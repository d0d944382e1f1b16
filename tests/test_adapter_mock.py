"""adapter/b200_adapter.{h,cc} -- the Ceres-side classes of the drop-in -- cannot be compiled against Ceres here (every
Ceres header includes Eigen, which this image does not have).  tests/mock_ceres restates the handful of Ceres-internal
interfaces the adapter is written against; here the adapter is COMPILED (-Wall -Wextra -Werror) and LINKED against it and
libb200ba.so, its host-side logic (problem recognition, refusal messages, Huber scale recovery, the factory predicate) is
run on the CPU, and every restated signature is checked against the digests of the ceres-solver headers it was
found in (tests/golden/ceres_reference_digests.json).  The `-m gpu` part runs the driver's `solve` case on the device -- Create -> Evaluate -> Solve through the adapter
classes -- and compares it with the oracle."""
import hashlib
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    import ceres_solver_b200 as cs
    cs.lib()
    tmp = tmp_path_factory.mktemp("adapter")
    (tmp / "ceres").mkdir()
    shutil.copy(os.path.join(ROOT, "adapter", "b200_adapter.h"), tmp / "ceres" / "b200_adapter.h")   # Ceres' include path
    exe = str(tmp / "adapter_mock_driver")
    libdir = os.path.join(ROOT, "ceres_solver_b200")
    cmd = ["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-Werror", "-I", str(tmp), "-I", os.path.join(ROOT, "tests", "mock_ceres"),
           "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "adapter", "b200_adapter.cc"),
           os.path.join(ROOT, "tests", "adapter_mock_driver.cc"), "-o", exe, "-L", libdir, "-l:libb200ba.so", "-Wl,-rpath," + libdir]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


def run(exe, *args, timeout=300):
    return subprocess.run([exe, *args], capture_output=True, text=True, timeout=timeout)


def test_factory_predicate(driver):
    # ITERATIVE_SCHUR + CUDA_SPARSE only: SPARSE_SCHUR + CUDA_SPARSE (the reference's cuDSS configuration), other
    # libraries and CGNR + CUDA_SPARSE (the reference's own CUDA path) are left alone
    assert run(driver, "predicate").stdout.split() == ["1", "0", "0", "0"]


@pytest.mark.parametrize("a", ["0.5", "1", "0.1", "30000", "1e-9", "1e14"])
def test_huber_scale_is_recovered_exactly(driver, a):
    assert float(run(driver, "huber", a).stdout) == float(a)


def test_huber_scale_beyond_the_probe_is_refused(driver):
    assert run(driver, "huber", "1e31").stdout.strip() == "inf"


@pytest.mark.parametrize("case,needle", [
    ("bad_order", "points must form the first elimination group"),
    ("other_functor", "residual block 4 is not SnavelyReprojectionError<2,9,3>"),
    ("manifold", "residual block 0 is not SnavelyReprojectionError<2,9,3> on Euclidean"),
    ("cauchy", "only the trivial and Huber losses"),
    ("mixed_loss", "different loss functions (block 2)"),
    ("mixed_huber", "different loss functions (block 5)"),
    ("callback", "evaluation callbacks"),
])
def test_unsupported_programs_are_refused_with_a_message(driver, case, needle):
    """Evaluator::Create's contract (evaluator.cc:95-97): nullptr + *error, decided before the device is touched --
    never a silent CPU path, never a wrong loss."""
    r = run(driver, case)
    assert r.returncode == 4 and r.stdout.startswith("refused: B200Evaluator:") and needle in r.stdout, (r.stdout, r.stderr)


def _write_problem(path, rp, state):
    with open(path, "wb") as f:
        f.write(np.int32(rp.C).tobytes())
        f.write(np.int32(rp.P).tobytes())
        f.write(np.int64(rp.N).tobytes())
        f.write(np.ascontiguousarray(rp.row_cam, dtype=np.int32).tobytes())
        f.write(np.ascontiguousarray(rp.row_pt, dtype=np.int32).tobytes())
        f.write(np.ascontiguousarray(rp.row_obs, dtype=np.float64).tobytes())
        f.write(np.ascontiguousarray(state, dtype=np.float64).tobytes())


def _have_gpu():
    import torch
    return torch.cuda.is_available()


def test_valid_program_reaches_the_library_and_fails_loudly_without_a_gpu(driver, tmp_path):
    if _have_gpu():
        pytest.skip("a GPU is present: test_adapter_classes_match_oracle runs the case")
    from ceres_solver_b200 import bal as B
    bal = B.synthetic("tiny")
    rp = B.ReducedProgram(bal)
    _write_problem(tmp_path / "p.bin", rp, rp.state(bal))
    r = run(driver, "solve", str(tmp_path / "p.bin"))
    assert r.returncode == 3 and "no CPU fallback" in r.stderr, (r.stdout, r.stderr)


@pytest.mark.gpu
@pytest.mark.parametrize("huber", [False, True])
def test_adapter_classes_match_oracle(driver, tmp_path, oracle, huber):
    """Create -> CreateJacobian -> Evaluate (with and without apply_loss_function) -> SquaredColumnNorm ->
    B200IterativeSchurSolver::Solve -> RightMultiplyAndAccumulate -> ModelCostChange -> Plus through the adapter classes,
    against the oracle."""
    from ceres_solver_b200 import bal as B
    bal = B.synthetic_bal(64, 4000, 18000, seed=3)
    rp = B.ReducedProgram(bal)
    state = rp.state(bal)
    _write_problem(tmp_path / "p.bin", rp, state)
    r = run(driver, "solve", str(tmp_path / "p.bin"), *(["huber"] if huber else []))
    assert r.returncode == 0 and r.stdout.strip().endswith("done"), (r.stdout, r.stderr)
    out = {}
    for line in r.stdout.splitlines():
        w = line.split()
        out[w[0]] = w[1:]
    np_, nr = 3 * rp.P + 9 * rp.C, 2 * rp.N
    assert [int(v) for v in out["sizes"]] == [np_, np_, nr]
    assert [int(v) for v in out["jacobian"]] == [nr, np_, 24 * rp.N]
    orc = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel(), use_huber=huber, huber_a=1.0)
    ok, cost_o, res_o, grad_o = orc.evaluate(state, nt=8)
    assert abs(float(out["cost"][0]) - cost_o) <= 1e-12 * cost_o
    assert abs(float(out["gradient_max_norm"][0]) - np.abs(grad_o).max()) <= 1e-10 * np.abs(grad_o).max()
    if huber:
        plain = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())
        assert abs(float(out["raw_cost"][0]) - plain.evaluate(state, nt=8)[1]) <= 1e-12 * cost_o
    J = orc.jacobian()
    sq = J.squared_column_norm()
    assert abs(float(out["column_norm_sum"][0]) - sq.sum()) <= 1e-11 * sq.sum()
    D = np.sqrt(np.clip(sq, 1e-6, 1e32) / 1e4)
    xo, its_o, term_o = J.linear_solve(rp.P, res_o, D, solver=0, q_tolerance=1e-2, r_tolerance=-1.0, nt=8)
    assert (int(out["solve"][1]), int(out["solve"][3])) == (its_o, term_o)
    assert abs(float(out["solve"][5]) - np.linalg.norm(xo)) <= 1e-7 * np.linalg.norm(xo)
    Jx = J.right_multiply(xo, nt=8)
    assert abs(float(out["jx_norm"][0]) - np.linalg.norm(Jx)) <= 1e-7 * np.linalg.norm(Jx)
    mcc = float(np.dot(Jx, res_o - 0.5 * Jx))   # -(J s)'(r + J s / 2) for s = -x
    assert abs(float(out["model_cost_change"][0]) - mcc) <= 1e-6 * abs(mcc)
    assert float(out["plus_error"][0]) <= 1e-13 * np.linalg.norm(state)   # Plus on Euclidean blocks: x + delta up to rounding
    assert int(out["evaluator_calls"][0]) == (3 if huber else 1)


# ---------------------------------------------------------------------------------------------------------------------
# the mock against the ceres-solver headers

def _norm(text):
    text = re.sub(r"//[^\n]*", " ", text)
    text = re.sub(r"\b(CERES_NO_EXPORT|CERES_EXPORT|final|override)\b", " ", text)
    return re.sub(r"\s+", "", text)


SIGNATURES = {
    "internal/ceres/evaluator.h": [
        "virtual std::unique_ptr<SparseMatrix> CreateJacobian() const = 0;",
        "virtual bool Evaluate(const EvaluateOptions& evaluate_options, const double* state, double* cost, double* residuals, double* gradient, SparseMatrix* jacobian) = 0;",
        "virtual bool Plus(const double* state, const double* delta, double* state_plus_delta) const = 0;",
        "virtual int NumParameters() const = 0;", "virtual int NumEffectiveParameters() const = 0;", "virtual int NumResiduals() const = 0;",
        "virtual std::map<std::string, CallStatistics> Statistics() const {",
        "int num_eliminate_blocks = -1;", "EvaluationCallback* evaluation_callback = nullptr;",
        "bool apply_loss_function = true;", "bool new_evaluation_point = true;",
        "static std::unique_ptr<Evaluator> Create(const Options& options, Program* program, std::string* error);",
    ],
    "internal/ceres/block_sparse_matrix.h": [
        "class BlockSparseMatrix : public SparseMatrix {",
        "explicit BlockSparseMatrix(CompressedRowBlockStructure* block_structure, bool use_page_locked_memory = false);",
        "void SetZero() ;", "void SetZero(ContextImpl* context, int num_threads) ;",
        "void RightMultiplyAndAccumulate(const double* x, double* y) const ;",
        "void RightMultiplyAndAccumulate(const double* x, double* y, ContextImpl* context, int num_threads) const ;",
        "void LeftMultiplyAndAccumulate(const double* x, double* y) const ;",
        "void LeftMultiplyAndAccumulate(const double* x, double* y, ContextImpl* context, int num_threads) const ;",
        "void SquaredColumnNorm(double* x) const ;", "void SquaredColumnNorm(double* x, ContextImpl* context, int num_threads) const ;",
        "void ScaleColumns(const double* scale) ;", "void ScaleColumns(const double* scale, ContextImpl* context, int num_threads) ;",
        "double* mutable_values() { return values_; }", "const CompressedRowBlockStructure* block_structure() const;",
    ],
    "internal/ceres/sparse_matrix.h": [
        "virtual void SquaredColumnNorm(double* x) const = 0;", "virtual void ScaleColumns(const double* scale) = 0;", "virtual void SetZero() = 0;",
        "virtual void SquaredColumnNorm(double* x, ContextImpl* context, int num_threads) const;",
        "virtual void ScaleColumns(const double* scale, ContextImpl* context, int num_threads);",
    ],
    "internal/ceres/linear_operator.h": [
        "virtual void RightMultiplyAndAccumulate(const double* x, double* y) const = 0;",
        "virtual void RightMultiplyAndAccumulate(const double* x, double* y, ContextImpl* context, int num_threads) const;",
        "virtual void LeftMultiplyAndAccumulate(const double* x, double* y) const = 0;",
    ],
    "internal/ceres/linear_solver.h": [
        "enum class LinearSolverTerminationType {", "PreconditionerType preconditioner_type = JACOBI;", "int min_num_iterations = 1;",
        "int max_num_iterations = 1;", "int max_num_spse_iterations = 5;", "bool use_spse_initialization = false;", "double spse_tolerance = 0.1;",
        "int residual_reset_period = 10;", "double* D = nullptr;", "double r_tolerance = 0.0;", "double q_tolerance = 0.0;",
        "double residual_norm = -1.0;", "int num_iterations = -1;", "std::string message;",
        "virtual LinearSolver::Summary SolveImpl(MatrixType* A, const double* b, const LinearSolver::PerSolveOptions& per_solve_options, double* x) = 0;",
        "using BlockSparseMatrixSolver = TypedLinearSolver<BlockSparseMatrix>;",
    ],
    "internal/ceres/program.h": ["const std::vector<ResidualBlock*>& residual_blocks() const;", "int NumParameterBlocks() const;",
                                 "int NumParameters() const;", "int NumEffectiveParameters() const;", "int NumResiduals() const;"],
    "internal/ceres/residual_block.h": ["const CostFunction* cost_function() const {", "const LossFunction* loss_function() const {",
                                        "ParameterBlock* const* parameter_blocks() const {", "int NumParameterBlocks() const {"],
    "internal/ceres/parameter_block.h": ["int Size() const {", "const Manifold* manifold() const {", "int index() const {"],
    "internal/ceres/execution_summary.h": ["const std::map<std::string, CallStatistics>& statistics() const {",
                                           "ScopedExecutionTimer(std::string name, ExecutionSummary* summary)"],
    "internal/ceres/block_jacobian_writer.h": ["BlockJacobianWriter(const Evaluator::Options& options, Program* program);",
                                               "std::unique_ptr<SparseMatrix> CreateJacobian() const;"],
    "internal/ceres/block_structure.h": ["struct CompressedRowBlockStructure { std::vector<Block> cols; std::vector<CompressedRow> rows; };"],
    "include/ceres/loss_function.h": ["virtual void Evaluate(double sq_norm, double out[3]) const = 0;", "class HuberLoss : public LossFunction {",
                                      "explicit HuberLoss(double a)"],
    "include/ceres/autodiff_cost_function.h": ["const CostFunctor& functor() const { return *functor_; }"],
    "examples/snavely_reprojection_error.h": ["struct SnavelyReprojectionError {", "double observed_x;", "double observed_y;"],
}


@pytest.mark.parametrize("rel", sorted(SIGNATURES))
def test_mock_signatures_exist_in_the_reference(rel):
    """Every declaration the mock restates (and the adapter relies on) is present, token for token, in the ceres-solver
    header it cites -- `final` / `override` / export macros aside (the patch removes the `final`s, test_adapter_patch.py).
    tools/make_reference_digests.py looked each one up in the ceres-solver tree and stored the SHA-256 of the normalised
    declarations it found; a declaration added or changed here has to be looked up again the same way."""
    with open(os.path.join(ROOT, "tests", "golden", "ceres_reference_digests.json")) as f:
        found = set(json.load(f)["signatures"][rel])
    for sig in SIGNATURES[rel]:
        assert hashlib.sha256(_norm(sig).encode()).hexdigest() in found, (rel, sig)


@pytest.mark.parametrize("rel", sorted(SIGNATURES))
def test_mock_declares_what_the_list_says(rel):
    """...and the same declarations are in the mock (so the list above cannot drift from what was compiled)."""
    text = _norm(open(os.path.join(ROOT, "tests", "mock_ceres", "ceres", "mock_all.h")).read())
    for sig in SIGNATURES[rel]:
        if sig.startswith("static std::unique_ptr<Evaluator> Create("):
            continue   # the factory is Ceres' own (evaluator.cc); the adapter only mirrors its signature
        head = _norm(sig.rstrip(";").split("{")[0])   # declared in the reference, often DEFINED inline in the mock
        assert head in text, (rel, sig)
