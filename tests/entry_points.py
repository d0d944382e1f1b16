"""Every entry point of one problem against the oracle, shared by the modules that test a kernel configuration each
(tests/test_gpu_orders.py, tests/test_gpu_dispatch.py).

The kernels are FP64 and differ from the oracle only in summation order, so the bounds are tight on purpose: 1e-12 on
evaluate and the Jacobian products, 1e-9..1e-11 on the Schur pieces, identical CG counts under the eta stop.
"""
import re

import numpy as np


def relerr(a, b):
    a = np.asarray(a, dtype=float)
    b = np.asarray(b, dtype=float)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def parse_plan(text):
    """Fields of the `[b200ba] C=...` line b200_create prints under B200_VERBOSE (the kernel configuration it chose)."""
    lines = [ln for ln in text.splitlines() if ln.startswith("[b200ba] C=")]
    assert len(lines) == 1, text
    line = lines[0][len("[b200ba] "):]
    m = re.search(r"v2\(w=(\d+),s=(\d+),r=(\d+)\) mul\((\S+) w=(\d+),s=(\d+),r=(\d+),smem=(\d+)\)", line)
    assert m, line
    plan = dict(v2_w=int(m.group(1)), v2_s=int(m.group(2)), v2_r=int(m.group(3)), mul=m.group(4), mul_w=int(m.group(5)),
                mul_s=int(m.group(6)), mul_r=int(m.group(7)), mul_smem=int(m.group(8)))
    for key, value in re.findall(r"(\w+)(?:\(\+slices\))?=(\w+)", line[:m.start()] + line[m.end():]):
        plan[key] = int(value) if value.isdigit() else value
    return plan


class Case:
    """One BAL problem set up identically for the oracle and for the GPU library, with the trivial loss
    (loss_type = LOSS_TRIVIAL) or Huber(loss_a) (LOSS_HUBER)."""

    def __init__(self, cs, oracle, bal, loss_type=0, loss_a=1.0):
        from ceres_solver_b200 import bal as B
        self.rp = B.ReducedProgram(bal)
        self.orc = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel(),
                                    use_huber=loss_type == cs.LOSS_HUBER, huber_a=loss_a)
        self.gpu = cs.Problem(self.rp.C, self.rp.P, self.rp.row_cam, self.rp.row_pt, self.rp.row_obs, loss_type=loss_type,
                              loss_a=loss_a)
        self.state = self.rp.state(bal)

    def close(self):
        self.gpu.close()


def _inv_blocks(flat):
    return np.linalg.inv(flat.reshape(-1, 9, 9)).ravel()


def check_every_entry_point(case, oracle, shared_inputs=False):
    """shared_inputs: once evaluate has been checked, the oracle's Jacobian and residuals are replaced by the GPU's, so
    that every product and solve after it is compared on identical inputs.  A robust loss needs that: the weight
    sqrt(a / |r|) of an outlier row carries the relative rounding error of its residual, a small difference of two large
    numbers, into every entry of its Jacobian row (~1e-12 relative, measured on the fixtures of test_gpu_dispatch.py),
    three orders of magnitude above what the products below are held to."""
    gpu, orc = case.gpu, case.orc
    ok, cost, res, grad = gpu.evaluate(case.state)
    ok_o, cost_o, res_o, grad_o = orc.evaluate(case.state, nt=8)
    assert ok and ok_o and abs(cost - cost_o) <= 1e-12 * cost_o
    assert relerr(res, res_o) < 1e-12 and relerr(grad, grad_o) < 1e-10
    J = orc.jacobian()
    v = gpu.jacobian_values()
    assert relerr(v, J.values()) < 1e-12
    if shared_inputs:
        J.set_values(v)
        res_o = res
    # cost-only evaluation: same cost, Jacobian untouched
    ok, cost2, _, _ = gpu.evaluate(case.state, want_residuals=False, want_gradient=False, want_jacobian=False)
    assert ok and abs(cost2 - cost_o) <= 1e-12 * cost_o
    assert np.array_equal(gpu.jacobian_values(), v)
    rng = np.random.RandomState(3)
    x = rng.randn(gpu.num_parameters)
    y = rng.randn(gpu.num_residuals)
    assert relerr(gpu.squared_column_norm(), J.squared_column_norm()) < 1e-12
    assert relerr(gpu.right_multiply(x), J.right_multiply(x)) < 1e-12
    assert relerr(gpu.left_multiply(y), J.left_multiply(y)) < 1e-11
    # PartitionedMatrixView single products (E x, F x, E'y, F'y), accumulate semantics
    xe, xf = rng.randn(3 * gpu.P), rng.randn(9 * gpu.C)
    y0 = rng.randn(gpu.num_residuals)
    nr = gpu.num_residuals
    assert relerr(gpu.partitioned_multiply(0, xe, y0), y0 + J.pmv(gpu.P, 0, xe, nr, nt=8)) < 1e-12
    assert relerr(gpu.partitioned_multiply(1, xf, y0), y0 + J.pmv(gpu.P, 1, xf, nr, nt=8)) < 1e-12
    assert relerr(gpu.partitioned_multiply(2, y, xe), xe + J.pmv(gpu.P, 2, y, 3 * gpu.P, nt=8)) < 1e-12
    assert relerr(gpu.partitioned_multiply(3, y, xf), xf + J.pmv(gpu.P, 3, y, 9 * gpu.C, nt=8)) < 1e-11
    # set_values round trip (in the caller's layout)
    gpu.set_jacobian_values(2.0 * v)
    assert relerr(gpu.right_multiply(x), 2.0 * J.right_multiply(x)) < 1e-12
    gpu.set_jacobian_values(v)
    s = 1.0 / (1.0 + np.sqrt(J.squared_column_norm()))
    gpu.scale_columns(s)
    J.scale_columns(s, nt=8)
    assert relerr(gpu.jacobian_values(), J.values()) < 1e-14
    D = np.sqrt(np.clip(J.squared_column_norm(), 1e-6, 1e32) / 1e4)
    expect = J.left_multiply(J.right_multiply(x, nt=8), nt=8) + D * D * x
    assert relerr(gpu.jtj_multiply(x, D), expect) < 1e-11
    assert relerr(gpu.jtj_multiply(x, None), J.left_multiply(J.right_multiply(x, nt=8), nt=8)) < 1e-11
    isc = oracle.ImplicitSchur(J, gpu.P, want_ftf=False, nt=8)
    isc.init(D, res_o)
    gpu.schur_init(res, D)
    assert relerr(gpu.schur_rhs(), isc.rhs()) < 1e-9
    assert relerr(gpu.schur_ete_inverse(), isc.ete_inverse()) < 1e-9
    for _ in range(2):
        u = rng.randn(9 * gpu.C)
        assert relerr(gpu.schur_multiply(u), isc.right_multiply(u)) < 1e-9
    assert relerr(gpu.schur_back_substitute(u), isc.back_substitute(u)) < 1e-9
    C, P = gpu.C, gpu.P
    # SCHUR_JACOBI: the diagonal blocks of S and their inverses
    diag, _ = J.schur_eliminate(P, None, D, diagonal_only=True, diag_len=81 * C, nt=8, n_f=9 * C)
    blocks, inv = gpu.schur_jacobi_update()
    assert relerr(blocks, diag) < 1e-9
    assert relerr(inv, _inv_blocks(diag)) < 1e-7
    # JACOBI: (F'F + D_f^2)^-1
    ftf = J.block_diagonal(P, 1, nt=8).reshape(C, 9, 9) + np.einsum("ci,ij->cij", D[3 * P:].reshape(C, 9) ** 2, np.eye(9))
    assert relerr(gpu.block_jacobi_update(), _inv_blocks(ftf)) < 1e-7
    step = rng.randn(gpu.num_parameters) * 1e-3
    Js = J.right_multiply(step, nt=8)
    assert abs(gpu.model_cost_change(step) - (-Js @ (res_o + 0.5 * Js))) <= 1e-9 * abs(Js @ res_o)
    # linear solves under the eta stop, with each preconditioner the PCG supports.  Unpreconditioned, eta = 1e-3 takes
    # 100+ iterations on the larger problems, where last-bit differences grow past the 1e-7 bound on the solution
    # (tests/conftest.py compare_lm_traces); eta = 0.1 stops it after 4..21.
    for precond, eta in ((0, 1e-1), (1, 1e-3), (2, 1e-3)):
        o = gpu.solver_options(preconditioner_type=precond, q_tolerance=eta, r_tolerance=-1.0)
        xs, its, term = gpu.schur_solve(res, D, o)
        xo, its_o, term_o = J.linear_solve(P, res_o, D, solver=0, preconditioner=precond, q_tolerance=eta,
                                           r_tolerance=-1.0, nt=8)
        assert (precond, its, term) == (precond, its_o, term_o)
        assert relerr(xs, xo) < 1e-7, precond
    if 9 * C <= 4000:   # the explicit reduced system is dense: small camera counts only
        xd, _, td = gpu.dense_schur_solve(res, D)
        xdo, _, tdo = J.linear_solve(P, res_o, D, solver=1, nt=8)
        assert td == tdo and relerr(xd, xdo) < 1e-7
    # SCHUR_JACOBI after a write of J that no new initialisation followed: every configuration forms the blocks from the
    # current J and the initialisation's P = (E'E + D_e^2)^-1, F'F + D_f^2 - sum_k W_kc' P_k W_kc with W_kc the sum of
    # E_r'F_r over the rows of point k and camera c
    gpu.schur_init(res, D)
    Pk = gpu.schur_ete_inverse().reshape(P, 3, 3)
    gpu.scale_columns(rng.uniform(0.5, 2.0, gpu.num_parameters))
    v = gpu.jacobian_values()
    N = gpu.N
    E, F = v[:6 * N].reshape(N, 2, 3), v[6 * N:].reshape(N, 2, 9)
    cam, pt = np.asarray(case.rp.row_cam), np.asarray(case.rp.row_pt)
    expect = np.einsum("ci,ij->cij", D[3 * P:].reshape(C, 9) ** 2, np.eye(9))
    np.add.at(expect, cam, np.einsum("nri,nrj->nij", F, F))
    pairs, pair_of_row = np.unique(pt.astype(np.int64) * C + cam, return_inverse=True)
    W = np.zeros((pairs.size, 3, 9))
    np.add.at(W, pair_of_row.ravel(), np.einsum("nri,nrj->nij", E, F))
    np.subtract.at(expect, pairs % C, np.einsum("kij,kil,klm->kjm", W, Pk[pairs // C], W))
    blocks, _ = gpu.schur_jacobi_update()
    assert relerr(blocks, expect.ravel()) < 1e-9


def oracle_lm_traces(case, iterations, max_cg=None, threads=(8, 3)):
    """The oracle's LM run with several thread counts: the spread between them is what a change of summation order does
    to the inexact trajectory (tests/test_gpu_headline.py explains), i.e. the resolution of the comparison.  max_cg caps
    the CG iterations of every solve (None: the default of 500)."""
    out = []
    for nt in threads:
        o = case.orc.default_options()
        o.num_threads = nt
        o.max_num_iterations = iterations
        if max_cg is not None:
            o.max_linear_solver_iterations = max_cg
        _, recs_o, _ = case.orc.solve(case.state, o)
        out.append(recs_o)
    return out


def check_lm_trajectory(case, traces, iterations, host_boundary, max_cg=None):
    """`iterations` LM iterations on the GPU, device-resident or through the host-buffer boundary, against the oracle's
    traces (oracle_lm_traces with the same iterations and max_cg)."""
    from tests.conftest import compare_lm_traces
    o = case.gpu.lm_options(max_num_iterations=iterations)
    if max_cg is not None:
        o.linear_solver.max_num_iterations = max_cg
    _, recs = case.gpu.lm_solve(case.state, o, host_boundary=host_boundary)
    compare_lm_traces(recs, *traces, keys=("cost", "step_norm"))


INT_FIELDS = ("iteration", "ls_iterations", "step_is_valid", "step_is_successful")
RELATIVE_FIELDS = ("cost", "gradient_max_norm", "gradient_norm", "step_norm", "tr_radius", "model_cost_change")


def compare_lm_traces_exact(recs, recs_o):
    """Every field of every record of a short solve against the oracle's (the same options on both sides).  While every
    linear solve is short, the two trajectories differ only by summation order, ~1e-10 relative, so this holds them to
    1e-9: the iteration and CG counts and the valid / accepted decisions equal; cost, gradient norms, step norm, radius
    and model cost change to 1e-9 relative; the cost change to 1e-9 of the cost (it is a difference of two costs); the
    step quality rho to 1e-6 max(1, |rho|) (a quotient of two differences).  A zero on the oracle's side (the step norm
    before the first accepted step, an invalid step's model cost change) must be an exact zero on the GPU's.

    The gradient norms also get 1e-12 of the initial record's: the gradient J'r is a sum whose terms do not shrink as the
    solve converges, so its rounding error stays at the scale of the initial gradient while the gradient itself drops by
    orders of magnitude (measured on `tiny`: record 2's max norm, 1e4 below the initial one, moves by up to 1.6e-9
    relative between GPU and oracle and by 4e-10 between two oracle runs with the same thread count)."""
    assert len(recs) == len(recs_o), ([r["iteration"] for r in recs], [int(r["iteration"]) for r in recs_o])
    for a, b in zip(recs, recs_o):
        for key in INT_FIELDS:
            assert int(a[key]) == int(b[key]), (key, a, b)
        for key in RELATIVE_FIELDS:
            floor = 1e-12 * abs(recs_o[0][key]) if key in ("gradient_max_norm", "gradient_norm") else 0.0
            assert abs(a[key] - b[key]) <= 1e-9 * abs(b[key]) + floor, (key, a, b)
        assert abs(a["cost_change"] - b["cost_change"]) <= 1e-9 * abs(b["cost"]), ("cost_change", a, b)
        assert abs(a["tr_ratio"] - b["tr_ratio"]) <= 1e-6 * max(1.0, abs(b["tr_ratio"])), ("tr_ratio", a, b)
