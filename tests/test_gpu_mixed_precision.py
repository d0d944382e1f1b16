"""Mixed-precision exact solves and iterative refinement (b200_set_exact_solve_options; use_mixed_precision_solves and
max_num_refinement_iterations of b200_lm_options) on DENSE_SCHUR and SPARSE_SCHUR, against the extended-precision measures
of tests/test_gpu_sparse_factor.py (backward error eta of the reduced system, forward error against a refined longdouble
solution), on the camera graphs of tests/test_sparse_schur_plan.py that reach every supernode shape and schedule.

A float factorisation with k = 0 is held to eta <= C32 2^-24.  C32 is fixed from runs of every case of test_structure
(geometric and random values, radius 1e4, 1e-1 and D = NULL) on an H100 80GB HBM3 at a 700 W power limit: the largest
observed eta / 2^-24 at k = 0 was 1.50 (clique16, random values, radius 1e-1; 3e-9 .. 1.3 elsewhere), so C32 = 16 sits an
order of magnitude above it.  eta / 2^-24 for k = 0 .. 3 is printed per case (pytest -s).  With refinement, eta never
grows from k to k + 1 until it reaches the FP64 floor C_ETA 2^-53, and where kappa 2^-24 < 1/2 (kappa the scaled condition number of test_gpu_sparse_factor.py, computed per case) enough refinement
steps bring the camera block within the FP64 forward-error bound C_X kappa 2^-53.

A value-only change aimed at the solve-only pass: dropping the last descendant term of step 3 in sp_forward (q < u1 - 1
in the loop that subtracts L_d y_d).  It would leave each refinement's correction wrong by that term on every structure
with updates, which test_structure's monotonicity and refined forward-error checks are built to see.  That mutation has
not yet been run against this module.
"""
import ctypes
import math

import numpy as np
import pytest

from tests import lm_cases as L
from tests.entry_points import Case, compare_lm_traces_exact
from tests.test_gpu_sparse_factor import (C_ETA, C_X, RADII, U, Structure, check_solution, load, lm_diagonal,
                                          reference_for)
from tests.test_sparse_schur_plan import STRUCTURES

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
C32 = 16.0


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


def solve(gpu, solver, b, D, mixed, k):
    gpu.set_exact_solve_options(mixed, k)
    f = gpu.sparse_schur_solve if solver == "sparse" else gpu.dense_schur_solve
    x, its, term = f(b, D)
    assert its == 1
    return x, term


def refinement_steps(kappa):
    """Steps after which a contraction by kappa 2^-24 per step has taken an error of one down by 2^-53, plus two."""
    rho = kappa * U32
    return min(60, int(math.ceil(53.0 * math.log(2.0) / -math.log(rho))) + 2)


def check_mixed(gpu, s, b, D, solver, tag, report):
    ref, kappa, x_ref = reference_for(gpu, s, b, D)
    n_e = 3 * s.P
    etas = []
    for k in range(4):
        x, term = solve(gpu, solver, b, D, True, k)
        assert term == 0, (tag, k)
        etas.append(ref.eta(x[n_e:]))
    report.append("%-36s eta/2^-24 k=0..3: %s  kappa 2^-24 %.1e" % (tag, " ".join("%.2e" % (e / U32) for e in etas),
                                                                     kappa * U32))
    assert etas[0] <= C32 * U32, (tag, etas)
    for a, c in zip(etas, etas[1:]):
        assert c <= a or c <= C_ETA * U, (tag, etas)
    if kappa * U32 < 0.5:
        x, term = solve(gpu, solver, b, D, True, refinement_steps(kappa))
        assert term == 0
        check_solution(x, ref, kappa, x_ref, tag=tag + "/refined")
    # FP64 with refinement stays within the FP64 bounds
    x, term = solve(gpu, solver, b, D, False, 2)
    assert term == 0
    check_solution(x, ref, kappa, x_ref, tag=tag + "/fp64 k=2")
    gpu.set_exact_solve_options(False, 0)
    return ref, kappa


@pytest.mark.parametrize("name", STRUCTURES)
def test_structure(name, cs):
    s = Structure(cs, name)
    report = []
    for kind in ("geometric", "random"):
        gpu = s.problem(cs)
        b = load(gpu, s, kind)
        for radius in RADII:
            if radius is None and kind == "geometric":
                continue
            D = lm_diagonal(gpu, radius)
            tag = "%s/%s/%s" % (name, kind, radius)
            ref, kappa = check_mixed(gpu, s, b, D, "sparse", tag, report)
            if 9 * s.C <= 4000:
                check_mixed(gpu, s, b, D, "dense", tag + "/dense", report)
                # the two float factorisations agree after three refinements as far as the refinement has converged
                xs, _ = solve(gpu, "sparse", b, D, True, 3)
                xd, _ = solve(gpu, "dense", b, D, True, 3)
                gpu.set_exact_solve_options(False, 0)
                bound = max(2 * C_X * kappa * U, 2 * (kappa * U32) ** 4)
                assert ref.scaled_err(xs[3 * s.P:], xd[3 * s.P:]) <= bound, tag
        gpu.close()
    print("\n" + "\n".join(report))


def test_launch_counts(cs):
    """A sparse solve launches the factorisation once and the solve-only pass k times, with k S x products and 2 k
    conversion passes; mixed with k = 0 launches exactly the kernels the FP64 solve does.  The dense solve: one assembly,
    k products and 2 k conversion passes, with mixed precision 3 more (the matrix, the rhs and the widening)."""
    s = Structure(cs, "cliques")
    gpu = s.problem(cs)
    b = load(gpu, s, "random")
    D = lm_diagonal(gpu, 1e4)
    gpu.sparse_schur_solve(b, D)   # the analysis
    launched = {}
    for mixed in (False, True):
        for k in (0, 1, 3):
            gpu.stats_reset()
            solve(gpu, "sparse", b, D, mixed, k)
            st = {n: v["launches"] for n, v in gpu.stats().items() if v["launches"] > 0}
            launched[(mixed, k)] = st
            assert st["sparse_factor"] == 1 and st.get("sparse_solve", 0) == k
            assert gpu.stats()["schur_multiply"]["operations"] == k
            assert st.get("refine_convert", 0) == 2 * k
    assert launched[(True, 0)] == launched[(False, 0)]
    for mixed in (False, True):
        for k in (0, 2):
            gpu.stats_reset()
            solve(gpu, "dense", b, D, mixed, k)
            st = gpu.stats()
            assert st["schur_diag_blocks"]["launches"] == 1 and st["schur_multiply"]["operations"] == k
            assert st["refine_convert"]["launches"] == (3 + 2 * k if mixed else 2 * k), (mixed, k)
    gpu.close()


def raw_solve(cs, gpu, solver, b, D, sentinel=-7.25):
    from ceres_solver_b200 import binding as Bd
    x = np.full(gpu.num_parameters, sentinel)
    summ = Bd.SolverSummary()
    b = np.ascontiguousarray(b, dtype=float)
    f = cs.lib().b200_sparse_schur_solve if solver == "sparse" else cs.lib().b200_dense_schur_solve
    assert f(gpu.h, Bd._d(b), Bd._d(np.ascontiguousarray(D, dtype=float)), Bd._d(x), ctypes.byref(summ)) == 0
    return x, summ.termination_type


@pytest.mark.parametrize("solver", ["sparse", "dense"])
def test_failure_and_recovery(solver, cs):
    """The geometric Jacobian has bundle adjustment's gauge freedom: S is singular but for the damping, whose smallest
    eigenvalues are of the size of D_f^2.  Rounding S to float perturbs it by ~1e-7 of its norm, so between radius 1e6 and
    1e10 (D_f^2 = 1e-6 .. 1e-10 of the column norms; at 1e11 FP64 fails too) there is a radius where S + D_f^2 factors in
    FP64 and not in float.  Mixed: FAILURE with the caller's buffer untouched; the same handle then succeeds in mixed
    precision at radius 1e4 and matches a fresh handle's solve."""
    found = None
    for name in ("one", "two", "clique16", "band"):
        s = Structure(cs, name)
        gpu = s.problem(cs)
        b = load(gpu, s, "geometric")
        for radius in (1e6, 1e7, 1e8, 1e9, 1e10):
            D = lm_diagonal(gpu, radius)
            gpu.set_exact_solve_options(False, 0)
            _, term64 = raw_solve(cs, gpu, solver, b, D)
            gpu.set_exact_solve_options(True, 0)
            x, term32 = raw_solve(cs, gpu, solver, b, D)
            print(name, radius, "fp64", term64, "fp32", term32)
            if term64 == cs.LS_SUCCESS and term32 == cs.LS_FAILURE:
                found = (s, gpu, b)
                assert np.all(x == -7.25)
                break
        if found is not None:
            break
        gpu.close()
    assert found is not None
    s, gpu, b = found
    D = lm_diagonal(gpu, 1e4)
    gpu.set_exact_solve_options(True, 3)
    x, term = raw_solve(cs, gpu, solver, b, D)
    assert term == cs.LS_SUCCESS
    ref, kappa, x_ref = reference_for(gpu, s, b, D)
    assert ref.eta(x[3 * s.P:]) <= C32 * U32
    fresh = s.problem(cs)
    load(fresh, s, "geometric")
    fresh.set_exact_solve_options(True, 3)
    xf, term = raw_solve(cs, fresh, solver, b, D)
    assert term == cs.LS_SUCCESS
    assert ref.scaled_err(x[3 * s.P:], xf[3 * s.P:]) <= max(2 * C_X * kappa * U, 2 * (kappa * U32) ** 4)
    gpu.close()
    fresh.close()


def test_reuse(cs):
    """Two mixed solves at k = 0 on one handle: camera blocks bitwise equal (the float rounding of the FP64 right-hand side
    and S, the fixed-order factorisation); with k = 3 equal to 1e-15 relative (the FP64 products may sum with REDs)."""
    s = Structure(cs, "loop")
    gpu = s.problem(cs)
    b = load(gpu, s, "random")
    D = lm_diagonal(gpu, 1e4)
    n_e = 3 * s.P
    a, _ = solve(gpu, "sparse", b, D, True, 0)
    c, _ = solve(gpu, "sparse", b, D, True, 0)
    assert np.array_equal(a[n_e:], c[n_e:])
    a, _ = solve(gpu, "sparse", b, D, True, 3)
    c, _ = solve(gpu, "sparse", b, D, True, 3)
    assert np.linalg.norm(a - c) <= 1e-15 * np.linalg.norm(a)
    gpu.close()


def test_options(cs):
    """Defaults off; a flag other than 0 / 1 and k < 0 refused; mixed with ITERATIVE_SCHUR refused by b200_lm_solve (k is
    ignored there); the handle's options restored after b200_lm_solve, on success and on error."""
    case_bal = L.tiny_bal()
    from ceres_solver_b200 import bal as B
    from ceres_solver_b200 import binding as Bd
    rp = B.ReducedProgram(case_bal)
    gpu = cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs)
    state = rp.state(case_bal)
    o = gpu.lm_options()
    assert o.use_mixed_precision_solves == 0 and o.max_num_refinement_iterations == 0
    for args in ((2, 0), (-1, 0), (0, -1)):
        with pytest.raises(cs.B200Error) as e:
            gpu.set_exact_solve_options(*args)
        assert e.value.code == Bd.ERR_INVALID_ARGUMENT
    with pytest.raises(cs.B200Error) as e:
        gpu.lm_solve(state, gpu.lm_options(use_mixed_precision_solves=1))
    assert e.value.code == Bd.ERR_INVALID_ARGUMENT
    gpu.lm_solve(state, gpu.lm_options(max_num_iterations=2, max_num_refinement_iterations=3))   # ITERATIVE_SCHUR: k ignored
    ok, _, res, _ = gpu.evaluate(state)
    D = lm_diagonal(gpu, 1e4)
    gpu.set_exact_solve_options(False, 0)
    x0, _ = raw_solve(cs, gpu, "sparse", res, D)

    def launches():
        gpu.stats_reset()
        raw_solve(cs, gpu, "sparse", res, D)
        return gpu.stats()["sparse_solve"]["launches"]
    # success: the call's options are dropped afterwards
    gpu.set_exact_solve_options(False, 2)
    gpu.lm_solve(state, gpu.lm_options(max_num_iterations=2, linear_solver_type=cs.SPARSE_SCHUR,
                                       use_mixed_precision_solves=1, max_num_refinement_iterations=5))
    assert launches() == 2
    # errors: k < 0 in the options, mixed with ITERATIVE_SCHUR
    for kw in (dict(linear_solver_type=cs.SPARSE_SCHUR, max_num_refinement_iterations=-1),
               dict(use_mixed_precision_solves=1)):
        with pytest.raises(cs.B200Error):
            gpu.lm_solve(state, gpu.lm_options(**kw))
        assert launches() == 2
    gpu.close()


def _lm_cases(cs, oracle, c16):
    from ceres_solver_b200 import bal as B
    yield "c16", Case(cs, oracle, L.c16_bal(c16))
    yield "clusters", Case(cs, oracle, B.synthetic_clusters(150, 8000, 40000))


@pytest.mark.parametrize("host_boundary", [False, True])
def test_lm(host_boundary, cs, oracle, c16):
    """LM with mixed precision and 8 refinements against the oracle's FP64 DENSE_SCHUR trace (four iterations, as
    test_gpu_sparse_factor.py's many-supernode test), both exact solvers; with k = 0 the loop completes and its records are
    consistent: the cost only changes on accepted steps (a rejected step's record keeps the cost to rounding)."""
    for name, case in _lm_cases(cs, oracle, c16):
        _, recs_o, _ = L.oracle_solve(case.orc, case.state, linear_solver_type=L.DENSE_SCHUR, max_num_iterations=4)
        for solver in (cs.SPARSE_SCHUR, cs.DENSE_SCHUR):
            _, recs = L.gpu_solve(case.gpu, case.state, host_boundary, linear_solver_type=solver, max_num_iterations=4,
                                  use_mixed_precision_solves=1, max_num_refinement_iterations=8)
            compare_lm_traces_exact(recs, recs_o)
            _, recs = L.gpu_solve(case.gpu, case.state, host_boundary, linear_solver_type=solver, max_num_iterations=10,
                                  use_mixed_precision_solves=1)
            for a, c in zip(recs, recs[1:]):
                if not c["step_is_successful"]:
                    assert abs(c["cost"] - a["cost"]) <= 1e-12 * a["cost"], (name, c)
            print(name, solver, "k=0 cost after %d: %.9e (FP64 oracle after 4: %.9e)" % (len(recs) - 1, recs[-1]["cost"],
                                                                                      recs_o[-1]["cost"]))
        case.close()


@pytest.mark.parametrize("host_boundary", [False, True])
@pytest.mark.parametrize("dogleg_type", [0, 1])
def test_dogleg(dogleg_type, host_boundary, cs, oracle, c16):
    """DOGLEG's Gauss-Newton solves with mixed precision and 8 refinements.  The Gauss-Newton system is damped by mu = 1e-8
    only, and with bundle adjustment's gauge freedom its condition number times 2^-24 exceeds 1: refinement does not
    converge, and the trace leaves FP64's (measured on an H100: C16's cost after the first step 1.1e-3 relative from
    FP64's, and a later record's cost 4.4e6 against FP64's 3e5).  What holds is that the loop runs to the same number of
    records with every cost finite; the final costs are printed (pytest -s)."""
    for name, case in _lm_cases(cs, oracle, c16):
        for solver in (cs.SPARSE_SCHUR, cs.DENSE_SCHUR):
            kw = dict(linear_solver_type=solver, max_num_iterations=4, trust_region_strategy_type=cs.DOGLEG,
                      dogleg_type=dogleg_type)
            _, recs64 = L.gpu_solve(case.gpu, case.state, host_boundary, **kw)
            _, recs = L.gpu_solve(case.gpu, case.state, host_boundary, use_mixed_precision_solves=1,
                                  max_num_refinement_iterations=8, **kw)
            assert len(recs) == len(recs64)
            costs = [r["cost"] for r in recs]
            assert np.all(np.isfinite(costs)), costs
            print("dogleg %d %s solver %d: final cost %.9e, FP64 %.9e" % (dogleg_type, name, solver, costs[-1],
                                                                       recs64[-1]["cost"]))
        case.close()
