"""SPARSE_SCHUR (b200_sparse_schur_solve: csrc/sparse_plan.cuh, csrc/sparse_schur.cuh) against the oracle's DENSE_SCHUR and
against b200_dense_schur_solve: both are exact solves of the same damped reduced system.

  solve     C16, tiny, the huge-point problem and reduced-size sequence (explicit plan, duplicate rows), cluster and random
            shapes (implicit plans; internally re-ordered points; minimum degree taken on the random one)
  failure   S + D_f^2 singular: FAILURE as the dense solve, and the LM loop's invalid-step chain
  lm        the exact-step LM loop on C16, device-resident and through the host buffers
  pcg       on an explicit-plan handle, a sparse solve between two PCG solves leaves them as on a fresh handle
"""
import numpy as np
import pytest

from tests import lm_cases as L
from tests.entry_points import Case, compare_lm_traces_exact, relerr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


def _bal(name, c16):
    from ceres_solver_b200 import bal as B
    from tests.test_gpu_dispatch import _duplicate_row
    from tests.test_gpu_parity import huge_bal
    if name == "c16":
        return L.c16_bal(c16)
    if name == "huge":
        return huge_bal()
    if name == "sequence":   # large enough for the explicit S plan, with two duplicate (camera, point) rows
        return _duplicate_row(_duplicate_row(B.synthetic_sequence(300, 40000, 180000), 5), 77)
    if name == "clusters":
        return B.synthetic_clusters(150, 8000, 40000)
    if name == "random":
        return B.synthetic_bal(80, 4000, 20000)
    return B.synthetic(name)


# S plan b200_create prints, camera order of the sparse analysis (0 caller's, 1 minimum degree), internal point order
# re-ordered; the largest point's rows
EXPECT = {"c16": ("implicit", 0, None), "tiny": ("implicit", 0, True), "huge": ("implicit", 0, True),
          "sequence": ("explicit", 0, False), "clusters": ("implicit", 0, True), "random": ("implicit", 1, True)}


def _scaled_system(case, radius=1e4):
    """Jacobi-scaled J, residuals b and an LM diagonal D as an LM iteration with this trust region radius sees them."""
    ok, _, res, _ = case.gpu.evaluate(case.state)
    ok_o, _, _, _ = case.orc.evaluate(case.state, nt=8)
    assert ok and ok_o
    J = case.orc.jacobian()
    s = 1.0 / (1.0 + np.sqrt(J.squared_column_norm()))
    case.gpu.scale_columns(s)
    J.scale_columns(s, nt=8)
    D = np.sqrt(np.clip(J.squared_column_norm(), 1e-6, 1e32) / radius)
    return J, res, D


@pytest.mark.parametrize("which", list(EXPECT))
def test_solve(which, cs, oracle, c16, capfd):
    import os
    os.environ["B200_VERBOSE"] = "1"
    try:
        case = Case(cs, oracle, _bal(which, c16))
    finally:
        del os.environ["B200_VERBOSE"]
    err = capfd.readouterr().err
    plan, order, reordered = EXPECT[which]
    assert "[b200ba] S plan: %s," % plan in err, err
    perm, st = cs.plan_sparse_schur(case.rp.C, case.rp.P, case.rp.row_cam, case.rp.row_pt)
    assert st["order"] == order
    if reordered is not None:
        assert (cs.plan_point_order(case.rp.C, case.rp.P, case.rp.row_cam, case.rp.row_pt)[2] != 0) == reordered
    if which == "huge":
        assert np.bincount(case.rp.row_pt).max() > 128
    # the 300-camera sequence at radius 1e4 is conditioned so that the last-bit differences of the two assemblies move the
    # solution by ~3e-6 (observed); a smaller radius (a later LM iteration) keeps the comparison at the 1e-8 the others meet
    J, b, D = _scaled_system(case, 10.0 if which == "sequence" else 1e4)
    x_o, _, term_o = J.linear_solve(case.gpu.P, b, D, solver=1, nt=8)
    case.gpu.stats_reset()
    x, its, term = case.gpu.sparse_schur_solve(b, D)
    assert term == term_o == cs.LS_SUCCESS and its == 1
    assert relerr(x, x_o) < 1e-8
    stats = case.gpu.stats()
    assert stats["sparse_factor"]["launches"] == 1 and stats["sparse_scatter"]["operations"] == 1
    xd, _, termd = case.gpu.dense_schur_solve(b, D)
    assert termd == cs.LS_SUCCESS and relerr(x, xd) < 1e-9
    # the same answer from the device-resident residuals (the reduced right-hand side is summed with FP64 REDs, whose order
    # varies from run to run; the solve amplifies that last-bit noise by the condition number, as in the dense test)
    x2, its2, term2 = case.gpu.sparse_schur_solve(None, D)
    assert (its2, term2) == (1, cs.LS_SUCCESS) and relerr(x2, x) < 1e-9
    case.close()


def test_failure_and_invalid_steps(cs, oracle):
    """Zero focal length and no LM floor: S + D_f^2 is singular.  The sparse solve reports FAILURE and writes nothing, as the
    dense one; the LM loop then runs the invalid-step chain of the oracle's DENSE_SCHUR loop."""
    case = Case(cs, oracle, L.zero_focal_bal())
    ok, _, res, _ = case.gpu.evaluate(case.state)
    assert ok
    D = np.zeros(case.gpu.num_parameters)
    D[:3 * case.gpu.P] = 1.0
    _, its, term = case.gpu.sparse_schur_solve(res, D)
    _, itsd, termd = case.gpu.dense_schur_solve(res, D)
    assert (its, term) == (itsd, termd) == (1, cs.LS_FAILURE)
    for host_boundary in (False, True):
        state_o, recs_o, _ = L.oracle_solve(case.orc, case.state, **L.INVALID)
        state, recs = L.gpu_solve(case.gpu, case.state, host_boundary, **dict(L.INVALID, linear_solver_type=cs.SPARSE_SCHUR))
        compare_lm_traces_exact(recs, recs_o)
        assert np.array_equal(state, case.state)
        assert all(r["step_is_valid"] == 0 for r in recs[1:]) and len(recs) > 1
    case.close()


@pytest.mark.parametrize("host_boundary", [False, True])
def test_lm_trajectory(host_boundary, cs, oracle, c16):
    """The exact-step LM loop with B200_SPARSE_SCHUR against the oracle's DENSE_SCHUR loop on C16 (the reference's
    published transcript; tests/test_gpu_parity.py runs the same comparison with B200_DENSE_SCHUR)."""
    from tests.test_gpu_parity import _compare_traces
    case = Case(cs, oracle, L.c16_bal(c16))
    o = case.orc.default_options()
    o.linear_solver = 1
    o.num_threads = 8
    state_o, recs_o, _ = case.orc.solve(case.state, o)
    lo = case.gpu.lm_options()
    lo.linear_solver_type = cs.SPARSE_SCHUR
    state, recs = case.gpu.lm_solve(case.state, lo, host_boundary=host_boundary)
    _compare_traces(recs, recs_o)
    assert relerr(state, state_o) < 1e-6
    case.close()


def test_pcg_around_sparse_solve(cs, oracle, c16, capfd):
    """On a handle with the explicit S plan: PCG, sparse solve, PCG give the PCG results of a fresh handle (the sparse path
    reassembles S for its own initialisation and leaves the flags of the explicit PCG consistent)."""
    import os
    bal = _bal("sequence", c16)
    os.environ["B200_VERBOSE"] = "1"
    try:
        a = Case(cs, oracle, bal)
        f = Case(cs, oracle, bal)
    finally:
        del os.environ["B200_VERBOSE"]
    assert capfd.readouterr().err.count("[b200ba] S plan: explicit,") == 2
    opts = a.gpu.solver_options(q_tolerance=1e-3, r_tolerance=-1.0)
    _, b, D = _scaled_system(a)
    _scaled_system(f)
    x_f, its_f, term_f = f.gpu.schur_solve(b, D, opts)
    x1, its1, term1 = a.gpu.schur_solve(b, D, opts)
    xs, _, ts = a.gpu.sparse_schur_solve(b, 2.0 * D)
    assert ts == cs.LS_SUCCESS
    x2, its2, term2 = a.gpu.schur_solve(b, D, opts)
    assert (its1, term1) == (its2, term2) == (its_f, term_f)
    assert relerr(x1, x_f) < 1e-12 and relerr(x2, x_f) < 1e-12
    a.close()
    f.close()
