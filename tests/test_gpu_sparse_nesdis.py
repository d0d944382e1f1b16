"""SPARSE_SCHUR under linear_solver_ordering_type = NESDIS (b200_set_linear_solver_ordering_type, the
linear_solver_ordering_type field of b200_lm_options): the nested-dissection order of csrc/sparse_plan.cuh and the
topological task order of csrc/sparse_schur.cuh, against the extended-precision reference of
tests/test_gpu_sparse_factor.py and the LM / DOGLEG references.

  structure   every camera graph of tests/test_sparse_schur_plan.py at radius 1e4, 1e-1 and D = NULL: FP64 within the
              reference's bounds, mixed precision with k = 0 within test_gpu_mixed_precision.py's C32 2^-24 and with k = 2
              no worse than k = 0; the plan line and, where the task order is not the identity, that it is not
  switching   AMD -> NESDIS -> AMD on one handle: one analysis per switch, one factor launch per solve, AMD's solutions as
              on a handle that never switched, NESDIS's within the reference bound
  failure     a non-finite Jacobian block: FAILURE without writing x, then recovery on the same handle
  lm          b200_lm_solve with NESDIS (LM and traditional DOGLEG), device-resident and through the host boundary, against
              the oracle; the handle's own ordering type afterwards, also after an error

Bitwise comparisons use mixed precision with k = 0: the FP64 reduced right-hand side is summed with REDs whose order
varies from run to run (test_gpu_sparse_factor.py test_reuse), and rounding it to float hides that, as in
test_gpu_mixed_precision.py test_reuse.
"""
import os

import numpy as np
import pytest

from tests import dogleg_reference as R
from tests import lm_cases as L
from tests.entry_points import Case, compare_lm_traces_exact, relerr
from tests.test_gpu_dogleg import _compare
from tests.test_gpu_sparse_factor import (C_X, PLAN_RE, RADII, U, check_solution, geometry, lm_diagonal, load,
                                          raw_sparse_solve, reference_for)
from tests.test_sparse_nesdis_plan import check_ordered
from tests.test_sparse_schur_plan import STRUCTURES, structure

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
C32 = 16.0   # tests/test_gpu_mixed_precision.py


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


class NdStructure:
    """One camera graph of STRUCTURES with its NESDIS plan recounted (tests/test_sparse_nesdis_plan.py)."""

    def __init__(self, cs, name):
        self.name = name
        self.C, self.P, self.cam, self.pt = structure(name)
        self.perm, self.stats, self.lay, heights = check_ordered(cs, self.C, self.P, self.cam, self.pt, cs.NESDIS)
        self.task_order = sorted(range(self.lay.ns), key=lambda s: (heights[s], s))
        self.obs, self.state = geometry(self.C, self.P, self.cam, self.pt, seed=11)

    def problem(self, cs, ordering):
        gpu = cs.Problem(self.C, self.P, self.cam, self.pt, self.obs)
        gpu.set_linear_solver_ordering_type(ordering)
        return gpu


def verbose(fn, capfd):
    """fn() under B200_VERBOSE: (its result, the sparse plan lines it printed)."""
    capfd.readouterr()
    os.environ["B200_VERBOSE"] = "1"
    try:
        out = fn()
    finally:
        del os.environ["B200_VERBOSE"]
    return out, [ln for ln in capfd.readouterr().err.splitlines() if "sparse S plan" in ln]


@pytest.mark.parametrize("name", STRUCTURES)
def test_structure(name, cs, capfd, record_property):
    s = NdStructure(cs, name)
    if name in ("cliques", "band", "loop", "forest", "random400", "shuffled"):
        assert s.task_order != list(range(s.lay.ns))
    gpu = s.problem(cs, cs.NESDIS)
    b = load(gpu, s, "random")
    n_e = 3 * s.P
    for radius in RADII:
        D = lm_diagonal(gpu, radius)
        if radius == RADII[0]:
            (x, its, term), lines = verbose(lambda: gpu.sparse_schur_solve(b, D), capfd)
            assert len(lines) == 1 and "-> nested dissection," in lines[0], lines
            m = PLAN_RE.search(lines[0])
            assert m and int(m.group(1)) == s.lay.ns and int(m.group(2)) == 9 * s.lay.width.max()
            assert "critical path %d supernodes" % s.stats["critical_path_supernodes"] in lines[0]
        else:
            x, its, term = gpu.sparse_schur_solve(b, D)
        assert (its, term) == (1, cs.LS_SUCCESS)
        ref, kappa, x_ref = reference_for(gpu, s, b, D)
        tag = "%s/nesdis/%s" % (name, radius)
        check_solution(x, ref, kappa, x_ref, record_property, tag)
        etas = []
        for k in (0, 2):
            gpu.set_exact_solve_options(True, k)
            xm, _, tm = gpu.sparse_schur_solve(b, D)
            assert tm == cs.LS_SUCCESS, (tag, k)
            etas.append(ref.eta(xm[n_e:]))
        gpu.set_exact_solve_options(False, 0)
        record_property(tag + "/mixed", "eta/2^-24 k=0 %.2e k=2 %.2e" % (etas[0] / U32, etas[1] / U32))
        assert etas[0] <= C32 * U32, (tag, etas)
        assert etas[1] <= etas[0] or etas[1] <= 16.0 * U, (tag, etas)
    gpu.close()


def test_switching(cs, capfd):
    s = NdStructure(cs, "loop")
    gpu = s.problem(cs, cs.AMD)
    b = load(gpu, s, "random")
    D = lm_diagonal(gpu, 1e4)
    ref, kappa, x_ref = reference_for(gpu, s, b, D)
    n_e = 3 * s.P

    def solve_counted():
        gpu.stats_reset()
        x, its, term = gpu.sparse_schur_solve(b, D)
        assert (its, term) == (1, cs.LS_SUCCESS)
        assert gpu.stats()["sparse_factor"]["launches"] == 1
        return x

    def phase(ordering):
        """Set the type and solve three times (FP64, mixed k = 0 twice): one analysis, at the first solve."""
        gpu.set_exact_solve_options(False, 0)
        gpu.set_linear_solver_ordering_type(ordering)
        x, lines = verbose(solve_counted, capfd)
        assert len(lines) == 1 and ("-> nested dissection," in lines[0]) == (ordering == cs.NESDIS), lines
        check_solution(x, ref, kappa, x_ref, tag=str(ordering))
        gpu.set_exact_solve_options(True, 0)
        (xm, xm2), lines = verbose(lambda: (solve_counted(), solve_counted()), capfd)
        assert lines == [] and np.array_equal(xm[n_e:], xm2[n_e:])
        return x, xm

    x1, m1 = phase(cs.AMD)
    x2, m2 = phase(cs.NESDIS)
    # the same type again is a no-op: no analysis
    gpu.set_linear_solver_ordering_type(cs.NESDIS)
    _, lines = verbose(solve_counted, capfd)
    assert lines == []
    x3, m3 = phase(cs.AMD)
    assert ref.scaled_err(x2[n_e:], x1[n_e:]) <= 2 * C_X * kappa * U
    assert np.array_equal(m1[n_e:], m3[n_e:])
    fresh = s.problem(cs, cs.AMD)
    load(fresh, s, "random")
    fresh.set_exact_solve_options(True, 0)
    xf, _, tf = fresh.sparse_schur_solve(b, D)
    assert tf == cs.LS_SUCCESS and np.array_equal(xf[n_e:], m1[n_e:])
    # reproducible under NESDIS on a fresh handle too
    nd = s.problem(cs, cs.NESDIS)
    load(nd, s, "random")
    nd.set_exact_solve_options(True, 0)
    xn, _, _ = nd.sparse_schur_solve(b, D)
    assert np.array_equal(xn[n_e:], m2[n_e:])
    for bad in (2, -1):
        with pytest.raises(cs.B200Error) as e:
            gpu.set_linear_solver_ordering_type(bad)
        assert e.value.code == cs.binding.ERR_INVALID_ARGUMENT
    for h in (gpu, fresh, nd):
        h.close()


@pytest.mark.parametrize("fault", ["nan_first", "inf_root"])
def test_failure_and_recovery(fault, cs):
    s = NdStructure(cs, "band")
    gpu = s.problem(cs, cs.NESDIS)
    b = load(gpu, s, "random")
    v = gpu.jacobian_values()
    D = lm_diagonal(gpu, 1e4)
    vb = v.copy()
    N = len(s.cam)
    c = int(s.perm[0] if fault == "nan_first" else s.perm[-1])
    row = int(np.flatnonzero(s.cam == c)[0])
    vb[6 * N + 18 * row + 7] = np.nan if fault == "nan_first" else np.inf
    gpu.set_jacobian_values(vb)
    x, term = raw_sparse_solve(cs, gpu, b, D)
    assert term == cs.LS_FAILURE and np.all(x == -7.25)
    gpu.set_jacobian_values(v)
    x, term = raw_sparse_solve(cs, gpu, b, D)
    assert term == cs.LS_SUCCESS
    ref, kappa, x_ref = reference_for(gpu, s, b, D)
    check_solution(x, ref, kappa, x_ref, tag=fault)
    gpu.close()


def _lm_case(cs, oracle, c16, which):
    from tests.test_gpu_sparse_schur import _bal
    return Case(cs, oracle, _bal(which, c16))


def _assert_amd_after(cs, case, capfd):
    """The handle's ordering type is AMD again: its next sparse solve analyses in an AMD order."""
    ok, _, res, _ = case.gpu.evaluate(case.state)
    assert ok
    D = lm_diagonal(case.gpu, 1e4)
    (_, _, term), lines = verbose(lambda: case.gpu.sparse_schur_solve(res, D), capfd)
    assert term == cs.LS_SUCCESS
    assert len(lines) == 1 and "nested dissection" not in lines[0], lines


@pytest.mark.parametrize("which", ["c16", "sequence"])
@pytest.mark.parametrize("host_boundary", [False, True])
def test_lm(which, host_boundary, cs, oracle, c16, capfd):
    """Four LM iterations with SPARSE_SCHUR under NESDIS against the oracle's DENSE_SCHUR loop (the tolerances of
    tests/test_gpu_sparse_factor.py test_lm_loop_many_supernodes), and three traditional DOGLEG iterations against
    tests/dogleg_reference.py (those of tests/test_gpu_dogleg.py); the handle stays at AMD.  The sequence (300 frames,
    tests/test_gpu_sparse_schur.py) starts from radius 1, as tests/test_gpu_dogleg.py runs it: from the default 1e4 its
    first step is so long that the rejected candidate's cost (~1e58) differs between any two summation orders."""
    case = _lm_case(cs, oracle, c16, which)
    _, st = cs.plan_sparse_schur(case.rp.C, case.rp.P, case.rp.row_cam, case.rp.row_pt, cs.NESDIS)
    assert st["order"] == 2
    start = dict(initial_trust_region_radius=1.0) if which == "sequence" else {}
    _, recs_o, _ = L.oracle_solve(case.orc, case.state, linear_solver_type=L.DENSE_SCHUR, max_num_iterations=4, **start)
    (_, recs), lines = verbose(lambda: L.gpu_solve(case.gpu, case.state, host_boundary, linear_solver_type=cs.SPARSE_SCHUR,
                                                   linear_solver_ordering_type=cs.NESDIS, max_num_iterations=4, **start),
                               capfd)
    compare_lm_traces_exact(recs, recs_o)
    assert len(lines) == 1 and "-> nested dissection," in lines[0], lines
    _assert_amd_after(cs, case, capfd)
    options = dict(initial_trust_region_radius=1.0, max_num_iterations=3)
    state_o, recs_o, _ = R.minimize(case.orc, case.state, cs.TRADITIONAL_DOGLEG, **options)
    state, recs = case.gpu.lm_solve(case.state, case.gpu.lm_options(
        trust_region_strategy_type=cs.DOGLEG, dogleg_type=cs.TRADITIONAL_DOGLEG, linear_solver_type=cs.SPARSE_SCHUR,
        linear_solver_ordering_type=cs.NESDIS, **options), host_boundary=host_boundary)
    _compare(case, cs.TRADITIONAL_DOGLEG, options, recs, recs_o)
    assert relerr(state, state_o) < 1e-6
    case.close()


def test_lm_restores_after_error(cs, oracle, c16, capfd):
    """A non-finite initial state fails the loop's first evaluation after the call has switched to NESDIS: the handle is
    back at AMD (its next sparse solve analyses in an AMD order).  An invalid ordering type fails before any switch: the
    handle keeps its AMD analysis (no new one).  A NESDIS handle keeps NESDIS across an AMD call."""
    case = _lm_case(cs, oracle, c16, "c16")
    bad_state = case.state.copy()
    bad_state[0] = np.nan
    for host_boundary in (False, True):
        with pytest.raises(cs.B200Error):
            case.gpu.lm_solve(bad_state, case.gpu.lm_options(linear_solver_type=cs.SPARSE_SCHUR,
                                                              linear_solver_ordering_type=cs.NESDIS),
                              host_boundary=host_boundary)
        _assert_amd_after(cs, case, capfd)
    with pytest.raises(cs.B200Error) as e:
        case.gpu.lm_solve(case.state, case.gpu.lm_options(linear_solver_type=cs.SPARSE_SCHUR, linear_solver_ordering_type=2))
    assert e.value.code == cs.binding.ERR_INVALID_ARGUMENT
    ok, _, res, _ = case.gpu.evaluate(case.state)
    (_, _, term), lines = verbose(lambda: case.gpu.sparse_schur_solve(res, lm_diagonal(case.gpu, 1e4)), capfd)
    assert ok and term == cs.LS_SUCCESS and lines == [], lines
    # a NESDIS handle after an AMD call: NESDIS again, without a new analysis until a sparse solve needs one
    case.gpu.set_linear_solver_ordering_type(cs.NESDIS)
    case.gpu.lm_solve(case.state, case.gpu.lm_options(linear_solver_type=cs.SPARSE_SCHUR, max_num_iterations=1))
    ok, _, res, _ = case.gpu.evaluate(case.state)
    (_, _, term), lines = verbose(lambda: case.gpu.sparse_schur_solve(res, lm_diagonal(case.gpu, 1e4)), capfd)
    assert term == cs.LS_SUCCESS and len(lines) == 1 and "-> nested dissection," in lines[0], lines
    case.close()
