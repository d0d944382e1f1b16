"""b200_lm_solve with the DOGLEG strategy (traditional and subspace) against the CPU reference in tests/dogleg_reference.py,
which restates DoglegStrategy literally on the oracle's DENSE_SCHUR solve: the device-resident loop (dogleg_diagonal_kernel,
dogleg_gn_kernel, dogleg_gram_kernel, dogleg_step_kernel) and the host-boundary loop, with DENSE_SCHUR and SPARSE_SCHUR.

The option sets come from tests/dogleg_cases.py, whose branch coverage tests/test_oracle_dogleg.py checks on a CPU machine.
"""
import numpy as np
import pytest

from tests import dogleg_cases as K
from tests import dogleg_reference as R
from tests import lm_cases as L
from tests.entry_points import Case, compare_lm_traces_exact, relerr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.fixture(scope="module")
def cases(cs, oracle, c16):
    out = {"tiny": Case(cs, oracle, L.tiny_bal()), "c16": Case(cs, oracle, L.c16_bal(c16)),
           "zero_focal": Case(cs, oracle, L.zero_focal_bal())}
    yield out
    for c in out.values():
        c.close()


def _factor_launches(cs, stats, solver):
    # one dense assembly (then potrf) per DENSE_SCHUR solve; one sparse_factor launch per SPARSE_SCHUR solve
    return stats["schur_diag_blocks" if solver == cs.DENSE_SCHUR else "sparse_factor"]["launches"]


KEYS = ("cost", "step_norm", "gradient_max_norm", "gradient_norm", "tr_radius", "model_cost_change")


def _run(cs, case, dogleg_type, solver, host_boundary, options):
    state_o, recs_o, info = R.minimize(case.orc, case.state, dogleg_type, **options)
    case.gpu.stats_reset()
    state, recs = case.gpu.lm_solve(case.state, case.gpu.lm_options(
        trust_region_strategy_type=cs.DOGLEG, dogleg_type=dogleg_type, linear_solver_type=solver, **options),
        host_boundary=host_boundary)
    return state, state_o, recs, recs_o, info, case.gpu.stats()


def _compare(case, dogleg_type, options, recs, recs_o):
    """Linear solver iterations and every decision exact; the values to max(1e-5, 10 x the reference's own spread over two
    thread counts), as tests/conftest.py compare_lm_traces holds its inexact trajectories.  The Gauss-Newton system is
    damped by mu = 1e-8 only, and bundle adjustment's gauge freedom leaves it that ill-conditioned: near the minimum a
    new Gauss-Newton step moves by up to 2e-6 relative between the GPU's and the oracle's factorisations, where the LM
    loop's damped solves agree to 1e-10.  Measured on an H100, the largest deviation of any value over all of this module's
    traces is 2.1e-6: the step norm on `tiny` with the rejection set, iterations 5 and 6.  Every C16 trace stays below 6e-7.
    The worst deviation of each trace is printed (pytest -s)."""
    _, recs_alt, _ = R.minimize(case.orc, case.state, dogleg_type, nt=3, **options)
    assert len(recs) == len(recs_o) == len(recs_alt)
    worst = (0.0, None)
    for a, b, c in zip(recs, recs_o, recs_alt):
        for key in ("ls_iterations", "step_is_valid", "step_is_successful"):
            assert int(a[key]) == int(b[key]), (key, a, b)
        for key in KEYS:
            spread = abs(c[key] - b[key]) / max(abs(b[key]), 1e-300)
            dev = abs(a[key] - b[key]) / max(abs(b[key]), 1e-300)
            assert dev <= max(1e-5, 10.0 * spread), (key, a, b)
            worst = max(worst, (dev, "%s@%d" % (key, a["iteration"])), key=lambda w: w[0])
    print("dogleg trace worst relative deviation %.2e (%s)" % worst)


@pytest.mark.parametrize("host_boundary", [False, True])
@pytest.mark.parametrize("solver", ["dense", "sparse"])
@pytest.mark.parametrize("dogleg_type", [0, 1])
@pytest.mark.parametrize("problem,option_set", K.TRACES)
def test_trace(problem, option_set, dogleg_type, solver, host_boundary, cs, cases):
    """Every field of every record against the reference; the state returned; one factorisation per new Gauss-Newton
    step (none for a reused one) and, device-resident, one dogleg_gram pass per new step."""
    case = cases[problem]
    solver = cs.DENSE_SCHUR if solver == "dense" else cs.SPARSE_SCHUR
    options = K.OPTIONS[option_set]
    state, state_o, recs, recs_o, info, stats = _run(cs, case, dogleg_type, solver, host_boundary, options)
    _compare(case, dogleg_type, options, recs, recs_o)
    assert relerr(state, state_o) < 1e-8
    solves = sum(n for n, *_ in info)
    new_steps = sum(1 for n, *_ in info if n > 0)
    assert _factor_launches(cs, stats, solver) == solves
    for r, (n, *_) in zip(recs[1:], info[1:]):
        assert (r["ls_iterations"] == 0) == (n == 0)
    if not host_boundary:
        assert stats["dogleg_gram"]["launches"] == new_steps
        # one dogleg_diagonal and one dogleg_gn operation per new step, one dogleg_step per valid solve or reuse
        assert stats["dogleg_diagonal"]["operations"] == new_steps
        assert stats["dogleg_gn"]["launches"] == stats["dogleg_diagonal"]["launches"]
        assert stats["dogleg_step"]["operations"] == sum(1 for n, b, _ in info[1:] if b is not None)
        for name in ("dogleg_gram", "dogleg_diagonal", "dogleg_gn", "dogleg_step"):
            assert stats[name]["bytes_per_operation"] > 0


@pytest.mark.parametrize("host_boundary", [False, True])
@pytest.mark.parametrize("solver", ["dense", "sparse"])
@pytest.mark.parametrize("dogleg_type", [0, 1])
def test_zero_focal_invalid_steps(dogleg_type, solver, host_boundary, cs, cases):
    """Every factorisation fails (tests/test_gpu_lm_control.py explains the construction): the first iteration raises mu
    tenfold from 1e-8 to 1 through eight failed solves, later ones solve nothing (mu is past its cap) and record -1 linear
    solver iterations; the radius never changes; the state comes back untouched."""
    case = cases["zero_focal"]
    solver = cs.DENSE_SCHUR if solver == "dense" else cs.SPARSE_SCHUR
    state, _, recs, recs_o, info, stats = _run(cs, case, dogleg_type, solver, host_boundary, K.INVALID)
    compare_lm_traces_exact(recs, recs_o)
    assert np.array_equal(state, case.state)
    assert all(r["tr_radius"] == recs[0]["tr_radius"] for r in recs)
    assert [r["ls_iterations"] for r in recs[1:]] == [1] + [-1] * (len(recs) - 2)
    assert all(r["step_is_valid"] == 0 for r in recs[1:])
    assert _factor_launches(cs, stats, solver) == sum(n for n, *_ in info) == 8


@pytest.mark.parametrize("which", ["huge", "sequence"])
@pytest.mark.parametrize("dogleg_type", [0, 1])
def test_larger_problems(which, dogleg_type, cs, oracle, c16):
    """The huge-point problem (chunk tiles in dogleg_gram_kernel) and the sequence with the explicit S plan, both solvers and
    both loops, three iterations against the reference."""
    from tests.test_gpu_sparse_schur import _bal
    case = Case(cs, oracle, _bal(which, c16))
    options = dict(initial_trust_region_radius=1.0, max_num_iterations=3)
    state_o, recs_o, _ = R.minimize(case.orc, case.state, dogleg_type, **options)
    for solver in (cs.DENSE_SCHUR, cs.SPARSE_SCHUR):
        for host_boundary in (False, True):
            state, recs = case.gpu.lm_solve(case.state, case.gpu.lm_options(
                trust_region_strategy_type=cs.DOGLEG, dogleg_type=dogleg_type, linear_solver_type=solver, **options),
                host_boundary=host_boundary)
            _compare(case, dogleg_type, options, recs, recs_o)
            assert relerr(state, state_o) < 1e-6
    case.close()


def test_error_paths(cs, cases):
    """DOGLEG with ITERATIVE_SCHUR (solver.cc:431-438) and out-of-range enum values: B200_ERR_INVALID_ARGUMENT."""
    gpu = cases["tiny"].gpu
    state = cases["tiny"].state
    bad = [dict(trust_region_strategy_type=cs.DOGLEG, linear_solver_type=cs.ITERATIVE_SCHUR),
           dict(trust_region_strategy_type=2, linear_solver_type=cs.DENSE_SCHUR),
           dict(trust_region_strategy_type=-1),
           dict(trust_region_strategy_type=cs.DOGLEG, dogleg_type=2, linear_solver_type=cs.DENSE_SCHUR)]
    for kw in bad:
        with pytest.raises(cs.B200Error) as e:
            gpu.lm_solve(state, gpu.lm_options(**kw))
        assert e.value.code == cs.binding.ERR_INVALID_ARGUMENT, kw
    with pytest.raises(cs.B200Error) as e:
        gpu.lm_solve(state, gpu.lm_options(**bad[0]))
    assert "DOGLEG only supports exact factorization" in str(e.value)
    # the defaults are Levenberg-Marquardt and traditional dogleg (bundle_adjuster.cc:79-81)
    o = gpu.lm_options()
    assert (o.trust_region_strategy_type, o.dogleg_type) == (cs.LEVENBERG_MARQUARDT, cs.TRADITIONAL_DOGLEG)
