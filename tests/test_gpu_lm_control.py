"""The decisions of b200_lm_solve's trust-region loop against the oracle's, device-resident (lm_diagonal_kernel,
lm_step_kernel, grad_norm_kernel) and through the host-buffer boundary: every exit, chains of rejected steps and chains
of invalid steps.

The solves are short (tiny and C16, a few iterations of short CG solves), so both trajectories reproduce to ~1e-10 and
every field of every record is compared (tests/entry_points.py compare_lm_traces_exact).  The options that steer each
run come from tests/lm_cases.py, whose constructions tests/test_oracle_lm_control.py checks on a CPU machine.

Invalid steps: with camera 0's focal length 0, 8 of its 9 Jacobian columns are exactly zero, so with min_lm_diagonal = 0
the LM diagonal is 0 there too and the reduced camera matrix S has exact zero rows.  Each point's E'E + D_e^2 stays
positive definite, because each point is also seen by a camera with f != 0.  The dense Cholesky of S then fails on GPU
and oracle alike (FAILURE after one iteration), so every step is invalid: the loop halves the radius, then quarters it,
..., until max_num_consecutive_invalid_steps or the minimum radius ends it.
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


@pytest.fixture(scope="module")
def cases(cs, oracle, c16):
    out = {"tiny": Case(cs, oracle, L.tiny_bal()), "c16": Case(cs, oracle, L.c16_bal(c16)),
           "zero_focal": Case(cs, oracle, L.zero_focal_bal())}
    yield out
    for c in out.values():
        c.close()


def _run_both(case, host_boundary, options):
    """GPU and oracle solves with the same options: the GPU's trace and state against the oracle's, every field."""
    state_o, recs_o, _ = L.oracle_solve(case.orc, case.state, **options)
    state, recs = L.gpu_solve(case.gpu, case.state, host_boundary, **options)
    compare_lm_traces_exact(recs, recs_o)
    assert relerr(state, state_o) < 1e-9
    return state, recs


@pytest.mark.parametrize("host_boundary", [False, True])
@pytest.mark.parametrize("problem,name,k", L.EXITS)
def test_exit(problem, name, k, host_boundary, cases):
    """Each exit fires at the iteration the oracle's fires at; the state returned is the best one so far."""
    case = cases[problem]
    options, num_records = L.place_exit(case.orc, case.state, name, k, L.REJECTION if name == "min_trust_region_radius" else None)
    _, recs = _run_both(case, host_boundary, options)
    assert len(recs) == num_records
    L.assert_decisions_have_margin(recs, options.get("min_relative_decrease", 1e-3))


@pytest.mark.parametrize("host_boundary", [False, True])
@pytest.mark.parametrize("problem", ["tiny", "c16"])
def test_no_iterations(problem, host_boundary, cases):
    """max_num_iterations = 0: the initial record only, and the initial state back."""
    case = cases[problem]
    state, recs = _run_both(case, host_boundary, dict(max_num_iterations=0))
    assert len(recs) == 1 and np.array_equal(state, case.state)


@pytest.mark.parametrize("host_boundary", [False, True])
def test_rejection_chain(host_boundary, cases):
    """Four rejected steps in a row (tests/lm_cases.py REJECTION): each one divides the radius by 2, 4, 8, 16, solves
    again with the LM diagonal of the last accepted point (lm_diagonal_kernel without refresh; the host `diagonal`
    vector), records the candidate's cost and carries the gradient norms over."""
    case = cases["c16"]
    _, recs = _run_both(case, host_boundary, L.REJECTION)
    L.assert_decisions_have_margin(recs, L.REJECTION["min_relative_decrease"])
    first, last = L.REJECTED_RUN
    assert [r["step_is_successful"] for r in recs] == [1, 1, 0, 0, 0, 0, 1, 0]
    accepted = recs[first - 1]
    for j in range(first, last + 1):
        r = recs[j]
        assert r["step_is_valid"] == 1 and r["step_is_successful"] == 0
        assert r["tr_radius"] == recs[j - 1]["tr_radius"] / 2.0 ** (j - first + 1)
        assert abs(r["cost"] - (accepted["cost"] - r["cost_change"])) <= 1e-12 * accepted["cost"]
        assert r["gradient_max_norm"] == accepted["gradient_max_norm"]
        assert r["gradient_norm"] == accepted["gradient_norm"]
        assert r["step_norm"] > 0.0 and r["model_cost_change"] > 0.0


def _check_invalid_records(recs):
    assert recs[0]["step_is_valid"] == 1
    for i, r in enumerate(recs):
        assert r["tr_radius"] == L.INVALID_RADII[i]
        if i == 0:
            continue
        assert (r["step_is_valid"], r["step_is_successful"], r["ls_iterations"]) == (0, 0, 1)
        assert r["cost"] == recs[0]["cost"] and r["cost_change"] == 0.0
        assert r["step_norm"] == 0.0 and r["model_cost_change"] == 0.0
        assert r["gradient_max_norm"] == recs[0]["gradient_max_norm"]


@pytest.mark.parametrize("host_boundary", [False, True])
@pytest.mark.parametrize("limit", [1, 3, 5])
def test_invalid_steps(limit, host_boundary, cases):
    """Every dense solve fails: limit - 1 invalid records, then the loop stops with the state unchanged."""
    case = cases["zero_focal"]
    state, recs = _run_both(case, host_boundary, dict(L.INVALID, max_num_consecutive_invalid_steps=limit))
    assert len(recs) == limit
    _check_invalid_records(recs)
    assert np.array_equal(state, case.state)


@pytest.mark.parametrize("host_boundary", [False, True])
def test_invalid_steps_reach_min_radius(host_boundary, cases):
    """The radius of the second invalid record is exactly min_trust_region_radius = 1250: the loop stops there, since
    the test is radius <= min_trust_region_radius (trust_region_minimizer.cc:707-711)."""
    case = cases["zero_focal"]
    state, recs = _run_both(case, host_boundary, dict(L.INVALID, min_trust_region_radius=1250.0))
    assert len(recs) == 3
    _check_invalid_records(recs)
    assert np.array_equal(state, case.state)
