"""The constructions of tests/eval_failure_cases.py on the oracle alone: each gives the verdict the GPU tests
(tests/test_gpu_eval_failure.py) expect of it, with the margins it is built for, so that a change to a construction, a
generator or the oracle fails here on a CPU machine instead of quietly testing something else on an H100."""
import numpy as np
import pytest

from tests import eval_failure_cases as F
from tests import lm_cases as L


def _problem(oracle, bal, huber_a=None):
    from ceres_solver_b200 import bal as B
    rp = B.ReducedProgram(bal)
    kw = {} if huber_a is None else dict(use_huber=True, huber_a=huber_a)
    orc = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel(), **kw)
    return rp, orc, rp.state(bal)


def _bals(c16):
    from tests.test_gpu_parity import huge_bal
    return {"tiny": L.tiny_bal(), "c16": L.c16_bal(c16), "huge": huge_bal()}


def _placements(rp, state):
    import ceres_solver_b200 as cs
    perm, _, _ = cs.plan_point_order(rp.C, rp.P, rp.row_cam, rp.row_pt, 132)
    return F.placements(state, rp.row_cam, rp.row_pt, rp.P, perm)


def _overflow_rows(rp, state, places):
    return F.overflow_targets(places, state, rp.row_cam, rp.row_pt, rp.P)


def _constructions(rp, state, places):
    """(kind, rows, state) of every construction of a problem: each single-row kind at every placement, and the two
    cost_overflow sizes on rows spread over the problem."""
    out = []
    for row in places.values():
        for kind in ("residual_nonfinite", "jacobian_only") + F.PLAIN_KINDS:
            out.append((kind, [row], F.construct(state, rp.row_cam, rp.row_pt, rp.P, kind, row)))
    rows = _overflow_rows(rp, state, places)
    for kind, k in (("cost_overflow2", 2), ("cost_overflow3", 3)):
        out.append((kind, rows[:k], F.construct(state, rp.row_cam, rp.row_pt, rp.P, kind, rows[:k])))
    return out


@pytest.fixture(scope="module")
def bals(c16):
    return _bals(c16)


@pytest.mark.parametrize("problem", ["tiny", "c16", "huge"])
def test_placements(problem, bals, oracle):
    """Every placement the GPU tests rely on is there: both ends of the internal order, degree-1 and ordinary points,
    and on `huge` the 33..128-row and >128-row points; `tiny` and `c16` have none of more than 32 rows."""
    rp, _, state = _problem(oracle, bals[problem])
    places = _placements(rp, state)
    assert {"first", "last", "ordinary_0", "ordinary_1", "ordinary_2"} <= set(places)
    deg = np.bincount(rp.row_pt)
    if problem == "huge":
        assert {"rows33_128_0", "rows33_128_1", "rows129+_0", "rows129+_1"} <= set(places)
    else:
        assert deg.max() <= 32
    zeroable = F.zeroable_cameras(state, rp.row_cam, rp.row_pt, rp.P)
    for label, row in places.items():
        assert zeroable[rp.row_cam[row]], (label, row)
        if label.startswith("ordinary"):
            assert 2 <= deg[rp.row_pt[row]] <= 32


@pytest.mark.parametrize("problem", ["tiny", "c16", "huge"])
def test_verdicts(problem, bals, oracle):
    """Each construction's oracle verdict in every call mode is the one expected_ok states, with the trivial loss and
    under Huber(a) for a = the median row norm."""
    rp, orc, state = _problem(oracle, bals[problem])
    _, orc_h, _ = _problem(oracle, bals[problem], huber_a=L.huber_scale(orc, state))
    places = _placements(rp, state)
    for kind, rows, x in _constructions(rp, state, places):
        for mode, args in F.MODES.items():
            ok, cost, _, _ = orc.evaluate(x, *args, nt=8)
            assert ok == F.expected_ok(kind, mode), (kind, rows, mode, cost)
            if kind in ("jacobian_only", "residual_nonfinite") and rows[0] != places["first"]:
                continue   # under Huber: every kind at the first placement, the overflow kinds
            ok_h, cost_h, _, _ = orc_h.evaluate(x, *args, nt=8)
            assert ok_h == F.expected_ok(kind, mode, huber=True), (kind, rows, mode, cost_h)


@pytest.mark.parametrize("problem", ["tiny", "c16", "huge"])
def test_healthy_part(problem, bals, oracle):
    """The zeroed cameras of every construction, with the target points left as they are, evaluate in every mode: only
    the target rows make a construction fail."""
    rp, orc, state = _problem(oracle, bals[problem])
    places = _placements(rp, state)
    rows = _overflow_rows(rp, state, places)
    for kind in ("residual_nonfinite", "jacobian_only", "cost_overflow3"):
        targets = rows if kind == "cost_overflow3" else list(places.values())
        x = F.zeroed_cameras(state, rp.row_cam, rp.P, kind, targets)
        for mode, args in F.MODES.items():
            ok, cost, _, _ = orc.evaluate(x, *args, nt=8)
            assert ok and cost < 1e30, (kind, mode, cost)


@pytest.mark.parametrize("problem", ["tiny", "c16", "huge"])
def test_overflow_margins(problem, bals, oracle):
    """Two cost_overflow rows sum below 0.9 DBL_MAX with everything else, three above 1.1 DBL_MAX: every row costs
    0.72e308 (to 1e-6) and the rest of the problem is negligible beside it.  No row and no sum of two overflows."""
    rp, orc, state = _problem(oracle, bals[problem])
    rows = _overflow_rows(rp, state, _placements(rp, state))
    row_costs = [F.overflow_row_cost(rp.row_obs[r]) for r in rows]
    assert all(abs(c - 0.72e308) <= 1e-6 * 0.72e308 for c in row_costs), row_costs
    x2 = F.construct(state, rp.row_cam, rp.row_pt, rp.P, "cost_overflow2", rows[:2])
    ok, cost2, res, _ = orc.evaluate(x2, want_gradient=False, want_jacobian=False, nt=8)
    assert ok and cost2 < 0.9 * F.DBL_MAX
    rest = cost2 - sum(row_costs[:2])   # the other rows: below the last bit of the two overflow rows' sum
    assert 0.0 <= rest < 1e-6 * F.DBL_MAX
    assert (rest + sum(row_costs[:2])) / F.DBL_MAX < 0.9 and sum(c / F.DBL_MAX for c in row_costs) > 1.1
    # the overflow rows' residuals are exactly f x_p - o_x with x_p = 1.2e151 on the oracle's side as well
    for r in rows[:2]:
        assert res[2 * r] == 1e3 * 1.2e151 - rp.row_obs[r][0] and res[2 * r + 1] == -rp.row_obs[r][1]


def test_jacobian_only_margin():
    """x_p is 1 to 4 ulp whichever way p_x / p_z is rounded (-p_x * (1 / p_z) on the GPU, -p_x / p_z in the oracle), and
    the Jacobian entry f / p_z overflows by a factor of 4."""
    px, _, pz = F.JACOBIAN_ONLY_X
    assert pz > np.finfo(np.float64).tiny   # a normal number: no subnormal arithmetic on either side
    assert abs(-px * (1.0 / pz) - 1.0) <= 4 * np.finfo(np.float64).eps and -px / pz == 1.0
    assert F.JACOBIAN_ONLY_INTRINSICS[0] * (1.0 / pz) == np.inf
    assert F.JACOBIAN_ONLY_INTRINSICS[0] / pz / 4.0 > F.DBL_MAX


@pytest.mark.parametrize("kind", F.OBSERVATION_KINDS)
def test_observation_kinds(kind, bals, oracle):
    """A non-finite observation fails every mode, at a row of each class of `huge`."""
    bal = bals["huge"]
    rp, _, state = _problem(oracle, bal)
    places = _placements(rp, state)
    for label in ("first", "rows33_128_0", "rows129+_0"):
        _, orc, state = _problem(oracle, F.with_observation(bal, rp.obs_of_row, places[label], kind))
        for mode, args in F.MODES.items():
            ok, _, _, _ = orc.evaluate(state, *args, nt=8)
            assert not ok, (kind, label, mode)
