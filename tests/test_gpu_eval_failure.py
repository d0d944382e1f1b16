"""The other half of the Evaluator contract: when b200_evaluate fails (B200_ERR_EVALUATION_FAILED, where
Evaluator::Evaluate returns false), and what a call leaves behind on the handle.

The bad states come from tests/eval_failure_cases.py, whose verdicts tests/test_oracle_eval_failure_cases.py pins on
the oracle alone.  Each is only a new state vector on the same handle, so every construction runs at many placements:
a row of the first and the last point of the library's internal order, of points of 33..128 and >128 rows, a degree-1
point, a duplicated (camera, point) row and a seeded sample of ordinary points.  The problems are the six fixtures of
tests/test_gpu_dispatch.py, C16, `tiny` and the huge-point problem; together they run evaluate_v2_kernel,
evaluate_kernel<true> on the 33..128-row and >128-row tiles and everywhere under CTA-tile, and evaluate_kernel<false>
(cost-only and residual-only calls) under every configuration.

In each call mode (cost only, residuals only, gradient without the Jacobian, gradient with it, Jacobian only) the GPU's
verdict must be the expected one; the oracle is called on every successful call and on all calls at the first
placement, and must agree, with cost and residuals to the bounds of tests/entry_points.py.  After every failure:
b200_last_error names it, a failed call that asked for residuals leaves no resident residuals (b == NULL in the solves
and b200_model_cost_change is refused), and the next evaluate at the healthy state matches the oracle, so the failure
flag and the cost partials were reset.

Not covered: a failing candidate evaluation inside the LM loop (tests/eval_failure_cases.py explains why), and the
failure flag's exchange between ranks, which needs two GPUs.
"""
import numpy as np
import pytest

from tests import eval_failure_cases as F
from tests import lm_cases as L
from tests.entry_points import Case, compare_lm_traces_exact, relerr

pytestmark = pytest.mark.gpu

# the six dispatch fixtures, then C16, the huge-point problem, tiny and the ragged problem (degree-1 points)
PROBLEMS = ["dups_direct", "dups_id_range", "direct_v3", "id_range", "tile", "v4_narrow", "c16", "huge", "tiny", "ragged"]

# the point order b200_create plans for an H100 SXM's 132 SMs (on another SM count "first" and "last" are two more
# points of the sample)
NUM_SMS = 132


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


def _bal(name, c16):
    if name == "c16":
        return L.c16_bal(c16)
    if name == "tiny":
        return L.tiny_bal()
    if name == "huge":
        from tests.test_gpu_parity import huge_bal
        return huge_bal()
    if name == "ragged":
        from tests.test_gpu_parity import ragged_bal
        return ragged_bal()
    from tests.test_gpu_dispatch import _bal as dispatch_bal
    return dispatch_bal(name)


def _placements(cs, rp, state):
    perm, _, _ = cs.plan_point_order(rp.C, rp.P, rp.row_cam, rp.row_pt, NUM_SMS)
    return F.placements(state, rp.row_cam, rp.row_pt, rp.P, perm)


class Setup:
    def __init__(self, cs, oracle, bal, loss_type=0, loss_a=1.0):
        self.case = Case(cs, oracle, bal, loss_type, loss_a)
        rp, state = self.case.rp, self.case.state
        self.places = _placements(cs, rp, state)
        self.overflow = F.overflow_targets(self.places, state, rp.row_cam, rp.row_pt, rp.P)
        ok, self.cost_o, self.res_o, self.grad_o = self.case.orc.evaluate(state, nt=8)
        assert ok

    def construct(self, kind, rows):
        rp = self.case.rp
        return F.construct(self.case.state, rp.row_cam, rp.row_pt, rp.P, kind, rows)

    def constructions(self, kinds, labels=None):
        """(kind, label, state) for the single-row kinds at the placements `labels` (all if None), then cost_overflow2
        and cost_overflow3."""
        out = []
        for label, row in self.places.items():
            if labels is None or label in labels:
                out += [(kind, label, self.construct(kind, row)) for kind in kinds]
        out += [(kind, "spread", self.construct(kind, self.overflow[:F.overflow_count(kind)]))
                for kind in ("cost_overflow2", "cost_overflow3")]
        return out

    def check_healthy(self, args):
        """An evaluate at the healthy state in call mode `args` matches the oracle's."""
        ok, cost, res, grad = self.case.gpu.evaluate(self.case.state, *args)
        assert ok and abs(cost - self.cost_o) <= 1e-12 * self.cost_o
        if args[0]:
            assert relerr(res, self.res_o) < 1e-12
        if args[1]:
            assert relerr(grad, self.grad_o) < 1e-10


@pytest.fixture(scope="module", params=PROBLEMS)
def setup(request, cs, oracle, c16):
    s = Setup(cs, oracle, _bal(request.param, c16))
    s.name = request.param
    yield s
    s.case.close()


def _last_error(cs):
    return cs.lib().b200_last_error().decode()


def _assert_no_resident_residuals(cs, gpu):
    """b == NULL (the residuals of the last evaluate) is refused by both solves and by b200_model_cost_change."""
    D = np.ones(gpu.num_parameters)
    for call in (lambda: gpu.schur_solve(None, D), lambda: gpu.dense_schur_solve(None, D),
                 lambda: gpu.model_cost_change(np.zeros(gpu.num_parameters))):
        with pytest.raises(cs.B200Error) as e:
            call()
        assert e.value.code == cs.binding.ERR_INVALID_ARGUMENT


def _check_call(cs, s, x, mode, expect, with_oracle, orc=None):
    """One evaluate of state x in `mode` on the GPU: the verdict, the oracle's verdict and values, and after a failure
    the handle's state."""
    gpu = s.case.gpu
    orc = orc or s.case.orc
    args = F.MODES[mode]
    ok, cost, res, _ = gpu.evaluate(x, *args)
    assert ok == expect
    if ok or with_oracle:
        ok_o, cost_o, res_o, _ = orc.evaluate(x, *args, nt=8)
        assert ok_o == ok
        if ok:   # only modes that compute no J succeed: no gradient to compare
            assert abs(cost - cost_o) <= 1e-12 * cost_o
            if args[0]:   # scaled first: the overflow rows' residuals are 1.2e154, whose squares overflow
                scale = np.max(np.abs(res_o))
                assert relerr(res / scale, res_o / scale) < 1e-12
    if not ok:
        assert "non-finite" in _last_error(cs)
        if args[0]:
            _assert_no_resident_residuals(cs, gpu)
    return ok


def test_verdicts(setup, cs):
    """Every construction at every placement in every call mode, followed after each failure by an evaluate at the
    healthy state in the same mode."""
    s = setup
    for kind, label, x in s.constructions(("residual_nonfinite", "jacobian_only") + F.PLAIN_KINDS):
        for mode in F.MODES:
            try:
                ok = _check_call(cs, s, x, mode, F.expected_ok(kind, mode), with_oracle=label == "first")
                if not ok:
                    s.check_healthy(F.MODES[mode])
            except AssertionError as e:
                raise AssertionError("%s: %s at %s, %s" % (s.name, kind, label, mode)) from e


def test_cost_overflow_sum(setup):
    """Two overflow rows: the GPU's cost, summed over its tiles in its own order, is the oracle's to 1e-12, although it
    is 1.44e308."""
    s = setup
    x = s.construct("cost_overflow2", s.overflow[:2])
    for mode in ("cost", "residuals"):
        ok, cost, _, _ = s.case.gpu.evaluate(x, *F.MODES[mode])
        ok_o, cost_o, _, _ = s.case.orc.evaluate(x, *F.MODES[mode], nt=8)
        assert ok and ok_o and cost_o > 1.4e308
        assert abs(cost - cost_o) <= 1e-12 * cost_o


def test_resident_residuals(setup, cs):
    """A failed evaluate that asked for residuals leaves none resident; a failed cost-only one leaves the last good
    ones, which b == NULL then uses: same answers as passing them explicitly."""
    s = setup
    gpu = s.case.gpu
    bad = s.construct("residual_nonfinite", s.places["first"])
    for mode in ("residuals", "gradient", "gradient_jacobian"):
        ok, _, res, _ = gpu.evaluate(s.case.state)
        assert ok
        ok, _, _, _ = gpu.evaluate(bad, *F.MODES[mode])
        assert not ok
        _assert_no_resident_residuals(cs, gpu)
    ok, _, res, _ = gpu.evaluate(s.case.state)
    assert ok
    for mode in ("cost", "jacobian"):
        ok, _, _, _ = gpu.evaluate(bad, *F.MODES[mode])
        assert not ok
    ok, _, _, _ = gpu.evaluate(s.case.state, *F.MODES["jacobian"])   # J back to the healthy state's; residuals kept
    assert ok
    D = np.sqrt(np.clip(gpu.squared_column_norm(), 1e-6, 1e32) / 1e4)
    o = gpu.solver_options(q_tolerance=0.0, r_tolerance=0.0, max_num_iterations=10)   # exactly 10 CG iterations
    x0, its0, term0 = gpu.schur_solve(None, D, o)
    x1, its1, term1 = gpu.schur_solve(res, D, o)
    assert (its0, term0) == (its1, term1) and relerr(x0, x1) < 1e-9
    if 9 * gpu.C <= 4000:
        x0, _, term0 = gpu.dense_schur_solve(None, D)
        x1, _, term1 = gpu.dense_schur_solve(res, D)
        assert term0 == term1 == cs.LS_SUCCESS and relerr(x0, x1) < 1e-9
    step = np.random.RandomState(4).randn(gpu.num_parameters) * 1e-3
    Js = gpu.right_multiply(step)
    expect = -float(np.dot(Js, res + 0.5 * Js))
    assert abs(gpu.model_cost_change(step) - expect) <= 1e-10 * abs(expect)


def test_gradient_only_leaves_jacobian(setup):
    """The gradient without the Jacobian, at x1 != x0, is the oracle's at x1 and leaves the Jacobian of x0 stored, bit
    for bit, in whichever kernel computes J; so does such a call that fails on a non-finite J."""
    s = setup
    gpu, orc = s.case.gpu, s.case.orc
    ok, _, _, _ = gpu.evaluate(s.case.state)
    assert ok
    v0 = gpu.jacobian_values()
    x1 = s.case.state * (1.0 + 1e-4 * np.random.RandomState(5).randn(s.case.state.size))
    for args in ((True, True, False), (False, True, False)):
        ok, cost, res, grad = gpu.evaluate(x1, *args)
        ok_o, cost_o, res_o, grad_o = orc.evaluate(x1, *args, nt=8)
        assert ok and ok_o and abs(cost - cost_o) <= 1e-12 * cost_o
        assert relerr(grad, grad_o) < 1e-10
        if args[0]:
            assert relerr(res, res_o) < 1e-12
        assert np.array_equal(gpu.jacobian_values(), v0)
    rp = s.case.rp
    bad = F.construct(x1, rp.row_cam, rp.row_pt, rp.P, "jacobian_only", s.places["first"])
    ok, _, _, _ = gpu.evaluate(bad, True, True, False)
    assert not ok
    assert np.array_equal(gpu.jacobian_values(), v0)


@pytest.mark.parametrize("problem", ["tiny", "c16", "huge"])
def test_huber(problem, cs, oracle, c16):
    """Under Huber(a) (a = the median row norm) three overflow rows succeed in cost-only and residual-only mode, since
    rho grows linearly, and fail again once set_apply_loss_function(0) turns the loss off.  Jacobian modes fail under
    both losses, as do non-finite residuals."""
    from ceres_solver_b200 import bal as B
    bal = _bal(problem, c16)
    rp = B.ReducedProgram(bal)
    trivial = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())
    s = Setup(cs, oracle, bal, cs.LOSS_HUBER, L.huber_scale(trivial, rp.state(bal)))
    s.name = problem
    try:
        for kind, label, x in s.constructions(("residual_nonfinite", "jacobian_only"), labels=("first", "last")):
            for mode in F.MODES:
                ok = _check_call(cs, s, x, mode, F.expected_ok(kind, mode, huber=True), with_oracle=True)
                if not ok:
                    s.check_healthy(F.MODES[mode])
        s.case.gpu.set_apply_loss_function(0)
        for kind in ("cost_overflow2", "cost_overflow3"):
            x = s.construct(kind, s.overflow[:F.overflow_count(kind)])
            for mode in ("cost", "residuals"):
                _check_call(cs, s, x, mode, F.expected_ok(kind, mode), with_oracle=True, orc=trivial)
        s.case.gpu.set_apply_loss_function(1)
        s.check_healthy(F.MODES["gradient_jacobian"])
    finally:
        s.case.close()


@pytest.mark.parametrize("problem", ["tiny", "c16", "huge"])
def test_observations(problem, cs, oracle, c16):
    """A NaN or -inf observation, given at b200_create, fails every call mode; on `huge` in a row of each class."""
    from ceres_solver_b200 import bal as B
    bal = _bal(problem, c16)
    rp = B.ReducedProgram(bal)
    places = _placements(cs, rp, rp.state(bal))
    labels = ("first", "rows33_128_0", "rows129+_0") if problem == "huge" else ("first", "last")
    for kind in F.OBSERVATION_KINDS:
        for label in labels:
            case = Case(cs, oracle, F.with_observation(bal, rp.obs_of_row, places[label], kind))
            try:
                for mode, args in F.MODES.items():
                    ok, _, _, _ = case.gpu.evaluate(case.state, *args)
                    ok_o, _, _, _ = case.orc.evaluate(case.state, *args, nt=8)
                    assert not ok and not ok_o, (kind, label, mode)
                    assert "non-finite" in _last_error(cs)
            finally:
                case.close()


@pytest.fixture(scope="module")
def tiny(cs, oracle):
    s = Setup(cs, oracle, L.tiny_bal())
    yield s
    s.case.close()


@pytest.mark.parametrize("host_boundary", [False, True])
@pytest.mark.parametrize("kind", ["residual_nonfinite", "jacobian_only"])
def test_lm_from_failing_state(kind, host_boundary, tiny, cs):
    """b200_lm_solve from a state whose evaluation fails raises B200_ERR_EVALUATION_FAILED, as the oracle's solve fails;
    a solve from the healthy state on the same handle then matches the oracle's record by record."""
    s = tiny
    x = s.construct(kind, s.places["first"])
    with pytest.raises(RuntimeError, match="oracle solve failed"):
        L.oracle_solve(s.case.orc, x, max_num_iterations=3)
    with pytest.raises(cs.B200Error) as e:
        L.gpu_solve(s.case.gpu, x, host_boundary, max_num_iterations=3)
    assert e.value.code == cs.binding.ERR_EVALUATION_FAILED
    _, recs_o, _ = L.oracle_solve(s.case.orc, s.case.state, max_num_iterations=3)
    _, recs = L.gpu_solve(s.case.gpu, s.case.state, host_boundary, max_num_iterations=3)
    compare_lm_traces_exact(recs, recs_o)
