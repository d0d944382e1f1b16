"""Every robust loss of include/ceres/loss_function.h, ScaledLoss weights and per-row loss tables
(b200_set_loss_functions) in every evaluate kernel, against the oracle.

The loss and its Corrector are one device function (csrc/loss.cuh) in three instantiations of evaluate_v2_kernel (warp
tiles, points of up to 32 rows, Jacobian wanted) and evaluate_kernel (CTA tiles: every cost-only evaluate, points of
more than 32 rows, every row of the configurations without warp-tile evaluate).  The parameters of each loss come from
the problem's row norms at its initial state (loss_set), so that every branch of every loss runs in every class of rows;
tests/test_oracle_losses.py asserts that on a CPU machine.

  - each loss, and ScaledLoss(Cauchy), on the fixtures of tests/test_gpu_dispatch.py, C16 and the huge-point problem:
    the GPU's loss and Corrector on its own uncorrected rows against the numpy restatement (cost, residuals, Jacobian
    1e-12), and evaluate in every mode against the oracle (cost 1e-12; Jacobian 1e-12, or J_END_TO_END for the losses
    that amplify the last-bit differences of the residuals); every entry point (tests/entry_points.py) on the
    loss-corrected Jacobian for every loss but Tukey on C16 and the huge-point problem, and for SoftLOne and the
    per-observation weights on every fixture;
  - two tables, all seven types mixed over the rows and one ScaledLoss(Cauchy) per observation, on the same fixtures and
    on the circle problem of tests/test_gpu_orders.py, whose points the library reorders;
  - the setter's contract: bit-for-bit equal to the descriptor's trivial and Huber losses, resident residuals dropped,
    apply_loss_function(0), every refusal;
  - SoftLOne and Cauchy cost overflow fails exactly where the oracle fails;
  - LM trajectories on C16 for every loss, Tukey with points whose rows are all outliers, and an annealed Cauchy scale;
  - a 2-rank sharded handle with a table (run as `python -m torch.distributed.run ... tests/test_gpu_losses.py`).
"""
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests import lm_cases as L  # noqa: E402
from tests.entry_points import check_every_entry_point, compare_lm_traces_exact, relerr  # noqa: E402
from tests.test_oracle_losses import LossProgram  # noqa: E402

pytestmark = pytest.mark.gpu

TRIVIAL, HUBER, SOFT_L_ONE, CAUCHY, ARCTAN, TOLERANT, TUKEY = range(7)
LOSSES = ("trivial", "huber", "soft_l_one", "cauchy", "arctan", "tolerant", "tukey", "scaled_cauchy")
TOLERANT_LINEAR_QUANTILE = 0.9   # rows above this quantile of s take Tolerant's x > 36.7 branch
SCALE = 0.37                     # ScaledLoss factor of the scaled variant


# ---------------------------------------------------------------------------------------------------- shared set-up
def squared_norms(orc0, state):
    ok, _, res, _ = orc0.evaluate(state, want_gradient=False, want_jacobian=False, nt=8)
    assert ok
    return res[0::2] ** 2 + res[1::2] ** 2


def loss_set(s):
    """name -> (type, a, b, scale) for a problem whose rows have squared norms s at its initial state: the scale of every
    one-parameter loss is the median row norm m (ArctanLoss, whose a is a value of s, takes m^2); TolerantLoss(a, b) has
    a = m^2 and b such that the rows above the TOLERANT_LINEAR_QUANTILE of s are past x = 36.7."""
    m2 = float(np.median(s))
    m = float(np.sqrt(m2))
    s_hi = float(np.quantile(s, TOLERANT_LINEAR_QUANTILE))
    return {"trivial": (TRIVIAL, 1.0, 1.0, 1.0), "huber": (HUBER, m, 1.0, 1.0), "soft_l_one": (SOFT_L_ONE, m, 1.0, 1.0),
            "cauchy": (CAUCHY, m, 1.0, 1.0), "arctan": (ARCTAN, m2, 1.0, 1.0),
            "tolerant": (TOLERANT, m2, (s_hi - m2) / 36.7, 1.0), "tukey": (TUKEY, m, 1.0, 1.0),
            "scaled_cauchy": (CAUCHY, m, 1.0, SCALE)}


def table(kind, s, seed=0):
    """(losses, obs_loss) of a heterogeneous table over N observations: "mixed", the seven types (two of them scaled,
    ScaledLoss(nullptr, s) among them) drawn per observation; "weights", one ScaledLoss(Cauchy(m)) per observation with a
    weight in [0.25, 4]."""
    rng = np.random.RandomState(seed)
    ls = loss_set(s)
    N = s.size
    if kind == "mixed":
        losses = [ls[k] for k in LOSSES[:7]] + [(TRIVIAL, 1.0, 1.0, 2.5), ls["scaled_cauchy"]]
        return losses, rng.randint(0, len(losses), N).astype(np.int32)
    if kind == "weights":
        m = ls["cauchy"][1]
        w = np.exp(rng.uniform(np.log(0.25), np.log(4.0), N))
        return [(CAUCHY, m, 1.0, float(x)) for x in w], np.arange(N, dtype=np.int32)
    raise KeyError(kind)


class Fixture:
    """One problem on one GPU handle and on the CPU reference (tests/test_oracle_losses.py LossProgram: the oracle's
    program with a table of loss objects), whose losses each test sets on both: the GPU's through
    b200_set_loss_functions with the table index of each row in the problem's row order, the reference's per
    observation."""

    def __init__(self, cs, oracle, bal):
        from ceres_solver_b200 import bal as B
        self.bal = bal
        self.rp = B.ReducedProgram(bal)
        self.state = self.rp.state(bal)
        obs = np.ascontiguousarray(bal.obs).ravel()
        self.orc0 = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, obs)
        self.s_obs = np.empty(bal.N)
        self.s_obs[self.orc0.obs_of_row] = squared_norms(self.orc0, self.state)   # per input observation
        self.losses = loss_set(self.s_obs)
        self.orc = LossProgram(oracle, bal, [self.losses["trivial"]])
        self.gpu = cs.Problem(self.rp.C, self.rp.P, self.rp.row_cam, self.rp.row_pt, self.rp.row_obs)

    def set(self, losses, obs_loss=None):
        self.orc.set_losses(losses, obs_loss)
        self.gpu.set_loss_functions(losses, None if obs_loss is None else obs_loss[self.rp.obs_of_row])

    def close(self):
        self.gpu.close()


def problem_bal(name, c16):
    from tests.test_gpu_dispatch import _bal
    from tests.test_gpu_orders import _make as make_orders
    from tests.test_gpu_parity import huge_bal
    if name == "c16":
        return L.c16_bal(c16)
    if name == "huge":
        return huge_bal()
    if name == "circle":
        return make_orders("circle")
    return _bal(name)


# End-to-end bound on the Jacobian against the oracle.  The GPU's residuals differ from the oracle's in the last bits
# (analytic derivative against autodiff, sincos against sin / cos), and a loss whose weight is steep in s carries that
# difference into its Jacobian rows amplified: Tukey's (1 - s / a^2)^2 near s = a^2, Tolerant's logistic in (s - a) / b
# with b a small fraction of a, Arctan's 1 / (1 + s^2 / a^2).  Measured on the fixtures below: up to 1.4e-11 (Tolerant
# on `tile`).  On identical inputs (check_loss_on_gpu_rows) every loss is held to 1e-12.
J_END_TO_END = {"tolerant": 1e-10, "tukey": 1e-10, "arctan": 1e-10, "mixed": 1e-10}

MODES = {   # (want_residuals, want_gradient, want_jacobian)
    "all": (True, True, True), "cost": (False, False, False), "gradient": (True, True, False),
    "jacobian": (False, False, True),
}


def check_evaluate_modes(fx, jtol=1e-12):
    """Evaluate in every mode against the oracle: cost and residuals 1e-12, Jacobian jtol (J_END_TO_END), gradient 1e-10;
    a gradient-only or cost-only call leaves the stored Jacobian as it is."""
    gpu, orc = fx.gpu, fx.orc
    ok, cost, res, grad = gpu.evaluate(fx.state)
    ok_o, cost_o, res_o, grad_o = orc.evaluate(fx.state, nt=8)
    assert ok and ok_o and abs(cost - cost_o) <= 1e-12 * cost_o, (cost, cost_o)
    assert relerr(res, res_o) < 1e-12 and relerr(grad, grad_o) < 1e-10
    v = gpu.jacobian_values()
    assert relerr(v, orc.jacobian().values()) < jtol
    for mode, (want_r, want_g, want_j) in MODES.items():
        ok, c, r, g = gpu.evaluate(fx.state, want_residuals=want_r, want_gradient=want_g, want_jacobian=want_j)
        assert ok and abs(c - cost_o) <= 1e-12 * cost_o, (mode, c, cost_o)
        if want_r:
            assert relerr(r, res_o) < 1e-12, mode
        if want_g:
            assert relerr(g, grad_o) < 1e-10, mode
        w = gpu.jacobian_values()
        assert (relerr(w, v) < 1e-12) if want_j else np.array_equal(w, v), mode


def check_loss_on_gpu_rows(fx, losses, obs_loss=None):
    """The GPU's loss and Corrector against the numpy restatement (tests/test_oracle_losses.py np_rho_rows, np_correct,
    both checked against the oracle there) applied to the GPU's own uncorrected rows: cost, residuals and Jacobian to
    1e-12, free of the amplification J_END_TO_END allows for."""
    from tests.test_oracle_losses import np_correct, np_rho_rows
    gpu, N = fx.gpu, fx.rp.N
    gpu.set_loss_functions([fx.losses["trivial"]])
    ok, _, r, _ = gpu.evaluate(fx.state, want_gradient=False)
    assert ok
    raw = gpu.jacobian_values()
    fx.set(losses, obs_loss)
    ok, cost, res, _ = gpu.evaluate(fx.state, want_gradient=False)
    assert ok
    v = gpu.jacobian_values()
    idx = np.zeros(N, dtype=np.int64) if obs_loss is None else obs_loss[fx.rp.obs_of_row]
    entries = np.asarray(losses, dtype=float).reshape(-1, 4)[idx]
    r = r.reshape(N, 2)
    rho = np_rho_rows(entries, r[:, 0] ** 2 + r[:, 1] ** 2)
    E, F = raw[:6 * N].reshape(N, 2, 3), raw[6 * N:].reshape(N, 2, 9)
    rc, Ec = np_correct(r, E, rho)
    _, Fc = np_correct(r, F, rho)
    cost_n = 0.5 * float(np.sum(rho[0]))
    assert abs(cost - cost_n) <= 1e-12 * cost_n, (cost, cost_n)
    assert relerr(res, rc.ravel()) < 1e-12
    assert relerr(v, np.concatenate([Ec.ravel(), Fc.ravel()])) < 1e-12


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.fixture(scope="module")
def fixtures(cs, oracle, c16):
    made = {}

    def get(name):
        if name not in made:
            made[name] = Fixture(cs, oracle, problem_bal(name, c16))
        return made[name]
    yield get
    for fx in made.values():
        fx.close()


# ---------------------------------------------------------------------------------------------------- every loss
@pytest.mark.parametrize("loss", LOSSES)
@pytest.mark.parametrize("name", ["id_range", "direct_v3", "v4_narrow", "dups_direct", "dups_id_range", "tile", "c16",
                                  "huge"])
def test_evaluate(name, loss, fixtures):
    fx = fixtures(name)
    check_loss_on_gpu_rows(fx, [fx.losses[loss]])
    check_evaluate_modes(fx, J_END_TO_END.get(loss, 1e-12))


# Tukey is left out: its zeroed rows leave the E'E blocks of points whose rows are all outliers at D^2 alone, and the
# solves on such a system are too ill-conditioned for entry_points' 1e-7 on the solution; test_lm_tukey_outlier_points
# runs them inside the LM loop instead.
@pytest.mark.parametrize("loss", [name for name in LOSSES if name != "tukey"])
@pytest.mark.parametrize("name", ["c16", "huge"])
def test_every_entry_point(name, loss, fixtures, oracle):
    fx = fixtures(name)
    fx.set([fx.losses[loss]])
    check_every_entry_point(fx, oracle, shared_inputs=True)


# (check_every_entry_point holds the Jacobian to 1e-12 end to end: the losses of J_END_TO_END are covered on these
# fixtures by test_evaluate and test_table)
@pytest.mark.parametrize("kind", ["soft_l_one", "weights"])
@pytest.mark.parametrize("name", ["id_range", "direct_v3", "v4_narrow", "dups_direct", "dups_id_range", "tile"])
def test_every_entry_point_dispatch(name, kind, fixtures, oracle):
    fx = fixtures(name)
    if kind == "weights":
        fx.set(*table("weights", fx.s_obs))
    else:
        fx.set([fx.losses[kind]])
    check_every_entry_point(fx, oracle, shared_inputs=True)


# ---------------------------------------------------------------------------------------------------- tables
@pytest.mark.parametrize("kind", ["mixed", "weights"])
@pytest.mark.parametrize("name", ["id_range", "direct_v3", "v4_narrow", "dups_direct", "dups_id_range", "tile", "c16",
                                  "huge", "circle"])
def test_table(name, kind, fixtures):
    fx = fixtures(name)
    losses, obs_loss = table(kind, fx.s_obs, seed=len(name))
    check_loss_on_gpu_rows(fx, losses, obs_loss)
    check_evaluate_modes(fx, J_END_TO_END.get(kind, 1e-12))


def test_table_order_is_the_callers(fixtures, cs):
    """A table whose objects differ only in scale: the row order of row_loss is the problem's (the library permutes it
    with its own point order), so the cost is the oracle's only if every row got its own weight."""
    fx = fixtures("circle")
    N = fx.bal.N
    w = np.arange(1, N + 1, dtype=float)
    fx.set([(TRIVIAL, 1.0, 1.0, float(x)) for x in w], np.arange(N, dtype=np.int32))
    ok, cost, _, _ = fx.gpu.evaluate(fx.state, want_residuals=False, want_gradient=False, want_jacobian=False)
    expect = 0.5 * float(np.dot(w, fx.s_obs))
    assert ok and abs(cost - expect) <= 1e-12 * expect


# ---------------------------------------------------------------------------------------------------- the setter
def _eval_all(gpu, state):
    ok, cost, res, grad = gpu.evaluate(state)
    assert ok
    return cost, res, grad, gpu.jacobian_values()


@pytest.mark.parametrize("name", ["c16", "tile"])
def test_setter_matches_descriptor(name, fixtures, cs):
    """Trivial and Huber(a) with scale 1 through the setter run the descriptor's instantiations: cost, residuals and
    Jacobian are equal to the last bit (the gradient's camera part is a sum of atomics, whose order is not fixed)."""
    fx = fixtures(name)
    a = fx.losses["huber"][1]
    rp = fx.rp
    for loss_type, entry in ((cs.LOSS_TRIVIAL, fx.losses["trivial"]), (cs.LOSS_HUBER, fx.losses["huber"])):
        ref = cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs, loss_type=loss_type, loss_a=a)
        try:
            c0, r0, g0, j0 = _eval_all(ref, fx.state)
            fx.gpu.set_loss_functions([(TUKEY, a, 1.0, 1.0)])   # something else first
            fx.gpu.set_loss_functions([entry])
            c1, r1, g1, j1 = _eval_all(fx.gpu, fx.state)
            assert c0 == c1 and np.array_equal(r0, r1) and np.array_equal(j0, j1), loss_type
            assert relerr(g1, g0) < 1e-14
        finally:
            ref.close()


def test_setter_drops_resident_residuals(fixtures, cs):
    from tests.test_gpu_eval_failure import _assert_no_resident_residuals
    fx = fixtures("c16")
    fx.set([fx.losses["cauchy"]])
    ok, _, res, _ = fx.gpu.evaluate(fx.state)
    assert ok
    D = np.ones(fx.gpu.num_parameters)
    x_resident, _, _ = fx.gpu.schur_solve(None, D)
    x_given, _, _ = fx.gpu.schur_solve(res, D)
    assert relerr(x_resident, x_given) < 1e-9   # (the PCG's products sum with atomics: not to the last bit)
    jac = fx.gpu.jacobian_values()
    fx.gpu.set_loss_functions([fx.losses["tukey"]])
    _assert_no_resident_residuals(cs, fx.gpu)
    assert np.array_equal(fx.gpu.jacobian_values(), jac)   # the stored Jacobian is left as it is
    ok, _, _, _ = fx.gpu.evaluate(fx.state, want_residuals=False, want_gradient=False, want_jacobian=False)
    assert ok
    _assert_no_resident_residuals(cs, fx.gpu)               # a cost-only evaluate produces none
    ok, _, _, _ = fx.gpu.evaluate(fx.state)
    assert ok
    fx.gpu.schur_solve(None, D)


@pytest.mark.parametrize("name", ["c16", "tile"])
def test_apply_loss_function(name, fixtures, cs):
    """apply_loss_function(0) turns off every row's loss, ScaledLoss factors included: the trivial oracle's values.
    (1) restores the table."""
    fx = fixtures(name)
    fx.set(*table("mixed", fx.s_obs, seed=3))
    gpu = fx.gpu
    for apply, orc in ((False, fx.orc0), (True, fx.orc)):
        gpu.set_apply_loss_function(apply)
        ok, cost, res, grad = gpu.evaluate(fx.state)
        ok_o, cost_o, res_o, grad_o = orc.evaluate(fx.state, nt=8)
        assert ok and ok_o and abs(cost - cost_o) <= 1e-12 * cost_o, apply
        assert relerr(res, res_o) < 1e-12 and relerr(grad, grad_o) < 1e-10, apply
        assert relerr(gpu.jacobian_values(), orc.jacobian().values()) < (J_END_TO_END["mixed"] if apply else 1e-12), apply
        ok, cost2, _, _ = gpu.evaluate(fx.state, want_residuals=False, want_gradient=False, want_jacobian=False)
        assert ok and abs(cost2 - cost_o) <= 1e-12 * cost_o, apply


REFUSED = [
    ("type_low", [(-1, 1.0, 1.0, 1.0)], None), ("type_high", [(7, 1.0, 1.0, 1.0)], None),
    ("a_zero", [(CAUCHY, 0.0, 1.0, 1.0)], None), ("a_negative", [(HUBER, -1.0, 1.0, 1.0)], None),
    ("a_nan", [(SOFT_L_ONE, float("nan"), 1.0, 1.0)], None), ("a_inf", [(TUKEY, float("inf"), 1.0, 1.0)], None),
    ("arctan_a_zero", [(ARCTAN, 0.0, 1.0, 1.0)], None),
    ("tolerant_a_negative", [(TOLERANT, -1.0, 1.0, 1.0)], None), ("tolerant_b_zero", [(TOLERANT, 1.0, 0.0, 1.0)], None),
    ("tolerant_b_negative", [(TOLERANT, 1.0, -1.0, 1.0)], None),
    ("tolerant_a_nan", [(TOLERANT, float("nan"), 1.0, 1.0)], None),
    ("tolerant_b_inf", [(TOLERANT, 1.0, float("inf"), 1.0)], None),
    ("scale_zero", [(TRIVIAL, 1.0, 1.0, 0.0)], None), ("scale_negative", [(HUBER, 1.0, 1.0, -2.0)], None),
    ("scale_nan", [(CAUCHY, 1.0, 1.0, float("nan"))], None), ("scale_inf", [(TRIVIAL, 1.0, 1.0, float("inf"))], None),
    ("no_losses", [], None), ("two_losses_no_rows", [(TRIVIAL, 1.0, 1.0, 1.0)] * 2, None),
    ("index_negative", [(TRIVIAL, 1.0, 1.0, 1.0)] * 2, -1), ("index_high", [(TRIVIAL, 1.0, 1.0, 1.0)] * 2, 2),
]


def test_refusals(fixtures, cs):
    """Each refused table returns B200_ERR_INVALID_ARGUMENT and leaves the handle as it was: same losses, resident
    residuals still there."""
    import ctypes as C
    fx = fixtures("c16")
    fx.set([fx.losses["huber"]])
    gpu = fx.gpu
    ok, cost, res, _ = gpu.evaluate(fx.state)
    assert ok
    D = np.ones(gpu.num_parameters)
    x0, _, _ = gpu.schur_solve(None, D)
    for label, losses, bad in REFUSED:
        tab = (cs.Loss * max(1, len(losses)))(*[cs.Loss(int(t), a, b, s) for t, a, b, s in losses])
        rows = None
        if bad is not None:
            rows = np.zeros(gpu.N, dtype=np.int32)
            rows[gpu.N // 2] = bad
        rc = cs.lib().b200_set_loss_functions(gpu.h, tab, len(losses),
                                              None if rows is None else rows.ctypes.data_as(C.POINTER(C.c_int32)))
        assert rc == cs.binding.ERR_INVALID_ARGUMENT, label
        x, _, _ = gpu.schur_solve(None, D)   # the resident residuals are still there
        assert relerr(x, x0) < 1e-7, label   # (a PCG solve: its products sum with atomics)
    ok, cost2, _, _ = gpu.evaluate(fx.state)
    assert ok and cost2 == cost
    assert cs.lib().b200_set_loss_functions(None, tab, 1, None) == cs.binding.ERR_INVALID_ARGUMENT
    assert cs.lib().b200_set_loss_functions(gpu.h, None, 1, None) == cs.binding.ERR_INVALID_ARGUMENT


@pytest.mark.parametrize("loss_type", [-1, 2, 3, 6, 7])
def test_create_refuses_other_losses(loss_type, fixtures, cs):
    rp = fixtures("c16").rp
    with pytest.raises(cs.B200Error) as e:
        cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs, loss_type=loss_type)
    assert e.value.code == cs.binding.ERR_INVALID_ARGUMENT


# ---------------------------------------------------------------------------------------------------- failures
def overflow_scale(s, factor):
    """a of SoftLOne / Cauchy such that s * (1 / a^2) overflows for the largest row at factor < 1 and for none at
    factor > 1: a^2 = factor * max(s) / DBL_MAX."""
    return float(np.sqrt(factor * np.max(s) / np.finfo(np.float64).max))


@pytest.mark.parametrize("loss", [SOFT_L_ONE, CAUCHY])
@pytest.mark.parametrize("name", ["c16", "tile", "huge"])
def test_cost_overflow(name, loss, fixtures, cs):
    """SoftLOne(a) and Cauchy(a) with 1 / a^2 so large that s / a^2 overflows on the largest row: rho = inf there, the cost
    is not finite and the evaluation fails in every mode, on GPU and oracle alike; a factor of 4 less and every mode
    succeeds.  After a failed call with residuals there are no resident residuals."""
    from tests.test_gpu_eval_failure import _assert_no_resident_residuals
    fx = fixtures(name)
    for factor, expect in ((0.5, False), (2.0, True)):
        fx.set([(loss, overflow_scale(fx.s_obs, factor), 1.0, 1.0)])
        for mode, (want_r, want_g, want_j) in MODES.items():
            ok_o, cost_o, _, _ = fx.orc.evaluate(fx.state, want_r, want_g, want_j, nt=8)
            ok, cost, _, _ = fx.gpu.evaluate(fx.state, want_residuals=want_r, want_gradient=want_g, want_jacobian=want_j)
            assert ok == ok_o == expect, (factor, mode, ok, ok_o)
            if ok:
                assert abs(cost - cost_o) <= 1e-12 * cost_o
            elif want_r:
                _assert_no_resident_residuals(cs, fx.gpu)


# ---------------------------------------------------------------------------------------------------- LM
@pytest.mark.parametrize("host_boundary", [False, True])
@pytest.mark.parametrize("loss", LOSSES)
def test_lm_trajectory_c16(loss, host_boundary, fixtures):
    fx = fixtures("c16")
    fx.set([fx.losses[loss]])
    state_o, recs_o, _ = L.oracle_solve(fx.orc, fx.state, max_num_iterations=5)
    state, recs = L.gpu_solve(fx.gpu, fx.state, host_boundary, max_num_iterations=5)
    compare_lm_traces_exact(recs, recs_o)
    assert relerr(state, state_o) < 1e-9


def tukey_outlier_points_bal(c16, count=5, shift=50.0):
    """C16 with every observation of `count` points moved by `shift` median row norms: under TukeyLoss(median norm) all
    their rows are outliers, with rho' = 0, so those points' rows and Jacobian blocks are zero."""
    from ceres_solver_b200 import bal as B
    bal = L.c16_bal(c16)
    rp = B.ReducedProgram(bal)
    res = B.snavely_project(bal.cameras, bal.points, bal.cam_idx, bal.pt_idx) - bal.obs
    m = float(np.median(np.hypot(res[:, 0], res[:, 1])))
    points = rp.point_of_eblock[:: max(1, rp.P // count)][:count]
    obs = np.array(bal.obs, dtype=float, copy=True)
    rows = np.isin(bal.pt_idx, points)
    obs[rows] += shift * m
    return B.Bal(bal.cam_idx, bal.pt_idx, obs, bal.cameras, bal.points), rows


@pytest.mark.parametrize("solver", ["iterative", "sparse"])
def test_lm_tukey_outlier_points(solver, cs, oracle, c16):
    """Five LM iterations with points whose Jacobian blocks are zero (their E'E blocks are D^2 alone).  The trajectory is
    held to the oracle's own spread between thread counts (tests/conftest.py compare_lm_traces) on every relative field:
    the near-singular blocks make the step quality move by ~1e-9 between summation orders, past
    compare_lm_traces_exact's bound."""
    from tests.conftest import compare_lm_traces
    from tests.entry_points import RELATIVE_FIELDS
    bal, rows = tukey_outlier_points_bal(c16)
    fx = Fixture(cs, oracle, bal)
    try:
        a = fx.losses["tukey"][1]
        assert fx.s_obs[rows].min() > a * a       # every row of the moved points is an outlier
        fx.set([fx.losses["tukey"]])
        ok, _, res, _ = fx.gpu.evaluate(fx.state)
        assert ok and not res.reshape(-1, 2)[rows[fx.rp.obs_of_row]].any()
        kind = cs.ITERATIVE_SCHUR if solver == "iterative" else cs.SPARSE_SCHUR
        # the oracle has no SPARSE_SCHUR: its exact solve is DENSE_SCHUR, which SPARSE_SCHUR matches to rounding
        oracle_kind = L.ITERATIVE_SCHUR if solver == "iterative" else L.DENSE_SCHUR
        traces = [L.oracle_solve(fx.orc, fx.state, nt=nt, max_num_iterations=5, linear_solver_type=oracle_kind)[1]
                  for nt in (8, 3)]
        for host_boundary in (False, True):
            _, recs = L.gpu_solve(fx.gpu, fx.state, host_boundary, max_num_iterations=5, linear_solver_type=kind)
            assert len(recs) == len(traces[0]) == 6
            compare_lm_traces(recs, *traces, keys=RELATIVE_FIELDS)
    finally:
        fx.close()


def test_lm_annealing(fixtures):
    """Cauchy(4a) for three iterations, then Cauchy(a) from the state reached, on one handle (LossFunctionWrapper::Reset
    between two solves), against the oracle doing the same."""
    fx = fixtures("c16")
    t, a, b, s = fx.losses["cauchy"]
    state_o, state = fx.state, fx.state
    for scale_a, iterations in ((4.0 * a, 3), (a, 4)):
        fx.set([(t, scale_a, b, s)])
        state_o, recs_o, _ = L.oracle_solve(fx.orc, state_o, max_num_iterations=iterations)
        state, recs = L.gpu_solve(fx.gpu, state, False, max_num_iterations=iterations)
        compare_lm_traces_exact(recs, recs_o)
        assert relerr(state, state_o) < 1e-9


# ---------------------------------------------------------------------------------------------------- sharded
def _free_port():
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        return sk.getsockname()[1]


def test_sharded_table():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs, %d visible" % torch.cuda.device_count())
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.abspath(__file__)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0 and "LOSSES-SHARDED-OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])


def _sharded_worker():
    """One rank of test_sharded_table: the rows of its point shard with their entries of the "mixed" table; cost and
    gradient against the oracle's over the whole problem."""
    import torch
    import torch.distributed as dist
    import ceres_solver_b200 as cs
    from ceres_solver_b200 import bal as B
    from oracle import pyoracle as po

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    idt = torch.zeros(128, dtype=torch.uint8, device="cuda")
    if rank == 0:
        idt.copy_(torch.frombuffer(bytearray(cs.nccl_unique_id()), dtype=torch.uint8))
    dist.broadcast(idt, 0)
    nccl_id = bytes(idt.cpu().numpy().tobytes())
    bal = B.synthetic("trafalgar-257")
    rp = B.ReducedProgram(bal)
    full = rp.state(bal)
    po.build()
    obs = np.ascontiguousarray(bal.obs).ravel()
    orc0 = po.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, obs)
    s_obs = np.empty(bal.N)
    s_obs[orc0.obs_of_row] = squared_norms(orc0, full)
    losses, obs_loss = table("mixed", s_obs, seed=5)
    orc = LossProgram(po, bal, losses, obs_loss)
    ok_o, cost_o, _, grad_o = orc.evaluate(full, want_residuals=False, nt=8)
    plo, phi, rlo, rhi = rp.shard(rank, world)
    gpu = cs.Problem(rp.C, phi - plo, rp.row_cam[rlo:rhi], rp.row_pt[rlo:rhi] - plo, rp.row_obs[rlo:rhi], device=local,
                     rank=rank, world_size=world, nccl_id=nccl_id)
    gpu.set_loss_functions(losses, obs_loss[rp.obs_of_row][rlo:rhi])
    state = np.concatenate([full[3 * plo:3 * phi], full[3 * rp.P:]])
    ok, cost, _, grad = gpu.evaluate(state, want_residuals=False)
    assert ok and ok_o and abs(cost - cost_o) <= 1e-12 * cost_o, (cost, cost_o)
    nP = 3 * (phi - plo)
    assert relerr(grad[:nP], grad_o[3 * plo:3 * phi]) < 1e-10
    assert relerr(grad[nP:], grad_o[3 * rp.P:]) < 1e-10
    gpu.close()
    dist.barrier()
    if rank == 0:
        print("LOSSES-SHARDED-OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    _sharded_worker()
