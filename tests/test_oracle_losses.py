"""The CPU reference of the robust losses that tests/test_gpu_losses.py checks the library against, on a CPU machine.

The oracle (oracle/bal.h) restates HuberLoss and the Corrector.  tests/loss_oracle.cc restates the other classes of
include/ceres/loss_function.h and ScaledLoss next to them, and LossProgram below applies a table of loss objects to the
oracle's own program (trivial loss) row by row, as ResidualBlock::Evaluate does, with the oracle's Jacobian products and
linear solves and the trust-region loop of tests/dogleg_reference.py running LevenbergMarquardtStrategy.  Checked here:
the values loss_function.h documents at s = 0, finite differences of rho' and rho'' in every region, the branch points,
ScaledLoss, an independent numpy restatement, LossProgram with HuberLoss against the oracle's own Huber evaluation and
LM transcript, the parameters of tests/test_gpu_losses.py doing on each fixture what those tests rely on, and the
layout of b200_loss in C against its ctypes mirror."""
import atexit
import ctypes
import math
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from tests import lm_cases as L

TRIVIAL, HUBER, SOFT_L_ONE, CAUCHY, ARCTAN, TOLERANT, TUKEY = range(7)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def np_rho(type_, a, b, scale, s):
    """{rho, rho', rho''} of a loss object, restated in numpy from loss_function.h's formulas (vectorised in s)."""
    s = np.asarray(s, dtype=float)
    tiny = np.finfo(np.float64).tiny
    if type_ == HUBER:
        out = s > a * a
        r = np.sqrt(np.where(out, s, 1.0))
        r1 = np.where(out, np.maximum(tiny, a / r), 1.0)
        rho = (np.where(out, 2.0 * a * r - a * a, s), r1, np.where(out, -r1 / (2.0 * np.where(out, s, 1.0)), 0.0))
    elif type_ in (SOFT_L_ONE, CAUCHY):
        c = 1.0 / (a * a)
        q = 1.0 + s * c
        if type_ == SOFT_L_ONE:
            r1 = np.maximum(tiny, 1.0 / np.sqrt(q))
            rho = (2.0 * (a * a) * (np.sqrt(q) - 1.0), r1, -(c * r1) / (2.0 * q))
        else:
            rho = (a * a * np.log(q), np.maximum(tiny, 1.0 / q), -c * (1.0 / q) ** 2)
    elif type_ == ARCTAN:
        c = 1.0 / (a * a)
        iq = 1.0 / (1.0 + s * s * c)
        rho = (a * np.arctan2(s, a), np.maximum(tiny, iq), -2.0 * s * c * iq * iq)
    elif type_ == TOLERANT:
        c0 = b * np.log(1.0 + np.exp(-a / b))
        x = (s - a) / b
        lin = x > 36.7
        xe = np.where(lin, 0.0, x)
        e = np.exp(xe)
        rho = (np.where(lin, s - a - c0, b * np.log(1.0 + e) - c0), np.where(lin, 1.0, np.maximum(tiny, e / (1.0 + e))),
               np.where(lin, 0.0, 0.5 / (b * (1.0 + np.cosh(xe)))))
    elif type_ == TUKEY:
        a2 = a * a
        inl = s <= a2
        t = 1.0 - s / a2
        rho = (np.where(inl, a2 / 3.0 * (1.0 - t * t * t), a2 / 3.0), np.where(inl, t * t, 0.0),
               np.where(inl, -2.0 / a2 * t, 0.0))
    else:
        rho = (s, np.ones_like(s), np.zeros_like(s))
    return tuple(scale * np.asarray(v, dtype=float) for v in rho)


def np_correct(r, J, rho):
    """The Corrector (corrector.cc) in numpy, per row: r [n, 2] residuals, J [n, 2, k] Jacobian rows, rho three [n] arrays.
    Returns the corrected copies."""
    s = r[:, 0] ** 2 + r[:, 1] ** 2
    sqrt_rho1 = np.sqrt(rho[1])
    second = (s > 0.0) & (rho[2] > 0.0)
    ss = np.where(second, s, 1.0)
    alpha = np.where(second, 1.0 - np.sqrt(np.where(second, 1.0 + 2.0 * ss * rho[2] / np.where(second, rho[1], 1.0), 1.0)), 0.0)
    scaling = np.where(second, sqrt_rho1 / (1.0 - alpha), sqrt_rho1)
    alpha_sq = np.where(second, alpha / ss, 0.0)
    rtj = np.einsum("ni,nik->nk", r, J)
    Jc = sqrt_rho1[:, None, None] * (J - alpha_sq[:, None, None] * r[:, :, None] * rtj[:, None, :])
    return r * scaling[:, None], Jc


def np_rho_rows(entries, s):
    """rho of each row, entries[i] = (type, a, b, scale) of row i (grouped by type, vectorised within a type)."""
    e = np.asarray(entries, dtype=float).reshape(-1, 4)
    out = [np.zeros_like(s) for _ in range(3)]
    types = e[:, 0].astype(int)
    for t in np.unique(types):
        k = types == t
        part = np_rho(int(t), e[k, 1], e[k, 2], e[k, 3], s[k])
        for j in range(3):
            out[j][k] = part[j]
    return out


# ---------------------------------------------------------------------------------------------------- the reference
_ref = None


class _Reference:
    """ctypes binding of tests/loss_oracle.cc, built with the oracle's compiler flags into a temporary directory."""

    def __init__(self):
        tmp = tempfile.mkdtemp(prefix="loss_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        path = os.path.join(tmp, "libloss_oracle.so")
        subprocess.check_call(["g++", "-O3", "-march=native", "-std=c++17", "-fPIC", "-shared", "-pthread", "-o", path,
                               os.path.join(ROOT, "tests", "loss_oracle.cc")])
        self.lib = ctypes.CDLL(path)

    def loss(self, type_, a, s, b=1.0, scale=1.0):
        """{rho(s), rho'(s), rho''(s)} of the loss object (type_, a, b) wrapped in ScaledLoss(scale)."""
        rho = np.zeros(3)
        d = ctypes.c_double
        self.lib.loss_rho(int(type_), d(a), d(b), d(scale), d(s), rho.ctypes.data_as(ctypes.POINTER(d)))
        return rho

    def rows(self, types, params, r, E, F):
        """loss_rows: the cost of each row; r, E and F (contiguous float64, E / F may be None) corrected in place."""
        n = types.size
        cost = np.zeros(n)
        dp = ctypes.POINTER(ctypes.c_double)
        ptr = (lambda a: None if a is None else a.ctypes.data_as(dp))
        self.lib.loss_rows(n, types.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), ptr(params), ptr(r), ptr(E), ptr(F),
                           ptr(cost))
        return cost


def reference():
    global _ref
    if _ref is None:
        _ref = _Reference()
    return _ref


@pytest.fixture(scope="module")
def ref():
    return reference()


class LevenbergMarquardtStrategy:
    """LevenbergMarquardtStrategy (levenberg_marquardt_strategy.cc:69-171) as oracle/bal.h Minimize runs it, in the
    interface of tests/dogleg_reference.py's DoglegStrategy: the LM diagonal from the scaled Jacobian's column norms
    (kept after a rejected or invalid step), the oracle's ITERATIVE_SCHUR or DENSE_SCHUR solve of min |J x - r|^2 +
    |D x|^2 with D = sqrt(diagonal / radius), and the radius updates."""

    def __init__(self, o, nt):
        self.o, self.nt = o, nt
        self.radius = o.initial_trust_region_radius
        self.decrease_factor, self.reuse_diagonal, self.diagonal = 2.0, False, None
        self.num_solves, self.branch, self.thresholds = 1, None, {}

    def compute_step(self, ops, residuals):
        o = self.o
        if not self.reuse_diagonal:
            self.diagonal = np.clip(ops.J.squared_column_norm(nt=self.nt), o.min_lm_diagonal, o.max_lm_diagonal)
        D = np.sqrt(self.diagonal / self.radius)
        x, its, term = ops.J.linear_solve(ops.num_elim, residuals, D, solver=o.linear_solver, preconditioner=o.preconditioner,
                                          min_iter=o.min_linear_solver_iterations, max_iter=o.max_linear_solver_iterations,
                                          q_tolerance=o.eta, r_tolerance=-1.0, nt=self.nt)
        self.reuse_diagonal = True
        if term != 2 and not np.isfinite(x).all():
            term = 2   # LS_FAILURE
        return -x, its, term

    def step_accepted(self, quality):
        self.radius = min(self.o.max_trust_region_radius, self.radius / max(1.0 / 3.0, 1.0 - (2.0 * quality - 1.0) ** 3))
        self.decrease_factor, self.reuse_diagonal = 2.0, False

    def step_rejected(self):
        self.radius /= self.decrease_factor
        self.decrease_factor *= 2.0
        self.reuse_diagonal = True

    step_is_invalid = step_rejected


class LossProgram:
    """The oracle's program of a BAL problem (trivial loss) with a table of loss objects: losses = (type, a, b, scale)
    tuples, obs_loss[i] the object of input observation i (None: losses[0] for every row).  Same interface as the
    oracle's BaProgram (evaluate, jacobian, default_options, solve), so tests/lm_cases.py drives either."""

    def __init__(self, oracle, bal, losses, obs_loss=None):
        self.base = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())
        b = self.base
        self.C, self.P, self.N = b.C, b.P, b.N
        self.obs_of_row, self.row_pt, self.row_cam = b.obs_of_row, b.row_pt, b.row_cam
        self.num_parameters, self.num_residuals = b.num_parameters, b.num_residuals
        self.set_losses(losses, obs_loss)

    def set_losses(self, losses, obs_loss=None):
        """Replaces the loss objects (as LossFunctionWrapper::Reset does between solves)."""
        table = np.asarray(losses, dtype=float).reshape(-1, 4)
        idx = np.zeros(self.N, dtype=np.int64) if obs_loss is None else np.asarray(obs_loss)[self.obs_of_row]
        self.types = np.ascontiguousarray(table[idx, 0], dtype=np.int32)
        self.params = np.ascontiguousarray(table[idx, 1:])

    def evaluate(self, state, want_residuals=True, want_gradient=True, want_jacobian=True, nt=1):
        """ProgramEvaluator::Evaluate with the losses: the base program evaluates each row (failing on a non-finite
        residual, or Jacobian entry when J is computed), then each row's loss and Corrector, then the cost's finiteness.
        The gradient is J'r of the corrected J and r.  With want_jacobian false the stored Jacobian is left as it was."""
        need_j = want_gradient or want_jacobian
        J = self.base.jacobian()
        kept = J.values() if need_j and not want_jacobian else None
        ok, cost, r, _ = self.base.evaluate(state, want_residuals=True, want_gradient=False, want_jacobian=need_j, nt=nt)
        # the base program returns false with the cost untouched (0) when a row failed, and with a non-finite cost when
        # only its trivial sum overflowed, which is no failure under a loss that sums its own cost
        if not ok and np.isfinite(cost):
            return False, float("nan"), None, None
        v = J.values() if need_j else None
        n6 = 6 * self.N
        E, F = (v[:n6].copy(), v[n6:].copy()) if need_j else (None, None)
        total = math.fsum(reference().rows(self.types, self.params, r, E, F))   # (correctly rounded: no summation order)
        if not np.isfinite(total):
            return False, total, None, None
        grad = None
        if need_j:
            J.set_values(np.concatenate([E, F]))
            if want_gradient:
                grad = J.left_multiply(r, nt=nt)
        if kept is not None:
            J.set_values(kept)
        return True, total, r if want_residuals else None, grad

    def jacobian(self):
        return self.base.jacobian()

    def default_options(self):
        return self.base.default_options()

    def solve(self, state, options=None):
        """TrustRegionMinimizer::Minimize with LevenbergMarquardtStrategy on this program (tests/dogleg_reference.py's
        loop, whose strategy class is looked up when it runs).  Returns (best state, records, {})."""
        from tests import dogleg_reference as R
        o = options or self.default_options()
        names = ("max_num_iterations", "initial_trust_region_radius", "min_trust_region_radius", "min_relative_decrease",
                 "min_lm_diagonal", "max_lm_diagonal", "function_tolerance", "gradient_tolerance", "parameter_tolerance",
                 "jacobi_scaling", "max_num_consecutive_invalid_steps")
        saved = R.DoglegStrategy
        R.DoglegStrategy = lambda *args: LevenbergMarquardtStrategy(o, o.num_threads)
        try:
            best, recs, _ = R.minimize(self, state, None, nt=o.num_threads, **{k: getattr(o, k) for k in names})
        finally:
            R.DoglegStrategy = saved
        return best, recs, {}


ONE_PARAMETER = [(HUBER, 1.3), (SOFT_L_ONE, 0.7), (CAUCHY, 2.0), (ARCTAN, 1.5), (TUKEY, 1.1)]
ONE_PARAMETER_B = [(t, a, 1.0) for t, a in ONE_PARAMETER] + [(TOLERANT, 3.0, 0.4)]   # (type, a, b)


def test_values_at_zero(ref, oracle):
    """The rho(0), rho'(0), rho''(0) loss_function.h documents for each class."""
    for a in (0.5, 1.0, 3.0):
        assert list(ref.loss(TRIVIAL, a, 0.0)) == [0.0, 1.0, 0.0]
        assert list(ref.loss(HUBER, a, 0.0)) == [0.0, 1.0, 0.0]
        assert list(ref.loss(SOFT_L_ONE, a, 0.0)) == pytest.approx([0.0, 1.0, -1.0 / (2.0 * a * a)], rel=1e-15)
        assert list(ref.loss(CAUCHY, a, 0.0)) == pytest.approx([0.0, 1.0, -1.0 / (a * a)], rel=1e-15)
        assert list(ref.loss(ARCTAN, a, 0.0)) == [0.0, 1.0, 0.0]
        assert list(ref.loss(TUKEY, a, 0.0)) == pytest.approx([0.0, 1.0, -2.0 / (a * a)], rel=1e-15)
    # TolerantLoss(a, b): rho(0) = 0 (c is rho's value at 0, up to a rounding); rho'(0), rho''(0) ~ 0 for a >> b
    for a, b in ((1.0, 0.5), (20.0, 1.0), (0.0, 2.0), (3.0, 0.4)):
        rho = ref.loss(TOLERANT, a, 0.0, b=b)
        assert abs(rho[0]) <= 1e-15 * b * np.log1p(np.exp(-a / b))
        assert rho[1] == pytest.approx(1.0 / (1.0 + np.exp(a / b)), rel=1e-14)
    rho = ref.loss(TOLERANT, 40.0, 0.0, b=1.0)
    assert rho[1] < 1e-17 and 0.0 < rho[2] < 1e-17


def _s_grid(type_, a, b):
    """Points of s in every region of a loss (away from its branch points)."""
    if type_ in (HUBER, TUKEY):
        return np.concatenate([np.linspace(0.05, 0.95, 7) * a * a, np.linspace(1.05, 6.0, 7) * a * a])
    if type_ == TOLERANT:
        return np.concatenate([a + b * np.array([-8.0, -2.0, -0.5, 0.0, 0.5, 2.0, 10.0, 30.0]),
                               a + b * np.array([37.0, 40.0, 60.0])])
    return np.array([1e-3, 0.1, 0.5, 1.0, 2.0, 10.0, 100.0]) * max(a * a, a)


@pytest.mark.parametrize("type_,a,b", ONE_PARAMETER_B)
def test_finite_differences(ref, oracle, type_, a, b):
    """rho' and rho'' against central differences of rho and rho' in each region."""
    for s in _s_grid(type_, a, b):
        h = 1e-5 * max(1.0, s)
        lo, hi, mid = ref.loss(type_, a, s - h, b=b), ref.loss(type_, a, s + h, b=b), ref.loss(type_, a, s, b=b)
        d0, d1 = (hi[0] - lo[0]) / (2.0 * h), (hi[1] - lo[1]) / (2.0 * h)
        scale0 = max(abs(mid[1]), 1e-300)
        assert abs(d0 - mid[1]) <= 1e-6 * max(scale0, abs(mid[0]) / max(s, 1.0)), (type_, s, d0, mid)
        assert abs(d1 - mid[2]) <= 1e-5 * max(abs(mid[2]), abs(mid[1]) / max(s, 1.0), 1e-12), (type_, s, d1, mid)


def test_tolerant_branch_point(ref, oracle):
    """TolerantLoss is continuous across x = (s - a) / b = 36.7, where it switches to rho = s - a - c."""
    for a, b in ((3.0, 0.4), (0.0, 1.0), (100.0, 7.0)):
        s0 = a + 36.7 * b
        below = ref.loss(TOLERANT, a, s0 * (1.0 - 1e-12), b=b)
        above = ref.loss(TOLERANT, a, s0 * (1.0 + 1e-12), b=b)
        assert abs(above[0] - below[0]) <= 1e-10 * abs(below[0])
        assert abs(above[1] - below[1]) <= 1e-14 and above[2] == 0.0 and 0.0 < below[2] < 1e-15 / b
        # rho(0) = b log(1 + e^(-a/b)) - c = 0 up to the rounding of the fused multiply-add the compiler may form
        assert abs(ref.loss(TOLERANT, a, 0.0, b=b)[0]) <= 1e-15 * b * np.log1p(np.exp(-a / b))


def test_tukey_boundary(ref, oracle):
    """TukeyLoss at s = a^2: rho = a^2 / 3 from both sides, rho' = rho'' = 0, and constant beyond (rho' = 0: the Corrector
    zeroes the row)."""
    for a in (0.5, 1.1, 4.0):
        a2 = a * a
        at = ref.loss(TUKEY, a, a2)
        assert at[0] == pytest.approx(a2 / 3.0, rel=1e-15) and at[1] == 0.0 and at[2] == 0.0
        inside = ref.loss(TUKEY, a, a2 * (1.0 - 1e-9))
        assert inside[1] > 0.0 and inside[0] == pytest.approx(a2 / 3.0, rel=1e-12)
        for s in (a2 * (1.0 + 1e-12), 2.0 * a2, 1e6 * a2):
            assert list(ref.loss(TUKEY, a, s)) == [a2 / 3.0, 0.0, 0.0]
        r, J = oracle.corrector(2.0 * a2, ref.loss(TUKEY, a, 2.0 * a2), np.array([1.0, -2.0]), np.ones(6))
        assert not r.any() and not J.any()


@pytest.mark.parametrize("type_,a,b", ONE_PARAMETER_B + [(TRIVIAL, 1.0, 1.0)])
def test_scaled_loss(ref, oracle, type_, a, b):
    """ScaledLoss(rho, k) is k rho in all three components; ScaledLoss(nullptr, k) is {k s, k, 0}."""
    for s in _s_grid(type_, a, b):
        base = ref.loss(type_, a, s, b=b)
        for k in (0.25, 3.0):
            assert np.array_equal(ref.loss(type_, a, s, b=b, scale=k), k * base)
    assert list(ref.loss(TRIVIAL, 1.0, 2.0, scale=0.5)) == [1.0, 0.5, 0.0]


@pytest.mark.parametrize("type_,a,b", ONE_PARAMETER_B + [(TRIVIAL, 1.0, 1.0), (TOLERANT, 0.0, 2.0)])
def test_numpy_restatement(ref, oracle, type_, a, b):
    """The oracle against np_rho to 1e-15 relative; Tolerant's rho, a difference of two terms of size c near s = 0, to
    1e-15 of c."""
    for scale in (1.0, 0.37):
        s = np.concatenate([[0.0], _s_grid(type_, a, b)])
        want = np_rho(type_, a, b, scale, s)
        c = scale * b * np.log1p(np.exp(-a / b)) if type_ == TOLERANT else 0.0
        for i, si in enumerate(s):
            got = ref.loss(type_, a, si, b=b, scale=scale)
            for k in range(3):
                floor = c if k == 0 else 1e-300
                assert abs(got[k] - want[k][i]) <= 1e-15 * max(abs(want[k][i]), floor), (type_, si, k, got, want[k][i])


def test_huber_against_the_oracle(oracle, c16):
    """LossProgram with one HuberLoss (and with the trivial loss) against the oracle's own evaluation and LM transcript of
    the same problem: cost, residuals, gradient and Jacobian, and every field of every record of five LM iterations under
    ITERATIVE_SCHUR and DENSE_SCHUR."""
    from ceres_solver_b200 import bal as B
    from tests.entry_points import compare_lm_traces_exact, relerr
    for name, bal in (("tiny", L.tiny_bal()), ("c16", L.c16_bal(c16))):
        state = B.ReducedProgram(bal).state(bal)
        obs = np.ascontiguousarray(bal.obs).ravel()
        orc0 = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, obs)
        a = L.huber_scale(orc0, state)
        for use_huber, entry in ((False, (TRIVIAL, 1.0, 1.0, 1.0)), (True, (HUBER, a, 1.0, 1.0))):
            orc = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, obs, use_huber=use_huber, huber_a=a)
            lp = LossProgram(oracle, bal, [entry])
            ok, cost, res, grad = lp.evaluate(state, nt=8)
            ok_o, cost_o, res_o, grad_o = orc.evaluate(state, nt=8)
            assert ok and ok_o and abs(cost - cost_o) <= 1e-14 * cost_o
            assert relerr(res, res_o) < 1e-15 and relerr(grad, grad_o) < 1e-13
            assert relerr(lp.jacobian().values(), orc.jacobian().values()) < 1e-15
            if name == "tiny":
                continue   # tiny converges in four iterations, to cost changes at the rounding level of its cost
            # one thread: threaded, the Schur elimination adds into shared blocks in lock order, and the distance of
            # the two programs' DENSE_SCHUR solutions moves from run to run across the bound on x below
            for solver in (L.ITERATIVE_SCHUR, L.DENSE_SCHUR):
                x_o, recs_o, _ = L.oracle_solve(orc, state, nt=1, max_num_iterations=5, linear_solver_type=solver)
                x, recs, _ = L.oracle_solve(lp, state, nt=1, max_num_iterations=5, linear_solver_type=solver)
                compare_lm_traces_exact(recs, recs_o)
                assert relerr(x, x_o) < 1e-12


def test_numpy_corrector(ref, oracle):
    """np_correct against the oracle's Corrector on both of its branches (Tolerant's rho'' > 0, Cauchy's < 0) and at s = 0."""
    rng = np.random.RandomState(1)
    for type_, a, b in ((TOLERANT, 3.0, 0.4), (CAUCHY, 2.0, 1.0), (TUKEY, 1.1, 1.0)):
        for scale_r in (0.0, 0.3, 1.0, 3.0):
            r = rng.randn(2) * scale_r
            J = rng.randn(2, 9)
            s = float(r @ r)
            rho = ref.loss(type_, a, s, b=b)
            r_o, J_o = oracle.corrector(s, rho, r, J)
            r_n, J_n = np_correct(r[None], J[None], [np.array([v]) for v in rho])
            assert np.allclose(r_n[0], r_o, rtol=1e-14, atol=0) and np.allclose(J_n[0], J_o.reshape(2, 9), rtol=1e-13, atol=1e-300)


# ---------------------------------------------------------------------------------------------------- GPU fixtures
def _branches(s, losses):
    """{loss: (rows in the first region, rows in the second)} of the branched losses at squared norms s."""
    _, a_h, _, _ = losses["huber"]
    _, a_t, b_t, _ = losses["tolerant"]
    _, a_k, _, _ = losses["tukey"]
    x = (s - a_t) / b_t
    rho2 = np_rho(TOLERANT, a_t, b_t, 1.0, s)[2]
    return {"huber": (int((s <= a_h * a_h).sum()), int((s > a_h * a_h).sum())),
            "tolerant": (int((x <= 36.7).sum()), int((x > 36.7).sum())),
            "tolerant_second_order": (int(((rho2 > 0.0) & (s > 0.0)).sum()), int(((rho2 <= 0.0) | (s == 0.0)).sum())),
            "tukey": (int((s <= a_k * a_k).sum()), int((s > a_k * a_k).sum()))}


def test_branches_on_gpu_fixtures(oracle, c16):
    """With the parameters of tests/test_gpu_losses.py, every branch of every branched loss (Huber and Tukey in / out,
    Tolerant's log and linear pieces, and the Corrector's second-order branch, which Tolerant's rows below x = 36.7 take)
    has rows in every class of rows (points of <= 32, 33..128, > 128 rows) of every fixture."""
    from ceres_solver_b200 import bal as B
    from tests.test_gpu_dispatch import EXPECT, _bal
    from tests.test_gpu_losses import loss_set, squared_norms
    from tests.test_gpu_parity import huge_bal
    problems = {name: _bal(name) for name in EXPECT}
    problems["huge"] = huge_bal()
    problems["c16"] = L.c16_bal(c16)
    for name, bal in problems.items():
        orc = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())
        s = squared_norms(orc, B.ReducedProgram(bal).state(bal))
        losses = loss_set(s)
        degree = np.bincount(orc.row_pt)[orc.row_pt]
        classes = 0
        for lo, hi in L.ROW_CLASSES:
            rows = (degree >= lo) & (degree <= hi)
            if rows.any():
                classes += 1
                for loss, (first, second) in _branches(s[rows], losses).items():
                    if loss == "tolerant_second_order":
                        assert first > 0, (name, lo, loss)
                    else:
                        assert first > 0 and second > 0, (name, lo, loss, first, second)
        if name in ("id_range", "tile", "huge"):
            assert classes == 3, name


def test_overflow_construction(oracle, c16):
    """The SoftLOne / Cauchy scale of test_cost_overflow: a^2 = 0.5 max(s) / DBL_MAX fails the evaluation (rho = inf on the
    largest row), 2 max(s) / DBL_MAX does not."""
    from ceres_solver_b200 import bal as B
    from tests.test_gpu_losses import overflow_scale, squared_norms
    bal = L.c16_bal(c16)
    obs = np.ascontiguousarray(bal.obs).ravel()
    orc0 = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, obs)
    state = B.ReducedProgram(bal).state(bal)
    s = squared_norms(orc0, state)
    for t in (SOFT_L_ONE, CAUCHY):
        for factor, expect in ((0.5, False), (2.0, True)):
            orc = LossProgram(oracle, bal, [(t, overflow_scale(s, factor), 1.0, 1.0)])
            for want_r, want_g, want_j in ((False, False, False), (True, True, True)):
                ok, cost, _, _ = orc.evaluate(state, want_r, want_g, want_j, nt=8)
                assert ok == expect and (not ok or np.isfinite(cost)), (t, factor)


def test_tukey_outlier_points(oracle, c16):
    """The construction of test_lm_tukey_outlier_points: every row of the moved points is a Tukey outlier."""
    from tests.test_gpu_losses import tukey_outlier_points_bal, squared_norms, loss_set
    from ceres_solver_b200 import bal as B
    bal, rows = tukey_outlier_points_bal(c16)
    orc = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())
    s = squared_norms(orc, B.ReducedProgram(bal).state(bal))
    a = loss_set(s)["tukey"][1]
    s_obs = np.empty_like(s)
    s_obs[orc.obs_of_row] = s
    assert rows.sum() > 0 and s_obs[rows].min() > a * a and (s_obs[~rows] <= a * a).any()


def test_loss_struct_layout(tmp_path):
    """b200_loss as gcc lays it out (include/b200ba.h) against ceres_solver_b200.binding.Loss."""
    from ceres_solver_b200.binding import Loss
    src = tmp_path / "layout.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "b200ba.h"\n'
                   'int main(void) { printf("%zu %zu %zu %zu %zu\\n", sizeof(b200_loss), offsetof(b200_loss, type), '
                   'offsetof(b200_loss, a), offsetof(b200_loss, b), offsetof(b200_loss, scale)); return 0; }\n')
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = [int(v) for v in subprocess.check_output([str(exe)], text=True).split()]
    assert got == [ctypes.sizeof(Loss), Loss.type.offset, Loss.a.offset, Loss.b.offset, Loss.scale.offset]
    assert got[0] == 32
