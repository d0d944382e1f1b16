"""CPU reference of the DOGLEG trust-region strategy, for the tests: a literal restatement of DoglegStrategy
(internal/ceres/dogleg_strategy.cc:54-717) driven by TrustRegionMinimizer::Minimize as the oracle restates it
(oracle/bal.h Minimize, which runs LevenbergMarquardtStrategy), with the oracle's evaluator, Jacobian products and
DENSE_SCHUR solve.

The library forms the subspace model from three dot products and a 2x2 Gram matrix (ceres_solver_b200/csrc/dogleg.h)
and finds the quartic's roots by simultaneous iteration.  This module keeps the reference's own formulation, so that the
tests check the reformulation against it:
  - the basis is the Q of a Householder QR with column pivoting of [g, gn] (Eigen's ColPivHouseholderQR: the column
    norms, the pivot, makeHouseholder's sign convention, the rank with the default threshold);
  - the roots are the eigenvalues of the balanced companion matrix (polynomial.cc:52-256); numpy's eigenvalue routine
    stands in for Eigen::EigenSolver.
"""
import numpy as np

EPS = np.finfo(float).eps
K_MIN_MU, K_MAX_MU, K_MU_INCREASE = 1e-8, 1.0, 10.0          # dogleg_strategy.cc:50-51, :63
TRADITIONAL, SUBSPACE = 0, 1
LS_SUCCESS, LS_FAILURE = 0, 2


# ------------------------------------------------------------------------------------------ polynomial.cc
def balance_companion_matrix(m):
    """BalanceCompanionMatrix (polynomial.cc:52-100), Parlett-Reinsch with gamma = 0.9."""
    m = np.array(m, dtype=float)
    off = m.copy()
    np.fill_diagonal(off, 0.0)
    degree = m.shape[0]
    gamma = 0.9
    changed = True
    while changed:
        changed = False
        for i in range(degree):
            col_norm = np.abs(off[:, i]).sum()
            if col_norm != 0.0:
                row_norm = np.abs(off[i, :]).sum()
                _, exponent = np.frexp(row_norm / col_norm)
                exponent = int(exponent)
                exponent = int(exponent / 2)   # C++ integer division truncates toward zero
                if exponent != 0:
                    scaled_col_norm = np.ldexp(col_norm, exponent)
                    scaled_row_norm = np.ldexp(row_norm, -exponent)
                    if scaled_col_norm + scaled_row_norm < gamma * (col_norm + row_norm):
                        changed = True
                        off[i, :] *= np.ldexp(1.0, -exponent)
                        off[:, i] *= np.ldexp(1.0, exponent)
    np.fill_diagonal(off, np.diag(m))
    return off


def build_companion_matrix(poly):
    """BuildCompanionMatrix (polynomial.cc:102-112): ones on the subdiagonal, -reverse(poly)[:degree] in the last column."""
    degree = len(poly) - 1
    m = np.zeros((degree, degree))
    for i in range(1, degree):
        m[i, i - 1] = 1.0
    m[:, degree - 1] = -np.asarray(poly[::-1][:degree])
    return m


def find_polynomial_roots(poly_in):
    """FindPolynomialRoots (polynomial.cc:190-256): (ok, real parts, imaginary parts), highest degree first."""
    poly = np.asarray(poly_in, dtype=float)
    if poly.size == 0:
        return False, None, None
    i = 0
    while i < poly.size - 1 and poly[i] == 0.0:
        i += 1
    poly = poly[i:]
    degree = poly.size - 1
    if degree == 0:
        return True, np.zeros(0), np.zeros(0)
    if degree == 1:
        return True, np.array([-poly[1] / poly[0]]), np.zeros(1)
    if degree == 2:
        a, b, c = poly
        D = b * b - 4 * a * c
        sqrt_D = np.sqrt(abs(D))
        if D >= 0:
            if b >= 0:
                return True, np.array([(-b - sqrt_D) / (2.0 * a), (2.0 * c) / (-b - sqrt_D)]), np.zeros(2)
            return True, np.array([(2.0 * c) / (-b + sqrt_D), (-b + sqrt_D) / (2.0 * a)]), np.zeros(2)
        return True, np.array([-b / (2.0 * a)] * 2), np.array([sqrt_D / (2.0 * a), -sqrt_D / (2.0 * a)])
    poly = poly / poly[0]
    m = balance_companion_matrix(build_companion_matrix(poly))
    if not np.all(np.isfinite(m)):
        return False, None, None   # Eigen's EigenSolver does not converge on non-finite input
    ev = np.linalg.eigvals(m)
    return True, ev.real.copy(), ev.imag.copy()


# ------------------------------------------------------------------------------------------ ColPivHouseholderQR
def _make_householder(x):
    """Eigen's MatrixBase::makeHouseholder: (essential, tau, beta) with H x = beta e0."""
    c0 = x[0]
    tail = x[1:]
    tail_sq = float(tail @ tail)
    tiny = np.finfo(float).tiny
    if tail_sq <= tiny:
        return np.zeros_like(tail), 0.0, c0
    beta = np.sqrt(c0 * c0 + tail_sq)
    if c0 >= 0:
        beta = -beta
    return tail / (c0 - beta), (beta - c0) / beta, beta


def col_piv_householder_qr(A):
    """(Q[:, :k], rank, R) of Eigen's ColPivHouseholderQR of A (n x k, k small), with the default threshold."""
    A = np.array(A, dtype=float)
    rows, cols = A.shape
    size = min(rows, cols)
    perm = list(range(cols))
    col_sq = np.array([A[:, j] @ A[:, j] for j in range(cols)])
    max_col_norm = np.sqrt(col_sq.max()) if cols else 0.0
    threshold_helper = (max_col_norm * EPS) ** 2 / rows
    nonzero_pivots = size
    max_pivot = 0.0
    hs = []
    for k in range(size):
        j = k + int(np.argmax(col_sq[k:]))   # first maximum, as maxCoeff
        if nonzero_pivots == size and col_sq[j] < threshold_helper * rows:
            nonzero_pivots = k
        if j != k:
            A[:, [k, j]] = A[:, [j, k]]
            col_sq[[k, j]] = col_sq[[j, k]]
            perm[k], perm[j] = perm[j], perm[k]
        ess, tau, beta = _make_householder(A[k:, k])
        A[k, k] = beta
        A[k + 1:, k] = ess
        max_pivot = max(max_pivot, abs(beta))
        v = np.concatenate([[1.0], ess])
        for c in range(k + 1, cols):   # applyHouseholderOnTheLeft
            A[k:, c] -= tau * v * (v @ A[k:, c])
        hs.append((k, v, tau))
        for c in range(k + 1, cols):   # column norm downdate, as Eigen (with recomputation on cancellation)
            if col_sq[c] != 0:
                temp = abs(A[k, c]) / np.sqrt(col_sq[c])
                temp = max(0.0, (1 + temp) * (1 - temp))
                col_sq[c] = A[k + 1:, c] @ A[k + 1:, c] if temp * col_sq[c] / col_sq[c] <= np.sqrt(EPS) else col_sq[c] * temp
    threshold = EPS * size
    rank = sum(1 for i in range(nonzero_pivots) if abs(A[i, i]) > abs(max_pivot) * threshold)
    Q = np.zeros((rows, size))
    Q[:size, :size] = np.eye(size)
    for k, v, tau in reversed(hs):   # householderQ() * I(n, size) = H_0 H_1 ... applied to I
        Q[k:, :] -= tau * np.outer(v, v @ Q[k:, :])
    return Q, rank, np.triu(A[:size, :size]), perm


# ------------------------------------------------------------------------------------------ DoglegStrategy
class DoglegStrategy:
    """dogleg_strategy.cc, on a Jacobian given by the callbacks of `ops`: squared_column_norm(), left_multiply(r),
    right_multiply(x) and solve(D) -> (y, num_iterations, termination_type)."""

    def __init__(self, dogleg_type, initial_radius, min_diagonal, max_diagonal):
        self.dogleg_type = dogleg_type
        self.radius = initial_radius
        self.min_diagonal, self.max_diagonal = min_diagonal, max_diagonal
        self.mu = K_MIN_MU
        self.dogleg_step_norm = 0.0
        self.reuse = False
        self.subspace_is_one_dimensional = False
        self.num_solves = 0        # linear solves of the last ComputeStep
        self.branch = None         # which step the last ComputeStep took (tests)

    def compute_step(self, ops, residuals):
        self.num_solves = 0
        if self.reuse:
            step = self._step()
            return step, 0, LS_SUCCESS
        self.reuse = True
        d = np.minimum(np.maximum(ops.squared_column_norm(), self.min_diagonal), self.max_diagonal)
        self.diagonal = np.sqrt(d)
        with np.errstate(all="ignore"):
            self.gradient = ops.left_multiply(residuals) / self.diagonal
            Jg = ops.right_multiply(self.gradient / self.diagonal)
            self.alpha = (self.gradient @ self.gradient) / (Jg @ Jg)
        num_iterations, term = self._gauss_newton_step(ops, residuals)
        if term != LS_FAILURE and self.dogleg_type == SUBSPACE and not self._subspace_model(ops):
            term = LS_FAILURE
        step = self._step() if term != LS_FAILURE else None
        return step, num_iterations, term

    def _step(self):
        with np.errstate(all="ignore"):
            return self._traditional() if self.dogleg_type == TRADITIONAL else self._subspace()

    def _gauss_newton_step(self, ops, residuals):
        num_iterations, term = -1, LS_FAILURE
        while self.mu < K_MAX_MU:
            D = self.diagonal * np.sqrt(self.mu)
            y, num_iterations, term = ops.solve(D)
            self.num_solves += 1
            if term == LS_FAILURE or not np.all(np.isfinite(y)):
                self.mu *= K_MU_INCREASE
                term = LS_FAILURE
                continue
            break
        if term != LS_FAILURE:
            self.gauss_newton_step = y * -self.diagonal
        return num_iterations, term

    def _traditional(self):
        g, gn = self.gradient, self.gauss_newton_step
        gradient_norm = np.sqrt(g @ g)
        gauss_newton_norm = np.sqrt(gn @ gn)
        # the two values the traditional step compares with the radius, relative to it (tests/dogleg_cases.py margins)
        self.thresholds = dict(gauss_newton=gauss_newton_norm / self.radius, cauchy=gradient_norm * self.alpha / self.radius)
        if gauss_newton_norm <= self.radius:
            self.branch = "gauss_newton"
            self.dogleg_step_norm = gauss_newton_norm
            return gn / self.diagonal
        if gradient_norm * self.alpha >= self.radius:
            self.branch = "cauchy"
            self.dogleg_step_norm = self.radius
            return (-(self.radius / gradient_norm) * g) / self.diagonal
        self.branch = "interpolated"
        b_dot_a = -self.alpha * (g @ gn)
        a_squared_norm = (self.alpha * gradient_norm) ** 2
        b_minus_a_squared_norm = a_squared_norm - 2 * b_dot_a + gauss_newton_norm ** 2
        c = b_dot_a - a_squared_norm
        d = np.sqrt(c * c + b_minus_a_squared_norm * (self.radius ** 2 - a_squared_norm))
        beta = (d - c) / b_minus_a_squared_norm if c <= 0 else (self.radius * self.radius - a_squared_norm) / (d + c)
        step = (-self.alpha * (1.0 - beta)) * g + beta * gn
        self.dogleg_step_norm = np.sqrt(step @ step)
        return step / self.diagonal

    def _subspace_model(self, ops):
        basis, rank, _, _ = col_piv_householder_qr(np.stack([self.gradient, self.gauss_newton_step], axis=1))
        self.rank = rank
        if rank == 0:
            return False
        if rank == 1:
            self.subspace_is_one_dimensional = True
            return True
        self.subspace_is_one_dimensional = False
        self.basis = basis
        self.sg = basis.T @ self.gradient
        Jb = np.stack([ops.right_multiply(basis[:, 0] / self.diagonal), ops.right_multiply(basis[:, 1] / self.diagonal)])
        self.B = Jb @ Jb.T
        return True

    def boundary_polynomial(self):
        B, g, r2 = self.B, self.sg, self.radius * self.radius
        detB = B[0, 0] * B[1, 1] - B[0, 1] * B[1, 0]
        trB = B[0, 0] + B[1, 1]
        adj = np.array([[B[1, 1], -B[0, 1]], [-B[1, 0], B[0, 0]]])
        return np.array([r2, 2.0 * r2 * trB, r2 * (trB * trB + 2.0 * detB) - g @ g,
                         -2.0 * (g @ adj @ g - r2 * detB * trB), r2 * detB * detB - (adj @ g) @ (adj @ g)])

    def _step_from_root(self, y):
        return -np.linalg.solve(self.B + y * np.eye(2), self.sg)

    def _model(self, x):
        return 0.5 * x @ (self.B @ x) + self.sg @ x

    def boundary_minimum(self):
        ok, roots, _ = find_polynomial_roots(self.boundary_polynomial())
        if not ok:
            return False, np.zeros(2)
        minimum_value, minimum, found = np.finfo(float).max, np.zeros(2), False
        for y in roots:
            try:
                x = self._step_from_root(y)
            except np.linalg.LinAlgError:
                continue
            n = np.sqrt(x @ x)
            if n > 0:
                f = self._model((self.radius / n) * x)
                found = True
                if f < minimum_value:
                    minimum_value, minimum = f, x
        return found, minimum

    def _subspace(self):
        gn = self.gauss_newton_step
        gauss_newton_norm = np.sqrt(gn @ gn)
        self.thresholds = dict(gauss_newton=gauss_newton_norm / self.radius)
        if gauss_newton_norm <= self.radius:
            self.branch = "gauss_newton"
            self.dogleg_step_norm = gauss_newton_norm
            return gn / self.diagonal
        if self.subspace_is_one_dimensional:
            self.branch = "one_dimensional"
            self.dogleg_step_norm = self.radius
            g = self.gradient
            return (-(self.radius / np.sqrt(g @ g)) * g) / self.diagonal
        ok, m = self.boundary_minimum()
        if not ok:
            step = self._traditional()
            self.branch = "root_failure"
            return step
        gm = self.B @ m + self.sg
        cosine = -(m @ gm) / (np.sqrt(m @ m) * np.sqrt(gm @ gm))
        if cosine < 0.99:
            step = self._traditional()
            self.branch = "cosine_fallback"
            return step
        self.branch = "boundary"
        self.dogleg_step_norm = self.radius
        return (self.basis @ m) / self.diagonal

    def step_accepted(self, quality):
        assert quality > 0.0
        if quality < 0.25:
            self.radius *= 0.5
        if quality > 0.75:
            self.radius = max(self.radius, 3.0 * self.dogleg_step_norm)
        self.mu = max(K_MIN_MU, 2.0 * self.mu / K_MU_INCREASE)
        self.reuse = False

    def step_rejected(self):
        self.radius *= 0.5
        self.reuse = True

    def step_is_invalid(self):
        self.mu *= K_MU_INCREASE
        self.reuse = False


class DenseOps:
    """A dense J (the known-answer tests): exact solve of (J'J + D^2) y = J'r."""

    def __init__(self, J, r):
        self.J = np.asarray(J, dtype=float)
        self.r = np.asarray(r, dtype=float)

    def squared_column_norm(self):
        return (self.J ** 2).sum(axis=0)

    def left_multiply(self, r):
        return self.J.T @ r

    def right_multiply(self, x):
        return self.J @ x

    def solve(self, D):
        A = self.J.T @ self.J + np.diag(D * D)
        try:
            np.linalg.cholesky(A)
        except np.linalg.LinAlgError:
            return np.full(A.shape[0], np.nan), 1, LS_FAILURE
        return np.linalg.solve(A, self.J.T @ self.r), 1, LS_SUCCESS


class OracleOps:
    """The oracle's Jacobian (scaled in place, as the minimizer leaves it) and its DENSE_SCHUR solve."""

    def __init__(self, J, num_elim, residuals, nt):
        self.J, self.num_elim, self.r, self.nt = J, num_elim, residuals, nt

    def squared_column_norm(self):
        return self.J.squared_column_norm(nt=self.nt)

    def left_multiply(self, r):
        return self.J.left_multiply(r, nt=self.nt)

    def right_multiply(self, x):
        return self.J.right_multiply(x, nt=self.nt)

    def solve(self, D):
        return self.J.linear_solve(self.num_elim, self.r, D, solver=1, nt=self.nt)


# ------------------------------------------------------------------------------------------ the minimizer
_DEFAULTS = dict(max_num_iterations=5, initial_trust_region_radius=1e4, min_trust_region_radius=1e-32,
                 min_relative_decrease=1e-3, min_lm_diagonal=1e-6, max_lm_diagonal=1e32, function_tolerance=1e-16,
                 gradient_tolerance=1e-16, parameter_tolerance=1e-16, jacobi_scaling=1,
                 max_num_consecutive_invalid_steps=5)


def minimize(orc, state, dogleg_type, nt=8, **options):
    """TrustRegionMinimizer::Minimize (oracle/bal.h Minimize, trust_region_minimizer.cc) with DoglegStrategy and
    DENSE_SCHUR.  Returns (best state, records in the binding's field names, per record (linear solves, branch, the
    step's threshold ratios))."""
    o = dict(_DEFAULTS)
    o.update({k: v for k, v in options.items() if k not in ("linear_solver_type", "trust_region_strategy_type",
                                                              "dogleg_type")})
    P = orc.P
    x = np.array(state, dtype=float)
    strategy = DoglegStrategy(dogleg_type, o["initial_trust_region_radius"], o["min_lm_diagonal"], o["max_lm_diagonal"])
    scaling = np.ones_like(x)
    recs, info = [], []
    st = dict(x_cost=np.finfo(float).max, iteration=0)

    def evaluate_gradient_and_jacobian(it):
        ok, cost, res, grad = orc.evaluate(x, nt=nt)
        assert ok
        J = orc.jacobian()
        if o["jacobi_scaling"]:
            if st["iteration"] == 0:
                scaling[:] = 1.0 / (1.0 + np.sqrt(J.squared_column_norm(nt=nt)))
            J.scale_columns(scaling, nt=nt)
        st.update(x_cost=cost, res=res, J=J)
        it["cost"] = cost
        d = x - (x + (-grad))
        it["gradient_max_norm"] = float(np.abs(d).max())
        it["gradient_norm"] = float(np.sqrt(d @ d))

    def new_record(iteration):
        return dict(iteration=iteration, ls_iterations=0, step_is_valid=0, step_is_successful=0, cost=0.0,
                    cost_change=0.0, gradient_max_norm=0.0, gradient_norm=0.0, step_norm=0.0, tr_ratio=0.0,
                    tr_radius=0.0, model_cost_change=0.0)

    it = new_record(0)
    evaluate_gradient_and_jacobian(it)
    it["step_is_valid"] = it["step_is_successful"] = 1
    se_min = se_cur = se_ref = se_cand = st["x_cost"]
    se_acc_ref = se_acc_cand = 0.0
    minimum_cost, best = np.finfo(float).max, x.copy()
    invalid, one_ok = 0, False
    solves = (0, None, {})
    while True:
        if it["step_is_successful"] and st["x_cost"] < minimum_cost:
            minimum_cost, best = st["x_cost"], x.copy()
        it["tr_radius"] = strategy.radius
        recs.append(it)
        info.append(solves)
        if it["iteration"] >= o["max_num_iterations"]:
            break
        if it["step_is_successful"] and it["gradient_max_norm"] <= o["gradient_tolerance"]:
            break
        if it["tr_radius"] <= o["min_trust_region_radius"]:
            break
        prev = it
        it = new_record(prev["iteration"] + 1)
        st["iteration"] = it["iteration"]
        ops = OracleOps(st["J"], P, st["res"], nt)
        strategy.thresholds = {}
        step, its, term = strategy.compute_step(ops, st["res"])
        solves = (strategy.num_solves, strategy.branch if term != LS_FAILURE else None, strategy.thresholds)
        it["ls_iterations"] = its
        if term != LS_FAILURE:
            with np.errstate(all="ignore"):
                Js = st["J"].right_multiply(step, nt=nt)
                mcc = -(Js @ (st["res"] + Js / 2.0))
            it["model_cost_change"] = mcc
            it["step_is_valid"] = int(mcc > 0.0)
        if not it["step_is_valid"]:
            invalid += 1
            if invalid >= o["max_num_consecutive_invalid_steps"]:
                break
            strategy.step_is_invalid()
            it.update(cost=st["x_cost"], cost_change=0.0, gradient_max_norm=prev["gradient_max_norm"],
                      gradient_norm=prev["gradient_norm"], step_norm=0.0, tr_ratio=0.0)
            continue
        invalid = 0
        cand = x + step * scaling
        ok, ccost, _, _ = orc.evaluate(cand, want_residuals=False, want_gradient=False, want_jacobian=False, nt=nt)
        if not ok:
            ccost = np.finfo(float).max
        sn = float((x - cand) @ (x - cand))
        it["step_norm"] = np.sqrt(sn) if one_ok else 0.0
        if one_ok and it["step_norm"] <= o["parameter_tolerance"] * (np.sqrt(x @ x) + o["parameter_tolerance"]):
            break
        it["cost_change"] = st["x_cost"] - ccost
        if abs(it["cost_change"]) <= o["function_tolerance"] * st["x_cost"]:
            break
        if ccost >= np.finfo(float).max:
            it["tr_ratio"] = -np.finfo(float).max
        else:
            it["tr_ratio"] = max((se_cur - ccost) / mcc, (se_ref - ccost) / (se_acc_ref + mcc))
        if it["tr_ratio"] > o["min_relative_decrease"]:
            one_ok = True
            x = cand
            evaluate_gradient_and_jacobian(it)
            it["step_is_successful"] = 1
            strategy.step_accepted(it["tr_ratio"])
            se_cur = ccost
            se_acc_cand += mcc
            se_acc_ref += mcc
            if se_cur < se_min:
                se_min = se_cand = se_cur
                se_acc_cand = 0.0
                se_ref, se_acc_ref = se_cand, se_acc_cand
            elif se_cur > se_cand:
                se_cand, se_acc_cand = se_cur, 0.0
        else:
            it.update(step_is_successful=0, cost=ccost, gradient_norm=prev["gradient_norm"],
                      gradient_max_norm=prev["gradient_max_norm"])
            strategy.step_rejected()
    return best, recs, info
