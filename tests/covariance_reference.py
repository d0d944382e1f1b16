"""The covariance of a bundle-adjustment problem's cameras and points, restated in numpy for the tests of
b200_covariance_compute (tests/test_gpu_covariance.py, guarded on the CPU by tests/test_covariance_reference.py).

Ceres' Covariance::Compute evaluates J on the reduced program (constant blocks removed, Program::RemoveFixedBlocks) and, with
SPARSE_QR, forms the covariance as R^-1 R^-T of J_red's QR factor, i.e. (J_red'J_red)^-1.  Two restatements:
  - literal_covariance: (J_red'J_red)^-1 itself, placed back in the full [3P | 9C] layout with zeros on constant blocks;
  - SchurCovariance: the Schur form the library computes, in np.longdouble: S = F'F - W'V^-1 W with D' = 1 on constant
    components (so constant blocks become decoupled identity blocks), its Cholesky factor (own code: numpy's linalg has no
    longdouble), Z = S^-1, and Cov(p, p) = V_p^-1 + V_p^-1 W_p Z W_p' V_p^-1.  It also reports the conditioning test of
    b200_covariance_compute: the smallest d_k / A_kk over the variable components of S's Cholesky and of every variable
    point's 3x3 Cholesky of V_p (d_k the k-th squared pivot, A_kk the matrix's diagonal).
Both take the Jacobian in the library's value layout (all E cells [N][2][3], then all F cells [N][2][9]).
"""
import numpy as np

from tests.constant_blocks_reference import jacobian_matrix

LD = np.longdouble


def literal_covariance(values, row_cam, row_pt, P, C, fixed):
    """(J_red'J_red)^-1 in float64 in the [3P + 9C] layout, zeros on the constant components."""
    J = jacobian_matrix(values, row_cam, row_pt, P, C).toarray()
    keep = np.flatnonzero(~fixed)
    Jr = J[:, keep]
    out = np.zeros((J.shape[1], J.shape[1]))
    out[np.ix_(keep, keep)] = np.linalg.inv(Jr.T @ Jr)
    return out


def cholesky(A):
    """Lower Cholesky factor of A (its dtype) and the squared pivots d_k; (None, pivots so far) at a non-positive pivot."""
    if A.dtype == np.float64 and A.shape[0] > 3:   # LAPACK's, for the larger float64 references
        try:
            L = np.linalg.cholesky(A)
        except np.linalg.LinAlgError:
            return None, np.zeros(1)
        return L, np.diag(L) ** 2
    A = np.array(A, copy=True)
    n = A.shape[0]
    L = np.zeros_like(A)
    d = np.zeros(n, dtype=A.dtype)
    for k in range(n):
        d[k] = A[k, k]
        if not d[k] > 0:
            return None, d[:k + 1]
        L[k, k] = np.sqrt(d[k])
        L[k + 1:, k] = A[k + 1:, k] / L[k, k]
        A[k + 1:, k + 1:] -= np.outer(L[k + 1:, k], L[k + 1:, k])
    return L, d


def cholesky_inverse(L):
    """(L L')^-1 by two triangular solves on the identity, in L's dtype."""
    n = L.shape[0]
    if L.dtype == np.float64 and n > 3:
        import scipy.linalg as sla
        Y = sla.solve_triangular(L, np.eye(n), lower=True)
        return sla.solve_triangular(L.T, Y, lower=False)
    Y = np.zeros_like(L)
    eye = np.eye(n, dtype=L.dtype)
    for k in range(n):   # L Y = I
        Y[k] = (eye[k] - L[k, :k] @ Y[:k]) / L[k, k]
    X = np.zeros_like(L)
    for k in range(n - 1, -1, -1):   # L' X = Y
        X[k] = (Y[k] - L[k + 1:, k] @ X[k + 1:]) / L[k, k]
    return X


class SchurCovariance:
    """The Schur form of the covariance in `dtype` (np.longdouble by default).  Attributes: S [9C x 9C] (as factored: D' = 1
    on constant components), Z = S^-1 (None when S is not positive definite), points [P, 3, 3], rcond (the conditioning
    test's minimum; 0 when a factorisation fails), kappa (the 2-norm condition number of S, in float64), and
    point_ok (every variable point's V_p positive definite)."""

    def __init__(self, values, row_cam, row_pt, P, C, fixed, dtype=LD):
        row_cam = np.asarray(row_cam, dtype=np.int64)
        row_pt = np.asarray(row_pt, dtype=np.int64)
        N = row_cam.size
        values = np.asarray(values, dtype=float)
        E = values[:6 * N].reshape(N, 2, 3).astype(dtype)
        F = values[6 * N:].reshape(N, 2, 9).astype(dtype)
        fp = np.asarray(fixed[:3 * P:3], dtype=bool)
        fc = np.asarray(fixed[3 * P::9], dtype=bool)
        self.fixed_points, self.fixed_cameras = fp, fc
        E[fp[row_pt]] = 0   # the reduced program has no columns for constant blocks (the library stores those cells as 0)
        F[fc[row_cam]] = 0
        n = 9 * C
        S = np.zeros((n, n), dtype=dtype)
        # F'F
        for r in range(N):
            c = row_cam[r]
            S[9 * c:9 * c + 9, 9 * c:9 * c + 9] += F[r].T @ F[r]
        # points: V_p, W_p = E_p'F_p [3 x 9C]
        order = np.argsort(row_pt, kind="stable")
        starts = np.searchsorted(row_pt[order], np.arange(P + 1))
        self.V = np.zeros((P, 3, 3), dtype=dtype)
        self.W = []
        rc = [1.0]
        self.point_ok = True
        for p in range(P):
            rows = order[starts[p]:starts[p + 1]]
            cams = np.unique(row_cam[rows])
            cols = (9 * cams[:, None] + np.arange(9)).ravel()
            Wc = np.zeros((3, cols.size), dtype=dtype)   # W_p on the point's cameras only
            V = np.zeros((3, 3), dtype=dtype)
            for r in rows:
                V += E[r].T @ E[r]
                k = int(np.searchsorted(cams, row_cam[r]))
                Wc[:, 9 * k:9 * k + 9] += E[r].T @ F[r]
            self.W.append((cols, Wc))
            if fp[p]:
                self.V[p] = np.eye(3, dtype=dtype)
                continue
            self.V[p] = V
            Lv, dv = cholesky(V)
            if Lv is None:
                self.point_ok = False
                rc.append(0.0)
                continue
            rc.append(min(dv / np.diag(V)))
            Vi = cholesky_inverse(Lv)
            S[np.ix_(cols, cols)] -= Wc.T @ Vi @ Wc
        idx = np.flatnonzero(np.repeat(fc, 9))
        S[idx, :] = 0
        S[:, idx] = 0
        S[idx, idx] = 1
        self.S = S
        Ls, ds = cholesky(S)
        var = ~np.repeat(fc, 9)
        self.Z = None
        self.points = None
        if Ls is None or not self.point_ok:
            self.rcond = 0.0
        else:
            rc.append(min((ds / np.diag(S))[var]))
            self.rcond = float(min(rc))
            self.Z = cholesky_inverse(Ls)
            self.points = np.zeros((P, 3, 3), dtype=dtype)
            for p in range(P):
                if fp[p]:
                    continue
                Vi = cholesky_inverse(cholesky(self.V[p])[0])
                cols, Wc = self.W[p]
                G = Wc @ self.Z[np.ix_(cols, cols)] @ Wc.T
                self.points[p] = Vi + Vi @ G @ Vi
        ev = np.linalg.eigvalsh(np.asarray(S, dtype=float)[np.ix_(var, var)]) if var.any() else np.ones(1)
        self.kappa = float(ev[-1] / ev[0]) if ev[0] > 0 else float("inf")

    def _dense_w(self, p, C):
        cols, Wc = self.W[p]
        Wp = np.zeros((3, 9 * C), dtype=Wc.dtype)
        Wp[:, cols] = Wc
        return Wp

    def camera_block(self, i, j):
        return np.asarray(self.Z[9 * i:9 * i + 9, 9 * j:9 * j + 9], dtype=float)

    def full(self, P, C):
        """The whole covariance [3P + 9C] from the Schur form, cross blocks included (for the comparison with the literal
        inverse): [[V^-1 + V^-1 W Z W' V^-1, -V^-1 W Z], [-Z W' V^-1, Z]] per point, zeros on constant blocks."""
        n = 3 * P + 9 * C
        out = np.zeros((n, n), dtype=self.Z.dtype)
        out[3 * P:, 3 * P:] = self.Z
        Vi = [np.zeros((3, 3), dtype=self.Z.dtype) if self.fixed_points[p] else cholesky_inverse(cholesky(self.V[p])[0])
              for p in range(P)]
        for p in range(P):
            if self.fixed_points[p]:
                continue
            Wp = self._dense_w(p, C)
            X = -Vi[p] @ Wp @ self.Z   # Cov(p, cameras)
            out[3 * p:3 * p + 3, 3 * P:] = X
            out[3 * P:, 3 * p:3 * p + 3] = X.T
            for q in range(P):
                if self.fixed_points[q]:
                    continue
                out[3 * p:3 * p + 3, 3 * q:3 * q + 3] = (p == q) * Vi[p] + Vi[p] @ Wp @ self.Z @ self._dense_w(q, C).T @ Vi[q]
        idx = np.flatnonzero(np.repeat(self.fixed_cameras, 9)) + 3 * P
        out[idx, :] = 0
        out[:, idx] = 0
        return out
