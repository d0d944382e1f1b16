"""The device SPARSE_SCHUR factorisation (b200_sparse_schur_solve: csrc/sparse_plan.cuh, csrc/sparse_schur.cuh) against an
extended-precision reference that shares nothing with the library's Schur path, on camera graphs built to reach each path
of the supernodal kernel (tests/test_sparse_schur_plan.py builds them and recounts their layout).

Reference.  J is rebuilt as a scipy CSR matrix from b200_jacobian_get_values and the row structure, and checked against
the library's J x and J'y to 1e-14 before it is used.  Two measures of the solve are then taken:

  backward error  of the camera block x_f as a solution of the reduced system (S + D_f^2) x_f = rhs_S, in np.longdouble
                  (80-bit, eps ~ 1.1e-19): V = E'E + D_e^2 and its 3x3 inverses by the adjugate formula; S x_f = F'F x_f +
                  D_f^2 x_f - F'E V^-1 E'F x_f and rhs_S = F'b - F'E V^-1 E'b as products, S is never formed;
                      eta = |rhs_S - (S + D_f^2) x_f| / ((|F'F| + |W'K V^-1 W| + |D_f^2|) |x_f| + |F'b| + ||W|'|K V^-1 E'b||),
                  W = E'F, matrix norms Frobenius.  The denominator holds the magnitudes of the terms S and rhs_S are summed
                  from, so the float64 assembly's own cancellation does not inflate eta.  K weighs each point's terms by
                  the condition number kappa(V_p) of its block: the library inverts V_p in float64, which leaves a relative
                  error of kappa(V_p) u in that point's contribution (observed: without K, eta reaches 190 u on the
                  geometric Jacobian at radius 1e4, where the solo points' V_p reach kappa 2e4).  Everything is taken on
                  the system scaled to a unit diagonal of F'F + D_f^2 (and kappa(V_p) on V_p scaled to a unit diagonal),
                  which the Cholesky factorisation is invariant under: unscaled, with column scales spread over six
                  decades, the norms would see only the largest columns.  A dropped or misplaced update leaves a residual
                  of the size of that update.  At radius 1e-1 every kappa(V_p) is about 1 and eta is at its sharpest.
  forward error   of the whole step against x_ref, the solution of (J'J + D^2) x = J'b in float64 (the points eliminated
                  with this module's V^-1, S + D_f^2 factored by scipy's splu), refined with residuals of the full system
                  computed in longdouble from J.  Refinement stops when the camera block's relative correction falls below
                  1e-18 or stops halving; with 80-bit residuals it cannot fall much below kappa x 1e-19, so what is
                  asserted is that it stops within REFINE_STEPS steps at a correction 100 times below the bound the solve
                  is held to.  The camera block is held, in the norm of the scaled system, to
                      |x_f - x_ref,f| <= C_X kappa u |x_ref,f|,   u = 2^-53,
                      kappa = |(S + D_f^2)^-1| (den_mat + den_vec / |x_ref,f|),
                  den_mat and den_vec the two parts of eta's denominator: the forward error a backward error of C_X u
                  implies.  kappa >= kappa_2(S + D_f^2), which is too small a factor here because the float64 assembly's
                  error is relative to the terms' magnitudes, not to S; kappa_2 alone (unscaled, 1e12 with random
                  values) would make the bound vacuous.  |(S + D_f^2)^-1| comes from eigvalsh of S + D_f^2, formed here in
                  float64 from J, per connected component of the camera graph.  The point block comes from back
                  substitution, x_e = V^-1 (E'b - W x_f), which passes the camera block's error on through V^-1 W and adds
                  the rounding of one 3x3 solve per point:
                      |x_e - x_ref,e| <= |V^-1 W| |x_f - x_ref,f| + C_X u kappa_V (|x_ref,e| + |V^-1 W| |x_ref,f|),
                  kappa_V the largest kappa(V_p).

C_ETA and C_X are fixed from runs of the unchanged kernel on every case of test_structure (one H100 80GB HBM3, 700 W
power limit): the largest observed eta / u was 1.45 and the largest camera-block forward error / (kappa u) 1.3 (both on
clique16 at radius 1e-1), and the largest point-block error 0.39 of its bound, so both constants sit at 16: an order of
magnitude above every observation, while a dropped or misplaced update moves eta by the relative size of that update,
orders of magnitude above C_ETA u = 1.8e-15.  Observed / bound for eta, camera block and point block, with kappa_V in
brackets; where kappa_V is ~1 (radius 1e-1) eta is unweighted and the check is at its sharpest:

             geometric 1e4            geometric 1e-1           random 1e4               random 1e-1              random D=NULL           
  one        1e-03/5e-04/0.39 (2e+04) 0.05/0.04/0.08 (1e+00)   8e-04/4e-04/9e-07 (3e+02) 0.06/0.05/5e-05 (1e+00)  6e-04/4e-04/1e-06 (3e+02)
  two        2e-03/5e-04/0.34 (2e+04) 0.04/0.03/0.07 (1e+00)   2e-03/9e-04/6e-07 (6e+02) 0.05/0.05/4e-05 (1e+00)  3e-03/1e-03/1e-06 (6e+02)
  clique16   3e-04/5e-05/0.05 (2e+04) 0.08/0.07/0.05 (1e+00)   7e-04/2e-04/2e-07 (3e+03) 0.08/0.08/8e-06 (1e+00)  4e-04/1e-04/9e-08 (3e+03)
  cliques    2e-04/3e-05/5e-03 (2e+04) 0.04/0.04/0.02 (1e+00)   4e-04/1e-05/5e-09 (2e+04) 0.06/0.05/3e-06 (1e+00)  4e-04/1e-05/2e-08 (5e+04)
  hub        2e-04/8e-05/7e-03 (2e+04) 0.02/0.02/0.03 (1e+00)   2e-04/1e-05/1e-08 (7e+03) 0.03/0.03/2e-06 (1e+00)  2e-04/7e-06/6e-08 (1e+04)
  band       2e-04/2e-05/6e-03 (2e+04) 0.05/0.05/0.03 (1e+00)   3e-04/1e-05/1e-08 (2e+04) 0.06/0.06/2e-06 (1e+00)  1e-04/4e-06/4e-09 (7e+04)
  loop       2e-04/8e-06/5e-03 (2e+04) 0.05/0.05/0.03 (1e+00)   5e-04/4e-05/9e-09 (6e+03) 0.06/0.06/3e-06 (1e+00)  3e-04/2e-05/7e-09 (1e+04)
  forest     6e-05/2e-05/9e-04 (2e+04) 9e-03/8e-03/9e-03 (1e+00) 7e-05/2e-06/2e-09 (2e+04) 0.01/0.01/5e-07 (1e+00)  2e-05/2e-07/5e-09 (1e+06)
  random400  2e-03/8e-05/0.03 (2e+01) 0.04/0.03/0.03 (1e+00)   7e-04/4e-04/1e-08 (2e+03) 0.05/0.04/2e-06 (1e+00)  8e-04/4e-04/2e-08 (2e+03)
  shuffled   1e-04/5e-06/0.01 (2e+04) 0.04/0.04/0.03 (1e+00)   5e-04/4e-05/3e-09 (6e+03) 0.06/0.06/3e-06 (1e+00)  3e-04/3e-05/2e-09 (9e+03)

Each of these value-only changes to sparse_schur.cuh fails this module (test_structure, test_failure_and_recovery and
test_reuse run against each; test_reuse compares a handle with a fresh one, so a consistent error passes it):

  change                                             fails here                                   tests/test_gpu_sparse_schur.py
  step 1 drops each supernode's last update          structure: 7 of 10 (all with updates);       test_solve: huge, sequence,
    (q < u1 - 1)                                     failure_and_recovery: all 3                  clusters, random
  partial last stage zeroed (t0 + kSpK <= Wd)        structure: cliques, hub, loop, forest,       test_solve: sequence, random
                                                     random400, shuffled
  trailing update j < jmax                           structure: all but `one`; failure: all 3     all 8 solve and LM tests
  backward sum omits the last block row              structure: 7 of 10; failure: all 3           test_solve: huge, sequence,
                                                                                                  clusters, random
  forward descendant term sums Wd - 9 columns        structure: 7 of 10; failure: all 3           the same 4

The refinement of x_ref shrinks its correction by 1e-3 .. 1e-10 from the first step to the second on these cases and
ends within 2 .. 4 steps at a correction of 3e-20 .. 1.4e-15, at least 100 times below the bound; np.longdouble must be
wider than float64 (asserted).

Each structure is solved with two kinds of Jacobian values: the geometric Jacobian of `evaluate` (Jacobi-scaled, as the LM
loop sees it) and random values whose column scales spread over 1e-3..1e3, and with three LM diagonals: radius 1e4,
radius 1e-1 and D = NULL (random values only: S is positive definite without damping thanks to every camera's solo
points).  The plan line b200_create's analysis prints under B200_VERBOSE at the first sparse solve is checked against the
recount.  Failure, recovery, reuse of one handle, and the exact-step LM loop on a problem of many supernodes follow.
"""
import ctypes
import os
import re

import numpy as np
import pytest
import scipy.sparse as sps
import scipy.sparse.linalg as spla
from scipy.sparse.csgraph import connected_components

from tests import lm_cases as L
from tests.entry_points import Case, compare_lm_traces_exact, relerr
from tests.test_sparse_schur_plan import STRUCTURES, check_plan, structure, structure_properties

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
LD = np.longdouble
C_ETA = 16.0
C_X = 16.0
REFINE_STEPS = 5
RADII = (1e4, 1e-1, None)
PLAN_RE = re.compile(r"\[b200ba\] sparse S plan: .*, (\d+) supernodes \(widest (\d+) columns\), tree height (\d+), "
                     r"factor [\d.]+ MB, (\d+) CTAs")


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.fixture(scope="module")
def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- problems

def geometry(C, P, cam, pt, seed):
    """Observations and an initial state for any camera graph: cameras on a circle of radius 100 looking at its centre,
    points within 60 of it, so every point is in front of every camera (tracks may be arbitrary)."""
    from ceres_solver_b200 import bal as B
    rng = np.random.RandomState(seed)
    phi = 2.0 * np.pi * (np.arange(C) + 0.5) / C
    centers = np.stack([100.0 * np.cos(phi), 100.0 * np.sin(phi), 5.0 * np.sin(3.0 * phi)], axis=1)
    cams = B._look_at_cameras(centers, np.zeros((C, 3)), rng)
    pts = rng.normal(0.0, 15.0, (P, 3))
    pts *= np.minimum(1.0, 60.0 / np.linalg.norm(pts, axis=1))[:, None]
    bal = B._finish(rng, cams, pts, cam, pt)
    return bal.obs, np.concatenate([bal.points.ravel(), bal.cameras.ravel()])


class Structure:
    def __init__(self, cs, name):
        self.name = name
        self.C, self.P, self.cam, self.pt = structure(name)
        self.perm, _, self.lay = check_plan(cs, self.C, self.P, self.cam, self.pt)
        structure_properties(name, self.perm, self.lay)
        self.obs, self.state = geometry(self.C, self.P, self.cam, self.pt, seed=11)

    def problem(self, cs):
        return cs.Problem(self.C, self.P, self.cam, self.pt, self.obs)


def random_values(s, seed):
    """Jacobian values with random signs and column scales spread over 1e-3..1e3, and a random right-hand side."""
    rng = np.random.RandomState(seed)
    scale = 10.0 ** rng.uniform(-3.0, 3.0, 3 * s.P + 9 * s.C)
    N = len(s.cam)
    vE = rng.randn(N, 2, 3) * scale[:3 * s.P].reshape(s.P, 3)[s.pt][:, None, :]
    vF = rng.randn(N, 2, 9) * scale[3 * s.P:].reshape(s.C, 9)[s.cam][:, None, :]
    return np.concatenate([vE.ravel(), vF.ravel()]), rng.randn(2 * N)


def load(gpu, s, kind):
    """Puts one kind of Jacobian values on the handle; returns the right-hand side b."""
    ok, _, res, _ = gpu.evaluate(s.state)
    assert ok
    if kind == "geometric":
        gpu.scale_columns(1.0 / (1.0 + np.sqrt(gpu.squared_column_norm())))
        return res
    v, b = random_values(s, seed=5)
    gpu.set_jacobian_values(v)
    return b


def lm_diagonal(gpu, radius):
    return None if radius is None else np.sqrt(np.clip(gpu.squared_column_norm(), 1e-6, 1e32) / radius)


# ---- reference

def jacobian(gpu, C, P, cam, pt):
    """J as a CSR matrix from the handle's values (all E cells [N][2][3], then all F cells [N][2][9]), checked against the
    handle's own products."""
    v = gpu.jacobian_values()
    N = len(cam)
    r = np.arange(2 * N).reshape(N, 2, 1)
    ce = 3 * np.asarray(pt).reshape(N, 1, 1) + np.arange(3)
    cf = 3 * P + 9 * np.asarray(cam).reshape(N, 1, 1) + np.arange(9)
    rows = np.concatenate([np.broadcast_to(r, (N, 2, 3)).ravel(), np.broadcast_to(r, (N, 2, 9)).ravel()])
    cols = np.concatenate([np.broadcast_to(ce, (N, 2, 3)).ravel(), np.broadcast_to(cf, (N, 2, 9)).ravel()])
    J = sps.csr_matrix((v, (rows, cols)), shape=(2 * N, 3 * P + 9 * C))
    rng = np.random.RandomState(1)
    x, y = rng.randn(J.shape[1]), rng.randn(J.shape[0])
    assert relerr(gpu.right_multiply(x), J @ x) <= 1e-14
    assert relerr(gpu.left_multiply(y), J.T @ y) <= 1e-14
    return J


def _norm(a):
    return float(np.sqrt(np.sum(np.asarray(a, dtype=LD) ** 2)))


def _inv3(M):
    """Inverses of a stack of 3x3 matrices by the adjugate formula, in M's precision."""
    a, b, c = M[:, 0, 0], M[:, 0, 1], M[:, 0, 2]
    d, e, f = M[:, 1, 0], M[:, 1, 1], M[:, 1, 2]
    g, h, i = M[:, 2, 0], M[:, 2, 1], M[:, 2, 2]
    adj = np.stack([np.stack([e * i - f * h, c * h - b * i, b * f - c * e], axis=1),
                    np.stack([f * g - d * i, a * i - c * g, c * d - a * f], axis=1),
                    np.stack([d * h - e * g, b * g - a * h, a * e - b * d], axis=1)], axis=1)
    det = a * adj[:, 0, 0] + b * adj[:, 1, 0] + c * adj[:, 2, 0]
    return adj / det[:, None, None]


class Reference:
    """The damped reduced system of one (J, b, D), and the full system's extended-precision solution."""

    def __init__(self, J, P, C, b, D):
        # the reference rests on a longdouble wider than float64 (x87 80-bit or quad)
        assert np.finfo(LD).eps < 1e-18, np.finfo(LD)
        self.P, self.C = P, C
        n_e = 3 * P
        d2 = np.zeros(J.shape[1]) if D is None else np.asarray(D) ** 2
        Jc = J.tocsc()
        E64, F64 = Jc[:, :n_e].tocsr(), Jc[:, n_e:].tocsr()
        self.E, self.F = E64.astype(LD), F64.astype(LD)
        self.Df2 = d2[n_e:].astype(LD)
        EtE = (self.E.T @ self.E).tocoo()
        V = np.zeros((P, 3, 3), dtype=LD)
        np.add.at(V, (EtE.row // 3, EtE.row % 3, EtE.col % 3), EtE.data)
        V[:, np.arange(3), np.arange(3)] += d2[:n_e].reshape(P, 3).astype(LD)
        self.Vinv = _inv3(V)
        bL = np.asarray(b, dtype=LD)
        self.rhs = self.F.T @ bL - self.F.T @ (self.E @ self._vinv(self.E.T @ bL))
        # magnitudes of the terms, in float64
        V64 = V.astype(float)
        sv = 1.0 / np.sqrt(np.einsum("pii->pi", V64))
        ev = np.linalg.eigvalsh(sv[:, :, None] * V64 * sv[:, None, :])
        kp = ev[:, -1] / ev[:, 0]   # condition number of each point block scaled to a unit diagonal
        self.kappa_V = float(kp.max())
        Vi = np.linalg.inv(V64)
        Vinv64 = sps.bsr_matrix((Vi, np.arange(P), np.arange(P + 1)), shape=(n_e, n_e)).tocsr()
        W = (E64.T @ F64).tocsr()
        VW = Vinv64 @ W
        T = (W.T @ VW).tocsr()
        FtF = (F64.T @ F64).tocsr()
        # a float64 V_p^-1 carries a relative error of kappa(V_p) u, so each point's terms enter with that weight
        Vk = sps.bsr_matrix((kp[:, None, None] * Vi, np.arange(P), np.arange(P + 1)), shape=(n_e, n_e)).tocsr()
        Tk = W.T @ (Vk @ W)
        yk = np.abs(Vk @ (E64.T @ b))
        # taken on the system scaled to a unit diagonal of F'F + D_f^2, which the factorisation is invariant under: with
        # column scales spread over six decades unscaled norms would see only the largest columns
        self.h = h = 1.0 / np.sqrt(FtF.diagonal() + d2[n_e:])
        H = sps.diags(h)
        self.den_mat = spla.norm(H @ FtF @ H) + spla.norm(H @ Tk @ H) + float((h * h * d2[n_e:]).max(initial=0.0))
        self.den_vec = np.linalg.norm(h * (F64.T @ b)) + np.linalg.norm(h * (abs(W).T @ yk))
        self.S = (FtF - T + sps.diags(d2[n_e:])).tocsr()
        self.norm_VW = spla.norm(VW)
        self.VW, self.Vinv64 = VW, Vinv64
        self.J, self.b, self.d2 = J, np.asarray(b, dtype=float), d2

    def _vinv(self, y):
        return np.einsum("pij,pj->pi", self.Vinv, y.reshape(self.P, 3)).ravel()

    def eta(self, x_f):
        xL = np.asarray(x_f, dtype=LD)
        Fx = self.F @ xL
        Sx = self.F.T @ Fx + self.Df2 * xL - self.F.T @ (self.E @ self._vinv(self.E.T @ Fx))
        return _norm(self.h.astype(LD) * (self.rhs - Sx)) / (self.den_mat * np.linalg.norm(x_f / self.h) + self.den_vec)

    def scaled_err(self, a, b):
        """|a - b| / |b| of camera blocks in the norm of the scaled system."""
        return float(np.linalg.norm((a - b) / self.h) / np.linalg.norm(b / self.h))

    def kappa(self, x_f):
        """The condition number the camera block's forward error is bounded with: |(H S H)^-1| (den_mat + den_vec /
        |H^-1 x_f|), H = diag(h), from the smallest eigenvalue over the connected components of S's block pattern.
        Sets kappa2 = kappa_2(H S H) <= kappa."""
        C = self.C
        S = self.S.tocoo()
        nc, label = connected_components(sps.csr_matrix((np.ones(S.nnz), (S.row // 9, S.col // 9)), shape=(C, C)), directed=False)
        lo, hi = np.inf, 0.0
        for k in range(nc):
            idx = (9 * np.flatnonzero(label == k)[:, None] + np.arange(9)).ravel()
            h = self.h[idx]
            ev = np.linalg.eigvalsh(h[:, None] * self.S[idx][:, idx].toarray() * h[None, :])
            assert ev[0] > 0.0
            lo, hi = min(lo, ev[0]), max(hi, ev[-1])
        self.kappa2 = hi / lo
        return (self.den_mat + self.den_vec / np.linalg.norm(x_f / self.h)) / lo

    def solution(self):
        """x_ref, refined with longdouble residuals of the full system; (x_ref, relative correction of each step).  The
        float64 solver inside the refinement eliminates the points with this class's V^-1 and factors S + D_f^2 with
        scipy's splu (SuperLU on the whole of J'J + D^2 takes a minute where the camera block is dense)."""
        n_e = 3 * self.P
        lu = spla.splu(self.S.tocsc())

        def solve(r):
            re, rf = r[:n_e], r[n_e:]
            xf = lu.solve(rf - self.VW.T @ re)
            return np.concatenate([self.Vinv64 @ re - self.VW @ xf, xf])
        JL, d2L = self.J.astype(LD), self.d2.astype(LD)
        JtbL = JL.T @ self.b.astype(LD)
        x = solve(self.J.T @ self.b).astype(LD)
        rel = []
        for step in range(1, REFINE_STEPS + 2):
            r = JtbL - JL.T @ (JL @ x) - d2L * x
            dx = solve(r.astype(float))
            x = x + dx.astype(LD)
            rel.append(float(np.linalg.norm(dx[n_e:] / self.h) / _norm(x[n_e:] / self.h)))
            if rel[-1] < 1e-18 or (len(rel) > 1 and rel[-1] > 0.5 * rel[-2]):
                break
        return x, rel


def check_solution(x, ref, kappa, x_ref, record=None, tag=""):
    """Backward error of the camera block, forward error of both blocks; returns (eta / u, camera forward error /
    (kappa u))."""
    n_e = 3 * ref.P
    eta = ref.eta(x[n_e:])
    xr = np.asarray(x_ref, dtype=float)
    ef = np.linalg.norm(x[n_e:] - xr[n_e:])
    ee = np.linalg.norm(x[:n_e] - xr[:n_e])
    bound_e = ref.norm_VW * ef + C_X * U * ref.kappa_V * (np.linalg.norm(xr[:n_e]) + ref.norm_VW * np.linalg.norm(xr[n_e:]))
    fwd = ref.scaled_err(x[n_e:], xr[n_e:])
    out = (eta / U, fwd / (kappa * U))
    if record is not None:
        record(tag, "eta/bound %.3g  fwd/bound %.3g  pts/bound %.3g  kappa %.2e  kappa2 %.2e  kappa_V %.2e  refine %s" % (
            out[0] / C_ETA, out[1] / C_X, ee / max(bound_e, 1e-300), kappa, ref.kappa2, ref.kappa_V,
            "/".join("%.1e" % r for r in ref.rel)))
    assert eta <= C_ETA * U, (tag, eta)
    assert fwd <= C_X * kappa * U, (tag, fwd, kappa)
    assert ee <= bound_e, (tag, ee, bound_e)
    return out


def reference_for(gpu, s, b, D):
    J = jacobian(gpu, s.C, s.P, s.cam, s.pt)
    return checked_reference(J, s.P, s.C, b, D)


def checked_reference(J, P, C, b, D):
    """(Reference, kappa, x_ref).  The refinement is asserted to have converged: within REFINE_STEPS steps, to a last
    correction 100 times below the forward bound, and contracting by at least 10 from its first correction to its second
    (unless the first is already that far below the bound), so that the error left in x_ref is of the order of the last
    correction, not a multiple of it.  ref.rel keeps the corrections."""
    ref = Reference(J, P, C, b, D)
    x_ref, rel = ref.solution()
    kappa = ref.kappa(np.asarray(x_ref[3 * P:], dtype=float))
    target = 1e-2 * C_X * kappa * U
    assert len(rel) <= REFINE_STEPS and (rel[-1] < 1e-18 or rel[-1] <= target), (rel, kappa)
    assert len(rel) == 1 or rel[1] <= 0.1 * rel[0] or rel[0] <= target, (rel, kappa)
    ref.rel = rel
    return ref, kappa, x_ref


def first_sparse_solve(gpu, b, D, capfd):
    """The first sparse solve of a handle, which runs the analysis, with its plan line: (x, its, term, plan fields)."""
    capfd.readouterr()
    os.environ["B200_VERBOSE"] = "1"
    try:
        out = gpu.sparse_schur_solve(b, D)
    finally:
        del os.environ["B200_VERBOSE"]
    err = capfd.readouterr().err
    m = PLAN_RE.search(err)
    assert m, err
    return out + (tuple(int(g) for g in m.groups()),)


# ---- section: every structure, value kind and damping

@pytest.mark.parametrize("name", STRUCTURES)
def test_structure(name, cs, sm_count, capfd, record_property):
    s = Structure(cs, name)
    for kind in ("geometric", "random"):
        gpu = s.problem(cs)
        b = load(gpu, s, kind)
        for radius in RADII:
            if radius is None and kind == "geometric":
                continue
            D = lm_diagonal(gpu, radius)
            if radius == RADII[0]:
                x, its, term, (ns, widest, height, ctas) = first_sparse_solve(gpu, b, D, capfd)
                assert ns == s.lay.ns and widest == 9 * s.lay.width.max()
                # one 256-thread CTA per SM (sparse_factor_kernel's registers allow no second), at most 2 ns of them
                assert ctas == min(2 * ns, sm_count)
                if name == "forest":
                    assert 2 * ns >= 4 * ctas
            else:
                x, its, term = gpu.sparse_schur_solve(b, D)
            assert (its, term) == (1, cs.LS_SUCCESS)
            ref, kappa, x_ref = reference_for(gpu, s, b, D)
            tag = "%s/%s/%s" % (name, kind, radius)
            check_solution(x, ref, kappa, x_ref, record_property, tag)
            if 9 * s.C <= 4000:
                xd, _, termd = gpu.dense_schur_solve(b, D)
                assert termd == cs.LS_SUCCESS
                assert ref.scaled_err(x[3 * s.P:], xd[3 * s.P:]) <= 2 * C_X * kappa * U, tag
        gpu.close()


# ---- failure, recovery and reuse

def raw_sparse_solve(cs, gpu, b, D, sentinel=-7.25):
    """b200_sparse_schur_solve into a sentinel-filled buffer (the binding pre-fills NaN): (x, termination)."""
    from ceres_solver_b200 import binding as Bd
    x = np.full(gpu.num_parameters, sentinel)
    summ = Bd.SolverSummary()
    b = np.ascontiguousarray(b, dtype=float)
    D = None if D is None else np.ascontiguousarray(D, dtype=float)
    rc = cs.lib().b200_sparse_schur_solve(gpu.h, Bd._d(b), Bd._d(D), Bd._d(x), ctypes.byref(summ))
    assert rc == 0
    return x, summ.termination_type


@pytest.mark.parametrize("fault", ["nan_first", "inf_root", "inf_D"])
def test_failure_and_recovery(fault, cs):
    """A non-finite Jacobian block in the first supernode eliminated or in a root, or an infinite entry of D_f: FAILURE
    with the caller's buffer untouched; the same handle then solves the clean system as a fresh handle does."""
    s = Structure(cs, "band")
    gpu = s.problem(cs)
    b = load(gpu, s, "random")
    v = gpu.jacobian_values()
    D = lm_diagonal(gpu, 1e4)
    vb, Db = v.copy(), D.copy()
    N, P = len(s.cam), s.P
    if fault == "inf_D":
        Db[3 * P + 9 * int(s.perm[s.C // 2]) + 4] = np.inf
    else:
        c = int(s.perm[0] if fault == "nan_first" else s.perm[-1])
        row = int(np.flatnonzero(s.cam == c)[0])
        vb[6 * N + 18 * row + 7] = np.nan if fault == "nan_first" else np.inf
    gpu.set_jacobian_values(vb)
    x, term = raw_sparse_solve(cs, gpu, b, Db)
    assert term == cs.LS_FAILURE and np.all(x == -7.25)
    gpu.set_jacobian_values(v)
    x, term = raw_sparse_solve(cs, gpu, b, D)
    assert term == cs.LS_SUCCESS
    ref, kappa, x_ref = reference_for(gpu, s, b, D)
    check_solution(x, ref, kappa, x_ref, tag=fault)
    fresh = s.problem(cs)
    load(fresh, s, "random")
    xf, _, tf = fresh.sparse_schur_solve(b, D)
    assert tf == cs.LS_SUCCESS and ref.scaled_err(x[3 * P:], xf[3 * P:]) <= 2 * C_X * kappa * U
    gpu.close()
    fresh.close()


def test_singular_then_recovery(cs, oracle):
    """Zero focal length and no damping of the cameras: S + D_f^2 singular, FAILURE with the buffer untouched; then the
    same handle with the LM diagonal."""
    case = Case(cs, oracle, L.zero_focal_bal())
    gpu = case.gpu
    ok, _, res, _ = gpu.evaluate(case.state)
    assert ok
    D = np.zeros(gpu.num_parameters)
    D[:3 * gpu.P] = 1.0
    x, term = raw_sparse_solve(cs, gpu, res, D)
    assert term == cs.LS_FAILURE and np.all(x == -7.25)
    D = lm_diagonal(gpu, 1e4)
    x, term = raw_sparse_solve(cs, gpu, res, D)
    assert term == cs.LS_SUCCESS
    J = jacobian(gpu, case.rp.C, case.rp.P, case.rp.row_cam, case.rp.row_pt)
    ref, kappa, x_ref = checked_reference(J, gpu.P, gpu.C, res, D)
    check_solution(x, ref, kappa, x_ref, tag="zero_focal")
    case.close()


def test_reuse(cs):
    """Several solves with different D on one handle, each against a fresh handle (L is re-zeroed, the counters and the
    ticket reset; the results are not bitwise equal because the reduced right-hand side is summed with FP64 REDs)."""
    s = Structure(cs, "loop")
    gpu = s.problem(cs)
    b = load(gpu, s, "random")
    J = jacobian(gpu, s.C, s.P, s.cam, s.pt)
    for radius in (1e4, 1e-1, None, 10.0, 1e4):
        D = lm_diagonal(gpu, radius)
        x, _, term = gpu.sparse_schur_solve(b, D)
        fresh = s.problem(cs)
        load(fresh, s, "random")
        xf, _, tf = fresh.sparse_schur_solve(b, D)
        fresh.close()
        assert term == tf == cs.LS_SUCCESS
        ref = Reference(J, s.P, s.C, b, D)
        assert ref.scaled_err(x[3 * s.P:], xf[3 * s.P:]) <= 2 * C_X * ref.kappa(xf[3 * s.P:]) * U, radius
    gpu.close()


@pytest.mark.parametrize("host_boundary", [False, True])
def test_lm_loop_many_supernodes(host_boundary, cs, oracle):
    """Four iterations of the exact-step LM loop with SPARSE_SCHUR against the oracle's DENSE_SCHUR loop, on a photo
    collection whose factor has 10 supernodes (the C16 transcript has one).  A fifth iteration is not compared: the
    reduced right-hand side is summed with FP64 REDs, so the trajectory moves from run to run, and by the fifth record the
    gradient has dropped far enough for that to show.  Measured over eight GPU runs (H100): the gradient max norm of
    record 5 spreads by 1.2e-8 relative between runs and lies up to 7.9e-9 from the oracle's, above
    compare_lm_traces_exact's 1e-9; record 4's lies up to 2.1e-9 from it, inside the 1e-12 x initial-gradient floor."""
    from ceres_solver_b200 import bal as B
    bal = B.synthetic_clusters(150, 8000, 40000)
    case = Case(cs, oracle, bal)
    _, st = cs.plan_sparse_schur(case.rp.C, case.rp.P, case.rp.row_cam, case.rp.row_pt)
    assert st["supernodes"] >= 10
    _, recs_o, _ = L.oracle_solve(case.orc, case.state, linear_solver_type=L.DENSE_SCHUR, max_num_iterations=4)
    _, recs = L.gpu_solve(case.gpu, case.state, host_boundary, linear_solver_type=cs.SPARSE_SCHUR, max_num_iterations=4)
    compare_lm_traces_exact(recs, recs_o)
    case.close()
