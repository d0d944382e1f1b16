"""The covariance reference of tests/covariance_reference.py, on the CPU: the Schur form against the literal
(J_red'J_red)^-1 (what SuiteSparseQR's R^-1 R^-T computes), against scipy's SVD inverse on a full-rank problem (the
DENSE_SVD semantics), zeros on constant blocks, and the conditioning test of b200_covariance_compute on C16: the ungauged
problem and two gauged ones fall on the intended sides of min_reciprocal_condition_number = 1e-14, in float64 and in
np.longdouble (the values are recorded in DESIGN §3.9).  The Jacobians come from the oracle's own program."""
import numpy as np
import pytest
import scipy.linalg as sla

from tests.constant_blocks_reference import fixed_components, jacobian_matrix
from tests.covariance_reference import SchurCovariance, literal_covariance

THRESHOLD = 1e-14


class _Rows:
    """The oracle's program of a BAL problem: its C, P and row structure, which its Jacobian values are laid out in."""

    def __init__(self, orc):
        self.C, self.P = orc.C, orc.P
        self.row_cam, self.row_pt = np.asarray(orc.row_cam), np.asarray(orc.row_pt)


def _oracle_problem(oracle, bal):
    """(rows, Jacobian values) of the oracle's own program of `bal` at the library's state, built from the original BAL
    rows as every oracle caller does; the values are in the oracle's row order, whose structure comes with them."""
    from ceres_solver_b200 import bal as B
    rp = B.ReducedProgram(bal)
    state = rp.state(bal)
    orc = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())
    rows = _Rows(orc)
    # the oracle's program is the library's reduced program: the same rows, the same block order
    assert np.array_equal(rows.row_cam, rp.row_cam) and np.array_equal(rows.row_pt, rp.row_pt)
    ok, _, _, _ = orc.evaluate(state)
    assert ok
    return rows, np.asarray(orc.jacobian().values(), float)


@pytest.fixture(scope="module")
def tiny(oracle):
    from tests import lm_cases as L
    return _oracle_problem(oracle, L.tiny_bal())


def _gauge(rp, cameras=(0,), points=3, seed=0):
    cam = np.zeros(rp.C, bool)
    cam[list(cameras)] = True
    row_cam, row_pt = np.asarray(rp.row_cam), np.asarray(rp.row_pt)
    seen = np.zeros(rp.P, bool)
    seen[row_pt[cam[row_cam]]] = True
    pts = np.zeros(rp.P, bool)
    if points:
        pts[np.random.RandomState(seed).choice(np.flatnonzero(~seen), size=points, replace=False)] = True
    return cam, pts


def test_schur_form_is_the_literal_inverse(tiny):
    rp, v = tiny
    cam, pts = _gauge(rp)
    fixed = fixed_components(rp.C, rp.P, cam, pts)
    lit = literal_covariance(v, rp.row_cam, rp.row_pt, rp.P, rp.C, fixed)
    sc = SchurCovariance(v, rp.row_cam, rp.row_pt, rp.P, rp.C, fixed)
    assert sc.Z is not None and sc.rcond >= THRESHOLD
    full = np.asarray(sc.full(rp.P, rp.C), float)
    assert np.abs(full - lit).max() <= 1e-9 * np.abs(lit).max()
    # the point blocks the library returns are the diagonal 3x3 blocks of it
    for p in range(rp.P):
        assert np.allclose(np.asarray(sc.points[p], float), lit[3 * p:3 * p + 3, 3 * p:3 * p + 3], rtol=1e-9,
                           atol=1e-9 * np.abs(lit).max())


def test_full_rank_equals_svd_inverse(tiny):
    """With the gauge fixed the reduced J'J has full rank, and DENSE_SVD's pseudo-inverse is the inverse."""
    rp, v = tiny
    cam, pts = _gauge(rp, cameras=(0, 1), points=0)
    fixed = fixed_components(rp.C, rp.P, cam, pts)
    J = jacobian_matrix(v, rp.row_cam, rp.row_pt, rp.P, rp.C).toarray()[:, ~fixed]
    pinv = sla.pinv(J.T @ J)
    sc = SchurCovariance(v, rp.row_cam, rp.row_pt, rp.P, rp.C, fixed)
    full = np.asarray(sc.full(rp.P, rp.C), float)[np.ix_(~fixed, ~fixed)]
    assert np.abs(full - pinv).max() <= 1e-8 * np.abs(pinv).max()


def test_constant_blocks_are_zero(tiny):
    rp, v = tiny
    cam, pts = _gauge(rp)
    fixed = fixed_components(rp.C, rp.P, cam, pts)
    sc = SchurCovariance(v, rp.row_cam, rp.row_pt, rp.P, rp.C, fixed)
    full = np.asarray(sc.full(rp.P, rp.C), float)
    assert not full[fixed].any() and not full[:, fixed].any()
    assert not np.asarray(sc.points, float)[pts].any()


@pytest.fixture(scope="module")
def c16_program(oracle, c16):
    from tests import lm_cases as L
    return _oracle_problem(oracle, L.c16_bal(c16))


# The minimum of d_k / A_kk on C16 (DESIGN §3.9), the same in float64 and np.longdouble: on the ungauged problem S keeps
# the 7-dimensional similarity gauge (seven eigenvalues of the unit-diagonal S below 4e-15) and its Cholesky factorisation
# meets a non-positive pivot, so the minimum is 0; with camera 0 and 1 % of the points constant, or cameras 0 and 1, it is
# 2.825e-4.  Both sides are asserted with a 100x margin around min_reciprocal_condition_number = 1e-14.
C16_SETS = {"ungauged": dict(cameras=(), points=0), "camera0_points1pct": dict(cameras=(0,), points=-1),
            "two_cameras": dict(cameras=(0, 1), points=0)}


@pytest.mark.parametrize("name", sorted(C16_SETS))
def test_c16_conditioning(c16_program, name):
    rp, v = c16_program
    kw = dict(C16_SETS[name])
    if kw["points"] == -1:
        kw["points"] = rp.P // 100
    cam, pts = _gauge(rp, **kw)
    fixed = fixed_components(rp.C, rp.P, cam, pts)
    vals = {}
    for dtype in (np.float64, np.longdouble):
        sc = SchurCovariance(v, rp.row_cam, rp.row_pt, rp.P, rp.C, fixed, dtype=dtype)
        vals["float64" if dtype is np.float64 else "longdouble"] = sc.rcond
    print("[covariance] C16 %s: min d_k / A_kk float64 %.4e, longdouble %.4e" % (name, vals["float64"], vals["longdouble"]))
    for r in vals.values():
        if name == "ungauged":
            assert r <= THRESHOLD / 100
        else:
            assert r >= THRESHOLD * 100
