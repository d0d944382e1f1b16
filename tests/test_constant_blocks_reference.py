"""CPU guard of tests/constant_blocks_reference.py, the reduced-program reference the GPU tests of
b200_set_constant_blocks compare against, and of the construction their failure test relies on."""
import numpy as np
import pytest

from tests import constant_blocks_reference as R
from tests import eval_failure_cases as F
from tests import lm_cases as L
from tests.entry_points import compare_lm_traces_exact


@pytest.fixture(scope="module")
def tiny(oracle):
    from ceres_solver_b200 import bal as B
    bal = B.synthetic("tiny")
    rp = B.ReducedProgram(bal)
    orc = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())
    state = rp.state(bal)
    ok, _, res, _ = orc.evaluate(state)
    assert ok
    return rp, orc, state, res


def _sets(rp):
    cam0 = np.zeros(rp.C, dtype=bool)
    cam0[0] = True
    seen0 = np.zeros(rp.P, dtype=bool)
    seen0[rp.row_pt[rp.row_cam == 0]] = True
    pts = np.zeros(rp.P, dtype=bool)
    pts[np.flatnonzero(~seen0)[:3]] = True
    return {"camera0": (cam0, None), "camera0_points": (cam0, pts), "points": (None, pts)}


def test_nothing_constant_is_the_oracle_solve(tiny):
    """With no constant block, the reference's solve is the oracle's DENSE_SCHUR solve of the full program."""
    rp, orc, _, res = tiny
    J = orc.jacobian()
    Js = R.jacobian_matrix(J.values(), rp.row_cam, rp.row_pt, rp.P, rp.C)
    D = np.random.RandomState(0).uniform(0.1, 1.0, rp.num_parameters)
    x = R.reduced_solve(Js, res, D, R.fixed_components(rp.C, rp.P))
    xo, _, _ = J.linear_solve(rp.P, res, D, solver=1)
    assert np.linalg.norm(x - xo) <= 1e-9 * np.linalg.norm(xo)
    # and the products: J x against the oracle's
    v = np.random.RandomState(1).normal(size=rp.num_parameters)
    assert np.allclose(Js @ v, J.right_multiply(v), rtol=0, atol=1e-12 * np.abs(Js @ v).max())


@pytest.mark.parametrize("name", ["camera0", "camera0_points", "points"])
@pytest.mark.parametrize("d_scale", [0.3, 1.0])
def test_reduced_solve_is_the_dense_solve(tiny, name, d_scale):
    """(Holding one camera constant leaves the scale gauge: without D the reduced normal equations are singular.)"""
    rp, orc, _, res = tiny
    cam, pts = _sets(rp)[name]
    fixed = R.fixed_components(rp.C, rp.P, cam, pts)
    Js = R.jacobian_matrix(orc.jacobian().values(), rp.row_cam, rp.row_pt, rp.P, rp.C)
    D = d_scale * np.random.RandomState(2).uniform(0.1, 1.0, rp.num_parameters)
    x = R.reduced_solve(Js, res, D, fixed)
    xd = R.reduced_dense_solve(Js, res, D, fixed)
    assert np.all(x[fixed] == 0.0)
    assert np.linalg.norm(x - xd) <= 1e-10 * np.linalg.norm(xd)


def test_constant_sets_cover_every_row_class():
    """constant_sets never makes a row fully constant, and takes points of each class it finds."""
    rng = np.random.RandomState(3)
    P, C = 400, 30
    deg = np.concatenate([rng.randint(2, 30, size=P - 4), [40, 90, 150, 300]])
    row_pt = np.repeat(np.arange(P), deg)
    row_cam = np.concatenate([rng.choice(C, size=d, replace=d > C) for d in deg])
    cam, pts = R.constant_sets(row_cam, row_pt, P, C, per_class=1)
    assert cam.sum() == 2
    assert not np.any(cam[row_cam] & pts[row_pt])
    assert pts.sum() >= 1


def test_cost_overflow2_point_cells_are_finite():
    """The failure test holds the camera of each cost_overflow row constant and expects every J mode to succeed: its only
    non-finite cells must be the camera's.  The analytic cells of snavely_reprojection_error.h on a zeroed camera
    (R = I, t = 0, f = 1e3, l1 = l2 = 0) and X = (-1.2e151, 0, 1): d r / d X is f (-1/z, 0, x/z^2) per coordinate
    (the distortion terms are 0 * finite), d r / d l1 = f r2 x_p with r2 = x_p^2 = 1.44e302 overflows."""
    f, l1, l2 = F.OVERFLOW_INTRINSICS
    X = np.array(F.OVERFLOW_X)
    p = X.copy()
    xp, yp = -p[0] / p[2], -p[1] / p[2]
    r2 = xp * xp + yp * yp
    dist = 1.0 + r2 * (l1 + l2 * r2)
    ddist = l1 + 2.0 * l2 * r2
    ip2 = 1.0 / p[2]
    fd, fx, fy = f * dist, f * ddist * xp, f * ddist * yp
    q = (-2.0 * xp * ip2, -2.0 * yp * ip2, -2.0 * r2 * ip2)
    with np.errstate(over="ignore", invalid="ignore"):
        A = np.array([[fx * q[0] - fd * ip2, fx * q[1], fx * q[2] - fd * xp * ip2],
                      [fy * q[0], fy * q[1] - fd * ip2, fy * q[2] - fd * yp * ip2]])
        d_l1 = f * r2 * xp
    assert np.all(np.isfinite(A)), A      # the point cells (R = I)
    assert not np.isfinite(d_l1)           # a camera cell


def c16_sets(P, C, row_cam, row_pt):
    """The constant sets of the C16 trajectories: camera 0 (the gauge), camera 0 and three points no row of camera 0
    sees, and the three points alone.  (Shared with tests/test_gpu_constant_blocks.py.)"""
    cam = np.zeros(C, bool)
    cam[0] = True
    seen = np.zeros(P, bool)
    seen[np.asarray(row_pt)[np.asarray(row_cam) == 0]] = True
    pts = np.zeros(P, bool)
    pts[np.flatnonzero(~seen)[[0, 100, 1000]]] = True
    return {"gauge": (cam, None), "gauge_points": (cam, pts), "points": (None, pts)}


@pytest.fixture(scope="module")
def c16_state(c16):
    from ceres_solver_b200 import bal as B
    bal = L.c16_bal(c16)
    return bal, B.ReducedProgram(bal).state(bal)


@pytest.mark.parametrize("solver", ["iterative", "dense"])
def test_nothing_constant_is_the_oracle_transcript(oracle, c16_state, solver):
    """With nothing constant the reduced program is the oracle's program: its LM loop reproduces the oracle's own C16
    transcript (ITERATIVE_SCHUR with SCHUR_JACOBI, and DENSE_SCHUR)."""
    bal, state = c16_state
    rp = R.ReducedProgram(oracle, bal)
    o = rp.default_options()
    o.num_threads = 8
    o.max_num_iterations = 5
    o.linear_solver = 0 if solver == "iterative" else 1
    best_o, recs_o, _ = rp.base.solve(state, o)
    best, recs = rp.solve(state, o)
    compare_lm_traces_exact(recs, recs_o)
    assert np.linalg.norm(best - best_o) <= 1e-9 * np.linalg.norm(best_o)


@pytest.mark.parametrize("name", ["gauge", "gauge_points", "points"])
def test_reduced_program_solve_is_the_dense_solve(oracle, c16_state, name):
    """The reduced program's Jacobian is the full one without the constant columns, and its DENSE_SCHUR solve (num_elim
    = the variable points, the constant points' rows without an e block) equals a direct solve of its normal equations."""
    bal, state = c16_state
    full = R.ReducedProgram(oracle, bal)
    cam, pts = c16_sets(full.P, full.C, full.base.row_cam, full.base.row_pt)[name]
    rp = R.ReducedProgram(oracle, bal, cam, pts)
    rp.state0 = state
    ok, cost, r, g = rp.evaluate(rp.reduce(state))
    full.state0 = state
    ok_f, cost_f, r_f, g_f = full.evaluate(state)
    assert ok and ok_f and cost == cost_f
    keep = ~rp.fixed
    assert np.linalg.norm(g - g_f[keep]) <= 1e-12 * np.linalg.norm(g_f[keep])
    Jf = R.jacobian_matrix(full.base.jacobian().values(), full.base.row_cam, full.base.row_pt, full.P, full.C)
    D = np.random.RandomState(4).uniform(0.5, 1.0, full.num_parameters)
    x_dense = R.reduced_solve(Jf, r_f, D, rp.fixed)   # (pinned to a dense numpy solve on `tiny` above)
    x, _, term = rp.jacobian().linear_solve(rp.P, r, D[keep], solver=1)
    assert term == 0
    assert np.linalg.norm(x - x_dense[keep]) <= 1e-8 * np.linalg.norm(x_dense[keep])   # (unscaled normal equations: cond ~1e8)


@pytest.mark.parametrize("name", ["gauge", "gauge_points", "points"])
def test_reduced_program_lm_keeps_constant_blocks(oracle, c16_state, name):
    """The reduced loop converges, leaves the constant blocks as they were and moves the others."""
    bal, state = c16_state
    full = R.ReducedProgram(oracle, bal)
    cam, pts = c16_sets(full.P, full.C, full.base.row_cam, full.base.row_pt)[name]
    rp = R.ReducedProgram(oracle, bal, cam, pts)
    o = rp.default_options()
    o.num_threads, o.max_num_iterations, o.linear_solver = 8, 3, 1
    best, recs = rp.solve(state, o)
    assert np.array_equal(best[rp.fixed], state[rp.fixed])
    assert recs[-1]["cost"] < recs[0]["cost"]
