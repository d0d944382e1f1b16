"""b200_set_constant_blocks (Problem::SetParameterBlockConstant) on the device, against the handle without constant blocks
and against the reduced program of tests/constant_blocks_reference.py.

A constant block is handled as Ceres' reduced program handles it: its Jacobian columns are exactly zero, and the solves use
D' = 1 on its components.  So, on every kernel configuration of the evaluate (warp tiles, CTA tiles for > 32-row points,
the huge-point slices, CTA tiles everywhere):
  - with nothing constant, every bit is the one of a handle that never made the call;
  - with constant blocks, their cells are exactly 0 and every other cell, the residuals and the cost are bit-identical;
  - every solve returns exact zeros on the constant components and the reduced program's solution elsewhere;
  - the trust-region loop returns the constant blocks bitwise unchanged and takes |x| over the variable blocks.
Each fixture asserts the plan it ran (B200_VERBOSE), as tests/test_gpu_dispatch.py does.
"""
import os

import numpy as np
import pytest

from tests import constant_blocks_reference as R
from tests import eval_failure_cases as F
from tests import lm_cases as L
from tests.entry_points import compare_lm_traces_exact
from tests.test_constant_blocks_reference import c16_sets
from tests.test_gpu_dispatch import EXPECT, _make, problem_plan  # noqa: F401  (problem_plan: a fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as cs
    cs.lib()
    return cs


def _bal(name, c16):
    if name == "c16":
        return L.c16_bal(c16)
    if name == "circle":
        from tests.test_gpu_orders import _make as make_orders
        return make_orders("circle")
    if name == "sequence":
        from tests.test_gpu_explicit_schur import _sequence_with_duplicates
        return _sequence_with_duplicates()
    return _make(name)


# (fixture, plan fields asserted): C16 runs the warp-tile evaluate with its > 32-row points on CTA tiles (one camera vector
# per warp); circle the same with shared camera vectors (16 warps); id_range and tile the CTA-tile evaluate with huge
# points; v4_narrow, direct_v3, dups_direct and dups_id_range the remaining warp-tile configurations of
# tests/test_gpu_dispatch.py; sequence a sparse camera graph, on which the PCG runs on the explicit S
FIXTURES = {"c16": dict(mul="v4-owned"), "circle": dict(mul="v4", mul_w=16),
            **{name: EXPECT[name][0] for name in ("id_range", "tile", "v4_narrow", "direct_v3", "dups_direct", "dups_id_range")},
            "sequence": {}}
# the fixtures on which ITERATIVE_SCHUR with SCHUR_JACOBI runs the explicit-S PCG (the camera graph is sparse)
EXPLICIT = ("sequence",)


class Setup:
    def __init__(self, cs, bal):
        from ceres_solver_b200 import bal as B
        self.rp = rp = B.ReducedProgram(bal)
        self.state = rp.state(bal)
        self.free = cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs)     # never holds anything constant
        self.gpu = cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs)
        self.cam, self.pts = R.constant_sets(rp.row_cam, rp.row_pt, rp.P, rp.C)
        self.fixed = R.fixed_components(rp.C, rp.P, self.cam, self.pts)

    def cell_mask(self):
        """[24N] True on the cells of constant blocks, in the library's value layout."""
        rp, N = self.rp, self.rp.N
        e = np.repeat(self.pts[rp.row_pt], 6)
        f = np.repeat(self.cam[rp.row_cam], 18)
        return np.concatenate([e, f])

    def close(self):
        self.free.close()
        self.gpu.close()


@pytest.fixture(scope="module", params=sorted(FIXTURES))
def setup(request, cs, c16):
    s = Setup(cs, _bal(request.param, c16))
    s.name = request.param
    yield s
    s.close()


def test_plan(setup, problem_plan, cs, monkeypatch, capfd):
    rp = setup.rp
    if setup.name in EXPLICIT:
        monkeypatch.setenv("B200_VERBOSE", "1")
        capfd.readouterr()
        cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs).close()
        monkeypatch.delenv("B200_VERBOSE")
        err = capfd.readouterr().err
        assert "[b200ba] S plan: explicit," in err, err
    plan = problem_plan(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs)
    for k, v in FIXTURES[setup.name].items():
        assert plan[k] == v, (setup.name, k, plan[k], v)
    deg = np.bincount(rp.row_pt, minlength=rp.P)
    # the constant set covers constant and variable points of every row class the problem has
    for lo, hi in ((1, 32), (33, 128), (129, 1 << 30)):
        cls = (deg >= lo) & (deg <= hi)
        if cls.sum() > 2:
            assert setup.pts[cls].any() and (~setup.pts[cls]).any(), (lo, hi)


def _eval_all(gpu, state):
    ok, cost, res, grad = gpu.evaluate(state)
    assert ok
    return cost, res, grad, gpu.jacobian_values()


def test_nothing_constant_is_the_old_path(setup):
    """Bit for bit wherever two runs of the untouched handle agree bit for bit (cost, residuals, J); the gradient's camera
    part is summed with atomics in some configurations, and is held to 1e-13 where it is not reproducible."""
    s = setup
    a = _eval_all(s.free, s.state)
    b = _eval_all(s.free, s.state)
    exact = [np.array_equal(x, y) for x, y in zip(a, b)]
    assert exact[0] and exact[1] and exact[3]
    for flags in ((None, None), (np.zeros(s.rp.C, bool), np.zeros(s.rp.P, bool))):
        s.gpu.set_constant_blocks(*flags)
        c = _eval_all(s.gpu, s.state)
        for x, y, bits in zip(a, c, exact):
            if bits:
                assert np.array_equal(x, y)
            else:
                assert np.linalg.norm(np.asarray(x) - y) <= 1e-13 * np.linalg.norm(x)
    if s.name == "c16":   # the LM trace with DENSE_SCHUR: bit for bit where two runs of the untouched handle agree so,
        # else (the gradient's atomics) as the untouched handle's second run compares with its first
        o = s.free.lm_options(max_num_iterations=5, linear_solver_type=1)
        xa, ra = s.free.lm_solve(s.state, o)
        xb, rb = s.free.lm_solve(s.state, o)
        xc, rc = s.gpu.lm_solve(s.state, o)
        if ra == rb:
            assert rc == ra and np.array_equal(xc, xa)
        else:
            compare_lm_traces_exact(rb, ra)
            compare_lm_traces_exact(rc, ra)


def test_evaluate_every_mode(setup):
    s = setup
    cost0, res0, grad0, J0 = _eval_all(s.free, s.state)
    s.gpu.set_constant_blocks(s.cam, s.pts)
    mask = s.cell_mask()
    try:
        # residuals, gradient and Jacobian
        ok, cost, res, grad = s.gpu.evaluate(s.state)
        assert ok and cost == cost0 and np.array_equal(res, res0)
        J = s.gpu.jacobian_values()
        assert np.all(J[mask] == 0.0)
        assert np.array_equal(J[~mask], J0[~mask])
        assert np.all(grad[s.fixed] == 0.0)
        g = ~s.fixed
        assert np.linalg.norm(grad[g] - grad0[g]) <= 1e-13 * np.linalg.norm(grad0[g])
        # the same against the reduced program: J'r of the masked Jacobian
        Js = R.jacobian_matrix(J, s.rp.row_cam, s.rp.row_pt, s.rp.P, s.rp.C)
        gr = Js.T @ res
        assert np.linalg.norm(grad - gr) <= 1e-12 * np.linalg.norm(gr)
        assert np.all(s.gpu.squared_column_norm()[s.fixed] == 0.0)
        # gradient only: J is computed and masked, the stored J is left as it is
        ok, cost_g, _, grad_g = s.gpu.evaluate(s.state, want_jacobian=False)
        assert ok and cost_g == cost0
        assert np.all(grad_g[s.fixed] == 0.0) and np.linalg.norm(grad_g - grad) <= 1e-13 * np.linalg.norm(grad)
        # Jacobian only
        s.gpu.set_jacobian_values(np.zeros_like(J))
        ok, cost_j, _, _ = s.gpu.evaluate(s.state, want_residuals=False, want_gradient=False)
        assert ok and cost_j == cost0 and np.array_equal(s.gpu.jacobian_values(), J)
        # J' x is 0 on the constant components; J x and the model cost change are those of the unconstrained handle's J
        # without the constant columns
        y = s.gpu.left_multiply(np.random.RandomState(0).normal(size=2 * s.rp.N))
        assert np.all(y[s.fixed] == 0.0)
        ok, _, res, _ = s.gpu.evaluate(s.state)
        J0m = np.where(mask, 0.0, J0)
        Jr = R.jacobian_matrix(J0m, s.rp.row_cam, s.rp.row_pt, s.rp.P, s.rp.C)
        x = np.random.RandomState(2).normal(size=s.rp.num_parameters)
        jx = Jr @ x
        assert np.linalg.norm(s.gpu.right_multiply(x) - jx) <= 1e-12 * np.linalg.norm(jx)
        mcc = -(jx @ (res + jx / 2.0))
        assert abs(s.gpu.model_cost_change(x) - mcc) <= 1e-12 * (abs(jx @ res) + jx @ jx / 2.0)
    finally:
        s.gpu.set_constant_blocks(None, None)


def _lm_D(gpu, radius=1e4):
    sq = gpu.squared_column_norm()
    return np.sqrt(np.clip(sq, 1e-6, 1e32) / radius)


def test_solves_against_the_reduced_program(setup, cs):
    s = setup
    s.gpu.set_constant_blocks(s.cam, s.pts)
    try:
        ok, _, res, _ = s.gpu.evaluate(s.state)
        assert ok
        J = s.gpu.jacobian_values()
        Js = R.jacobian_matrix(J, s.rp.row_cam, s.rp.row_pt, s.rp.P, s.rp.C)
        D = _lm_D(s.gpu)
        D0 = D.copy()
        D0[s.fixed] = 0.0
        # (the reference's direct solve of the reduced normal equations is only affordable on C16; on the larger fixtures
        # the solves are held to exact zeros on the constant components)
        full = s.name == "c16"
        x_ref = R.reduced_solve(Js, res, D, s.fixed) if full else None
        exact = [("dense", lambda d: s.gpu.dense_schur_solve(None, d)),
                 ("sparse_amd", lambda d: s.gpu.sparse_schur_solve(None, d))] if full else []
        for name, solve in exact:
            for d in (D, D0):
                x = solve(d)[0]
                assert np.all(x[s.fixed] == 0.0), name
                assert np.linalg.norm(x - x_ref) <= 1e-8 * np.linalg.norm(x_ref), name
        if full:
            s.gpu.set_linear_solver_ordering_type(cs.NESDIS)
            for mixed in (False, True):
                s.gpu.set_exact_solve_options(mixed, 2 if mixed else 0)
                for solve in (s.gpu.sparse_schur_solve, s.gpu.dense_schur_solve):
                    x = solve(None, D)[0]
                    assert np.all(x[s.fixed] == 0.0), (solve, mixed)
                    assert np.linalg.norm(x - x_ref) <= (1e-6 if mixed else 1e-8) * np.linalg.norm(x_ref), (solve, mixed)
            s.gpu.set_exact_solve_options(False, 0)
            s.gpu.set_linear_solver_ordering_type(cs.AMD)
        # ITERATIVE_SCHUR, every preconditioner and the SPSE initialisation, and with D = NULL: exact zeros on the
        # constant components.  On C16 also the values, against the reduced direct solve: every preconditioned solve
        # converges to it (to ~1e-9 measured); IDENTITY does not converge in 500 iterations on C16's unscaled system, with or
        # without constant blocks (NO_CONVERGENCE), so its values are not compared
        for pre, spse in ((cs.PRECOND_IDENTITY, 0), (cs.PRECOND_JACOBI, 0), (cs.PRECOND_SCHUR_JACOBI, 0),
                          (cs.PRECOND_SCHUR_POWER_SERIES_EXPANSION, 0), (cs.PRECOND_SCHUR_JACOBI, 1)):
            o = s.gpu.solver_options(preconditioner_type=pre, use_spse_initialization=spse,
                                     max_num_iterations=500 if full else 30, q_tolerance=0.0, r_tolerance=1e-14)
            for d in (D, D0, None):
                x = s.gpu.schur_solve(None, d, o)[0]
                assert np.all(x[s.fixed] == 0.0), (pre, spse)
            if full and pre != cs.PRECOND_IDENTITY:
                x, _, term = s.gpu.schur_solve(None, D, o)
                assert term == cs.LS_SUCCESS, (pre, spse)
                assert np.linalg.norm(x - x_ref) <= 1e-7 * np.linalg.norm(x_ref), (pre, spse)
        # the Schur pieces: (E'E + D'^2)^-1 is the identity on constant points, the back substitution 0 there
        s.gpu.schur_init(res, D)
        ete = s.gpu.schur_ete_inverse().reshape(-1, 9)
        assert np.array_equal(ete[s.pts], np.tile(np.eye(3).ravel(), (int(s.pts.sum()), 1)))
        y = s.gpu.schur_back_substitute(np.random.RandomState(1).normal(size=9 * s.rp.C))
        assert np.all(y[s.fixed] == 0.0)
    finally:
        s.gpu.set_constant_blocks(None, None)


def test_failure_only_in_constant_cells(cs, c16):
    """cost_overflow2 (tests/eval_failure_cases.py): the only non-finite cells are its cameras' (pinned on the CPU by
    tests/test_constant_blocks_reference.py).  With those cameras constant every J mode succeeds; with the points constant
    instead, it still fails."""
    s = Setup(cs, L.c16_bal(c16))
    try:
        rp = s.rp
        perm, _, _ = cs.plan_point_order(rp.C, rp.P, rp.row_cam, rp.row_pt)
        places = F.placements(s.state, rp.row_cam, rp.row_pt, rp.P, perm)
        rows = F.overflow_targets(places, s.state, rp.row_cam, rp.row_pt, rp.P)[:2]
        x = F.construct(s.state, rp.row_cam, rp.row_pt, rp.P, "cost_overflow2", rows)
        ok, _, _, _ = s.free.evaluate(x)
        assert not ok
        cam = np.zeros(rp.C, bool)
        cam[rp.row_cam[rows]] = True
        s.gpu.set_constant_blocks(cam, None)
        for kw in (dict(), dict(want_jacobian=False), dict(want_residuals=False, want_gradient=False)):
            ok, cost, _, _ = s.gpu.evaluate(x, **kw)
            assert ok and np.isfinite(cost), kw
        pts = np.zeros(rp.P, bool)
        pts[rp.row_pt[rows]] = True
        s.gpu.set_constant_blocks(None, pts)
        ok, _, _, _ = s.gpu.evaluate(x)
        assert not ok
        # a non-finite residual fails whatever is constant
        xr = F.construct(s.state, rp.row_cam, rp.row_pt, rp.P, "residual_nonfinite", rows[:1])
        cam1 = np.zeros(rp.C, bool)
        cam1[rp.row_cam[rows[0]]] = True
        s.gpu.set_constant_blocks(cam1, None)
        for kw in (dict(), dict(want_jacobian=False), dict(want_residuals=False, want_gradient=False, want_jacobian=False)):
            ok, _, _, _ = s.gpu.evaluate(xr, **kw)
            assert not ok, kw
    finally:
        s.close()


SETS = ("gauge", "gauge_points", "points")


def _c16_set(rp, name):
    return c16_sets(rp.P, rp.C, rp.row_cam, rp.row_pt)[name]


@pytest.fixture(scope="module")
def c16_setup(cs, c16):
    s = Setup(cs, L.c16_bal(c16))
    yield s
    s.close()


@pytest.fixture(scope="module")
def reduced(oracle, c16):
    """{set name: tests/constant_blocks_reference.py ReducedProgram of C16 with that set constant}."""
    bal = L.c16_bal(c16)
    out = {}
    for name in SETS:
        full = R.ReducedProgram(oracle, bal)
        cam, pts = c16_sets(full.P, full.C, full.base.row_cam, full.base.row_pt)[name]
        out[name] = R.ReducedProgram(oracle, bal, cam, pts)
    return out


# ITERATIVE_SCHUR's CG is capped at 10 iterations on both sides: the solves stay short, and the two trajectories differ
# by summation order only, as tests/entry_points.py compare_lm_traces_exact requires
SOLVERS = {"schur_jacobi": 2, "jacobi": 1, "spse": 3, "dense": None, "sparse": None, "dogleg": None, "subspace": None}
MAX_CG = 10


@pytest.mark.parametrize("name", SETS)
@pytest.mark.parametrize("solver", sorted(SOLVERS))
def test_lm_trajectory(c16_setup, reduced, cs, name, solver):
    """Every record of the device-resident and of the host-boundary loop against the reduced program's own loop (the
    oracle's solves on the reduced structure, tests/dogleg_reference.py's minimize) to 1e-9, and the constant blocks of
    the returned state bitwise equal to the input."""
    s = c16_setup
    ref = reduced[name]
    cam, pts = ref.cam_const, ref.pt_const
    fixed = ref.fixed
    o = ref.default_options()
    o.num_threads, o.max_num_iterations = 8, 5
    opts = dict(max_num_iterations=5)
    dogleg_type = None
    if SOLVERS[solver] is not None:
        opts["linear_solver"] = s.gpu.solver_options(preconditioner_type=SOLVERS[solver], max_num_iterations=MAX_CG)
        o.linear_solver, o.preconditioner, o.max_linear_solver_iterations = 0, SOLVERS[solver], MAX_CG
    else:
        opts["linear_solver_type"] = cs.SPARSE_SCHUR if solver == "sparse" else cs.DENSE_SCHUR
        o.linear_solver = 1
    if solver in ("dogleg", "subspace"):
        opts["trust_region_strategy_type"] = cs.DOGLEG
        dogleg_type = cs.SUBSPACE_DOGLEG if solver == "subspace" else cs.TRADITIONAL_DOGLEG
        opts["dogleg_type"] = dogleg_type
    best_o, recs_o = ref.solve(s.state, o, dogleg_type=dogleg_type)
    s.gpu.set_constant_blocks(cam, pts)
    try:
        xd, recs_d = s.gpu.lm_solve(s.state, s.gpu.lm_options(**opts))
        xh, recs_h = s.gpu.lm_solve(s.state, s.gpu.lm_options(**opts), host_boundary=True)
    finally:
        s.gpu.set_constant_blocks(None, None)
    assert len(recs_o) >= 3
    # (DOGLEG on a set that leaves a gauge free -- the scale with camera 0 alone, the whole similarity with points alone --
    # solves a Gauss-Newton system damped by mu = 1e-8 only: summation-order differences grow to ~1.3e-9 in the gradient
    # and the cost change after a step, measured, so those combinations are held to 1e-7)
    loose = solver in ("dogleg", "subspace") and name in ("gauge", "points")
    for x, recs in ((xd, recs_d), (xh, recs_h)):
        assert np.array_equal(x[fixed].view(np.int64), s.state[fixed].view(np.int64))   # bitwise
        if loose:
            assert len(recs) == len(recs_o)
            for a, b in zip(recs, recs_o):
                for k in ("iteration", "ls_iterations", "step_is_valid", "step_is_successful"):
                    assert int(a[k]) == int(b[k]), (k, a, b)
                for k in ("cost", "gradient_max_norm", "gradient_norm", "step_norm", "tr_radius", "model_cost_change"):
                    assert abs(a[k] - b[k]) <= 1e-7 * abs(b[k]), (k, a, b)
                assert abs(a["cost_change"] - b["cost_change"]) <= 1e-7 * abs(b["cost"]), (a, b)
        else:
            compare_lm_traces_exact(recs, recs_o)
        assert np.linalg.norm(x - best_o) <= (1e-7 if loose else 1e-9) * np.linalg.norm(best_o)


@pytest.mark.parametrize("host_boundary", [False, True])
def test_parameter_tolerance_uses_the_reduced_x(c16_setup, cs, host_boundary):
    """parameter_tolerance compares |step| with |x| over the variable blocks: a threshold between the step / |x_reduced|
    and step / |x_full| ratios of the second accepted step fires with the reduced norm and not with the full one."""
    s = c16_setup
    cam = np.zeros(s.rp.C, bool)
    norms = np.linalg.norm(s.state[:3 * s.rp.P].reshape(-1, 3), axis=1)
    pts = norms >= np.quantile(norms, 0.7)   # the points of largest |X|: |x_reduced| well below |x|
    fixed = R.fixed_components(s.rp.C, s.rp.P, cam, pts)
    s.gpu.set_constant_blocks(cam, pts)

    def solve(**kw):   # DENSE_SCHUR, on the side under test
        return s.gpu.lm_solve(s.state, s.gpu.lm_options(linear_solver_type=cs.DENSE_SCHUR, **kw), host_boundary=host_boundary)
    try:
        _, recs = solve(max_num_iterations=5)
        k = next(i for i, r in enumerate(recs) if i >= 2 and r["step_is_successful"])
        step = recs[k]["step_norm"]
        # the state the step was taken from: replay k - 1 iterations
        xk, _ = solve(max_num_iterations=k - 1)
        nr, nf = np.linalg.norm(xk[~fixed]), np.linalg.norm(xk)
        assert nf > 1.5 * nr
        tol = step / np.sqrt(nr * nf)     # step <= tol * |x_reduced| fails, step <= tol * |x_full| would fire
        _, recs_t = solve(max_num_iterations=5, parameter_tolerance=tol)
        assert len(recs_t) > k            # does not fire at k
        tol2 = step / nr * (1 + 1e-6)
        _, recs_t2 = solve(max_num_iterations=5, parameter_tolerance=tol2)
        assert len(recs_t2) == k          # fires at k: its record is not written
    finally:
        s.gpu.set_constant_blocks(None, None)


def test_setter_contract(c16_setup, cs):
    s = c16_setup
    rp = s.rp
    cam, pts = _c16_set(rp, "gauge_points")
    fixed = R.fixed_components(rp.C, rp.P, cam, pts)
    before = _eval_all(s.gpu, s.state)
    # refused: a row with both blocks constant, and the handle is unchanged
    bad = pts.copy()
    bad[rp.row_pt[rp.row_cam == 0][0]] = True
    with pytest.raises(cs.B200Error):
        s.gpu.set_constant_blocks(cam, bad)
    after = _eval_all(s.gpu, s.state)
    for i in (0, 1, 3):   # cost, residuals, J (the gradient's atomics are not bit-reproducible)
        assert np.array_equal(before[i], after[i])
    # the setter zeroes the stored J's constant cells at once, and set_jacobian_values after each upload
    s.gpu.set_constant_blocks(cam, pts)
    mask = np.concatenate([np.repeat(pts[rp.row_pt], 6), np.repeat(cam[rp.row_cam], 18)])
    J = s.gpu.jacobian_values()
    assert np.all(J[mask] == 0.0) and np.array_equal(J[~mask], before[3][~mask])
    s.gpu.set_jacobian_values(before[3])
    assert np.all(s.gpu.jacobian_values()[mask] == 0.0)
    # the resident residuals survive the call
    s.gpu.evaluate(s.state)
    s.gpu.set_constant_blocks(cam, pts)
    x = s.gpu.dense_schur_solve(None, np.ones(rp.num_parameters))[0]
    assert np.all(x[fixed] == 0.0)
    # set -> solve -> clear -> solve equals a fresh handle's solve from the first solve's state
    o = s.gpu.lm_options(max_num_iterations=3, linear_solver_type=cs.DENSE_SCHUR)
    x1, _ = s.gpu.lm_solve(s.state, o)
    s.gpu.set_constant_blocks(None, None)
    x2, recs2 = s.gpu.lm_solve(x1, o)
    x3, recs3 = s.free.lm_solve(x1, s.free.lm_options(max_num_iterations=3, linear_solver_type=cs.DENSE_SCHUR))
    assert len(recs2) == len(recs3)
    for a, b in zip(recs2, recs3):
        for k, v in b.items():
            assert abs(a[k] - v) <= 1e-9 * max(abs(v), 1e-300), (k, a, b)
    assert np.linalg.norm(x2 - x3) <= 1e-9 * np.linalg.norm(x3)


def _free_port():
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        return sk.getsockname()[1]


def test_sharded():
    """Two ranks, points sharded and cameras replicated, with a camera and points of both shards constant: cost, gradient
    and an ITERATIVE_SCHUR LM run (device-resident: its x_norm goes through the sharded reduction) against the unsharded
    handle, as tests/test_gpu_losses.py::test_sharded_table does for loss tables.  Skipped below 2 GPUs."""
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs, %d visible" % torch.cuda.device_count())
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.abspath(__file__)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=root)
    assert r.returncode == 0 and "CONSTANT-SHARDED-OK" in r.stdout, (r.stdout[-3000:], r.stderr[-3000:])


def _sharded_worker():
    import torch
    import torch.distributed as dist
    import ceres_solver_b200 as cs
    from ceres_solver_b200 import bal as B

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
    cam, pts = R.constant_sets(rp.row_cam, rp.row_pt, rp.P, rp.C, cameras=1, per_class=4)
    fixed = R.fixed_components(rp.C, rp.P, cam, pts)
    one = cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs, device=local)
    one.set_constant_blocks(cam, pts)
    ok1, cost1, _, grad1 = one.evaluate(full, want_residuals=False)
    o = one.lm_options(max_num_iterations=3)
    x1, recs1 = one.lm_solve(full, o)
    plo, phi, rlo, rhi = rp.shard(rank, world)
    gpu = cs.Problem(rp.C, phi - plo, rp.row_cam[rlo:rhi], rp.row_pt[rlo:rhi] - plo, rp.row_obs[rlo:rhi], device=local,
                     rank=rank, world_size=world, nccl_id=nccl_id)
    gpu.set_constant_blocks(cam, pts[plo:phi])
    state = np.concatenate([full[3 * plo:3 * phi], full[3 * rp.P:]])
    ok, cost, _, grad = gpu.evaluate(state, want_residuals=False)
    assert ok and ok1 and abs(cost - cost1) <= 1e-12 * cost1, (cost, cost1)
    nP = 3 * (phi - plo)
    g1 = np.concatenate([grad1[3 * plo:3 * phi], grad1[3 * rp.P:]])
    f = np.concatenate([fixed[3 * plo:3 * phi], fixed[3 * rp.P:]])
    assert np.all(grad[f] == 0.0)
    assert np.linalg.norm(grad - g1) <= 1e-10 * np.linalg.norm(g1)
    x, recs = gpu.lm_solve(state, o)
    x1s = np.concatenate([x1[3 * plo:3 * phi], x1[3 * rp.P:]])
    assert np.array_equal(x[f], state[f])
    assert len(recs) == len(recs1)
    for a, b in zip(recs, recs1):
        assert a["ls_iterations"] == b["ls_iterations"] and a["step_is_successful"] == b["step_is_successful"], (a, b)
        for k in ("cost", "step_norm", "gradient_max_norm"):
            assert abs(a[k] - b[k]) <= 1e-6 * max(abs(b[k]), 1e-300), (k, a, b)
    assert np.linalg.norm(x - x1s) <= 1e-6 * np.linalg.norm(x1s)
    gpu.close()
    one.close()
    dist.barrier()
    if rank == 0:
        print("CONSTANT-SHARDED-OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    _sharded_worker()
