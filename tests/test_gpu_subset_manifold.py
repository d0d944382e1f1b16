"""b200_set_subset_manifolds (Problem::SetManifold with SubsetManifold) on the device, against the handle without masks,
against b200_set_constant_blocks, and against the tangent-space program of tests/subset_manifold_reference.py.

A coordinate held by a SubsetManifold is a Jacobian column that is exactly zero, with D' = 1 in every solve, as a constant
block's columns are; it differs from a constant block in the finiteness check (the ambient Jacobian is checked before
the column is dropped), in |x| of parameter_tolerance (Ceres' x holds it) and in the covariance (zero rows and columns).
Fixtures: those of tests/test_gpu_constant_blocks.py (every evaluate configuration, each asserting its plan).
"""
import numpy as np
import pytest

from tests import constant_blocks_reference as R
from tests import eval_failure_cases as F
from tests import lm_cases as L
from tests import subset_manifold_reference as S
from tests.entry_points import compare_lm_traces_exact
from tests.test_gpu_constant_blocks import EXPLICIT, FIXTURES, _bal, _eval_all, _lm_D
from tests.test_gpu_dispatch import problem_plan  # noqa: F401  (a fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as cs
    cs.lib()
    return cs


class Setup:
    def __init__(self, cs, bal):
        from ceres_solver_b200 import bal as B
        self.rp = rp = B.ReducedProgram(bal)
        self.state = rp.state(bal)
        self.free = cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs)     # never holds anything constant
        self.gpu = cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs)
        self.cm, self.pm = S.mask_sets(rp.row_cam, rp.row_pt, rp.P, rp.C)
        _, _, self.fixed, self.masked = S.effective(rp.C, rp.P, None, None, self.cm, self.pm)
        self.cells = S.cell_mask(rp.row_cam, rp.row_pt, None, None, self.cm, self.pm)

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
    masked_pt = setup.pm.any(axis=1)
    assert setup.cm.any(axis=1).all() and not setup.cm.all(axis=1).any()
    for lo, hi in ((1, 32), (33, 128), (129, 1 << 30)):
        cls = (deg >= lo) & (deg <= hi)
        if cls.sum() > 2:
            assert masked_pt[cls].any() and (~masked_pt[cls]).any(), (lo, hi)


def test_empty_masks_are_the_old_path(setup):
    """Bit for bit wherever two runs of the untouched handle agree bit for bit (cost, residuals, J)."""
    s = setup
    a = _eval_all(s.free, s.state)
    b = _eval_all(s.free, s.state)
    exact = [np.array_equal(x, y) for x, y in zip(a, b)]
    assert exact[0] and exact[1] and exact[3]
    for masks in ((None, None), (np.zeros((s.rp.C, 9), bool), np.zeros((s.rp.P, 3), bool))):
        s.gpu.set_subset_manifolds(*masks)
        c = _eval_all(s.gpu, s.state)
        for x, y, bits in zip(a, c, exact):
            if bits:
                assert np.array_equal(x, y)
            else:
                assert np.linalg.norm(np.asarray(x) - y) <= 1e-13 * np.linalg.norm(x)
    s.gpu.set_subset_manifolds(None, None)


def test_full_masks_are_constant_blocks(setup, cs):
    """A full mask is a constant block: evaluate gives the bits of b200_set_constant_blocks on those blocks, every solve
    its exact zeros and its solution (the PCG sums with atomics, so two handles agree to rounding, not to the bit), and
    on C16 the LM trace."""
    s = setup
    cam, pts = R.constant_sets(s.rp.row_cam, s.rp.row_pt, s.rp.P, s.rp.C)
    cm = np.repeat(cam[:, None], 9, axis=1)
    pm = np.repeat(pts[:, None], 3, axis=1)
    s.gpu.set_subset_manifolds(cm, pm)
    s.free.set_constant_blocks(cam, pts)
    try:
        a, c = _eval_all(s.free, s.state), _eval_all(s.gpu, s.state)   # (the gradient's atomics: not compared)
        assert a[0] == c[0] and np.array_equal(a[1], c[1]) and np.array_equal(a[3], c[3])
        D = _lm_D(s.gpu)
        solves = [lambda g: g.schur_solve(None, D, g.solver_options(max_num_iterations=20))]
        if s.name == "c16":
            solves += [lambda g: g.dense_schur_solve(None, D), lambda g: g.sparse_schur_solve(None, D)]
        fixed = R.fixed_components(s.rp.C, s.rp.P, cam, pts)
        for solve in solves:
            xa, xc = solve(s.free)[0], solve(s.gpu)[0]
            assert np.all(xc[fixed] == 0.0) and np.all(xa[fixed] == 0.0)
            assert np.linalg.norm(xc - xa) <= 1e-10 * np.linalg.norm(xa)
        if s.name == "c16":
            o = s.free.lm_options(max_num_iterations=4, linear_solver_type=cs.DENSE_SCHUR)
            xa, ra = s.free.lm_solve(s.state, o)
            xb, rb = s.free.lm_solve(s.state, o)
            xc, rc = s.gpu.lm_solve(s.state, o)
            if ra == rb:   # else (the gradient's atomics) as the constant handle's second run compares with its first
                assert rc == ra and np.array_equal(xc, xa)
            else:
                compare_lm_traces_exact(rc, ra)
    finally:
        s.gpu.set_subset_manifolds(None, None)
        s.free.set_constant_blocks(None, None)


def test_evaluate_every_mode(setup):
    s = setup
    cost0, res0, grad0, J0 = _eval_all(s.free, s.state)
    s.gpu.set_subset_manifolds(s.cm, s.pm)
    mask, fixed = s.cells, s.fixed
    try:
        ok, cost, res, grad = s.gpu.evaluate(s.state)
        assert ok and cost == cost0 and np.array_equal(res, res0)
        J = s.gpu.jacobian_values()
        assert np.all(J[mask] == 0.0)
        assert np.array_equal(J[~mask], J0[~mask])
        assert np.all(grad[fixed] == 0.0)
        Js = R.jacobian_matrix(J, s.rp.row_cam, s.rp.row_pt, s.rp.P, s.rp.C)
        gr = Js.T @ res
        assert np.linalg.norm(grad - gr) <= 1e-12 * np.linalg.norm(gr)
        sq = s.gpu.squared_column_norm()
        assert np.all(sq[fixed] == 0.0)
        sq0 = np.asarray(Js.multiply(Js).sum(axis=0)).ravel()
        assert np.linalg.norm(sq - sq0) <= 1e-12 * np.linalg.norm(sq0)
        ok, cost_g, _, grad_g = s.gpu.evaluate(s.state, want_jacobian=False)
        assert ok and cost_g == cost0
        assert np.all(grad_g[fixed] == 0.0) and np.linalg.norm(grad_g - grad) <= 1e-13 * np.linalg.norm(grad)
        s.gpu.set_jacobian_values(np.zeros_like(J))
        ok, cost_j, _, _ = s.gpu.evaluate(s.state, want_residuals=False, want_gradient=False)
        assert ok and cost_j == cost0 and np.array_equal(s.gpu.jacobian_values(), J)
        y = s.gpu.left_multiply(np.random.RandomState(0).normal(size=2 * s.rp.N))
        assert np.all(y[fixed] == 0.0)
        ok, _, res, _ = s.gpu.evaluate(s.state)
        Jr = R.jacobian_matrix(np.where(mask, 0.0, J0), s.rp.row_cam, s.rp.row_pt, s.rp.P, s.rp.C)
        x = np.random.RandomState(2).normal(size=s.rp.num_parameters)
        jx = Jr @ x
        assert np.linalg.norm(s.gpu.right_multiply(x) - jx) <= 1e-12 * np.linalg.norm(jx)
        mcc = -(jx @ (res + jx / 2.0))
        assert abs(s.gpu.model_cost_change(x) - mcc) <= 1e-12 * (abs(jx @ res) + jx @ jx / 2.0)
    finally:
        s.gpu.set_subset_manifolds(None, None)


def test_failure_in_masked_columns(cs, c16):
    """cost_overflow2: the camera's non-finite cells (d r / d l1, d r / d l2) lie in masked columns while its column 3
    (d r / d t_x = -f / p_z, finite) stays free.  Ceres checks the ambient Jacobian, so every J mode fails; with the
    whole camera constant the same construction succeeds."""
    s = Setup(cs, L.c16_bal(c16))
    try:
        rp = s.rp
        perm, _, _ = cs.plan_point_order(rp.C, rp.P, rp.row_cam, rp.row_pt)
        places = F.placements(s.state, rp.row_cam, rp.row_pt, rp.P, perm)
        rows = F.overflow_targets(places, s.state, rp.row_cam, rp.row_pt, rp.P)[:2]
        x = F.construct(s.state, rp.row_cam, rp.row_pt, rp.P, "cost_overflow2", rows)
        cams = np.unique(rp.row_cam[rows])
        cm = np.zeros((rp.C, 9), bool)
        cm[cams] = True
        cm[cams, 3] = False
        s.gpu.set_subset_manifolds(cm, None)
        for kw in (dict(), dict(want_jacobian=False), dict(want_residuals=False, want_gradient=False)):
            ok, _, _, _ = s.gpu.evaluate(x, **kw)
            assert not ok, kw
        ok, cost, _, _ = s.gpu.evaluate(x, want_residuals=False, want_gradient=False, want_jacobian=False)
        assert ok and np.isfinite(cost)
        cm[cams, 3] = True   # a full mask: the camera is constant
        s.gpu.set_subset_manifolds(cm, None)
        for kw in (dict(), dict(want_jacobian=False), dict(want_residuals=False, want_gradient=False)):
            ok, cost, _, _ = s.gpu.evaluate(x, **kw)
            assert ok and np.isfinite(cost), kw
    finally:
        s.close()


# ---------------------------------------------------------------------------------------------------------- C16
@pytest.fixture(scope="module")
def c16_setup(cs, c16):
    s = Setup(cs, L.c16_bal(c16))
    yield s
    s.close()


SETS = ("intrinsics", "mixed", "heights", "combined")


@pytest.fixture(scope="module")
def tangent(oracle, c16):
    """{set name: (the set, SubsetProgram of C16)}."""
    bal = L.c16_bal(c16)
    full = R.ReducedProgram(oracle, bal)
    sets = S.c16_mask_sets(full.P, full.C, full.base.row_cam, full.base.row_pt)
    return {name: (sets[name], S.SubsetProgram(oracle, bal, *sets[name])) for name in SETS}


def _apply(gpu, st):
    cam, pts, cm, pm = st
    gpu.set_constant_blocks(cam, pts)
    gpu.set_subset_manifolds(cm, pm)


def _clear(gpu):
    gpu.set_constant_blocks(None, None)
    gpu.set_subset_manifolds(None, None)


@pytest.mark.parametrize("name", SETS)
def test_solves_against_the_tangent_program(c16_setup, tangent, cs, name):
    s = c16_setup
    st, sp = tangent[name]
    _apply(s.gpu, st)
    try:
        ok, _, res, _ = s.gpu.evaluate(s.state)
        assert ok
        J = s.gpu.jacobian_values()
        Js = R.jacobian_matrix(J, s.rp.row_cam, s.rp.row_pt, s.rp.P, s.rp.C)
        D = _lm_D(s.gpu)
        x_ref = R.reduced_solve(Js, res, D, sp.fixed)
        x_t, _, term = sp.tangent_solve(J, res, D)
        assert term == 0 and np.linalg.norm(x_t - x_ref) <= 1e-8 * np.linalg.norm(x_ref)
        for order in (cs.AMD, cs.NESDIS):
            s.gpu.set_linear_solver_ordering_type(order)
            for mixed in (False, True):
                s.gpu.set_exact_solve_options(mixed, 2 if mixed else 0)
                for solve in (s.gpu.sparse_schur_solve, s.gpu.dense_schur_solve):
                    x = solve(None, D)[0]
                    assert np.all(x[sp.fixed] == 0.0), (solve, order, mixed)
                    assert np.linalg.norm(x - x_ref) <= (1e-6 if mixed else 1e-8) * np.linalg.norm(x_ref), (solve, order, mixed)
        s.gpu.set_exact_solve_options(False, 0)
        s.gpu.set_linear_solver_ordering_type(cs.AMD)
        for pre, spse in ((cs.PRECOND_IDENTITY, 0), (cs.PRECOND_JACOBI, 0), (cs.PRECOND_SCHUR_JACOBI, 0),
                          (cs.PRECOND_SCHUR_POWER_SERIES_EXPANSION, 0), (cs.PRECOND_SCHUR_JACOBI, 1)):
            o = s.gpu.solver_options(preconditioner_type=pre, use_spse_initialization=spse, max_num_iterations=500,
                                     q_tolerance=0.0, r_tolerance=1e-14)
            for d in (D, None):
                x = s.gpu.schur_solve(None, d, o)[0]
                assert np.all(x[sp.fixed] == 0.0), (pre, spse)
            if pre != cs.PRECOND_IDENTITY:
                # (with intrinsics held on every camera the similarity gauge is free and S is regularised by D alone: the
                # PCG, whose sums use atomics, lands within 7e-7 of the direct solve in one H100 run and within 1e-7 in
                # another; the other sets fix the gauge and are held to 1e-7)
                x, _, term = s.gpu.schur_solve(None, D, o)
                assert term == cs.LS_SUCCESS, (pre, spse)
                assert np.linalg.norm(x - x_ref) <= (1e-5 if name == "intrinsics" else 1e-7) * np.linalg.norm(x_ref), (pre, spse)
        # PCG iteration counts: the decoupled components have rhs 0 and x0 = 0, so the iterates are the tangent program's
        # (the LM loop's stopping rule, as tests/test_gpu_parity.py compares the counts; IDENTITY on C16's unscaled system
        # converges too erratically for a count to be reproducible across summation orders: 55 against 51 measured)
        for pre in (cs.PRECOND_JACOBI, cs.PRECOND_SCHUR_JACOBI):
            o = s.gpu.solver_options(preconditioner_type=pre, q_tolerance=1e-2, r_tolerance=-1.0)
            _, it_gpu, term = s.gpu.schur_solve(None, D, o)
            _, it_ref, term_ref = sp.tangent_solve(J, res, D, solver=0, preconditioner=pre, max_iter=500, q_tolerance=1e-2,
                                                   r_tolerance=-1.0, nt=8)
            assert term == term_ref and it_gpu == it_ref, (pre, it_gpu, it_ref)
    finally:
        _clear(s.gpu)


# ITERATIVE_SCHUR's CG is capped at 10 iterations on both sides, as in tests/test_gpu_constant_blocks.py
SOLVERS = {"schur_jacobi": 2, "dense": None, "sparse": None, "dogleg": None, "subspace": None}
MAX_CG = 10


@pytest.mark.parametrize("name", ["intrinsics", "mixed"])
@pytest.mark.parametrize("solver", sorted(SOLVERS))
def test_lm_trajectory(c16_setup, tangent, cs, name, solver):
    """Every record of the device-resident and of the host-boundary loop against the tangent program's own loop to 1e-9,
    and the masked coordinates of the returned state bitwise equal to the input."""
    s = c16_setup
    st, ref = tangent[name]
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
    _apply(s.gpu, st)
    try:
        xd, recs_d = s.gpu.lm_solve(s.state, s.gpu.lm_options(**opts))
        xh, recs_h = s.gpu.lm_solve(s.state, s.gpu.lm_options(**opts), host_boundary=True)
    finally:
        _clear(s.gpu)
    assert len(recs_o) >= 3
    # (DOGLEG's Gauss-Newton system is damped by mu = 1e-8 only, and intrinsics held on every camera leave the whole
    # similarity gauge free: summation-order differences then grow past 1e-9, as in tests/test_gpu_constant_blocks.py's
    # gauge sets.  Measured on an H100: 2e-9 in the step norm of DENSE_SCHUR's fifth step and 1.2e-7 in SUBSPACE_DOGLEG's,
    # with intrinsics held.  Those combinations are held to 1e-7 and 1e-6, every decision still equal)
    dl = solver in ("dogleg", "subspace")
    loose = dl or name == "intrinsics"
    tol = 1e-6 if dl and name == "intrinsics" else 1e-7
    for x, recs in ((xd, recs_d), (xh, recs_h)):
        assert np.array_equal(x[fixed].view(np.int64), s.state[fixed].view(np.int64))
        if loose:
            assert len(recs) == len(recs_o)
            for a, b in zip(recs, recs_o):
                for k in ("iteration", "ls_iterations", "step_is_valid", "step_is_successful"):
                    assert int(a[k]) == int(b[k]), (k, a, b)
                for k in ("cost", "gradient_max_norm", "gradient_norm", "step_norm", "tr_radius", "model_cost_change"):
                    assert abs(a[k] - b[k]) <= tol * abs(b[k]), (k, a, b)
        else:
            compare_lm_traces_exact(recs, recs_o)
        assert np.linalg.norm(x - best_o) <= (tol if loose else 1e-9) * np.linalg.norm(best_o)


@pytest.mark.parametrize("host_boundary", [False, True])
def test_parameter_tolerance_counts_masked_coordinates(c16_setup, cs, host_boundary):
    """|x| of parameter_tolerance is Ceres' ambient x of the variable blocks: masked coordinates count, constant blocks do
    not.  With two coordinates of the points of largest |X| masked, a threshold between step / |x_ambient| and
    step / |x without the masked coordinates| (the tangent program's |x|) fires at step k."""
    s = c16_setup
    rp = s.rp
    norms = np.linalg.norm(s.state[:3 * rp.P].reshape(-1, 3), axis=1)
    big = norms >= np.quantile(norms, 0.7)
    pm = np.zeros((rp.P, 3), bool)
    pm[big, :2] = True            # masked: in |x|
    _, _, fixed, masked = S.effective(rp.C, rp.P, None, None, None, pm)
    s.gpu.set_subset_manifolds(None, pm)

    def solve(**kw):
        return s.gpu.lm_solve(s.state, s.gpu.lm_options(linear_solver_type=cs.DENSE_SCHUR, **kw), host_boundary=host_boundary)
    try:
        _, recs = solve(max_num_iterations=5, parameter_tolerance=1e-16)
        k = next(i for i, r in enumerate(recs) if i >= 2 and r["step_is_successful"])
        step = recs[k]["step_norm"]
        xk, _ = solve(max_num_iterations=k - 1, parameter_tolerance=1e-16)
        n_amb, n_var = np.linalg.norm(xk), np.linalg.norm(xk[~fixed])
        assert n_amb > 1.1 * n_var

        def threshold(n):   # the tolerance t at which step = t (|x| + t), trust_region_minimizer.cc:725-742
            return (np.sqrt(n * n + 4.0 * step) - n) / 2.0
        t_amb, t_var = threshold(n_amb), threshold(n_var)
        assert t_var > 1.05 * t_amb
        # between the two: fires with the ambient |x| (Ceres'), would not with the variable coordinates' alone
        _, recs_t = solve(max_num_iterations=5, parameter_tolerance=np.sqrt(t_amb * t_var))
        assert len(recs_t) == k           # fires at k: its record is not written
        _, recs_t2 = solve(max_num_iterations=5, parameter_tolerance=t_amb * (1 - 1e-6))
        assert len(recs_t2) > k
    finally:
        s.gpu.set_subset_manifolds(None, None)


# ---------------------------------------------------------------------------------------------------------- covariance
def _lifted_reference(gpu, fx, cm, pm):
    """tests/covariance_reference.py's Schur form of the tangent program, lifted with zero rows and columns: the stored J
    (masked columns 0) with one extra row per masked coordinate that puts 1 on its diagonal (V_p for a point's, F'F for a
    camera's) and nothing elsewhere, which is D' = 1 there; then Z and Cov(p, p) with the masked rows and columns zeroed."""
    from tests.covariance_reference import SchurCovariance
    J = gpu.jacobian_values()
    N = fx.cam.size
    E = list(J[:6 * N].reshape(N, 6))
    Fv = list(J[6 * N:].reshape(N, 18))
    cam, pt = list(fx.cam), list(fx.pt)
    var_pt = int(np.flatnonzero(~fx.pc)[0])
    for p, k in zip(*np.nonzero(pm & ~fx.pc[:, None])):
        e = np.zeros(6)
        e[k] = 1.0
        E.append(e), Fv.append(np.zeros(18)), cam.append(0), pt.append(p)
    for c, k in zip(*np.nonzero(cm & ~fx.cc[:, None])):
        f = np.zeros(18)
        f[k] = 1.0
        E.append(np.zeros(6)), Fv.append(f), cam.append(c), pt.append(var_pt)
    values = np.concatenate([np.ravel(E), np.ravel(Fv)])
    ref = SchurCovariance(values, cam, pt, fx.P, fx.C, fx.fixed, dtype=np.float64)
    if ref.Z is not None:
        idx = np.flatnonzero(cm.ravel())
        ref.Z[idx, :] = 0
        ref.Z[:, idx] = 0
        for p in np.flatnonzero(pm.any(axis=1)):
            ref.points[p][pm[p], :] = 0
            ref.points[p][:, pm[p]] = 0
    return ref


@pytest.mark.parametrize("algorithm", ["sparse_amd", "sparse_nesdis", "dense"])
def test_covariance(cs, c16, algorithm):
    from tests.test_gpu_covariance import c16_fixture, check_accuracy, pattern_pairs
    fx = c16_fixture(cs, c16)
    cm = np.zeros((fx.C, 9), bool)
    cm[1:, 6:] = True                      # intrinsics held on every variable camera
    pm = np.zeros((fx.P, 3), bool)
    rng = np.random.RandomState(3)
    pm[rng.choice(np.flatnonzero(~fx.pc), size=fx.P // 20, replace=False), 2] = True
    gpu = fx.problem()
    try:
        gpu.set_subset_manifolds(cm, pm)
        if algorithm == "sparse_nesdis":
            gpu.set_linear_solver_ordering_type(cs.NESDIS)
        alg = cs.DENSE_SCHUR if algorithm == "dense" else cs.SPARSE_SCHUR
        assert gpu.covariance_compute(fx.state, algorithm=alg)
        ref = _lifted_reference(gpu, fx, cm, pm)
        assert ref.Z is not None and ref.rcond >= 1e-14
        pairs = pattern_pairs(fx.C, fx.cam, fx.pt)
        cams = gpu.covariance_cameras(pairs)
        pts = gpu.covariance_points()
        for (i, j), blk in zip(pairs, cams):   # exact zeros on masked rows of camera i and masked columns of camera j
            assert not blk[cm[i], :].any() and not blk[:, cm[j]].any(), (i, j)
        for p in np.flatnonzero(pm.any(axis=1)):
            assert not pts[p][pm[p], :].any() and not pts[p][:, pm[p]].any(), p
        check_accuracy(fx, gpu, ref, pairs, cams, pts, "c16 masked/" + algorithm)
    finally:
        gpu.close()


def test_covariance_gauge_by_masks(cs, c16):
    """Masks alone fix the similarity gauge -- camera 0's pose (coordinates 0-5) and camera 1's t_x -- and the compute is
    valid; without them it is not."""
    from tests.test_gpu_covariance import c16_fixture
    fx = c16_fixture(cs, c16)
    gpu = cs.Problem(fx.C, fx.P, fx.cam, fx.pt, fx.obs)
    try:
        assert not gpu.covariance_compute(fx.state)
        cm = np.zeros((fx.C, 9), bool)
        cm[0, :6] = True
        cm[1, 3] = True
        gpu.set_subset_manifolds(cm, None)
        for alg in (cs.SPARSE_SCHUR, cs.DENSE_SCHUR):
            assert gpu.covariance_compute(fx.state, algorithm=alg)
            blk = gpu.covariance_cameras([(0, 0), (1, 1), (0, 1)])
            assert not blk[0][:6].any() and not blk[0][:, :6].any() and np.all(np.diag(blk[0])[6:] > 0)
            assert not blk[1][3].any() and not blk[1][:, 3].any()
            assert not blk[2][:6].any() and not blk[2][:, 3].any()
    finally:
        gpu.close()


# ---------------------------------------------------------------------------------------------------------- contract
def test_setter_contract(c16_setup, cs):
    s = c16_setup
    rp = s.rp
    before = _eval_all(s.gpu, s.state)
    cm = np.zeros((rp.C, 9), bool)
    cm[:, 6:] = True
    pm = np.zeros((rp.P, 3), bool)
    pm[:50, 2] = True
    lib = cs.lib()
    import ctypes as C

    def raw(cam, pts):
        return lib.b200_set_subset_manifolds(s.gpu.h, None if cam is None else cam.ctypes.data_as(C.POINTER(C.c_uint16)),
                                             None if pts is None else pts.ctypes.data_as(C.POINTER(C.c_uint8)))
    # bits above the block's coordinates are refused, and the handle is unchanged
    bad_c = np.zeros(rp.C, np.uint16)
    bad_c[3] = 1 << 9
    bad_p = np.zeros(rp.P, np.uint8)
    bad_p[7] = 1 << 3
    assert raw(bad_c, None) != 0 and raw(None, bad_p) != 0
    after = _eval_all(s.gpu, s.state)
    for i in (0, 1, 3):
        assert np.array_equal(before[i], after[i])
    # a row whose camera and point are both constant, through either setter: refused, handle (both sets) unchanged
    cam0 = np.zeros(rp.C, bool)
    cam0[0] = True
    p0 = rp.row_pt[rp.row_cam == 0][0]
    full_p = np.zeros((rp.P, 3), bool)
    full_p[p0] = True
    s.gpu.set_subset_manifolds(cm, pm)
    J_masked = s.gpu.jacobian_values()
    s.gpu.set_constant_blocks(cam0, None)
    J_both = s.gpu.jacobian_values()
    with pytest.raises(cs.B200Error):
        s.gpu.set_subset_manifolds(cm, full_p)
    ok, _, _, _ = s.gpu.evaluate(s.state)
    assert ok and np.array_equal(s.gpu.jacobian_values(), J_both)
    pts0 = np.zeros(rp.P, bool)
    pts0[p0] = True
    s.gpu.set_constant_blocks(None, None)
    full_c = np.zeros((rp.C, 9), bool)
    full_c[0] = True
    s.gpu.set_subset_manifolds(full_c, None)
    with pytest.raises(cs.B200Error):
        s.gpu.set_constant_blocks(None, pts0)
    # the setters are independent: clearing one keeps the other
    s.gpu.set_subset_manifolds(cm, pm)
    s.gpu.set_constant_blocks(cam0, None)
    s.gpu.set_constant_blocks(None, None)
    ok, _, _, _ = s.gpu.evaluate(s.state)
    assert ok and np.array_equal(s.gpu.jacobian_values(), J_masked)
    # the stored J is zeroed by the call and after set_jacobian_values
    mask = S.cell_mask(rp.row_cam, rp.row_pt, None, None, cm, pm)
    s.gpu.set_subset_manifolds(None, None)
    s.gpu.set_jacobian_values(before[3])
    s.gpu.set_subset_manifolds(cm, pm)
    J = s.gpu.jacobian_values()
    assert np.all(J[mask] == 0.0) and np.array_equal(J[~mask], before[3][~mask])
    s.gpu.set_jacobian_values(before[3])
    J = s.gpu.jacobian_values()
    assert np.all(J[mask] == 0.0) and np.array_equal(J[~mask], before[3][~mask])
    # the solves return exact zeros on masked coordinates
    _, _, fixed, _ = S.effective(rp.C, rp.P, None, None, cm, pm)
    x = s.gpu.dense_schur_solve(None, np.ones(rp.num_parameters))[0]
    assert np.all(x[fixed] == 0.0)
    s.gpu.set_subset_manifolds(None, None)
