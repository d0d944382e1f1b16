"""b200_covariance_compute / b200_covariance_cameras / b200_covariance_points (csrc/covariance.cuh) against the Schur-form
reference of tests/covariance_reference.py, built from the Jacobian the handle stored at the state (so the losses and
apply_loss_function the call used are in it).

Accuracy.  Each camera block of every served pair and each point block is held to
    |block - reference block|_F <= c n kappa u |ref|,   u = 2^-53, n = 9C,
with kappa = kappa_2(S) of the variable components (from the reference) and |ref| = |Z|_2 for camera blocks, and
|Cov(p, p)|_2 (kappa_2(S) + kappa_2(V_p)) / kappa_2(S) for point blocks.  The reference is np.longdouble on C16 and the
small structures, LAPACK float64 on the larger ones.  n kappa u alone is far above what the kernels reach, so c is set from
the largest observed ratio to it on an H100, with a margin of about 50: C_CAM = 3e-5 for camera blocks (largest observed
5.4e-7, the `two` structure) and C_PT = 1e-3 for point blocks (largest observed 1.9e-5, C16 with a Cauchy / ScaledLoss
table).  The ratio to n kappa u is printed per fixture and recorded in DESIGN §3.9.

Fixtures: C16 with camera 0 and 1 % of the points constant (none seen by camera 0), and the camera graphs of
tests/test_sparse_schur_plan.py that reach each path of the supernodal kernel, each under AMD and NESDIS, with their solo
points (seen twice by one camera, so E'E is singular; ten per camera, which fix the gauge) constant.  Each asserts its
plan.
"""
import numpy as np
import pytest

from tests.covariance_reference import SchurCovariance
from tests.test_sparse_schur_plan import camera_edges, check_plan, structure, structure_properties

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
C_CAM = 3e-5
C_PT = 1e-3
STRUCTS = ("two", "clique16", "cliques", "hub", "band", "loop", "random400", "shuffled")
LONGDOUBLE_MAX_CAMERAS = 64


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


def geometry(C, P, cam, pt, seed=11):
    from tests.test_gpu_sparse_factor import geometry as g
    return g(C, P, cam, pt, seed)


def gauge(C, P, cam, pt):
    """Every point seen by fewer than two distinct cameras constant (the solo points: each camera sees ten, which fix it)."""
    cam, pt = np.asarray(cam), np.asarray(pt)
    distinct = np.array([len(np.unique(cam[pt == p])) for p in range(P)])
    return np.zeros(C, bool), distinct < 2


def fixed_of(C, P, cc, pc):
    return np.concatenate([np.repeat(pc, 3), np.repeat(cc, 9)])


def pattern_pairs(C, cam, pt):
    return [(i, i) for i in range(C)] + sorted(camera_edges(C, cam, pt))


class Fixture:
    def __init__(self, cs, C, P, cam, pt, obs, state, cc, pc):
        self.C, self.P, self.cam, self.pt, self.obs, self.state = C, P, np.asarray(cam, np.int32), np.asarray(pt, np.int32), obs, state
        self.cc, self.pc = cc, pc
        self.fixed = fixed_of(C, P, cc, pc)
        self.cs = cs

    def problem(self):
        g = self.cs.Problem(self.C, self.P, self.cam, self.pt, self.obs)
        g.set_constant_blocks(self.cc, self.pc)
        return g

    def reference(self, gpu):
        dtype = np.longdouble if self.C <= LONGDOUBLE_MAX_CAMERAS else np.float64
        return SchurCovariance(gpu.jacobian_values(), self.cam, self.pt, self.P, self.C, self.fixed, dtype=dtype)


def structure_fixture(cs, name):
    C, P, cam, pt = structure(name)
    perm, _, lay = check_plan(cs, C, P, cam, pt)
    structure_properties(name, perm, lay)
    obs, state = geometry(C, P, cam, pt)
    cc, pc = gauge(C, P, cam, pt)
    return Fixture(cs, C, P, cam, pt, obs, state, cc, pc)


def c16_fixture(cs, c16):
    from ceres_solver_b200 import bal as B
    from tests import lm_cases as L
    bal = L.c16_bal(c16)
    rp = B.ReducedProgram(bal)
    cc = np.zeros(rp.C, bool)
    cc[0] = True
    seen = np.zeros(rp.P, bool)
    seen[np.asarray(rp.row_pt)[np.asarray(rp.row_cam) == 0]] = True
    pc = np.zeros(rp.P, bool)
    pc[np.random.RandomState(0).choice(np.flatnonzero(~seen), size=rp.P // 100, replace=False)] = True
    return Fixture(cs, rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs, rp.state(bal), cc, pc)


def check_accuracy(fx, gpu, ref, pairs, cams, pts, label):
    """Asserts the bounds of the module docstring; returns the largest observed ratios to n kappa u (cameras, points)."""
    n = 9 * fx.C
    Z = np.asarray(ref.Z, dtype=float)
    var = ~np.repeat(fx.cc, 9)
    znorm = np.linalg.norm(Z[np.ix_(var, var)], 2)
    worst_c = 0.0
    for (i, j), blk in zip(pairs, cams):
        if fx.cc[i] or fx.cc[j]:
            assert not blk.any(), (label, i, j)
            continue
        err = np.linalg.norm(blk - ref.camera_block(i, j))
        worst_c = max(worst_c, err / (n * ref.kappa * U * znorm))
    worst_p = 0.0
    refp = np.asarray(ref.points, dtype=float)
    for p in range(fx.P):
        if fx.pc[p]:
            assert not pts[p].any(), (label, p)
            continue
        ev = np.linalg.eigvalsh(np.asarray(ref.V[p], dtype=float))
        kv = ev[-1] / ev[0]
        bound = n * U * (ref.kappa + kv) * np.linalg.norm(refp[p], 2)
        worst_p = max(worst_p, np.linalg.norm(pts[p] - refp[p]) / bound)
    print("[covariance] %s: kappa(S) %.2e, observed / (n kappa u): cameras %.2e, points %.2e" % (label, ref.kappa, worst_c, worst_p))
    assert worst_c <= C_CAM and worst_p <= C_PT, (label, worst_c, worst_p)
    return worst_c, worst_p


@pytest.fixture(scope="module")
def c16fx(cs, c16):
    return c16_fixture(cs, c16)


@pytest.mark.parametrize("name", STRUCTS)
@pytest.mark.parametrize("ordering", ["amd", "nesdis"])
def test_structures(cs, name, ordering):
    fx = structure_fixture(cs, name)
    _, st = cs.plan_sparse_schur(fx.C, fx.P, fx.cam, fx.pt, ordering_type=cs.NESDIS if ordering == "nesdis" else cs.AMD)
    assert st["order"] == (2 if ordering == "nesdis" else st["order"])
    gpu = fx.problem()
    try:
        gpu.set_linear_solver_ordering_type(cs.NESDIS if ordering == "nesdis" else cs.AMD)
        valid = gpu.covariance_compute(fx.state)
        ref = fx.reference(gpu)
        print("[covariance] %s/%s: reference min d_k / A_kk %.3e" % (name, ordering, ref.rcond))
        # the device takes the reference's decision; every structure but random400 (tracks from synthetic_bal, no solo
        # points, so nothing holds its gauge) is valid
        assert valid == (ref.Z is not None and ref.rcond >= 1e-14)
        if name == "random400":
            return
        assert valid
        pairs = pattern_pairs(fx.C, fx.cam, fx.pt)
        cams = gpu.covariance_cameras(pairs)
        pts = gpu.covariance_points()
        check_accuracy(fx, gpu, ref, pairs, cams, pts, "%s/%s" % (name, ordering))
        # (j, i) is the transpose of (i, j), bit for bit
        rev = gpu.covariance_cameras([(j, i) for i, j in pairs])
        assert np.array_equal(rev, np.transpose(cams, (0, 2, 1)))
        # determinism: a second compute of the same state gives the same bits
        assert gpu.covariance_compute(fx.state)
        assert np.array_equal(gpu.covariance_cameras(pairs), cams)
        assert np.array_equal(gpu.covariance_points(), pts)
    finally:
        gpu.close()


@pytest.mark.parametrize("algorithm", ["sparse_amd", "sparse_nesdis", "dense"])
def test_c16(cs, c16fx, algorithm):
    fx = c16fx
    gpu = fx.problem()
    try:
        if algorithm == "sparse_nesdis":
            gpu.set_linear_solver_ordering_type(cs.NESDIS)
        alg = cs.DENSE_SCHUR if algorithm == "dense" else cs.SPARSE_SCHUR
        assert gpu.covariance_compute(fx.state, algorithm=alg)
        ref = fx.reference(gpu)
        pairs = pattern_pairs(fx.C, fx.cam, fx.pt)
        check_accuracy(fx, gpu, ref, pairs, gpu.covariance_cameras(pairs), gpu.covariance_points(), "c16/" + algorithm)
    finally:
        gpu.close()


def test_dense_against_sparse(cs):
    fx = structure_fixture(cs, "band")
    gpu = fx.problem()
    try:
        pairs = pattern_pairs(fx.C, fx.cam, fx.pt)
        assert gpu.covariance_compute(fx.state, algorithm=cs.SPARSE_SCHUR)
        sc, sp_ = gpu.covariance_cameras(pairs), gpu.covariance_points()
        assert gpu.covariance_compute(fx.state, algorithm=cs.DENSE_SCHUR)
        dc, dp = gpu.covariance_cameras(pairs), gpu.covariance_points()
        scale = np.abs(dc).max()
        assert np.abs(sc - dc).max() <= 1e-8 * scale
        assert np.abs(sp_ - dp).max() <= 1e-8 * np.abs(dp).max()
        # a pair outside the pattern: the dense algorithm serves it (frames 1 and C - 1 share no point), against the reference
        far = (1, fx.C - 1)
        assert far not in set(pairs)
        ref = fx.reference(gpu)
        blk = gpu.covariance_cameras([far])[0]
        assert np.linalg.norm(blk - ref.camera_block(*far)) <= C_CAM * 9 * fx.C * ref.kappa * U * np.linalg.norm(np.asarray(ref.Z, float), 2)
    finally:
        gpu.close()


def test_losses_and_apply_loss_function(cs, c16fx):
    fx = c16fx
    gpu = fx.problem()
    try:
        rng = np.random.RandomState(3)
        losses = [(cs.LOSS_CAUCHY, 1.0, 0.0, 1.0), (cs.LOSS_TRIVIAL, 0.0, 0.0, 2.5), (cs.LOSS_CAUCHY, 0.5, 0.0, 0.7)]
        gpu.set_loss_functions(losses, rng.randint(0, 3, size=len(fx.cam)))
        _, cost_loss, _, _ = gpu.evaluate(fx.state)
        results = {}
        for apply in (True, False):
            assert gpu.covariance_compute(fx.state, apply_loss_function=apply)
            ref = fx.reference(gpu)
            pairs = pattern_pairs(fx.C, fx.cam, fx.pt)
            cams = gpu.covariance_cameras(pairs)
            check_accuracy(fx, gpu, ref, pairs, cams, gpu.covariance_points(), "c16/losses apply=%d" % apply)
            results[apply] = cams
            # the handle's own setting (apply) is back: its evaluation still applies the losses
            _, c, _, _ = gpu.evaluate(fx.state)
            assert c == cost_loss
        assert not np.array_equal(results[True], results[False])
    finally:
        gpu.close()


def test_contract(cs, c16fx):
    from ceres_solver_b200.binding import B200Error, ERR_INVALID_ARGUMENT, ERR_UNSUPPORTED
    fx = c16fx
    gpu = fx.problem()
    free = cs.Problem(fx.C, fx.P, fx.cam, fx.pt, fx.obs)
    try:
        # getters refuse before any compute
        for call in (lambda: gpu.covariance_points(), lambda: gpu.covariance_cameras([(0, 1)])):
            with pytest.raises(B200Error) as e:
                call()
            assert e.value.code == ERR_INVALID_ARGUMENT
        with pytest.raises(B200Error) as e:
            gpu.covariance_compute(fx.state, algorithm=cs.ITERATIVE_SCHUR)
        assert e.value.code == ERR_UNSUPPORTED
        # the ungauged problem: S keeps the similarity gauge, so the compute is invalid, and the getters refuse
        for alg in (cs.SPARSE_SCHUR, cs.DENSE_SCHUR):
            assert not free.covariance_compute(fx.state, algorithm=alg)
            with pytest.raises(B200Error) as e:
                free.covariance_points()
            assert e.value.code == ERR_INVALID_ARGUMENT
        # mixed precision and refinement stay the handle's: a later sparse solve still refines in float
        gpu.set_exact_solve_options(True, 2)
        assert gpu.covariance_compute(fx.state)
        pairs = pattern_pairs(fx.C, fx.cam, fx.pt)
        cams, pts = gpu.covariance_cameras(pairs), gpu.covariance_points()
        assert not gpu.stats().get("refine_convert", {}).get("launches", 0)
        gpu.stats_reset()
        ok, _, res, _ = gpu.evaluate(fx.state)
        x, _, term = gpu.sparse_schur_solve(None, np.full(gpu.num_parameters, 1e-2))
        assert term == cs.LS_SUCCESS and gpu.stats()["refine_convert"]["launches"] > 0
        gpu.set_exact_solve_options(False, 0)
        # out-of-range and (C16's graph is complete, so) nothing out of pattern here: refused with the snapshot intact
        for bad in ([(0, fx.C)], [(-1, 0)]):
            with pytest.raises(B200Error) as e:
                gpu.covariance_cameras(bad)
            assert e.value.code == ERR_INVALID_ARGUMENT
        # the snapshot survives later evaluations, solves and setters
        gpu.lm_solve(fx.state, gpu.lm_options(max_num_iterations=2, linear_solver_type=cs.SPARSE_SCHUR))
        gpu.set_constant_blocks(None, None)
        gpu.set_linear_solver_ordering_type(cs.NESDIS)
        assert np.array_equal(gpu.covariance_cameras(pairs), cams)
        assert np.array_equal(gpu.covariance_points(), pts)
    finally:
        gpu.close()
        free.close()


def test_out_of_pattern_and_single_observation(cs):
    from ceres_solver_b200.binding import B200Error, ERR_INVALID_ARGUMENT
    fx = structure_fixture(cs, "band")
    gpu = fx.problem()
    try:
        assert gpu.covariance_compute(fx.state)
        pts = gpu.covariance_points()
        with pytest.raises(B200Error) as e:
            gpu.covariance_cameras([(0, 1), (1, fx.C - 1)])
        assert e.value.code == ERR_INVALID_ARGUMENT and "(1, %d)" % (fx.C - 1) in str(e.value)
        assert np.array_equal(gpu.covariance_points(), pts)
    finally:
        gpu.close()
    # one more point, seen once by camera 1 and variable: its E'E is singular
    cam = np.r_[fx.cam, 1].astype(np.int32)
    pt = np.r_[fx.pt, fx.P].astype(np.int32)
    obs, state = geometry(fx.C, fx.P + 1, cam, pt)
    one = Fixture(cs, fx.C, fx.P + 1, cam, pt, obs, state, fx.cc, np.r_[fx.pc, False])
    gpu = one.problem()
    try:
        assert not gpu.covariance_compute(one.state)
        with pytest.raises(B200Error):
            gpu.covariance_cameras([(0, 0)])
    finally:
        gpu.close()


def test_no_side_effects_on_lm(cs, c16fx):
    """An LM solve after compute gives the same trace as on a handle that never called it, wherever two runs of that handle
    agree bit for bit."""
    fx = c16fx
    opts = dict(max_num_iterations=4, linear_solver_type=cs.SPARSE_SCHUR)
    traces = []
    for with_cov in (False, False, True):
        gpu = fx.problem()
        try:
            if with_cov:
                assert gpu.covariance_compute(fx.state)
            traces.append(gpu.lm_solve(fx.state, gpu.lm_options(**opts)))
        finally:
            gpu.close()
    (s0, r0), (s1, r1), (s2, r2) = traces
    if np.array_equal(s0, s1) and r0 == r1:
        assert np.array_equal(s2, s0) and r2 == r0


def test_full_size_ladybug(cs):
    """Ladybug-1723-shaped data (the synthetic video sequence) with camera 0 and 1 % of the points constant: sparse (NESDIS)
    and dense agree, and sampled camera blocks match scipy splu solves of S on unit vectors."""
    import scipy.sparse as sps
    import scipy.sparse.linalg as spla
    from ceres_solver_b200 import bal as B
    from tests.constant_blocks_reference import jacobian_matrix
    bal = B.synthetic("ladybug-1723")
    rp = B.ReducedProgram(bal)
    state = rp.state(bal)
    cam, pt = np.asarray(rp.row_cam), np.asarray(rp.row_pt)
    cc = np.zeros(rp.C, bool)
    cc[0] = True
    seen = np.zeros(rp.P, bool)
    seen[pt[cam == 0]] = True
    pc = np.zeros(rp.P, bool)
    pc[np.random.RandomState(0).choice(np.flatnonzero(~seen), size=rp.P // 100, replace=False)] = True
    gpu = cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs)
    try:
        gpu.set_constant_blocks(cc, pc)
        gpu.set_linear_solver_ordering_type(cs.NESDIS)
        assert gpu.covariance_compute(state)
        pairs = pattern_pairs(rp.C, cam, pt)
        sc, sp_ = gpu.covariance_cameras(pairs), gpu.covariance_points()
        assert gpu.covariance_compute(state, algorithm=cs.DENSE_SCHUR)
        dc, dp = gpu.covariance_cameras(pairs), gpu.covariance_points()
        dc_rel = np.abs(sc - dc).max() / np.abs(dc).max()
        dp_rel = np.abs(sp_ - dp).max() / np.abs(dp).max()
        print("[covariance] ladybug-1723: sparse vs dense max rel. difference cameras %.2e, points %.2e" % (dc_rel, dp_rel))
        assert dc_rel <= 1e-6 and dp_rel <= 1e-6
        # S from the stored J in scipy, constant components as identity, and splu solves on unit vectors
        J = jacobian_matrix(gpu.jacobian_values(), cam, pt, rp.P, rp.C).tocsc()
        P3 = 3 * rp.P
        Je, Jf = J[:, :P3], J[:, P3:]
        V = (Je.T @ Je).tocsr()
        blocks = [np.eye(3) if pc[p] else np.linalg.inv(V[3 * p:3 * p + 3, 3 * p:3 * p + 3].toarray()) for p in range(rp.P)]
        Vi = sps.block_diag(blocks, format="csr")
        S = (Jf.T @ Jf - (Jf.T @ Je) @ Vi @ (Je.T @ Jf)).tolil()
        idx = np.flatnonzero(np.repeat(cc, 9))
        S[idx, :] = 0
        S[:, idx] = 0
        S[idx, idx] = 1
        lu = spla.splu(S.tocsc())
        rng = np.random.RandomState(1)
        sample = [pairs[k] for k in rng.choice(len(pairs), size=12, replace=False)] + [(5, 5)]
        got = gpu.covariance_cameras(sample)
        worst = 0.0
        for (i, j), blk in zip(sample, got):
            cols = np.zeros((9 * rp.C, 9))
            cols[9 * j + np.arange(9), np.arange(9)] = 1.0
            ref = lu.solve(cols)[9 * i:9 * i + 9]
            if cc[i] or cc[j]:
                assert not blk.any()
                continue
            worst = max(worst, np.abs(blk - ref).max() / np.abs(ref).max())
        print("[covariance] ladybug-1723: sampled blocks vs splu max rel. difference %.2e" % worst)
        assert worst <= 1e-6
    finally:
        gpu.close()
