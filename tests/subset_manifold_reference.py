"""The tangent-space program of a problem with SubsetManifolds on its cameras and points, restated on the oracle for the
tests of b200_set_subset_manifolds (tests/test_gpu_subset_manifold.py, guarded on the CPU by
tests/test_subset_manifold_reference.py).

Ceres minimises over each block's tangent space: the Jacobian it solves with is J_ambient * PlusJacobian, and
SubsetManifold's PlusJacobian is a 0/1 selection matrix (manifold.cc:168-180), so the columns of the constant coordinates
are not there.  A block whose every coordinate is held has tangent size 0 and is constant (ParameterBlock::IsConstant),
so the program drops it as Program::RemoveFixedBlocks drops a constant block.  SubsetProgram is
tests/constant_blocks_reference.py's ReducedProgram with that extension: column blocks of 9 - popcount(camera mask) and
3 - popcount(point mask), cells with the variable columns only, the oracle's dynamic-size Schur path for the solves, and
tests/dogleg_reference.py's trust-region loop on the reduced (tangent) state.

Two things follow Ceres here because the base program does them: evaluate() checks the ambient Jacobian (a non-finite
value in a masked column fails the evaluation), and the reduced state has no masked coordinate.  The latter differs from
Ceres in one place, |x| of parameter_tolerance, which Ceres takes over the variable blocks' ambient state; the GPU test
of that rule computes its threshold itself.
"""
import numpy as np

from tests import constant_blocks_reference as R


def masked_components(C, P, camera_mask=None, point_mask=None):
    """[3P + 9C] bool: True on the coordinates the masks hold ((C, 9) and (P, 3) bool, or None)."""
    out = np.zeros(3 * P + 9 * C, dtype=bool)
    if point_mask is not None:
        out[:3 * P] = np.asarray(point_mask, dtype=bool).reshape(P, 3).ravel()
    if camera_mask is not None:
        out[3 * P:] = np.asarray(camera_mask, dtype=bool).reshape(C, 9).ravel()
    return out


def effective(C, P, camera_constant=None, point_constant=None, camera_mask=None, point_mask=None):
    """(camera constant [C], point constant [P], fixed [3P + 9C], masked [3P + 9C]) as ParameterBlock sees them: a block is
    constant when set constant or when its mask is full; `fixed` is True on every constant component (the components the
    solves return as 0), `masked` on the held coordinates of variable blocks only."""
    cm = np.zeros((C, 9), bool) if camera_mask is None else np.asarray(camera_mask, bool).reshape(C, 9)
    pm = np.zeros((P, 3), bool) if point_mask is None else np.asarray(point_mask, bool).reshape(P, 3)
    cc = (np.zeros(C, bool) if camera_constant is None else np.asarray(camera_constant, bool)) | cm.all(axis=1)
    pc = (np.zeros(P, bool) if point_constant is None else np.asarray(point_constant, bool)) | pm.all(axis=1)
    block = R.fixed_components(C, P, cc, pc)
    fixed = block | masked_components(C, P, cm, pm)
    return cc, pc, fixed, fixed & ~block


class SubsetProgram(R.ReducedProgram):
    """ReducedProgram with SubsetManifolds: camera_mask (C, 9) / point_mask (P, 3) bool in the library's block order,
    True = coordinate held constant.  Fully masked blocks count as constant."""

    def __init__(self, oracle, bal, camera_constant=None, point_constant=None, camera_mask=None, point_mask=None):
        C, P = bal.C, bal.P
        cc, pc, fixed, masked = effective(C, P, camera_constant, point_constant, camera_mask, point_mask)
        super().__init__(oracle, bal, cc, pc)
        self.cam_mask = np.zeros((C, 9), bool) if camera_mask is None else np.asarray(camera_mask, bool).reshape(C, 9)
        self.pt_mask = np.zeros((P, 3), bool) if point_mask is None else np.asarray(point_mask, bool).reshape(P, 3)
        self.block_fixed = self.fixed
        self.fixed = fixed        # reduce / expand: the tangent coordinates of the variable blocks
        self.masked = masked
        vp, vc = np.flatnonzero(~self.pt_const), np.flatnonzero(~self.cam_const)
        self.col_sizes = [int(3 - self.pt_mask[p].sum()) for p in vp] + [int(9 - self.cam_mask[c].sum()) for c in vc]
        self.num_parameters = int(sum(self.col_sizes))
        assert self.num_parameters == int((~fixed).sum())
        # [N, 24] True on the cells the tangent Jacobian keeps, in the library's value layout of each row
        row_pt, row_cam = np.asarray(self.base.row_pt), np.asarray(self.base.row_cam)
        keep_e = ~self.pt_const[row_pt][:, None, None] & ~self.pt_mask[row_pt][:, None, :]
        keep_f = ~self.cam_const[row_cam][:, None, None] & ~self.cam_mask[row_cam][:, None, :]
        self.keep_cells = np.concatenate([np.broadcast_to(keep_e, (self.N, 2, 3)).reshape(self.N, 6),
                                          np.broadcast_to(keep_f, (self.N, 2, 9)).reshape(self.N, 18)], axis=1)

    def reduced_values(self, v):
        """The tangent Jacobian's values (cell order of self.cells, each cell [2][tangent size] row-major)."""
        n6 = 6 * self.N
        cells = np.concatenate([np.asarray(v[:n6]).reshape(self.N, 6), np.asarray(v[n6:]).reshape(self.N, 18)], axis=1)
        return cells[self.rows][self.keep_cells[self.rows]]

    def tangent_solve(self, J_full_values, b, D, solver=1, **kw):
        """The oracle's solve (pyoracle.BlockSparseMatrix.linear_solve: solver 0 = ITERATIVE_SCHUR, 1 = DENSE_SCHUR, and
        its keywords) of the tangent program's regularised normal equations, from a Jacobian in the library's layout
        (masked and constant columns dropped) and a full-length D.  Returns (full-length solution with 0 on every constant
        component, the oracle's iteration count, its termination type)."""
        J = self.oracle.BlockSparseMatrix(self.col_sizes, [2] * self.rows.size, self.cells, self.reduced_values(J_full_values))
        rr = np.asarray(b, dtype=float)[self.res_idx]
        Dr = None if D is None else np.asarray(D, dtype=float)[~self.fixed]
        x, iterations, term = J.linear_solve(self.P, rr, Dr, solver=solver, **kw)
        out = np.zeros(3 * self.P_full + 9 * self.C_full)
        out[~self.fixed] = x
        return out, iterations, term


def c16_mask_sets(P, C, row_cam, row_pt, seed=0):
    """The SubsetManifold sets of the C16 tests, {name: (camera_constant, point_constant, camera_mask, point_mask)}:
      - intrinsics: focal length and distortion held on every camera, SubsetManifold(9, {6, 7, 8}) (calibrated cameras);
      - mixed: a random non-empty, non-full subset on every camera and one or two coordinates on a tenth of the points;
      - heights: the third coordinate of a tenth of the points, SubsetManifold(3, {2}) (control points of known height);
      - combined: camera 0 constant, intrinsics held on the others, and three points no row of camera 0 sees constant,
        with heights held on other points."""
    row_cam, row_pt = np.asarray(row_cam), np.asarray(row_pt)
    rng = np.random.RandomState(seed)
    out = {}
    cm = np.zeros((C, 9), bool)
    cm[:, 6:] = True
    out["intrinsics"] = (None, None, cm, None)
    cm = np.zeros((C, 9), bool)
    for c in range(C):
        cm[c, rng.choice(9, size=rng.randint(1, 9), replace=False)] = True
    pm = np.zeros((P, 3), bool)
    for p in rng.choice(P, size=P // 10, replace=False):
        pm[p, rng.choice(3, size=rng.randint(1, 3), replace=False)] = True
    out["mixed"] = (None, None, cm, pm)
    pm = np.zeros((P, 3), bool)
    pm[rng.choice(P, size=P // 10, replace=False), 2] = True
    out["heights"] = (None, None, None, pm)
    cam = np.zeros(C, bool)
    cam[0] = True
    seen = np.zeros(P, bool)
    seen[row_pt[row_cam == 0]] = True
    pts = np.zeros(P, bool)
    pts[np.flatnonzero(~seen)[[0, 100, 1000]]] = True
    cm = np.zeros((C, 9), bool)
    cm[1:, 6:] = True
    pm2 = pm.copy()
    pm2[pts] = False
    out["combined"] = (cam, pts, cm, pm2)
    return out


def mask_sets(row_cam, row_pt, P, C, seed=0, per_class=2):
    """(camera_mask (C, 9), point_mask (P, 3)) for the larger fixtures: a random non-empty, non-full subset on every camera,
    and in each class of points by rows (<= 32, 33..128, > 128: the warp tiles, the CTA tiles and the huge points of the
    evaluate kernels) up to `per_class` points with one or two held coordinates.  Every class keeps unmasked points, and no
    block is fully masked."""
    row_pt = np.asarray(row_pt)
    rng = np.random.RandomState(seed)
    cm = np.zeros((C, 9), bool)
    for c in range(C):
        cm[c, rng.choice(9, size=rng.randint(1, 9), replace=False)] = True
    deg = np.bincount(row_pt, minlength=P)
    pm = np.zeros((P, 3), bool)
    for lo, hi in ((1, 32), (33, 128), (129, 1 << 30)):
        cand = np.flatnonzero((deg >= lo) & (deg <= hi))
        if cand.size > per_class:
            for p in rng.choice(cand, size=per_class, replace=False):
                pm[p, rng.choice(3, size=rng.randint(1, 3), replace=False)] = True
    return cm, pm


def cell_mask(row_cam, row_pt, camera_constant, point_constant, camera_mask, point_mask):
    """[24N] True on the cells the library stores as 0 (constant blocks and masked columns), in its value layout."""
    row_cam, row_pt = np.asarray(row_cam), np.asarray(row_pt)
    N = row_cam.size
    C, P = len(camera_mask), len(point_mask)
    cc, pc, _, _ = effective(C, P, camera_constant, point_constant, camera_mask, point_mask)
    pm = np.asarray(point_mask, bool)[row_pt] | pc[row_pt][:, None]
    cm = np.asarray(camera_mask, bool)[row_cam] | cc[row_cam][:, None]
    e = np.broadcast_to(pm[:, None, :], (N, 2, 3)).reshape(-1)
    f = np.broadcast_to(cm[:, None, :], (N, 2, 9)).reshape(-1)
    return np.concatenate([e, f])
