"""The reduced program of a problem with constant parameter blocks, restated in numpy / scipy for the tests of
b200_set_constant_blocks (tests/test_gpu_constant_blocks.py, guarded on the CPU by tests/test_constant_blocks_reference.py).

Ceres removes constant blocks from the program it minimises (Program::RemoveFixedBlocks): their Jacobian columns are never
formed and the linear solves see only the variable columns.  Two restatements:
  - ReducedProgram: the oracle's own program with the constant blocks removed, a BlockSparseMatrix of the reduced
    structure, the oracle's solves and tests/dogleg_reference.py's trust-region loop on the reduced state;
  - jacobian_matrix / reduced_solve: a Jacobian in the library's value layout (all E cells [N][2][3], then all F cells
    [N][2][9]) as a scipy matrix, and a direct solve of the reduced regularised normal equations, for the larger fixtures.
"""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla


def fixed_components(C, P, camera_constant=None, point_constant=None):
    """[3P + 9C] bool: True on the components of constant blocks."""
    fixed = np.zeros(3 * P + 9 * C, dtype=bool)
    if point_constant is not None:
        fixed[:3 * P] = np.repeat(np.asarray(point_constant, dtype=bool), 3)
    if camera_constant is not None:
        fixed[3 * P:] = np.repeat(np.asarray(camera_constant, dtype=bool), 9)
    return fixed


def jacobian_matrix(values, row_cam, row_pt, P, C):
    """The [2N x (3P + 9C)] sparse Jacobian of a value array in the library's layout."""
    row_cam = np.asarray(row_cam, dtype=np.int64)
    row_pt = np.asarray(row_pt, dtype=np.int64)
    N = row_cam.size
    values = np.asarray(values, dtype=float)
    E = values[:6 * N].reshape(N, 2, 3)
    F = values[6 * N:].reshape(N, 2, 9)
    r = np.arange(N)
    rows_e = (2 * r[:, None, None] + np.arange(2)[None, :, None]).repeat(3, axis=2)
    cols_e = (3 * row_pt[:, None, None] + np.arange(3)[None, None, :]).repeat(2, axis=1)
    rows_f = (2 * r[:, None, None] + np.arange(2)[None, :, None]).repeat(9, axis=2)
    cols_f = (3 * P + 9 * row_cam[:, None, None] + np.arange(9)[None, None, :]).repeat(2, axis=1)
    data = np.concatenate([E.ravel(), F.ravel()])
    rows = np.concatenate([rows_e.ravel(), rows_f.ravel()])
    cols = np.concatenate([cols_e.ravel(), cols_f.ravel()])
    return sp.csr_matrix((data, (rows, cols)), shape=(2 * N, 3 * P + 9 * C))


def reduced_solve(J, b, D, fixed):
    """x of min |J_r x_r - b|^2 + |D_r x_r|^2 over the variable columns (fixed == False), 0 on the constant ones.
    D None: no regularisation."""
    keep = np.flatnonzero(~fixed)
    Jr = J[:, keep].tocsc()
    A = (Jr.T @ Jr).tocsc()
    if D is not None:
        A = A + sp.diags(np.asarray(D, dtype=float)[keep] ** 2)
    x = np.zeros(J.shape[1])
    x[keep] = spla.spsolve(A.tocsc(), Jr.T @ np.asarray(b, dtype=float))
    return x


def reduced_dense_solve(J, b, D, fixed):
    """reduced_solve by a dense numpy solve of the same normal equations (the guard of reduced_solve)."""
    keep = np.flatnonzero(~fixed)
    Jr = J[:, keep].toarray()
    A = Jr.T @ Jr
    if D is not None:
        A = A + np.diag(np.asarray(D, dtype=float)[keep] ** 2)
    x = np.zeros(J.shape[1])
    x[keep] = np.linalg.solve(A, Jr.T @ np.asarray(b, dtype=float))
    return x


def constant_sets(row_cam, row_pt, P, C, seed=0, cameras=2, per_class=2):
    """(camera_constant, point_constant) with `cameras` constant cameras and, in each class of points by rows (<= 32,
    33..128, > 128: the warp tiles, the CTA tiles and the huge points of the evaluate kernels), up to `per_class` constant
    points that no constant camera sees, so that no row has both blocks constant.  Every class keeps variable points."""
    row_cam = np.asarray(row_cam)
    row_pt = np.asarray(row_pt)
    rng = np.random.RandomState(seed)
    cam_const = np.zeros(C, dtype=bool)
    cam_const[rng.choice(C, size=cameras, replace=False)] = True
    seen = np.zeros(P, dtype=bool)
    seen[row_pt[cam_const[row_cam]]] = True
    deg = np.bincount(row_pt, minlength=P)
    pt_const = np.zeros(P, dtype=bool)
    for lo, hi in ((1, 32), (33, 128), (129, 1 << 30)):
        cand = np.flatnonzero((deg >= lo) & (deg <= hi) & ~seen)
        if cand.size > per_class:
            pt_const[rng.choice(cand, size=per_class, replace=False)] = True
    return cam_const, pt_const


class ReducedProgram:
    """Program::RemoveFixedBlocks restated on the oracle's own program of a BAL problem: the variable blocks only, with
    the same interface as the oracle's BaProgram (evaluate, jacobian, P = the eliminated blocks, default_options, solve)
    so that tests/dogleg_reference.py's trust-region loop runs on it.

    camera_constant / point_constant: [C] / [P] bool in the reduced program's block order (the order of the library's
    vectors).  The reduced state holds the variable points, then the variable cameras.  The Jacobian is a
    pyoracle.BlockSparseMatrix of the reduced structure: the rows of variable points first, grouped by point, each with its
    E cell and, unless its camera is constant, its F cell; then the rows of constant points, with their F cell only (the
    rows the Schur eliminator handles without an e block).  Its solves are the oracle's, with num_elim = the number of
    variable points."""

    def __init__(self, oracle, bal, camera_constant=None, point_constant=None):
        self.oracle = oracle
        self.base = b = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())
        C, P, N = b.C, b.P, b.N
        self.C_full, self.P_full, self.N = C, P, N
        self.cam_const = np.zeros(C, bool) if camera_constant is None else np.asarray(camera_constant, bool)
        self.pt_const = np.zeros(P, bool) if point_constant is None else np.asarray(point_constant, bool)
        row_pt, row_cam = np.asarray(b.row_pt), np.asarray(b.row_cam)
        assert not np.any(self.pt_const[row_pt] & self.cam_const[row_cam]), "a row with both blocks constant"
        self.fixed = fixed_components(C, P, self.cam_const, self.pt_const)
        vp, vc = np.flatnonzero(~self.pt_const), np.flatnonzero(~self.cam_const)
        self.P, self.C = int(vp.size), int(vc.size)
        pcol = np.full(P, -1)
        pcol[vp] = np.arange(vp.size)
        ccol = np.full(C, -1)
        ccol[vc] = self.P + np.arange(vc.size)
        self.rows = np.concatenate([np.flatnonzero(~self.pt_const[row_pt]), np.flatnonzero(self.pt_const[row_pt])])
        self.cells = [[c for c in (pcol[row_pt[r]], ccol[row_cam[r]]) if c >= 0] for r in self.rows]
        self.has_e = ~self.pt_const[row_pt[self.rows]]
        self.has_f = ~self.cam_const[row_cam[self.rows]]
        self.col_sizes = [3] * self.P + [9] * self.C
        self.num_parameters = 3 * self.P + 9 * self.C
        self.num_residuals = 2 * N
        self.res_idx = (2 * self.rows[:, None] + np.arange(2)).ravel()   # reduced residual k <- base residual res_idx[k]
        self.J = None
        self.state0 = None

    # ---- the reduced state and the full one
    def reduce(self, full):
        return np.asarray(full, dtype=float)[~self.fixed]

    def expand(self, x):
        full = np.array(self.state0, dtype=float)
        full[~self.fixed] = x
        return full

    def reduced_values(self, v):
        """The reduced Jacobian's values (cell order of self.cells) from a value array in the library's layout."""
        n6 = 6 * self.N
        cells = np.concatenate([np.asarray(v[:n6]).reshape(self.N, 6), np.asarray(v[n6:]).reshape(self.N, 18)], axis=1)
        keep = np.concatenate([np.repeat(self.has_e[:, None], 6, axis=1), np.repeat(self.has_f[:, None], 18, axis=1)], axis=1)
        return cells[self.rows][keep]

    def evaluate(self, x, want_residuals=True, want_gradient=True, want_jacobian=True, nt=1):
        """x: the reduced state.  The base program evaluates the full state (constant blocks at their values in
        state0); the kept cells make the reduced Jacobian."""
        need_j = want_gradient or want_jacobian
        ok, cost, r, _ = self.base.evaluate(self.expand(x), want_residuals=True, want_gradient=False,
                                            want_jacobian=need_j, nt=nt)
        if not ok:
            return False, float("nan"), None, None
        rr = r[self.res_idx]
        grad = None
        if need_j:
            J = self.oracle.BlockSparseMatrix(self.col_sizes, [2] * self.rows.size, self.cells,
                                              self.reduced_values(self.base.jacobian().values()))
            if want_jacobian:
                self.J = J
            if want_gradient:
                grad = J.left_multiply(rr, nt=nt)
        return True, cost, rr if want_residuals else None, grad

    def jacobian(self):
        return self.J

    def default_options(self):
        return self.base.default_options()

    def solve(self, state, options=None, dogleg_type=None):
        """TrustRegionMinimizer::Minimize on the reduced program from the full state `state`: LevenbergMarquardtStrategy
        (tests/test_oracle_losses.py) when dogleg_type is None, else DoglegStrategy over DENSE_SCHUR.  Returns (full best
        state, records)."""
        from tests import dogleg_reference as DR
        from tests.test_oracle_losses import LevenbergMarquardtStrategy
        o = options or self.default_options()
        self.state0 = np.array(state, dtype=float)
        names = ("max_num_iterations", "initial_trust_region_radius", "min_trust_region_radius", "min_relative_decrease",
                 "min_lm_diagonal", "max_lm_diagonal", "function_tolerance", "gradient_tolerance", "parameter_tolerance",
                 "jacobi_scaling", "max_num_consecutive_invalid_steps")
        kw = {k: getattr(o, k) for k in names}
        if dogleg_type is not None:
            best, recs, _ = DR.minimize(self, self.reduce(state), dogleg_type, nt=o.num_threads, **kw)
        else:
            saved = DR.DoglegStrategy
            DR.DoglegStrategy = lambda *args: LevenbergMarquardtStrategy(o, o.num_threads)
            try:
                best, recs, _ = DR.minimize(self, self.reduce(state), None, nt=o.num_threads, **kw)
            finally:
                DR.DoglegStrategy = saved
        return self.expand(best), recs
