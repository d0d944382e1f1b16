"""ctypes binding of libb200ba.so (include/b200ba.h).

This is plumbing for tests and bench.py: numpy arrays in, numpy arrays out, every call going through the
C ABI exactly as the Ceres adapters would.  There is no CPU fallback: a missing library or a missing GPU
raises.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
# (B200BA_LIB: tooling only -- lets tools/ A/B scripts load a -DB200_DEV_KNOBS build of the same library)
LIB_PATH = os.environ.get("B200BA_LIB") or os.path.join(_HERE, "libb200ba.so")

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int32)

OK = 0
ERR_INVALID_ARGUMENT = -1
ERR_EVALUATION_FAILED = -3
ERR_UNSUPPORTED = -6
LS_SUCCESS, LS_NO_CONVERGENCE, LS_FAILURE, LS_FATAL_ERROR = 0, 1, 2, 3
PRECOND_IDENTITY, PRECOND_JACOBI, PRECOND_SCHUR_JACOBI, PRECOND_SCHUR_POWER_SERIES_EXPANSION = 0, 1, 2, 3
ITERATIVE_SCHUR, DENSE_SCHUR, SPARSE_SCHUR = 0, 1, 2
LEVENBERG_MARQUARDT, DOGLEG = 0, 1                  # trust_region_strategy_type
TRADITIONAL_DOGLEG, SUBSPACE_DOGLEG = 0, 1          # dogleg_type
AMD, NESDIS = 0, 1                                  # linear_solver_ordering_type
# b200_plan_sparse_schur's statistics (B200_SPARSE_STAT_*), in order
SPARSE_STATS = ("s_blocks", "l_blocks", "l_blocks_caller", "l_blocks_min_degree", "flops_caller", "flops_min_degree",
                "supernodes", "tree_height", "order", "factor_bytes", "flops", "critical_path_supernodes",
                "critical_path_flops")
# B200_LOSS_*, in the order of include/ceres/loss_function.h
LOSS_TRIVIAL, LOSS_HUBER, LOSS_SOFT_L_ONE, LOSS_CAUCHY, LOSS_ARCTAN, LOSS_TOLERANT, LOSS_TUKEY = range(7)


class B200Error(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libb200ba error %d: %s" % (code, msg))
        self.code = code


class BaDesc(C.Structure):
    _fields_ = [("num_cameras", C.c_int32), ("num_points", C.c_int32), ("num_observations", C.c_int64),
                ("cam_idx", _ip), ("pt_idx", _ip), ("obs", _dp), ("loss_type", C.c_int32), ("loss_a", C.c_double),
                ("device", C.c_int32), ("stream", C.c_void_p), ("rank", C.c_int32), ("world_size", C.c_int32),
                ("nccl_unique_id", C.c_void_p)]


class Loss(C.Structure):
    """b200_loss: one loss object; a, b its constructor arguments (only TolerantLoss reads b), scale ScaledLoss's factor."""
    _fields_ = [("type", C.c_int32), ("a", C.c_double), ("b", C.c_double), ("scale", C.c_double)]


class SolverOptions(C.Structure):
    _fields_ = [("preconditioner_type", C.c_int32), ("min_num_iterations", C.c_int32),
                ("max_num_iterations", C.c_int32), ("residual_reset_period", C.c_int32),
                ("q_tolerance", C.c_double), ("r_tolerance", C.c_double),
                ("max_num_spse_iterations", C.c_int32), ("use_spse_initialization", C.c_int32),
                ("spse_tolerance", C.c_double)]


class SolverSummary(C.Structure):
    _fields_ = [("residual_norm", C.c_double), ("num_iterations", C.c_int32), ("termination_type", C.c_int32)]


class LmOptions(C.Structure):
    _fields_ = [("max_num_iterations", C.c_int32), ("jacobi_scaling", C.c_int32),
                ("max_num_consecutive_invalid_steps", C.c_int32), ("linear_solver_type", C.c_int32), ("eta", C.c_double),
                ("initial_trust_region_radius", C.c_double), ("max_trust_region_radius", C.c_double),
                ("min_trust_region_radius", C.c_double), ("min_relative_decrease", C.c_double),
                ("min_lm_diagonal", C.c_double), ("max_lm_diagonal", C.c_double), ("function_tolerance", C.c_double),
                ("gradient_tolerance", C.c_double), ("parameter_tolerance", C.c_double),
                ("linear_solver", SolverOptions), ("trust_region_strategy_type", C.c_int32), ("dogleg_type", C.c_int32),
                ("use_mixed_precision_solves", C.c_int32), ("max_num_refinement_iterations", C.c_int32),
                ("linear_solver_ordering_type", C.c_int32)]


class CovarianceOptions(C.Structure):
    """b200_covariance_options: Covariance::Options' algorithm_type, min_reciprocal_condition_number, apply_loss_function."""
    _fields_ = [("algorithm", C.c_int32), ("min_reciprocal_condition_number", C.c_double),
                ("apply_loss_function", C.c_int32)]


class LmIteration(C.Structure):
    _fields_ = [("iteration", C.c_int32), ("linear_solver_iterations", C.c_int32), ("step_is_valid", C.c_int32),
                ("step_is_successful", C.c_int32), ("cost", C.c_double), ("cost_change", C.c_double),
                ("gradient_max_norm", C.c_double), ("gradient_norm", C.c_double), ("step_norm", C.c_double),
                ("relative_decrease", C.c_double), ("trust_region_radius", C.c_double),
                ("model_cost_change", C.c_double)]


class KernelStat(C.Structure):
    _fields_ = [("name", C.c_char * 32), ("launches", C.c_int64), ("operations", C.c_int64),
                ("device_ms", C.c_double), ("bytes_per_operation", C.c_double)]


# Every symbol include/b200ba.h declares (tests/test_abi.py checks the library exports all of them).
SYMBOLS = [
    "b200_plan_point_order", "b200_plan_sparse_schur", "b200_plan_sparse_schur_ordered", "b200_sparse_schur_solve", "b200_nccl_unique_id", "b200_create", "b200_destroy", "b200_last_error", "b200_num_parameters",
    "b200_num_residuals", "b200_evaluate", "b200_set_apply_loss_function", "b200_set_loss_functions", "b200_set_constant_blocks", "b200_set_subset_manifolds", "b200_plus", "b200_jacobian_squared_column_norm",
    "b200_jacobian_scale_columns", "b200_jacobian_right_multiply", "b200_jacobian_left_multiply", "b200_model_cost_change",
    "b200_jacobian_get_values", "b200_jacobian_set_values", "b200_partitioned_multiply", "b200_jtj_multiply", "b200_solver_options_default",
    "b200_schur_solve", "b200_dense_schur_solve", "b200_set_exact_solve_options",
    "b200_set_linear_solver_ordering_type", "b200_schur_init", "b200_schur_rhs", "b200_schur_ete_inverse", "b200_schur_multiply",
    "b200_schur_back_substitute", "b200_schur_jacobi_update", "b200_block_jacobi_update",
    "b200_lm_options_default", "b200_lm_solve", "b200_profile_enable", "b200_stats_reset", "b200_stats_get",
    "b200_total_launches", "b200_synchronize", "b200_transfer_bytes", "b200_covariance_options_default",
    "b200_covariance_compute", "b200_covariance_cameras", "b200_covariance_points", "b200_plan_sparse_selinv",
]

_lib = None


def lib():
    """Loads libb200ba.so (built by __graft_entry__.build()); raises if it is missing."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("%s not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(there is no CPU fallback)" % LIB_PATH)
        _lib = C.CDLL(LIB_PATH)
        _lib.b200_last_error.restype = C.c_char_p
        _lib.b200_num_residuals.restype = C.c_int64
        _lib.b200_total_launches.restype = C.c_int64
    return _lib


def _d(a):
    return None if a is None else a.ctypes.data_as(_dp)


def _f64(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64)


def _check(rc):
    if rc != OK:
        raise B200Error(rc, lib().b200_last_error().decode())


def plan_point_order(num_cameras, num_points, cam_idx, pt_idx, num_chunks=132):
    """Host-only: the internal point order b200_create would choose.  Returns (perm, metrics[4], choice)."""
    cam = np.ascontiguousarray(cam_idx, dtype=np.int32)
    pt = np.ascontiguousarray(pt_idx, dtype=np.int32)
    d = BaDesc()
    d.num_cameras, d.num_points, d.num_observations = int(num_cameras), int(num_points), len(cam)
    d.cam_idx = cam.ctypes.data_as(_ip)
    d.pt_idx = pt.ctypes.data_as(_ip)
    perm = np.zeros(int(num_points), dtype=np.int32)
    metrics = (C.c_int64 * 4)()
    choice = C.c_int()
    _check(lib().b200_plan_point_order(C.byref(d), int(num_chunks), perm.ctypes.data_as(_ip), metrics, C.byref(choice)))
    return perm, [int(m) for m in metrics], choice.value


def plan_sparse_schur(num_cameras, num_points, cam_idx, pt_idx, ordering_type=AMD):
    """Host-only: the symbolic analysis b200_sparse_schur_solve runs for this structure under `ordering_type` (AMD or
    NESDIS).  Returns (camera elimination order, dict of SPARSE_STATS)."""
    cam = np.ascontiguousarray(cam_idx, dtype=np.int32)
    pt = np.ascontiguousarray(pt_idx, dtype=np.int32)
    d = BaDesc()
    d.num_cameras, d.num_points, d.num_observations = int(num_cameras), int(num_points), len(cam)
    d.cam_idx = cam.ctypes.data_as(_ip)
    d.pt_idx = pt.ctypes.data_as(_ip)
    perm = np.zeros(int(num_cameras), dtype=np.int32)
    stats = (C.c_int64 * len(SPARSE_STATS))()
    _check(lib().b200_plan_sparse_schur_ordered(C.byref(d), int(ordering_type), perm.ctypes.data_as(_ip), stats))
    return perm, {k: int(v) for k, v in zip(SPARSE_STATS, stats)}


def plan_sparse_selinv(num_cameras, num_points, cam_idx, pt_idx, ordering_type=AMD):
    """Host-only: the selected inversion's task graph for this structure.  Returns (sn_first [ns + 1], order [ns],
    counter init [ns])."""
    cam = np.ascontiguousarray(cam_idx, dtype=np.int32)
    pt = np.ascontiguousarray(pt_idx, dtype=np.int32)
    d = BaDesc()
    d.num_cameras, d.num_points, d.num_observations = int(num_cameras), int(num_points), len(cam)
    d.cam_idx = cam.ctypes.data_as(_ip)
    d.pt_idx = pt.ctypes.data_as(_ip)
    ns = C.c_int32()
    first = np.zeros(int(num_cameras) + 1, dtype=np.int32)
    order = np.zeros(int(num_cameras), dtype=np.int32)
    cnt = np.zeros(int(num_cameras), dtype=np.int32)
    _check(lib().b200_plan_sparse_selinv(C.byref(d), int(ordering_type), C.byref(ns), first.ctypes.data_as(_ip),
                                         order.ctypes.data_as(_ip), cnt.ctypes.data_as(_ip)))
    n = ns.value
    return first[:n + 1].copy(), order[:n].copy(), cnt[:n].copy()


def subset_manifold_masks(num_cameras, num_points, camera_constant=None, point_constant=None):
    """The bit masks b200_set_subset_manifolds takes, from boolean arrays of shape (C, 9) and (P, 3) (True = coordinate
    held constant: SubsetManifold(9 | 3, {k : True})), or None for no SubsetManifold on any block of that kind.  Returns
    (uint16 [C] or None, uint8 [P] or None); ValueError on a shape mismatch."""
    out = []
    for a, n, width, dtype, what in ((camera_constant, num_cameras, 9, np.uint16, "camera_constant"),
                                     (point_constant, num_points, 3, np.uint8, "point_constant")):
        if a is None:
            out.append(None)
            continue
        a = np.asarray(a).astype(bool)
        if a.shape != (int(n), width):
            raise ValueError("%s has shape %s for (%d, %d)" % (what, a.shape, int(n), width))
        out.append(np.ascontiguousarray((a.astype(np.uint32) << np.arange(width, dtype=np.uint32)).sum(axis=1).astype(dtype)))
    return out[0], out[1]


def nccl_unique_id():
    buf = (C.c_char * 128)()
    _check(lib().b200_nccl_unique_id(buf))
    return bytes(buf)


class Problem:
    """One b200_handle: a BAL-shaped problem resident on one GPU.

    cam_idx / pt_idx / obs are in reduced-program row order (rows grouped by point)."""

    def __init__(self, num_cameras, num_points, cam_idx, pt_idx, obs, loss_type=LOSS_TRIVIAL, loss_a=1.0, device=0,
                 stream=None, rank=0, world_size=1, nccl_id=None):
        self._cam = np.ascontiguousarray(cam_idx, dtype=np.int32)
        self._pt = np.ascontiguousarray(pt_idx, dtype=np.int32)
        self._obs = _f64(obs).ravel()
        d = BaDesc()
        d.num_cameras, d.num_points, d.num_observations = int(num_cameras), int(num_points), len(self._cam)
        d.cam_idx = self._cam.ctypes.data_as(_ip)
        d.pt_idx = self._pt.ctypes.data_as(_ip)
        d.obs = _d(self._obs)
        d.loss_type, d.loss_a, d.device = int(loss_type), float(loss_a), int(device)
        d.stream = stream
        d.rank, d.world_size = int(rank), int(world_size)
        self._nccl = C.create_string_buffer(nccl_id, 128) if nccl_id is not None else None
        d.nccl_unique_id = C.cast(self._nccl, C.c_void_p) if self._nccl is not None else None
        self.h = C.c_void_p()
        rc = lib().b200_create(C.byref(d), C.byref(self.h))
        if rc != OK:
            msg = lib().b200_last_error().decode()
            if self.h:
                lib().b200_destroy(self.h)
                self.h = C.c_void_p()
            raise B200Error(rc, msg)
        self.C, self.P, self.N = int(num_cameras), int(num_points), len(self._cam)
        self.num_parameters = lib().b200_num_parameters(self.h)
        self.num_residuals = lib().b200_num_residuals(self.h)

    def close(self):
        if getattr(self, "h", None):
            lib().b200_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- Evaluator
    def evaluate(self, state, want_residuals=True, want_gradient=True, want_jacobian=True):
        state = _f64(state)
        cost = C.c_double()
        res = np.zeros(self.num_residuals) if want_residuals else None
        grad = np.zeros(self.num_parameters) if want_gradient else None
        rc = lib().b200_evaluate(self.h, _d(state), C.byref(cost), _d(res), _d(grad), int(want_jacobian))
        if rc == ERR_EVALUATION_FAILED:
            return False, float("nan"), res, grad
        _check(rc)
        return True, cost.value, res, grad

    def set_apply_loss_function(self, apply):
        _check(lib().b200_set_apply_loss_function(self.h, int(bool(apply))))

    def set_loss_functions(self, losses, row_loss=None):
        """b200_set_loss_functions: `losses` is a sequence of (type, a, b, scale) tuples (or Loss structures), the table of
        loss objects; `row_loss` the table index of each row, in this problem's row order (None: every row uses losses[0],
        which needs exactly one loss)."""
        table = (Loss * max(1, len(losses)))()
        for k, l in enumerate(losses):
            table[k] = l if isinstance(l, Loss) else Loss(*(int(l[0]),) + tuple(float(v) for v in l[1:]))
        rows = None if row_loss is None else np.ascontiguousarray(row_loss, dtype=np.int32)
        if rows is not None and rows.size != self.N:
            raise ValueError("row_loss has %d entries for %d rows" % (rows.size, self.N))
        _check(lib().b200_set_loss_functions(self.h, table, len(losses), None if rows is None else rows.ctypes.data_as(_ip)))

    def set_constant_blocks(self, camera_constant=None, point_constant=None):
        """b200_set_constant_blocks: boolean arrays of C cameras and of this problem's P points (True = constant); None =
        none.  Replaces the problem's set (Problem::SetParameterBlockConstant / SetParameterBlockVariable)."""
        flags = []
        for a, n, what in ((camera_constant, self.C, "camera_constant"), (point_constant, self.P, "point_constant")):
            if a is None:
                flags.append(None)
                continue
            a = np.ascontiguousarray(np.asarray(a).astype(bool).astype(np.uint8))
            if a.size != n:
                raise ValueError("%s has %d entries for %d blocks" % (what, a.size, n))
            flags.append(a)
        _check(lib().b200_set_constant_blocks(self.h, *(None if a is None else a.ctypes.data_as(C.POINTER(C.c_uint8))
                                                       for a in flags)))

    def set_subset_manifolds(self, camera_constant=None, point_constant=None):
        """b200_set_subset_manifolds: boolean arrays of shape (C, 9) and (this problem's P, 3), True on the coordinates
        each block's SubsetManifold holds constant; None = no SubsetManifold on any block of that kind.  Replaces the
        problem's masks (Problem::SetManifold) and leaves its constant blocks alone."""
        cam, pts = subset_manifold_masks(self.C, self.P, camera_constant, point_constant)
        _check(lib().b200_set_subset_manifolds(self.h, None if cam is None else cam.ctypes.data_as(C.POINTER(C.c_uint16)),
                                               None if pts is None else pts.ctypes.data_as(C.POINTER(C.c_uint8))))

    # ---- Jacobian as a SparseMatrix
    def squared_column_norm(self):
        out = np.zeros(self.num_parameters)
        _check(lib().b200_jacobian_squared_column_norm(self.h, _d(out)))
        return out

    def scale_columns(self, scale):
        _check(lib().b200_jacobian_scale_columns(self.h, _d(_f64(scale))))

    def right_multiply(self, x, y=None):
        y = np.zeros(self.num_residuals) if y is None else _f64(y).copy()
        _check(lib().b200_jacobian_right_multiply(self.h, _d(_f64(x)), _d(y)))
        return y

    def left_multiply(self, x, y=None):
        y = np.zeros(self.num_parameters) if y is None else _f64(y).copy()
        _check(lib().b200_jacobian_left_multiply(self.h, _d(_f64(x)), _d(y)))
        return y

    def partitioned_multiply(self, op, x, y=None):
        """op: 0 y += E x_e, 1 y += F x_f, 2 y += E'x, 3 y += F'x  (PartitionedMatrixView)."""
        n_out = (self.num_residuals, self.num_residuals, 3 * self.P, 9 * self.C)[op]
        y = np.zeros(n_out) if y is None else _f64(y).copy()
        _check(lib().b200_partitioned_multiply(self.h, int(op), _d(_f64(x)), _d(y)))
        return y

    def jtj_multiply(self, x, D=None):
        y = np.zeros(self.num_parameters)
        _check(lib().b200_jtj_multiply(self.h, _d(_f64(x)), _d(_f64(D)), _d(y)))
        return y

    def jacobian_values(self):
        v = np.zeros(24 * self.N)
        _check(lib().b200_jacobian_get_values(self.h, _d(v)))
        return v

    def set_jacobian_values(self, v):
        v = _f64(v)
        assert v.size == 24 * self.N
        _check(lib().b200_jacobian_set_values(self.h, _d(v)))

    # ---- LinearSolver
    @staticmethod
    def solver_options(**kw):
        o = SolverOptions()
        lib().b200_solver_options_default(C.byref(o))
        for k, v in kw.items():
            setattr(o, k, v)
        return o

    def schur_solve(self, b, D, options=None):
        o = options or self.solver_options()
        x = np.full(self.num_parameters, np.nan)
        s = SolverSummary()
        bp = _d(_f64(b)) if b is not None else None  # None: the residuals of the last evaluate(), still in HBM
        _check(lib().b200_schur_solve(self.h, bp, _d(_f64(D)), C.byref(o), _d(x), C.byref(s)))
        return x, s.num_iterations, s.termination_type

    def dense_schur_solve(self, b, D):
        x = np.full(self.num_parameters, np.nan)
        s = SolverSummary()
        bp = _d(_f64(b)) if b is not None else None
        _check(lib().b200_dense_schur_solve(self.h, bp, _d(_f64(D)), _d(x), C.byref(s)))
        return x, s.num_iterations, s.termination_type

    def sparse_schur_solve(self, b, D):
        x = np.full(self.num_parameters, np.nan)
        s = SolverSummary()
        bp = _d(_f64(b)) if b is not None else None
        _check(lib().b200_sparse_schur_solve(self.h, bp, _d(_f64(D)), _d(x), C.byref(s)))
        return x, s.num_iterations, s.termination_type

    def set_exact_solve_options(self, use_mixed_precision_solves=False, max_num_refinement_iterations=0):
        """LinearSolver::Options::use_mixed_precision_solves / max_num_refinement_iterations of the later dense and sparse
        Schur solves on this handle."""
        _check(lib().b200_set_exact_solve_options(self.h, int(use_mixed_precision_solves), int(max_num_refinement_iterations)))

    def set_linear_solver_ordering_type(self, ordering_type):
        """Solver::Options::linear_solver_ordering_type (AMD or NESDIS) of the later sparse Schur solves on this handle; a
        change drops the handle's sparse analysis, which the next sparse solve runs again."""
        _check(lib().b200_set_linear_solver_ordering_type(self.h, int(ordering_type)))

    def model_cost_change(self, step):
        out = C.c_double(0.0)
        _check(lib().b200_model_cost_change(self.h, _d(_f64(step)), C.byref(out)))
        return out.value

    def schur_init(self, b, D):
        _check(lib().b200_schur_init(self.h, _d(_f64(b)), _d(_f64(D))))

    def schur_rhs(self):
        out = np.zeros(9 * self.C)
        _check(lib().b200_schur_rhs(self.h, _d(out)))
        return out

    def schur_ete_inverse(self):
        out = np.zeros(9 * self.P)
        _check(lib().b200_schur_ete_inverse(self.h, _d(out)))
        return out

    def schur_multiply(self, x):
        y = np.zeros(9 * self.C)
        _check(lib().b200_schur_multiply(self.h, _d(_f64(x)), _d(y)))
        return y

    def schur_back_substitute(self, z):
        y = np.zeros(self.num_parameters)
        _check(lib().b200_schur_back_substitute(self.h, _d(_f64(z)), _d(y)))
        return y

    def schur_jacobi_update(self):
        blocks = np.zeros(81 * self.C)
        inv = np.zeros(81 * self.C)
        _check(lib().b200_schur_jacobi_update(self.h, _d(blocks), _d(inv)))
        return blocks, inv

    def block_jacobi_update(self):
        inv = np.zeros(81 * self.C)
        _check(lib().b200_block_jacobi_update(self.h, _d(inv)))
        return inv

    # ---- Covariance
    def covariance_compute(self, state, algorithm=SPARSE_SCHUR, min_reciprocal_condition_number=1e-14,
                           apply_loss_function=True):
        """b200_covariance_compute: Covariance::Compute at `state`; returns its bool (False: not positive definite or
        worse conditioned than min_reciprocal_condition_number)."""
        o = CovarianceOptions()
        lib().b200_covariance_options_default(C.byref(o))
        o.algorithm = int(algorithm)
        o.min_reciprocal_condition_number = float(min_reciprocal_condition_number)
        o.apply_loss_function = int(bool(apply_loss_function))
        valid = C.c_int()
        _check(lib().b200_covariance_compute(self.h, _d(_f64(state)), C.byref(o), C.byref(valid)))
        return bool(valid.value)

    def covariance_cameras(self, pairs):
        """Cov(c_i, c_j) of each (i, j) in `pairs`: (n, 9, 9), row-major blocks."""
        p = np.ascontiguousarray(np.asarray(pairs, dtype=np.int32).reshape(-1, 2))
        out = np.zeros((len(p), 9, 9))
        _check(lib().b200_covariance_cameras(self.h, len(p), p.ctypes.data_as(_ip), _d(out)))
        return out

    def covariance_points(self):
        """Cov(p, p) of every point: (P, 3, 3)."""
        out = np.zeros((self.P, 3, 3))
        _check(lib().b200_covariance_points(self.h, _d(out)))
        return out

    # ---- trust region loop
    @staticmethod
    def lm_options(**kw):
        o = LmOptions()
        lib().b200_lm_options_default(C.byref(o))
        for k, v in kw.items():
            setattr(o, k, v)
        return o

    def lm_solve(self, state, options=None, host_boundary=False, max_records=256):
        o = options or self.lm_options()
        state = _f64(state).copy()
        trace = (LmIteration * max_records)()
        n = C.c_int()
        _check(lib().b200_lm_solve(self.h, C.byref(o), _d(state), trace, max_records, C.byref(n), int(host_boundary)))
        recs = []
        for i in range(n.value):
            t = trace[i]
            recs.append(dict(iteration=t.iteration, ls_iterations=t.linear_solver_iterations,
                             step_is_valid=t.step_is_valid, step_is_successful=t.step_is_successful, cost=t.cost,
                             cost_change=t.cost_change, gradient_max_norm=t.gradient_max_norm,
                             gradient_norm=t.gradient_norm, step_norm=t.step_norm, tr_ratio=t.relative_decrease,
                             tr_radius=t.trust_region_radius, model_cost_change=t.model_cost_change))
        return state, recs

    # ---- instrumentation
    def profile(self, on):
        _check(lib().b200_profile_enable(self.h, int(on)))

    def stats_reset(self):
        _check(lib().b200_stats_reset(self.h))

    def stats(self):
        arr = (KernelStat * 64)()
        n = C.c_int()
        _check(lib().b200_stats_get(self.h, arr, 64, C.byref(n)))
        return {arr[i].name.decode(): dict(launches=arr[i].launches, operations=arr[i].operations, ms=arr[i].device_ms,
                                           bytes_per_operation=arr[i].bytes_per_operation) for i in range(n.value)}

    def total_launches(self):
        return int(lib().b200_total_launches(self.h))

    def transfer_bytes(self):
        a, b = C.c_int64(), C.c_int64()
        _check(lib().b200_transfer_bytes(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def synchronize(self):
        _check(lib().b200_synchronize(self.h))
