"""ctypes binding of the CPU oracle (oracle/libceres_oracle.so).

ORACLE — TEST INFRASTRUCTURE ONLY.  Importable from tests/, __graft_entry__.smoke() and
bench.py's cpu_baseline / --impl reference legs; never from the product package.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "libceres_oracle.so")

_dp = C.POINTER(C.c_double)
_ip = C.POINTER(C.c_int)


def build(force=False):
    """Compile the oracle with g++ (seconds)."""
    srcs = ["capi.cc", "block_ops.h", "parallel.h", "block_sparse.h", "schur.h", "bal.h"]
    if not force and os.path.exists(_LIB_PATH):
        newest = max(os.path.getmtime(os.path.join(_HERE, s)) for s in srcs)
        if os.path.getmtime(_LIB_PATH) >= newest:
            return _LIB_PATH
    subprocess.check_call(["make", "-C", _HERE, "-B", "libceres_oracle.so"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB_PATH):
            build()
        _lib = C.CDLL(_LIB_PATH)
        _lib.orc_bsm_create.restype = C.c_void_p
        _lib.orc_isc_create.restype = C.c_void_p
        _lib.orc_bal_read.restype = C.c_void_p
        _lib.orc_bal_from_arrays.restype = C.c_void_p
        _lib.orc_ba_create.restype = C.c_void_p
        _lib.orc_ba_jacobian.restype = C.c_void_p
        _lib.orc_bsm_num_nonzeros.restype = C.c_long
    return _lib


def _d(a):
    return None if a is None else a.ctypes.data_as(_dp)


def _i(a):
    return None if a is None else a.ctypes.data_as(_ip)


def _f64(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64)


def _i32(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.int32)


def max_threads():
    return int(lib().orc_max_threads())


class BlockSparseMatrix:
    """Generic block sparse matrix: col_sizes, row_sizes, rows = list of (block ids), values in cell order."""

    def __init__(self, col_sizes=None, row_sizes=None, row_cells=None, values=None, handle=None):
        self._owned = handle is None
        if handle is None:
            col_sizes = _i32(col_sizes)
            row_sizes = _i32(row_sizes)
            ptr = np.zeros(len(row_cells) + 1, dtype=np.int32)
            ids = []
            for r, cells in enumerate(row_cells):
                ids.extend(cells)
                ptr[r + 1] = len(ids)
            ids = _i32(ids)
            values = _f64(values)
            handle = lib().orc_bsm_create(len(col_sizes), _i(col_sizes), len(row_sizes), _i(row_sizes), _i(ptr),
                                          _i(ids), _d(values))
        self.h = C.c_void_p(handle)
        self.num_rows = lib().orc_bsm_num_rows(self.h)
        self.num_cols = lib().orc_bsm_num_cols(self.h)
        self.nnz = lib().orc_bsm_num_nonzeros(self.h)

    def __del__(self):
        if getattr(self, "_owned", False) and lib is not None:
            try:
                lib().orc_bsm_free(self.h)
            except Exception:
                pass

    def values(self):
        out = np.empty(self.nnz)
        lib().orc_bsm_get_values(self.h, _d(out))
        return out

    def set_values(self, v):
        v = _f64(v)
        assert v.size == self.nnz
        lib().orc_bsm_set_values(self.h, _d(v))

    def right_multiply(self, x, nt=1):
        x = _f64(x)
        y = np.zeros(self.num_rows)
        lib().orc_bsm_right_multiply(self.h, _d(x), _d(y), nt)
        return y

    def left_multiply(self, x, nt=1):
        x = _f64(x)
        y = np.zeros(self.num_cols)
        lib().orc_bsm_left_multiply(self.h, _d(x), _d(y), nt)
        return y

    def squared_column_norm(self, nt=1):
        out = np.empty(self.num_cols)
        lib().orc_bsm_squared_column_norm(self.h, _d(out), nt)
        return out

    def scale_columns(self, s, nt=1):
        s = _f64(s)
        lib().orc_bsm_scale_columns(self.h, _d(s), nt)

    # ---- partitioned view
    def pmv(self, num_elim, op, x, out_len, nt=1, force_dynamic=0):
        x = _f64(x)
        y = np.zeros(out_len)
        lib().orc_pmv_multiply(self.h, num_elim, op, _d(x), _d(y), nt, force_dynamic)
        return y

    def block_diagonal(self, num_elim, which, nt=1, force_dynamic=0):
        n = lib().orc_pmv_block_diagonal(self.h, num_elim, which, None, nt, force_dynamic)
        out = np.zeros(n)
        lib().orc_pmv_block_diagonal(self.h, num_elim, which, _d(out), nt, force_dynamic)
        return out

    # ---- Schur eliminator
    def schur_eliminate(self, num_elim, b, D, diagonal_only=False, full_rank=True, nt=1, force_dynamic=0,
                        n_f=None, diag_len=None):
        b = _f64(b)
        D = _f64(D)
        if n_f is None:
            n_f = lib().orc_schur_eliminate(self.h, num_elim, None, None, 1, 1, None, None, 1, force_dynamic)
        if diagonal_only:
            assert diag_len is not None
            lhs = np.zeros(diag_len)
        else:
            lhs = np.zeros((n_f, n_f))
        rhs = np.zeros(n_f) if b is not None else None
        lib().orc_schur_eliminate(self.h, num_elim, _d(b), _d(D), int(diagonal_only), int(full_rank), _d(lhs),
                                  _d(rhs), nt, force_dynamic)
        return lhs, rhs

    def schur_back_substitute(self, num_elim, b, D, z, full_rank=True, nt=1, force_dynamic=0):
        y = np.zeros(self.num_cols)
        lib().orc_schur_back_substitute(self.h, num_elim, _d(_f64(b)), _d(_f64(D)), _d(_f64(z)), int(full_rank),
                                        _d(y), nt, force_dynamic)
        return y

    def linear_solve(self, num_elim, b, D, solver=0, preconditioner=2, min_iter=0, max_iter=500, reset_period=10,
                     q_tolerance=0.0, r_tolerance=0.0, nt=1, force_dynamic=0, max_num_spse_iterations=5,
                     use_spse_initialization=False, spse_tolerance=0.1):
        x = np.zeros(self.num_cols)
        summ = np.zeros(2, dtype=np.int32)
        lib().orc_linear_solve_spse(self.h, num_elim, solver, preconditioner, min_iter, max_iter, reset_period,
                                    C.c_double(q_tolerance), C.c_double(r_tolerance), _d(_f64(b)), _d(_f64(D)), _d(x),
                                    _i(summ), nt, force_dynamic, int(max_num_spse_iterations),
                                    int(bool(use_spse_initialization)), C.c_double(spse_tolerance))
        return x, int(summ[0]), int(summ[1])


def cg_dense(A, b, x0, min_iter=0, max_iter=500, reset_period=10, q_tolerance=0.0, r_tolerance=0.0):
    """The oracle's ConjugateGradientsSolver on a dense symmetric matrix with the identity preconditioner."""
    A = _f64(A)
    x = _f64(x0).copy()
    summ = np.zeros(2, dtype=np.int32)
    lib().orc_cg_dense(A.shape[0], _d(A), _d(_f64(b)), _d(x), min_iter, max_iter, reset_period, C.c_double(q_tolerance),
                       C.c_double(r_tolerance), _i(summ))
    return x, int(summ[0]), int(summ[1])


def angle_axis_rotate_point(angle_axis, pt):
    out = np.zeros(3)
    lib().orc_angle_axis_rotate_point(_d(_f64(angle_axis)), _d(_f64(pt)), _d(out))
    return out


def huber_loss(a, s):
    rho = np.zeros(3)
    lib().orc_huber_loss(C.c_double(a), C.c_double(s), _d(rho))
    return rho


def corrector(sq_norm, rho, residuals, jacobian=None):
    """Corrector(sq_norm, rho).CorrectJacobian + CorrectResiduals; returns the corrected copies."""
    r = _f64(residuals).copy()
    J = None if jacobian is None else _f64(jacobian).copy()
    rows = r.size
    cols = 0 if J is None else J.size // rows
    lib().orc_corrector(C.c_double(sq_norm), _d(_f64(rho)), rows, cols, _d(r), _d(J))
    return r, J


class ImplicitSchur:
    def __init__(self, A, num_elim, want_ftf=False, nt=1, force_dynamic=0):
        self.A = A
        self.h = C.c_void_p(lib().orc_isc_create(A.h, num_elim, int(want_ftf), nt, force_dynamic))
        self.n = lib().orc_isc_num_rows(self.h)

    def __del__(self):
        try:
            lib().orc_isc_free(self.h)
        except Exception:
            pass

    def init(self, D, b):
        self._D = _f64(D)
        self._b = _f64(b)  # keep alive: the oracle stores the pointers, like the reference
        lib().orc_isc_init(self.h, _d(self._D), _d(self._b))

    def right_multiply(self, x):
        y = np.zeros(self.n)
        lib().orc_isc_right_multiply(self.h, _d(_f64(x)), _d(y))
        return y

    def rhs(self):
        out = np.zeros(self.n)
        lib().orc_isc_rhs(self.h, _d(out))
        return out

    def back_substitute(self, x):
        y = np.zeros(self.A.num_cols)
        lib().orc_isc_back_substitute(self.h, _d(_f64(x)), _d(y))
        return y

    def power_series(self, x, max_num_spse_iterations=5, spse_tolerance=0.0):
        """PowerSeriesExpansionPreconditioner::RightMultiplyAndAccumulate on a zeroed y (needs want_ftf=True)."""
        y = np.zeros(self.n)
        lib().orc_isc_power_series(self.h, int(max_num_spse_iterations), C.c_double(spse_tolerance), _d(_f64(x)), _d(y))
        return y

    def ete_inverse(self):
        n = lib().orc_isc_ete_inverse(self.h, None)
        out = np.zeros(n)
        lib().orc_isc_ete_inverse(self.h, _d(out))
        return out


class BalProblem:
    """BAL text file (examples/bal_problem.cc) as arrays."""

    def __init__(self, path=None, arrays=None):
        if path is not None:
            h = lib().orc_bal_read(path.encode())
            if not h:
                raise IOError("cannot read BAL file %s" % path)
        else:
            cam_idx, pt_idx, obs, cameras, points = arrays
            cam_idx, pt_idx = _i32(cam_idx), _i32(pt_idx)
            obs, cameras, points = _f64(obs), _f64(cameras), _f64(points)
            h = lib().orc_bal_from_arrays(len(cameras) // 9 if cameras.ndim == 1 else cameras.shape[0],
                                          len(points) // 3 if points.ndim == 1 else points.shape[0], len(cam_idx),
                                          _i(cam_idx), _i(pt_idx), _d(obs), _d(cameras), _d(points))
        self.h = C.c_void_p(h)
        self._refresh()

    def _refresh(self):
        dims = np.zeros(3, dtype=np.int32)
        lib().orc_bal_dims(self.h, _i(dims))
        self.C, self.P, self.N = (int(v) for v in dims)
        self.cam_idx = np.zeros(self.N, dtype=np.int32)
        self.pt_idx = np.zeros(self.N, dtype=np.int32)
        self.obs = np.zeros(2 * self.N)
        self.cameras = np.zeros(9 * self.C)
        self.points = np.zeros(3 * self.P)
        lib().orc_bal_get(self.h, _i(self.cam_idx), _i(self.pt_idx), _d(self.obs), _d(self.cameras), _d(self.points))

    def normalize(self):
        lib().orc_bal_normalize(self.h)
        self._refresh()

    def __del__(self):
        try:
            lib().orc_bal_free(self.h)
        except Exception:
            pass


class SolveOptions(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("linear_solver", "preconditioner", "max_num_iterations",
                                       "max_linear_solver_iterations", "min_linear_solver_iterations",
                                       "jacobi_scaling", "num_threads", "use_spse_initialization",
                                       "max_num_consecutive_invalid_steps")] + \
               [(n, C.c_double) for n in ("eta", "initial_trust_region_radius", "max_trust_region_radius",
                                          "min_trust_region_radius", "min_relative_decrease", "min_lm_diagonal",
                                          "max_lm_diagonal", "function_tolerance", "gradient_tolerance",
                                          "parameter_tolerance")]


TRACE_FIELDS = ("iteration", "cost", "cost_change", "gradient_max_norm", "gradient_norm", "step_norm",
                "tr_ratio", "tr_radius", "ls_iterations", "step_is_valid", "step_is_successful",
                "model_cost_change")


class BaProgram:
    """Reduced program of a BAL-shaped problem in the reference's own ordering + evaluator + LM solve."""

    def __init__(self, C_, P_, cam_idx, pt_idx, obs, use_huber=False, huber_a=1.0):
        cam_idx, pt_idx, obs = _i32(cam_idx), _i32(pt_idx), _f64(obs)
        self.h = C.c_void_p(lib().orc_ba_create(C_, P_, len(cam_idx), _i(cam_idx), _i(pt_idx), _d(obs),
                                                int(use_huber), C.c_double(huber_a)))
        dims = np.zeros(3, dtype=np.int32)
        lib().orc_ba_dims(self.h, _i(dims))
        self.C, self.P, self.N = (int(v) for v in dims)
        self.point_of_eblock = np.zeros(self.P, dtype=np.int32)
        self.camera_of_fblock = np.zeros(self.C, dtype=np.int32)
        self.obs_of_row = np.zeros(self.N, dtype=np.int32)
        self.row_pt = np.zeros(self.N, dtype=np.int32)
        self.row_cam = np.zeros(self.N, dtype=np.int32)
        self.row_obs = np.zeros(2 * self.N)
        lib().orc_ba_order(self.h, _i(self.point_of_eblock), _i(self.camera_of_fblock), _i(self.obs_of_row),
                           _i(self.row_pt), _i(self.row_cam), _d(self.row_obs))
        self.num_parameters = 3 * self.P + 9 * self.C
        self.num_residuals = 2 * self.N

    def __del__(self):
        try:
            lib().orc_ba_free(self.h)
        except Exception:
            pass

    def state_from_parameters(self, cameras, points):
        state = np.zeros(self.num_parameters)
        lib().orc_ba_state_from_parameters(self.h, _d(_f64(cameras)), _d(_f64(points)), _d(state))
        return state

    def evaluate(self, state, want_residuals=True, want_gradient=True, want_jacobian=True, nt=1):
        state = _f64(state)
        cost = C.c_double(0.0)
        res = np.zeros(self.num_residuals) if want_residuals else None
        grad = np.zeros(self.num_parameters) if want_gradient else None
        ok = lib().orc_ba_evaluate(self.h, _d(state), C.byref(cost), _d(res), _d(grad), int(want_jacobian), nt)
        return bool(ok), cost.value, res, grad

    def jacobian(self):
        return BlockSparseMatrix(handle=lib().orc_ba_jacobian(self.h))

    @staticmethod
    def default_options():
        o = SolveOptions()
        lib().orc_solve_options_default(C.byref(o))
        return o

    def solve(self, state, options=None, max_records=256):
        o = options or self.default_options()
        state = _f64(state).copy()
        trace = np.zeros((max_records, 12))
        times = np.zeros(7)
        n = lib().orc_ba_solve(self.h, C.byref(o), _d(state), _d(trace), max_records, _d(times))
        if n < 0:
            raise RuntimeError("oracle solve failed")
        recs = [dict(zip(TRACE_FIELDS, row)) for row in trace[:n]]
        tdict = dict(residual_eval=times[0], jacobian_eval=times[1], linear_solver=times[2], total=times[3],
                     num_residual_evals=int(times[4]), num_jacobian_evals=int(times[5]),
                     num_linear_solves=int(times[6]))
        return state, recs, tdict
