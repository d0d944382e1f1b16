"""ceres_solver_b200 — H100-native (sm_90a) implementation of Ceres Solver's Levenberg-Marquardt inner-loop
hot path for bundle adjustment: CUDA kernels + C ABI in csrc/ (libb200ba.so), ctypes plumbing in binding.py,
host-side problem preparation in bal.py.  No CPU fallback: using the compute path without the built library
or without a GPU raises."""
from . import bal  # noqa: F401
from .binding import (B200Error, Problem, lib, nccl_unique_id, plan_point_order, plan_sparse_schur, LIB_PATH, SYMBOLS,  # noqa: F401
                      PRECOND_IDENTITY, PRECOND_JACOBI, PRECOND_SCHUR_JACOBI, PRECOND_SCHUR_POWER_SERIES_EXPANSION, ITERATIVE_SCHUR, DENSE_SCHUR,
                      SPARSE_SCHUR, SPARSE_STATS, LEVENBERG_MARQUARDT, DOGLEG, TRADITIONAL_DOGLEG, SUBSPACE_DOGLEG, AMD, NESDIS, LOSS_TRIVIAL, LOSS_HUBER,
                      LOSS_SOFT_L_ONE, LOSS_CAUCHY, LOSS_ARCTAN, LOSS_TOLERANT, LOSS_TUKEY, Loss, CovarianceOptions, plan_sparse_selinv,
                      subset_manifold_masks,
                      LS_SUCCESS, LS_NO_CONVERGENCE, LS_FAILURE, LS_FATAL_ERROR)
