// Camera-sized (9C) PCG vector kernels and parameter-sized (3P+9C) LM vector kernels.
//
// The PCG of the reference (conjugate_gradients_solver.h:109-306) runs ~12 tiny Eigen expressions and
// 3 dot products per iteration, each a host round trip in its CUDA variant (cuda_vector.cc:97-181).  Here one
// cooperative kernel per iteration (cg_kernel.cuh) carries all of it, with every scalar (rho, alpha, beta, Q, |r|,
// iteration count, termination code) living in a device-side CgState so that the host never synchronises inside the
// iteration: kernels exit immediately once `done` is set.  This header holds the state, the small helpers and the
// parameter-sized LM vector kernels.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int kVecThreads = 1024;

struct CgState {
  double rho, last_rho, Q0, norm_rhs, tol_r, norm_r, alpha, pq, beta;
  int iteration;    // summary.num_iterations
  int done;         // 1 once a termination criterion fired
  int termination;  // B200_LS_*
  int reason;       // 1 zeta, 2 |r|, 3 max iterations, 4 rho, 5 beta, 6 pq, 7 alpha, 8 |b| = 0
};

struct CgParams {
  int n;            // 9C
  int min_iterations, max_iterations;
  double q_tolerance, r_tolerance;
};

__device__ __forceinline__ bool zero_or_inf(double x) { return x == 0.0 || isinf(x); }

// y[i] = d[i]^2 * x[i]  (or 0 when d == nullptr)
__global__ void __launch_bounds__(256) diag_sq_mul_kernel(int n, const double* __restrict__ d,
                                                          const double* __restrict__ x, double* y,
                                                          const int* __restrict__ done_flag) {
  if (done_flag != nullptr && *done_flag != 0) return;
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    y[i] = d != nullptr ? d[i] * d[i] * x[i] : 0.0;
}

__global__ void flag_to_double_kernel(const int* flag, double* out) { out[0] = flag[0] != 0 ? 1.0 : 0.0; }
__global__ void double_to_flag_kernel(const double* in, int* flag) { flag[0] = in[0] != 0.0 ? 1 : 0; }

__global__ void __launch_bounds__(256) fill_kernel(size_t n, double* y, double v) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) y[i] = v;
}

// The per-component state of a handle's constant components (b200_handle::d_fixed / h_fixed): 0 = free, kComponentMasked =
// a coordinate held by a SubsetManifold on a variable block, kComponentConstant = a component of a constant block (a full
// SubsetManifold included: ParameterBlock::IsConstant).  Whatever only needs "zero column, D' = 1, x kept bitwise" tests
// != 0; |x| for parameter_tolerance leaves out kComponentConstant only (Ceres' reduced x holds masked coordinates).
constexpr uint8_t kComponentMasked = 1, kComponentConstant = 2;

// D' of the solves on a handle with constant components: 1 there, D (0 when null) elsewhere.  Their E'E + D'^2 and S
// entries are then identities decoupled from the rest, and the solves return exact zeros there.
__global__ void __launch_bounds__(256) solve_diagonal_kernel(int n, const double* __restrict__ D, const uint8_t* __restrict__ fixed,
                                                             double* out) {
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = fixed[i] != 0 ? 1.0 : D != nullptr ? D[i] : 0.0;
}

// ---------------------------------------------------------------- LM vector kernels (n = 3P+9C)
// scale = 1 / (1 + sqrt(colnorm^2))     trust_region_minimizer.cc:263-274
__global__ void __launch_bounds__(256) jacobi_scale_kernel(int n, const double* __restrict__ sqnorm, double* scale) {
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) scale[i] = 1.0 / (1.0 + sqrt(sqnorm[i]));
}
// sq <- sq * scale^2 : squared column norms after J <- J diag(scale)
__global__ void __launch_bounds__(256) rescale_sq_kernel(int n, const double* __restrict__ scale, double* sq) {
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) sq[i] *= scale[i] * scale[i];
}
// diagonal = clamp(colnorm^2, min, max) (if refresh) ; D = sqrt(diagonal / radius)   levenberg_marquardt_strategy.cc:79-95
__global__ void __launch_bounds__(256) lm_diagonal_kernel(int n, int refresh, const double* __restrict__ sqnorm,
                                                          double* diagonal, double* D, double min_d, double max_d,
                                                          double radius) {
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double v = diagonal[i];
    if (refresh) {
      v = fmin(fmax(sqnorm[i], min_d), max_d);
      diagonal[i] = v;
    }
    D[i] = sqrt(v / radius);
  }
}

// Generic two-stage deterministic reductions: partial[blockIdx.x*kSlots + s], then reduce_final_kernel.
constexpr int kRedBlocks = 296;
// step = -y ; delta = step*scale ; cand = x + delta ; partials: {|delta|^2, |x|^2, nonfinite count}
// fixed: null, or the component states (kComponentMasked, kComponentConstant): cand = x on every constant component, and
// |x|^2 is taken over Ceres' reduced x (trust_region_minimizer.cc:725-742), which holds the variable blocks' coordinates,
// masked ones included, and no constant block.
__global__ void __launch_bounds__(256)
    lm_step_kernel(int n, const double* __restrict__ y, const double* __restrict__ scale, const double* __restrict__ x,
                   const uint8_t* __restrict__ fixed, double* step, double* cand, double* partial) {
  __shared__ double scratch[32];
  double a = 0.0, b = 0.0, c = 0.0;
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const double yi = y[i];
    const double si = -yi;
    step[i] = si;
    const double di = si * scale[i];
    const double xi = x[i];
    const uint8_t fx = fixed != nullptr ? fixed[i] : 0;
    const double ci = fx != 0 ? xi : xi + di;
    cand[i] = ci;
    const double dd = xi - ci;
    a += dd * dd;
    if (fx != kComponentConstant) b += xi * xi;
    if (!isfinite(yi)) c += 1.0;
  }
  a = block_sum<256>(a, scratch);
  b = block_sum<256>(b, scratch);
  c = block_sum<256>(c, scratch);
  if (threadIdx.x == 0) {
    partial[blockIdx.x * 3 + 0] = a;
    partial[blockIdx.x * 3 + 1] = b;
    partial[blockIdx.x * 3 + 2] = c;
  }
}
// partials: {max |g|, |g|^2}   (gradient norms: trust_region_minimizer.cc:290-302 with Euclidean Plus)
__global__ void __launch_bounds__(256) grad_norm_kernel(int n, const double* __restrict__ g, double* partial) {
  __shared__ double scratch[32];
  double mx = 0.0, sq = 0.0;
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const double v = g[i];
    mx = fmax(mx, fabs(v));
    sq += v * v;
  }
  sq = block_sum<256>(sq, scratch);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    double m = 0.0;
    for (int w = 0; w < 8; ++w) m = fmax(m, scratch[w]);
    partial[blockIdx.x * 2 + 0] = m;
    partial[blockIdx.x * 2 + 1] = sq;
  }
}
// ---------------------------------------------------------------- DOGLEG vector kernels (dogleg_strategy.cc)
// refresh: diagonal = sqrt(clamp(colnorm^2, min, max)) (:123-128) and g = scale * gradient / diagonal.  The reference
// forms g as J_s' r / diagonal (:176-181) with J_s the scaled Jacobian; J_s' r = scale * (J' r) up to rounding, and J' r
// is the gradient the evaluate already wrote, so no pass over J is needed.  Always: D = diagonal * sqrt(mu) (:561).
__global__ void __launch_bounds__(256) dogleg_diagonal_kernel(int n, int refresh, const double* __restrict__ sqnorm,
                                                              const double* __restrict__ gradient,
                                                              const double* __restrict__ scale, double* diagonal,
                                                              double* g, double* D, double min_d, double max_d,
                                                              double sqrt_mu) {
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double d = diagonal[i];
    if (refresh) {
      d = sqrt(fmin(fmax(sqnorm[i], min_d), max_d));
      diagonal[i] = d;
      g[i] = __dmul_rn(scale[i], gradient[i]) / d;
    }
    D[i] = __dmul_rn(d, sqrt_mu);
  }
}
// After a solve J'J + D^2 y = J'r: gn = -diagonal * y (:612); partials {|g|^2, g.gn, |gn|^2, non-finite y count} (:594).
__global__ void __launch_bounds__(256) dogleg_gn_kernel(int n, const double* __restrict__ y,
                                                        const double* __restrict__ diagonal,
                                                        const double* __restrict__ g, double* gn, double* partial) {
  __shared__ double scratch[32];
  double a = 0.0, b = 0.0, c = 0.0, bad = 0.0;
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const double yi = y[i];
    const double v = __dmul_rn(yi, -diagonal[i]);
    gn[i] = v;
    const double gi = g[i];
    a = __fma_rn(gi, gi, a);
    b = __fma_rn(gi, v, b);
    c = __fma_rn(v, v, c);
    if (!isfinite(yi)) bad += 1.0;
  }
  a = block_sum<256>(a, scratch);
  b = block_sum<256>(b, scratch);
  c = block_sum<256>(c, scratch);
  bad = block_sum<256>(bad, scratch);
  if (threadIdx.x == 0) {
    partial[blockIdx.x * 4 + 0] = a;
    partial[blockIdx.x * 4 + 1] = b;
    partial[blockIdx.x * 4 + 2] = c;
    partial[blockIdx.x * 4 + 3] = bad;
  }
}
// The dogleg step (dogleg.h StepKind): v = gn (kind 0), cg g (kind 1) or cg g + cn gn (kind 2), selected rather than
// multiplied by 0; step = v / diagonal; delta = step * scale; cand = x + delta.
// Partials {|x - cand|^2, |x|^2, non-finite step count, |v|^2 (dogleg_step_norm_ of the interpolation, :251)}.
// fixed: as in lm_step_kernel.
__global__ void __launch_bounds__(256)
    dogleg_step_kernel(int n, int kind, double cg, double cn, const double* __restrict__ g, const double* __restrict__ gn,
                       const double* __restrict__ diagonal, const double* __restrict__ scale,
                       const double* __restrict__ x, const uint8_t* __restrict__ fixed, double* step, double* cand,
                       double* partial) {
  __shared__ double scratch[32];
  double a = 0.0, b = 0.0, c = 0.0, e = 0.0;
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double v;
    if (kind == 0) v = gn[i];
    else if (kind == 1) v = __dmul_rn(cg, g[i]);
    else v = __dadd_rn(__dmul_rn(cg, g[i]), __dmul_rn(cn, gn[i]));
    const double si = v / diagonal[i];
    step[i] = si;
    const double xi = x[i];
    const uint8_t fx = fixed != nullptr ? fixed[i] : 0;
    const double ci = fx != 0 ? xi : __dadd_rn(xi, __dmul_rn(si, scale[i]));
    cand[i] = ci;
    const double dd = xi - ci;
    a = __fma_rn(dd, dd, a);
    if (fx != kComponentConstant) b = __fma_rn(xi, xi, b);
    if (!isfinite(si)) c += 1.0;
    e = __fma_rn(v, v, e);
  }
  a = block_sum<256>(a, scratch);
  b = block_sum<256>(b, scratch);
  c = block_sum<256>(c, scratch);
  e = block_sum<256>(e, scratch);
  if (threadIdx.x == 0) {
    partial[blockIdx.x * 4 + 0] = a;
    partial[blockIdx.x * 4 + 1] = b;
    partial[blockIdx.x * 4 + 2] = c;
    partial[blockIdx.x * 4 + 3] = e;
  }
}

// out[s] = reduce over blocks of partial[b*slots + s]; op_mask bit s set => max, else sum.
__global__ void __launch_bounds__(32) reduce_final_kernel(int blocks, int slots, unsigned op_mask,
                                                          const double* __restrict__ partial, double* out) {
  const int s = threadIdx.x;
  if (s >= slots) return;
  double acc = 0.0;
  const bool is_max = (op_mask >> s) & 1u;
  for (int b = 0; b < blocks; ++b) {
    const double v = partial[b * slots + s];
    acc = is_max ? fmax(acc, v) : acc + v;
  }
  out[s] = acc;
}
// out[0] = sum_t partial[t]   (per-tile cost partials, model cost partials): single CTA, fixed order
__global__ void __launch_bounds__(kVecThreads) sum_kernel(int n, const double* __restrict__ partial, double* out) {
  __shared__ double scratch[32];
  double acc = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) acc += partial[i];
  acc = block_sum<kVecThreads>(acc, scratch);
  if (threadIdx.x == 0) out[0] = acc;
}

// Boundary permutations between the caller's block order and the library's internal one (blocks of `w` doubles):
//   gather :  dst[i] = src[perm[i]]        (caller -> internal, perm[i] = caller index of internal block i)
//   scatter:  dst[perm[i]] = src[i]        (internal -> caller)
__global__ void __launch_bounds__(256) permute_gather_kernel(size_t n, int w, const int* __restrict__ perm,
                                                             const double* __restrict__ src, double* __restrict__ dst) {
  const size_t total = n * w, stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t b = i / w, j = i - b * w;
    dst[i] = src[static_cast<size_t>(perm[b]) * w + j];
  }
}
__global__ void __launch_bounds__(256) permute_scatter_kernel(size_t n, int w, const int* __restrict__ perm,
                                                              const double* __restrict__ src, double* __restrict__ dst) {
  const size_t total = n * w, stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
    const size_t b = i / w, j = i - b * w;
    dst[static_cast<size_t>(perm[b]) * w + j] = src[i];
  }
}

}  // namespace b200
