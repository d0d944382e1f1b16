// SURVEY 8f.1: the explicit reduced camera system for an exact (Cholesky) solve -- what DENSE_SCHUR / SPARSE_SCHUR do
// (schur_complement_solver.cc:101-159, SchurEliminator::Eliminate schur_eliminator_impl.h:184-347):
//     S = sum_k [ F_k'F_k - (E_k'F_k)' (E_k'E_k + D_e^2)^-1 (E_k'F_k) ] + D_f^2        (dense, 9C x 9C, FP64)
// assembled on the device from the Jacobian that is already there; the factorisation itself is cuSOLVER's potrf/potrs
// (library code, bound lazily).  Per point with d rows the eliminator makes d^2 rank-3 updates of 9x9 blocks
// (ChunkOuterProduct, :519-568); here one CTA takes a point, stages W_r = E_r'F_r (3x9) and P W_r for 96 rows at a time
// in shared memory and every thread walks the (r, s) pairs of the two staged slices, adding W_r' (P W_s) into the block
// (cam_r, cam_s) of the LOWER triangle (cam_r >= cam_s; column-major for cuSOLVER) with FP64 REDs -- the assembly is bound
// by the device's FP64 RED rate (81 per pair).  The diagonal blocks also receive F_r'F_r.
#pragma once
#include "kernels.cuh"

namespace b200 {

constexpr int kDsRows = 96;      // rows of a point staged per slice (2 x 96 x 27 doubles = 41 KB of static shared memory)
constexpr int kDsThreads = 256;

// A: [n][n] column-major, n = 9C, zeroed by the caller.  ete_inv from schur_init.
__global__ void __launch_bounds__(kDsThreads)
    dense_schur_assemble_kernel(ProblemView p, const double* __restrict__ ete_inv, double* A, size_t lda) {
  __shared__ double sW[kDsRows * 27];    // slice i: W_r   [3][9]
  __shared__ double sPW[kDsRows * 27];   // slice j: P W_s [3][9]
  __shared__ int sCi[kDsRows], sCj[kDsRows];
  const int tid = threadIdx.x;
  for (int k = blockIdx.x; k < p.P; k += gridDim.x) {
    const int r0 = p.pt_ptr[k], r1 = p.pt_ptr[k + 1];
    const double* pi = ete_inv + 6 * static_cast<size_t>(k);
    const double P00 = pi[0], P01 = pi[1], P02 = pi[2], P11 = pi[3], P12 = pi[4], P22 = pi[5];
    for (int i0 = r0; i0 < r1; i0 += kDsRows) {
      const int ni = min(kDsRows, r1 - i0);
      for (int j0 = r0; j0 <= i0; j0 += kDsRows) {
        const int nj = min(kDsRows, r1 - j0);
        __syncthreads();
        // stage W of slice i and P W of slice j (thread t < ni: row i0 + t; thread kDsRows + t < nj: row j0 + t)
        for (int t = tid; t < ni + nj; t += kDsThreads) {
          const bool is_i = t < ni;
          const int r = is_i ? i0 + t : j0 + (t - ni);
          const double2* e = reinterpret_cast<const double2*>(p.E() + 6 * static_cast<size_t>(r));
          const double2 e0 = e[0], e1 = e[1], e2 = e[2];   // E = (e0.x e0.y e1.x ; e1.y e2.x e2.y)
          const double* f = p.F() + 18 * static_cast<size_t>(r);
          double w[27];
#pragma unroll
          for (int b = 0; b < 9; ++b) {
            const double f0 = f[b], f1 = f[9 + b];
            w[b] = e0.x * f0 + e1.y * f1;
            w[9 + b] = e0.y * f0 + e2.x * f1;
            w[18 + b] = e1.x * f0 + e2.y * f1;
          }
          if (is_i) {
            double* dst = sW + t * 27;
#pragma unroll
            for (int q = 0; q < 27; ++q) dst[q] = w[q];
            sCi[t] = p.cam_idx[r];
          } else {
            double* dst = sPW + (t - ni) * 27;
#pragma unroll
            for (int b = 0; b < 9; ++b) {
              dst[b] = P00 * w[b] + P01 * w[9 + b] + P02 * w[18 + b];
              dst[9 + b] = P01 * w[b] + P11 * w[9 + b] + P12 * w[18 + b];
              dst[18 + b] = P02 * w[b] + P12 * w[9 + b] + P22 * w[18 + b];
            }
            sCj[t - ni] = p.cam_idx[r];
          }
        }
        __syncthreads();
        // all (r in slice i, s in slice j) pairs; within the diagonal slice pair only s <= r (the mirror image of s > r
        // is produced when the roles are swapped, see below)
        const int pairs = ni * nj;
        for (int q = tid; q < pairs; q += kDsThreads) {
          const int a = q / nj, b = q - a * nj;
          if (i0 == j0 && b > a) continue;
          const double* wi = sW + a * 27;
          const double* pw = sPW + b * 27;
          int ci = sCi[a], cj = sCj[b];
          // block(ci, cj) -= W_a' (P W_b); stored where row-camera >= column-camera.  When ci < cj the transposed block
          // goes to (cj, ci): (W_a' P W_b)' = W_b' P W_a.
          const bool swap = ci < cj;
          if (swap) {
            const int t = ci;
            ci = cj;
            cj = t;
          }
          double* base = A + (9 * static_cast<size_t>(ci)) + (9 * static_cast<size_t>(cj)) * lda;
          const bool same_row = (i0 == j0 && a == b);
          const double* f = same_row ? p.F() + 18 * static_cast<size_t>(i0 + a) : nullptr;
#pragma unroll 3
          for (int u = 0; u < 9; ++u) {
#pragma unroll
            for (int v = 0; v < 9; ++v) {
              // entry (u, v) of W_a' P W_b
              double val = wi[u] * pw[v] + wi[9 + u] * pw[9 + v] + wi[18 + u] * pw[18 + v];
              val = -val;
              if (same_row) val += f[u] * f[v] + f[9 + u] * f[9 + v];   // + F_r'F_r on the diagonal block
              // destination inside the stored block: (u, v) normally, (v, u) when transposed
              const int rr = swap ? v : u, cc = swap ? u : v;
              red_add(base + rr + static_cast<size_t>(cc) * lda, val);
              // a pair of distinct rows that see the SAME camera contributes the block and its transpose to the diagonal block
              if (!same_row && ci == cj && !(i0 == j0 && a == b)) red_add(base + cc + static_cast<size_t>(rr) * lda, val);
            }
          }
        }
      }
    }
  }
}

// A[j][j] += D_f[j]^2
__global__ void __launch_bounds__(256) dense_schur_diagonal_kernel(int n, const double* __restrict__ Df, double* A, size_t lda) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n && Df != nullptr) A[j + static_cast<size_t>(j) * lda] += Df[j] * Df[j];
}

// Iterative refinement of the exact solves (RefinedSparseCholesky::Solve sparse_cholesky.cc:160-170, RefinedDenseCholesky::
// Solve dense_cholesky.cc:337-349): x_f = solve(rhs_S), then k times r = rhs_S - (S + D_f^2) x_f in FP64 and x_f += solve(r).
// A solve's vector v is indexed by position pos(k) = 9 pinv[k / 9] + k % 9 (the sparse factor's elimination order) or, with
// pinv == NULL, by k itself (the dense factor).

// v[pos(k)] <- rhs[k] - Sx[k] (Sx may be NULL), rounded to T once.
template <typename T>
__global__ void __launch_bounds__(256) refine_residual_kernel(int n, const int* __restrict__ pinv, const double* __restrict__ rhs,
                                                             const double* __restrict__ Sx, T* __restrict__ v) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x)
    v[pinv != nullptr ? 9 * pinv[k / 9] + k % 9 : k] = static_cast<T>(Sx != nullptr ? rhs[k] - Sx[k] : rhs[k]);
}

// x[k] <- (add ? x[k] : 0) + v[pos(k)] widened to double.
template <typename T>
__global__ void __launch_bounds__(256) refine_accumulate_kernel(int n, const int* __restrict__ pinv, const T* __restrict__ v,
                                                               double* __restrict__ x, int add) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    const double d = static_cast<double>(v[pinv != nullptr ? 9 * pinv[k / 9] + k % 9 : k]);
    x[k] = add ? x[k] + d : d;
  }
}

// The lower triangle of the assembled A [n][n] (column-major), rounded to float for a single-precision potrf
// (CUDADenseCholeskyMixedPrecision::Factorize, dense_cholesky.cc:562-578).  The upper triangle of Af is not written.
__global__ void __launch_bounds__(256) dense_round_lower_kernel(int n, const double* __restrict__ A, float* __restrict__ Af) {
  const size_t total = static_cast<size_t>(n) * n;
  for (size_t e = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; e < total; e += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t j = e / n, i = e - j * n;
    if (i >= j) Af[e] = static_cast<float>(A[e]);
  }
}

}  // namespace b200
