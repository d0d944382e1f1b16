// Covariance of the cameras and the points on the device (ceres::Covariance, covariance.h; CovarianceImpl,
// covariance_impl.cc), in the Schur form.  With D = 0 on the variable components (D' = 1 on the constant ones, DESIGN §3.8),
// V_p = E_p'E_p, W_p = E_p'F_p and Z = S^-1:
//     Cov(cameras) = Z,     Cov(p, p) = V_p^-1 + V_p^-1 (sum over rows r, s of p of W_r Z_{c_r c_s} W_s') V_p^-1.
// Every camera pair (c_r, c_s) of that sum shares point p, so every block of Z a point reads lies in the block pattern of S,
// and so in the pattern of the supernodal factor L.  The selected inverse (Takahashi's recurrence) computes Z on exactly
// L's pattern, never a dense S^-1.
//
// sparse_selinv_kernel: one persistent cooperative launch over the factor of sparse_schur.cuh, writing Z into a second
// buffer with L's panel layout.  Per supernode s with panel [L_ss; L_Rs] (R: its rows below):
//     U = L_Rs L_ss^-1,   Z_Rs = -Z_RR U,   Z_ss = L_ss^-T L_ss^-1 - U' Z_Rs.
// U overwrites L_Rs in place (no other task reads s's factor panel; the factor is rebuilt by the next solve).  Z_ss is
// written as a full symmetric block (both triangles from the lower one), so every block of Z can be read either way round.
// Z_RR is read from the panels of the supernodes that own R's columns: entry (a, b) of R x R, positions a >= b, lies in the
// panel of the supernode t owning b, in its row of a (the structure of a supernode's rows below contains that of every
// column it updates: sparse_plan.cuh).
//
// Tasks: ns tickets taken in order from a global counter.  Ticket t is supernode s = order[ns - 1 - t]: the reverse of the
// factor's topological order, ancestors first.  Task s waits until every supernode owning one of its rows below is done:
// its counter starts at that count (SparsePlan::cnt_inv; 0 for a root) and each such supernode, when done, decrements the
// counter of every descendant in its update list, as sparse_factor_kernel's backward tasks do.  Those supernodes are
// ancestors of s, which come after s in `order` and so before it in the tickets: every task waits only on tasks with
// smaller tickets, which have all been taken by CTAs that are running (the launch is cooperative: every CTA is resident),
// so the walk cannot deadlock.  Each Z entry is written once, by the CTA that owns its supernode, in a fixed order: no
// atomics on values, and the result is bitwise reproducible.  A task's writes are fenced before it releases its
// dependants, and other supernodes' panels are read with ld.global.cg.
#pragma once
#include "sparse_schur.cuh"

namespace b200 {

// Dynamic shared memory of sparse_selinv_kernel for supernodes of at most W scalar columns: the GEMM stages, then
// L_ss^-1 [W][W].
inline size_t selinv_smem_bytes(int W) {
  return sizeof(double) * (kSpK * (kSpMaxCols + kSpTileRows) + static_cast<size_t>(W) * W);
}

// The supernode owning position p (binary search on sn_first).
__device__ __forceinline__ int sn_of_position(const SparseView<double>& sv, int p) {
  int lo = 0, hi = sv.ns - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (sv.sn_first[mid] <= p) lo = mid;
    else hi = mid - 1;
  }
  return lo;
}

// Offset in the panel storage of block (hi, lo), positions hi >= lo, and its leading dimension (column-major 9 x 9).
__device__ __forceinline__ long long panel_block(const SparseView<double>& sv, int hi, int lo, int* ld) {
  const int t = sn_of_position(sv, lo);
  const int f = sv.sn_first[t], w = sv.sn_first[t + 1] - f, rp = sv.row_ptr[t], R = sv.row_ptr[t + 1] - rp;
  int idx;
  if (hi < f + w) {
    idx = hi - f;
  } else {
    int a = w, b = R;
    while (a < b) {
      const int mid = (a + b) >> 1;
      if (sv.rows[rp + mid] < hi) a = mid + 1;
      else b = mid;
    }
    idx = a;
  }
  *ld = 9 * R;
  return sv.val[t] + 9LL * idx + 9LL * (lo - f) * (9LL * R);
}

// out[tile rows r0.., column blocks] over K inner steps: acc[h][rr][m] = sum_k A(k, r0 + 2 lane + rr) B(k, 9 (warp + 8 h) + m),
// staged kSpK steps at a time as in sparse_factor_kernel's update (lane l of warp g: rows 2l, 2l + 1 of the tile against
// column blocks g and g + 8).  stage(t0) fills sA [kSpK][kSpTileRows] and sB [kSpK][kSpMaxCols] (zeros past the ends).
template <typename Stage>
__device__ __forceinline__ void selinv_gemm(int K, int ncb, double* sA, double* sB, double (&acc)[2][2][9], Stage&& stage) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int m = 0; m < 9; ++m) acc[h][0][m] = acc[h][1][m] = 0.0;
  for (int t0 = 0; t0 < K; t0 += kSpK) {
    __syncthreads();
    stage(t0);
    __syncthreads();
    if (warp < ncb) {
#pragma unroll 4
      for (int k = 0; k < kSpK; ++k) {
        const double2 a = *reinterpret_cast<const double2*>(sA + k * kSpTileRows + 2 * lane);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const double* b = sB + k * kSpMaxCols + 9 * (warp + 8 * h);
#pragma unroll
          for (int m = 0; m < 9; ++m) {
            const double bm = b[m];
            acc[h][0][m] += a.x * bm;
            acc[h][1][m] += a.y * bm;
          }
        }
      }
    }
  }
}

// The selected-inversion task of supernode s (file comment).
__device__ void selinv_task(const SparseView<double>& sv, double* Z, int s, double* sm) {
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
  const int f = sv.sn_first[s], w = sv.sn_first[s + 1] - f, W = 9 * w;
  const int rp = sv.row_ptr[s], R = sv.row_ptr[s + 1] - rp, ld = 9 * R, nR = ld - W;
  double* Ls = sv.L + sv.val[s];
  double* Zs = Z + sv.val[s];
  double* sB = sm;
  double* sA = sB + kSpK * kSpMaxCols;
  double* sM = sA + kSpK * kSpTileRows;   // L_ss^-1, column-major [W][W]
  __shared__ long long sOff[27];          // blocks of Z_RR a GEMM stage reads: 8 row blocks x 3 column blocks (9 x 3 kept)
  __shared__ int sLd[27], sHow[27];
  // a. L_ss^-1, one column per thread (forward substitution on e_j)
  for (int j = tid; j < W; j += nt) {
    for (int k = 0; k < j; ++k) sM[k + j * W] = 0.0;
    for (int k = j; k < W; ++k) {
      double a = k == j ? 1.0 : 0.0;
      for (int t = j; t < k; ++t) a -= Ls[k + static_cast<long long>(t) * ld] * sM[t + j * W];
      sM[k + j * W] = a / Ls[k + static_cast<long long>(k) * ld];
    }
  }
  __syncthreads();
  // b. U = L_Rs L_ss^-1 in place, one row per thread: column c reads L_Rs columns >= c only, so ascending c is safe
  for (int i = W + tid; i < ld; i += nt) {
    for (int c = 0; c < W; ++c) {
      double u = 0.0;
      for (int t = c; t < W; ++t) u += Ls[i + static_cast<long long>(t) * ld] * sM[t + c * W];
      Ls[i + static_cast<long long>(c) * ld] = u;
    }
  }
  double acc[2][2][9];
  // c. Z_Rs = -Z_RR U, in tiles of kSpTileRows rows of R
  for (int r0 = 0; r0 < nR; r0 += kSpTileRows) {
    selinv_gemm(nR, w, sA, sB, acc, [&](int t0) {
      const int ra0 = (W + r0) / 9, kb0 = (W + t0) / 9;
      if (tid < 27) {
        const int ia = tid / 3, ib = tid % 3;
        const int ra = ra0 + ia, kb = kb0 + ib;
        if (ra < R && kb < R) {
          const int pa = sv.rows[rp + ra], pb = sv.rows[rp + kb];
          int l = 0;
          sOff[tid] = pa >= pb ? panel_block(sv, pa, pb, &l) : panel_block(sv, pb, pa, &l);
          sLd[tid] = l;
          sHow[tid] = pa > pb ? 0 : pa < pb ? 1 : 2;   // as stored / transposed / a diagonal block: either way
        }
      }
      __syncthreads();
      for (int e = tid; e < kSpK * kSpTileRows; e += nt) {
        const int k = e / kSpTileRows, r = e - k * kSpTileRows;
        double a = 0.0;
        if (r0 + r < nR && t0 + k < nR) {
          const int i = W + r0 + r, j = W + t0 + k;
          const int q = 3 * (i / 9 - ra0) + (j / 9 - kb0), ui = i % 9, uj = j % 9;
          const long long o = sOff[q];
          const int l = sLd[q];
          a = __ldcg(Z + (sHow[q] == 1 ? o + uj + static_cast<long long>(ui) * l : o + ui + static_cast<long long>(uj) * l));
        }
        sA[e] = a;
      }
      for (int e = tid; e < kSpK * kSpMaxCols; e += nt) {
        const int k = e / kSpMaxCols, c = e - k * kSpMaxCols;
        sB[e] = c < W && t0 + k < nR ? Ls[W + t0 + k + static_cast<long long>(c) * ld] : 0.0;
      }
    });
    if (warp < w) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int i = r0 + 2 * lane + rr;
        if (i >= nR) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int cb = warp + 8 * h;
          if (cb >= w) continue;
#pragma unroll
          for (int m = 0; m < 9; ++m) Zs[W + i + static_cast<long long>(9 * cb + m) * ld] = -acc[h][rr][m];
        }
      }
    }
  }
  __syncthreads();
  // d. Z_ss = L_ss^-T L_ss^-1 - U' Z_Rs: the lower triangle, mirrored
  for (int r0 = 0; r0 < W; r0 += kSpTileRows) {
    selinv_gemm(nR, w, sA, sB, acc, [&](int t0) {
      for (int e = tid; e < kSpK * kSpTileRows; e += nt) {
        const int k = e / kSpTileRows, r = e - k * kSpTileRows;
        sA[e] = r0 + r < W && t0 + k < nR ? Ls[W + t0 + k + static_cast<long long>(r0 + r) * ld] : 0.0;
      }
      for (int e = tid; e < kSpK * kSpMaxCols; e += nt) {
        const int k = e / kSpMaxCols, c = e - k * kSpMaxCols;
        sB[e] = c < W && t0 + k < nR ? __ldcg(Zs + W + t0 + k + static_cast<long long>(c) * ld) : 0.0;
      }
    });
    if (warp < w) {
#pragma unroll
      for (int rr = 0; rr < 2; ++rr) {
        const int i = r0 + 2 * lane + rr;
        if (i >= W) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int cb = warp + 8 * h;
          if (cb >= w) continue;
#pragma unroll
          for (int m = 0; m < 9; ++m) {
            const int j = 9 * cb + m;
            if (j > i) continue;
            double a = 0.0;
            for (int k = i; k < W; ++k) a += sM[k + i * W] * sM[k + j * W];
            const double z = a - acc[h][rr][m];
            Zs[i + static_cast<long long>(j) * ld] = z;
            Zs[j + static_cast<long long>(i) * ld] = z;
          }
        }
      }
    }
  }
}

// Z on the pattern of L from the factor in sv.L (sparse_factor_kernel's, which this overwrites below the diagonal blocks).
// sv.cnt [ns]: SparsePlan::cnt_inv; ticket reset before the launch.
__global__ void __launch_bounds__(kSpThreads, 1) sparse_selinv_kernel(SparseView<double> sv, double* Z) {
  extern __shared__ __align__(16) unsigned char si_smem_raw[];
  double* sm = reinterpret_cast<double*>(si_smem_raw);
  __shared__ int s_task;
  const int ns = sv.ns;
  for (;;) {
    __syncthreads();
    if (threadIdx.x == 0) s_task = atomicAdd(sv.ticket, 1);
    __syncthreads();
    const int t = s_task;
    if (t >= ns) return;
    const int s = sv.order[ns - 1 - t];
    sp_wait(sv.cnt + s);
    selinv_task(sv, Z, s, sm);
    sp_release_begin();
    if (threadIdx.x == 0)
      for (int k = sv.upd_ptr[s]; k < sv.upd_ptr[s + 1]; ++k) atomicSub(sv.cnt + sv.upd[k].x, 1);
  }
}

// The smallest of the positive doubles offered, as the bits of a double (positive doubles order as their bit patterns); a
// value that is not a finite non-negative number counts as 0.
__device__ __forceinline__ void offer_min(unsigned long long* slot, double v) {
  if (!(v >= 0.0) || !isfinite(v)) v = 0.0;
  atomicMin(slot, static_cast<unsigned long long>(__double_as_longlong(v)));
}

// The conditioning test of the sparse factor: min over variable components k of L_kk^2 / A_kk, A = S + D_f^2 as factored
// (A_kk from the assembled diagonal block of S, the first block of its block row).
__global__ void __launch_bounds__(256) selinv_pivots_kernel(SparseView<double> sv, XsView xv, const int* __restrict__ blk_row_ptr,
                                                           const double* __restrict__ Df, const uint8_t* __restrict__ fixed_f,
                                                           unsigned long long* min_slot) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < 9 * sv.C; k += gridDim.x * blockDim.x) {
    if (fixed_f != nullptr && fixed_f[k] != 0) continue;
    const int c = k / 9, u = k % 9, p = sv.pinv[c];
    const int t = sn_of_position(sv, p);
    const int f = sv.sn_first[t], ld = 9 * (sv.row_ptr[t + 1] - sv.row_ptr[t]);
    const long long i = 9LL * (p - f) + u;
    const double l = sv.L[sv.val[t] + i + i * ld];
    double a = xv.S[81LL * blk_row_ptr[c] + 10 * u];
    if (Df != nullptr) a += Df[k] * Df[k];
    offer_min(min_slot, l * l / a);
  }
}

// cov_s [81 x blocks of S], row-major 9 x 9 blocks Z_ij in S's block order, from the panels (one warp per block).
__global__ void __launch_bounds__(256) selinv_blocks_kernel(SparseView<double> sv, int num_blocks, const double* __restrict__ Z,
                                                           double* __restrict__ cov_s) {
  const int lane = threadIdx.x & 31;
  const int nw = gridDim.x * (blockDim.x / 32);
  for (int b = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); b < num_blocks; b += nw) {
    const long long off = sv.blk_off[b];
    const int ldt = sv.blk_ld[b], ld = ldt < 0 ? -ldt : ldt;
    for (int e = lane; e < 81; e += 32) {
      const int u = e / 9, w = e - 9 * u;
      cov_s[81LL * b + e] = Z[off + (ldt < 0 ? w + static_cast<long long>(u) * ld : u + static_cast<long long>(w) * ld)];
    }
  }
}

// Dense path: diag[k] = A_kk before the factorisation; then the conditioning test on the factor's diagonal.
__global__ void __launch_bounds__(256) dense_diagonal_copy_kernel(int n, const double* __restrict__ A, double* diag) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) diag[k] = A[k + static_cast<size_t>(k) * n];
}
__global__ void __launch_bounds__(256) dense_pivots_kernel(int n, const double* __restrict__ L, const double* __restrict__ diag,
                                                          const uint8_t* __restrict__ fixed_f, unsigned long long* min_slot) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
    if (fixed_f != nullptr && fixed_f[k] != 0) continue;
    const double l = L[k + static_cast<size_t>(k) * n];
    offer_min(min_slot, l * l / diag[k]);
  }
}

// Where the point and gather kernels read Z_ij: the S-ordered block copy of the sparse path (kDense = false; the block of
// the pair found by bisection in the block row's columns, S's diagonal block first) or the dense matrix, made symmetric
// after potri (kDense = true).  Entry (u, v) of Z_ij is base[u su + v sv].
template <bool kDense>
struct ZAccess {
  const double* Z;           // cov_s [81 x blocks] or the dense [9C][9C]
  const int* blk_row_ptr;    // [C + 1] (sparse)
  const int* blk_col;        // [blocks] (sparse)
  long long n;               // 9C (dense)
  __device__ __forceinline__ const double* block(int i, int j, long long* su, long long* sv) const {
    if (kDense) {
      *su = 1;
      *sv = n;
      return Z + 9LL * i + 9LL * j * n;
    }
    const int a = i < j ? i : j, b = i < j ? j : i;
    int lo = blk_row_ptr[a], hi = blk_row_ptr[a + 1];
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (blk_col[mid] < b) lo = mid + 1;
      else hi = mid;
    }
    *su = i <= j ? 9 : 1;
    *sv = i <= j ? 1 : 9;
    return Z + 81LL * lo;
  }
};

// The dense Z: the upper triangle from the lower one potri leaves (one thread per entry below the diagonal).
__global__ void __launch_bounds__(256) dense_symmetrize_kernel(long long n, double* Z) {
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < n * n;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long j = e / n, i = e - j * n;
    if (i > j) Z[j + i * n] = Z[e];
  }
}

// Cov(p, p) of every point, one warp per point, into out [9P] in the caller's point order (row-major 3 x 3), zero for a
// constant point; the pivots of each variable point's Cholesky of V_p = E_p'E_p go to the conditioning test.  A coordinate
// held by a SubsetManifold (fixed == kComponentMasked) has a zero E column: V_p takes D' = 1 there, the coordinate stays
// out of the conditioning test, and its row and column of the block are written as 0 (GetCovarianceBlock lifts the
// tangent covariance with the 0/1 plus Jacobian).  Lane q takes
// the row pairs q, q + 32, ... in a fixed order and the warp sums with a fixed butterfly: no atomics on values.
template <bool kDense>
__global__ void __launch_bounds__(256) covariance_point_kernel(ProblemView p, ZAccess<kDense> z, const uint8_t* __restrict__ fixed,
                                                              const int* __restrict__ pt_perm, double* __restrict__ out,
                                                              unsigned long long* min_slot) {
  const int lane = threadIdx.x & 31;
  const int nw = gridDim.x * (blockDim.x / 32);
  const double* __restrict__ E = p.E();
  const double* __restrict__ F = p.F();
  for (int k = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); k < p.P; k += nw) {
    double* o = out + 9LL * (pt_perm != nullptr ? pt_perm[k] : k);
    if (fixed != nullptr && fixed[3LL * k] == kComponentConstant) {
      if (lane < 9) o[lane] = 0.0;
      continue;
    }
    const unsigned m = fixed == nullptr ? 0u : (fixed[3LL * k] != 0) | (fixed[3LL * k + 1] != 0) << 1 | (fixed[3LL * k + 2] != 0) << 2;
    const int r0 = p.pt_ptr[k], d = p.pt_ptr[k + 1] - r0;
    // V = sum_r E_r'E_r (upper triangle: 00 01 02 11 12 22)
    double v[6] = {0, 0, 0, 0, 0, 0};
    for (int r = r0 + lane; r < r0 + d; r += 32) {
      const double* e = E + 6LL * r;
      v[0] += e[0] * e[0] + e[3] * e[3];
      v[1] += e[0] * e[1] + e[3] * e[4];
      v[2] += e[0] * e[2] + e[3] * e[5];
      v[3] += e[1] * e[1] + e[4] * e[4];
      v[4] += e[1] * e[2] + e[4] * e[5];
      v[5] += e[2] * e[2] + e[5] * e[5];
    }
    // sum over row pairs of W_r Z_{c_r c_s} W_s' (3 x 3, all 9 entries)
    double g[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    const long long pairs = static_cast<long long>(d) * d;
    for (long long q = lane; q < pairs; q += 32) {
      const int r = r0 + static_cast<int>(q / d), s = r0 + static_cast<int>(q % d);
      const int ci = p.cam_idx[r], cj = p.cam_idx[s];
      double wr[27], ws[27];   // W = E'F: [3][9]
      const double* er = E + 6LL * r;
      const double* es = E + 6LL * s;
      const double* fr = F + 18LL * r;
      const double* fs = F + 18LL * s;
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 9; ++b) {
          wr[9 * a + b] = er[a] * fr[b] + er[3 + a] * fr[9 + b];
          ws[9 * a + b] = es[a] * fs[b] + es[3 + a] * fs[9 + b];
        }
      long long su, sv;
      const double* zb = z.block(ci, cj, &su, &sv);
      // row u of Z_{ci cj} W_s' at a time, straight into g += W_r (Z W_s')
#pragma unroll
      for (int u = 0; u < 9; ++u) {
        double t0 = 0.0, t1 = 0.0, t2 = 0.0;
#pragma unroll
        for (int w = 0; w < 9; ++w) {
          const double zz = zb[u * su + w * sv];
          t0 += zz * ws[w];
          t1 += zz * ws[9 + w];
          t2 += zz * ws[18 + w];
        }
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          g[3 * a] += wr[9 * a + u] * t0;
          g[3 * a + 1] += wr[9 * a + u] * t1;
          g[3 * a + 2] += wr[9 * a + u] * t2;
        }
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
#pragma unroll
      for (int m = 0; m < 6; ++m) v[m] += __shfl_xor_sync(0xffffffffu, v[m], off);
#pragma unroll
      for (int m = 0; m < 9; ++m) g[m] += __shfl_xor_sync(0xffffffffu, g[m], off);
    }
    if (lane == 0) {
      if (m & 1u) v[0] = 1.0;   // D' = 1 on masked coordinates (their off-diagonal entries are already 0)
      if (m & 2u) v[3] = 1.0;
      if (m & 4u) v[5] = 1.0;
      // Cholesky of V, its pivots against V's diagonal, V^-1 = L^-T L^-1
      const double l00 = sqrt(v[0]), l10 = v[1] / l00, l20 = v[2] / l00;
      const double d1 = v[3] - l10 * l10, l11 = sqrt(d1), l21 = (v[4] - l20 * l10) / l11;
      const double d2 = v[5] - l20 * l20 - l21 * l21, l22 = sqrt(d2);
      // NaN (v[0] = 0) counts as 0; a masked coordinate offers NaN, which fmin drops
      const double nan = __longlong_as_double(0x7ff8000000000000LL);
      offer_min(min_slot, fmin(fmin((m & 1u) ? nan : v[0] / v[0], (m & 2u) ? nan : d1 / v[3]), (m & 4u) ? nan : d2 / v[5]));
      const double m00 = 1.0 / l00, m11 = 1.0 / l11, m22 = 1.0 / l22;   // M = L^-1 (lower)
      const double m10 = -l10 * m00 * m11, m21 = -l21 * m11 * m22;
      const double m20 = -(l20 * m00 + l21 * m10) * m22;
      double vi[9];
      vi[0] = m00 * m00 + m10 * m10 + m20 * m20;
      vi[1] = vi[3] = m10 * m11 + m20 * m21;
      vi[2] = vi[6] = m20 * m22;
      vi[4] = m11 * m11 + m21 * m21;
      vi[5] = vi[7] = m21 * m22;
      vi[8] = m22 * m22;
      double h[9];   // V^-1 G
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) h[3 * a + b] = vi[3 * a] * g[b] + vi[3 * a + 1] * g[3 + b] + vi[3 * a + 2] * g[6 + b];
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b)
          o[3 * a + b] = ((m >> a) | (m >> b)) & 1u ? 0.0
                                                     : vi[3 * a + b] + h[3 * a] * vi[b] + h[3 * a + 1] * vi[3 + b] + h[3 * a + 2] * vi[6 + b];
    }
  }
}

// The requested camera blocks: out [81 x n] row-major, pair q = {i, j, -, zero mask}: bit u (u < 9) zeroes row u, bit
// 9 + v column v (the constant coordinates of camera i and of camera j; all of them for a constant camera).
template <bool kDense>
__global__ void __launch_bounds__(256) covariance_gather_kernel(ZAccess<kDense> z, int n, const int4* __restrict__ pairs,
                                                               double* __restrict__ out) {
  for (long long e = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; e < 81LL * n;
       e += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int q = static_cast<int>(e / 81), uv = static_cast<int>(e % 81), u = uv / 9, v = uv % 9;
    const int4 pr = pairs[q];
    long long su, sv;
    const double* zb = z.block(pr.x, pr.y, &su, &sv);
    out[e] = ((pr.w >> u) | (pr.w >> (9 + v))) & 1 ? 0.0 : zb[u * su + v * sv];
  }
}

}  // namespace b200
