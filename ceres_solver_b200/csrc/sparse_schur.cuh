// SPARSE_SCHUR on the device (SparseSchurComplementSolver, schur_complement_solver.cc:205-335): S + D_f^2, assembled by
// xs_assemble_kernel, is scattered into the supernodal panels of sparse_plan.cuh and factored by a supernodal Cholesky; the
// factorisation and both triangular solves run as one persistent kernel.  The factor and the vector it solves in are of one
// type T: double, or float for use_mixed_precision_solves (solver.h:572-590), where S + D_f^2 is formed in FP64 and rounded
// once as it is scattered (FloatSuiteSparseCholesky::Factorize, suitesparse.cc:487-498).  Either way the schedule, the tickets
// and the summation order are the same.  A solve-only launch (kFactor = false) reuses a factor for the corrections of
// iterative refinement: its forward task runs step 3 alone, which depends on exactly the descendants step 1 does.
//
// Tasks: 2 ns tickets, taken in order from a global counter by whichever CTA is free.  Ticket t < ns is the forward task of
// supernode s = order[t]: it waits until every descendant that updates s is done, then (left-looking) subtracts their updates
// from its panel in ascending order of descendant, factors the panel (right-looking, one 9-column block at a time), and
// computes its part of y = L^-1 rhs.  Ticket t >= ns is the backward task of s = order[2 ns - 1 - t]: once every supernode
// holding one of its rows below is done (a root: once its own forward task is), x_s = L_ss^-T (y_s - L_below,s' x_below).
// `order` (sparse_plan.cuh) is topological, every descendant before its ancestors: the identity with AMD, leaves first with
// nested dissection.  So a forward task waits only on descendants, whose forward tickets are smaller; a backward task only on
// ancestors, whose backward tickets are smaller, or (a root) on its own forward ticket.  A task thus only waits on tasks with
// smaller tickets, which have all been taken by CTAs that are running (the launch is cooperative: every CTA is resident), so
// the walk cannot deadlock.  Each panel entry and each entry of y and x is written by the one CTA that owns the supernode, in
// a fixed order: no atomics on values, and the result is bitwise reproducible.  The counters themselves are atomics.
//
// Memory ordering: a task's writes are fenced before it decrements its dependants' counters, and a CTA reads another
// supernode's panel or vector entries with ld.global.cg (L2), never through its L1.
#pragma once
#include "explicit_schur.cuh"

namespace b200 {

constexpr int kSpThreads = 256;   // 8 warps: warp g takes column blocks g and g + 8 of an update
constexpr int kSpMaxCols = 144;   // 9 x kSnMaxCams (sparse_plan.cuh): the widest supernode
constexpr int kSpTileRows = 64;   // rows of an update tile: two per lane
constexpr int kSpK = 16;          // columns of the descendant staged per step

template <typename T>
struct SparseView {
  int C, ns;
  const int* pinv;            // [C] camera -> position
  const int* sn_first;        // [ns + 1]
  const int* row_ptr;         // [ns + 1]
  const int* rows;            // positions: the supernode's columns, then its rows below
  const long long* val;       // [ns] panel offsets (column-major, leading dimension 9 x rows)
  const int* upd_ptr;         // [ns + 1]
  const int4* upd;            // {descendant d, k0, k1, 0}
  const int* ntf_ptr;         // [ns + 1]
  const int* ntf;             // supernodes each supernode updates
  const int* order;           // [ns] supernode of each forward ticket, topological
  const long long* blk_off;   // per block of S: offset of its place in L
  const int* blk_ld;          // ... leading dimension there, negative: the block goes in transposed
  T* L;
  T* v;                       // [9C] by position: rhs, then y, then x
  int* cnt;                   // [2 ns] dependency counters of the forward / backward tasks
  int* ticket;
  int* fail;                  // set on a non-positive or non-finite pivot
};

// L <- the blocks of S (as assembled: the upper triangle, without D_f^2) + D_f^2 on the diagonal, into zeroed storage; v <- the
// reduced right-hand side in the elimination order, each value rounded to T once.  One warp per block of S.
template <typename T>
__global__ void __launch_bounds__(256) sparse_scatter_kernel(SparseView<T> sv, XsView xv, const double* __restrict__ Df,
                                                            const double* __restrict__ rhs) {
  const int lane = threadIdx.x & 31;
  const int nw = gridDim.x * (blockDim.x / 32);
  for (int b = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5); b < xv.num_blocks; b += nw) {
    const long long off = sv.blk_off[b];
    const int ldt = sv.blk_ld[b], ld = ldt < 0 ? -ldt : ldt;
    const int i = xv.blk_row[b];
    const bool diag = i == xv.blk_col[b];
    for (int e = lane; e < 81; e += 32) {
      const int u = e / 9, w = e - 9 * u;
      double s = xv.S[81 * static_cast<size_t>(b) + e];
      if (diag && u == w && Df != nullptr) s += Df[9 * i + u] * Df[9 * i + u];
      sv.L[off + (ldt < 0 ? w + static_cast<long long>(u) * ld : u + static_cast<long long>(w) * ld)] = static_cast<T>(s);
    }
  }
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < 9 * sv.C; k += gridDim.x * blockDim.x)
    sv.v[9 * sv.pinv[k / 9] + k % 9] = static_cast<T>(rhs[k]);
}

// sol [9C] in the caller's camera order <- x by position, widened to double.
template <typename T>
__global__ void __launch_bounds__(256) sparse_gather_kernel(SparseView<T> sv, double* __restrict__ sol) {
  for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < 9 * sv.C; k += gridDim.x * blockDim.x)
    sol[k] = static_cast<double>(sv.v[9 * sv.pinv[k / 9] + k % 9]);
}

// Dynamic shared memory of sparse_factor_kernel for supernodes of at most W scalar columns: the update stages, the block
// column being factored [W][9], and y_s / z_s [W].
template <typename T>
inline size_t sparse_smem_bytes(int W) {
  return sizeof(T) * (kSpK * (kSpMaxCols + kSpTileRows) + 9 * static_cast<size_t>(W) + W);
}

template <typename T> struct SpPair;
template <> struct SpPair<double> { using type = double2; };
template <> struct SpPair<float> { using type = float2; };

__device__ __forceinline__ void sp_wait(int* c) {
  if (threadIdx.x == 0) {
    while (*reinterpret_cast<volatile int*>(c) > 0) __nanosleep(32);
    __threadfence();
  }
  __syncthreads();
}
// every thread's writes of the task are fenced before thread 0 releases the dependants
__device__ __forceinline__ void sp_release_begin() {
  __threadfence();
  __syncthreads();
}

// The forward task of supernode s: steps 1 and 2 only when kFactor.
template <typename T, bool kFactor>
__device__ void sp_forward(const SparseView<T>& sv, int s, T* sm) {
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
  const int f = sv.sn_first[s], w = sv.sn_first[s + 1] - f, W = 9 * w;
  const int rp = sv.row_ptr[s], R = sv.row_ptr[s + 1] - rp, ld = 9 * R;
  T* Ls = sv.L + sv.val[s];
  T* sB = sm;                                        // update stages: B [kSpK][kSpMaxCols], then A [kSpK][kSpTileRows]
  T* sX = sm + kSpK * (kSpMaxCols + kSpTileRows);    // block column K of the rows of the diagonal block: [9w][9]
  T* sY = sX + 9 * W;                                // y_s
  __shared__ T sK[81];                               // diagonal block K, column-major
  const int u0 = sv.upd_ptr[s], u1 = sv.upd_ptr[s + 1];
  if (kFactor) {
  // 1. left-looking updates: Ls -= L_d[rows k0.., :] L_d[rows k0..k1-1, :]', in tiles of kSpTileRows rows: A = the tile's
  //    rows and B = the rows in s's columns, both staged kSpK columns of L_d at a time.  Lane l of warp g accumulates rows
  //    2l, 2l + 1 of the tile against column blocks g and g + 8 (9 columns each): 36 products per 2 + 18 shared loads.
  T* sA = sB + kSpK * kSpMaxCols;
  for (int q = u0; q < u1; ++q) {
    const int4 u = sv.upd[q];
    const int d = u.x, k0 = u.y, k1 = u.z;
    const int fd = sv.sn_first[d], Wd = 9 * (sv.sn_first[d + 1] - fd);
    const int rpd = sv.row_ptr[d], Rd = sv.row_ptr[d + 1] - rpd, ldd = 9 * Rd;
    const T* Ld = sv.L + sv.val[d];
    const int ncb = k1 - k0, nc = 9 * ncb, iend = 9 * Rd;
    for (int r0 = 9 * k0; r0 < iend; r0 += kSpTileRows) {
      T acc[2][2][9];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int m = 0; m < 9; ++m) acc[h][0][m] = acc[h][1][m] = T(0);
      for (int t0 = 0; t0 < Wd; t0 += kSpK) {
        __syncthreads();
        for (int e = tid; e < kSpK * kSpTileRows; e += nt) {
          const int k = e / kSpTileRows, r = e - k * kSpTileRows;
          sA[e] = r0 + r < iend && t0 + k < Wd ? __ldcg(Ld + r0 + r + static_cast<long long>(t0 + k) * ldd) : T(0);
        }
        for (int e = tid; e < kSpK * kSpMaxCols; e += nt) {
          const int k = e / kSpMaxCols, c = e - k * kSpMaxCols;
          sB[e] = c < nc && t0 + k < Wd ? __ldcg(Ld + 9 * k0 + c + static_cast<long long>(t0 + k) * ldd) : T(0);
        }
        __syncthreads();
        if (warp < ncb) {
#pragma unroll 4
          for (int k = 0; k < kSpK; ++k) {
            const typename SpPair<T>::type a = *reinterpret_cast<const typename SpPair<T>::type*>(sA + k * kSpTileRows + 2 * lane);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const T* b = sB + k * kSpMaxCols + 9 * (warp + 8 * h);
#pragma unroll
              for (int m = 0; m < 9; ++m) {
                const T bm = b[m];
                acc[h][0][m] += a.x * bm;
                acc[h][1][m] += a.y * bm;
              }
            }
          }
        }
      }
      if (warp < ncb) {
#pragma unroll
        for (int rr = 0; rr < 2; ++rr) {
          const int i = r0 + 2 * lane + rr;
          if (i >= iend) continue;
          const int pos = sv.rows[rpd + i / 9];
          int idx;
          if (pos < f + w) {
            idx = pos - f;
          } else {   // binary search among the rows below
            int lo = w, hi = R;
            while (lo < hi) {
              const int mid = (lo + hi) >> 1;
              if (sv.rows[rp + mid] < pos) lo = mid + 1;
              else hi = mid;
            }
            idx = lo;
          }
          const long long trow = 9LL * idx + i % 9;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int cb = warp + 8 * h;
            if (cb >= ncb) continue;
            const long long col = 9LL * (sv.rows[rpd + k0 + cb] - f);
#pragma unroll
            for (int m = 0; m < 9; ++m) Ls[trow + (col + m) * ld] -= acc[h][rr][m];
          }
        }
      }
    }
  }
  // 2. the panel: for each block column K, Cholesky of its diagonal block, the rows below it times L_KK^-T, and the update of
  //    the trailing columns
  for (int K = 0; K < w; ++K) {
    __syncthreads();
    if (tid < 81) sK[tid] = Ls[9 * K + tid % 9 + static_cast<long long>(9 * K + tid / 9) * ld];
    __syncthreads();
    if (tid == 0) {
      bool bad = false;
      for (int c = 0; c < 9; ++c) {
        T dcc = sK[c * 9 + c];
        for (int t = 0; t < c; ++t) dcc -= sK[t * 9 + c] * sK[t * 9 + c];
        if (!(dcc > T(0)) || !isfinite(dcc)) bad = true;
        const T lcc = sqrt(dcc);
        sK[c * 9 + c] = lcc;
        for (int r = c + 1; r < 9; ++r) {
          T a = sK[c * 9 + r];
          for (int t = 0; t < c; ++t) a -= sK[t * 9 + r] * sK[t * 9 + c];
          sK[c * 9 + r] = a / lcc;
        }
      }
      if (bad) *sv.fail = 1;
    }
    __syncthreads();
    if (tid < 81 && tid % 9 >= tid / 9) Ls[9 * K + tid % 9 + static_cast<long long>(9 * K + tid / 9) * ld] = sK[tid];
    const int i0 = 9 * (K + 1);
    auto solve_row = [&](int i, T* x) {   // x = A_iK L_KK^-T
#pragma unroll
      for (int c = 0; c < 9; ++c) {
        T a = Ls[i + static_cast<long long>(9 * K + c) * ld];
#pragma unroll
        for (int t = 0; t < c; ++t) a -= x[t] * sK[t * 9 + c];
        x[c] = a / sK[c * 9 + c];
      }
#pragma unroll
      for (int c = 0; c < 9; ++c) Ls[i + static_cast<long long>(9 * K + c) * ld] = x[c];
    };
    for (int i = i0 + tid; i < W; i += nt) {   // rows of the diagonal block: staged for the trailing update
      T x[9];
      solve_row(i, x);
#pragma unroll
      for (int c = 0; c < 9; ++c) sX[(i - i0) * 9 + c] = x[c];
    }
    __syncthreads();
    for (int i = i0 + tid; i < 9 * R; i += nt) {
      T x[9];
      if (i < W) {
#pragma unroll
        for (int c = 0; c < 9; ++c) x[c] = sX[(i - i0) * 9 + c];
      } else {
        solve_row(i, x);
      }
      const int jmax = i < W ? i : W - 1;   // lower triangle of the diagonal block, every column below it
      for (int j = i0; j <= jmax; ++j) {
        const T* xj = sX + (j - i0) * 9;
        T a = T(0);
#pragma unroll
        for (int c = 0; c < 9; ++c) a += x[c] * xj[c];
        Ls[i + static_cast<long long>(j) * ld] -= a;
      }
    }
  }
  }   // kFactor
  __syncthreads();
  // 3. y_s = L_ss^-1 (rhs_s - sum over the descendants of L_d[rows in s] y_d)
  for (int c = tid; c < W; c += nt) sY[c] = __ldcg(sv.v + 9LL * f + c);
  __syncthreads();
  for (int q = u0; q < u1; ++q) {
    const int4 u = sv.upd[q];
    const int d = u.x, k0 = u.y, k1 = u.z;
    const int fd = sv.sn_first[d], Wd = 9 * (sv.sn_first[d + 1] - fd);
    const int rpd = sv.row_ptr[d], ldd = 9 * (sv.row_ptr[d + 1] - rpd);
    const T* Ld = sv.L + sv.val[d];
    const int nc = 9 * (k1 - k0);
    for (int c = tid; c < nc; c += nt) {
      T a = T(0);
      for (int t = 0; t < Wd; ++t) a += __ldcg(Ld + 9 * k0 + c + static_cast<long long>(t) * ldd) * __ldcg(sv.v + 9LL * fd + t);
      sY[9 * (sv.rows[rpd + k0 + c / 9] - f) + c % 9] -= a;
    }
    __syncthreads();
  }
  if (warp == 0) {
    for (int j = 0; j < W; ++j) {
      const T yj = sY[j] / Ls[j + static_cast<long long>(j) * ld];
      __syncwarp();
      if (lane == 0) sY[j] = yj;
      for (int i = j + 1 + lane; i < W; i += 32) sY[i] -= Ls[i + static_cast<long long>(j) * ld] * yj;
      __syncwarp();
    }
  }
  __syncthreads();
  for (int c = tid; c < W; c += nt) sv.v[9LL * f + c] = sY[c];
}

// The backward task of supernode s.
template <typename T>
__device__ void sp_backward(const SparseView<T>& sv, int s, T* sm) {
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
  const int f = sv.sn_first[s], w = sv.sn_first[s + 1] - f, W = 9 * w;
  const int rp = sv.row_ptr[s], R = sv.row_ptr[s + 1] - rp, ld = 9 * R;
  const T* Ls = sv.L + sv.val[s];
  T* sZ = sm;
  // z_c = y_c - sum over the rows below of L[i][c] x_i: one warp per column, a fixed butterfly
  for (int c = warp; c < W; c += nt / 32) {
    T a = T(0);
    for (int i = W + lane; i < 9 * R; i += 32) a += Ls[i + static_cast<long long>(c) * ld] * __ldcg(sv.v + 9LL * sv.rows[rp + i / 9] + i % 9);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) sZ[c] = __ldcg(sv.v + 9LL * f + c) - a;
  }
  __syncthreads();
  if (warp == 0) {
    for (int j = W - 1; j >= 0; --j) {
      const T xj = sZ[j] / Ls[j + static_cast<long long>(j) * ld];
      __syncwarp();
      if (lane == 0) sZ[j] = xj;
      for (int i = lane; i < j; i += 32) sZ[i] -= Ls[j + static_cast<long long>(i) * ld] * xj;
      __syncwarp();
    }
  }
  __syncthreads();
  for (int c = tid; c < W; c += nt) sv.v[9LL * f + c] = sZ[c];
}

// The factorisation (kFactor) and both triangular solves: a cooperative launch of at most the resident CTAs, counters and
// ticket reset before it.
template <typename T, bool kFactor>
__global__ void __launch_bounds__(kSpThreads, 1) sparse_factor_kernel(SparseView<T> sv) {
  extern __shared__ __align__(16) unsigned char sp_smem_raw[];
  T* sp_smem = reinterpret_cast<T*>(sp_smem_raw);
  __shared__ int s_task;
  const int ns = sv.ns;
  for (;;) {
    __syncthreads();
    if (threadIdx.x == 0) s_task = atomicAdd(sv.ticket, 1);
    __syncthreads();
    const int t = s_task;
    if (t >= 2 * ns) return;
    if (t < ns) {
      const int s = sv.order[t];
      sp_wait(sv.cnt + s);
      sp_forward<T, kFactor>(sv, s, sp_smem);
      sp_release_begin();
      if (threadIdx.x == 0) {
        const int n0 = sv.ntf_ptr[s], n1 = sv.ntf_ptr[s + 1];
        for (int k = n0; k < n1; ++k) atomicSub(sv.cnt + sv.ntf[k], 1);
        if (n0 == n1) atomicSub(sv.cnt + ns + s, 1);   // a root: its backward task may start
      }
    } else {
      const int s = sv.order[2 * ns - 1 - t];
      sp_wait(sv.cnt + ns + s);
      sp_backward<T>(sv, s, sp_smem);
      sp_release_begin();
      if (threadIdx.x == 0)
        for (int k = sv.upd_ptr[s]; k < sv.upd_ptr[s + 1]; ++k) atomicSub(sv.cnt + ns + sv.upd[k].x, 1);
    }
  }
}

}  // namespace b200
