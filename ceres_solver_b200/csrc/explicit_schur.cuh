// The reduced camera system S = sum_p [F'F - W' (E'E + D_e^2)^-1 W]_p as an explicit block-sparse matrix, for problems
// whose camera graph is sparse enough that S is much smaller than the stream the implicit product reads (DESIGN §1, §3).
// S is assembled once per linear solve and then multiplied once per CG iteration; it is the operator of
// ImplicitSchurComplement (implicit_schur_complement.cc:49-276) stored, as the reference does with
// use_explicit_schur_complement + SCHUR_JACOBI (iterative_schur_complement_solver.cc:64-157).
//
// Storage: the upper triangle (blocks (i, j >= i)) as 9x9 row-major blocks, block row i owning its blocks, the diagonal
// block first.  D_f^2 is not stored: the PCG seeds D_f^2 p into the product's output and invert9_kernel adds it to the
// diagonal blocks.
//
// Assembly.  With G_rs = E_r (E'E + D_e^2)^-1 E_s' (2x2) for two rows r, s of one point,
//     S_ij = sum over row pairs (r, s) of one point with cam r = i, cam s = j of  -F_r' (G_rs - [r == s] I) F_s,
// i.e. W_r' P W_s = F_r' E_r P E_s' F_s and F_r'F_r on the diagonal.  b200_create lists, for every block, its row pairs
// (a diagonal block (i, i) gets all ordered pairs, so two rows of one point that see camera i contribute the block and
// its transpose).  One warp owns one block, or one CTA a block with many pairs (the diagonal blocks): no atomics, fixed
// summation order, plain stores.
//
// Product (one pass over the stored triangle).  The warp that owns block row i streams it once, three blocks per step
// (lane 9e + w holds column w of the step's block e, lanes 27..31 idle).  For each block (i, j) it adds S_ij x_j into
// the row part a_i, and for j > i it also forms t_ij = S_ij' x_i, which it stores in the block's slot of T.  It writes
// y_i = seed + a_i; the column part sum_{i<j} t_ij of q_j is added by whoever reads q next: the PCG's vector kernel or
// the vector phase of the resident PCG (xs_col_sum, xs_pcg.cuh) or, outside the PCG, xs_gather_kernel.  T is ordered by column, so that sum reads contiguous slots.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int kXsThreads = 256;       // product: 8 warps per CTA
constexpr int kXsWarps = kXsThreads / 32;
constexpr int kXsMinCtas = 2;         // product CTAs per SM its register budget (__launch_bounds__) is sized for
constexpr int kXsStep = 3;            // blocks per product step: lane 9e + w owns column w of block e
constexpr int kXsAsmThreads = 256;    // assembly: one warp per block, or one CTA per block with a long pair list
constexpr int kXsLongPairs = 96;      // ... longer than this
// product step descriptor {first block, row | count << 27 | first of row | last of row}
constexpr int kXsStepCountShift = 27;
constexpr int kXsStepFirst = 1 << 29;
constexpr int kXsStepLast = 1 << 30;

struct XsView {
  int C;
  int num_blocks;
  const int* blk_row;        // [num_blocks] i of block (i, j)
  const int* blk_col;        // [num_blocks] j
  const int* pair_ptr;       // [num_blocks + 1] row pairs of each block
  const int2* pairs;         // (r, s): cam r = i, cam s = j, same point
  const int2* cols;          // [num_blocks] {j, T slot of the block; -1 for a diagonal block}
  const int* col_ptr;        // [C + 1] T slots of column j: its blocks (i, j), i < j, in order of i
  const int2* steps;         // product steps, each warp's in order (descriptor above)
  const int* warp_step;      // [warps + 1] first step of each product warp
  double* S;                 // [num_blocks][81]
  double* T;                 // [pairs][9] t_ij = S_ij' x_i of the last product, by T slot
};

// Row pairs [q_begin, q_end) of one block into the lane's entries (u, w0 .. w0 + 2); lanes 0..26 own entries.  G of 8
// pairs at a time (lane 4q + 2a + c computes G_rs[a][c] of pair q), then the F rows of 4 pairs are fetched together.
__device__ __forceinline__ void xs_pairs(const XsView& v, const ProblemView& p, const double* __restrict__ ete_inv, int q_begin,
                                         int q_end, int lane, double& acc0, double& acc1, double& acc2) {
  const double* __restrict__ E = p.E();
  const double* __restrict__ F = p.F();
  const bool owner = lane < 27;
  const int u = owner ? lane / 3 : 0, w0 = owner ? 3 * (lane - 3 * (lane / 3)) : 0;
  const int q = lane >> 2, ga = (lane >> 1) & 1, gc = lane & 1;
  for (int q0 = q_begin; q0 < q_end; q0 += 8) {
    const int nq = min(8, q_end - q0);
    int r = 0, s = 0;
    double g = 0.0;
    if (q < nq) {
      const int2 rs = __ldg(v.pairs + q0 + q);
      r = rs.x;
      s = rs.y;
      const double* er = E + 6 * static_cast<size_t>(r) + 3 * ga;
      const double* es = E + 6 * static_cast<size_t>(s) + 3 * gc;
      const double e0 = es[0], e1 = es[1], e2 = es[2], f0 = er[0], f1 = er[1], f2 = er[2];
      const double* pp = ete_inv + 6 * static_cast<size_t>(__ldg(p.pt_of_row + r));
      const double P00 = pp[0], P01 = pp[1], P02 = pp[2], P11 = pp[3], P12 = pp[4], P22 = pp[5];
      const double pe0 = P00 * e0 + P01 * e1 + P02 * e2;
      const double pe1 = P01 * e0 + P11 * e1 + P12 * e2;
      const double pe2 = P02 * e0 + P12 * e1 + P22 * e2;
      g = f0 * pe0 + f1 * pe1 + f2 * pe2;
      if (r == s && ga == gc) g -= 1.0;   // F_r'F_r of the diagonal: -F_r'(G - I)F_r
    }
    for (int t0 = 0; t0 < nq; t0 += 4) {
      double fr[4][2], fs[4][6], gg[4][4];
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int src = 4 * (t0 + t);   // lanes of pairs past nq hold r = s = 0 and g = 0: a zero contribution
#pragma unroll
        for (int k = 0; k < 4; ++k) gg[t][k] = __shfl_sync(0xffffffffu, g, (src + k) & 31);
        const int rr = __shfl_sync(0xffffffffu, r, src & 31), ss = __shfl_sync(0xffffffffu, s, src & 31);
        const double* pr = F + 18 * static_cast<size_t>(rr) + u;
        const double* ps = F + 18 * static_cast<size_t>(ss) + w0;
        fr[t][0] = pr[0];
        fr[t][1] = pr[9];
#pragma unroll
        for (int m = 0; m < 3; ++m) {
          fs[t][m] = ps[m];
          fs[t][3 + m] = ps[9 + m];
        }
      }
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        if (t0 + t >= nq) continue;
        const double a0 = gg[t][0] * fr[t][0] + gg[t][2] * fr[t][1], a1 = gg[t][1] * fr[t][0] + gg[t][3] * fr[t][1];   // G' F_r[:, u]
#pragma unroll
        acc0 -= a0 * fs[t][0] + a1 * fs[t][3];
        acc1 -= a0 * fs[t][1] + a1 * fs[t][4];
        acc2 -= a0 * fs[t][2] + a1 * fs[t][5];
      }
    }
  }
}

// S (and, for the diagonal blocks, their upper triangles in upper45, the layout invert9_kernel reads) from J and
// (E'E + D_e^2)^-1.  kLong: one CTA per block of `blocks`, its warps take contiguous eighths of the pair list and add
// their sums in warp order; otherwise one warp per block.
template <bool kLong>
__global__ void __launch_bounds__(kXsAsmThreads) xs_assemble_kernel(XsView v, ProblemView p, const int* __restrict__ blocks,
                                                                   int num, const double* __restrict__ ete_inv,
                                                                   double* __restrict__ upper45) {
  __shared__ double s_part[kLong ? kXsAsmThreads / 32 : 1][81];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool owner = lane < 27;
  const int u = owner ? lane / 3 : 0, w0 = owner ? 3 * (lane - 3 * (lane / 3)) : 0;
  const int item0 = kLong ? static_cast<int>(blockIdx.x) : static_cast<int>(blockIdx.x) * (kXsAsmThreads / 32) + warp;
  const int items = kLong ? static_cast<int>(gridDim.x) : static_cast<int>(gridDim.x) * (kXsAsmThreads / 32);
  for (int it = item0; it < num; it += items) {
    const int b = __ldg(blocks + it);
    const int p0 = __ldg(v.pair_ptr + b), p1 = __ldg(v.pair_ptr + b + 1);
    double acc[3] = {0.0, 0.0, 0.0};
    if (kLong) {
      constexpr int W = kXsAsmThreads / 32;
      const int n = p1 - p0;
      xs_pairs(v, p, ete_inv, p0 + static_cast<int>(static_cast<long long>(n) * warp / W),
               p0 + static_cast<int>(static_cast<long long>(n) * (warp + 1) / W), lane, acc[0], acc[1], acc[2]);
      __syncthreads();
      if (owner)
#pragma unroll
        for (int m = 0; m < 3; ++m) s_part[warp][9 * u + w0 + m] = acc[m];
      __syncthreads();
      if (warp != 0) continue;
      if (owner)
#pragma unroll
        for (int m = 0; m < 3; ++m) {
          double t = 0.0;
#pragma unroll
          for (int k = 0; k < W; ++k) t += s_part[k][9 * u + w0 + m];
          acc[m] = t;
        }
    } else {
      xs_pairs(v, p, ete_inv, p0, p1, lane, acc[0], acc[1], acc[2]);
    }
    if (owner) {
      double* sb = v.S + 81 * static_cast<size_t>(b) + 9 * u + w0;
      sb[0] = acc[0];
      sb[1] = acc[1];
      sb[2] = acc[2];
      const int i = __ldg(v.blk_row + b);
      if (upper45 != nullptr && __ldg(v.blk_col + b) == i) {
        double* o = upper45 + 45 * static_cast<size_t>(i) + u * 9 - u * (u - 1) / 2 - u;
        if (u <= w0) o[w0] = acc[0];
        if (u <= w0 + 1) o[w0 + 1] = acc[1];
        if (u <= w0 + 2) o[w0 + 2] = acc[2];
      }
    }
  }
}

// The lane's column of the blocks of one product step and the column entry it reads them with.
struct XsStepData {
  int2 d;        // step descriptor
  int2 c;        // {j, T slot} of the lane's block ({0, -1}: no block)
  double s[9];   // S[u][w] of the lane's block, u = 0..8
};
// kShared: v.steps and v.cols point into shared memory (the resident PCG's staged copies), not at the global arrays
template <bool kShared>
__device__ __forceinline__ int2 xs_step_desc(const XsView& v, int k, int k1) {
  return k < k1 ? (kShared ? v.steps[k] : __ldg(v.steps + k)) : make_int2(0, 0);   // past the end: a step of no blocks
}
__device__ __forceinline__ bool xs_lane_in(int2 d, int e) { return e < ((d.y >> kXsStepCountShift) & 3); }
template <bool kShared>
__device__ __forceinline__ int2 xs_step_col(const XsView& v, int2 d, int e) {
  return xs_lane_in(d, e) ? (kShared ? v.cols[d.x + e] : __ldg(v.cols + d.x + e)) : make_int2(0, -1);
}
__device__ __forceinline__ void xs_step_s(const XsView& v, int2 d, int e, int w, double* s) {
  const bool in = xs_lane_in(d, e);
  const int b = in ? d.x + e : 0;
  const double* sb = v.S + 81 * static_cast<size_t>(b) + w;
#pragma unroll
  for (int u = 0; u < 9; ++u) s[u] = in ? __ldg(sb + 9 * u) : 0.0;
}

// The walk of one warp over its product steps [k0, k1), shared by xs_mul_kernel and the resident PCG (xs_pcg.cuh), so that
// both form S x with the same arithmetic in the same order: lane 9e + w, the next step's S and x_j in flight and the
// column entries of the one after, the butterfly of each row sum, and t_ij stored into its T slot.  load_s(d, e, w, s)
// fills the lane's column of step d's block e, load_x(j, w) returns entry w of x_j, row_out(i, lane, a_i[lane], x_i[lane])
// takes the row part of row i in lanes 0..8.  xs_walk_begin loads what does not depend on x (before a grid dependency
// resolves); xs_walk returns the lane's share of x . S x (x_i . a_i over its rows, x_j . t_ij over its blocks).
// kShared: the descriptors and column entries come from shared memory (xs_step_desc).
// A range may begin or end inside a row (the resident PCG splits long rows over warps): a range that begins inside row
// i reads x_i with load_xi(i, u) instead of from its diagonal block, and one that ends inside a row passes row_out the
// sum of that row's blocks in the range.  Either way x_i . (that sum) goes into the returned share.
struct XsWalk {
  XsStepData nx;   // step k + 1
  int2 d2, c2;     // step k + 2: descriptor and column entry
};
template <bool kShared = false, class LoadS>
__device__ __forceinline__ void xs_walk_begin(const XsView& v, int k0, int k1, int e, int w, LoadS load_s, XsWalk& wk) {
  wk.nx.d = xs_step_desc<kShared>(v, k0, k1);
  wk.nx.c = xs_step_col<kShared>(v, wk.nx.d, e);
  load_s(wk.nx.d, e, w, wk.nx.s);
  wk.d2 = xs_step_desc<kShared>(v, k0 + 1, k1);
  wk.c2 = xs_step_col<kShared>(v, wk.d2, e);
}
constexpr int kXsStepRowMask = (1 << kXsStepCountShift) - 1;
template <bool kShared = false, class LoadS, class LoadX, class LoadXi, class RowOut>
__device__ __forceinline__ double xs_walk(const XsView& v, int k0, int k1, int lane, int e, int w, LoadS load_s, LoadX load_x,
                                          LoadXi load_xi, RowOut row_out, XsWalk& wk) {
  XsStepData& nx = wk.nx;
  int2 d2 = wk.d2, c2 = wk.c2;
  double nx_x = xs_lane_in(nx.d, e) ? load_x(nx.c.x, w) : 0.0;
  double acc[9], xi[9];
#pragma unroll
  for (int u = 0; u < 9; ++u) acc[u] = xi[u] = 0.0;
  if (k0 < k1 && !(nx.d.y & kXsStepFirst))
#pragma unroll
    for (int u = 0; u < 9; ++u) xi[u] = load_xi(nx.d.y & kXsStepRowMask, u);
  double pq = 0.0;
  for (int k = k0; k < k1; ++k) {
    const int2 d = nx.d, c = nx.c;
    double s[9];
#pragma unroll
    for (int u = 0; u < 9; ++u) s[u] = nx.s[u];
    const double xj = nx_x;
    // refill: step k + 1 from the entries loaded one step ago, the column entries of step k + 2
    nx.d = d2;
    nx.c = c2;
    load_s(nx.d, e, w, nx.s);
    nx_x = xs_lane_in(nx.d, e) ? load_x(nx.c.x, w) : 0.0;
    d2 = xs_step_desc<kShared>(v, k + 2, k1);
    c2 = xs_step_col<kShared>(v, d2, e);
    // a row begins with its diagonal block in lanes 0..8: their x_j is x_i
    if (d.y & kXsStepFirst)
#pragma unroll
      for (int u = 0; u < 9; ++u) xi[u] = __shfl_sync(0xffffffffu, xj, u);
    double t = 0.0;
#pragma unroll
    for (int u = 0; u < 9; ++u) {
      acc[u] += s[u] * xj;   // lanes without a block hold s = 0, x_j = 0
      t += s[u] * xi[u];
    }
    if (c.y >= 0) {
      v.T[9 * static_cast<size_t>(c.y) + w] = t;
      pq += xj * t;
    }
    if ((d.y & kXsStepLast) || k + 1 == k1) {
      // a_i[u] = sum over the lanes of acc[u]: a butterfly, so every lane holds the same bits
      double mine = 0.0, xo = 0.0;
#pragma unroll
      for (int u = 0; u < 9; ++u) {
        double a = acc[u];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == u) {
          mine = a;
          xo = xi[u];
        }
        acc[u] = 0.0;
      }
      if (lane < 9) {
        pq += xo * mine;
        row_out(d.y & kXsStepRowMask, lane, mine, xo);
      }
    }
  }
  return pq;
}

// y = [y if accumulate] + [D_f^2 x if Df] + (row part of S x), and T = the column part (file comment), S as assembled
// (without D_f^2).  Inside the PCG: accumulate onto the output the vector kernel seeded, no-op once done_flag is set, and
// pq_part[CTA] = sum over this CTA's rows of x_i . a_i + sum over its off-diagonal blocks of x_j . t_ij, i.e. its share of
// x . S x -- the product protocol of schur_mul_v4_kernel.  Launched with programmatic stream serialisation behind the
// vector kernel: the steps, column entries and S of the first two steps are static and are read before the wait.
__global__ void __launch_bounds__(kXsThreads, kXsMinCtas) xs_mul_kernel(XsView v, const double* __restrict__ x, double* y,
                                                                        const double* __restrict__ Df, int accumulate,
                                                                        const int* __restrict__ done_flag, double* pq_part) {
  __shared__ double s_pq[kXsWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int e = lane / 9, w = lane - 9 * (lane / 9);   // e == 3: lanes 27..31, no block
  const int gw = blockIdx.x * kXsWarps + warp;
  const int k0 = __ldg(v.warp_step + gw), k1 = __ldg(v.warp_step + gw + 1);
  auto load_s = [&](int2 d, int e, int w, double* s) { xs_step_s(v, d, e, w, s); };
  XsWalk wk;
  xs_walk_begin(v, k0, k1, e, w, load_s, wk);
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (done_flag != nullptr && __ldcg(done_flag) != 0) return;
  auto load_x = [&](int j, int w) { return __ldcg(x + 9 * static_cast<size_t>(j) + w); };
  double pq = xs_walk(
      v, k0, k1, lane, e, w, load_s, load_x, load_x,
      [&](int i, int u, double a, double xo) {
        const size_t o = 9 * static_cast<size_t>(i) + u;
        double out = a;
        if (Df != nullptr) out += Df[o] * Df[o] * xo;
        if (accumulate) out += __ldcg(y + o);
        y[o] = out;
      },
      wk);
  if (pq_part == nullptr) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) pq += __shfl_xor_sync(0xffffffffu, pq, o);
  if (lane == 0) s_pq[warp] = pq;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
#pragma unroll
    for (int ww = 0; ww < kXsWarps; ++ww) tot += s_pq[ww];
    pq_part[blockIdx.x] = tot;
  }
}

// q + entry w of the column part over T slots [c0, c1): sum of t_ij[w] in slot order, i.e. in order of i (a column's
// slots are contiguous), loaded 8 at a time.  src holds slot c at 9 (c - base): T itself (base 0, read with ld.global.cg,
// as the product that wrote it may run in the same launch), or, kStaged, a copy of slots from `base` on in shared memory.
template <bool kStaged>
__device__ __forceinline__ double xs_col_sum(const double* src, int base, int c0, int c1, int w, double q) {
  for (int c = c0; c < c1; c += 8) {
    double t[8];
#pragma unroll
    for (int m = 0; m < 8; ++m) {
      const double* s = src + 9 * static_cast<size_t>(c + m - base) + w;
      t[m] = c + m < c1 ? (kStaged ? *s : __ldcg(s)) : 0.0;
    }
#pragma unroll
    for (int m = 0; m < 8; ++m)
      if (c + m < c1) q += t[m];
  }
  return q;
}
// q + the column part of entry k = 9j + w of S x: sum over the blocks (i, j), i < j, of t_ij[w] in order of i.
__device__ __forceinline__ double xs_col_sum(const int* __restrict__ col_ptr, const double* T, int k, double q) {
  const int j = k / 9, w = k - 9 * (k / 9);
  return xs_col_sum<false>(T, 0, __ldg(col_ptr + j), __ldg(col_ptr + j + 1), w, q);
}

// Completes a product outside the PCG: y += the column part held in T.
__global__ void __launch_bounds__(256) xs_gather_kernel(XsView v, double* y) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < 9 * v.C) y[k] = xs_col_sum(v.col_ptr, v.T, k, y[k]);
}

}  // namespace b200
