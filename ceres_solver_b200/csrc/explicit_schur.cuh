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
// Product.  Each output camera i owns y_i = sum_{j >= i} S_ij x_j + sum_{j < i} S_ji' x_j: a pair of warps walks the list
// of block row i followed by the blocks of column i above the diagonal (each off-diagonal block is read twice, from a
// footprint that is half of the full matrix), accumulates with fixed order and writes y_i once.
#pragma once
#include "common.cuh"

namespace b200 {

constexpr int kXsThreads = 256;       // product: 8 warps per CTA
constexpr int kXsWarps = kXsThreads / 32;
constexpr int kXsSplit = 2;           // warps per output camera
constexpr int kXsGroups = kXsWarps / kXsSplit;   // groups of kXsSplit warps per CTA, each owning a contiguous camera range
constexpr int kXsBatch = 4;           // blocks in flight per warp in the product
constexpr int kXsAsmThreads = 256;    // assembly: one warp per block, or one CTA per block with a long pair list
constexpr int kXsLongPairs = 96;      // ... longer than this
constexpr uint32_t kXsTransposed = 0x80000000u;

struct XsView {
  int C;
  int num_blocks;
  const int* blk_row;        // [num_blocks] i of block (i, j)
  const int* blk_col;        // [num_blocks] j
  const int* pair_ptr;       // [num_blocks + 1] row pairs of each block
  const int2* pairs;         // (r, s): cam r = i, cam s = j, same point
  const int* list_ptr;       // [C + 1] product list of output camera i
  const int2* list;          // {block, j | kXsTransposed when the block is (j, i), j < i}
  const int* warp_cam;       // [groups + 1] first output camera of each product warp group
  double* S;                 // [num_blocks][81]
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

// y = [y if accumulate] + [D_f^2 x if Df] + S x, S as assembled (without D_f^2).  Inside the PCG: accumulate onto the
// output the vector kernel seeded, no-op once done_flag is set, and pq_part[CTA] = x . (this CTA's rows of S x) -- the
// product protocol of schur_mul_v4_kernel.  Launched with programmatic stream serialisation behind the vector kernel.
// kXsSplit warps share each output camera (alternate batches of its list) and add their sums in warp order.
__global__ void __launch_bounds__(kXsThreads, 3) xs_mul_kernel(XsView v, const double* __restrict__ x, double* y,
                                                               const double* __restrict__ Df, int accumulate,
                                                               const int* __restrict__ done_flag, double* pq_part) {
  __shared__ double s_acc[kXsWarps][2][81];
  __shared__ double s_pq[kXsWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int grp = warp / kXsSplit, h = warp - kXsSplit * grp;
  const int gid = blockIdx.x * kXsGroups + grp;
  // static data first: it may be read before the kernel that produces x has finished
  const int c0 = __ldg(v.warp_cam + gid), c1 = __ldg(v.warp_cam + gid + 1);
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (done_flag != nullptr && __ldcg(done_flag) != 0) return;
  // lane entries k = lane + 32 m of a block: row u_m, column w_m (m = 2 only for lanes < 17)
  const bool ok2 = lane < 17;
  int um[3], wm[3];
#pragma unroll
  for (int m = 0; m < 3; ++m) {
    const int k = (m < 2 || ok2) ? lane + 32 * m : 0;
    um[m] = k / 9;
    wm[m] = k - 9 * (k / 9);
  }
  double pq = 0.0;
  for (int i = c0; i < c1; ++i) {
    double a[3] = {0.0, 0.0, 0.0};   // sum over blocks (i, j) of S_ij[u][w] x_j[w]  -> y_i[u]
    double t[3] = {0.0, 0.0, 0.0};   // sum over blocks (j, i) of S_ji[u][w] x_j[u]  -> y_i[w]
    const int l0 = __ldg(v.list_ptr + i), l1 = __ldg(v.list_ptr + i + 1);
    for (int l = l0 + h * kXsBatch; l < l1; l += kXsBatch * kXsSplit) {
      double sv[kXsBatch][3], xv[kXsBatch][3];
      unsigned tr = 0u;   // bit e: entry e is a transposed block
#pragma unroll
      for (int e = 0; e < kXsBatch; ++e) {
        const bool ok = l + e < l1;
        const int2 ent = ok ? __ldg(v.list + l + e) : make_int2(0, 0);
        const bool te = (static_cast<uint32_t>(ent.y) & kXsTransposed) != 0;
        tr |= te ? 1u << e : 0u;
        const int j = static_cast<int>(static_cast<uint32_t>(ent.y) & ~kXsTransposed);
        const double* sb = v.S + 81 * static_cast<size_t>(ent.x);
        const double* xj = x + 9 * static_cast<size_t>(j);
#pragma unroll
        for (int m = 0; m < 3; ++m) {
          const bool use = ok && (m < 2 || ok2);
          sv[e][m] = use ? __ldg(sb + lane + 32 * m) : 0.0;
          xv[e][m] = use ? __ldcg(xj + (te ? um[m] : wm[m])) : 0.0;
        }
      }
#pragma unroll
      for (int e = 0; e < kXsBatch; ++e)
#pragma unroll
        for (int m = 0; m < 3; ++m) {
          const double prod = sv[e][m] * xv[e][m];
          if ((tr >> e) & 1u) t[m] += prod;
          else a[m] += prod;
        }
    }
#pragma unroll
    for (int m = 0; m < 3; ++m)
      if (m < 2 || ok2) {
        s_acc[warp][0][lane + 32 * m] = a[m];
        s_acc[warp][1][lane + 32 * m] = t[m];
      }
    // the warps of the group meet on a named barrier (id 1 + group; 0 is __syncthreads)
    asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "r"(32 * kXsSplit) : "memory");
    if (h == 0 && lane < 9) {
      double acc = 0.0;
#pragma unroll
      for (int hh = 0; hh < kXsSplit; ++hh) {
        const double(*sa)[81] = s_acc[kXsSplit * grp + hh];
#pragma unroll
        for (int w = 0; w < 9; ++w) acc += sa[0][9 * lane + w];
#pragma unroll
        for (int uu = 0; uu < 9; ++uu) acc += sa[1][9 * uu + lane];
      }
      const size_t o = 9 * static_cast<size_t>(i) + lane;
      const double xo = __ldcg(x + o);
      pq += xo * acc;
      double out = acc;
      if (Df != nullptr) out += Df[o] * Df[o] * xo;
      if (accumulate) out += __ldcg(y + o);
      y[o] = out;
    }
    asm volatile("bar.sync %0, %1;" ::"r"(1 + grp), "r"(32 * kXsSplit) : "memory");
  }
  if (pq_part == nullptr) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) pq += __shfl_xor_sync(0xffffffffu, pq, o);
  if (lane == 0) s_pq[warp] = pq;
  __syncthreads();
  if (threadIdx.x == 0) {
    double tot = 0.0;
#pragma unroll
    for (int w = 0; w < kXsWarps; ++w) tot += s_pq[w];
    pq_part[blockIdx.x] = tot;
  }
}

}  // namespace b200
