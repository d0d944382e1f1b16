// Once-per-LM-iteration kernels on the v4 machinery (kernels_v2.cuh: every operand of a warp tile through the warp's
// TMA slot, the CTA's cameras addressed through its camera list, per-warp private camera vectors, segmented sums by
// shuffles): the implicit-Schur initialisation fused with the per-row 2x2 blocks the camera-major block-diagonal pass
// needs, and that camera-major pass itself.  Together they are the "Schur eliminate" of the metric
// (SchurEliminator<2,3,9>::Eliminate against a block-diagonal lhs, schur_eliminator_impl.h:184-568, plus
// ImplicitSchurComplement::Init / UpdateRhs, implicit_schur_complement.cc:49-97, :251-276).
#pragma once
#include "kernels_v2b.cuh"

namespace b200 {

// (A + D^2)^-1 of a symmetric 3x3 through its Cholesky factor, like invert_sym3_llt (the reference's
// selfadjointView<Upper>().llt().solve(I), implicit_schur_complement.cc:201-202), but with reciprocal square roots only:
// three rsqrt instead of three sqrt + six divisions.  FP64 sqrt / division are ~25-instruction sequences on a pipe that
// issues a warp instruction every ~4.5 cycles: ncu attributed a third of the first version of the init kernel to them.
// rsqrt(double) is accurate to 1-2 ulp, so the result differs from the division form by O(1e-16) relative.
__device__ __forceinline__ void invert_sym3_llt_rsqrt(const double m[6], double inv[6]) {
  const double i00 = rsqrt(m[0]);                 // 1 / l00
  const double l10 = m[1] * i00, l20 = m[2] * i00;
  const double i11 = rsqrt(m[3] - l10 * l10);     // 1 / l11
  const double l21 = (m[4] - l20 * l10) * i11;
  const double i22 = rsqrt(m[5] - l20 * l20 - l21 * l21);
  // L^-1 (lower)
  const double i10 = -l10 * i00 * i11;
  const double i21 = -l21 * i11 * i22;
  const double i20 = -(l20 * i00 + l21 * i10) * i22;
  // inv = L^-T L^-1
  inv[0] = i00 * i00 + i10 * i10 + i20 * i20;
  inv[1] = i10 * i11 + i20 * i21;
  inv[2] = i20 * i22;
  inv[3] = i11 * i11 + i21 * i21;
  inv[4] = i21 * i22;
  inv[5] = i22 * i22;
}

struct InitV4Args {
  const double* b;   // [2N]
  const double* D;   // [3P+9C] or null
  double* ete_inv;   // [6P]
  double* rhs;       // [9C], zeroed by the caller
  double* ye;        // [3P] or null
  double* q3;        // [kQStride N] or null: Q_r = I - E_r (E'E + D^2)^-1 E_r'  (2x2 symmetric: q00, q01, q11, pad) per row
};

// slot: [0,4608) F | [4608,6144) E | [6144,6656) b (16 B per row) | [6656,7440) the tile's slice of D_e (24 B per point, the
// 16-byte-aligned superset) | [7680,7840) descriptor block
__device__ __forceinline__ void init_v4_issue(const V2View& v, const InitV4Args& a, unsigned char* stage, uint64_t* bar, int tile,
                                              int row_begin, int pt_begin, int row_count, int pt_count) {
  const uint32_t xoff = (pt_begin & 1) ? 8u : 0u;
  const uint32_t dbytes = a.D != nullptr ? ((24u * pt_count + xoff + 15u) & ~15u) : 0u;
  mbar_arrive_expect_tx(bar, row_count * 208u + dbytes + kV4MetaWords * 4u);
  bulk_g2s(stage, v.p.F() + 18 * static_cast<size_t>(row_begin), row_count * 144u, bar);
  bulk_g2s(stage + 4608, v.p.E() + 6 * static_cast<size_t>(row_begin), row_count * 48u, bar);
  bulk_g2s(stage + 6144, a.b + 2 * static_cast<size_t>(row_begin), row_count * 16u, bar);
  if (a.D != nullptr)
    bulk_g2s(stage + 6656, reinterpret_cast<const unsigned char*>(a.D + 3 * static_cast<size_t>(pt_begin)) - xoff, dbytes, bar);
  bulk_g2s(stage + 7680, v.tile_meta + static_cast<size_t>(kV4MetaWords) * tile, kV4MetaWords * 4u, bar);
}

template <int K>
__device__ __forceinline__ void seg_suffix_sum(double (&w)[K], int seg_end, int maxlen) {
  const int lane = threadIdx.x & 31;
  for (int d = 1; d < maxlen; d <<= 1) {
    double a[K];
#pragma unroll
    for (int k = 0; k < K; ++k) a[k] = __shfl_down_sync(0xffffffffu, w[k], d);
    if (lane + d < seg_end) {
#pragma unroll
      for (int k = 0; k < K; ++k) w[k] += a[k];
    }
  }
}

// The 33..kTile-row points of the CTA for the implicit-Schur initialisation (staging as in schur_mul_big_points_impl): the
// nine sums of E'E and E'b go through a CTA reduction, every row then finishes like a warp-tile row; the camera part is
// added to replica 0 of the private camera vector with shared-memory atomics.
__device__ __forceinline__ void init_big_points_impl(const V2View& v, const BigStage& st, uint32_t& parity, double* sy_rep0, int2 cr,
                                                     const InitV4Args& a) {
  const int2 br = v.cta_big[blockIdx.x];
  const int tid = threadIdx.x;
  double* sU = st.sU;
  for (int b = br.x; b < br.y; ++b) {
    const TileDesc d = v.big_tiles[b];
    if (tid == 0) {
      mbar_arrive_expect_tx(st.bar, d.obs_count * 192u);
      for (int r0 = 0, k = 0; r0 < d.obs_count; r0 += st.chunk_rows, ++k) {
        const int rows = min(st.chunk_rows, d.obs_count - r0);
        unsigned char* dst = st.base + static_cast<size_t>(k) * st.chunk_stride;
        bulk_g2s(dst, v.p.F() + 18 * static_cast<size_t>(d.obs_begin + r0), rows * 144u, st.bar);
        bulk_g2s(dst + st.chunk_rows * 144, v.p.E() + 6 * static_cast<size_t>(d.obs_begin + r0), rows * 48u, st.bar);
      }
    }
    const bool active = tid < d.obs_count;
    const int chunk = tid / st.chunk_rows, rr = tid - chunk * st.chunk_rows;
    const double* sF = reinterpret_cast<const double*>(st.base + static_cast<size_t>(chunk) * st.chunk_stride) + rr * 18;
    const double* sE = reinterpret_cast<const double*>(st.base + static_cast<size_t>(chunk) * st.chunk_stride + st.chunk_rows * 144) + rr * 6;
    const size_t row = static_cast<size_t>(d.obs_begin) + tid;
    const size_t pt = static_cast<size_t>(d.pt_begin);
    int cam_l = 0;
    double2 bb = make_double2(0, 0);
    if (active) {
      cam_l = meta_local(v, __ldg(v.row_meta + row), cr);
      bb = *reinterpret_cast<const double2*>(a.b + 2 * row);
    }
    double d0 = 0.0, d1 = 0.0, d2 = 0.0;
    if (a.D != nullptr) {
      d0 = __ldg(a.D + 3 * pt);
      d1 = __ldg(a.D + 3 * pt + 1);
      d2 = __ldg(a.D + 3 * pt + 2);
    }
    mbar_wait(st.bar, parity);
    parity ^= 1;
    double f[18];
    double2 e0 = make_double2(0, 0), e1 = e0, e2 = e0;
    double m[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (active) {
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 w = lds2(sF + 2 * k);
        f[2 * k] = w.x;
        f[2 * k + 1] = w.y;
      }
      e0 = lds2(sE);
      e1 = lds2(sE + 2);
      e2 = lds2(sE + 4);
      m[0] = e0.x * e0.x + e1.y * e1.y;
      m[1] = e0.x * e0.y + e1.y * e2.x;
      m[2] = e0.x * e1.x + e1.y * e2.y;
      m[3] = e0.y * e0.y + e2.x * e2.x;
      m[4] = e0.y * e1.x + e2.x * e2.y;
      m[5] = e1.x * e1.x + e2.y * e2.y;
      m[6] = e0.x * bb.x + e1.y * bb.y;
      m[7] = e0.y * bb.x + e2.x * bb.y;
      m[8] = e1.x * bb.x + e2.y * bb.y;
    }
    if (tid < kTile) {  // the first four warps hold all rows
#pragma unroll
      for (int k = 0; k < 9; ++k) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) m[k] += __shfl_xor_sync(0xffffffffu, m[k], o);
      }
      if ((tid & 31) == 0) {
#pragma unroll
        for (int k = 0; k < 9; ++k) sU[(tid >> 5) * 9 + k] = m[k];
      }
    }
    __syncthreads();
    if (active) {
#pragma unroll
      for (int k = 0; k < 9; ++k) m[k] = (sU[k] + sU[9 + k]) + (sU[18 + k] + sU[27 + k]);
      m[0] += d0 * d0;
      m[3] += d1 * d1;
      m[5] += d2 * d2;
      double inv[6];
      invert_sym3_llt_rsqrt(m, inv);
      const double v0 = inv[0] * m[6] + inv[1] * m[7] + inv[2] * m[8];
      const double v1 = inv[1] * m[6] + inv[3] * m[7] + inv[4] * m[8];
      const double v2 = inv[2] * m[6] + inv[4] * m[7] + inv[5] * m[8];
      if (tid == 0) {
#pragma unroll
        for (int k = 0; k < 6; ++k) a.ete_inv[6 * pt + k] = inv[k];
        if (a.ye != nullptr) {
          a.ye[3 * pt] = v0;
          a.ye[3 * pt + 1] = v1;
          a.ye[3 * pt + 2] = v2;
        }
      }
      const double t0 = bb.x - (e0.x * v0 + e0.y * v1 + e1.x * v2);
      const double t1 = bb.y - (e1.y * v0 + e2.x * v1 + e2.y * v2);
      double* yc = sy_rep0 + 9 * cam_l;
#pragma unroll
      for (int k = 0; k < 9; ++k) atomicAdd(yc + k, f[k] * t0 + f[9 + k] * t1);
      if (a.q3 != nullptr) {
        const double pa = inv[0] * e0.x + inv[1] * e0.y + inv[2] * e1.x, pb = inv[1] * e0.x + inv[3] * e0.y + inv[4] * e1.x,
                     pc = inv[2] * e0.x + inv[4] * e0.y + inv[5] * e1.x;
        const double pd = inv[0] * e1.y + inv[1] * e2.x + inv[2] * e2.y, pe = inv[1] * e1.y + inv[3] * e2.x + inv[4] * e2.y,
                     pf = inv[2] * e1.y + inv[4] * e2.x + inv[5] * e2.y;
        double2* q = reinterpret_cast<double2*>(a.q3 + kQStride * row);
        q[0] = make_double2(1.0 - (e0.x * pa + e0.y * pb + e1.x * pc), -(e1.y * pa + e2.x * pb + e2.y * pc));
        q[1] = make_double2(1.0 - (e1.y * pd + e2.x * pe + e2.y * pf), 0.0);
      }
    }
    __syncthreads();  // staging and sU are reused by the next point
  }
}

// ete_inv[k] = (sum_rows E'E + D_k^2)^-1 ; ye = ete_inv E'b ; rhs += F'(b - E ye) ; q3[r] = I - E_r ete_inv E_r'
// Warp tiles and the CTA's 33..kTile-row points; the slices of larger points go through huge_schur_init_kernel and
// row_q_tiles_kernel.
template <bool kOwned>
__global__ void __launch_bounds__(kV4MaxThreads, 1) schur_init_v4_kernel(V2View v, InitV4Args a) {
  const V4Ctx c = v4_ctx(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int2 part = c.part, cr = c.cr;
  v4_init(v, c);
  if (lane == 0) {
    int t = part.x + warp;
    for (int s = 0; s < v.stages && t < part.y; ++s, t += v.warps) {
      const WarpTile wt = v.wtiles[t];
      init_v4_issue(v, a, c.wbase() + s * kV4StageBytes, c.bars() + s, t, wt.row_begin, wt.pt_begin, wt.row_count, wt.pt_count);
    }
  }
  {
    const int n = c.sy_stride * v.replicas;
    for (int i = threadIdx.x; i < n; i += blockDim.x) c.sy()[i] = 0.0;
  }
  __syncthreads();
  double* my_y = c.sy() + (kOwned ? warp : warp % v.replicas) * c.sy_stride;
  const int reissue = v.warps * v.stages;
  int it = 0;
  for (int tile = part.x + warp; tile < part.y; tile += v.warps, ++it) {
    const int s = it % v.stages;
    const uint32_t parity = (it / v.stages) & 1u;
    unsigned char* stage = c.wbase() + s * kV4StageBytes;
    const double* sF = reinterpret_cast<const double*>(stage);
    const double* sE = reinterpret_cast<const double*>(stage + 4608);
    const double* sB = reinterpret_cast<const double*>(stage + 6144);
    const uint32_t* sM = reinterpret_cast<const uint32_t*>(stage + 7680);
    mbar_wait(c.bars() + s, parity);
    const uint4 own = *reinterpret_cast<const uint4*>(sM + 32);
    const uint4 nxt = *reinterpret_cast<const uint4*>(sM + 36);
    const int row_begin = static_cast<int>(own.x), pt_begin = static_cast<int>(own.y);
    const int row_count = static_cast<int>(own.z & 0xffffu);
    const bool active = lane < row_count;
    const uint32_t meta = active ? sM[lane] : 0u;
    const int cam_l = meta_local(v, meta, cr);
    const Seg sg = v2_segment(active && meta_head(meta), row_count);
    double f[18];
    double2 e0 = make_double2(0, 0), e1 = e0, e2 = e0, bb = e0;
    double d0 = 0.0, d1 = 0.0, d2 = 0.0;
    if (active) {
      const double* fr = sF + lane * 18;
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 w = lds2(fr + 2 * k);
        f[2 * k] = w.x;
        f[2 * k + 1] = w.y;
      }
      e0 = lds2(sE + lane * 6);
      e1 = lds2(sE + lane * 6 + 2);
      e2 = lds2(sE + lane * 6 + 4);
      bb = lds2(sB + 2 * lane);
      if (a.D != nullptr) {
        const double* dp = reinterpret_cast<const double*>(stage + 6656 + ((pt_begin & 1) ? 8 : 0)) + 3 * sg.lpt;
        d0 = dp[0];
        d1 = dp[1];
        d2 = dp[2];
      }
    }
    __syncwarp();  // every lane is done with the ring slot
    if (lane == 0 && (nxt.z & 0xffffu) != 0u)
      init_v4_issue(v, a, stage, c.bars() + s, tile + reissue, static_cast<int>(nxt.x), static_cast<int>(nxt.y),
                    static_cast<int>(nxt.z & 0xffffu), static_cast<int>(nxt.z >> 16));
    // E'E (6 unique) and E'b (3) of the row, summed over the rows of its point
    double m[9];
    m[0] = e0.x * e0.x + e1.y * e1.y;
    m[1] = e0.x * e0.y + e1.y * e2.x;
    m[2] = e0.x * e1.x + e1.y * e2.y;
    m[3] = e0.y * e0.y + e2.x * e2.x;
    m[4] = e0.y * e1.x + e2.x * e2.y;
    m[5] = e1.x * e1.x + e2.y * e2.y;
    m[6] = e0.x * bb.x + e1.y * bb.y;
    m[7] = e0.y * bb.x + e2.x * bb.y;
    m[8] = e1.x * bb.x + e2.y * bb.y;
    seg_suffix_sum<9>(m, sg.end, static_cast<int>(own.w));
#pragma unroll
    for (int k = 0; k < 9; ++k) m[k] = __shfl_sync(0xffffffffu, m[k], sg.first);
    double g[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (active) {
      m[0] += d0 * d0;
      m[3] += d1 * d1;
      m[5] += d2 * d2;
      double inv[6];
      invert_sym3_llt_rsqrt(m, inv);   // every lane of the point computes the same inverse
      const double v0 = inv[0] * m[6] + inv[1] * m[7] + inv[2] * m[8];
      const double v1 = inv[1] * m[6] + inv[3] * m[7] + inv[4] * m[8];
      const double v2 = inv[2] * m[6] + inv[4] * m[7] + inv[5] * m[8];
      const size_t pt = static_cast<size_t>(pt_begin + sg.lpt);
      if (lane == sg.first) {
        double2* pi = reinterpret_cast<double2*>(a.ete_inv + 6 * pt);
        pi[0] = make_double2(inv[0], inv[1]);
        pi[1] = make_double2(inv[2], inv[3]);
        pi[2] = make_double2(inv[4], inv[5]);
        if (a.ye != nullptr) {
          a.ye[3 * pt] = v0;
          a.ye[3 * pt + 1] = v1;
          a.ye[3 * pt + 2] = v2;
        }
      }
      const double t0 = bb.x - (e0.x * v0 + e0.y * v1 + e1.x * v2);
      const double t1 = bb.y - (e1.y * v0 + e2.x * v1 + e2.y * v2);
#pragma unroll
      for (int k = 0; k < 9; ++k) g[k] = f[k] * t0 + f[9 + k] * t1;
      if (a.q3 != nullptr) {
        // P e_r' for the two rows of E
        const double pa = inv[0] * e0.x + inv[1] * e0.y + inv[2] * e1.x, pb = inv[1] * e0.x + inv[3] * e0.y + inv[4] * e1.x,
                     pc = inv[2] * e0.x + inv[4] * e0.y + inv[5] * e1.x;
        const double pd = inv[0] * e1.y + inv[1] * e2.x + inv[2] * e2.y, pe = inv[1] * e1.y + inv[3] * e2.x + inv[4] * e2.y,
                     pf = inv[2] * e1.y + inv[4] * e2.x + inv[5] * e2.y;
        double2* q = reinterpret_cast<double2*>(a.q3 + kQStride * (static_cast<size_t>(row_begin) + lane));
        q[0] = make_double2(1.0 - (e0.x * pa + e0.y * pb + e1.x * pc), -(e1.y * pa + e2.x * pb + e2.y * pc));
        q[1] = make_double2(1.0 - (e1.y * pd + e2.x * pe + e2.y * pf), 0.0);
      }
    }
    if (kOwned) cam_accumulate9_owned(my_y, cam_l, active, g);
    else cam_accumulate9(my_y, cam_l, active, g);
  }
  {  // the CTA's 33..kTile-row points (uniform per CTA), processed by the whole CTA
    const int2 br = v.cta_big[blockIdx.x];
    if (br.y > br.x) {
      double* sw0 = reinterpret_cast<double*>(c.ring() + v.stages * kV4StageBytes);
      BigStage st;
      st.base = c.ring();
      st.chunk_rows = kV4BigChunkRows;
      st.chunk_stride = v.per_warp_bytes;
      st.sU = sw0 + 48;   // 4 warps x 9 partial sums
      st.bar = reinterpret_cast<uint64_t*>(c.ring() + v4_extra_offset(v.stages));
      __syncthreads();  // every warp is done with its ring slot
      uint32_t parity = 0;
      init_big_points_impl(v, st, parity, c.sy(), cr, a);
    }
  }
  v2_epilogue(v, c.sy(), cr, a.rhs);
}

// Q_r for the rows of CTA tiles that hold ONE point each (the 33..kTile-row points and the slices of larger ones).
__global__ void __launch_bounds__(kTile) row_q_tiles_kernel(ProblemView p, const double* __restrict__ ete_inv, double* q3) {
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileDesc d = p.tiles[tile];
    if (static_cast<int>(threadIdx.x) >= d.obs_count) continue;
    const size_t r = static_cast<size_t>(d.obs_begin) + threadIdx.x;
    const double2* ep = reinterpret_cast<const double2*>(p.E() + 6 * r);
    const double2 a0 = __ldg(ep), a1 = __ldg(ep + 1), a2 = __ldg(ep + 2);
    const double e00 = a0.x, e01 = a0.y, e02 = a1.x, e10 = a1.y, e11 = a2.x, e12 = a2.y;
    const double* pi = ete_inv + 6 * static_cast<size_t>(d.pt_begin);
    const double p0 = __ldg(pi), p1 = __ldg(pi + 1), p2 = __ldg(pi + 2), p3 = __ldg(pi + 3), p4 = __ldg(pi + 4), p5 = __ldg(pi + 5);
    const double a = p0 * e00 + p1 * e01 + p2 * e02, b = p1 * e00 + p3 * e01 + p4 * e02, c = p2 * e00 + p4 * e01 + p5 * e02;
    const double dd = p0 * e10 + p1 * e11 + p2 * e12, e = p1 * e10 + p3 * e11 + p4 * e12, f = p2 * e10 + p4 * e11 + p5 * e12;
    double2* q = reinterpret_cast<double2*>(q3 + kQStride * r);
    q[0] = make_double2(1.0 - (e00 * a + e01 * b + e02 * c), -(e10 * a + e11 * b + e12 * c));
    q[1] = make_double2(1.0 - (e10 * dd + e11 * e + e12 * f), 0.0);
  }
}

// ------------------------------------------------------------------------------------------------
// Camera-major block diagonal, second version (cam_blocks_kernel of kernels_v2b.cuh: ncu showed 8 resident warps per SM at
// 162 registers, 43 % long-scoreboard stalls, and 450 shuffles per item for the final reduction).  One warp per item (a
// slice of one camera's row list), 4-warp CTAs (three per SM at ~165 registers: 12 resident warps keep more loads in
// flight than one 8-warp CTA did); the 45 packed entries are reduced across the lanes by recursive halving (each lane ends with <= 2 entries: 46 64-bit exchanges
// instead of 225) and added with <= 2 REDs per lane.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(kPending) : "memory"); }

constexpr int kCamBlkRowBytes = 144 + 32;                 // F row + Q block (q00, q01, q11, pad)
constexpr int kCamBlkDepth = 2;                           // buffers per warp: the next 32 rows land while 32 are computed
constexpr int kCamBlkWarpBytes = kCamBlkDepth * 32 * kCamBlkRowBytes;
constexpr int kCamBlkThreads = 128;

// Sum of the 46 (zero padded) per-lane entries over the lanes by recursive halving: 46 -> 23 -> 12 -> 6 -> 3 -> 2 entries per
// lane (46 64-bit exchanges instead of 45 x 5), then <= 2 REDs per lane into the camera's packed block.
__device__ __forceinline__ void cam_block_flush(double (&m)[46], double* dst) {
  const int lane = threadIdx.x & 31;
  int base = 0;
  double r1[23], r2[12], r3[6], r4[3], r5[2];
  {
    const bool up = (lane & 16) != 0;
#pragma unroll
    for (int k = 0; k < 23; ++k) {
      const double keep = up ? m[23 + k] : m[k], give = up ? m[k] : m[23 + k];
      r1[k] = keep + __shfl_xor_sync(0xffffffffu, give, 16);
    }
    base += up ? 23 : 0;
  }
  {
    const bool up = (lane & 8) != 0;
#pragma unroll
    for (int k = 0; k < 12; ++k) {
      const double hi = (12 + k < 23) ? r1[(12 + k < 23) ? 12 + k : 0] : 0.0;
      const double keep = up ? hi : r1[k], give = up ? r1[k] : hi;
      r2[k] = keep + __shfl_xor_sync(0xffffffffu, give, 8);
    }
    base += up ? 12 : 0;
  }
  {
    const bool up = (lane & 4) != 0;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      const double keep = up ? r2[6 + k] : r2[k], give = up ? r2[k] : r2[6 + k];
      r3[k] = keep + __shfl_xor_sync(0xffffffffu, give, 4);
    }
    base += up ? 6 : 0;
  }
  {
    const bool up = (lane & 2) != 0;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const double keep = up ? r3[3 + k] : r3[k], give = up ? r3[k] : r3[3 + k];
      r4[k] = keep + __shfl_xor_sync(0xffffffffu, give, 2);
    }
    base += up ? 3 : 0;
  }
  {
    const bool up = (lane & 1) != 0;
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const double hi = (k == 0) ? r4[2] : 0.0;
      const double keep = up ? hi : r4[k], give = up ? r4[k] : hi;
      r5[k] = keep + __shfl_xor_sync(0xffffffffu, give, 1);
    }
    base += up ? 2 : 0;
  }
#pragma unroll
  for (int k = 0; k < 2; ++k)
    if (r5[k] != 0.0) red_add(dst + base + k, r5[k]);   // padding entries are exactly zero and never reach an index >= 45
}

// Camera-major block diagonal.  One warp per item (a slice of one camera's row list, the reference's transpose block
// structure, block_sparse_matrix.cc:784-808); each lane copies ITS (gathered) row of the next 32 rows into the warp's
// shared-memory buffer with cp.async while the warp computes on the previous 32; the 45 packed entries stay in registers per
// lane and are reduced across the lanes when the item ends.  The kernel is bound by the DRAM access pattern of 144-byte
// gathers, not by latency; register-only, one continuous cp.async stream across items, and CTA-local streaming with the
// regrouping by camera done in shared memory (FP64-issue-bound) were slower and are not in the build.
template <bool kSchur>
__global__ void __launch_bounds__(kCamBlkThreads, 3)
    cam_blocks_v2_kernel(ProblemView p, int num_items, const CamItem* __restrict__ items, const int* __restrict__ cam_rows,
                         const double* __restrict__ q3, double* out45) {
  extern __shared__ __align__(128) unsigned char cb_smem[];
  const int lane = threadIdx.x & 31;
  const int warps_per_block = blockDim.x >> 5;
  unsigned char* wbuf = cb_smem + (threadIdx.x >> 5) * kCamBlkWarpBytes;
  for (int item = blockIdx.x * warps_per_block + (threadIdx.x >> 5); item < num_items; item += gridDim.x * warps_per_block) {
    const CamItem it = items[item];
    double m[46];
#pragma unroll
    for (int k = 0; k < 46; ++k) m[k] = 0.0;
    const int iters = (it.end - it.begin + 31) >> 5;
    auto row_of = [&](int iter) -> int {
      const int j = it.begin + 32 * iter + lane;
      return (iter < iters && j < it.end) ? __ldg(cam_rows + j) : -1;
    };
    // Two adjacent lanes fetch ONE row together, 32 bytes per step: a row is 144 B = 4.5 sectors, and with each lane on its
    // own row every 16-byte cp.async was a separate half-empty sector request to L2 (11 requests per row, counting Q);
    // paired on sector boundaries it takes 6 (rows start at 144 r: the pairs of row r begin at chunk r & 1).
    auto issue = [&](int r, int buf) {
      unsigned char* fbuf = wbuf + buf * 32 * kCamBlkRowBytes;
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int slot = 16 * half + (lane >> 1);                    // row slot served by this lane pair
        const int rr = __shfl_sync(0xffffffffu, r, slot);             // its row (held by lane `slot`)
        if (rr >= 0) {
          const unsigned char* src = reinterpret_cast<const unsigned char*>(p.F() + 18 * static_cast<size_t>(rr));
          unsigned char* dst = fbuf + slot * 144;
          const int first = (lane & 1) - (rr & 1);                   // chunk of this lane in step 0: -1, 0 or 1
#pragma unroll
          for (int c = 0; c < 5; ++c) {
            const int chunk = 2 * c + first;
            if (chunk >= 0 && chunk <= 8) cp_async16(dst + 16 * chunk, src + 16 * chunk);
          }
          if (kSchur) cp_async16(fbuf + 32 * 144 + slot * 32 + 16 * (lane & 1), q3 + kQStride * static_cast<size_t>(rr) + 2 * (lane & 1));
        }
      }
      cp_async_commit();
    };
    int r_cur = row_of(0), r_nxt = row_of(1);
    issue(r_cur, 0);
    for (int i = 0; i < iters; ++i) {
      const int r_nn = row_of(i + 2);
      issue(r_nxt, (i + 1) & 1);
      cp_async_wait<1>();
      __syncwarp();
      if (r_cur >= 0) {
        const double* fr = reinterpret_cast<const double*>(wbuf + (i & 1) * 32 * kCamBlkRowBytes + lane * 144);
        double f[18];
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          const double2 w = lds2(fr + 2 * k);
          f[2 * k] = w.x;
          f[2 * k + 1] = w.y;
        }
        double q00 = 1.0, q01 = 0.0, q11 = 1.0;
        if (kSchur) {
          const double* q = reinterpret_cast<const double*>(wbuf + (i & 1) * 32 * kCamBlkRowBytes + 32 * 144 + lane * 32);
          q00 = q[0];
          q01 = q[1];
          q11 = q[2];
        }
        int idx = 0;
#pragma unroll
        for (int aa = 0; aa < 9; ++aa) {
          const double ga = q00 * f[aa] + q01 * f[9 + aa], gb = q01 * f[aa] + q11 * f[9 + aa];   // row aa of F'Q
#pragma unroll
          for (int bb = aa; bb < 9; ++bb) {
            m[idx] += ga * f[bb] + gb * f[9 + bb];
            ++idx;
          }
        }
      }
      __syncwarp();   // the buffer is refilled two iterations later
      r_cur = r_nxt;
      r_nxt = r_nn;
    }
    cp_async_wait<0>();
    cam_block_flush(m, out45 + 45 * static_cast<size_t>(it.cam));
  }
}

}  // namespace b200
