// Warp-tile kernels (v2): the camera-scatter kernels built around three properties of the memory system:
//   * FP64 global REDs have a chip-wide rate limit regardless of locality -> 9 REDs per row make S*x RED-bound far
//     below the HBM roofline;
//   * FP64 atomics on SHARED memory (ATOMS.CAST.SPIN.64) sustain several times that rate;
//   * a TMA bulk-copy ring streams HBM close to its peak.
// So: one persistent CTA per SM keeps a PRIVATE copy of the camera-sized output in shared memory, rows are
// processed in warp-sized tiles (whole points, <= 32 rows) so that the per-point reduction needs only
// __syncwarp (no CTA barrier anywhere in the main loop), every warp runs its own TMA ring for the 2x9 F
// cells (E cells are read straight from global: a warp's 32 cells are one contiguous 1.5 KB run), and the
// per-CTA partial vectors are summed in a fixed order by a tiny second kernel (no global atomics at all).
#pragma once
#include "common.cuh"

namespace b200 {

struct WarpTile {
  int row_begin;
  int pt_begin;
  unsigned short row_count;  // <= 32
  unsigned short pt_count;   // <= 32, every point has >= 1 row
};

struct V2View {
  ProblemView p;
  const WarpTile* wtiles;
  const uint32_t* row_meta;  // [N] camera (bits 0..19) | index of the camera in the CTA's camera list (bits 20..30, direct mode)
                             //     | (first row of its point ? 1u << 31 : 0)
  const int2* cta_part;      // per CTA: [tile_begin, tile_end)
  const int2* cta_cam;       // per CTA, direct mode: {offset into cta_cams, number of distinct cameras its tiles touch};
                             //          otherwise: [cam_lo, cam_hi) touched by its tiles
  const int* cta_cams;       // direct mode: the CTAs' sorted camera lists, concatenated
  const int2* cta_big;       // per CTA: [begin, end) into big_tiles: the >32-row points inside its row range
  const TileDesc* big_tiles; // one point each, 33..kTile rows
  const uint32_t* tile_meta; // v4: [num tiles][kV4MetaWords] row words + own descriptor + descriptor of the tile that reuses the stage
  double* partials;         // [num_ctas][9 * max_cam_span]
  int num_ctas;
  int max_cam_span;
  int warps;                 // warps per CTA
  int stages;                // TMA ring depth per warp
  int replicas;              // copies of the private camera vector (warp w uses copy w % replicas)
  int direct;                // 1: CTAs RED their (narrow) camera range straight into the output vector; 0: partials
  int per_warp_bytes;
  // L2 residency plan of S*x (b200_create), the same for every CTA: a fraction l2_stream / 65536 of its tiles, spread
  // evenly over its tile range, is copied with evict_first; the rest with evict_normal (evict_last if l2_last, development
  // builds), so that it stays in L2 from one product of a PCG to the next.  0: every copy evict_normal, the default policy.
  uint32_t l2_stream;
  int l2_last;
};

// L2 policy of the bulk copies of entry i of a CTA's tile range under the residency plan: entry i is streamed when
// floor((i + 1) s) != floor(i s) with s = l2_stream / 65536.  Created per copy instead of once per thread:
// schur_mul_v4_kernel sits at the 128-register limit of 16 warps per SM.
__device__ __forceinline__ uint64_t v4_l2_policy(const V2View& v, int i) {
  const uint64_t s = v.l2_stream, k = static_cast<uint64_t>(i);
  if (((k + 1) * s >> 16) != (k * s >> 16)) return l2_policy_evict_first();
  return v.l2_last ? l2_policy_evict_last() : l2_policy_evict_normal();
}

// Row word accessors.  A CTA addresses its cameras by their position in its own camera list (direct mode: the list is
// short, the private camera vectors live in shared memory and are flushed with REDs), or by the offset inside its camera
// id range (no camera locality: per-CTA partial vectors, cam_reduce_kernel).
constexpr uint32_t kMetaCamMask = 0xfffffu;   // camera ids below 2^20 on this path
constexpr int kMetaLocalShift = 20;
constexpr uint32_t kMetaLocalMask = 0x7ffu;   // at most 2047 cameras per CTA in direct mode
__device__ __forceinline__ int meta_cam(uint32_t meta) { return static_cast<int>(meta & kMetaCamMask); }
__device__ __forceinline__ bool meta_head(uint32_t meta) { return (meta & 0x80000000u) != 0u; }
__device__ __forceinline__ int meta_local(const V2View& v, uint32_t meta, int2 cr) {
  return v.direct ? static_cast<int>((meta >> kMetaLocalShift) & kMetaLocalMask) : meta_cam(meta) - cr.x;
}
__device__ __forceinline__ int v2_span(const V2View& v, int2 cr) { return v.direct ? cr.y : cr.y - cr.x; }
// index into a camera-major global array with `per_cam` doubles per camera of entry i of the CTA's private array
__device__ __forceinline__ size_t v2_global_entry(const V2View& v, int2 cr, int i, int per_cam) {
  if (!v.direct) return static_cast<size_t>(per_cam) * cr.x + i;
  const int c = i / per_cam;
  return static_cast<size_t>(per_cam) * __ldg(v.cta_cams + cr.x + c) + (i - c * per_cam);
}

constexpr int kV2MaxThreads = 384;
constexpr int kV2Scratch = 3;  // doubles of per-lane exchange scratch in every v2 kernel

__host__ __device__ inline int v2_per_warp_bytes(int stages, int scratch_doubles_per_lane) {
  return (stages * 32 * 144 + 32 * scratch_doubles_per_lane * 8 + 8 * stages + 15) & ~15;
}
__host__ __device__ inline size_t v2_sy_stride(int max_cam_span) {  // doubles per replica
  return (static_cast<size_t>(9) * max_cam_span + 15) & ~static_cast<size_t>(15);
}
__host__ __device__ inline size_t v2_sy_bytes(int max_cam_span, int replicas) {
  return v2_sy_stride(max_cam_span) * 8 * replicas;
}

// Per-warp context: F ring, scratch, barriers.
struct WarpCtx {
  double* sF;
  double* sW;
  uint64_t* bars;
};

__device__ __forceinline__ WarpCtx v2_warp_ctx(const V2View& v, unsigned char* smem, int scratch_per_lane) {
  const int warp = threadIdx.x >> 5;
  unsigned char* base = smem + v2_sy_bytes(v.max_cam_span, v.replicas) + static_cast<size_t>(warp) * v.per_warp_bytes;
  WarpCtx c;
  c.sF = reinterpret_cast<double*>(base);
  c.sW = c.sF + v.stages * 576;
  c.bars = reinterpret_cast<uint64_t*>(c.sW + 32 * scratch_per_lane);
  return c;
}

__device__ __forceinline__ void v2_issue(const V2View& v, const WarpCtx& c, int tile, int stage) {
  const WarpTile wt = v.wtiles[tile];
  const uint32_t bytes = wt.row_count * 144u;
  mbar_arrive_expect_tx(c.bars + stage, bytes);
  bulk_g2s(c.sF + stage * 576, v.p.F() + 18 * static_cast<size_t>(wt.row_begin), bytes, c.bars + stage);
}

// Segment bookkeeping inside a warp tile from the per-row head flags.
struct Seg {
  int first;     // first lane of my point
  int end;       // one past the last lane of my point
  int lpt;       // index of my point inside the tile
};
__device__ __forceinline__ Seg v2_segment(bool head, int row_count) {
  const int lane = threadIdx.x & 31;
  const unsigned heads = __ballot_sync(0xffffffffu, head);
  const unsigned le = heads & (0xffffffffu >> (31 - lane));
  const unsigned gt = (lane == 31) ? 0u : (heads & (0xffffffffu << (lane + 1)));
  Seg s;
  s.first = 31 - __clz(le | 1u);
  s.end = gt ? (__ffs(gt) - 1) : row_count;
  s.lpt = __popc(le) - 1;
  return s;
}

// Common prologue: zero the private camera vector, arm the barriers, prime the TMA ring.
__device__ __forceinline__ void v2_prologue(const V2View& v, double* sy, const WarpCtx& c, int2 part, int2 cr,
                                            int& t_issue) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  (void)cr;
  const int n = static_cast<int>(v2_sy_stride(v.max_cam_span)) * v.replicas;
  for (int i = threadIdx.x; i < n; i += blockDim.x) sy[i] = 0.0;
  if (lane == 0) {
    for (int s = 0; s < v.stages; ++s) mbar_init(c.bars + s, 1);
    fence_mbar_init();
  }
  __syncthreads();
  t_issue = part.x + warp;
  if (lane == 0) {
    for (int s = 0; s < v.stages && t_issue < part.y; ++s) {
      v2_issue(v, c, t_issue, s);
      t_issue += v.warps;
    }
  } else {
    for (int s = 0; s < v.stages && t_issue < part.y; ++s) t_issue += v.warps;
  }
}

// Flush of the CTA-private camera vector.  With camera locality a CTA touches a few dozen cameras, so it adds its
// range straight into the (pre-seeded) output with a few hundred REDs; otherwise (every CTA touches every camera)
// it writes a partial vector that cam_reduce_kernel sums in a fixed order.
__device__ __forceinline__ void v2_epilogue(const V2View& v, const double* sy, int2 cr, double* y_direct) {
  __syncthreads();
  const int n = 9 * v2_span(v, cr);
  const int stride = static_cast<int>(v2_sy_stride(v.max_cam_span));
  double* dst = v.partials + static_cast<size_t>(blockIdx.x) * 9 * v.max_cam_span;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double acc = sy[i];
    for (int r = 1; r < v.replicas; ++r) acc += sy[r * stride + i];
    if (v.direct) {
      if (acc != 0.0) red_add(y_direct + v2_global_entry(v, cr, i, 9), acc);
    } else {
      dst[i] = acc;
    }
  }
}

// Accumulate one 9-vector per row into the CTA-private camera vector.
//  1. rows of the warp that hit the same camera are summed through shuffles first (binary tree over the rank inside
//     each __match_any group): with the camera locality of real captures a warp tile touches a handful of cameras,
//     and un-aggregated lanes would fight over the same shared-memory words;
//  2. the group leaders add into replica `rep` of the vector (one replica per warp when shared memory allows, so
//     different warps never collide) with shared-memory FP64 atomics (ATOMS.CAST.SPIN.64).
__device__ __forceinline__ void cam_accumulate9(double* sy_rep, int cam_local, bool active, double (&g)[9]) {
  const int lane = threadIdx.x & 31;
  const int key = active ? cam_local : (0x40000000 | lane);
  const unsigned m = __match_any_sync(0xffffffffu, key);
  // Linked list of the lanes that share my camera (ascending lane order); pointer jumping turns it into a suffix
  // sum in ceil(log2(group size)) rounds, after which the first lane of every group holds the group total.
  const unsigned above = (lane == 31) ? 0u : (m & (0xfffffffeu << lane));
  int nxt = above ? (__ffs(above) - 1) : -1;
  while (__any_sync(0xffffffffu, nxt >= 0)) {
    const int src = nxt >= 0 ? nxt : lane;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const double v = __shfl_sync(0xffffffffu, g[k], src);
      g[k] += (nxt >= 0) ? v : 0.0;
    }
    nxt = __shfl_sync(0xffffffffu, nxt, src);
    nxt = (src == lane) ? -1 : nxt;
  }
  if (active && (m & ((1u << lane) - 1u)) == 0u) {  // first lane of its group
    double* yc = sy_rep + 9 * cam_local;
#pragma unroll
    for (int k = 0; k < 9; ++k) atomicAdd(yc + k, g[k]);
  }
}

// ------------------------------------------------------------------------------------------------
// partial_y(camera part) = F'(F x - E (E'E+D^2)^-1 E'F x)     x: [9C]   -- the product for problems WITHOUT camera
// locality (every CTA touches cameras all over the index range: per-CTA partial vectors + cam_reduce_kernel).
// F cells through the per-warp TMA ring; nothing is carried in registers from one tile to the next (the E cells, row
// words and (E'E)^-1 of the NEXT tile are only pulled towards L2 with prefetch.global.L2, one 128-byte line per lane),
// which keeps the kernel under 128 registers so that 16 warps per SM are resident.
// ------------------------------------------------------------------------------------------------
// The few points with 33..kTile rows that fall inside this CTA's row range: processed by the whole CTA after the
// warp tiles (the warps' TMA rings are idle by then and provide the staging memory), one point at a time:
// u = sum_rows E'(F x) through a CTA reduction, then the same update as the warp path, accumulated into the
// CTA-private camera vector.  Every thread of the CTA must call this (it contains CTA barriers).
// x of a row's camera is read from the global vector (x_staged = false) or from the CTA's staged copy of its cameras.
// Staging layout: rows are staged in chunks of `chunk_rows`; chunk k lives at base + k * chunk_stride as
// [chunk_rows x 18 F][chunk_rows x 6 E].  sU: 16 doubles of scratch, bar: an INITIALISED mbarrier whose current phase
// parity is *parity_io (updated on return; only thread 0's copy matters to the caller).
struct BigStage {
  unsigned char* base;
  int chunk_rows;
  int chunk_stride;
  double* sU;
  uint64_t* bar;
};

__device__ __forceinline__ void schur_mul_big_points_impl(const V2View& v, const BigStage& st, uint32_t& parity, double* sy_rep0,
                                                          int2 cr, const double* __restrict__ ete_inv, const double* xbase,
                                                          bool x_staged) {
  const int2 br = v.cta_big[blockIdx.x];
  const int tid = threadIdx.x;
  double* sU = st.sU;
  for (int b = br.x; b < br.y; ++b) {
    const TileDesc d = v.big_tiles[b];
    if (tid == 0) {
      const uint64_t pol = v4_l2_policy(v, b - br.x);
      mbar_arrive_expect_tx(st.bar, d.obs_count * 192u);
      for (int r0 = 0, k = 0; r0 < d.obs_count; r0 += st.chunk_rows, ++k) {
        const int rows = min(st.chunk_rows, d.obs_count - r0);
        unsigned char* dst = st.base + static_cast<size_t>(k) * st.chunk_stride;
        bulk_g2s(dst, v.p.F() + 18 * static_cast<size_t>(d.obs_begin + r0), rows * 144u, st.bar, pol);
        bulk_g2s(dst + st.chunk_rows * 144, v.p.E() + 6 * static_cast<size_t>(d.obs_begin + r0), rows * 48u, st.bar, pol);
      }
    }
    const bool active = tid < d.obs_count;
    const int chunk = tid / st.chunk_rows, rr = tid - chunk * st.chunk_rows;
    const double* sF = reinterpret_cast<const double*>(st.base + static_cast<size_t>(chunk) * st.chunk_stride) + rr * 18;
    const double* sE = reinterpret_cast<const double*>(st.base + static_cast<size_t>(chunk) * st.chunk_stride + st.chunk_rows * 144) + rr * 6;
    int cam_l = 0;
    double xc[9];
    double p0 = 0.0, p1 = 0.0, p2 = 0.0, p3 = 0.0, p4 = 0.0, p5 = 0.0;
    if (active) {  // everything that does not come through the bulk copy is requested while it is in flight
      const uint32_t meta = __ldg(v.row_meta + d.obs_begin + tid);
      cam_l = meta_local(v, meta, cr);
      const double* pi = ete_inv + 6 * static_cast<size_t>(d.pt_begin);
      p0 = __ldg(pi), p1 = __ldg(pi + 1), p2 = __ldg(pi + 2), p3 = __ldg(pi + 3), p4 = __ldg(pi + 4), p5 = __ldg(pi + 5);
      const double* xcp = xbase + 9 * static_cast<size_t>(x_staged ? cam_l : meta_cam(meta));
#pragma unroll
      for (int k = 0; k < 9; ++k) xc[k] = xcp[k];
    }
    mbar_wait(st.bar, parity);
    parity ^= 1;
    double t0 = 0.0, t1 = 0.0, w0 = 0.0, w1 = 0.0, w2 = 0.0;
    double f[18];
    double2 e0 = make_double2(0, 0), e1 = e0, e2 = e0;
    if (active) {
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 a = lds2(sF + 2 * k);
        f[2 * k] = a.x;
        f[2 * k + 1] = a.y;
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        t0 += f[k] * xc[k];
        t1 += f[9 + k] * xc[k];
      }
      e0 = lds2(sE);
      e1 = lds2(sE + 2);
      e2 = lds2(sE + 4);
      w0 = e0.x * t0 + e1.y * t1;
      w1 = e0.y * t0 + e2.x * t1;
      w2 = e1.x * t0 + e2.y * t1;
    }
    if (tid < kTile) {  // the first four warps hold all rows
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        w0 += __shfl_xor_sync(0xffffffffu, w0, o);
        w1 += __shfl_xor_sync(0xffffffffu, w1, o);
        w2 += __shfl_xor_sync(0xffffffffu, w2, o);
      }
      if ((tid & 31) == 0) {
        sU[(tid >> 5) * 3 + 0] = w0;
        sU[(tid >> 5) * 3 + 1] = w1;
        sU[(tid >> 5) * 3 + 2] = w2;
      }
    }
    __syncthreads();
    if (active) {
      const double u0 = sU[0] + sU[3] + sU[6] + sU[9], u1 = sU[1] + sU[4] + sU[7] + sU[10], u2 = sU[2] + sU[5] + sU[8] + sU[11];
      const double v0 = -(p0 * u0 + p1 * u1 + p2 * u2);
      const double v1 = -(p1 * u0 + p3 * u1 + p4 * u2);
      const double v2 = -(p2 * u0 + p4 * u1 + p5 * u2);
      t0 += e0.x * v0 + e0.y * v1 + e1.x * v2;
      t1 += e1.y * v0 + e2.x * v1 + e2.y * v2;
      double* yc = sy_rep0 + 9 * cam_l;
#pragma unroll
      for (int k = 0; k < 9; ++k) atomicAdd(yc + k, f[k] * t0 + f[9 + k] * t1);
    }
    __syncthreads();  // staging and sU are reused by the next point
  }
}

// v2/v3 layout: the (idle) ring is used as one contiguous staging area; the kernel ends afterwards, so overwriting the
// warps' barriers is harmless.
__device__ __forceinline__ void schur_mul_big_points(const V2View& v, unsigned char* ring, double* sy_rep0, int2 cr,
                                                     const double* __restrict__ ete_inv, const double* xbase, bool x_staged) {
  const int2 br = v.cta_big[blockIdx.x];
  if (br.y <= br.x) return;  // uniform per CTA
  BigStage st;
  st.base = ring;
  st.chunk_rows = kTile;
  st.chunk_stride = kTile * 192;
  st.sU = reinterpret_cast<double*>(ring + kTile * 192);
  st.bar = reinterpret_cast<uint64_t*>(st.sU + 16);
  __syncthreads();
  if (threadIdx.x == 0) {
    mbar_init(st.bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
  uint32_t parity = 0;
  schur_mul_big_points_impl(v, st, parity, sy_rep0, cr, ete_inv, xbase, x_staged);
}

constexpr int kV3MaxThreads = 512;

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

__global__ void __launch_bounds__(kV3MaxThreads, 1)
    schur_mul_v3_kernel(V2View v, const double* __restrict__ ete_inv, const double* __restrict__ x, double* y,
                        const int* __restrict__ done_flag) {
  if (done_flag != nullptr && *done_flag != 0) return;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  double* sy = reinterpret_cast<double*>(smem_raw);
  const WarpCtx c = v2_warp_ctx(v, smem_raw, kV2Scratch);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int2 part = v.cta_part[blockIdx.x];
  const int2 cr = v.cta_cam[blockIdx.x];
  int t_issue;
  v2_prologue(v, sy, c, part, cr, t_issue);
  double* my_y = sy + (warp % v.replicas) * v2_sy_stride(v.max_cam_span);
  const char* Ebytes = reinterpret_cast<const char*>(v.p.E());
  int it = 0;
  for (int tile = part.x + warp; tile < part.y; tile += v.warps, ++it) {
    const int s = it % v.stages;
    const uint32_t parity = (it / v.stages) & 1;
    const WarpTile wt = v.wtiles[tile];
    if (tile + v.warps < part.y) {  // pull the next tile's non-TMA operands towards L2
      const WarpTile nt = v.wtiles[tile + v.warps];
      if (lane < 12) {
        if (128 * lane < 48 * nt.row_count) prefetch_l2(Ebytes + 48 * static_cast<size_t>(nt.row_begin) + 128 * lane);
      } else if (lane < 24) {
        if (128 * (lane - 12) < 48 * nt.pt_count)
          prefetch_l2(reinterpret_cast<const char*>(ete_inv + 6 * static_cast<size_t>(nt.pt_begin)) + 128 * (lane - 12));
      } else if (lane == 24) {
        prefetch_l2(v.row_meta + nt.row_begin);
      }
    }
    const bool active = lane < wt.row_count;
    const size_t row = static_cast<size_t>(wt.row_begin) + lane;
    const uint32_t meta = active ? __ldg(v.row_meta + row) : 0u;
    const int cam = meta_cam(meta), cam_l = meta_local(v, meta, cr);
    const Seg sg = v2_segment(active && meta_head(meta), wt.row_count);
    double2 e0 = make_double2(0, 0), e1 = e0, e2 = e0;
    double t0 = 0.0, t1 = 0.0;
    if (active) {
      const double2* ep = reinterpret_cast<const double2*>(v.p.E() + 6 * row);
      e0 = __ldg(ep);
      e1 = __ldg(ep + 1);
      e2 = __ldg(ep + 2);
    }
    {
      double xc[9];
      if (active) {
        const double* xcp = x + 9 * static_cast<size_t>(cam);
#pragma unroll
        for (int k = 0; k < 9; ++k) xc[k] = __ldg(xcp + k);
      }
      mbar_wait(c.bars + s, parity);
      if (active) {
        const double* fr = c.sF + s * 576 + lane * 18;
        double ta = 0.0, tb = 0.0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {  // row 0 = elements 0..8, row 1 = 9..17; element 8|9 share a double2
          const double2 a = lds2(fr + 2 * k);
          t0 += a.x * xc[2 * k];
          ta += a.y * xc[2 * k + 1];
        }
        {
          const double2 a = lds2(fr + 8);
          t0 += a.x * xc[8];
          t1 += a.y * xc[0];
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const double2 a = lds2(fr + 10 + 2 * k);
          t1 += a.x * xc[2 * k + 1];
          tb += a.y * xc[2 * k + 2];
        }
        t0 += ta;
        t1 += tb;
        c.sW[lane * 3 + 0] = e0.x * t0 + e1.y * t1;
        c.sW[lane * 3 + 1] = e0.y * t0 + e2.x * t1;
        c.sW[lane * 3 + 2] = e1.x * t0 + e2.y * t1;
      }
    }
    __syncwarp();
    double g[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (active) {
      double u0 = 0.0, u1 = 0.0, u2 = 0.0;
      for (int j = sg.first; j < sg.end; ++j) {
        u0 += c.sW[j * 3 + 0];
        u1 += c.sW[j * 3 + 1];
        u2 += c.sW[j * 3 + 2];
      }
      const double* pi = ete_inv + 6 * static_cast<size_t>(wt.pt_begin + sg.lpt);
      const double2 pa = __ldg(reinterpret_cast<const double2*>(pi)), pb = __ldg(reinterpret_cast<const double2*>(pi) + 1),
                    pc = __ldg(reinterpret_cast<const double2*>(pi) + 2);
      const double v0 = -(pa.x * u0 + pa.y * u1 + pb.x * u2);
      const double v1 = -(pa.y * u0 + pb.y * u1 + pc.x * u2);
      const double v2 = -(pb.x * u0 + pc.x * u1 + pc.y * u2);
      t0 += e0.x * v0 + e0.y * v1 + e1.x * v2;
      t1 += e1.y * v0 + e2.x * v1 + e2.y * v2;
      const double* fr = c.sF + s * 576 + lane * 18;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const double2 a = lds2(fr + 2 * k);
        g[2 * k] = a.x * t0;
        g[2 * k + 1] = a.y * t0;
      }
      {
        const double2 a = lds2(fr + 8);
        g[8] = a.x * t0;
        g[0] += a.y * t1;
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const double2 a = lds2(fr + 10 + 2 * k);
        g[2 * k + 1] += a.x * t1;
        g[2 * k + 2] += a.y * t1;
      }
    }
    cam_accumulate9(my_y, cam_l, active, g);
    __syncwarp();
    if (t_issue < part.y && lane == 0) v2_issue(v, c, t_issue, s);
    t_issue += v.warps;
  }
  schur_mul_big_points(v, smem_raw + v2_sy_bytes(v.max_cam_span, v.replicas), sy, cr, ete_inv, x, false);
  v2_epilogue(v, sy, cr, y);
}

// ------------------------------------------------------------------------------------------------
// v4: every operand of a warp tile arrives through the warp's TMA ring -- the 2x9 F cells, the 2x3 E cells, the
// (E'E+D^2)^-1 blocks of its points and a 160-byte descriptor block (row words, the tile's own extents and the extents
// of the tile that will reuse the ring slot) -- and x of the CTA's camera range is staged once in shared memory, so the
// main loop issues no global load at all (no long-scoreboard waits on the row word -> x -> (E'E)^-1 dependency chain).  The slot's contents go to
// registers first (the F cells stay there, 36 registers; the kernel sits at 122-126 of the 128 registers that 16 warps
// allow) and the slot is refilled at once, so one slot per warp is enough; with one private camera vector per warp the
// accumulation needs no atomics (cam_accumulate9_owned).
// ------------------------------------------------------------------------------------------------
// Segmented suffix sums of three per-lane values over runs of consecutive lanes (the rows of one point): after
// ceil(log2(maxlen)) steps lane i holds the sum over lanes [i, seg_end) of its run; seg_end is one past the run's last lane.
__device__ __forceinline__ void seg_suffix_sum3(double& w0, double& w1, double& w2, int seg_end, int maxlen) {
  const int lane = threadIdx.x & 31;
  for (int d = 1; d < maxlen; d <<= 1) {
    const double a0 = __shfl_down_sync(0xffffffffu, w0, d), a1 = __shfl_down_sync(0xffffffffu, w1, d),
                 a2 = __shfl_down_sync(0xffffffffu, w2, d);
    if (lane + d < seg_end) {
      w0 += a0;
      w1 += a1;
      w2 += a2;
    }
  }
}

constexpr int kV4MaxThreads = 512;
constexpr int kV4MetaWords = 40;
constexpr int kV4StageBytes = 32 * 144 + 32 * 48 + 32 * 48 + kV4MetaWords * 4;  // F | E | P | descriptor block

// [stages x slot][scratch 96 doubles][slot barriers][16 B: warp 0 keeps the barrier + parity word of the >32-row points]
__host__ __device__ inline int v4_bars_offset(int stages) { return stages * kV4StageBytes + 32 * kV2Scratch * 8; }
__host__ __device__ inline int v4_extra_offset(int stages) { return v4_bars_offset(stages) + ((8 * stages + 15) & ~15); }
__host__ __device__ inline int v4_per_warp_bytes(int stages) { return v4_extra_offset(stages) + 16; }
__host__ __device__ inline size_t v4_sx_bytes(int max_cam_span) { return v2_sy_stride(max_cam_span) * 8; }

// `part_begin`: first tile of the CTA's range (the residency plan is indexed by the position of the tile inside it).
__device__ __forceinline__ void v4_issue(const V2View& v, const double* ete_inv, unsigned char* stage, uint64_t* bar, int tile,
                                         int row_begin, int pt_begin, int row_count, int pt_count, int part_begin) {
  const uint64_t pol = v4_l2_policy(v, tile - part_begin);
  mbar_arrive_expect_tx(bar, row_count * 192u + pt_count * 48u + kV4MetaWords * 4u);
  bulk_g2s(stage, v.p.F() + 18 * static_cast<size_t>(row_begin), row_count * 144u, bar, pol);
  bulk_g2s(stage + 4608, v.p.E() + 6 * static_cast<size_t>(row_begin), row_count * 48u, bar, pol);
  bulk_g2s(stage + 6144, ete_inv + 6 * static_cast<size_t>(pt_begin), pt_count * 48u, bar, pol);
  bulk_g2s(stage + 7680, v.tile_meta + static_cast<size_t>(kV4MetaWords) * tile, kV4MetaWords * 4u, bar, pol);
}

// Adds one 9-vector per row into replica `sy_rep` that only THIS warp touches: after the same warp-level
// aggregation as cam_accumulate9 the group leaders hold distinct cameras, so plain read-modify-write is race-free
// and the nine updates are independent (the shared-memory FP64 atomic is a CAS loop: nine dependent round trips).
__device__ __forceinline__ void cam_accumulate9_owned(double* sy_rep, int cam_local, bool active, double (&g)[9]) {
  const int lane = threadIdx.x & 31;
  const int key = active ? cam_local : (0x40000000 | lane);
  const unsigned m = __match_any_sync(0xffffffffu, key);
  const unsigned above = (lane == 31) ? 0u : (m & (0xfffffffeu << lane));
  int nxt = above ? (__ffs(above) - 1) : -1;
  while (__any_sync(0xffffffffu, nxt >= 0)) {
    const int src = nxt >= 0 ? nxt : lane;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const double v = __shfl_sync(0xffffffffu, g[k], src);
      g[k] += (nxt >= 0) ? v : 0.0;
    }
    nxt = __shfl_sync(0xffffffffu, nxt, src);
    nxt = (src == lane) ? -1 : nxt;
  }
  if (active && (m & ((1u << lane) - 1u)) == 0u) {
    double* yc = sy_rep + 9 * cam_local;
    double o[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) o[k] = yc[k];
#pragma unroll
    for (int k = 0; k < 9; ++k) yc[k] = o[k] + g[k];
  }
  __syncwarp();
}

// Shared-memory map of a v4 CTA: [replicas of the private camera vector][x of the camera range][per-warp areas],
// per-warp area = [stages x {F | E | P | descriptor block}][exchange scratch 96 doubles][mbarriers].
// The context holds OFFSETS into the dynamic shared memory, not pointers: a pointer that crosses a (non-inlined)
// function boundary loses its address space and every access through it becomes a generic LD/ST instead of LDS/STS.
__device__ __forceinline__ unsigned char* v4_smem() {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  return smem_raw;
}
struct V4Ctx {
  int sy_stride;
  int sx_off, ring_off, wbase_off, sW_off, bars_off;
  int2 part, cr;
  __device__ __forceinline__ double* sy() const { return reinterpret_cast<double*>(v4_smem()); }
  __device__ __forceinline__ double* sx() const { return reinterpret_cast<double*>(v4_smem() + sx_off); }
  __device__ __forceinline__ unsigned char* ring() const { return v4_smem() + ring_off; }
  __device__ __forceinline__ unsigned char* wbase() const { return v4_smem() + wbase_off; }
  __device__ __forceinline__ double* sW() const { return reinterpret_cast<double*>(v4_smem() + sW_off); }
  __device__ __forceinline__ uint64_t* bars() const { return reinterpret_cast<uint64_t*>(v4_smem() + bars_off); }
};

__device__ __forceinline__ V4Ctx v4_ctx(const V2View& v) {
  V4Ctx c;
  const int warp = threadIdx.x >> 5;
  c.sy_stride = static_cast<int>(v2_sy_stride(v.max_cam_span));
  c.sx_off = static_cast<int>(v2_sy_bytes(v.max_cam_span, v.replicas));
  c.ring_off = c.sx_off + static_cast<int>(v4_sx_bytes(v.max_cam_span));
  c.wbase_off = c.ring_off + warp * v.per_warp_bytes;
  c.sW_off = c.wbase_off + v.stages * kV4StageBytes;
  c.bars_off = c.sW_off + 32 * kV2Scratch * 8;
  c.part = v.cta_part[blockIdx.x];
  c.cr = v.cta_cam[blockIdx.x];
  return c;
}

// Barriers are initialised ONCE per kernel (re-initialising a live mbarrier is undefined); a kernel that runs several
// products keeps them and tracks the phase parity of every ring slot in `flip` (bit s = parity of the next phase of
// slot s).  The >32-row points use one more barrier and a parity word in warp 0's scratch.
constexpr int kV4BigChunkRows = 40;  // 40 rows x 192 B = 7680 B: one chunk per warp slot
__device__ __forceinline__ void v4_init(const V2View& v, const V4Ctx& c) {
  if ((threadIdx.x & 31) == 0) {
    for (int s = 0; s < v.stages; ++s) mbar_init(c.bars() + s, 1);
    if (threadIdx.x == 0) {
      unsigned char* extra = c.ring() + v4_extra_offset(v.stages);  // warp 0's spare words
      mbar_init(reinterpret_cast<uint64_t*>(extra), 1);
      *reinterpret_cast<uint32_t*>(extra + 8) = 0u;
    }
    fence_mbar_init();
  }
}

// Requests the warp's first tiles.  Its ring slots must be idle.
__device__ __forceinline__ void v4_prime(const V2View& v, const double* ete_inv, const V4Ctx& c) {
  if ((threadIdx.x & 31) == 0) {
    int t = c.part.x + (threadIdx.x >> 5);
    for (int s = 0; s < v.stages && t < c.part.y; ++s, t += v.warps) {
      const WarpTile wt = v.wtiles[t];
      v4_issue(v, ete_inv, c.wbase() + s * kV4StageBytes, c.bars() + s, t, wt.row_begin, wt.pt_begin, wt.row_count, wt.pt_count, c.part.x);
    }
  }
}

// Waits for the tiles requested by v4_prime without consuming them (before the CTA exits).
__device__ __forceinline__ void v4_drain(const V2View& v, const V4Ctx& c, uint32_t flip) {
  int t = c.part.x + (threadIdx.x >> 5);
  for (int s = 0; s < v.stages && t < c.part.y; ++s, t += v.warps) mbar_wait(c.bars() + s, (flip >> s) & 1u);
}

// The >32-row points of the CTA on the v4 layout: staged in 40-row chunks, one per warp slot (slots 0..3), scratch
// in warp 0's scratch words [64, 80), barrier + parity in its spare words -- nothing a later product needs is
// overwritten.
__device__ __forceinline__ void v4_big_points(const V2View& v, const V4Ctx& c, const double* __restrict__ ete_inv) {
  const int2 br = v.cta_big[blockIdx.x];
  if (br.y <= br.x) return;  // uniform per CTA
  double* sw0 = reinterpret_cast<double*>(c.ring() + v.stages * kV4StageBytes);
  BigStage st;
  st.base = c.ring();
  st.chunk_rows = kV4BigChunkRows;
  st.chunk_stride = v.per_warp_bytes;
  st.sU = sw0 + 64;
  unsigned char* extra = c.ring() + v4_extra_offset(v.stages);
  st.bar = reinterpret_cast<uint64_t*>(extra);
  uint32_t* pword = reinterpret_cast<uint32_t*>(extra + 8);
  __syncthreads();  // every warp is done with its ring slot and scratch
  uint32_t parity = *pword;
  schur_mul_big_points_impl(v, st, parity, c.sy(), c.cr, ete_inv, c.sx(), true);
  if (threadIdx.x == 0) *pword = parity;
}

// The warp-tile loop: accumulates F'(F x - E P E'F x) of the CTA's tiles into the private camera vector(s).
// Expects primed barriers, zeroed c.sy(), x of the camera range in c.sx(), and a CTA barrier after those.
// `flip` carries the slots' phase parities from one product to the next (0 for a kernel that runs a single product).
template <bool kOwned>
__device__ __forceinline__ void v4_tiles(const V2View& v, const double* ete_inv, const V4Ctx& c, uint32_t& flip) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int2 part = c.part, cr = c.cr;
  const double* sx = c.sx();
  double* sW = c.sW();
  double* my_y = c.sy() + (kOwned ? warp : warp % v.replicas) * c.sy_stride;
  const int reissue = v.warps * v.stages;
  int it = 0;
  for (int tile = part.x + warp; tile < part.y; tile += v.warps, ++it) {
    const int s = it % v.stages;
    const uint32_t parity = ((it / v.stages) ^ (flip >> s)) & 1u;
    unsigned char* stage = c.wbase() + s * kV4StageBytes;
    const double* sF = reinterpret_cast<const double*>(stage);
    const double* sE = reinterpret_cast<const double*>(stage + 4608);
    const double* sP = reinterpret_cast<const double*>(stage + 6144);
    const uint32_t* sM = reinterpret_cast<const uint32_t*>(stage + 7680);
    mbar_wait(c.bars() + s, parity);
    // ---- everything the tile needs from its ring slot goes to registers first, so that the slot can be refilled
    //      while the arithmetic runs (the ring needs a single stage per warp: more resident warps instead)
    const uint4 own = *reinterpret_cast<const uint4*>(sM + 32);   // row_begin, pt_begin, rows | pts << 16, -
    const uint4 nxt = *reinterpret_cast<const uint4*>(sM + 36);   // same for tile + warps * stages (rows == 0: none)
    const int row_count = static_cast<int>(own.z & 0xffffu);
    const bool active = lane < row_count;
    const uint32_t meta = active ? sM[lane] : 0u;
    const int cam = meta_cam(meta), cam_l = meta_local(v, meta, cr);
    const Seg sg = v2_segment(active && meta_head(meta), row_count);
    double f[18];
    double2 e0 = make_double2(0, 0), e1 = e0, e2 = e0, pa = e0, pb = e0, pc = e0;
    if (active) {
      const double* fr = sF + lane * 18;
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 a = lds2(fr + 2 * k);
        f[2 * k] = a.x;
        f[2 * k + 1] = a.y;
      }
      e0 = lds2(sE + lane * 6);
      e1 = lds2(sE + lane * 6 + 2);
      e2 = lds2(sE + lane * 6 + 4);
      const double* pi = sP + 6 * sg.lpt;
      pa = lds2(pi);
      pb = lds2(pi + 2);
      pc = lds2(pi + 4);
    }
    __syncwarp();  // every lane is done with the ring slot (and with the previous tile's scratch)
    if (lane == 0 && (nxt.z & 0xffffu) != 0u)
      v4_issue(v, ete_inv, stage, c.bars() + s, tile + reissue, static_cast<int>(nxt.x), static_cast<int>(nxt.y),
               static_cast<int>(nxt.z & 0xffffu), static_cast<int>(nxt.z >> 16), part.x);
    double t0 = 0.0, t1 = 0.0, w0 = 0.0, w1 = 0.0, w2 = 0.0;
    if (active) {
      double xc[9];
      const double* xcp = sx + 9 * cam_l;
#pragma unroll
      for (int k = 0; k < 9; ++k) xc[k] = xcp[k];
      double ta = 0.0, tb = 0.0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        t0 += f[2 * k] * xc[2 * k];
        ta += f[2 * k + 1] * xc[2 * k + 1];
        t1 += f[9 + 2 * k] * xc[2 * k];
        tb += f[10 + 2 * k] * xc[2 * k + 1];
      }
      t0 += f[8] * xc[8];
      t1 += f[17] * xc[8];
      t0 += ta;
      t1 += tb;
      w0 = e0.x * t0 + e1.y * t1;
      w1 = e0.y * t0 + e2.x * t1;
      w2 = e1.x * t0 + e2.y * t1;
    }
    // u = sum over the rows of the point of E'(F x): segmented suffix sums by shuffles (log2(longest point of the tile)
    // steps, fewer LSU wavefronts than an exchange through shared memory), the
    // total sits in the point's first lane and is broadcast from there
    seg_suffix_sum3(w0, w1, w2, sg.end, static_cast<int>(own.w));
    const double u0 = __shfl_sync(0xffffffffu, w0, sg.first), u1 = __shfl_sync(0xffffffffu, w1, sg.first),
                 u2 = __shfl_sync(0xffffffffu, w2, sg.first);
    double g[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    if (active) {
      const double v0 = -(pa.x * u0 + pa.y * u1 + pb.x * u2);
      const double v1 = -(pa.y * u0 + pb.y * u1 + pc.x * u2);
      const double v2 = -(pb.x * u0 + pc.x * u1 + pc.y * u2);
      t0 += e0.x * v0 + e0.y * v1 + e1.x * v2;
      t1 += e1.y * v0 + e2.x * v1 + e2.y * v2;
#pragma unroll
      for (int k = 0; k < 9; ++k) g[k] = f[k] * t0 + f[9 + k] * t1;
    }
    if (kOwned) cam_accumulate9_owned(my_y, cam_l, active, g);
    else cam_accumulate9(my_y, cam_l, active, g);
  }
  // phases consumed on slot s: tiles it = s, s + stages, ... < `it`
  for (int s = 0; s < v.stages; ++s) flip ^= (((it - s + v.stages - 1) / v.stages) & 1u) << s;
}

// pq_part (may be null): the CTA also writes x . (its partial of y) there -- the p.q of the PCG without a pass over q
// (the D_f^2 term is added by the vector kernel, which seeds y with it).
template <bool kOwned>
__global__ void __launch_bounds__(kV4MaxThreads, 1)
    schur_mul_v4_kernel(V2View v, const double* __restrict__ ete_inv, const double* __restrict__ x, double* y,
                        const int* __restrict__ done_flag, double* pq_part) {
  // Everything up to the wait below only touches data that is constant during a PCG (J, (E'E)^-1, the tile tables), so
  // that with programmatic dependent launch this prologue and the first TMA requests overlap the tail of the vector
  // kernel that produces x (griddepcontrol.wait is a no-op for an ordinary launch).
  const V4Ctx c = v4_ctx(v);
  v4_init(v, c);
  v4_prime(v, ete_inv, c);
  {
    const int n = c.sy_stride * v.replicas;
    for (int i = threadIdx.x; i < n; i += blockDim.x) c.sy()[i] = 0.0;
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (done_flag != nullptr && __ldcg(done_flag) != 0) {  // PCG already terminated: nothing to do but let the TMA land
      v4_drain(v, c, 0);
      return;
    }
    for (int i = threadIdx.x; i < 9 * v2_span(v, c.cr); i += blockDim.x) c.sx()[i] = __ldcg(x + v2_global_entry(v, c.cr, i, 9));
  }
  __syncthreads();
  uint32_t flip = 0;
  v4_tiles<kOwned>(v, ete_inv, c, flip);
  v4_big_points(v, c, ete_inv);
  if (pq_part == nullptr || !v.direct) {
    v2_epilogue(v, c.sy(), c.cr, y);
    return;
  }
  // direct flush + x . partial
  __shared__ double s_pq;
  if (threadIdx.x == 0) s_pq = 0.0;
  __syncthreads();
  const int n = 9 * v2_span(v, c.cr);
  const double* sy = c.sy();
  const double* sx = c.sx();
  double pq = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double acc = sy[i];
    for (int r = 1; r < v.replicas; ++r) acc += sy[r * c.sy_stride + i];
    if (acc != 0.0) red_add(y + v2_global_entry(v, c.cr, i, 9), acc);
    pq += sx[i] * acc;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) pq += __shfl_xor_sync(0xffffffffu, pq, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(&s_pq, pq);
  __syncthreads();
  if (threadIdx.x == 0) pq_part[blockIdx.x] = s_pq;
}

// ------------------------------------------------------------------------------------------------
// (J'J + D^2) x with the v4 machinery: the slot carries F, E, the descriptor block and -- in the place of the (E'E)^-1
// blocks -- the point part of x for the tile's points (24 B per point: the bulk copy fetches the 16-byte-aligned superset,
// `xoff` is where the tile's first point starts inside it); x of the CTA's cameras is staged like in S*x.  Per row
// t = E x_p + F x_c; the camera part F't goes through the per-warp private vectors and the direct flush, the point part
// D_p^2 x_p + sum_rows E't is written by the point's first lane (segmented shuffle sum; the tile owns its points).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void jtj_v4_issue(const V2View& v, const double* x, unsigned char* stage, uint64_t* bar, int tile,
                                             int row_begin, int pt_begin, int row_count, int pt_count) {
  const uint32_t xoff = (pt_begin & 1) ? 8u : 0u;                       // (24 * pt_begin) mod 16
  const uint32_t xbytes = (24u * pt_count + xoff + 15u) & ~15u;         // <= 784
  mbar_arrive_expect_tx(bar, row_count * 192u + xbytes + kV4MetaWords * 4u);
  bulk_g2s(stage, v.p.F() + 18 * static_cast<size_t>(row_begin), row_count * 144u, bar);
  bulk_g2s(stage + 4608, v.p.E() + 6 * static_cast<size_t>(row_begin), row_count * 48u, bar);
  bulk_g2s(stage + 6144, reinterpret_cast<const unsigned char*>(x + 3 * static_cast<size_t>(pt_begin)) - xoff, xbytes, bar);
  bulk_g2s(stage + 7680, v.tile_meta + static_cast<size_t>(kV4MetaWords) * tile, kV4MetaWords * 4u, bar);
}

// The 33..kTile-row points of the CTA for J'J x, processed by the whole CTA after its warp tiles (same staging as
// schur_mul_big_points_impl): t = E x_p + F x_c per row, the point part D_p^2 x_p + sum E't is WRITTEN by thread 0 (the
// CTA owns the point), the camera part F't goes into replica 0 of the private camera vector with shared-memory atomics.
__device__ __forceinline__ void jtj_big_points_impl(const V2View& v, const BigStage& st, uint32_t& parity, double* sy_rep0, int2 cr,
                                                    const double* __restrict__ x, const double* __restrict__ D, const double* sx,
                                                    double* y) {
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
    int cam_l = 0;
    double xc[9];
    const size_t po = 3 * static_cast<size_t>(d.pt_begin);
    const double xp0 = __ldg(x + po), xp1 = __ldg(x + po + 1), xp2 = __ldg(x + po + 2);
    if (active) {
      cam_l = meta_local(v, __ldg(v.row_meta + d.obs_begin + tid), cr);
      const double* xcp = sx + 9 * cam_l;
#pragma unroll
      for (int k = 0; k < 9; ++k) xc[k] = xcp[k];
    }
    mbar_wait(st.bar, parity);
    parity ^= 1;
    double t0 = 0.0, t1 = 0.0, w0 = 0.0, w1 = 0.0, w2 = 0.0;
    double f[18];
    if (active) {
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 a = lds2(sF + 2 * k);
        f[2 * k] = a.x;
        f[2 * k + 1] = a.y;
      }
      const double2 e0 = lds2(sE), e1 = lds2(sE + 2), e2 = lds2(sE + 4);
      t0 = e0.x * xp0 + e0.y * xp1 + e1.x * xp2;
      t1 = e1.y * xp0 + e2.x * xp1 + e2.y * xp2;
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        t0 += f[k] * xc[k];
        t1 += f[9 + k] * xc[k];
      }
      w0 = e0.x * t0 + e1.y * t1;
      w1 = e0.y * t0 + e2.x * t1;
      w2 = e1.x * t0 + e2.y * t1;
    }
    if (tid < kTile) {  // the first four warps hold all rows
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        w0 += __shfl_xor_sync(0xffffffffu, w0, o);
        w1 += __shfl_xor_sync(0xffffffffu, w1, o);
        w2 += __shfl_xor_sync(0xffffffffu, w2, o);
      }
      if ((tid & 31) == 0) {
        sU[(tid >> 5) * 3 + 0] = w0;
        sU[(tid >> 5) * 3 + 1] = w1;
        sU[(tid >> 5) * 3 + 2] = w2;
      }
    }
    __syncthreads();
    if (tid == 0) {
      const double d0 = D != nullptr ? __ldg(D + po) : 0.0, d1 = D != nullptr ? __ldg(D + po + 1) : 0.0,
                   d2 = D != nullptr ? __ldg(D + po + 2) : 0.0;
      y[po] = d0 * d0 * xp0 + (sU[0] + sU[3] + sU[6] + sU[9]);
      y[po + 1] = d1 * d1 * xp1 + (sU[1] + sU[4] + sU[7] + sU[10]);
      y[po + 2] = d2 * d2 * xp2 + (sU[2] + sU[5] + sU[8] + sU[11]);
    }
    if (active) {
      double* yc = sy_rep0 + 9 * cam_l;
#pragma unroll
      for (int k = 0; k < 9; ++k) atomicAdd(yc + k, f[k] * t0 + f[9 + k] * t1);
    }
    __syncthreads();  // staging and sU are reused by the next point
  }
}

// y = (J'J + D^2) x in ONE launch: the point part of y is written by the tile that owns the point (D_p^2 x_p + sum E't,
// no seeding pass, no REDs), the camera part is added into y_c, which the caller seeds with D_c^2 x_c (a 9C-element
// kernel).  D may be null.
template <bool kOwned>
__global__ void __launch_bounds__(kV4MaxThreads, 1)
    jtj_v4_kernel(V2View v, const double* __restrict__ x, const double* __restrict__ D, double* y) {
  const V4Ctx c = v4_ctx(v);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int2 part = c.part, cr = c.cr;
  const size_t off = 3 * static_cast<size_t>(v.p.P);
  v4_init(v, c);
  if (lane == 0) {
    int t = part.x + warp;
    for (int s = 0; s < v.stages && t < part.y; ++s, t += v.warps) {
      const WarpTile wt = v.wtiles[t];
      jtj_v4_issue(v, x, c.wbase() + s * kV4StageBytes, c.bars() + s, t, wt.row_begin, wt.pt_begin, wt.row_count, wt.pt_count);
    }
  }
  {
    const int n = c.sy_stride * v.replicas;
    for (int i = threadIdx.x; i < n; i += blockDim.x) c.sy()[i] = 0.0;
    for (int i = threadIdx.x; i < 9 * v2_span(v, cr); i += blockDim.x) c.sx()[i] = __ldcg(x + off + v2_global_entry(v, cr, i, 9));
  }
  __syncthreads();
  const double* sx = c.sx();
  double* my_y = c.sy() + (kOwned ? warp : warp % v.replicas) * c.sy_stride;
  const int reissue = v.warps * v.stages;
  int it = 0;
  for (int tile = part.x + warp; tile < part.y; tile += v.warps, ++it) {
    const int s = it % v.stages;
    const uint32_t parity = (it / v.stages) & 1u;
    unsigned char* stage = c.wbase() + s * kV4StageBytes;
    const double* sF = reinterpret_cast<const double*>(stage);
    const double* sE = reinterpret_cast<const double*>(stage + 4608);
    const uint32_t* sM = reinterpret_cast<const uint32_t*>(stage + 7680);
    mbar_wait(c.bars() + s, parity);
    const uint4 own = *reinterpret_cast<const uint4*>(sM + 32);
    const uint4 nxt = *reinterpret_cast<const uint4*>(sM + 36);
    const int row_count = static_cast<int>(own.z & 0xffffu);
    const int pt_begin = static_cast<int>(own.y);
    const bool active = lane < row_count;
    const uint32_t meta = active ? sM[lane] : 0u;
    const int cam_l = meta_local(v, meta, cr);
    const Seg sg = v2_segment(active && meta_head(meta), row_count);
    const bool head = active && lane == sg.first;
    double f[18];
    double2 e0 = make_double2(0, 0), e1 = e0, e2 = e0;
    double xp0 = 0.0, xp1 = 0.0, xp2 = 0.0, dp0 = 0.0, dp1 = 0.0, dp2 = 0.0;
    const size_t po = 3 * static_cast<size_t>(pt_begin + sg.lpt);
    if (head && D != nullptr) {  // needed only at the end of the tile: in flight during the arithmetic
      dp0 = __ldg(D + po);
      dp1 = __ldg(D + po + 1);
      dp2 = __ldg(D + po + 2);
    }
    if (active) {
      const double* fr = sF + lane * 18;
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 a = lds2(fr + 2 * k);
        f[2 * k] = a.x;
        f[2 * k + 1] = a.y;
      }
      e0 = lds2(sE + lane * 6);
      e1 = lds2(sE + lane * 6 + 2);
      e2 = lds2(sE + lane * 6 + 4);
      const double* xp = reinterpret_cast<const double*>(stage + 6144 + ((pt_begin & 1) ? 8 : 0)) + 3 * sg.lpt;
      xp0 = xp[0];
      xp1 = xp[1];
      xp2 = xp[2];
    }
    __syncwarp();  // every lane is done with the ring slot
    if (lane == 0 && (nxt.z & 0xffffu) != 0u)
      jtj_v4_issue(v, x, stage, c.bars() + s, tile + reissue, static_cast<int>(nxt.x), static_cast<int>(nxt.y),
                   static_cast<int>(nxt.z & 0xffffu), static_cast<int>(nxt.z >> 16));
    double t0 = 0.0, t1 = 0.0, w0 = 0.0, w1 = 0.0, w2 = 0.0;
    if (active) {
      const double* xcp = sx + 9 * cam_l;
      t0 = e0.x * xp0 + e0.y * xp1 + e1.x * xp2;
      t1 = e1.y * xp0 + e2.x * xp1 + e2.y * xp2;
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double xk = xcp[k];
        t0 += f[k] * xk;
        t1 += f[9 + k] * xk;
      }
      w0 = e0.x * t0 + e1.y * t1;
      w1 = e0.y * t0 + e2.x * t1;
      w2 = e1.x * t0 + e2.y * t1;
    }
    seg_suffix_sum3(w0, w1, w2, sg.end, static_cast<int>(own.w));   // point part: the first lane of the point holds the sum
    if (head) {
      y[po] = dp0 * dp0 * xp0 + w0;
      y[po + 1] = dp1 * dp1 * xp1 + w1;
      y[po + 2] = dp2 * dp2 * xp2 + w2;
    }
    double g[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) g[k] = active ? f[k] * t0 + f[9 + k] * t1 : 0.0;
    if (kOwned) cam_accumulate9_owned(my_y, cam_l, active, g);
    else cam_accumulate9(my_y, cam_l, active, g);
  }
  {  // the CTA's 33..kTile-row points (uniform per CTA)
    const int2 br = v.cta_big[blockIdx.x];
    if (br.y > br.x) {
      double* sw0 = reinterpret_cast<double*>(c.ring() + v.stages * kV4StageBytes);
      BigStage st;
      st.base = c.ring();
      st.chunk_rows = kV4BigChunkRows;
      st.chunk_stride = v.per_warp_bytes;
      st.sU = sw0 + 64;
      unsigned char* extra = c.ring() + v4_extra_offset(v.stages);
      st.bar = reinterpret_cast<uint64_t*>(extra);
      __syncthreads();  // every warp is done with its ring slot
      uint32_t parity = 0;
      jtj_big_points_impl(v, st, parity, c.sy(), cr, x, D, sx, y);
    }
  }
  v2_epilogue(v, c.sy(), cr, y + off);
}

// ------------------------------------------------------------------------------------------------
// y = J'(J x) + D^2 x in one pass: point part written directly (owned by the tile), camera part -> partials.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kV2MaxThreads, 1)
    jtj_v2_kernel(V2View v, const double* __restrict__ x, const double* __restrict__ D, double* y) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  double* sy = reinterpret_cast<double*>(smem_raw);
  const WarpCtx c = v2_warp_ctx(v, smem_raw, kV2Scratch);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int2 part = v.cta_part[blockIdx.x];
  const int2 cr = v.cta_cam[blockIdx.x];
  int t_issue;
  v2_prologue(v, sy, c, part, cr, t_issue);
  const size_t off = 3 * static_cast<size_t>(v.p.P);
  int it = 0;
  for (int tile = part.x + warp; tile < part.y; tile += v.warps, ++it) {
    const int s = it % v.stages;
    const uint32_t parity = (it / v.stages) & 1;
    const WarpTile wt = v.wtiles[tile];
    const bool active = lane < wt.row_count;
    const size_t row = static_cast<size_t>(wt.row_begin) + lane;
    const uint32_t meta = active ? v.row_meta[row] : 0x80000000u;
    const int cam = meta_cam(meta), cam_l = meta_local(v, meta, cr);
    const Seg sg = v2_segment(active && meta_head(meta), wt.row_count);
    double xc[9], xp[3] = {0, 0, 0};
    double2 e0 = make_double2(0, 0), e1 = e0, e2 = e0;
    size_t po = 0;
    if (active) {
      const double* xcp = x + off + 9 * static_cast<size_t>(cam);
#pragma unroll
      for (int k = 0; k < 9; ++k) xc[k] = __ldg(xcp + k);
      po = 3 * static_cast<size_t>(wt.pt_begin + sg.lpt);
#pragma unroll
      for (int k = 0; k < 3; ++k) xp[k] = __ldg(x + po + k);
      const double2* ep = reinterpret_cast<const double2*>(v.p.E() + 6 * row);
      e0 = __ldg(ep);
      e1 = __ldg(ep + 1);
      e2 = __ldg(ep + 2);
    }
    mbar_wait(c.bars + s, parity);
    double f[18] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    double t0 = 0.0, t1 = 0.0;
    if (active) {
      const double* fr = c.sF + s * 576 + lane * 18;
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 a = lds2(fr + 2 * k);
        f[2 * k] = a.x;
        f[2 * k + 1] = a.y;
      }
      t0 = e0.x * xp[0] + e0.y * xp[1] + e1.x * xp[2];
      t1 = e1.y * xp[0] + e2.x * xp[1] + e2.y * xp[2];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        t0 += f[k] * xc[k];
        t1 += f[9 + k] * xc[k];
      }
      c.sW[lane * 3 + 0] = e0.x * t0 + e1.y * t1;
      c.sW[lane * 3 + 1] = e0.y * t0 + e2.x * t1;
      c.sW[lane * 3 + 2] = e1.x * t0 + e2.y * t1;
    }
    {
      double g[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) g[k] = active ? f[k] * t0 + f[9 + k] * t1 : 0.0;
      cam_accumulate9(sy + (warp % v.replicas) * v2_sy_stride(v.max_cam_span), cam_l, active, g);
    }
    __syncwarp();
    if (active && lane == sg.first) {
      double u0 = 0.0, u1 = 0.0, u2 = 0.0;
      for (int j = sg.first; j < sg.end; ++j) {
        u0 += c.sW[j * 3 + 0];
        u1 += c.sW[j * 3 + 1];
        u2 += c.sW[j * 3 + 2];
      }
      if (D != nullptr) {
        u0 += D[po] * D[po] * xp[0];
        u1 += D[po + 1] * D[po + 1] * xp[1];
        u2 += D[po + 2] * D[po + 2] * xp[2];
      }
      y[po] = u0;
      y[po + 1] = u1;
      y[po + 2] = u2;
    }
    __syncwarp();
    if (t_issue < part.y && lane == 0) v2_issue(v, c, t_issue, s);
    t_issue += v.warps;
  }
  v2_epilogue(v, sy, cr, y + off);
}

// ------------------------------------------------------------------------------------------------
// y[j] = (seed ? d[j]^2 x[j] : 0) + sum over CTAs (fixed order) of their partial for camera entry j.
// add != 0: y[j] += ... instead (accumulate on top of an existing vector).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    cam_reduce_kernel(int n, int num_ctas, const int2* __restrict__ cta_cam, const double* __restrict__ partials,
                      int stride, const double* __restrict__ d, const double* __restrict__ x, double* y, int add,
                      const int* __restrict__ done_flag) {
  if (done_flag != nullptr && *done_flag != 0) return;
  // 64 camera entries per block x 4 slices of the CTA list; slices are combined in a fixed order.
  extern __shared__ int2 s_ranges[];
  __shared__ double s_part[4][64];
  for (int b = threadIdx.x; b < num_ctas; b += blockDim.x) s_ranges[b] = cta_cam[b];
  __syncthreads();
  const int e = threadIdx.x & 63, slice = threadIdx.x >> 6;
  const int j = blockIdx.x * 64 + e;
  double acc = 0.0;
  if (j < n) {
    const int cidx = j / 9;
    const int b0 = num_ctas * slice / 4, b1 = num_ctas * (slice + 1) / 4;
    double a0 = 0.0, a1 = 0.0;
    int b = b0;
    for (; b + 1 < b1; b += 2) {
      const int2 r0 = s_ranges[b], r1 = s_ranges[b + 1];
      if (cidx >= r0.x && cidx < r0.y) a0 += partials[static_cast<size_t>(b) * stride + (j - 9 * r0.x)];
      if (cidx >= r1.x && cidx < r1.y) a1 += partials[static_cast<size_t>(b + 1) * stride + (j - 9 * r1.x)];
    }
    if (b < b1) {
      const int2 r0 = s_ranges[b];
      if (cidx >= r0.x && cidx < r0.y) a0 += partials[static_cast<size_t>(b) * stride + (j - 9 * r0.x)];
    }
    acc = a0 + a1;
  }
  s_part[slice][e] = acc;
  __syncthreads();
  if (slice == 0 && j < n) {
    double v = (d != nullptr) ? d[j] * d[j] * x[j] : 0.0;
    if (add) v += y[j];
    v += ((s_part[0][e] + s_part[1][e]) + (s_part[2][e] + s_part[3][e]));
    y[j] = v;
  }
}

}  // namespace b200
