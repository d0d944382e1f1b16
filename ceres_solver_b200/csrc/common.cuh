// Device-side plumbing shared by every tile kernel of libb200ba: the HBM-resident problem layout,
// TMA (cp.async.bulk) + mbarrier wrappers for sm_90a, and the per-tile bookkeeping.
//
// Layout in HBM (SURVEY Appendix B; reference origin in brackets):
//   values      [24N] f64   all E cells [N][2][3] then all F cells [N][2][9]   (block_jacobian_writer.cc:68-167)
//   cam_idx     [N]   i32   f block of row i                                   (cells[1].block_id - P)
//   pt_ptr      [P+1] i32   chunk boundaries: rows of point k are [pt_ptr[k], pt_ptr[k+1])
//                                                                               (schur_eliminator_impl.h:128-163)
//   obs         [2N]  f64   observed image point of row i
//   tiles       [T]         whole points packed into <= TILE rows; one CTA pass each
// Vectors use the reduced program's order  [ 3 per point | 9 per camera ].
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

constexpr int kTile = 128;  // rows (observations) per tile == threads per CTA

struct TileDesc {
  int obs_begin = 0;   // first row of the tile
  int obs_count = 0;   // rows in the tile (<= kTile)
  int pt_begin = 0;    // first point
  int pt_count = 0;    // points in the tile
  int chunk = 0;       // 1: the rows are a slice of the single point pt_begin, which has more than kTile rows: point-sized
                       // outputs are accumulated with REDs (the caller zeroes them), and the kernels that couple all rows
                       // of a point skip the tile (huge_kernels.cuh does those points)
};

struct ProblemView {
  int C, P;
  int N;
  int num_tiles;
  const TileDesc* tiles;
  const int* cam_idx;
  const int* pt_ptr;
  const int* pt_of_row;  // [N] point of row i (flat kernels)
  const double* obs;
  double* values;  // 24N: E then F
  __device__ __host__ double* E() const { return values; }
  __device__ __host__ double* F() const { return values + 6 * static_cast<size_t>(N); }
};

// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a bulk copy that never lands (wrong byte count, bad descriptor) must not hang the GPU -- after
// ~2 s the kernel traps and the host sees a launch failure.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}
// TMA 1-D bulk copy global -> shared, completion on an mbarrier (SASS: UBLKCP). 16 B aligned, size % 16 == 0.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// L2 cache policies for the hinted bulk copy below (createpolicy: a 64-bit policy word, no memory access).
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_normal() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p));
  return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// bulk_g2s with an L2 eviction-priority hint for the lines it brings into L2.  The hint only decides which lines L2 gives
// up first; the bytes copied are the same.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
// TMA 1-D bulk copy shared -> global (bulk async-group completion).
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
// generic-proxy smem writes -> visible to the async proxy (TMA store source)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ double2 lds2(const double* p) { return *reinterpret_cast<const double2*>(p); }

// ---------------------------------------------------------------- per-CTA tile context
// Shared memory carve-up common to every tile kernel.  E/F staging areas are TMA destinations (16 B aligned).
struct TileSmem {
  double* sE;       // [kTile*6]
  double* sF;       // [kTile*18]
  double* sObs;     // [kTile*kObsScratch]  per-row scratch handed from the per-row to the per-point phase
  double* sPt;      // [kTile*kPtScratch]   per-point scratch handed back to the rows
  int* sPtOfs;      // [kTile+1] first local row of local point k
  int* sSlotPt;     // [kTile]   local point of local row j
  int* sCam;        // [kTile]   camera of local row j
  uint64_t* bar;    // TMA completion barrier
};

template <int kObsScratch, int kPtScratch>
__host__ __device__ constexpr size_t tile_smem_bytes() {
  return sizeof(double) * kTile * (6 + 18 + kObsScratch + kPtScratch) + sizeof(int) * (3 * kTile + 4) + 16;
}

template <int kObsScratch, int kPtScratch>
__device__ __forceinline__ TileSmem carve_smem(unsigned char* base) {
  TileSmem s;
  s.sE = reinterpret_cast<double*>(base);
  s.sF = s.sE + kTile * 6;
  s.sObs = s.sF + kTile * 18;
  s.sPt = s.sObs + kTile * kObsScratch;
  double* end = s.sPt + kTile * kPtScratch;
  s.bar = reinterpret_cast<uint64_t*>(end);
  s.sPtOfs = reinterpret_cast<int*>(s.bar + 2);
  s.sSlotPt = s.sPtOfs + kTile + 2;
  s.sCam = s.sSlotPt + kTile;
  return s;
}

// Once per CTA: arm the TMA completion barrier (one arriving thread: the issuing lane).
__device__ __forceinline__ void tile_prologue(const TileSmem& s) {
  if (threadIdx.x == 0) {
    mbar_init(s.bar, 1);
    fence_mbar_init();
  }
  __syncthreads();
}

// Starts the TMA loads of a tile's E and/or F cells and builds the row<->point maps.
// Ends with a __syncthreads(); the caller waits on s.bar (parity) before touching sE/sF.
__device__ __forceinline__ void tile_begin(const ProblemView& p, const TileDesc& d, const TileSmem& s, bool load_e,
                                           bool load_f) {
  const int tid = threadIdx.x;
  if (tid == 0 && (load_e || load_f)) {
    // One arrival per tile completes the barrier phase once all bytes have landed (an empty tile — only
    // zero-degree points — arrives with 0 bytes so the waiters still pass).
    const uint32_t bytes = (load_e ? d.obs_count * 48u : 0u) + (load_f ? d.obs_count * 144u : 0u);
    mbar_arrive_expect_tx(s.bar, bytes);
    if (d.obs_count > 0) {
      if (load_e) bulk_g2s(s.sE, p.E() + 6 * static_cast<size_t>(d.obs_begin), d.obs_count * 48u, s.bar);
      if (load_f) bulk_g2s(s.sF, p.F() + 18 * static_cast<size_t>(d.obs_begin), d.obs_count * 144u, s.bar);
    }
  }
  // (clamped to the tile: a chunk tile sees its own rows as the rows of its point)
  if (tid <= d.pt_count) s.sPtOfs[tid] = min(max(p.pt_ptr[d.pt_begin + tid] - d.obs_begin, 0), d.obs_count);
  if (tid < d.obs_count) s.sCam[tid] = p.cam_idx[d.obs_begin + tid];
  __syncthreads();
  if (tid < d.pt_count) {
    const int e = s.sPtOfs[tid + 1];
    for (int j = s.sPtOfs[tid]; j < e; ++j) s.sSlotPt[j] = tid;
  }
  __syncthreads();
}

// FP64 atomic accumulate without return (SASS: RED.E.ADD.F64).
__device__ __forceinline__ void red_add(double* addr, double v) { atomicAdd(addr, v); }

template <int BLOCK>
__device__ __forceinline__ double block_sum(double v, double* scratch /* >= BLOCK/32 doubles */) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) scratch[warp] = v;
  __syncthreads();
  double r = 0.0;
  if (warp == 0) {
    r = lane < BLOCK / 32 ? scratch[lane] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) r += __shfl_xor_sync(0xffffffffu, r, o);
  }
  return r;  // valid on warp 0
}

}  // namespace b200
