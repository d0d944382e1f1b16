// Warp-tile (v2) versions of the once-per-LM-iteration kernels: evaluate (+ fused column norms) and the block diagonal
// of the Schur complement.  Same structure as kernels_v2.cuh: one
// persistent CTA per SM, whole points in <= 32-row warp tiles, per-point sums through __syncwarp + a per-warp
// scratch, camera-sized results accumulated in CTA-private shared memory after a warp-level pre-reduction and
// flushed with a few hundred REDs per CTA.  Used when the CTAs' camera ranges are narrow (V2View::direct); the
// CTA-tile kernels of kernels.cuh remain the general fallback.
#pragma once
#include "kernels.cuh"
#include "kernels_v2.cuh"

namespace b200 {

// Flush `count` doubles per camera of a replicated private accumulator into global memory with REDs.
__device__ __forceinline__ void v2_flush(const V2View& v, int2 cr, const double* sacc, int per_cam, int replicas,
                                         size_t rep_stride, double* dst /* camera-major, per_cam doubles per camera */) {
  const int n = per_cam * v2_span(v, cr);
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    double acc = sacc[i];
    for (int r = 1; r < replicas; ++r) acc += sacc[r * rep_stride + i];
    if (acc != 0.0) red_add(dst + v2_global_entry(v, cr, i, per_cam), acc);
  }
}

// Segmented sum of K per-lane values over the rows of each point of the warp tile (through the per-warp scratch).
template <int K>
__device__ __forceinline__ void v2_point_sum(double* sW, const Seg& sg, bool active, const double (&in)[K], double (&out)[K]) {
  const int lane = threadIdx.x & 31;
  __syncwarp();
  if (active) {
#pragma unroll
    for (int k = 0; k < K; ++k) sW[lane * K + k] = in[k];
  }
  __syncwarp();
#pragma unroll
  for (int k = 0; k < K; ++k) out[k] = 0.0;
  if (active) {
    for (int j = sg.first; j < sg.end; ++j) {
#pragma unroll
      for (int k = 0; k < K; ++k) out[k] += sW[j * K + k];
    }
  }
}

// Pointer-jumping warp pre-reduction for K values + shared-memory accumulation (see cam_accumulate9).
template <int K>
__device__ __forceinline__ void cam_accumulate(double* sacc_rep, int cam_local, bool active, double (&g)[K],
                                               int stride = K, int offset = 0) {
  const int lane = threadIdx.x & 31;
  const int key = active ? cam_local : (0x40000000 | lane);
  const unsigned m = __match_any_sync(0xffffffffu, key);
  const unsigned above = (lane == 31) ? 0u : (m & (0xfffffffeu << lane));
  int nxt = above ? (__ffs(above) - 1) : -1;
  while (__any_sync(0xffffffffu, nxt >= 0)) {
    const int src = nxt >= 0 ? nxt : lane;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const double v = __shfl_sync(0xffffffffu, g[k], src);
      g[k] += (nxt >= 0) ? v : 0.0;
    }
    nxt = __shfl_sync(0xffffffffu, nxt, src);
    nxt = (src == lane) ? -1 : nxt;
  }
  if (active && (m & ((1u << lane) - 1u)) == 0u) {
    double* yc = sacc_rep + stride * cam_local + offset;
#pragma unroll
    for (int k = 0; k < K; ++k) atomicAdd(yc + k, g[k]);
  }
}

// (row, col) of entry idx of the row-major packed upper triangle of a 9x9 matrix.
__host__ __device__ constexpr int upper9_row(int idx) {
  int a = 0;
  while (idx >= 9 - a) {
    idx -= 9 - a;
    ++a;
  }
  return a;
}
__host__ __device__ constexpr int upper9_col(int idx) {
  int a = 0;
  while (idx >= 9 - a) {
    idx -= 9 - a;
    ++a;
  }
  return a + idx;
}

constexpr int kEvalScratch = 3;  // doubles per lane in the exchange scratch
__host__ __device__ inline int eval_v2_per_warp_bytes() { return 32 * 144 + 32 * 48 + 32 * kEvalScratch * 8; }

// Evaluate residuals, Jacobian (written through a per-warp staging buffer + TMA bulk store), cost, gradient and the
// squared column norms of the Jacobian as written (i.e. after the fused Jacobi scaling).
// kStoreJ = false (gradient without the Jacobian): as evaluate_kernel<kLoss, true, false>, the Jacobian is left as it is.
// kFixed: constant blocks' cells and coordinates held by a SubsetManifold are 0 (evaluate_row).
template <int kLoss, bool kStoreJ, bool kFixed = false>
__global__ void __launch_bounds__(kV2MaxThreads, 1) evaluate_v2_kernel(V2View v, EvalArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int2 part = v.cta_part[blockIdx.x];
  const int2 cr = v.cta_cam[blockIdx.x];
  const size_t rstride = v2_sy_stride(v.max_cam_span);
  double* sg_acc = reinterpret_cast<double*>(smem_raw);                 // gradient, [replicas][rstride]
  double* sq_acc = sg_acc + rstride * v.replicas;                       // column norms
  unsigned char* wbase = smem_raw + 2 * rstride * v.replicas * 8 + static_cast<size_t>(warp) * eval_v2_per_warp_bytes();
  double* sF = reinterpret_cast<double*>(wbase);
  double* sE = sF + 32 * 18;
  double* sW = sE + 32 * 6;
  for (int i = threadIdx.x; i < static_cast<int>(2 * rstride * v.replicas); i += blockDim.x) sg_acc[i] = 0.0;
  __syncthreads();
  double* my_g = sg_acc + (warp % v.replicas) * rstride;
  double* my_q = sq_acc + (warp % v.replicas) * rstride;
  const bool owned = v.replicas >= static_cast<int>(blockDim.x >> 5);   // (uniform) no other warp touches this warp's copies
  const size_t camoff = 3 * static_cast<size_t>(v.p.P);
  double cost = 0.0;
  bool store_pending = false;
  for (int tile = part.x + warp; tile < part.y; tile += v.warps) {
    const WarpTile wt = v.wtiles[tile];
    const bool active = lane < wt.row_count;
    const size_t row = static_cast<size_t>(wt.row_begin) + lane;
    const uint32_t meta = active ? __ldg(v.row_meta + row) : 0u;
    const int cam = meta_cam(meta), cam_l = meta_local(v, meta, cr);
    const Seg sg = v2_segment(active && meta_head(meta), wt.row_count);
    double r0 = 0.0, r1 = 0.0;
    double jc[18], jp[6];
#pragma unroll
    for (int k = 0; k < 18; ++k) jc[k] = 0.0;
#pragma unroll
    for (int k = 0; k < 6; ++k) jp[k] = 0.0;
    const int pt = wt.pt_begin + sg.lpt;
    const size_t po = 3 * static_cast<size_t>(pt);
    if (active) cost += evaluate_row<kLoss, true, kFixed>(v.p, a, row, wt.pt_begin, sg.lpt, cam, r0, r1, jc, jp);
    // gradient of the unscaled Jacobian (program_evaluator.h:242-259)
    if (a.gradient != nullptr) {
      double gp[3], gps[3], gc[9];
#pragma unroll
      for (int k = 0; k < 3; ++k) gp[k] = jp[k] * r0 + jp[3 + k] * r1;
#pragma unroll
      for (int k = 0; k < 9; ++k) gc[k] = jc[k] * r0 + jc[9 + k] * r1;
      v2_point_sum<3>(sW, sg, active, gp, gps);
      if (active && lane == sg.first) {
        a.gradient[po] = gps[0];
        a.gradient[po + 1] = gps[1];
        a.gradient[po + 2] = gps[2];
      }
      if (owned) cam_accumulate9_owned(my_g, cam_l, active, gc);   // one private copy per warp: plain read-modify-write
      else cam_accumulate<9>(my_g, cam_l, active, gc);
    }
    if (a.scale != nullptr && active) scale_row(a.scale, v.p.P, pt, cam, jc, jp);
    if (a.sqnorm != nullptr) {
      double qp[3], qps[3], qc[9];
#pragma unroll
      for (int k = 0; k < 3; ++k) qp[k] = jp[k] * jp[k] + jp[3 + k] * jp[3 + k];
#pragma unroll
      for (int k = 0; k < 9; ++k) qc[k] = jc[k] * jc[k] + jc[9 + k] * jc[9 + k];
      v2_point_sum<3>(sW, sg, active, qp, qps);
      if (active && lane == sg.first) {
        a.sqnorm[po] = qps[0];
        a.sqnorm[po + 1] = qps[1];
        a.sqnorm[po + 2] = qps[2];
      }
      if (owned) cam_accumulate9_owned(my_q, cam_l, active, qc);
      else cam_accumulate<9>(my_q, cam_l, active, qc);
    }
    if (!kStoreJ) continue;
    // Jacobian cells: stage the warp's rows contiguously, then one TMA bulk store each for E and F
    if (store_pending) {
      if (lane == 0) bulk_wait_read_all();
      __syncwarp();
    }
    if (active) {
#pragma unroll
      for (int k = 0; k < 3; ++k) *reinterpret_cast<double2*>(sE + lane * 6 + 2 * k) = make_double2(jp[2 * k], jp[2 * k + 1]);
#pragma unroll
      for (int k = 0; k < 9; ++k) *reinterpret_cast<double2*>(sF + lane * 18 + 2 * k) = make_double2(jc[2 * k], jc[2 * k + 1]);
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) {
      bulk_s2g(v.p.E() + 6 * static_cast<size_t>(wt.row_begin), sE, wt.row_count * 48u);
      bulk_s2g(v.p.F() + 18 * static_cast<size_t>(wt.row_begin), sF, wt.row_count * 144u);
      bulk_commit();
    }
    store_pending = true;
  }
  if (lane == 0) bulk_wait_all();
  // cost: warp sums -> CTA sum (fixed order) -> one partial per CTA
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cost += __shfl_xor_sync(0xffffffffu, cost, o);
  __shared__ double s_cost[kV2MaxThreads / 32];
  if (lane == 0) s_cost[warp] = cost;
  __syncthreads();
  if (threadIdx.x == 0) {
    double c = 0.0;
    for (int w = 0; w < static_cast<int>(blockDim.x >> 5); ++w) c += s_cost[w];
    a.cost_partial[blockIdx.x] = c;
  }
  if (a.gradient != nullptr) v2_flush(v, cr, sg_acc, 9, v.replicas, rstride, a.gradient + camoff);
  if (a.sqnorm != nullptr) v2_flush(v, cr, sq_acc, 9, v.replicas, rstride, a.sqnorm + camoff);
}

// ------------------------------------------------------------------------------------------------
// Block diagonal of the Schur complement (kSchur) or of F'F, upper triangle packed (45 per camera), accumulated into
// out45 (zeroed by the caller).  Same maths as diag_blocks_kernel (schur_eliminator_impl.h:449-568).
// Shared memory: [replicas][45 * max_cam_span] accumulators + per-warp {F ring, E rows, camera ids}.
// ------------------------------------------------------------------------------------------------
__host__ __device__ inline size_t diag_v2_acc_stride(int max_cam_span) {
  return (static_cast<size_t>(45) * max_cam_span + 15) & ~static_cast<size_t>(15);
}
__host__ __device__ inline int diag_v2_per_warp_bytes(int stages) { return (stages * 4608 + 32 * 48 + 32 * 4 + 8 * stages + 15) & ~15; }

__host__ __device__ constexpr int upper9_offset(int a) { return a * 9 - a * (a - 1) / 2; }

// Rows [A0, A1) of the packed upper triangle of  F_i'F_i - W_i' (P buf)  for one Jacobian row, accumulated per camera.
template <bool kSchur, int A0, int A1>
__device__ __forceinline__ void diag_rows(const double (&f)[18], const double (&W)[27], const double (&PB)[27],
                                          double* my_acc, int cam_local, bool active) {
  constexpr int K = upper9_offset(A1) - upper9_offset(A0);
  double mb[K];
  int q = 0;
#pragma unroll
  for (int aa = A0; aa < A1; ++aa) {
#pragma unroll
    for (int bb = aa; bb < 9; ++bb) {
      double mm = f[aa] * f[bb] + f[9 + aa] * f[9 + bb];
      if (kSchur) mm -= W[aa] * PB[bb] + W[9 + aa] * PB[9 + bb] + W[18 + aa] * PB[18 + bb];
      mb[q++] = mm;
    }
  }
  cam_accumulate<K>(my_acc, cam_local, active, mb, 45, upper9_offset(A0));
}

template <bool kSchur>
__global__ void __launch_bounds__(kV2MaxThreads, 1)
    diag_blocks_v2_kernel(V2View v, int replicas, const double* __restrict__ ete_inv, double* out45) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  double* sacc = reinterpret_cast<double*>(smem_raw);
  const size_t astride = diag_v2_acc_stride(v.max_cam_span);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned char* wbase = smem_raw + astride * replicas * 8 + static_cast<size_t>(warp) * diag_v2_per_warp_bytes(v.stages);
  WarpCtx c;
  c.sF = reinterpret_cast<double*>(wbase);
  double* sE = c.sF + v.stages * 576;
  int* sCam = reinterpret_cast<int*>(sE + 32 * 6);
  c.bars = reinterpret_cast<uint64_t*>(sCam + 32);
  c.sW = nullptr;
  const int2 part = v.cta_part[blockIdx.x];
  const int2 cr = v.cta_cam[blockIdx.x];
  for (int i = threadIdx.x; i < static_cast<int>(astride * replicas); i += blockDim.x) sacc[i] = 0.0;
  if (lane == 0) {
    for (int s = 0; s < v.stages; ++s) mbar_init(c.bars + s, 1);
    fence_mbar_init();
  }
  __syncthreads();
  int t_issue = part.x + warp;
  for (int s = 0; s < v.stages && t_issue < part.y; ++s) {
    if (lane == 0) v2_issue(v, c, t_issue, s);
    t_issue += v.warps;
  }
  double* my_acc = sacc + (warp % replicas) * astride;
  int it = 0;
  for (int tile = part.x + warp; tile < part.y; tile += v.warps, ++it) {
    const int s = it % v.stages;
    const uint32_t parity = (it / v.stages) & 1;
    const WarpTile wt = v.wtiles[tile];
    const bool active = lane < wt.row_count;
    const size_t row = static_cast<size_t>(wt.row_begin) + lane;
    const uint32_t meta = active ? __ldg(v.row_meta + row) : 0u;
    const int cam = meta_cam(meta), cam_l = meta_local(v, meta, cr);
    const Seg sg = v2_segment(active && meta_head(meta), wt.row_count);
    double e[6] = {0, 0, 0, 0, 0, 0};
    double pinv[6] = {0, 0, 0, 0, 0, 0};
    if (active && kSchur) {
      const double2* ep = reinterpret_cast<const double2*>(v.p.E() + 6 * row);
      const double2 a0 = __ldg(ep), a1 = __ldg(ep + 1), a2 = __ldg(ep + 2);
      e[0] = a0.x; e[1] = a0.y; e[2] = a1.x; e[3] = a1.y; e[4] = a2.x; e[5] = a2.y;
      const double* pi = ete_inv + 6 * static_cast<size_t>(wt.pt_begin + sg.lpt);
#pragma unroll
      for (int k = 0; k < 6; ++k) pinv[k] = __ldg(pi + k);
    }
    if (kSchur) {
      __syncwarp();
#pragma unroll
      for (int k = 0; k < 6; ++k) sE[lane * 6 + k] = e[k];
      sCam[lane] = active ? cam : -1;
    }
    mbar_wait(c.bars + s, parity);
    __syncwarp();
    double f[18];
#pragma unroll
    for (int k = 0; k < 18; ++k) f[k] = 0.0;
    if (active) {
      const double* fr = c.sF + s * 576 + lane * 18;
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 w = lds2(fr + 2 * k);
        f[2 * k] = w.x;
        f[2 * k + 1] = w.y;
      }
    }
    double W[27], PB[27];
    if (kSchur) {
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        W[k] = e[0] * f[k] + e[3] * f[9 + k];
        W[9 + k] = e[1] * f[k] + e[4] * f[9 + k];
        W[18 + k] = e[2] * f[k] + e[5] * f[9 + k];
      }
      double B[27];
#pragma unroll
      for (int k = 0; k < 27; ++k) B[k] = W[k];
      if (active) {  // other rows of my point that see my camera (a camera seeing a point twice: rare)
        for (int j = sg.first; j < sg.end; ++j) {
          if (j != lane && sCam[j] == cam) {
            const double* ej = sE + j * 6;
            const double* fj = c.sF + s * 576 + j * 18;
#pragma unroll
            for (int k = 0; k < 9; ++k) {
              B[k] += ej[0] * fj[k] + ej[3] * fj[9 + k];
              B[9 + k] += ej[1] * fj[k] + ej[4] * fj[9 + k];
              B[18 + k] += ej[2] * fj[k] + ej[5] * fj[9 + k];
            }
          }
        }
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        PB[k] = pinv[0] * B[k] + pinv[1] * B[9 + k] + pinv[2] * B[18 + k];
        PB[9 + k] = pinv[1] * B[k] + pinv[3] * B[9 + k] + pinv[4] * B[18 + k];
        PB[18 + k] = pinv[2] * B[k] + pinv[4] * B[9 + k] + pinv[5] * B[18 + k];
      }
    }
    // 45 packed upper-triangle entries per row, accumulated in three groups of matrix rows ({0,1}, {2,3,4}, {5..8}:
    // 17 + 18 + 10 entries) to bound the live registers; all indices are compile-time after unrolling.
    diag_rows<kSchur, 0, 2>(f, W, PB, my_acc, cam_l, active);
    diag_rows<kSchur, 2, 5>(f, W, PB, my_acc, cam_l, active);
    diag_rows<kSchur, 5, 9>(f, W, PB, my_acc, cam_l, active);
    __syncwarp();
    if (t_issue < part.y && lane == 0) v2_issue(v, c, t_issue, s);
    t_issue += v.warps;
  }
  __syncthreads();
  v2_flush(v, cr, sacc, 45, replicas, astride, out45);
}

}  // namespace b200

namespace b200 {

// ------------------------------------------------------------------------------------------------
// Camera-major block diagonal (no atomics on the hot loop).  For a row i of point k (no camera seeing a point twice):
//   F_i'F_i - (E_i'F_i)' P_k (E_i'F_i) = F_i' Q_i F_i ,   Q_i = I - E_i P_k E_i'   (2x2 symmetric)
// so  M_c = sum_{i in camera c} F_i' Q_i F_i.  Q_i (q00, q01, q11 + one pad per row) is written by the implicit-Schur
// initialisation (kernels_v4b.cuh) or, on the fallback paths, by row_q_kernel in one flat pass over E; the camera-major
// kernels of kernels_v4b.cuh keep the 45 packed entries in registers while they walk a camera's rows.  Same result as SchurEliminator against a block-diagonal lhs
// (schur_eliminator_impl.h:449-568) / UpdateBlockDiagonalFtF (partitioned_matrix_view_impl.h:531-658, Q = I).
// ------------------------------------------------------------------------------------------------
constexpr int kQStride = 4;   // doubles per row of the Q array: q00, q01, q11 and one pad (32-byte rows: aligned bulk copies)

__global__ void __launch_bounds__(256) row_q_kernel(ProblemView p, const double* __restrict__ ete_inv, double* q3) {
  const int stride = gridDim.x * blockDim.x;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < p.N; r += stride) {
    const double2* ep = reinterpret_cast<const double2*>(p.E() + 6 * static_cast<size_t>(r));
    const double2 a0 = __ldg(ep), a1 = __ldg(ep + 1), a2 = __ldg(ep + 2);
    const double e00 = a0.x, e01 = a0.y, e02 = a1.x, e10 = a1.y, e11 = a2.x, e12 = a2.y;
    const double* pi = ete_inv + 6 * static_cast<size_t>(p.pt_of_row[r]);
    const double p0 = __ldg(pi), p1 = __ldg(pi + 1), p2 = __ldg(pi + 2), p3 = __ldg(pi + 3), p4 = __ldg(pi + 4), p5 = __ldg(pi + 5);
    // P e_r' for both rows of E
    const double a = p0 * e00 + p1 * e01 + p2 * e02, b = p1 * e00 + p3 * e01 + p4 * e02, c = p2 * e00 + p4 * e01 + p5 * e02;
    const double d = p0 * e10 + p1 * e11 + p2 * e12, e = p1 * e10 + p3 * e11 + p4 * e12, f = p2 * e10 + p4 * e11 + p5 * e12;
    double2* q = reinterpret_cast<double2*>(q3 + kQStride * static_cast<size_t>(r));
    q[0] = make_double2(1.0 - (e00 * a + e01 * b + e02 * c), -(e10 * a + e11 * b + e12 * c));
    q[1] = make_double2(1.0 - (e10 * d + e11 * e + e12 * f), 0.0);
  }
}

struct CamItem {
  int cam;
  int begin, end;  // range in cam_rows
};

}  // namespace b200
