// One cooperative kernel per PCG iteration carries everything that is not the S*p product:
//   phase A  partial p.q                               (q = S*p was assembled by the product kernels)
//   ---- grid sync ----
//   phase B  alpha = rho / p.q ; x += alpha p ; r -= alpha q ; z = M^-1 r (9x9 block per camera) ;
//            partial x.(b+r), r.r, r.z
//   ---- grid sync ----
//   phase C  the reference's termination tests (conjugate_gradients_solver.h:245-299) evaluated identically by
//            every CTA from the same partials, beta = rho_new / rho, p = z + beta p, and the seed D_f^2 p of the next
//            product ; CTA 0 publishes the state.
// CTAs own whole cameras (28 cameras = 252 entries per 256-thread CTA), so the block-diagonal preconditioner
// needs only the CTA's own slice of r.  All dot products are reduced in a fixed order: the PCG is deterministic
// given q.  The kernel is latency-bound (a few KB per CTA), so every operand that does not depend on a grid-wide
// result is loaded before the grid sync that precedes its use, and each thread keeps its entry of x, r, p, z in
// registers across the phases.  Replaces the reference's ~12 Eigen expressions + 3 host-synchronising dots per
// iteration (conjugate_gradients_solver.h:162-299; cuda_vector.cc:97-181 in its CUDA variant).
#pragma once
#include <cooperative_groups.h>

#include "explicit_schur.cuh"
#include "vector_kernels.cuh"

namespace b200 {
namespace cg = cooperative_groups;

constexpr int kCgCamsPerCta = 28;
constexpr int kCgThreads = 256;

enum CgMode { CG_NORMAL = 0, CG_RESET_FIRST = 1, CG_RESET_SECOND = 2, CG_BEGIN = 3 };

constexpr int kMaxXchgRanks = 8;
struct XchgPeers {
  uint4* buf[kMaxXchgRanks];   // every rank's exchange buffer [2 slots][world][9C + 1] packets, as mapped into THIS process
  int world, rank;
};

__device__ __forceinline__ void xchg_store(uint4* dst, double v, unsigned epoch) {
  const unsigned lo = static_cast<unsigned>(__double2loint(v)), hi = static_cast<unsigned>(__double2hiint(v));
  asm volatile("st.volatile.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(dst), "r"(lo), "r"(epoch), "r"(hi), "r"(epoch) : "memory");
}
__device__ __forceinline__ double xchg_wait_load(const uint4* src, unsigned epoch) {
  unsigned a, b, c, d;
  const long long t0 = clock64();
  for (;;) {
    asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "l"(src) : "memory");
    if (b == epoch && d == epoch) break;
    if (clock64() - t0 > 8000000000LL) __trap();   // a peer that never arrives must not hang this GPU
  }
  return __hiloint2double(static_cast<int>(c), static_cast<int>(a));
}
// this rank's partial v of entry j -> every peer; returns the rank-ordered sum over all ranks' partials of entry j
// (n: packets per rank and slot = 9C entries of q + 1 for the scalar p.q partial)
__device__ __forceinline__ double xchg_allsum(const XchgPeers& xg, int slot, unsigned epoch, int n, int j, double v) {
  const size_t base = static_cast<size_t>(slot) * xg.world * n;
#pragma unroll
  for (int p = 0; p < kMaxXchgRanks; ++p)
    if (p < xg.world && p != xg.rank) xchg_store(xg.buf[p] + base + static_cast<size_t>(xg.rank) * n + j, v, epoch);
  double acc = 0.0;
  for (int r = 0; r < xg.world; ++r)
    acc += (r == xg.rank) ? v : xchg_wait_load(xg.buf[xg.rank] + base + static_cast<size_t>(r) * n + j, epoch);
  return acc;
}

struct CgVecArgs {
  CgParams prm;
  int mode;
  int C;
  double* seed_target;         // non-null: this launch also writes the seed of the NEXT product there,
                               // seed_target = Df^2 * (p_new, or x_new in CG_RESET_FIRST)  (0 if Df is null)
  const double* Df;
  int precond;                 // 0 identity, 1 block-diagonal inverse blocks
  const double* minv;
  const double* rhs;
  double *x, *r, *z, *p, *q;   // q holds S*p (S*x_new in CG_RESET_SECOND)
  // explicit S (explicit_schur.cuh): q holds the product's row part; its column part is summed here from T (xs_col_sum).
  // Null: q is complete.
  const int* xs_col_ptr;
  const double* xs_T;
  double* red;                 // [gridDim.x][4] partial sums
  CgState* st;
  // p.q without a pass over q (single GPU, direct-flush products): pq_parts[0..num_pq_parts) hold p . (partial of S0 p)
  // from the product's CTAs, seed_pq[gridDim.x] the partials of sum D_f^2 p^2 this kernel wrote when it formed p.
  // Null: phase A computes p.q from q (one more grid sync).
  const double* pq_parts;
  int num_pq_parts;
  double* seed_pq;
  // Multi-GPU (observations sharded, cameras replicated): q = S p is the sum over ranks of the ranks' partial products.
  // The exchange happens INSIDE this kernel, NCCL-LL style: every thread packs its entries of this rank's partial (a.q)
  // into 16-byte packets {lo32, epoch, hi32, epoch} and stores them straight into every peer's exchange buffer
  // (peer-mapped pointers, NVLink), then polls its own buffer until the packets of all ranks carry the current epoch and
  // sums the partials in RANK ORDER -- the same order on every rank, so the replicated PCG state stays bit-identical.
  // No fences, no flags kernel, no collective: one NVLink write latency on top of the vector update.
  XchgPeers xg;                // xg.world == 0: single GPU / q already complete
  int xg_slot;
  unsigned xg_epoch;
};

// Sums up to three values over a CTA of kWarps warps with one barrier pair; results valid in every thread.
template <int kWarps = kCgThreads / 32>
__device__ __forceinline__ void cg_block_sum3(double& a, double& b, double& c, double (*scratch)[3]) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) {
    scratch[warp][0] = a;
    scratch[warp][1] = b;
    scratch[warp][2] = c;
  }
  __syncthreads();
  a = b = c = 0.0;
#pragma unroll
  for (int w = 0; w < kWarps; ++w) {
    a += scratch[w][0];
    b += scratch[w][1];
    c += scratch[w][2];
  }
}

// Fixed-order totals of slots [slot0, slot0 + count) over all CTAs' partials; every thread gets them.
__device__ __forceinline__ void cg_totals(const double* red, int nb, int slot0, int count, double* out, double* s_tot) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (warp < count) {
    double acc = 0.0;
    for (int b = lane; b < nb; b += 32) acc += __ldcg(red + b * 4 + slot0 + warp);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) s_tot[warp] = acc;
  }
  __syncthreads();
  for (int k = 0; k < count; ++k) out[k] = s_tot[k];
}

// The reference's tests of one PCG iteration (conjugate_gradients_solver.h:162-299), shared by cg_vector_kernel and the
// resident PCG (xs_pcg.cuh).  Every CTA evaluates them on identical totals, so every CTA takes the same branch; `writer`
// (one thread of the grid) publishes the state the host reads.
//
// p.q of iteration `it`: false when the solve stops here, else alpha = rho_old / p.q.
__device__ __forceinline__ bool cg_alpha(double pq, double rho_old, int it, CgState* st, bool writer, double* alpha) {
  int term = 0, reason = 0;
  if (!(pq > 0.0) || isinf(pq)) {
    term = isnan(pq) ? 2 : 1;
    reason = 6;
  } else {
    *alpha = rho_old / pq;
    if (!isinf(*alpha)) return true;
    term = 2;
    reason = 7;
  }
  if (writer) {
    st->pq = pq;
    st->done = 1;
    st->termination = term;
    st->reason = reason;
    st->iteration = it;
  }
  return false;
}

// Phase C: the termination tests of iteration `it` (or, `begin`, of the initial residual) on the totals x.(b+r), r.r and
// r.z, then the rho / beta checks of iteration it + 1.  False when the solve ends here; otherwise beta (0 for it == 0),
// the Q0 and |r| tolerance the next iteration tests against, and the state of the next iteration published.
__device__ __forceinline__ bool cg_phase_c(const CgParams& prm, bool begin, int it, double rho_old, double Q0, double tol_r,
                                           double dotQ, double sqR, double rho_new, CgState* st, bool writer, double* beta,
                                           double* Q0_next, double* tol_r_next) {
  const double norm_r = sqrt(sqR);
  *Q0_next = 0.0;
  *tol_r_next = tol_r;
  if (begin) {
    if (writer) {
      st->norm_rhs = norm_r;
      st->tol_r = prm.r_tolerance * norm_r;
      st->norm_r = norm_r;
      st->Q0 = 0.0;
      st->iteration = 0;
      st->done = 0;
      st->termination = 1;
      st->reason = 0;
      st->last_rho = 1.0;
    }
    const double tol0 = prm.r_tolerance * norm_r;
    *tol_r_next = tol0;
    if (norm_r == 0.0 || (prm.min_iterations == 0 && norm_r <= tol0)) {
      if (writer) {
        st->done = 1;
        st->termination = 0;
        st->reason = norm_r == 0.0 ? 8 : 2;
      }
      return false;
    }
  } else {
    // termination tests of iteration `it`
    const double Q1 = -dotQ;
    const double zeta = it * (Q1 - Q0) / Q1;
    int done = 0, term = 1, reason = 0;
    if (zeta < prm.q_tolerance && it >= prm.min_iterations) {
      done = 1; term = 0; reason = 1;
    } else if (norm_r <= tol_r && it >= prm.min_iterations) {
      done = 1; term = 0; reason = 2;
    } else if (it >= prm.max_iterations) {
      done = 1; term = 1; reason = 3;
    }
    if (done) {
      if (writer) {
        st->norm_r = norm_r;
        st->iteration = it;
        st->done = 1;
        st->termination = term;
        st->reason = reason;
      }
      return false;
    }
    *Q0_next = Q1;
  }
  // rho / beta checks of iteration it + 1
  *beta = 0.0;
  int fail_reason = 0;
  if (zero_or_inf(rho_new) || isnan(rho_new)) {
    fail_reason = 4;
  } else if (it >= 1) {
    *beta = rho_new / rho_old;
    if (zero_or_inf(*beta)) fail_reason = 5;
  }
  if (fail_reason) {
    if (writer) {
      st->iteration = it + 1;
      st->done = 1;
      st->termination = 2;
      st->reason = fail_reason;
    }
    return false;
  }
  if (writer) {
    st->norm_r = norm_r;
    st->last_rho = rho_old;
    st->rho = rho_new;
    st->Q0 = *Q0_next;
    st->iteration = it;
  }
  return true;
}

// The next search direction p = z + beta p (p = z in the first iteration), one expression for every kernel that forms it.
__device__ __forceinline__ double cg_next_p(int it, double z, double beta, double p) { return it == 0 ? z : __fma_rn(beta, p, z); }

__global__ void __launch_bounds__(kCgThreads) cg_vector_kernel(CgVecArgs a) {
  cg::grid_group grid = cg::this_grid();
  // (A/B on hardware, round 2: an ordinary launch with a grid barrier in global memory was 3 % slower per CG iteration than
  //  this cooperative launch, and launching it as a programmatic dependent of the product bought nothing on top.)
  __shared__ double scratch[kCgThreads / 32][3];
  __shared__ double s_tot[4];
  __shared__ double s_r[kCgCamsPerCta * 9];
  // lets a product kernel launched with programmatic stream serialisation start its prologue now (it waits for this
  // grid's completion before it touches anything this kernel writes)
  asm volatile("griddepcontrol.launch_dependents;");
  CgState* st = a.st;
  const int mode = a.mode;
  // state of the previous iteration, read before anybody rewrites it; all the loads that do not depend on a grid-wide
  // result are issued together (one L2 round trip), the done test comes after them
  const int st_done = __ldcg(&st->done);
  const double st_rho = __ldcg(&st->rho), Q0 = __ldcg(&st->Q0), tol_r = __ldcg(&st->tol_r);
  const int st_it = __ldcg(&st->iteration);
  const int tid = threadIdx.x;
  const int n = a.prm.n;
  const int nblocks = (a.C + kCgCamsPerCta - 1) / kCgCamsPerCta;
  const bool lane_ok = tid < kCgCamsPerCta * 9;
  const bool writer = (blockIdx.x == 0 && tid == 0);
  // Fast path: one camera block per CTA (grid == nblocks) — entries stay in registers across the phases.
  const bool single = (gridDim.x >= nblocks);
  const int j0 = blockIdx.x * kCgCamsPerCta * 9 + tid;
  const bool ok0 = single && lane_ok && j0 < n && blockIdx.x < nblocks;

  // operands that do not depend on grid-wide results: fetch them now
  double pj = 0.0, qj = 0.0, xj = 0.0, rj = 0.0, bj = 0.0, dj = 0.0;
  double mrow[9];
  double pq_pre = 0.0;  // this lane's share of the fused p.q partials (warps 0 and 1)
  if (ok0) {
    bj = a.rhs[j0];
    if (mode != CG_BEGIN) {
      pj = a.p[j0];
      xj = a.x[j0];
      if (mode != CG_RESET_SECOND) rj = a.r[j0];
    }
    if (a.Df != nullptr) dj = a.Df[j0];
    if (a.precond != 0 && mode != CG_RESET_FIRST) {
      const int cl = tid / 9, row = tid - 9 * cl;
      const double* m = a.minv + 81 * static_cast<size_t>(blockIdx.x * kCgCamsPerCta + cl) + 9 * row;
#pragma unroll
      for (int k = 0; k < 9; ++k) mrow[k] = m[k];
    }
  }
  if (a.pq_parts != nullptr && (mode == CG_NORMAL || mode == CG_RESET_FIRST)) {
    const int warp = tid >> 5, lane = tid & 31;
    if (warp == 0) {
      for (int b = lane; b < a.num_pq_parts; b += 32) pq_pre += __ldcg(a.pq_parts + b);
    } else if (warp == 1) {
      for (int b = lane; b < static_cast<int>(gridDim.x); b += 32) pq_pre += __ldcg(a.seed_pq + b);
    }
  }
  // q of entry j: the product's output, plus the column part of an explicit-S product
  auto load_q = [&](int j) -> double {
    const double q = __ldcg(a.q + j);
    return a.xs_T != nullptr ? xs_col_sum(a.xs_col_ptr, a.xs_T, j, q) : q;
  };
  if (ok0 && mode != CG_BEGIN && a.xg.world <= 1) qj = load_q(j0);

  if (mode != CG_BEGIN && st_done) return;
  if (a.xg.world > 1 && mode != CG_BEGIN) {
    // exchange + rank-ordered sum of the partial products (replaces qj / a.q)
    if (single) {
      if (ok0) {
        qj = xchg_allsum(a.xg, a.xg_slot, a.xg_epoch, n + 1, j0, __ldcg(a.q + j0));
        a.q[j0] = qj;
      }
    } else {
      for (int blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
        const int j = blk * kCgCamsPerCta * 9 + tid;
        if (lane_ok && j < n) a.q[j] = xchg_allsum(a.xg, a.xg_slot, a.xg_epoch, n + 1, j, __ldcg(a.q + j));
      }
    }
  }
  const double rho_old = (mode == CG_BEGIN) ? 1.0 : st_rho;
  const int it = (mode == CG_BEGIN) ? 0 : st_it + (mode == CG_RESET_SECOND ? 0 : 1);

  // ------------------------------------------------------------------ phase A: p.q
  const bool fused_pq = a.pq_parts != nullptr;
  if ((mode == CG_NORMAL || mode == CG_RESET_FIRST) && !fused_pq) {
    double acc = 0.0, d1 = 0.0, d2 = 0.0;
    if (single) {
      acc = pj * qj;
    } else {
      for (int blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
        const int j = blk * kCgCamsPerCta * 9 + tid;
        if (lane_ok && j < n) acc += a.p[j] * load_q(j);
      }
    }
    cg_block_sum3(acc, d1, d2, scratch);
    if (tid == 0) a.red[blockIdx.x * 4 + 0] = acc;
    grid.sync();
  }

  // ------------------------------------------------------------------ phase B
  double alpha = 0.0;
  if (mode == CG_NORMAL || mode == CG_RESET_FIRST) {
    double pq;
    if (fused_pq) {
      // fixed-order sum of the product's per-CTA partials and of this kernel's own seed partials
      const int warp = tid >> 5, lane = tid & 31;
      __syncthreads();
      if (warp < 2) {
        double acc = pq_pre;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) s_tot[warp] = acc;
      }
      __syncthreads();
      pq = s_tot[0] + s_tot[1];
      if (a.xg.world > 1) {
        // sharded: that was this rank's share of p.q (its partial product dotted with p; the D_f^2 term lives on rank 0);
        // the ranks' shares travel as one more packet (index n) and are summed in rank order like the entries of q
        __syncthreads();
        if (tid == 0) s_tot[2] = xchg_allsum(a.xg, a.xg_slot, a.xg_epoch, n + 1, n, pq);
        __syncthreads();
        pq = s_tot[2];
      }
    } else {
      cg_totals(a.red, gridDim.x, 0, 1, &pq, s_tot);
    }
    if (!cg_alpha(pq, rho_old, it, st, writer, &alpha)) return;  // every CTA takes this branch together
  }
  double zj = 0.0;
  {
    double accQ = 0.0, accR = 0.0, accRho = 0.0;
    for (int blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
      const int j = blk * kCgCamsPerCta * 9 + tid;
      const bool ok = lane_ok && j < n;
      if (ok && !single) {  // generic path: operands from memory
        bj = a.rhs[j];
        if (mode != CG_BEGIN) {
          pj = a.p[j];
          qj = load_q(j);
          xj = a.x[j];
          if (mode != CG_RESET_SECOND) rj = a.r[j];
        }
        dj = a.Df != nullptr ? a.Df[j] : 0.0;
      }
      if (ok) {
        if (mode == CG_BEGIN) {
          xj = 0.0;
          rj = bj;
          a.x[j] = 0.0;
        } else if (mode == CG_RESET_SECOND) {
          rj = bj - qj;                       // r = b - S x   (q holds S x here)
        } else {
          xj += alpha * pj;
          a.x[j] = xj;
          rj -= alpha * qj;
          if (mode == CG_RESET_FIRST && a.seed_target != nullptr) a.seed_target[j] = dj * dj * xj;
        }
        if (mode != CG_RESET_FIRST) {
          a.r[j] = rj;
          accQ += xj * (bj + rj);
          accR += rj * rj;
        }
      }
      if (mode != CG_RESET_FIRST) {
        __syncthreads();
        if (lane_ok) s_r[tid] = ok ? rj : 0.0;
        __syncthreads();
        if (ok) {
          if (a.precond == 0) {
            zj = rj;
          } else {
            const int cl = tid / 9;
            const double* rc = s_r + 9 * cl;
            if (!single) {
              const int row = tid - 9 * cl;
              const double* m = a.minv + 81 * static_cast<size_t>(blk * kCgCamsPerCta + cl) + 9 * row;
#pragma unroll
              for (int k = 0; k < 9; ++k) mrow[k] = m[k];
            }
            zj = 0.0;
#pragma unroll
            for (int k = 0; k < 9; ++k) zj += mrow[k] * rc[k];
          }
          a.z[j] = zj;
          accRho += rj * zj;
        }
      }
    }
    if (mode == CG_RESET_FIRST) {
      if (writer) {
        st->alpha = alpha;
        st->iteration = it;   // iteration `it` is half done; the second half reads it back
      }
      return;
    }
    cg_block_sum3(accQ, accR, accRho, scratch);
    if (tid == 0) {
      a.red[blockIdx.x * 4 + 1] = accQ;
      a.red[blockIdx.x * 4 + 2] = accR;
      a.red[blockIdx.x * 4 + 3] = accRho;
    }
  }
  grid.sync();

  // ------------------------------------------------------------------ phase C
  double tot[3];
  cg_totals(a.red, gridDim.x, 1, 3, tot, s_tot);
  // termination tests, then the rho / beta checks of iteration it + 1 and the state of the next launch; then p
  double beta = 0.0, Q0_next = 0.0, tol_next = 0.0;
  if (!cg_phase_c(a.prm, mode == CG_BEGIN, it, rho_old, Q0, tol_r, tot[0], tot[1], tot[2], st, writer, &beta, &Q0_next,
                  &tol_next))
    return;
  double seed_acc = 0.0;
  if (single) {
    if (ok0) {
      const double pn = cg_next_p(it, zj, beta, pj);
      a.p[j0] = pn;
      if (a.seed_target != nullptr) a.seed_target[j0] = dj * dj * pn;
      seed_acc = dj * dj * pn * pn;
    }
  } else {
    for (int blk = blockIdx.x; blk < nblocks; blk += gridDim.x) {
      const int j = blk * kCgCamsPerCta * 9 + tid;
      if (lane_ok && j < n) {
        const double pn = cg_next_p(it, a.z[j], beta, a.p[j]);
        a.p[j] = pn;
        const double d = a.Df != nullptr ? a.Df[j] : 0.0;
        if (a.seed_target != nullptr) a.seed_target[j] = d * d * pn;
        seed_acc += d * d * pn * pn;
      }
    }
  }
  if (a.seed_pq != nullptr) {
    double d1 = 0.0, d2 = 0.0;
    cg_block_sum3(seed_acc, d1, d2, scratch);
    if (tid == 0) a.seed_pq[blockIdx.x] = seed_acc;
  }
}

}  // namespace b200
