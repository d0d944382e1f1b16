// The whole SCHUR_JACOBI PCG on an explicit S in one cooperative launch (DESIGN §3.2), for an S that fits the aggregate
// shared memory of the SMs.  One CTA per SM owns a contiguous range of block rows -- the cameras of those rows and their
// stored blocks -- and copies its blocks of S (each transposed, so that a step's loads conflict least) and its cameras'
// preconditioner blocks M^-1 into shared memory once per solve.  Each iteration is then
//   product  S p with S from shared memory (xs_walk, the arithmetic of xs_mul_kernel): the row part a_i of every owned
//            camera stays in shared memory, t_ij goes to T, and the CTA's share of p.q (plus sum D_f^2 p^2) to red[.][0]
//   ---- grid barrier ----
//   vector   on the owned cameras: q = (a + D_f^2 p) + the column part from T (xs_col_sum), p.q, alpha, x, r, z = M^-1 r,
//            and the partials of x.(b+r), r.r, r.z
//   ---- grid barrier ----
//   tests    the reference's termination and failure tests (cg_alpha, cg_phase_c) on identical fixed-order totals in
//            every CTA, beta, and the new p of the owned cameras.
// The product's steps are cut into one contiguous range per warp, balanced by steps plus one per row segment for its
// sum; a range may begin and end inside a row.  A row split over warps gets its first segment's sum in s_a and each
// later segment's in the segment scratch, and join_rows adds those into s_a in segment order once the walks are done.
// The product reads p_j of every column j its blocks touch.  A foreign column's p_j (j past the CTA's last row; only the
// upper triangle is stored) is not read back from its owner (that would need a third barrier): the CTA forms it itself
// from z_j and the previous p_j (cg_next_p, the owner's expression, so the bits agree), p double-buffered by iteration
// parity for that.  It does so for all its foreign columns at once, in the same pass that forms the owned cameras' new p,
// into a shared buffer: the walk then reads every x_j from shared memory, through the plan's CTA-local column index of
// each block ([owned cameras | foreign columns]), and its steps and column entries from copies the prologue makes, so
// it reads nothing from global memory.  Likewise the vector phase first copies the T slots of the owned
// columns (one contiguous range of T) into shared memory in one coalesced pass and sums each column from that copy, in
// every CTA whose slots fit the room the plan left (stage_slots); any other CTA sums from T in L2, in the same order.  A
// residual reset adds a barrier, the product on x (its foreign x_j gathered into the same buffer) and a second barrier,
// as CG_RESET_FIRST / CG_RESET_SECOND of the two-kernel loop do.  Every branch around a barrier is taken by the whole
// grid: it depends only on the iteration count and on totals every CTA sums in the same order.  Everything another CTA
// wrote during the launch (z, p, x, T, red) is read with ld.global.cg.  No atomics, and every sum has a fixed order: the
// solve is deterministic given its inputs.  S q is not bit-identical to xs_mul_kernel + xs_col_sum: a split row's part
// a_i is the sum of its segments' sums, where xs_mul_kernel sums the row in one warp.
#pragma once
#include "cg_kernel.cuh"

namespace b200 {

constexpr int kXpThreads = 512;
constexpr int kXpWarps = kXpThreads / 32;
// dynamic shared memory per CTA: S blocks, M^-1 blocks, seven vectors (x r p b D_f a z) of the owned cameras, the
// product's input [owned cameras | foreign columns], one split row's segment sum per warp, `slots` staged T slots; the
// product's steps and its blocks' column entries (int2); then the owned columns' col_ptr, the foreign columns' ids and
// the warps' first steps
inline size_t xs_pcg_smem_bytes(int max_blocks, int max_cams, int max_foreign, int max_steps, int slots) {
  return sizeof(double) * (81 * static_cast<size_t>(max_blocks) + (81 + 7 * 9) * static_cast<size_t>(max_cams) +
                           9 * static_cast<size_t>(max_cams + max_foreign) + 9 * kXpWarps + 9 * static_cast<size_t>(slots)) +
         sizeof(int2) * (static_cast<size_t>(max_steps) + static_cast<size_t>(max_blocks)) +
         sizeof(int) * (static_cast<size_t>(max_cams) + 1 + static_cast<size_t>(max_foreign) + kXpWarps + 1);
}

struct XsPcgArgs {
  XsView v;                   // v.cols: {CTA-local column, T slot} of every block (KernelPlan::xs_pcg_cols)
  CgParams prm;
  int reset;                  // residual reset period (iterations)
  const int2* cta;            // [grid + 1] {first block row, first block} of each CTA
  const int* warp_step;       // [grid * kXpWarps + 1] first product step of each warp
  const int* fptr;            // [grid + 1] each CTA's foreign columns in fcol
  const int* fcol;            // the foreign columns of each CTA, ascending
  int max_blocks, max_cams;   // the shared-memory geometry: the largest CTA's blocks and cameras,
  int max_foreign;            // ... the most foreign columns of a CTA
  int max_steps;              // ... and the most product steps of a CTA
  int stage_slots;            // a CTA whose owned columns have at most this many T slots sums them from shared memory
  const double* minv;         // [C][81] M^-1
  const double* rhs;          // [9C]
  const double* Df;           // [9C] or null
  double *x, *z;              // [9C]
  double* p[2];               // [9C] each: p of the even / odd iterations
  double* red;                // [grid][4] per-CTA partials: p.q | x.(b+r), r.r, r.z
  CgState* st;
#ifdef B200_DEV_KNOBS
  long long* stamps;          // B200_XS_STAMPS: clock64() cycles of CTA 0 by phase, accumulated over the solve (kXpPhases)
#endif
};

// phases of the stamps: prologue and CG_BEGIN, product, wait at barrier 1, vector phase (with a reset's product and
// barriers), wait at barrier 2, tests and the new p
constexpr int kXpPhases = 6;
#ifdef B200_DEV_KNOBS
#define XP_STAMP(k)                                                   \
  if (a.stamps != nullptr && blockIdx.x == 0 && threadIdx.x == 0) {   \
    const long long t_now = clock64();                                \
    a.stamps[k] += t_now - t_mark;                                    \
    t_mark = t_now;                                                   \
  }
#else
#define XP_STAMP(k)
#endif

__global__ void __launch_bounds__(kXpThreads, 1) xs_pcg_kernel(XsPcgArgs a) {
  cg::grid_group grid = cg::this_grid();
#ifdef B200_DEV_KNOBS
  long long t_mark = clock64();
#endif
  extern __shared__ double smem[];
  __shared__ double scratch[kXpWarps][3];
  __shared__ double s_tot[4];
  __shared__ int s_nfe;   // entries of the foreign columns (kept here: the product's walk needs every register)
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int e = lane / 9, w = lane - 9 * (lane / 9);   // e == 3: lanes 27..31, no block
  const int2 lo = a.cta[blockIdx.x], hi = a.cta[blockIdx.x + 1];
  const int r0 = lo.x, ncam = hi.x - lo.x, nent = 9 * ncam, b0 = lo.y, nblk = hi.y - lo.y;
  double* s_S = smem;
  double* s_minv = s_S + 81 * static_cast<size_t>(a.max_blocks);
  double* s_x = s_minv + 81 * static_cast<size_t>(a.max_cams);
  double* s_r = s_x + 9 * a.max_cams;
  double* s_p = s_r + 9 * a.max_cams;
  double* s_b = s_p + 9 * a.max_cams;
  double* s_d = s_b + 9 * a.max_cams;
  double* s_a = s_d + 9 * a.max_cams;
  double* s_z = s_a + 9 * a.max_cams;
  double* s_v = s_z + 9 * a.max_cams;                           // the product's input x_l at 9 l: [owned | foreign]
  double* s_seg = s_v + 9 * (a.max_cams + a.max_foreign);       // [kXpWarps][9] a split row's segment sum, by warp
  double* s_T = s_seg + 9 * kXpWarps;                           // T slots of the owned columns, from slot s_cp[0] on
  int2* s_steps = reinterpret_cast<int2*>(s_T + 9 * a.stage_slots);  // the CTA's product steps
  int2* s_cols = s_steps + a.max_steps;                               // column entries of its blocks
  int* s_cp = reinterpret_cast<int*>(s_cols + a.max_blocks);          // col_ptr[r0 .. r0 + ncam]
  int* s_fc = s_cp + a.max_cams + 1;                            // the foreign columns
  int* s_ws = s_fc + a.max_foreign;                             // [kXpWarps + 1] the warps' first steps
  const XsView& v = a.v;
  const int kc = __ldg(a.warp_step + blockIdx.x * kXpWarps);   // the CTA's first step
  XsView vs = v;                                                // the walk's view: steps and column entries staged
  vs.steps = s_steps - kc;
  vs.cols = s_cols - b0;
  const size_t o0 = 9 * static_cast<size_t>(r0);   // first owned entry
  const bool writer = blockIdx.x == 0 && tid == 0;
  const int k0 = __ldg(a.warp_step + blockIdx.x * kXpWarps + warp), k1 = __ldg(a.warp_step + blockIdx.x * kXpWarps + warp + 1);

  // ---- prologue: the CTA's blocks of S (contiguous: block rows own their blocks), each transposed (load_s), and M^-1
  // blocks, b and D_f
  {
    const double* src = v.S + 81 * static_cast<size_t>(b0);
    const int n = 81 * nblk;
    auto transposed = [](int i) {   // entry (u, w) of a block at 9 w + u
      const int b = i / 81, uw = i - 81 * b, u = uw / 9;
      return 81 * b + 9 * (uw - 9 * u) + u;
    };
    int i = tid;
    for (; i + 3 * kXpThreads < n; i += 4 * kXpThreads) {
      double t[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) t[k] = __ldcg(src + i + k * kXpThreads);
#pragma unroll
      for (int k = 0; k < 4; ++k) s_S[transposed(i + k * kXpThreads)] = t[k];
    }
    for (; i < n; i += kXpThreads) s_S[transposed(i)] = __ldcg(src + i);
    for (int k = tid; k < 81 * ncam; k += kXpThreads) s_minv[k] = __ldcg(a.minv + 81 * static_cast<size_t>(r0) + k);
    for (int k = tid; k <= ncam; k += kXpThreads) s_cp[k] = __ldg(v.col_ptr + r0 + k);
    const int nsteps = __ldg(a.warp_step + (blockIdx.x + 1) * kXpWarps) - kc;
    for (int k = tid; k < nsteps; k += kXpThreads) s_steps[k] = __ldg(v.steps + kc + k);
    for (int k = tid; k < nblk; k += kXpThreads) s_cols[k] = __ldg(v.cols + b0 + k);
    const int f0 = __ldg(a.fptr + blockIdx.x), nf = __ldg(a.fptr + blockIdx.x + 1) - f0;
    for (int k = tid; k < nf; k += kXpThreads) s_fc[k] = __ldg(a.fcol + f0 + k);
    if (tid == 0) s_nfe = 9 * nf;
    if (tid <= kXpWarps) s_ws[tid] = __ldg(a.warp_step + blockIdx.x * kXpWarps + tid);
  }
  for (int k = tid; k < nent; k += kXpThreads) {
    s_b[k] = a.rhs[o0 + k];
    s_d[k] = a.Df != nullptr ? a.Df[o0 + k] : 0.0;
    s_p[k] = 0.0;
  }
  // column w of block e of step d: 9 consecutive doubles of the transposed copy.  The three blocks' columns (blocks
  // 81 doubles apart) then fall on distinct banks but for pairs; a lane without a block reads lane w's address of the
  // step's first block (a broadcast, no further conflict)
  auto load_s = [&](int2 d, int e, int w, double* s) {
    const bool in = xs_lane_in(d, e);
    const double* sb = s_S + 81 * (xs_lane_in(d, 0) ? d.x + (in ? e : 0) - b0 : 0) + 9 * w;
#pragma unroll
    for (int u = 0; u < 9; ++u) s[u] = in ? sb[u] : 0.0;
  };
  // a warp whose range begins inside row i takes x_i from the product's input (the row is owned)
  auto load_xi = [&](int i, int u) { return s_v[9 * (i - r0) + u]; };
  // the sum of a row's blocks in this warp's range: a_i, or the first segment of a split row, into s_a; a later segment
  // (the range begins inside row i) into the warp's segment scratch
  auto keep_row = [&](int i, int u, double av, double) {
    const int2 d0 = vs.steps[k0];
    if (!(d0.y & kXsStepFirst) && (d0.y & kXsStepRowMask) == i) s_seg[9 * warp + u] = av;
    else s_a[9 * (i - r0) + u] = av;
  };
  // after the walks (and a CTA barrier): each split row gets its later segments added into s_a in warp order, by the 9
  // threads of the warp that holds its first segment
  auto join_rows = [&]() {
    if (tid >= 9 * kXpWarps) return;
    const int wv = tid / 9, u = tid - 9 * wv;
    const int ka = s_ws[wv], kb = s_ws[wv + 1];
    if (ka == kb) return;
    const int2 dl = vs.steps[kb - 1], df = vs.steps[ka];
    const int i = dl.y & kXsStepRowMask;
    if ((dl.y & kXsStepLast) || (!(df.y & kXsStepFirst) && (df.y & kXsStepRowMask) == i)) return;   // not a first segment
    double* out = s_a + 9 * (i - r0) + u;
    double acc = *out;
    for (int w2 = wv + 1; w2 < kXpWarps; ++w2) {
      const int kb2 = s_ws[w2 + 1];
      if (s_ws[w2] == kb2) continue;
      acc += s_seg[9 * w2 + u];
      const int2 d2 = vs.steps[kb2 - 1];
      if ((d2.y & kXsStepLast) || (d2.y & kXsStepRowMask) != i) break;
    }
    *out = acc;
  };
  // the owned columns' T slots into s_T, one coalesced pass (made visible by the caller's next __syncthreads), if they fit
  auto staged = [&]() { return s_cp[ncam] - s_cp[0] <= a.stage_slots; };
  auto stage_T = [&]() {
    if (!staged()) return;
    const int c0 = s_cp[0];
    const double* src = v.T + 9 * static_cast<size_t>(c0);
    const int n = 9 * (s_cp[ncam] - c0);
    int i = tid;
    for (; i + 7 * kXpThreads < n; i += 8 * kXpThreads) {
      double t[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) t[k] = __ldcg(src + i + k * kXpThreads);
#pragma unroll
      for (int k = 0; k < 8; ++k) s_T[i + k * kXpThreads] = t[k];
    }
    for (; i < n; i += kXpThreads) s_T[i] = __ldcg(src + i);
  };
  // q_k = init + the column part of owned entry k, from s_T or else from T (the same sum in the same order)
  auto col_sum = [&](bool from_s, int k, double init) {
    const int cl = k / 9;
    return from_s ? xs_col_sum<true>(s_T, s_cp[0], s_cp[cl], s_cp[cl + 1], k - 9 * cl, init)
                  : xs_col_sum(v.col_ptr, v.T, static_cast<int>(o0) + k, init);
  };
  // z = M^-1 r of the owned cameras (s_r complete), and the partials x.(b+r), r.r, r.z into red[CTA][1..3]
  auto precondition = [&]() {
    __syncthreads();
    double accQ = 0.0, accR = 0.0, accRho = 0.0;
    for (int k = tid; k < nent; k += kXpThreads) {
      const int cl = k / 9, row = k - 9 * cl;
      const double* m = s_minv + 81 * cl + 9 * row;
      const double* rc = s_r + 9 * cl;
      double zj = 0.0;
#pragma unroll
      for (int t = 0; t < 9; ++t) zj += m[t] * rc[t];
      s_z[k] = zj;
      a.z[o0 + k] = zj;
      const double xj = s_x[k], rj = s_r[k];
      accQ += xj * (s_b[k] + rj);
      accR += rj * rj;
      accRho += rj * zj;
    }
    cg_block_sum3<kXpWarps>(accQ, accR, accRho, scratch);
    if (tid == 0) {
      a.red[blockIdx.x * 4 + 1] = accQ;
      a.red[blockIdx.x * 4 + 2] = accR;
      a.red[blockIdx.x * 4 + 3] = accRho;
    }
  };

  // ---- CG_BEGIN: x = 0, r = b, z = M^-1 r
  for (int k = tid; k < nent; k += kXpThreads) {
    s_x[k] = 0.0;
    s_r[k] = s_b[k];
    a.x[o0 + k] = 0.0;
  }
  // The foreign entry of this thread's first pass (k = tid) of the p formation: z_j and the previous p_j, loaded right
  // after the barrier that makes z visible, so that these loads overlap the totals' instead of following the tests.
  int it = 0;
  double fz = 0.0, fp = 0.0;
  auto prefetch_foreign = [&]() {
    const int k = tid - nent;
    if (k < 0 || k >= s_nfe) return;
    const int fl = k / 9;
    const size_t o = 9 * static_cast<size_t>(s_fc[fl]) + (k - 9 * fl);
    fz = __ldcg(a.z + o);
    fp = __ldcg(a.p[it & 1] + o);
  };
  precondition();
  grid.sync();
  prefetch_foreign();
  double tot[3];
  cg_totals(a.red, gridDim.x, 1, 3, tot, s_tot);
  XP_STAMP(0);
  double rho = 1.0, Q0 = 0.0, tol_r = 0.0, beta = 0.0;
  if (!cg_phase_c(a.prm, true, 0, rho, Q0, tol_r, tot[0], tot[1], tot[2], a.st, writer, &beta, &Q0, &tol_r)) return;
  rho = tot[2];

  for (;;) {
    // ---- p of iteration it + 1: the owned cameras' (and their share of D_f^2 p.p), and in the threads past them the
    // foreign columns', from z and p of iteration it
    double pq = 0.0;
    const double* p_prev = a.p[it & 1];
    for (int k = tid; k < nent + s_nfe; k += kXpThreads) {
      if (k < nent) {
        const double pn = cg_next_p(it, s_z[k], beta, s_p[k]);
        s_p[k] = pn;
        s_v[k] = pn;
        a.p[(it + 1) & 1][o0 + k] = pn;
        pq += s_d[k] * s_d[k] * pn * pn;
      } else if (k < kXpThreads) {
        s_v[k] = cg_next_p(it, fz, beta, fp);
      } else {
        const int fl = (k - nent) / 9;
        const size_t o = 9 * static_cast<size_t>(s_fc[fl]) + (k - nent - 9 * fl);
        s_v[k] = cg_next_p(it, __ldcg(a.z + o), beta, __ldcg(p_prev + o));
      }
    }
    ++it;
    __syncthreads();
    // ---- product S p
    {
      XsWalk wk;
      xs_walk_begin<true>(vs, k0, k1, e, w, load_s, wk);
      pq += xs_walk<true>(vs, k0, k1, lane, e, w, load_s, [&](int l, int w) { return s_v[9 * l + w]; }, load_xi, keep_row, wk);
    }
    {
      double d1 = 0.0, d2 = 0.0;
      cg_block_sum3<kXpWarps>(pq, d1, d2, scratch);   // its barriers also end the walks
      if (tid == 0) a.red[blockIdx.x * 4] = pq;
    }
    join_rows();
    XP_STAMP(1);
    grid.sync();
    XP_STAMP(2);
    // ---- vector phase (cg_totals' __syncthreads make the staged T visible)
    double pq_tot, alpha = 0.0;
    const bool reset = it % a.reset == 0;
    if (!reset) stage_T();
    cg_totals(a.red, gridDim.x, 0, 1, &pq_tot, s_tot);
    if (!cg_alpha(pq_tot, rho, it, a.st, writer, &alpha)) return;
    const bool from_s = staged();
    for (int k = tid; k < nent; k += kXpThreads) {
      const double pj = s_p[k];
      double xj = s_x[k];
      xj += alpha * pj;
      s_x[k] = xj;
      a.x[o0 + k] = xj;
      if (reset) {
        s_v[k] = xj;
      } else {
        const double dj = s_d[k];
        const double q = col_sum(from_s, k, __dadd_rn(s_a[k], __dmul_rn(__dmul_rn(dj, dj), pj)));
        double rj = s_r[k];
        rj -= alpha * q;
        s_r[k] = rj;
      }
    }
    if (reset) {
      // r = b - S x: the product on x, its foreign columns read back from their owners
      grid.sync();
      for (int k = tid; k < s_nfe; k += kXpThreads) {
        const int fl = k / 9;
        s_v[nent + k] = __ldcg(a.x + 9 * static_cast<size_t>(s_fc[fl]) + (k - 9 * fl));
      }
      __syncthreads();
      {
        XsWalk wk;
        xs_walk_begin<true>(vs, k0, k1, e, w, load_s, wk);
        xs_walk<true>(vs, k0, k1, lane, e, w, load_s, [&](int l, int w) { return s_v[9 * l + w]; }, load_xi, keep_row, wk);
      }
      __syncthreads();
      join_rows();
      grid.sync();
      stage_T();
      __syncthreads();
      for (int k = tid; k < nent; k += kXpThreads) {
        const double dj = s_d[k];
        const double q = col_sum(from_s, k, __dadd_rn(s_a[k], __dmul_rn(__dmul_rn(dj, dj), s_x[k])));
        s_r[k] = s_b[k] - q;
      }
    }
    precondition();
    XP_STAMP(3);
    grid.sync();
    prefetch_foreign();
    XP_STAMP(4);
    // ---- tests of iteration it, beta
    cg_totals(a.red, gridDim.x, 1, 3, tot, s_tot);
    if (!cg_phase_c(a.prm, false, it, rho, Q0, tol_r, tot[0], tot[1], tot[2], a.st, writer, &beta, &Q0, &tol_r)) return;
    rho = tot[2];
    XP_STAMP(5);
  }
}

}  // namespace b200
