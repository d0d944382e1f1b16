// Tile kernels of libb200ba (sm_90a).  One CTA processes one tile (<= kTile rows = whole points) per
// loop iteration; E/F cells are staged into shared memory by TMA bulk copies (UBLKCP) and read back with
// conflict-free 128-bit LDS; per-point quantities are reduced in shared memory inside the tile (points never
// straddle tiles, so there is no cross-CTA traffic for the e blocks); camera-sized results are accumulated
// with FP64 RED atomics into L2-resident vectors.
//
// Kernel            reference function it replaces (internal/ceres/ unless noted)
//  evaluate_kernel   ProgramEvaluator::Evaluate program_evaluator.h:137-304 + ResidualBlock::Evaluate
//                    residual_block.cc:70-198 + SnavelyReprojectionError (examples/snavely_reprojection_error.h:57-92,
//                    include/ceres/rotation.h:864-930) + the loss and its Corrector (loss.cuh)
//  sqnorm_kernel     BlockSparseMatrix::SquaredColumnNorm block_sparse_matrix.cc:351-401
//  scale_kernel      BlockSparseMatrix::ScaleColumns :403-450
//  jmul_kernel       BlockSparseMatrix::RightMultiplyAndAccumulate :239-274
//  jtmul_kernel      BlockSparseMatrix::LeftMultiplyAndAccumulate :278-349 (and J'J x in one pass)
//  schur_init_kernel ImplicitSchurComplement::Init implicit_schur_complement.cc:49-97 (UpdateBlockDiagonalEtE
//                    partitioned_matrix_view_impl.h:447-523, AddDiagonalAndInvert :179-204, UpdateRhs :251-276)
//  schur_mul_kernel  ImplicitSchurComplement::RightMultiplyAndAccumulate :106-144 — the four partitioned SpMVs
//                    (partitioned_matrix_view_impl.h:113-375) fused into one pass over J
//  schur_diag_kernel SchurEliminator<2,3,9>::Eliminate against a block-diagonal lhs
//                    (schur_eliminator_impl.h:184-311,449-568; schur_jacobi_preconditioner.cc:87-97)
//  ftf_diag_kernel   PartitionedMatrixView::UpdateBlockDiagonalFtF :531-658 (JACOBI preconditioner)
//  backsub_kernel    ImplicitSchurComplement::BackSubstitute :208-243
#pragma once
#include <math_constants.h>

#include "common.cuh"
#include "loss.cuh"

namespace b200 {

// ------------------------------------------------------------------------------------------------
// Snavely reprojection residual and its analytic Jacobian.  The derivative is that of the very
// expression the reference differentiates with Jet<double,12> (Rodrigues formula away from theta==0,
// first-order R = I + [w]x at exactly zero), so it agrees with the autodiff Jacobian to rounding.
// jc = d r / d camera, row-major [2][9];  jp = d r / d point, row-major [2][3].
// ------------------------------------------------------------------------------------------------
template <bool kWantJ>
__device__ __forceinline__ void snavely(const double* __restrict__ cam, double X0, double X1, double X2, double ox,
                                        double oy, double& r0, double& r1, double* jc, double* jp) {
  const double w0 = cam[0], w1 = cam[1], w2 = cam[2];
  const double theta = norm3d(w0, w1, w2);
  double p0, p1, p2;
  double R[9], dpw[9];
  if (theta != 0.0) {
    double s, c;
    sincos(theta, &s, &c);
    const double ti = 1.0 / theta;
    const double a0 = w0 * ti, a1 = w1 * ti, a2 = w2 * ti;
    const double cx0 = a1 * X2 - a2 * X1, cx1 = a2 * X0 - a0 * X2, cx2 = a0 * X1 - a1 * X0;
    const double d = a0 * X0 + a1 * X1 + a2 * X2;
    const double omc = 1.0 - c;
    const double tmp = d * omc;
    p0 = X0 * c + cx0 * s + a0 * tmp;
    p1 = X1 * c + cx1 * s + a1 * tmp;
    p2 = X2 * c + cx2 * s + a2 * tmp;
    if (kWantJ) {
      R[0] = c + omc * a0 * a0;
      R[1] = -s * a2 + omc * a0 * a1;
      R[2] = s * a1 + omc * a0 * a2;
      R[3] = s * a2 + omc * a1 * a0;
      R[4] = c + omc * a1 * a1;
      R[5] = -s * a0 + omc * a1 * a2;
      R[6] = -s * a1 + omc * a2 * a0;
      R[7] = s * a0 + omc * a2 * a1;
      R[8] = c + omc * a2 * a2;
      const double a[3] = {a0, a1, a2};
      const double X[3] = {X0, X1, X2};
      const double cx[3] = {cx0, cx1, cx2};
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        const double aj = a[j];
        // d(axis)/d(w_j) = (e_j - axis * axis_j) / theta
        const double da0 = ((j == 0 ? 1.0 : 0.0) - a0 * aj) * ti;
        const double da1 = ((j == 1 ? 1.0 : 0.0) - a1 * aj) * ti;
        const double da2 = ((j == 2 ? 1.0 : 0.0) - a2 * aj) * ti;
        const double dcx0 = da1 * X2 - da2 * X1, dcx1 = da2 * X0 - da0 * X2, dcx2 = da0 * X1 - da1 * X0;
        const double dd = da0 * X0 + da1 * X1 + da2 * X2;
        const double dtmp = dd * omc + d * s * aj;
        const double msa = -s * aj, ca = c * aj;
        dpw[0 + j] = X[0] * msa + dcx0 * s + cx[0] * ca + da0 * tmp + a0 * dtmp;
        dpw[3 + j] = X[1] * msa + dcx1 * s + cx[1] * ca + da1 * tmp + a1 * dtmp;
        dpw[6 + j] = X[2] * msa + dcx2 * s + cx[2] * ca + da2 * tmp + a2 * dtmp;
      }
    }
  } else {
    p0 = X0 + (w1 * X2 - w2 * X1);
    p1 = X1 + (w2 * X0 - w0 * X2);
    p2 = X2 + (w0 * X1 - w1 * X0);
    if (kWantJ) {
      R[0] = 1.0; R[1] = -w2; R[2] = w1;
      R[3] = w2;  R[4] = 1.0; R[5] = -w0;
      R[6] = -w1; R[7] = w0;  R[8] = 1.0;
      dpw[0] = 0.0; dpw[1] = X2;  dpw[2] = -X1;
      dpw[3] = -X2; dpw[4] = 0.0; dpw[5] = X0;
      dpw[6] = X1;  dpw[7] = -X0; dpw[8] = 0.0;
    }
  }
  p0 += cam[3];
  p1 += cam[4];
  p2 += cam[5];
  const double ip2 = 1.0 / p2;
  const double xp = -p0 * ip2, yp = -p1 * ip2;
  const double l1 = cam[7], l2 = cam[8], f = cam[6];
  const double r2 = xp * xp + yp * yp;
  const double dist = 1.0 + r2 * (l1 + l2 * r2);
  const double fd = f * dist;
  r0 = fd * xp - ox;
  r1 = fd * yp - oy;
  if (kWantJ) {
    const double ddist = l1 + 2.0 * l2 * r2;  // d dist / d r2
    // d r2 / d p = (-2 xp, -2 yp, -2 r2) / p2
    const double q0 = -2.0 * xp * ip2, q1 = -2.0 * yp * ip2, q2 = -2.0 * r2 * ip2;
    const double fx = f * ddist * xp, fy = f * ddist * yp;
    // A = d predicted / d p   (2x3)
    const double A00 = fx * q0 - fd * ip2, A01 = fx * q1, A02 = fx * q2 - fd * xp * ip2;
    const double A10 = fy * q0, A11 = fy * q1 - fd * ip2, A12 = fy * q2 - fd * yp * ip2;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      jc[k] = A00 * dpw[k] + A01 * dpw[3 + k] + A02 * dpw[6 + k];
      jc[9 + k] = A10 * dpw[k] + A11 * dpw[3 + k] + A12 * dpw[6 + k];
      jp[k] = A00 * R[k] + A01 * R[3 + k] + A02 * R[6 + k];
      jp[3 + k] = A10 * R[k] + A11 * R[3 + k] + A12 * R[6 + k];
    }
    jc[3] = A00; jc[4] = A01; jc[5] = A02;
    jc[12] = A10; jc[13] = A11; jc[14] = A12;
    jc[6] = dist * xp;
    jc[15] = dist * yp;
    const double fr2 = f * r2;
    jc[7] = fr2 * xp;
    jc[16] = fr2 * yp;
    jc[8] = fr2 * r2 * xp;
    jc[17] = fr2 * r2 * yp;
  }
}

// The packed state of one block, as the evaluate kernels read it (b200_set_constant_blocks, b200_set_subset_manifolds):
// kBlockConstant for a constant block (a full SubsetManifold included), else bit k = coordinate k held by a SubsetManifold.
constexpr uint16_t kBlockConstant = 0x8000;

struct EvalArgs {
  const double* state;   // [3P+9C]
  double* residuals;     // [2N] or null
  double* gradient;      // [3P+9C] or null; camera part must be zeroed by the caller
  double* sqnorm;        // [3P+9C] or null, evaluate_v2_kernel only; camera part zeroed by the caller: squared column
                         // norms of the Jacobian as written
  double* cost_partial;  // [num_tiles] (evaluate_kernel) or [num_ctas] (evaluate_v2_kernel)
  const double* scale;   // null or [3P+9C]: Jacobi scaling fused into the Jacobian write (J <- J diag(scale))
  int* fail_flag;        // set to 1 on a non-finite residual/Jacobian entry
  LossArgs loss;
  const uint16_t* block_state;  // [P + C] points then cameras, read with kFixed only: the packed states (kBlockConstant)
};

// One row of both evaluate kernels: residual and Jacobian (kWantJ) at point pt_begin + lpt (the tile's first point and
// the row's index within the tile, kept apart so that the kFixed instantiations keep their registers) and camera `cam`,
// the constant blocks and coordinates (kFixed), the finiteness check, the loss and the residual store.  Returns the
// row's cost.  The order is Ceres':
// - a constant block's cells are zeroed before the check: Ceres evaluates it with jacobians[i] == nullptr;
// - a coordinate held by a SubsetManifold is zeroed after it: Ceres checks the ambient Jacobian before it multiplies by
//   the 0/1 PlusJacobian (residual_block.cc:85-159).  The Corrector is linear per column, so before or after it is the
//   same.
// The caller takes the gradient from the returned row, then applies the Jacobi scaling (scale_row).
template <int kLoss, bool kWantJ, bool kFixed>
__device__ __forceinline__ double evaluate_row(const ProblemView& p, const EvalArgs& a, size_t row, int pt_begin, int lpt,
                                               int cam, double& r0, double& r1, double (&jc)[18], double (&jp)[6]) {
  const double* X = a.state + 3 * static_cast<size_t>(pt_begin + lpt);
  const double* cp = a.state + 3 * static_cast<size_t>(p.P) + 9 * static_cast<size_t>(cam);
  const double2 o = *reinterpret_cast<const double2*>(p.obs + 2 * row);
  snavely<kWantJ>(cp, X[0], X[1], X[2], o.x, o.y, r0, r1, jc, jp);
  uint32_t mp = 0, mc = 0;
  if (kFixed && kWantJ) {
    mp = __ldg(a.block_state + pt_begin + lpt);
    mc = __ldg(a.block_state + p.P + cam);
    if (mp & kBlockConstant) {
#pragma unroll
      for (int k = 0; k < 6; ++k) jp[k] = 0.0;
    }
    if (mc & kBlockConstant) {
#pragma unroll
      for (int k = 0; k < 18; ++k) jc[k] = 0.0;
    }
  }
  bool finite = isfinite(r0) && isfinite(r1);
  if (kWantJ) {
#pragma unroll
    for (int k = 0; k < 18; ++k) finite = finite && isfinite(jc[k]);
#pragma unroll
    for (int k = 0; k < 6; ++k) finite = finite && isfinite(jp[k]);
  }
  if (!finite) atomicExch(a.fail_flag, 1);
  if (kFixed && kWantJ && ((mp | mc) & 0x1ffu) != 0) {
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      const bool m = (mp >> k) & 1u;
      jp[k] = m ? 0.0 : jp[k];
      jp[3 + k] = m ? 0.0 : jp[3 + k];
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const bool m = (mc >> k) & 1u;
      jc[k] = m ? 0.0 : jc[k];
      jc[9 + k] = m ? 0.0 : jc[9 + k];
    }
  }
  const double cost = apply_loss<kLoss, kWantJ>(row_loss_entry<kLoss>(a.loss, row), r0, r1, jc, jp);
  if (a.residuals != nullptr) *reinterpret_cast<double2*>(a.residuals + 2 * row) = make_double2(r0, r1);
  return cost;
}

// The fused Jacobi scaling of one row, J <- J diag(scale).
__device__ __forceinline__ void scale_row(const double* scale, int P, int pt, int cam, double (&jc)[18], double (&jp)[6]) {
  const double* sp = scale + 3 * static_cast<size_t>(pt);
  const double* sc = scale + 3 * static_cast<size_t>(P) + 9 * static_cast<size_t>(cam);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double v = sp[k];
    jp[k] *= v;
    jp[3 + k] *= v;
  }
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const double v = sc[k];
    jc[k] *= v;
    jc[9 + k] *= v;
  }
}

// kStoreJ = false (gradient without the Jacobian): J is computed, checked and used for the gradient, but the stored
// Jacobian is left as it is.  A template parameter, so that the instantiation the LM loop runs is the same code.
// kLoss: the class of the handle's loss set (loss.cuh).
// kFixed: the handle holds blocks or coordinates constant (evaluate_row).  Their columns are stored, summed into the
// gradient and scaled as 0: the columns Program::RemoveFixedBlocks and the PlusJacobian leave out.
// a.sqnorm is not read: sqnorm_kernel forms the column norms of these tiles.
template <int kLoss, bool kWantJ, bool kStoreJ = kWantJ, bool kFixed = false>
__global__ void __launch_bounds__(kTile) evaluate_kernel(ProblemView p, EvalArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const TileSmem s = carve_smem<3, 1>(smem_raw);
  tile_prologue(s);
  const int tid = threadIdx.x;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileDesc d = p.tiles[tile];
    tile_begin(p, d, s, false, false);
    double cost = 0.0;
    const bool active = tid < d.obs_count;
    double r0 = 0.0, r1 = 0.0;
    double jc[18], jp[6];
    int cam = 0, lpt = 0;
    if (active) {
      cam = s.sCam[tid];
      lpt = s.sSlotPt[tid];
      const size_t row = static_cast<size_t>(d.obs_begin) + tid;
      cost = evaluate_row<kLoss, kWantJ, kFixed>(p, a, row, d.pt_begin, lpt, cam, r0, r1, jc, jp);
      if (kWantJ) {
        if (a.gradient != nullptr) {
          // g += J_i' r_i  (program_evaluator.h:242-259), taken before the column scaling
          double* gc = a.gradient + 3 * static_cast<size_t>(p.P) + 9 * static_cast<size_t>(cam);
#pragma unroll
          for (int k = 0; k < 9; ++k) red_add(gc + k, jc[k] * r0 + jc[9 + k] * r1);
#pragma unroll
          for (int k = 0; k < 3; ++k) s.sObs[tid * 3 + k] = jp[k] * r0 + jp[3 + k] * r1;
        }
        if (a.scale != nullptr) scale_row(a.scale, p.P, d.pt_begin + lpt, cam, jc, jp);
#pragma unroll
        for (int k = 0; k < 3; ++k) *reinterpret_cast<double2*>(s.sE + tid * 6 + 2 * k) = make_double2(jp[2 * k], jp[2 * k + 1]);
#pragma unroll
        for (int k = 0; k < 9; ++k) *reinterpret_cast<double2*>(s.sF + tid * 18 + 2 * k) = make_double2(jc[2 * k], jc[2 * k + 1]);
      }
    }
    if (kWantJ) {
      fence_proxy_async_smem();
      __syncthreads();
      if (kStoreJ && tid == 0) {
        bulk_s2g(p.E() + 6 * static_cast<size_t>(d.obs_begin), s.sE, d.obs_count * 48u);
        bulk_s2g(p.F() + 18 * static_cast<size_t>(d.obs_begin), s.sF, d.obs_count * 144u);
        bulk_commit();
      }
      if (a.gradient != nullptr && tid < d.pt_count) {
        double g0 = 0.0, g1 = 0.0, g2 = 0.0;
        const int e = s.sPtOfs[tid + 1];
        for (int j = s.sPtOfs[tid]; j < e; ++j) {
          g0 += s.sObs[j * 3 + 0];
          g1 += s.sObs[j * 3 + 1];
          g2 += s.sObs[j * 3 + 2];
        }
        double* gp = a.gradient + 3 * static_cast<size_t>(d.pt_begin + tid);
        if (d.chunk) {
          red_add(gp, g0);
          red_add(gp + 1, g1);
          red_add(gp + 2, g2);
        } else {
          gp[0] = g0;
          gp[1] = g1;
          gp[2] = g2;
        }
      }
    }
    const double total = block_sum<kTile>(cost, s.sPt);
    if (tid == 0) {
      a.cost_partial[tile] = total;
      if (kWantJ) bulk_wait_read_all();
    }
    __syncthreads();
  }
  if (kWantJ && tid == 0) bulk_wait_all();
}

// ------------------------------------------------------------------------------------------------
// Squared column norms of J: point part reduced inside the tile, camera part by RED.
// out: [3P+9C]; the camera part must be zeroed by the caller.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTile) sqnorm_kernel(ProblemView p, double* out) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const TileSmem s = carve_smem<3, 1>(smem_raw);
  tile_prologue(s);
  const int tid = threadIdx.x;
  uint32_t parity = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileDesc d = p.tiles[tile];
    tile_begin(p, d, s, true, true);
    mbar_wait(s.bar, parity);
    parity ^= 1;
    if (tid < d.obs_count) {
      const double* e = s.sE + tid * 6;
      const double2 e0 = lds2(e), e1 = lds2(e + 2), e2 = lds2(e + 4);  // row0: e0.x e0.y e1.x ; row1: e1.y e2.x e2.y
      s.sObs[tid * 3 + 0] = e0.x * e0.x + e1.y * e1.y;
      s.sObs[tid * 3 + 1] = e0.y * e0.y + e2.x * e2.x;
      s.sObs[tid * 3 + 2] = e1.x * e1.x + e2.y * e2.y;
      double f[18];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 v = lds2(s.sF + tid * 18 + 2 * k);
        f[2 * k] = v.x;
        f[2 * k + 1] = v.y;
      }
      double* oc = out + 3 * static_cast<size_t>(p.P) + 9 * static_cast<size_t>(s.sCam[tid]);
#pragma unroll
      for (int k = 0; k < 9; ++k) red_add(oc + k, f[k] * f[k] + f[9 + k] * f[9 + k]);
    }
    __syncthreads();
    if (tid < d.pt_count) {
      double g0 = 0.0, g1 = 0.0, g2 = 0.0;
      const int e = s.sPtOfs[tid + 1];
      for (int j = s.sPtOfs[tid]; j < e; ++j) {
        g0 += s.sObs[j * 3 + 0];
        g1 += s.sObs[j * 3 + 1];
        g2 += s.sObs[j * 3 + 2];
      }
      double* op = out + 3 * static_cast<size_t>(d.pt_begin + tid);
      if (d.chunk) {
        red_add(op, g0);
        red_add(op + 1, g1);
        red_add(op + 2, g2);
      } else {
        op[0] = g0;
        op[1] = g1;
        op[2] = g2;
      }
    }
    __syncthreads();
  }
}

// Zeroes the stored cells of constant components (fixed: [3P+9C], nonzero on the components of constant blocks and on
// coordinates held by a SubsetManifold), column by column.  Same flat walk as scale_kernel: E cell [2][3] as 3 double2,
// element e -> column e % 3; F cell [2][9] as 9 double2, element e -> column e % 9.
__global__ void __launch_bounds__(256) fixed_mask_kernel(ProblemView p, const uint8_t* __restrict__ fixed) {
  const size_t nE2 = 3 * static_cast<size_t>(p.N), nF2 = 9 * static_cast<size_t>(p.N);
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  double2* E2 = reinterpret_cast<double2*>(p.E());
  double2* F2 = reinterpret_cast<double2*>(p.F());
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nE2 + nF2; i += stride) {
    const bool e_cell = i < nE2;
    const size_t j = e_cell ? i : i - nE2;
    const int w = e_cell ? 3 : 9, el = 2 * static_cast<int>(j % w);
    const uint8_t* f = e_cell ? fixed + 3 * static_cast<size_t>(p.pt_of_row[j / 3])
                              : fixed + 3 * static_cast<size_t>(p.P) + 9 * static_cast<size_t>(p.cam_idx[j / 9]);
    const bool zx = f[el % w] != 0, zy = f[(el + 1) % w] != 0;
    if (!zx && !zy) continue;
    double2* c = e_cell ? E2 + j : F2 + j;
    double2 v = *c;
    if (zx) v.x = 0.0;
    if (zy) v.y = 0.0;
    *c = v;
  }
}

// J <- J diag(scale): flat, fully coalesced read-modify-write of the value array, one double2 per step.
// E cell [2][3] as 3 double2: (00 01)(02 10)(11 12);  F cell [2][9] as 9 double2: element e -> column e % 9.
__global__ void __launch_bounds__(256) scale_kernel(ProblemView p, const double* __restrict__ scale) {
  const size_t nE2 = 3 * static_cast<size_t>(p.N);  // double2 elements in E
  const size_t nF2 = 9 * static_cast<size_t>(p.N);
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  double2* E2 = reinterpret_cast<double2*>(p.E());
  double2* F2 = reinterpret_cast<double2*>(p.F());
  for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < nE2 + nF2; i += stride) {
    if (i < nE2) {
      const size_t row = i / 3;
      const int k = static_cast<int>(i - row * 3) * 2;  // element 0, 2, 4 of the 2x3 cell
      const double* sp = scale + 3 * static_cast<size_t>(p.pt_of_row[row]);
      double2 v = E2[i];
      v.x *= sp[k % 3];
      v.y *= sp[(k + 1) % 3];
      E2[i] = v;
    } else {
      const size_t j = i - nE2;
      const size_t row = j / 9;
      const int k = static_cast<int>(j - row * 9) * 2;  // element 0..16 of the 2x9 cell
      const double* sc = scale + 3 * static_cast<size_t>(p.P) + 9 * static_cast<size_t>(p.cam_idx[row]);
      double2 v = F2[j];
      v.x *= sc[k % 9];
      v.y *= sc[(k + 1) % 9];
      F2[j] = v;
    }
  }
}

// model_cost_change = -(J step)'(r + J step / 2)   (trust_region_minimizer.cc:430-438) without materialising
// J*step: per-tile partial sums, reduced in fixed order afterwards.
__global__ void __launch_bounds__(kTile) model_cost_kernel(ProblemView p, const double* __restrict__ step,
                                                           const double* __restrict__ residuals, double* partial) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const TileSmem s = carve_smem<1, 1>(smem_raw);
  tile_prologue(s);
  const int tid = threadIdx.x;
  uint32_t parity = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileDesc d = p.tiles[tile];
    tile_begin(p, d, s, true, true);
    double xc[9], xp[3], r0 = 0.0, r1 = 0.0;
    const bool active = tid < d.obs_count;
    if (active) {
      const double* xcp = step + 3 * static_cast<size_t>(p.P) + 9 * static_cast<size_t>(s.sCam[tid]);
#pragma unroll
      for (int k = 0; k < 9; ++k) xc[k] = xcp[k];
      const double* xpp = step + 3 * static_cast<size_t>(d.pt_begin + s.sSlotPt[tid]);
#pragma unroll
      for (int k = 0; k < 3; ++k) xp[k] = xpp[k];
      const double2 v = *reinterpret_cast<const double2*>(residuals + 2 * (static_cast<size_t>(d.obs_begin) + tid));
      r0 = v.x;
      r1 = v.y;
    }
    mbar_wait(s.bar, parity);
    parity ^= 1;
    double acc = 0.0;
    if (active) {
      const double* e = s.sE + tid * 6;
      const double2 e0 = lds2(e), e1 = lds2(e + 2), e2 = lds2(e + 4);
      double t0 = e0.x * xp[0] + e0.y * xp[1] + e1.x * xp[2];
      double t1 = e1.y * xp[0] + e2.x * xp[1] + e2.y * xp[2];
      double f[18];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 v = lds2(s.sF + tid * 18 + 2 * k);
        f[2 * k] = v.x;
        f[2 * k + 1] = v.y;
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        t0 += f[k] * xc[k];
        t1 += f[9 + k] * xc[k];
      }
      acc = -(t0 * (r0 + t0 / 2.0) + t1 * (r1 + t1 / 2.0));
    }
    const double total = block_sum<kTile>(acc, s.sPt);
    if (tid == 0) partial[tile] = total;
    __syncthreads();
  }
}

// DOGLEG's one pass over J per Gauss-Newton step (dogleg_strategy.cc:185-194, :699-714): with a = g / diagonal and
// b = gn / diagonal, the per-tile partials of |J a|^2 and, when gn != nullptr, of |J b|^2 and (J a).(J b), stored at
// partial[k * num_tiles + tile] and reduced in fixed order afterwards.
__global__ void __launch_bounds__(kTile) dogleg_gram_kernel(ProblemView p, const double* __restrict__ g,
                                                            const double* __restrict__ gn,
                                                            const double* __restrict__ diagonal, double* partial) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const TileSmem s = carve_smem<1, 1>(smem_raw);
  tile_prologue(s);
  const int tid = threadIdx.x;
  const bool two = gn != nullptr;
  uint32_t parity = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileDesc d = p.tiles[tile];
    tile_begin(p, d, s, true, true);
    double ac[9], ap[3], bc[9], bp[3];
    const bool active = tid < d.obs_count;
    if (active) {
      const size_t oc = 3 * static_cast<size_t>(p.P) + 9 * static_cast<size_t>(s.sCam[tid]);
      const size_t op = 3 * static_cast<size_t>(d.pt_begin + s.sSlotPt[tid]);
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double dk = diagonal[oc + k];
        ac[k] = g[oc + k] / dk;
        bc[k] = two ? gn[oc + k] / dk : 0.0;
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double dk = diagonal[op + k];
        ap[k] = g[op + k] / dk;
        bp[k] = two ? gn[op + k] / dk : 0.0;
      }
    }
    mbar_wait(s.bar, parity);
    parity ^= 1;
    double aa = 0.0, bb = 0.0, ab = 0.0;
    if (active) {
      const double* e = s.sE + tid * 6;
      const double2 e0 = lds2(e), e1 = lds2(e + 2), e2 = lds2(e + 4);
      const double ev[6] = {e0.x, e0.y, e1.x, e1.y, e2.x, e2.y};
      double t0 = 0.0, t1 = 0.0, u0 = 0.0, u1 = 0.0;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        t0 += ev[k] * ap[k];
        t1 += ev[3 + k] * ap[k];
        u0 += ev[k] * bp[k];
        u1 += ev[3 + k] * bp[k];
      }
      double f[18];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 v = lds2(s.sF + tid * 18 + 2 * k);
        f[2 * k] = v.x;
        f[2 * k + 1] = v.y;
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        t0 += f[k] * ac[k];
        t1 += f[9 + k] * ac[k];
        u0 += f[k] * bc[k];
        u1 += f[9 + k] * bc[k];
      }
      aa = t0 * t0 + t1 * t1;
      bb = u0 * u0 + u1 * u1;
      ab = t0 * u0 + t1 * u1;
    }
    const double taa = block_sum<kTile>(aa, s.sPt);
    if (tid == 0) partial[tile] = taa;
    if (two) {
      const double tbb = block_sum<kTile>(bb, s.sPt);
      const double tab = block_sum<kTile>(ab, s.sPt);
      if (tid == 0) {
        partial[static_cast<size_t>(p.num_tiles) + tile] = tbb;
        partial[2 * static_cast<size_t>(p.num_tiles) + tile] = tab;
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// y += J x  (rows are independent; x = [points | cameras])
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTile) jmul_kernel(ProblemView p, const double* __restrict__ x, double* y) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const TileSmem s = carve_smem<1, 1>(smem_raw);
  tile_prologue(s);
  const int tid = threadIdx.x;
  uint32_t parity = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileDesc d = p.tiles[tile];
    tile_begin(p, d, s, true, true);
    double xc[9], xp[3];
    if (tid < d.obs_count) {
      const double* xcp = x + 3 * static_cast<size_t>(p.P) + 9 * static_cast<size_t>(s.sCam[tid]);
#pragma unroll
      for (int k = 0; k < 9; ++k) xc[k] = xcp[k];
      const double* xpp = x + 3 * static_cast<size_t>(d.pt_begin + s.sSlotPt[tid]);
#pragma unroll
      for (int k = 0; k < 3; ++k) xp[k] = xpp[k];
    }
    mbar_wait(s.bar, parity);
    parity ^= 1;
    if (tid < d.obs_count) {
      const double* e = s.sE + tid * 6;
      const double2 e0 = lds2(e), e1 = lds2(e + 2), e2 = lds2(e + 4);
      double t0 = e0.x * xp[0] + e0.y * xp[1] + e1.x * xp[2];
      double t1 = e1.y * xp[0] + e2.x * xp[1] + e2.y * xp[2];
      double f[18];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 v = lds2(s.sF + tid * 18 + 2 * k);
        f[2 * k] = v.x;
        f[2 * k + 1] = v.y;
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        t0 += f[k] * xc[k];
        t1 += f[9 + k] * xc[k];
      }
      double2* yp = reinterpret_cast<double2*>(y + 2 * (static_cast<size_t>(d.obs_begin) + tid));
      double2 v = *yp;
      v.x += t0;
      v.y += t1;
      *yp = v;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// kNormal == false:  y += J' r          (r: [2N] rows)
// kNormal == true :  y  = J'(J x) + D^2 x   in ONE pass over J (the J'J x bandwidth kernel)
// Point part of y is owned by the tile (plain stores); camera part accumulates with RED: for kNormal the
// caller pre-initialises y_cam = D_cam^2 x_cam (or zero).
// ------------------------------------------------------------------------------------------------
template <bool kNormal>
__global__ void __launch_bounds__(kTile)
    jtmul_kernel(ProblemView p, const double* __restrict__ x, const double* __restrict__ D, double* y) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const TileSmem s = carve_smem<3, 1>(smem_raw);
  tile_prologue(s);
  const int tid = threadIdx.x;
  uint32_t parity = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileDesc d = p.tiles[tile];
    tile_begin(p, d, s, true, true);
    double xc[9], xp[3];
    double t0 = 0.0, t1 = 0.0;
    const bool active = tid < d.obs_count;
    if (active) {
      if (kNormal) {
        const double* xcp = x + 3 * static_cast<size_t>(p.P) + 9 * static_cast<size_t>(s.sCam[tid]);
#pragma unroll
        for (int k = 0; k < 9; ++k) xc[k] = xcp[k];
        const double* xpp = x + 3 * static_cast<size_t>(d.pt_begin + s.sSlotPt[tid]);
#pragma unroll
        for (int k = 0; k < 3; ++k) xp[k] = xpp[k];
      } else {
        const double2 v = *reinterpret_cast<const double2*>(x + 2 * (static_cast<size_t>(d.obs_begin) + tid));
        t0 = v.x;
        t1 = v.y;
      }
    }
    mbar_wait(s.bar, parity);
    parity ^= 1;
    if (active) {
      const double* e = s.sE + tid * 6;
      const double2 e0 = lds2(e), e1 = lds2(e + 2), e2 = lds2(e + 4);
      double f[18];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 v = lds2(s.sF + tid * 18 + 2 * k);
        f[2 * k] = v.x;
        f[2 * k + 1] = v.y;
      }
      if (kNormal) {
        t0 = e0.x * xp[0] + e0.y * xp[1] + e1.x * xp[2];
        t1 = e1.y * xp[0] + e2.x * xp[1] + e2.y * xp[2];
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          t0 += f[k] * xc[k];
          t1 += f[9 + k] * xc[k];
        }
      }
      s.sObs[tid * 3 + 0] = e0.x * t0 + e1.y * t1;
      s.sObs[tid * 3 + 1] = e0.y * t0 + e2.x * t1;
      s.sObs[tid * 3 + 2] = e1.x * t0 + e2.y * t1;
      double* yc = y + 3 * static_cast<size_t>(p.P) + 9 * static_cast<size_t>(s.sCam[tid]);
#pragma unroll
      for (int k = 0; k < 9; ++k) red_add(yc + k, f[k] * t0 + f[9 + k] * t1);
    }
    __syncthreads();
    if (tid < d.pt_count) {
      double g0 = 0.0, g1 = 0.0, g2 = 0.0;
      const int e = s.sPtOfs[tid + 1];
      for (int j = s.sPtOfs[tid]; j < e; ++j) {
        g0 += s.sObs[j * 3 + 0];
        g1 += s.sObs[j * 3 + 1];
        g2 += s.sObs[j * 3 + 2];
      }
      const size_t o = 3 * static_cast<size_t>(d.pt_begin + tid);
      if (d.chunk) {
        // slice of a huge point: accumulate (kNormal: into the entry the caller zeroed; the D^2 x term once, with the
        // slice that holds the point's first row)
        if (kNormal && D != nullptr && p.pt_ptr[d.pt_begin] == d.obs_begin) {
          g0 += D[o] * D[o] * x[o];
          g1 += D[o + 1] * D[o + 1] * x[o + 1];
          g2 += D[o + 2] * D[o + 2] * x[o + 2];
        }
        red_add(y + o, g0);
        red_add(y + o + 1, g1);
        red_add(y + o + 2, g2);
      } else if (kNormal) {
        if (D != nullptr) {
          g0 += D[o] * D[o] * x[o];
          g1 += D[o + 1] * D[o + 1] * x[o + 1];
          g2 += D[o + 2] * D[o + 2] * x[o + 2];
        }
        y[o] = g0;
        y[o + 1] = g1;
        y[o + 2] = g2;
      } else {
        y[o] += g0;
        y[o + 1] += g1;
        y[o + 2] += g2;
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// Symmetric 3x3 helpers.  (E'E + D^2)^-1 is stored as its 6 unique entries [00 01 02 11 12 22].
// inverse via Cholesky solve against I, as the reference does with selfadjointView<Upper>().llt().solve(I)
// (implicit_schur_complement.cc:201-202).
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void invert_sym3_llt(const double m[6], double inv[6]) {
  const double l00 = sqrt(m[0]);
  const double l10 = m[1] / l00, l20 = m[2] / l00;
  const double l11 = sqrt(m[3] - l10 * l10);
  const double l21 = (m[4] - l20 * l10) / l11;
  const double l22 = sqrt(m[5] - l20 * l20 - l21 * l21);
  // L^-1 (lower)
  const double i00 = 1.0 / l00, i11 = 1.0 / l11, i22 = 1.0 / l22;
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

struct SchurState {
  const double* b;   // [2N] residuals (rhs of the least squares problem)
  const double* D;   // [3P+9C] or null
  double* ete_inv;   // [6P]
  double* rhs;       // [9C]  zeroed by the caller
  double* ye;        // scratch [3P]: (E'E)^-1 E'b  (kept for tests / back-substitution reuse)
};

// EtE_inv[k] = (sum_i E_i'E_i + D_k^2)^-1 ;  rhs += F_i'(b_i - E_i EtE_inv E'b)
__global__ void __launch_bounds__(kTile) schur_init_kernel(ProblemView p, SchurState st) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const TileSmem s = carve_smem<9, 3>(smem_raw);
  tile_prologue(s);
  const int tid = threadIdx.x;
  uint32_t parity = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileDesc d = p.tiles[tile];
    if (d.chunk) continue;  // slice of a huge point: huge_kernels.cuh
    tile_begin(p, d, s, true, true);
    const bool active = tid < d.obs_count;
    double b0 = 0.0, b1 = 0.0;
    if (active) {
      const double2 v = *reinterpret_cast<const double2*>(st.b + 2 * (static_cast<size_t>(d.obs_begin) + tid));
      b0 = v.x;
      b1 = v.y;
    }
    mbar_wait(s.bar, parity);
    parity ^= 1;
    double2 e0, e1, e2;
    if (active) {
      const double* e = s.sE + tid * 6;
      e0 = lds2(e); e1 = lds2(e + 2); e2 = lds2(e + 4);
      double* o = s.sObs + tid * 9;
      o[0] = e0.x * e0.x + e1.y * e1.y;  // 00
      o[1] = e0.x * e0.y + e1.y * e2.x;  // 01
      o[2] = e0.x * e1.x + e1.y * e2.y;  // 02
      o[3] = e0.y * e0.y + e2.x * e2.x;  // 11
      o[4] = e0.y * e1.x + e2.x * e2.y;  // 12
      o[5] = e1.x * e1.x + e2.y * e2.y;  // 22
      o[6] = e0.x * b0 + e1.y * b1;      // E'b
      o[7] = e0.y * b0 + e2.x * b1;
      o[8] = e1.x * b0 + e2.y * b1;
    }
    __syncthreads();
    if (tid < d.pt_count) {
      double m[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) m[k] = 0.0;
      const int e = s.sPtOfs[tid + 1];
      for (int j = s.sPtOfs[tid]; j < e; ++j) {
#pragma unroll
        for (int k = 0; k < 9; ++k) m[k] += s.sObs[j * 9 + k];
      }
      const size_t pt = static_cast<size_t>(d.pt_begin + tid);
      if (st.D != nullptr) {
        const double d0 = st.D[3 * pt], d1 = st.D[3 * pt + 1], d2 = st.D[3 * pt + 2];
        m[0] += d0 * d0;
        m[3] += d1 * d1;
        m[5] += d2 * d2;
      }
      double inv[6];
      invert_sym3_llt(m, inv);
#pragma unroll
      for (int k = 0; k < 6; ++k) st.ete_inv[6 * pt + k] = inv[k];
      const double v0 = inv[0] * m[6] + inv[1] * m[7] + inv[2] * m[8];
      const double v1 = inv[1] * m[6] + inv[3] * m[7] + inv[4] * m[8];
      const double v2 = inv[2] * m[6] + inv[4] * m[7] + inv[5] * m[8];
      s.sPt[tid * 3 + 0] = v0;
      s.sPt[tid * 3 + 1] = v1;
      s.sPt[tid * 3 + 2] = v2;
      if (st.ye != nullptr) {
        st.ye[3 * pt] = v0;
        st.ye[3 * pt + 1] = v1;
        st.ye[3 * pt + 2] = v2;
      }
    }
    __syncthreads();
    if (active) {
      const double* v = s.sPt + s.sSlotPt[tid] * 3;
      const double t0 = b0 - (e0.x * v[0] + e0.y * v[1] + e1.x * v[2]);
      const double t1 = b1 - (e1.y * v[0] + e2.x * v[1] + e2.y * v[2]);
      double f[18];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 w = lds2(s.sF + tid * 18 + 2 * k);
        f[2 * k] = w.x;
        f[2 * k + 1] = w.y;
      }
      double* rc = st.rhs + 9 * static_cast<size_t>(s.sCam[tid]);
#pragma unroll
      for (int k = 0; k < 9; ++k) red_add(rc + k, f[k] * t0 + f[9 + k] * t1);
    }
    __syncthreads();
  }
}

// y += F'(F x - E (E'E+D^2)^-1 E'F x): the implicit Schur complement product, one pass over J.
// The caller pre-initialises y = D_f^2 x (or zero).  x, y: [9C].
__global__ void __launch_bounds__(kTile)
    schur_mul_kernel(ProblemView p, const double* __restrict__ ete_inv, const double* __restrict__ x, double* y,
                     const int* __restrict__ done_flag) {
  if (done_flag != nullptr && *done_flag != 0) return;  // PCG already terminated: the launch is a no-op
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const TileSmem s = carve_smem<3, 3>(smem_raw);
  tile_prologue(s);
  const int tid = threadIdx.x;
  uint32_t parity = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileDesc d = p.tiles[tile];
    if (d.chunk) continue;  // slice of a huge point: huge_kernels.cuh
    tile_begin(p, d, s, true, true);
    const bool active = tid < d.obs_count;
    double xc[9];
    int cam = 0;
    if (active) {
      cam = s.sCam[tid];
      const double* xcp = x + 9 * static_cast<size_t>(cam);
#pragma unroll
      for (int k = 0; k < 9; ++k) xc[k] = xcp[k];
    }
    double pinv[6];
    if (tid < d.pt_count) {
      const double* pi = ete_inv + 6 * static_cast<size_t>(d.pt_begin + tid);
#pragma unroll
      for (int k = 0; k < 6; ++k) pinv[k] = pi[k];
    }
    mbar_wait(s.bar, parity);
    parity ^= 1;
    double t0 = 0.0, t1 = 0.0;
    double2 e0, e1, e2;
    if (active) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {  // F row 0 is elements 0..8, row 1 is 9..17; element 8|9 share a double2
        const double2 a = lds2(s.sF + tid * 18 + 2 * k);
        t0 += a.x * xc[2 * k] + a.y * xc[2 * k + 1];
      }
      {
        const double2 a = lds2(s.sF + tid * 18 + 8);
        t0 += a.x * xc[8];
        t1 += a.y * xc[0];
      }
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const double2 a = lds2(s.sF + tid * 18 + 10 + 2 * k);
        t1 += a.x * xc[2 * k + 1] + a.y * xc[2 * k + 2];
      }
      const double* e = s.sE + tid * 6;
      e0 = lds2(e); e1 = lds2(e + 2); e2 = lds2(e + 4);
      s.sObs[tid * 3 + 0] = e0.x * t0 + e1.y * t1;
      s.sObs[tid * 3 + 1] = e0.y * t0 + e2.x * t1;
      s.sObs[tid * 3 + 2] = e1.x * t0 + e2.y * t1;
    }
    __syncthreads();
    if (tid < d.pt_count) {
      double u0 = 0.0, u1 = 0.0, u2 = 0.0;
      const int e = s.sPtOfs[tid + 1];
      for (int j = s.sPtOfs[tid]; j < e; ++j) {
        u0 += s.sObs[j * 3 + 0];
        u1 += s.sObs[j * 3 + 1];
        u2 += s.sObs[j * 3 + 2];
      }
      s.sPt[tid * 3 + 0] = -(pinv[0] * u0 + pinv[1] * u1 + pinv[2] * u2);
      s.sPt[tid * 3 + 1] = -(pinv[1] * u0 + pinv[3] * u1 + pinv[4] * u2);
      s.sPt[tid * 3 + 2] = -(pinv[2] * u0 + pinv[4] * u1 + pinv[5] * u2);
    }
    __syncthreads();
    if (active) {
      const double* v = s.sPt + s.sSlotPt[tid] * 3;
      t0 += e0.x * v[0] + e0.y * v[1] + e1.x * v[2];
      t1 += e1.y * v[0] + e2.x * v[1] + e2.y * v[2];
      double f[18];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 w = lds2(s.sF + tid * 18 + 2 * k);
        f[2 * k] = w.x;
        f[2 * k + 1] = w.y;
      }
      double* yc = y + 9 * static_cast<size_t>(cam);
#pragma unroll
      for (int k = 0; k < 9; ++k) red_add(yc + k, f[k] * t0 + f[9 + k] * t1);
    }
    __syncthreads();
  }
}

// y_e = (E'E+D^2)^-1 E'(b - F z);   z: [9C], y_e: [3P]
__global__ void __launch_bounds__(kTile) backsub_kernel(ProblemView p, const double* __restrict__ ete_inv,
                                                        const double* __restrict__ b, const double* __restrict__ z,
                                                        double* ye) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const TileSmem s = carve_smem<3, 1>(smem_raw);
  tile_prologue(s);
  const int tid = threadIdx.x;
  uint32_t parity = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileDesc d = p.tiles[tile];
    if (d.chunk) continue;  // slice of a huge point: huge_kernels.cuh
    tile_begin(p, d, s, true, true);
    const bool active = tid < d.obs_count;
    double zc[9], t0 = 0.0, t1 = 0.0;
    if (active) {
      const double* zp = z + 9 * static_cast<size_t>(s.sCam[tid]);
#pragma unroll
      for (int k = 0; k < 9; ++k) zc[k] = zp[k];
      const double2 v = *reinterpret_cast<const double2*>(b + 2 * (static_cast<size_t>(d.obs_begin) + tid));
      t0 = v.x;
      t1 = v.y;
    }
    mbar_wait(s.bar, parity);
    parity ^= 1;
    if (active) {
      double f[18];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 w = lds2(s.sF + tid * 18 + 2 * k);
        f[2 * k] = w.x;
        f[2 * k + 1] = w.y;
      }
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        t0 -= f[k] * zc[k];
        t1 -= f[9 + k] * zc[k];
      }
      const double* e = s.sE + tid * 6;
      const double2 e0 = lds2(e), e1 = lds2(e + 2), e2 = lds2(e + 4);
      s.sObs[tid * 3 + 0] = e0.x * t0 + e1.y * t1;
      s.sObs[tid * 3 + 1] = e0.y * t0 + e2.x * t1;
      s.sObs[tid * 3 + 2] = e1.x * t0 + e2.y * t1;
    }
    __syncthreads();
    if (tid < d.pt_count) {
      double u0 = 0.0, u1 = 0.0, u2 = 0.0;
      const int e = s.sPtOfs[tid + 1];
      for (int j = s.sPtOfs[tid]; j < e; ++j) {
        u0 += s.sObs[j * 3 + 0];
        u1 += s.sObs[j * 3 + 1];
        u2 += s.sObs[j * 3 + 2];
      }
      const size_t pt = static_cast<size_t>(d.pt_begin + tid);
      const double* pi = ete_inv + 6 * pt;
      ye[3 * pt + 0] = pi[0] * u0 + pi[1] * u1 + pi[2] * u2;
      ye[3 * pt + 1] = pi[1] * u0 + pi[3] * u1 + pi[4] * u2;
      ye[3 * pt + 2] = pi[2] * u0 + pi[4] * u1 + pi[5] * u2;
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------
// Block diagonal of the Schur complement (SCHUR_JACOBI) or of F'F (JACOBI):
//   kSchur: M_c += sum_{i in cam c} F_i'F_i - W_i' P_k buf_{k,c},  W_i = E_i'F_i,
//           buf_{k,c} = sum of W_j over the rows j of point k that see camera c  (schur_eliminator_impl.h:449-568;
//           normally a single row), P_k = (E'E + D^2)^-1.
// Only the upper triangle (45 entries, row-major packed) is accumulated; out: [45C], zeroed by the caller.
// ------------------------------------------------------------------------------------------------
template <bool kSchur>
__global__ void __launch_bounds__(kTile)
    diag_blocks_kernel(ProblemView p, const double* __restrict__ ete_inv, double* out45) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const TileSmem s = carve_smem<1, 1>(smem_raw);
  tile_prologue(s);
  const int tid = threadIdx.x;
  uint32_t parity = 0;
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const TileDesc d = p.tiles[tile];
    tile_begin(p, d, s, true, true);
    mbar_wait(s.bar, parity);
    parity ^= 1;
    if (tid < d.obs_count) {
      const int cam = s.sCam[tid];
      double f[18];
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double2 w = lds2(s.sF + tid * 18 + 2 * k);
        f[2 * k] = w.x;
        f[2 * k + 1] = w.y;
      }
      double W[27], PB[27];
      if (kSchur) {
        const int lpt = s.sSlotPt[tid];
        const double* e = s.sE + tid * 6;
        const double e00 = e[0], e01 = e[1], e02 = e[2], e10 = e[3], e11 = e[4], e12 = e[5];
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          W[k] = e00 * f[k] + e10 * f[9 + k];
          W[9 + k] = e01 * f[k] + e11 * f[9 + k];
          W[18 + k] = e02 * f[k] + e12 * f[9 + k];
        }
        double B[27];
#pragma unroll
        for (int k = 0; k < 27; ++k) B[k] = W[k];
        // other rows of the same point observing the same camera (duplicates are rare; loop is over <= degree)
        const int jb = s.sPtOfs[lpt], je = s.sPtOfs[lpt + 1];
        for (int j = jb; j < je; ++j) {
          if (j != tid && s.sCam[j] == cam) {
            const double* ej = s.sE + j * 6;
            const double* fj = s.sF + j * 18;
#pragma unroll
            for (int k = 0; k < 9; ++k) {
              B[k] += ej[0] * fj[k] + ej[3] * fj[9 + k];
              B[9 + k] += ej[1] * fj[k] + ej[4] * fj[9 + k];
              B[18 + k] += ej[2] * fj[k] + ej[5] * fj[9 + k];
            }
          }
        }
        const double* pi = ete_inv + 6 * static_cast<size_t>(d.pt_begin + lpt);
        const double p0 = pi[0], p1 = pi[1], p2 = pi[2], p3 = pi[3], p4 = pi[4], p5 = pi[5];
#pragma unroll
        for (int k = 0; k < 9; ++k) {
          PB[k] = p0 * B[k] + p1 * B[9 + k] + p2 * B[18 + k];
          PB[9 + k] = p1 * B[k] + p3 * B[9 + k] + p4 * B[18 + k];
          PB[18 + k] = p2 * B[k] + p4 * B[9 + k] + p5 * B[18 + k];
        }
      }
      double* oc = out45 + 45 * static_cast<size_t>(cam);
      int idx = 0;
#pragma unroll
      for (int a = 0; a < 9; ++a) {
#pragma unroll
        for (int bb = a; bb < 9; ++bb) {
          double m = f[a] * f[bb] + f[9 + a] * f[9 + bb];
          if (kSchur) m -= W[a] * PB[bb] + W[9 + a] * PB[9 + bb] + W[18 + a] * PB[18 + bb];
          red_add(oc + idx, m);
          ++idx;
        }
      }
    }
    __syncthreads();
  }
}

// One warp per camera: M = sym(upper45) + D_c^2; inverse by Cholesky solve against I, as the reference does with
// selfadjointView<Upper>().llt().solve(I) (block_random_access_diagonal_matrix.cc:90-100 / AddDiagonalAndInvert).
// blocks / inverse: [81C], either may be null.  The factor lives in shared memory; lanes 0..8 each solve one column.
constexpr int kInvWarps = 4;
__global__ void __launch_bounds__(32 * kInvWarps) invert9_kernel(int C, const double* __restrict__ upper45,
                                                                 const double* __restrict__ Df, double* blocks,
                                                                 double* inverse) {
  __shared__ double sM[kInvWarps][81];
  __shared__ double sL[kInvWarps][81];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x * kInvWarps + warp;
  if (c >= C) return;
  double* M = sM[warp];
  double* L = sL[warp];
  const double* u = upper45 + 45 * static_cast<size_t>(c);
  for (int e = lane; e < 81; e += 32) {
    const int a = e / 9, b = e - 9 * a;
    const int lo = a < b ? a : b, hi = a < b ? b : a;
    double v = u[lo * 9 - lo * (lo - 1) / 2 + (hi - lo)];
    if (a == b && Df != nullptr) v += Df[9 * static_cast<size_t>(c) + a] * Df[9 * static_cast<size_t>(c) + a];
    M[e] = v;
    L[e] = 0.0;
    if (blocks != nullptr) blocks[81 * static_cast<size_t>(c) + e] = v;
  }
  __syncwarp();
  if (inverse == nullptr) return;
  for (int j = 0; j < 9; ++j) {
    if (lane == 0) {
      double d = M[j * 9 + j];
      for (int k = 0; k < j; ++k) d -= L[j * 9 + k] * L[j * 9 + k];
      L[j * 9 + j] = sqrt(d);
    }
    __syncwarp();
    if (lane > j && lane < 9) {
      double sv = M[j * 9 + lane];
      for (int k = 0; k < j; ++k) sv -= L[lane * 9 + k] * L[j * 9 + k];
      L[lane * 9 + j] = sv / L[j * 9 + j];
    }
    __syncwarp();
  }
  if (lane < 9) {
    double yv[9], xv[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      double sv = (i == lane) ? 1.0 : 0.0;
#pragma unroll
      for (int k = 0; k < 9; ++k)
        if (k < i) sv -= L[i * 9 + k] * yv[k];
      yv[i] = sv / L[i * 9 + i];
    }
#pragma unroll
    for (int i = 8; i >= 0; --i) {
      double sv = yv[i];
#pragma unroll
      for (int k = 0; k < 9; ++k)
        if (k > i) sv -= L[k * 9 + i] * xv[k];
      xv[i] = sv / L[i * 9 + i];
    }
    double* inv = inverse + 81 * static_cast<size_t>(c);
#pragma unroll
    for (int i = 0; i < 9; ++i) inv[i * 9 + lane] = xv[i];
  }
}

}  // namespace b200
