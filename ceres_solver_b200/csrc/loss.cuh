// Robust losses and the Corrector on the device: rho(s) of each class of include/ceres/loss_function.h
// (loss_function.cc), the ScaledLoss factor around it, and the correction of a row's residual and Jacobian
// (corrector.cc:41-155, applied as residual_block.cc:170-195 does).  One copy, used by evaluate_kernel and
// evaluate_v2_kernel.
//
// The evaluate kernels are instantiated for three classes of a handle's loss set (b200ba.cu: loss_class):
//   kLossTrivial  one trivial loss with scale 1, or the loss turned off: cost 0.5 s, no correction;
//   kLossHuber    one HuberLoss with scale 1;
//   kLossGeneral  anything else: a switch on the type per row.  One loss object comes in the kernel arguments; a table
//                 is read per row through the read-only path (4 B of index + one 40 B entry).
#pragma once
#include "../../include/b200ba.h"
#include "common.cuh"

namespace b200 {

enum LossClass : int { kLossTrivial = 0, kLossHuber = 1, kLossGeneral = 2 };

// One loss object as the kernels read it: the constants each class's constructor derives from its arguments, computed
// once on the host (b200ba.cu: make_loss_entry).
//   HUBER p = a, q = a^2;  SOFT_L_ONE, CAUCHY q = a^2, r = 1 / a^2;  ARCTAN p = a, q = 1 / a^2;
//   TOLERANT p = a, q = b, r = b log(1 + exp(-a / b));  TUKEY q = a^2;  TRIVIAL none.
struct LossEntry {
  double p, q, r, scale;
  int type;
};

struct LossArgs {
  LossEntry one;             // the loss of every row when row_loss is null
  const int* row_loss;       // null, or [N] table index of each row (internal row order): kLossGeneral only
  const LossEntry* table;
};

constexpr double kDblMin = 2.2250738585072014e-308;   // std::numeric_limits<double>::min(): the floor of rho'

__device__ __forceinline__ void huber_rho(double a, double b, double s, double (&rho)[3]) {
  if (s > b) {
    const double rr = sqrt(s);
    rho[0] = 2.0 * a * rr - b;
    rho[1] = fmax(kDblMin, a / rr);
    rho[2] = -rho[1] / (2.0 * s);
  } else {
    rho[0] = s;
    rho[1] = 1.0;
    rho[2] = 0.0;
  }
}

// {rho(s), rho'(s), rho''(s)} of one loss object, times its ScaledLoss factor.
__device__ __forceinline__ void loss_rho(const LossEntry& L, double s, double (&rho)[3]) {
  switch (L.type) {
    case B200_LOSS_HUBER:
      huber_rho(L.p, L.q, s, rho);
      break;
    case B200_LOSS_SOFT_L_ONE: {   // 2 a^2 (sqrt(1 + s / a^2) - 1)
      const double u = 1.0 + s * L.r;
      const double su = sqrt(u);
      rho[0] = 2.0 * L.q * (su - 1.0);
      rho[1] = fmax(kDblMin, 1.0 / su);
      rho[2] = -(L.r * rho[1]) / (2.0 * u);
      break;
    }
    case B200_LOSS_CAUCHY: {       // a^2 log(1 + s / a^2)
      const double u = 1.0 + s * L.r;
      const double iu = 1.0 / u;
      rho[0] = L.q * log(u);
      rho[1] = fmax(kDblMin, iu);
      rho[2] = -L.r * (iu * iu);
      break;
    }
    case B200_LOSS_ARCTAN: {       // a atan(s / a)
      const double u = 1.0 + s * s * L.q;
      const double iu = 1.0 / u;
      rho[0] = L.p * atan2(s, L.p);
      rho[1] = fmax(kDblMin, iu);
      rho[2] = -2.0 * s * L.q * (iu * iu);
      break;
    }
    case B200_LOSS_TOLERANT: {     // b log(1 + exp((s - a) / b)) - c
      const double x = (s - L.p) / L.q;
      if (x > 36.7) {              // beyond ln(2^53), 1 + e^x == e^x in double: log(1 + e^x) = x
        rho[0] = s - L.p - L.r;
        rho[1] = 1.0;
        rho[2] = 0.0;
      } else {
        const double ex = exp(x);
        rho[0] = L.q * log(1.0 + ex) - L.r;
        rho[1] = fmax(kDblMin, ex / (1.0 + ex));
        rho[2] = 0.5 / (L.q * (1.0 + cosh(x)));   // > 0: the Corrector's second-order branch
      }
      break;
    }
    case B200_LOSS_TUKEY:          // a^2 / 3 (1 - (1 - s / a^2)^3) inside, a^2 / 3 outside (rho' = 0 zeroes the row)
      if (s <= L.q) {
        const double v = 1.0 - s / L.q;
        const double v2 = v * v;
        rho[0] = L.q / 3.0 * (1.0 - v2 * v);
        rho[1] = v2;
        rho[2] = -2.0 / L.q * v;
      } else {
        rho[0] = L.q / 3.0;
        rho[1] = 0.0;
        rho[2] = 0.0;
      }
      break;
    default:                       // B200_LOSS_TRIVIAL
      rho[0] = s;
      rho[1] = 1.0;
      rho[2] = 0.0;
      break;
  }
  rho[0] *= L.scale;
  rho[1] *= L.scale;
  rho[2] *= L.scale;
}

// The loss object of a row.
template <int kLoss>
__device__ __forceinline__ LossEntry row_loss_entry(const LossArgs& l, size_t row) {
  if (kLoss != kLossGeneral || l.row_loss == nullptr) return l.one;
  const LossEntry* e = l.table + __ldg(l.row_loss + row);
  LossEntry L;
  L.p = __ldg(&e->p);
  L.q = __ldg(&e->q);
  L.r = __ldg(&e->r);
  L.scale = __ldg(&e->scale);
  L.type = __ldg(&e->type);
  return L;
}

// The loss of one row of residuals (r0, r1) and, with kWantJ, Jacobian jc [2][9] / jp [2][3]: returns the row's cost
// 0.5 rho(s) and leaves r and J corrected in place (Jacobian first, from the uncorrected residuals).
template <int kLoss, bool kWantJ>
__device__ __forceinline__ double apply_loss(const LossEntry& L, double& r0, double& r1, double* jc, double* jp) {
  const double sq = r0 * r0 + r1 * r1;
  if (kLoss == kLossTrivial) return 0.5 * sq;
  double rho[3];
  if (kLoss == kLossHuber) huber_rho(L.p, L.q, sq, rho);
  else loss_rho(L, sq, rho);
  const double sqrt_rho1 = sqrt(rho[1]);
  double residual_scaling, alpha_sq_norm;
  if (sq == 0.0 || rho[2] <= 0.0) {
    residual_scaling = sqrt_rho1;
    alpha_sq_norm = 0.0;
  } else {
    const double Dd = 1.0 + 2.0 * sq * rho[2] / rho[1];
    const double alpha = 1.0 - sqrt(Dd);
    residual_scaling = sqrt_rho1 / (1.0 - alpha);
    alpha_sq_norm = alpha / sq;
  }
  if (kWantJ) {
    if (alpha_sq_norm == 0.0) {
#pragma unroll
      for (int k = 0; k < 18; ++k) jc[k] *= sqrt_rho1;
#pragma unroll
      for (int k = 0; k < 6; ++k) jp[k] *= sqrt_rho1;
    } else {
#pragma unroll
      for (int k = 0; k < 9; ++k) {
        const double rtj = jc[k] * r0 + jc[9 + k] * r1;
        jc[k] = sqrt_rho1 * (jc[k] - alpha_sq_norm * r0 * rtj);
        jc[9 + k] = sqrt_rho1 * (jc[9 + k] - alpha_sq_norm * r1 * rtj);
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double rtj = jp[k] * r0 + jp[3 + k] * r1;
        jp[k] = sqrt_rho1 * (jp[k] - alpha_sq_norm * r0 * rtj);
        jp[3 + k] = sqrt_rho1 * (jp[3 + k] - alpha_sq_norm * r1 * rtj);
      }
    }
  }
  r0 *= residual_scaling;
  r1 *= residual_scaling;
  return 0.5 * rho[0];
}

}  // namespace b200
