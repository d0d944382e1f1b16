// TEST INFRASTRUCTURE ONLY (tests/test_oracle_losses.py builds it into a temporary directory and loads it with ctypes).
//
// The robust losses of include/ceres/loss_function.h that the oracle (oracle/bal.h) does not restate -- SoftLOne,
// Cauchy, Arctan, Tolerant, Tukey -- and ScaledLoss around any of them, for the tests of b200_set_loss_functions.
// HuberLoss and the Corrector are the oracle's own (HuberLossEvaluate, Corrector), applied per row in the order
// ResidualBlock::Evaluate applies them (residual_block.cc:170-195: Jacobian first, from the uncorrected residuals).
#include <cmath>
#include <limits>

#include "../oracle/bal.h"

namespace orc {

// The loss objects of include/ceres/loss_function.h, in its order, and ScaledLoss around any of them: type = the
// class, a and b its constructor arguments (only TolerantLoss takes b), scale the ScaledLoss factor (1: not wrapped;
// ScaledLoss(nullptr, s) is {TRIVIAL, -, -, s}).  Each class's Evaluate is restated from its documented rho(s).
enum LossType { LOSS_TRIVIAL = 0, LOSS_HUBER, LOSS_SOFT_L_ONE, LOSS_CAUCHY, LOSS_ARCTAN, LOSS_TOLERANT, LOSS_TUKEY };
struct RobustLoss {
  int type = LOSS_TRIVIAL;
  double a = 1.0, b = 1.0, scale = 1.0;
  double tolerant_c = 0.0;   // TolerantLoss: b log(1 + exp(-a / b)), so that rho(0) = 0; computed once, as its constructor does
  RobustLoss() = default;
  RobustLoss(int type_, double a_, double b_, double scale_) : type(type_), a(a_), b(b_), scale(scale_) {
    if (type == LOSS_TOLERANT) tolerant_c = b * std::log(1.0 + std::exp(-a / b));
  }
  void Evaluate(double s, double rho[3]) const {
    const double kMin = std::numeric_limits<double>::min();   // rho' is kept positive
    switch (type) {
      case LOSS_HUBER:
        HuberLossEvaluate(a, s, rho);
        break;
      case LOSS_SOFT_L_ONE: {   // rho = 2 a^2 (sqrt(1 + s / a^2) - 1)
        const double a2 = a * a, inv_a2 = 1.0 / a2;
        const double q = 1.0 + s * inv_a2;
        const double root = std::sqrt(q);
        rho[0] = 2.0 * a2 * (root - 1.0);
        rho[1] = std::max(kMin, 1.0 / root);
        rho[2] = -(inv_a2 * rho[1]) / (2.0 * q);
        break;
      }
      case LOSS_CAUCHY: {       // rho = a^2 log(1 + s / a^2)
        const double a2 = a * a, inv_a2 = 1.0 / a2;
        const double q = 1.0 + s * inv_a2;
        const double inv_q = 1.0 / q;
        rho[0] = a2 * std::log(q);
        rho[1] = std::max(kMin, inv_q);
        rho[2] = -inv_a2 * (inv_q * inv_q);
        break;
      }
      case LOSS_ARCTAN: {       // rho = a atan(s / a)
        const double inv_a2 = 1.0 / (a * a);
        const double q = 1.0 + s * s * inv_a2;
        const double inv_q = 1.0 / q;
        rho[0] = a * std::atan2(s, a);
        rho[1] = std::max(kMin, inv_q);
        rho[2] = -2.0 * s * inv_a2 * (inv_q * inv_q);
        break;
      }
      case LOSS_TOLERANT: {     // rho = b log(1 + exp((s - a) / b)) - c
        const double x = (s - a) / b;
        if (x > 36.7) {         // ln(2^53): 1 + e^x rounds to e^x, and b log(e^x) = s - a
          rho[0] = s - a - tolerant_c;
          rho[1] = 1.0;
          rho[2] = 0.0;
        } else {
          const double e = std::exp(x);
          rho[0] = b * std::log(1.0 + e) - tolerant_c;
          rho[1] = std::max(kMin, e / (1.0 + e));
          rho[2] = 0.5 / (b * (1.0 + std::cosh(x)));
        }
        break;
      }
      case LOSS_TUKEY: {        // rho = a^2 / 3 (1 - (1 - s / a^2)^3) for s <= a^2, a^2 / 3 beyond
        const double a2 = a * a;
        if (s <= a2) {
          const double t = 1.0 - s / a2;
          const double t2 = t * t;
          rho[0] = a2 / 3.0 * (1.0 - t2 * t);
          rho[1] = t2;
          rho[2] = -2.0 / a2 * t;
        } else {
          rho[0] = a2 / 3.0;
          rho[1] = 0.0;
          rho[2] = 0.0;
        }
        break;
      }
      default:
        rho[0] = s;
        rho[1] = 1.0;
        rho[2] = 0.0;
        break;
    }
    for (int k = 0; k < 3; ++k) rho[k] *= scale;   // ScaledLoss
  }
};

}  // namespace orc

extern "C" {

// rho3 = {rho(s), rho'(s), rho''(s)} of the loss object {type, a, b} wrapped in ScaledLoss(scale)
void loss_rho(int type, double a, double b, double scale, double s, double* rho3) {
  orc::RobustLoss(type, a, b, scale).Evaluate(s, rho3);
}

// The loss of n rows: row i has the object {types[i], params[3i..3i+2] = a, b, scale}, residuals r[2i..2i+1] and, when
// not null, Jacobian cells E [n][2][3] and F [n][2][9] (the oracle's value layout).  Writes row i's cost 0.5 rho(s) to
// cost[i] and corrects r, E and F in place.
void loss_rows(int n, const int* types, const double* params, double* r, double* E, double* F, double* cost) {
  for (int i = 0; i < n; ++i) {
    const orc::RobustLoss loss(types[i], params[3 * i], params[3 * i + 1], params[3 * i + 2]);
    double* ri = r + 2 * static_cast<size_t>(i);
    const double s = ri[0] * ri[0] + ri[1] * ri[1];
    double rho[3];
    loss.Evaluate(s, rho);
    cost[i] = 0.5 * rho[0];
    const orc::Corrector correct(s, rho);
    if (F != nullptr) correct.CorrectJacobian(2, 9, ri, F + 18 * static_cast<size_t>(i));
    if (E != nullptr) correct.CorrectJacobian(2, 3, ri, E + 6 * static_cast<size_t>(i));
    correct.CorrectResiduals(2, ri);
  }
}

}  // extern "C"
