// DOGLEG trust-region strategy (internal/ceres/dogleg_strategy.cc:54-717), host-only scalar part.
//
// The vectors stay where the loop keeps them (HBM, or the host buffers of the host-boundary loop).  What the strategy
// decides is a function of a few scalars of the current Gauss-Newton step: |g|^2, g.gn, |gn|^2 and the Gram matrix of
// J(g/diagonal) and J(gn/diagonal).  This header holds that part: the state kept across iterations, the traditional
// and subspace steps expressed as coefficients on g and gn, and the quartic of the subspace problem.  It includes no
// CUDA header so that it can be compiled and tested on a machine without a GPU.
#pragma once
#include <algorithm>
#include <cmath>
#include <complex>
#include <limits>

namespace b200dl {

constexpr double kMinMu = 1e-8, kMaxMu = 1.0, kMuIncreaseFactor = 10.0;   // dogleg_strategy.cc:50-51, :63
constexpr double kIncreaseThreshold = 0.75, kDecreaseThreshold = 0.25;      // :64-65
constexpr double kCosineThreshold = 0.99;                                    // :344
enum { kTraditional = 0, kSubspace = 1 };                                    // DoglegType, include/ceres/types.h

// How the step is formed from g and gn, element by element: step_i = (cg g_i + cn gn_i) / diagonal_i.  The two pure
// cases select instead of multiplying by 0, as the reference assigns (:209, :221, :281, :311): g is NaN wherever
// diagonal_ is 0 (possible with min_lm_diagonal = 0), and 0 * NaN would leak it into a Gauss-Newton step.
enum StepKind { kGaussNewton = 0, kGradient = 1, kCombination = 2 };
struct Step {
  int kind;
  double cg, cn;
  double norm;         // dogleg_step_norm_ (|step| before the division by diagonal_)
  bool measure_norm;   // the traditional interpolation: norm is |cg g + cn gn|, measured by the pass that forms the step
};

// The scalars of one Gauss-Newton step.  a = g / diagonal_, b = gn / diagonal_.
struct Model {
  double gg = 0, ggn = 0, gngn = 0;    // |g|^2, g.gn, |gn|^2
  double jaja = 0, jajb = 0, jbjb = 0; // |J a|^2, (J a).(J b), |J b|^2
  double alpha = 0;                    // Cauchy point: alpha * -g (:185-194)
  // subspace model (ComputeSubspaceModel, :648-717) in the basis U = [p q] R^-1, where [p q] is [g gn] after column
  // pivoting and R the upper triangle of its QR factorisation
  int rank = 0;
  bool pivot_gn = false;               // p = gn, q = g
  double i11 = 0, i12 = 0, i22 = 0;    // R^-1
  double sg[2] = {0, 0};               // subspace_g_ = U' g
  double B[2][2] = {{0, 0}, {0, 0}};   // subspace_B_ = (J D^-1 U)' (J D^-1 U)
};

inline void cauchy_point(Model* m) { m->alpha = m->gg / m->jaja; }

// Rank and 2-D model from the dot products.  Rank rule: Eigen's ColPivHouseholderQR counts |R_ii| > threshold * max|R_jj|
// with the default threshold epsilon * min(rows, cols) = 2 epsilon.  Column pivoting puts the longer of g and gn first,
// so max|R_jj| = R_11 and the test is R_22 > 2 epsilon R_11 (R_11 = 0: rank 0).  Here R_22 = sqrt(|q|^2 - (p.q)^2/|p|^2)
// is formed from dot products, which resolves it to about sqrt(epsilon) |q| rather than epsilon |q|: g and gn closer than
// that to parallel are classed as rank 1 here and may be rank 2 in the reference.
inline void subspace_model(Model* m) {
  m->pivot_gn = m->gngn > m->gg;   // ties keep g first (Eigen takes the first maximal column)
  const double pp = m->pivot_gn ? m->gngn : m->gg, qq = m->pivot_gn ? m->gg : m->gngn, pq = m->ggn;
  const double r11 = std::sqrt(pp);
  if (!(r11 > 0.0)) {
    m->rank = 0;
    return;
  }
  const double r12 = pq / r11;
  const double r22 = std::sqrt(std::max(0.0, qq - r12 * r12));
  if (!(r22 > 2.0 * std::numeric_limits<double>::epsilon() * r11)) {
    m->rank = 1;
    return;
  }
  m->rank = 2;
  m->i11 = 1.0 / r11;
  m->i12 = -r12 / (r11 * r22);
  m->i22 = 1.0 / r22;
  // U' g = R^-T [p.g, q.g]
  const double pg = m->pivot_gn ? pq : pp, qg = m->pivot_gn ? qq : pq;
  m->sg[0] = pg / r11;
  m->sg[1] = (qg - r12 * m->sg[0]) / r22;
  // B = R^-T G R^-1, G the Gram matrix of J(p/diagonal_), J(q/diagonal_)
  const double Gpp = m->pivot_gn ? m->jbjb : m->jaja, Gqq = m->pivot_gn ? m->jaja : m->jbjb, Gpq = m->jajb;
  const double M00 = Gpp * m->i11, M01 = Gpp * m->i12 + Gpq * m->i22;   // M = G R^-1
  const double M10 = Gpq * m->i11, M11 = Gpq * m->i12 + Gqq * m->i22;
  m->B[0][0] = m->i11 * M00;
  m->B[0][1] = m->i11 * M01;
  m->B[1][0] = m->i12 * M00 + m->i22 * M10;
  m->B[1][1] = m->i12 * M01 + m->i22 * M11;
}

// MakePolynomialForBoundaryConstrainedProblem (:419-438), highest degree first.
inline void boundary_polynomial(const Model& m, double radius, double poly[5]) {
  const double (&B)[2][2] = m.B;
  const double detB = B[0][0] * B[1][1] - B[0][1] * B[1][0];
  const double trB = B[0][0] + B[1][1];
  const double r2 = radius * radius;
  const double adj[2][2] = {{B[1][1], -B[0][1]}, {-B[1][0], B[0][0]}};
  const double ag0 = adj[0][0] * m.sg[0] + adj[0][1] * m.sg[1], ag1 = adj[1][0] * m.sg[0] + adj[1][1] * m.sg[1];
  poly[0] = r2;
  poly[1] = 2.0 * r2 * trB;
  poly[2] = r2 * (trB * trB + 2.0 * detB) - (m.sg[0] * m.sg[0] + m.sg[1] * m.sg[1]);
  poly[3] = -2.0 * ((m.sg[0] * ag0 + m.sg[1] * ag1) - r2 * detB * trB);
  poly[4] = r2 * detB * detB - (ag0 * ag0 + ag1 * ag1);
}

// FindPolynomialRoots (polynomial.cc:190-256): the real parts of all roots, leading zeros removed, closed forms for
// degrees 1 and 2.  From degree 3 the reference takes the eigenvalues of the balanced companion matrix; here the roots
// come from Aberth-Ehrlich simultaneous iteration, which returns the same roots to rounding for the simple roots of the
// boundary quartic.  Returns the number of roots written to `re`, or -1 where the reference's eigen-solver fails
// (non-finite coefficients).
inline int polynomial_roots_real(const double* poly_in, int size, double* re) {
  for (int i = 0; i < size; ++i)
    if (!std::isfinite(poly_in[i])) return -1;
  int lead = 0;
  while (lead < size - 1 && poly_in[lead] == 0.0) ++lead;
  const double* p = poly_in + lead;
  const int degree = size - lead - 1;
  if (degree <= 0) return 0;
  if (degree == 1) {
    re[0] = -p[1] / p[0];
    return 1;
  }
  if (degree == 2) {   // FindQuadraticPolynomialRoots (polynomial.cc:141-180)
    const double a = p[0], b = p[1], c = p[2];
    const double D = b * b - 4 * a * c;
    const double sqrt_D = std::sqrt(std::fabs(D));
    if (D >= 0) {
      if (b >= 0) {
        re[0] = (-b - sqrt_D) / (2.0 * a);
        re[1] = (2.0 * c) / (-b - sqrt_D);
      } else {
        re[0] = (2.0 * c) / (-b + sqrt_D);
        re[1] = (-b + sqrt_D) / (2.0 * a);
      }
    } else {
      re[0] = re[1] = -b / (2.0 * a);
    }
    return 2;
  }
  using cd = std::complex<double>;
  constexpr int kMaxDegree = 8;
  if (degree > kMaxDegree) return -1;
  double a[kMaxDegree + 1];
  double bound = 0.0;
  for (int i = 0; i <= degree; ++i) a[i] = p[i] / p[0];
  for (int i = 1; i <= degree; ++i) bound = std::max(bound, std::fabs(a[i]));
  const double rad = 1.0 + bound;   // Cauchy's bound on the roots' moduli
  cd z[kMaxDegree];
  for (int k = 0; k < degree; ++k) z[k] = std::polar(rad, 6.283185307179586 * k / degree + 0.4);
  for (int iter = 0; iter < 200; ++iter) {
    bool moved = false;
    for (int k = 0; k < degree; ++k) {
      cd f = 1.0, df = 0.0;
      for (int i = 1; i <= degree; ++i) {
        df = df * z[k] + f;
        f = f * z[k] + a[i];
      }
      if (f == 0.0) continue;
      const cd ratio = f / df;
      cd sum = 0.0;
      for (int j = 0; j < degree; ++j)
        if (j != k) sum += 1.0 / (z[k] - z[j]);
      const cd w = ratio / (1.0 - ratio * sum);
      if (!(std::isfinite(w.real()) && std::isfinite(w.imag()))) continue;
      z[k] -= w;
      if (std::abs(w) > 4.0 * std::numeric_limits<double>::epsilon() * std::abs(z[k])) moved = true;
    }
    if (!moved) break;
  }
  for (int k = 0; k < degree; ++k) {
    if (!std::isfinite(z[k].real())) return -1;
    re[k] = z[k].real();
  }
  return degree;
}

// ComputeSubspaceStepFromRoot (:448-452): -(B + y I)^-1 g by LU with partial pivoting, as Eigen's partialPivLu.
inline void step_from_root(const Model& m, double y, double x[2]) {
  double a00 = m.B[0][0] + y, a01 = m.B[0][1], a10 = m.B[1][0], a11 = m.B[1][1] + y, b0 = m.sg[0], b1 = m.sg[1];
  if (std::fabs(a10) > std::fabs(a00)) {
    std::swap(a00, a10);
    std::swap(a01, a11);
    std::swap(b0, b1);
  }
  const double l = a10 / a00;
  const double u11 = a11 - l * a01;
  const double x1 = (b1 - l * b0) / u11;
  const double x0 = (b0 - a01 * x1) / a00;
  x[0] = -x0;
  x[1] = -x1;
}

inline double subspace_model_value(const Model& m, const double x[2]) {   // EvaluateSubspaceModel (:456-458)
  const double bx0 = m.B[0][0] * x[0] + m.B[0][1] * x[1], bx1 = m.B[1][0] * x[0] + m.B[1][1] * x[1];
  return 0.5 * (x[0] * bx0 + x[1] * bx1) + (m.sg[0] * x[0] + m.sg[1] * x[1]);
}

// FindMinimumOnTrustRegionBoundary (:473-515).
inline bool boundary_minimum(const Model& m, double radius, double minimum[2]) {
  minimum[0] = minimum[1] = 0.0;
  double poly[5], roots[4];
  boundary_polynomial(m, radius, poly);
  const int n = polynomial_roots_real(poly, 5, roots);
  if (n < 0) return false;
  double minimum_value = std::numeric_limits<double>::max();
  bool valid_root_found = false;
  for (int i = 0; i < n; ++i) {
    double x[2];
    step_from_root(m, roots[i], x);
    const double xn = std::sqrt(x[0] * x[0] + x[1] * x[1]);
    if (xn > 0) {
      const double s = radius / xn;
      const double xs[2] = {s * x[0], s * x[1]};
      const double f = subspace_model_value(m, xs);
      valid_root_found = true;
      if (f < minimum_value) {
        minimum_value = f;
        minimum[0] = x[0];
        minimum[1] = x[1];
      }
    }
  }
  return valid_root_found;
}

// ComputeTraditionalDoglegStep (:201-255).
inline Step traditional_step(const Model& m, double radius) {
  const double gradient_norm = std::sqrt(m.gg);
  const double gauss_newton_norm = std::sqrt(m.gngn);
  if (gauss_newton_norm <= radius) return {kGaussNewton, 0.0, 1.0, gauss_newton_norm, false};
  if (gradient_norm * m.alpha >= radius) return {kGradient, -(radius / gradient_norm), 0.0, radius, false};
  const double b_dot_a = -m.alpha * m.ggn;
  const double a_squared_norm = std::pow(m.alpha * gradient_norm, 2.0);
  const double b_minus_a_squared_norm = a_squared_norm - 2 * b_dot_a + std::pow(gauss_newton_norm, 2);
  const double c = b_dot_a - a_squared_norm;
  const double d = std::sqrt(c * c + b_minus_a_squared_norm * (std::pow(radius, 2.0) - a_squared_norm));
  const double beta = (c <= 0) ? (d - c) / b_minus_a_squared_norm : (radius * radius - a_squared_norm) / (d + c);
  return {kCombination, -m.alpha * (1.0 - beta), beta, 0.0, true};
}

// Which branch a subspace step took, for tests.
enum SubspaceBranch { kSubGaussNewton = 0, kSubOneDimensional, kSubRootFailure, kSubCosineFallback, kSubBoundary };

// ComputeSubspaceDoglegStep (:266-366).  The step U m is written as coefficients on g and gn: U m = [p q] R^-1 m.
inline Step subspace_step(const Model& m, double radius, int* branch = nullptr) {
  int br = kSubBoundary;
  Step s;
  const double gauss_newton_norm = std::sqrt(m.gngn);
  double mn[2];
  if (gauss_newton_norm <= radius) {
    br = kSubGaussNewton;
    s = {kGaussNewton, 0.0, 1.0, gauss_newton_norm, false};
  } else if (m.rank == 1) {
    br = kSubOneDimensional;
    s = {kGradient, -(radius / std::sqrt(m.gg)), 0.0, radius, false};
  } else if (!boundary_minimum(m, radius, mn)) {
    br = kSubRootFailure;
    s = traditional_step(m, radius);
  } else {
    const double gm0 = m.B[0][0] * mn[0] + m.B[0][1] * mn[1] + m.sg[0];
    const double gm1 = m.B[1][0] * mn[0] + m.B[1][1] * mn[1] + m.sg[1];
    const double cosine_angle = -(mn[0] * gm0 + mn[1] * gm1) /
                                (std::sqrt(mn[0] * mn[0] + mn[1] * mn[1]) * std::sqrt(gm0 * gm0 + gm1 * gm1));
    if (cosine_angle < kCosineThreshold) {
      br = kSubCosineFallback;
      s = traditional_step(m, radius);
    } else {
      const double cp = m.i11 * mn[0] + m.i12 * mn[1], cq = m.i22 * mn[1];
      s = {kCombination, m.pivot_gn ? cq : cp, m.pivot_gn ? cp : cq, radius, false};
    }
  }
  if (branch != nullptr) *branch = br;
  return s;
}

// The strategy's state across iterations (:54-68) and its updates after a step (:618-644).
struct Strategy {
  int type = kTraditional;
  double radius = 0.0;
  double mu = kMinMu;
  double step_norm = 0.0;   // dogleg_step_norm_
  bool reuse = false;

  Step step(const Model& m) const { return type == kSubspace ? subspace_step(m, radius) : traditional_step(m, radius); }
  void accepted(double step_quality) {
    if (step_quality < kDecreaseThreshold) radius *= 0.5;
    if (step_quality > kIncreaseThreshold) radius = std::max(radius, 3.0 * step_norm);
    mu = std::max(kMinMu, 2.0 * mu / kMuIncreaseFactor);
    reuse = false;
  }
  void rejected() {
    radius *= 0.5;
    reuse = true;
  }
  void invalid() {
    mu *= kMuIncreaseFactor;
    reuse = false;
  }
};

}  // namespace b200dl
