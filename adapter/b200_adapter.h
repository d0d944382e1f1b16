// Ceres-side adapters over libb200ba.so (include/b200ba.h).  Compiled INSIDE a Ceres tree (they include Ceres'
// internal headers, which need Eigen — not available in the development image, so these files are source only here;
// see INTEGRATION.md).  Three classes, all in ceres::internal:
//
//   B200Jacobian             : BlockSparseMatrix   the handle Solver::Solve / TrustRegionMinimizer see as "the
//                                                   Jacobian"; the values live in HBM, the virtuals the minimizer calls
//                                                   (sparse_matrix.h:67-116) forward to the C ABI
//   B200Evaluator            : Evaluator           evaluator.h:60-168
//   B200IterativeSchurSolver : BlockSparseMatrixSolver (TypedLinearSolver<BlockSparseMatrix>, linear_solver.h:366-387)
// (The exact solve on the explicit reduced system, b200_dense_schur_solve, is reachable through the C ABI and the
//  library's own LM loop; it is not routed through a Ceres factory: SPARSE_SCHUR + CUDA_SPARSE is Ceres' own cuDSS path.)
//
// Selected from the unmodified bundle_adjuster CLI with
//   --linear_solver=iterative_schur --sparse_linear_algebra_library=cuda_sparse --preconditioner=schur_jacobi
//   --ordering_type=user      (bundle_adjuster's default automatic ordering may put points into the camera group; the device
//                              path needs the points to be the first elimination group and refuses anything else)
// The Ceres-side hunks (adapter/ceres_b200.patch, generated and verified by tools/make_adapter_patch.py) drop `final` from
// BlockSparseMatrix and from the ten virtuals B200Jacobian overrides (block_sparse_matrix.h:60-95) and add one branch to
// each of the two factories (evaluator.cc:64-70, linear_solver.cc:111-116), both on the SAME predicate (B200Selected).
#ifndef CERES_INTERNAL_B200_ADAPTER_H_
#define CERES_INTERNAL_B200_ADAPTER_H_

#include <cmath>
#include <map>
#include <memory>
#include <string>

#include "b200ba.h"
#include "ceres/block_sparse_matrix.h"
#include "ceres/evaluator.h"
#include "ceres/execution_summary.h"
#include "ceres/linear_solver.h"
#include "ceres/loss_function.h"
#include "ceres/program.h"

namespace ceres::internal {

// The one predicate both factory hunks use, so that the evaluator and the linear solver are always selected together.
inline bool B200Selected(LinearSolverType linear_solver_type, SparseLinearAlgebraLibraryType sparse_library) {
  return linear_solver_type == ITERATIVE_SCHUR && sparse_library == CUDA_SPARSE;
}

// The scale a of a HuberLoss (its members are private).  Beyond s = a^2 the loss is 2 a sqrt(s) - a^2 with
// rho'(s) = a / sqrt(s) (loss_function.cc:52-66): probed at s = 2^200, whose square root is the exact power 2^100, the
// product rho'(s) * 2^100 returns a to the last bit for every a < 2^100 (the difference rho(4s) - 2 rho(s) = a^2 would
// cancel: 6e-6 relative error at a = 3e4).  A loss that is still in its inlier region there (rho' = 1) has no usable
// scale: HUGE_VAL, which B200Evaluator::Create refuses.
inline double B200HuberScale(const LossFunction& loss) {
  const double root = std::ldexp(1.0, 100);
  double rho[3];
  loss.Evaluate(root * root, rho);
  if (rho[1] >= 1.0 || !(rho[1] > 0.0)) return HUGE_VAL;
  return rho[1] * root;
}

// Shared owner of the device problem; evaluator, Jacobian and linear solver all point at it.
struct B200Context {
  b200_handle* handle = nullptr;
  // Host vector the last Evaluate() filled with residuals: when the minimizer hands the same pointer to the linear
  // solver (trust_region_minimizer.cc:399-402) the copy that is still in HBM is used instead of uploading it again.
  const double* last_residuals = nullptr;
  bool apply_loss_function = true;   // what the device evaluator is currently set to (EvaluateOptions, evaluator.h:101)
  ~B200Context() { b200_destroy(handle); }
};

class B200Jacobian final : public BlockSparseMatrix {  // ceres_b200.patch drops `final` from the base and its virtuals
 public:
  B200Jacobian(CompressedRowBlockStructure* bs, std::shared_ptr<B200Context> ctx)
      : BlockSparseMatrix(bs), ctx_(std::move(ctx)) {}
  b200_handle* handle() const { return ctx_->handle; }
  const B200Context& context() const { return *ctx_; }
  // -(J step)'(r + J step / 2) in one pass, r = residuals of the last Evaluate (optional minimizer hunk, ceres_b200.patch)
  bool ModelCostChange(const double* step, double* model_cost_change) const {
    return b200_model_cost_change(ctx_->handle, step, model_cost_change) == B200_OK;
  }

  // The calls TrustRegionMinimizer, LevenbergMarquardtStrategy and DoglegStrategy make on the Jacobian
  // (trust_region_minimizer.cc:269,277,431; levenberg_marquardt_strategy.cc:84;
  // dogleg_strategy.cc:123,179,192,710-712), threaded overloads included.
  void SquaredColumnNorm(double* x) const override;
  void SquaredColumnNorm(double* x, ContextImpl*, int) const override { SquaredColumnNorm(x); }
  void ScaleColumns(const double* scale) override;
  void ScaleColumns(const double* scale, ContextImpl*, int) override { ScaleColumns(scale); }
  void RightMultiplyAndAccumulate(const double* x, double* y) const override;
  void RightMultiplyAndAccumulate(const double* x, double* y, ContextImpl*, int) const override {
    RightMultiplyAndAccumulate(x, y);
  }
  void LeftMultiplyAndAccumulate(const double* x, double* y) const override;
  void LeftMultiplyAndAccumulate(const double* x, double* y, ContextImpl*, int) const override {
    LeftMultiplyAndAccumulate(x, y);
  }
  void SetZero() override {}  // the evaluator overwrites every cell on the device
  void SetZero(ContextImpl*, int) override {}
  // CPU consumers (problem dumps, CLUSTER_* preconditioners) pull the values explicitly:
  void SyncValuesToHost() { b200_jacobian_get_values(handle(), mutable_values()); }

 private:
  std::shared_ptr<B200Context> ctx_;
};

class B200Evaluator final : public Evaluator {
 public:
  // Returns nullptr + *error (as Evaluator::Create does, evaluator.cc:95-97) unless every residual block is
  // AutoDiffCostFunction<SnavelyReprojectionError, 2, 9, 3> on (camera[9], point[3]) with a null or Huber loss.
  static std::unique_ptr<Evaluator> Create(const Evaluator::Options& options, Program* program, std::string* error);

  std::unique_ptr<SparseMatrix> CreateJacobian() const final;
  bool Evaluate(const Evaluator::EvaluateOptions& evaluate_options, const double* state, double* cost,
                double* residuals, double* gradient, SparseMatrix* jacobian) final;
  bool Plus(const double* state, const double* delta, double* state_plus_delta) const final;
  int NumParameters() const final { return program_->NumParameters(); }
  int NumEffectiveParameters() const final { return program_->NumEffectiveParameters(); }
  int NumResiduals() const final { return program_->NumResiduals(); }
  std::map<std::string, CallStatistics> Statistics() const final { return execution_summary_.statistics(); }

 private:
  B200Evaluator(Program* program, std::shared_ptr<B200Context> ctx, int num_eliminate_blocks)
      : program_(program), ctx_(std::move(ctx)), num_eliminate_blocks_(num_eliminate_blocks) {}
  Program* program_;
  std::shared_ptr<B200Context> ctx_;
  int num_eliminate_blocks_;
  ExecutionSummary execution_summary_;
};

class B200IterativeSchurSolver final : public BlockSparseMatrixSolver {
 public:
  explicit B200IterativeSchurSolver(LinearSolver::Options options) : options_(std::move(options)) {}

 private:
  LinearSolver::Summary SolveImpl(BlockSparseMatrix* A, const double* b,
                                  const LinearSolver::PerSolveOptions& per_solve_options, double* x) final;
  LinearSolver::Options options_;
};

}  // namespace ceres::internal
#endif  // CERES_INTERNAL_B200_ADAPTER_H_
