// ORACLE — TEST INFRASTRUCTURE ONLY. Never linked into the product library.
// Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
// load this library; it is the checker, never the thing measured as the product.
//
// C entry points (for ctypes) over the CPU restatement in block_sparse.h / schur.h / bal.h.
// Parity status: PINNED — checked in tests/test_oracle_*.py against the reference's own
// known-answer fixtures (internal/ceres/linear_least_squares_problems.cc:73-928), dense
// re-computations in the style of the reference's unit tests, and the two published
// per-iteration solver transcripts on data/problem-16-22106-pre.txt
// (docs/source/installation.rst:187-215, docs/source/solving_faqs.rst:72-100).
#include <cstring>

#include "bal.h"

using namespace orc;

namespace {

// detect_structure.cc: static <2,3,9> when every e-row is 2 rows, e block 3, all f cells 9.
bool Is239(const BlockStructure& bs, int num_elim) {
  bool any = false;
  for (const auto& row : bs.rows) {
    if (row.cells.empty() || row.cells[0].block_id >= num_elim) break;
    any = true;
    if (row.block.size != 2 || bs.cols[row.cells[0].block_id].size != 3) return false;
    for (size_t c = 1; c < row.cells.size(); ++c)
      if (bs.cols[row.cells[c].block_id].size != 9) return false;
  }
  return any;
}

template <typename F239, typename FDyn>
auto Dispatch(const BlockSparseMatrix& A, int num_elim, int force_dynamic, F239&& f239, FDyn&& fdyn) {
  if (!force_dynamic && Is239(A.bs, num_elim)) return f239();
  return fdyn();
}

struct IscHolder {
  std::unique_ptr<ImplicitSchur<2, 3, 9>> s239;
  std::unique_ptr<ImplicitSchur<kDyn, kDyn, kDyn>> sdyn;
};

}  // namespace

extern "C" {

int orc_max_threads() { return static_cast<int>(std::thread::hardware_concurrency()); }

// ------------------------------------------------------------------ generic block sparse matrix
void* orc_bsm_create(int num_col_blocks, const int* col_sizes, int num_row_blocks, const int* row_sizes,
                     const int* row_cell_ptr, const int* cell_block_ids, const double* values) {
  auto* A = new BlockSparseMatrix;
  A->bs.cols.resize(num_col_blocks);
  int pos = 0;
  for (int c = 0; c < num_col_blocks; ++c) {
    A->bs.cols[c].size = col_sizes[c];
    A->bs.cols[c].position = pos;
    pos += col_sizes[c];
  }
  A->bs.rows.resize(num_row_blocks);
  int rpos = 0, vpos = 0;
  for (int r = 0; r < num_row_blocks; ++r) {
    A->bs.rows[r].block.size = row_sizes[r];
    A->bs.rows[r].block.position = rpos;
    rpos += row_sizes[r];
    for (int k = row_cell_ptr[r]; k < row_cell_ptr[r + 1]; ++k) {
      Cell cell;
      cell.block_id = cell_block_ids[k];
      cell.position = vpos;
      vpos += row_sizes[r] * col_sizes[cell.block_id];
      A->bs.rows[r].cells.push_back(cell);
    }
  }
  A->Finalize();
  if (values != nullptr) std::memcpy(A->values.data(), values, sizeof(double) * A->values.size());
  return A;
}
void orc_bsm_free(void* h) { delete static_cast<BlockSparseMatrix*>(h); }
int orc_bsm_num_rows(void* h) { return static_cast<BlockSparseMatrix*>(h)->num_rows; }
int orc_bsm_num_cols(void* h) { return static_cast<BlockSparseMatrix*>(h)->num_cols; }
long orc_bsm_num_nonzeros(void* h) { return static_cast<BlockSparseMatrix*>(h)->num_nonzeros; }
void orc_bsm_get_values(void* h, double* out) {
  auto* A = static_cast<BlockSparseMatrix*>(h);
  std::memcpy(out, A->values.data(), sizeof(double) * A->values.size());
}
void orc_bsm_set_values(void* h, const double* in) {
  auto* A = static_cast<BlockSparseMatrix*>(h);
  std::memcpy(A->values.data(), in, sizeof(double) * A->values.size());
}
void orc_bsm_right_multiply(void* h, const double* x, double* y, int nt) {
  static_cast<BlockSparseMatrix*>(h)->RightMultiplyAndAccumulate(x, y, nt);
}
void orc_bsm_left_multiply(void* h, const double* x, double* y, int nt) {
  static_cast<BlockSparseMatrix*>(h)->LeftMultiplyAndAccumulate(x, y, nt);
}
void orc_bsm_squared_column_norm(void* h, double* x, int nt) {
  static_cast<BlockSparseMatrix*>(h)->SquaredColumnNorm(x, nt);
}
void orc_bsm_scale_columns(void* h, const double* s, int nt) {
  static_cast<BlockSparseMatrix*>(h)->ScaleColumns(s, nt);
}

// ------------------------------------------------------------------ partitioned view
// op: 0 = y += E x, 1 = y += F x, 2 = y += E' x, 3 = y += F' x
void orc_pmv_multiply(void* h, int num_elim, int op, const double* x, double* y, int nt, int force_dynamic) {
  auto& A = *static_cast<BlockSparseMatrix*>(h);
  auto run = [&](auto& v) {
    switch (op) {
      case 0: v.RightMultiplyAndAccumulateE(x, y); break;
      case 1: v.RightMultiplyAndAccumulateF(x, y); break;
      case 2: v.LeftMultiplyAndAccumulateE(x, y); break;
      default: v.LeftMultiplyAndAccumulateF(x, y); break;
    }
    return 0;
  };
  Dispatch(A, num_elim, force_dynamic,
           [&] { PartitionedView<2, 3, 9> v(A, num_elim, nt); return run(v); },
           [&] { PartitionedView<kDyn, kDyn, kDyn> v(A, num_elim, nt); return run(v); });
}
// which: 0 = blockdiag(E'E), 1 = blockdiag(F'F); out = concatenated square cells. Returns #doubles.
int orc_pmv_block_diagonal(void* h, int num_elim, int which, double* out, int nt, int force_dynamic) {
  auto& A = *static_cast<BlockSparseMatrix*>(h);
  auto run = [&](auto& v) {
    int total = 0;
    std::vector<int> layout = which == 0 ? v.DiagonalLayout(0, v.num_col_blocks_e, &total)
                                         : v.DiagonalLayout(v.num_col_blocks_e, v.num_col_blocks_e + v.num_col_blocks_f, &total);
    if (out != nullptr) {
      if (which == 0) v.UpdateBlockDiagonalEtE(layout, out);
      else v.UpdateBlockDiagonalFtF(layout, out);
    }
    return total;
  };
  return Dispatch(A, num_elim, force_dynamic,
                  [&] { PartitionedView<2, 3, 9> v(A, num_elim, nt); return run(v); },
                  [&] { PartitionedView<kDyn, kDyn, kDyn> v(A, num_elim, nt); return run(v); });
}

// ------------------------------------------------------------------ implicit Schur complement
void* orc_isc_create(void* h, int num_elim, int want_ftf, int nt, int force_dynamic) {
  auto& A = *static_cast<BlockSparseMatrix*>(h);
  auto* holder = new IscHolder;
  if (!force_dynamic && Is239(A.bs, num_elim)) holder->s239.reset(new ImplicitSchur<2, 3, 9>(A, num_elim, want_ftf, nt));
  else holder->sdyn.reset(new ImplicitSchur<kDyn, kDyn, kDyn>(A, num_elim, want_ftf, nt));
  return holder;
}
void orc_isc_free(void* s) { delete static_cast<IscHolder*>(s); }
#define ORC_ISC_CALL(s, expr)                      \
  do {                                             \
    auto* hh = static_cast<IscHolder*>(s);         \
    if (hh->s239) { auto& isc = *hh->s239; expr; } \
    else { auto& isc = *hh->sdyn; expr; }          \
  } while (0)
int orc_isc_num_rows(void* s) { int n = 0; ORC_ISC_CALL(s, n = isc.num_rows()); return n; }
void orc_isc_init(void* s, const double* D, const double* b) { ORC_ISC_CALL(s, isc.Init(D, b)); }
void orc_isc_right_multiply(void* s, const double* x, double* y) { ORC_ISC_CALL(s, isc.RightMultiplyAndAccumulate(x, y)); }
void orc_isc_rhs(void* s, double* out) { ORC_ISC_CALL(s, std::memcpy(out, isc.rhs.data(), sizeof(double) * isc.rhs.size())); }
void orc_isc_back_substitute(void* s, const double* x, double* y) { ORC_ISC_CALL(s, isc.BackSubstitute(x, y)); }
// y = power series approximation of S^-1 x (needs want_ftf at creation)
void orc_isc_power_series(void* s, int max_num_spse_iterations, double spse_tolerance, const double* x, double* y) {
  ORC_ISC_CALL(s, PowerSeriesExpansion(&isc, max_num_spse_iterations, spse_tolerance, x, y));
}
int orc_isc_ete_inverse(void* s, double* out) {
  int n = 0;
  ORC_ISC_CALL(s, { n = static_cast<int>(isc.ete_inv.values.size()); if (out) std::memcpy(out, isc.ete_inv.values.data(), sizeof(double) * n); });
  return n;
}

// ------------------------------------------------------------------ Schur eliminator
// diagonal_only = 0: lhs is dense n_f x n_f row-major (upper block triangle filled, as the reference
// does); = 1: lhs is the concatenated diagonal cells (what SCHUR_JACOBI asks for).
// Returns n_f (scalar size of the reduced system). b, D, rhs may be null.
int orc_schur_eliminate(void* h, int num_elim, const double* b, const double* D, int diagonal_only,
                        int assume_full_rank_ete, double* lhs_out, double* rhs, int nt, int force_dynamic) {
  auto& A = *static_cast<BlockSparseMatrix*>(h);
  std::vector<int> sizes;
  for (size_t i = num_elim; i < A.bs.cols.size(); ++i) sizes.push_back(A.bs.cols[i].size);
  RandomAccessLhs lhs(sizes, diagonal_only != 0);
  auto run = [&](auto& e) {
    e.Init(num_elim, assume_full_rank_ete != 0, A.bs);
    e.Eliminate(A, b, D, &lhs, rhs);
    return 0;
  };
  Dispatch(A, num_elim, force_dynamic,
           [&] { SchurEliminator<2, 3, 9> e(nt); return run(e); },
           [&] { SchurEliminator<kDyn, kDyn, kDyn> e(nt); return run(e); });
  if (lhs_out != nullptr) std::memcpy(lhs_out, lhs.values.data(), sizeof(double) * lhs.values.size());
  return lhs.n;
}
void orc_schur_back_substitute(void* h, int num_elim, const double* b, const double* D, const double* z,
                               int assume_full_rank_ete, double* y, int nt, int force_dynamic) {
  auto& A = *static_cast<BlockSparseMatrix*>(h);
  auto run = [&](auto& e) {
    e.Init(num_elim, assume_full_rank_ete != 0, A.bs);
    e.BackSubstitute(A, b, D, z, y);
    return 0;
  };
  Dispatch(A, num_elim, force_dynamic,
           [&] { SchurEliminator<2, 3, 9> e(nt); return run(e); },
           [&] { SchurEliminator<kDyn, kDyn, kDyn> e(nt); return run(e); });
}

// ------------------------------------------------------------------ linear solvers
// solver: 0 = ITERATIVE_SCHUR, 1 = DENSE_SCHUR. out_summary = {num_iterations, termination_type}.
void orc_linear_solve_spse(void* h, int num_elim, int solver, int preconditioner, int min_iter, int max_iter,
                           int residual_reset_period, double q_tolerance, double r_tolerance, const double* b,
                           const double* D, double* x, int* out_summary, int nt, int force_dynamic,
                           int max_num_spse_iterations, int use_spse_initialization, double spse_tolerance);
void orc_linear_solve(void* h, int num_elim, int solver, int preconditioner, int min_iter, int max_iter,
                      int residual_reset_period, double q_tolerance, double r_tolerance, const double* b,
                      const double* D, double* x, int* out_summary, int nt, int force_dynamic) {
  orc_linear_solve_spse(h, num_elim, solver, preconditioner, min_iter, max_iter, residual_reset_period, q_tolerance,
                        r_tolerance, b, D, x, out_summary, nt, force_dynamic, 5, 0, 0.1);
}
void orc_linear_solve_spse(void* h, int num_elim, int solver, int preconditioner, int min_iter, int max_iter,
                           int residual_reset_period, double q_tolerance, double r_tolerance, const double* b,
                           const double* D, double* x, int* out_summary, int nt, int force_dynamic,
                           int max_num_spse_iterations, int use_spse_initialization, double spse_tolerance) {
  auto& A = *static_cast<BlockSparseMatrix*>(h);
  IterativeSchurOptions so;
  so.num_eliminate_blocks = num_elim;
  so.preconditioner_type = preconditioner;
  so.min_num_iterations = min_iter;
  so.max_num_iterations = max_iter;
  so.residual_reset_period = residual_reset_period;
  so.num_threads = nt;
  so.max_num_spse_iterations = max_num_spse_iterations;
  so.use_spse_initialization = use_spse_initialization != 0;
  so.spse_tolerance = spse_tolerance;
  std::unique_ptr<LinearSolverBase> ls;
  const bool s239 = !force_dynamic && Is239(A.bs, num_elim);
  if (solver == ITERATIVE_SCHUR) {
    if (s239) ls.reset(new IterativeSchurSolver<2, 3, 9>(so));
    else ls.reset(new IterativeSchurSolver<kDyn, kDyn, kDyn>(so));
  } else {
    if (s239) ls.reset(new DenseSchurSolver<2, 3, 9>(num_elim, nt));
    else ls.reset(new DenseSchurSolver<kDyn, kDyn, kDyn>(num_elim, nt));
  }
  LinearSummary s = ls->Solve(&A, b, D, q_tolerance, r_tolerance, x);
  out_summary[0] = s.num_iterations;
  out_summary[1] = s.termination_type;
}

// ------------------------------------------------------------------ ConjugateGradientsSolver on a dense symmetric matrix
// (conjugate_gradients_solver_test.cc): identity preconditioner, x is the initial guess and the result.
// out_summary = {num_iterations, termination_type}.
void orc_cg_dense(int n, const double* A_rowmajor, const double* b, double* x, int min_iter, int max_iter,
                  int residual_reset_period, double q_tolerance, double r_tolerance, int* out_summary) {
  CGOptions o;
  o.min_num_iterations = min_iter;
  o.max_num_iterations = max_iter;
  o.residual_reset_period = residual_reset_period;
  o.q_tolerance = q_tolerance;
  o.r_tolerance = r_tolerance;
  std::vector<double> rhs(b, b + n), sol(x, x + n);
  auto lhs = [&](const double* xx, double* yy) {
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < n; ++j) yy[i] += A_rowmajor[i * n + j] * xx[j];
  };
  auto identity = [&](const double* rr, double* zz) {
    for (int i = 0; i < n; ++i) zz[i] += rr[i];
  };
  LinearSummary s = ConjugateGradients(o, lhs, rhs, identity, sol);
  for (int i = 0; i < n; ++i) x[i] = sol[i];
  out_summary[0] = s.num_iterations;
  out_summary[1] = s.termination_type;
}

// ------------------------------------------------------------------ rotation (for the known-answer tests)
void orc_angle_axis_rotate_point(const double* angle_axis, const double* pt, double* result) {
  AngleAxisRotatePoint<double>(angle_axis, pt, result);
}

// ------------------------------------------------------------------ loss / corrector (for the known-answer tests)
void orc_huber_loss(double a, double s, double* rho3) { HuberLossEvaluate(a, s, rho3); }
// residuals [num_rows] and jacobian [num_rows x num_cols] are corrected in place (Jacobian first, like ResidualBlock::Evaluate)
void orc_corrector(double sq_norm, const double* rho3, int num_rows, int num_cols, double* residuals, double* jacobian) {
  const Corrector c(sq_norm, rho3);
  if (jacobian != nullptr) c.CorrectJacobian(num_rows, num_cols, residuals, jacobian);
  c.CorrectResiduals(num_rows, residuals);
}

// ------------------------------------------------------------------ BAL problem
void* orc_bal_read(const char* path) {
  auto* p = new BalProblem;
  if (!p->Read(path)) {
    delete p;
    return nullptr;
  }
  return p;
}
void* orc_bal_from_arrays(int C, int P, int N, const int* cam_idx, const int* pt_idx, const double* obs,
                          const double* cameras, const double* points) {
  auto* p = new BalProblem;
  p->num_cameras = C;
  p->num_points = P;
  p->num_observations = N;
  p->camera_index.assign(cam_idx, cam_idx + N);
  p->point_index.assign(pt_idx, pt_idx + N);
  p->observations.assign(obs, obs + 2 * static_cast<size_t>(N));
  p->parameters.resize(9 * static_cast<size_t>(C) + 3 * static_cast<size_t>(P));
  std::memcpy(p->cameras(), cameras, sizeof(double) * 9 * C);
  std::memcpy(p->points(), points, sizeof(double) * 3 * P);
  return p;
}
void orc_bal_free(void* p) { delete static_cast<BalProblem*>(p); }
void orc_bal_dims(void* p, int* out3) {
  auto* b = static_cast<BalProblem*>(p);
  out3[0] = b->num_cameras;
  out3[1] = b->num_points;
  out3[2] = b->num_observations;
}
void orc_bal_normalize(void* p) { static_cast<BalProblem*>(p)->Normalize(); }
void orc_bal_get(void* p, int* cam_idx, int* pt_idx, double* obs, double* cameras, double* points) {
  auto* b = static_cast<BalProblem*>(p);
  std::memcpy(cam_idx, b->camera_index.data(), sizeof(int) * b->num_observations);
  std::memcpy(pt_idx, b->point_index.data(), sizeof(int) * b->num_observations);
  std::memcpy(obs, b->observations.data(), sizeof(double) * 2 * b->num_observations);
  std::memcpy(cameras, b->cameras(), sizeof(double) * 9 * b->num_cameras);
  std::memcpy(points, b->points(), sizeof(double) * 3 * b->num_points);
}

// ------------------------------------------------------------------ BA program / evaluator / LM
void* orc_ba_create(int C, int P, int N, const int* cam_idx, const int* pt_idx, const double* obs,
                    int use_huber, double huber_a) {
  auto* prog = new BaProgram;
  prog->use_huber = use_huber != 0;
  prog->huber_a = huber_a;
  prog->Build(C, P, N, cam_idx, pt_idx, obs);
  return prog;
}
void orc_ba_free(void* h) { delete static_cast<BaProgram*>(h); }
void orc_ba_dims(void* h, int* out3) {
  auto* p = static_cast<BaProgram*>(h);
  out3[0] = p->C;
  out3[1] = p->P;
  out3[2] = p->N;
}
// Program order: e block -> input point, f block -> input camera, row -> input observation,
// and per-row (e block, f block) ids: exactly what a Ceres adapter reads off the reduced Program.
void orc_ba_order(void* h, int* point_of_eblock, int* camera_of_fblock, int* obs_of_row, int* row_pt,
                  int* row_cam, double* row_obs) {
  auto* p = static_cast<BaProgram*>(h);
  if (point_of_eblock) std::memcpy(point_of_eblock, p->point_of_eblock.data(), sizeof(int) * p->P);
  if (camera_of_fblock) std::memcpy(camera_of_fblock, p->camera_of_fblock.data(), sizeof(int) * p->C);
  if (obs_of_row) std::memcpy(obs_of_row, p->obs_of_row.data(), sizeof(int) * p->N);
  if (row_pt) std::memcpy(row_pt, p->row_pt.data(), sizeof(int) * p->N);
  if (row_cam) std::memcpy(row_cam, p->row_cam.data(), sizeof(int) * p->N);
  if (row_obs) std::memcpy(row_obs, p->row_obs.data(), sizeof(double) * 2 * p->N);
}
void orc_ba_state_from_parameters(void* h, const double* cameras, const double* points, double* state) {
  static_cast<BaProgram*>(h)->StateFromParameters(cameras, points, state);
}
void orc_ba_parameters_from_state(void* h, const double* state, double* cameras, double* points) {
  static_cast<BaProgram*>(h)->ParametersFromState(state, cameras, points);
}
// Returns 1 on success. residuals/gradient may be null. The Jacobian (if wanted) stays inside the
// program; orc_ba_jacobian() exposes it as a generic matrix handle (not owned by the caller).
int orc_ba_evaluate(void* h, const double* state, double* cost, double* residuals, double* gradient,
                    int want_jacobian, int nt) {
  auto* p = static_cast<BaProgram*>(h);
  p->num_threads = nt;
  return p->Evaluate(state, cost, residuals, gradient, want_jacobian != 0) ? 1 : 0;
}
void* orc_ba_jacobian(void* h) { return &static_cast<BaProgram*>(h)->jacobian; }

struct orc_solve_options {
  int linear_solver, preconditioner, max_num_iterations, max_linear_solver_iterations,
      min_linear_solver_iterations, jacobi_scaling, num_threads, use_spse_initialization,
      max_num_consecutive_invalid_steps;
  double eta, initial_trust_region_radius, max_trust_region_radius, min_trust_region_radius,
      min_relative_decrease, min_lm_diagonal, max_lm_diagonal, function_tolerance, gradient_tolerance,
      parameter_tolerance;
};
void orc_solve_options_default(orc_solve_options* o) {
  SolveOptions d;
  o->linear_solver = d.linear_solver;
  o->preconditioner = d.preconditioner;
  o->max_num_iterations = d.max_num_iterations;
  o->max_linear_solver_iterations = d.max_linear_solver_iterations;
  o->min_linear_solver_iterations = d.min_linear_solver_iterations;
  o->jacobi_scaling = d.jacobi_scaling;
  o->num_threads = d.num_threads;
  o->use_spse_initialization = 0;
  o->max_num_consecutive_invalid_steps = d.max_num_consecutive_invalid_steps;
  o->eta = d.eta;
  o->initial_trust_region_radius = d.initial_trust_region_radius;
  o->max_trust_region_radius = d.max_trust_region_radius;
  o->min_trust_region_radius = d.min_trust_region_radius;
  o->min_relative_decrease = d.min_relative_decrease;
  o->min_lm_diagonal = d.min_lm_diagonal;
  o->max_lm_diagonal = d.max_lm_diagonal;
  o->function_tolerance = d.function_tolerance;
  o->gradient_tolerance = d.gradient_tolerance;
  o->parameter_tolerance = d.parameter_tolerance;
}
// trace: max_records rows of 12 doubles:
//  {iteration, cost, cost_change, |g|_inf, |g|_2, |step|, tr_ratio, tr_radius, ls_iterations,
//   step_is_valid, step_is_successful, model_cost_change}
// times (7 doubles, may be null): residual, jacobian, linear solver, total seconds, then call counts.
// Returns number of records written (>=1) or -1 on failure.
int orc_ba_solve(void* h, const orc_solve_options* o, double* state_inout, double* trace, int max_records,
                 double* times_out) {
  auto* p = static_cast<BaProgram*>(h);
  SolveOptions so;
  so.linear_solver = o->linear_solver;
  so.preconditioner = o->preconditioner;
  so.max_num_iterations = o->max_num_iterations;
  so.max_linear_solver_iterations = o->max_linear_solver_iterations;
  so.min_linear_solver_iterations = o->min_linear_solver_iterations;
  so.jacobi_scaling = o->jacobi_scaling;
  so.num_threads = o->num_threads;
  so.use_spse_initialization = o->use_spse_initialization;
  so.max_num_consecutive_invalid_steps = o->max_num_consecutive_invalid_steps;
  so.eta = o->eta;
  so.initial_trust_region_radius = o->initial_trust_region_radius;
  so.max_trust_region_radius = o->max_trust_region_radius;
  so.min_trust_region_radius = o->min_trust_region_radius;
  so.min_relative_decrease = o->min_relative_decrease;
  so.min_lm_diagonal = o->min_lm_diagonal;
  so.max_lm_diagonal = o->max_lm_diagonal;
  so.function_tolerance = o->function_tolerance;
  so.gradient_tolerance = o->gradient_tolerance;
  so.parameter_tolerance = o->parameter_tolerance;
  std::vector<IterationRecord> recs;
  SolveTimes times;
  const int rc = Minimize(p, so, state_inout, &recs, &times);
  if (rc == FAILURE && recs.empty()) return -1;
  const int n = std::min<int>(static_cast<int>(recs.size()), max_records);
  for (int i = 0; i < n; ++i) {
    double* t = trace + 12 * i;
    const IterationRecord& r = recs[i];
    t[0] = r.iteration; t[1] = r.cost; t[2] = r.cost_change; t[3] = r.gradient_max_norm;
    t[4] = r.gradient_norm; t[5] = r.step_norm; t[6] = r.relative_decrease; t[7] = r.trust_region_radius;
    t[8] = r.linear_solver_iterations; t[9] = r.step_is_valid; t[10] = r.step_is_successful;
    t[11] = r.model_cost_change;
  }
  if (times_out != nullptr) {
    times_out[0] = times.residual_eval; times_out[1] = times.jacobian_eval; times_out[2] = times.linear_solver;
    times_out[3] = times.total; times_out[4] = times.num_residual_evals; times_out[5] = times.num_jacobian_evals;
    times_out[6] = times.num_linear_solves;
  }
  return n;
}

}  // extern "C"
