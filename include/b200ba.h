/* b200ba.h — C ABI of libb200ba.so: the H100-native (sm_90a) implementation of Ceres Solver's
 * Levenberg–Marquardt inner-loop hot path for bundle-adjustment-shaped problems
 * (row block 2, eliminated "e" blocks of size 3 = points, "f" blocks of size 9 = cameras).
 *
 * Ceres has no plugin registry or C ABI for evaluators/linear solvers; this header is what two thin
 * adapter classes (adapter/b200_evaluator.h, adapter/b200_iterative_schur_solver.h) bind, one entry
 * point per virtual of the two internal interfaces they subclass.  Each declaration cites the
 * reference interface it replaces (paths relative to the ceres-solver tree).
 *
 * Conventions: plain C types only; every array argument is a caller-owned HOST buffer unless the name
 * ends in _dev; functions return B200_OK (0) or a negative error code and never throw; the message of
 * the last error is available from b200_last_error().  A handle is NOT thread-safe (like the reference
 * objects: internal/ceres/program_evaluator.h:78-79).  All arithmetic is FP64.
 *
 * Vector layout (the reduced program's own order, internal/ceres/reorder_program.cc:262-273 and
 * block_jacobian_writer.cc:211-218):   x = [ e blocks: 3 doubles per point | f blocks: 9 per camera ].
 * Jacobian value layout (block_jacobian_writer.cc:68-167): all E cells [N][2][3] row-major first, then
 * all F cells [N][2][9] — identical to BlockSparseMatrix::values() for this structure.
 */
#ifndef B200BA_H_
#define B200BA_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct b200_handle b200_handle;

enum {
  B200_OK = 0,
  B200_ERR_INVALID_ARGUMENT = -1,
  B200_ERR_CUDA = -2,
  B200_ERR_EVALUATION_FAILED = -3, /* non-finite residual/Jacobian: Evaluator::Evaluate returns false */
  B200_ERR_NO_DEVICE = -4,
  B200_ERR_NCCL = -5,
  B200_ERR_UNSUPPORTED = -6
};

/* LinearSolverTerminationType, internal/ceres/linear_solver.h:58-74 (same numeric order). */
enum { B200_LS_SUCCESS = 0, B200_LS_NO_CONVERGENCE = 1, B200_LS_FAILURE = 2, B200_LS_FATAL_ERROR = 3 };
/* PreconditionerType subset valid for ITERATIVE_SCHUR here (include/ceres/types.h:93-119, same numeric order). */
enum {
  B200_PRECOND_IDENTITY = 0,
  B200_PRECOND_JACOBI = 1,
  B200_PRECOND_SCHUR_JACOBI = 2,
  B200_PRECOND_SCHUR_POWER_SERIES_EXPANSION = 3 /* power_series_expansion_preconditioner.cc:57-82 */
};
/* Robust losses, in the order of include/ceres/loss_function.h.  b200_ba_desc takes TRIVIAL or HUBER; every type goes
 * through b200_set_loss_functions. */
enum {
  B200_LOSS_TRIVIAL = 0,
  B200_LOSS_HUBER = 1,
  B200_LOSS_SOFT_L_ONE = 2,
  B200_LOSS_CAUCHY = 3,
  B200_LOSS_ARCTAN = 4,
  B200_LOSS_TOLERANT = 5,
  B200_LOSS_TUKEY = 6
};
/* One loss object (loss_function.h): type = B200_LOSS_*; a, b = the constructor arguments of that class (HuberLoss(a),
 * SoftLOneLoss(a), CauchyLoss(a), ArctanLoss(a), TolerantLoss(a, b), TukeyLoss(a); only TolerantLoss reads b, TRIVIAL
 * reads neither); scale = ScaledLoss's factor around it, 1 for an unwrapped loss.  ScaledLoss(NULL, s) is
 * {B200_LOSS_TRIVIAL, -, -, s}. */
typedef struct b200_loss {
  int32_t type;
  double a;
  double b;
  double scale;
} b200_loss;
/* LinearSolverType subset (include/ceres/types.h): the implicit iterative solver and the two exact solves of the explicit
 * reduced camera system, by a dense Cholesky (DENSE_SCHUR) and by a block-sparse supernodal Cholesky (SPARSE_SCHUR). */
enum { B200_ITERATIVE_SCHUR = 0, B200_DENSE_SCHUR = 1, B200_SPARSE_SCHUR = 2 };
/* TrustRegionStrategyType and DoglegType, in Ceres' numeric order (include/ceres/types.h) */
enum { B200_LEVENBERG_MARQUARDT = 0, B200_DOGLEG = 1 };
enum { B200_TRADITIONAL_DOGLEG = 0, B200_SUBSPACE_DOGLEG = 1 };

/* Problem structure = what the adapters read off the reduced ceres::internal::Program
 * (residual_block->parameter_blocks()[j]->index(), SnavelyReprojectionError::observed_x/y,
 * residual_block->loss_function()).  Rows must be grouped by e block (pt_idx non-decreasing): the same
 * precondition SchurEliminator has (internal/ceres/schur_eliminator.h:85-99), established by
 * LexicographicallyOrderResidualBlocks (reorder_program.cc:278-359). */
typedef struct b200_ba_desc {
  int32_t num_cameras;       /* C: number of f blocks                                   */
  int32_t num_points;        /* P: number of e blocks (of this shard)                   */
  int64_t num_observations;  /* N: number of row blocks (of this shard)                 */
  const int32_t* cam_idx;    /* [N] f block id of row i  (cells[1].block_id - P)        */
  const int32_t* pt_idx;     /* [N] e block id of row i  (cells[0].block_id), sorted    */
  const double* obs;         /* [2N] observed_x, observed_y of row i                    */
  int32_t loss_type;         /* B200_LOSS_TRIVIAL or B200_LOSS_HUBER (examples/bundle_adjuster.cc:331-332); other
                                losses: b200_set_loss_functions                          */
  double loss_a;             /* HuberLoss(a)                                             */
  int32_t device;            /* CUDA device ordinal                                      */
  void* stream;              /* cudaStream_t to launch on; NULL = a private stream       */
  /* Multi-GPU (SURVEY §8e): points (e blocks) are sharded, cameras replicated.  world_size==1 or
   * nccl_unique_id==NULL means single GPU.  nccl_unique_id = the 128 bytes of ncclUniqueId from
   * b200_nccl_unique_id() on rank 0, distributed by the caller (torch.distributed / MPI / files). */
  int32_t rank, world_size;
  const void* nccl_unique_id;
} b200_ba_desc;

/* The point order the library would keep privately for this structure (b200_create re-orders points -- with all their rows --
 * so that neighbouring points see the same few cameras, and undoes the permutation at every entry point: the layout above is
 * what the caller sees).  Host-only, needs no GPU: perm_out[k] = caller's e block at internal position k ([P], may be NULL);
 * metrics_out = distinct cameras per 1/num_chunks of the rows, summed, for {caller's order, by camera arc, by mean camera,
 * by smallest camera}; *choice_out = which of the four was taken (0 = the caller's order is kept). */
int b200_plan_point_order(const b200_ba_desc* desc, int num_chunks, int32_t* perm_out, int64_t metrics_out[4], int* choice_out);
/* LinearSolverOrderingType (include/ceres/types.h:208, same numeric order): how SPARSE_SCHUR orders the reduced camera
 * system.  B200_AMD: the caller's order or minimum degree, whichever needs fewer flops; B200_NESDIS: nested dissection of the
 * camera graph (solver.h:410).  DENSE_SCHUR and ITERATIVE_SCHUR ignore it. */
enum { B200_AMD = 0, B200_NESDIS = 1 };
/* The symbolic analysis b200_sparse_schur_solve runs at its first call on a handle of this structure.  Host-only, needs no GPU:
 * cam_perm_out[k] = camera eliminated k-th ([C], may be NULL); stats_out (may be NULL), indexed by B200_SPARSE_STAT_*:
 * blocks of the upper triangle of S (diagonal included); blocks of L (diagonal included) in the chosen order, in the caller's
 * order and in the minimum-degree order; factor flops in the caller's and in the minimum-degree order; supernodes; height of
 * the elimination tree (nodes on its longest path); which order was taken (0 the caller's, 1 minimum degree: the one of
 * fewer flops, the caller's on a tie; minimum degree is tried up to 32768 cameras and only with B200_AMD, and reported with
 * the caller's counts where it is not; 2 nested dissection); bytes of factor storage; factor flops in the order taken; and,
 * over the tree of supernodes, the most supernodes and the most flops on one path from a leaf to a root. */
enum {
  B200_SPARSE_STAT_S_BLOCKS = 0,
  B200_SPARSE_STAT_L_BLOCKS,
  B200_SPARSE_STAT_L_BLOCKS_CALLER,
  B200_SPARSE_STAT_L_BLOCKS_MIN_DEGREE,
  B200_SPARSE_STAT_FLOPS_CALLER,
  B200_SPARSE_STAT_FLOPS_MIN_DEGREE,
  B200_SPARSE_STAT_SUPERNODES,
  B200_SPARSE_STAT_TREE_HEIGHT,
  B200_SPARSE_STAT_ORDER,
  B200_SPARSE_STAT_FACTOR_BYTES,
  B200_SPARSE_STAT_FLOPS,
  B200_SPARSE_STAT_CRITICAL_PATH_SUPERNODES,
  B200_SPARSE_STAT_CRITICAL_PATH_FLOPS,
  B200_SPARSE_STATS
};
int b200_plan_sparse_schur(const b200_ba_desc* desc, int32_t* cam_perm_out, int64_t stats_out[B200_SPARSE_STATS]);
/* The same analysis under a given ordering type (B200_AMD: b200_plan_sparse_schur; B200_NESDIS); any other value:
 * B200_ERR_INVALID_ARGUMENT. */
int b200_plan_sparse_schur_ordered(const b200_ba_desc* desc, int ordering_type, int32_t* cam_perm_out,
                                   int64_t stats_out[B200_SPARSE_STATS]);
int b200_nccl_unique_id(void* out128);
int b200_create(const b200_ba_desc* desc, b200_handle** out);
void b200_destroy(b200_handle* h);
const char* b200_last_error(void); /* thread-local message of the last failing call */
int b200_num_parameters(const b200_handle* h);     /* Evaluator::NumParameters   evaluator.h:151 */
int64_t b200_num_residuals(const b200_handle* h);  /* Evaluator::NumResiduals    evaluator.h:158 */

/* ---- Evaluator (internal/ceres/evaluator.h:116-121, ProgramEvaluator::Evaluate program_evaluator.h:137-304)
 * residuals / gradient may be NULL; want_jacobian != 0 refreshes the device-resident Jacobian, and want_jacobian == 0
 * leaves it untouched, also when the gradient is asked for.  gradient = J'r of the unscaled Jacobian.
 * Returns B200_ERR_EVALUATION_FAILED where Evaluate returns false (residual_block.cc:100-131, program_evaluator.h:205-292):
 * a non-finite residual, a non-finite Jacobian entry whenever J is computed (for the Jacobian or the gradient), or a
 * non-finite total cost.  A failed call that asked for residuals leaves no resident residuals (see b200_schur_solve);
 * a failed call that asked for the Jacobian leaves the device-resident Jacobian undefined. */
int b200_evaluate(b200_handle* h, const double* state, double* cost, double* residuals, double* gradient,
                  int want_jacobian);
/* Evaluator::EvaluateOptions::apply_loss_function (evaluator.h:101-102): apply == 0 makes the following evaluations
 * skip the robust correction (rho, Corrector) of the handle's losses, ScaledLoss factors included (residual_block.cc skips
 * the loss object entirely); apply != 0 (the default) restores it. */
int b200_set_apply_loss_function(b200_handle* h, int apply);
/* The loss of every row, as Ceres keeps it: each residual block points at one loss object (problem.h AddResidualBlock).
 * losses[num_losses] is the table of loss objects; row_loss[N] holds the table index of each row of this handle (of this
 * shard), in the caller's row order; row_loss == NULL needs num_losses == 1 and gives every row losses[0].  The table
 * replaces the handle's losses (those of b200_create or of an earlier call) from the next evaluation on; the device-resident
 * Jacobian is left as it is, and the resident residuals are dropped (b == NULL solves and b200_model_cost_change return
 * B200_ERR_INVALID_ARGUMENT until the next successful evaluation with residuals), so that a loss schedule
 * (LossFunctionWrapper::Reset between solves) takes effect at once.  TolerantLoss's constant c = b log(1 + exp(-a / b)) is
 * computed here, as its constructor does.  B200_ERR_INVALID_ARGUMENT, with the handle unchanged: num_losses < 1, a NULL
 * table, row_loss == NULL with more than one loss, an index outside [0, num_losses), a type out of range, a non-finite
 * scale or scale <= 0, a non-finite a or a <= 0 for Huber, SoftLOne, Cauchy, Arctan and Tukey, and for Tolerant a
 * non-finite a or b, a < 0 or b <= 0 (TolerantLoss's CHECKs). */
int b200_set_loss_functions(b200_handle* h, const b200_loss* losses, int num_losses, const int32_t* row_loss);
/* Problem::SetParameterBlockConstant / SetParameterBlockVariable for every block at once.
   camera_constant[C], point_constant[P]: nonzero = constant. Points are this shard's, in the caller's order.
   NULL = none.
 * The call replaces the handle's set; the new set applies from the next evaluation on.  The layout stays [3P | 9C] and
 * b200_num_parameters is unchanged: a constant block is handled as Ceres' reduced program handles it
 * (Program::RemoveFixedBlocks), as Jacobian columns that are exactly zero.
 *  - Evaluation neither checks nor corrects a constant block's cells (a non-finite value there does not fail it) and
 *    stores them as 0, so J'r, the column norms and J'x are 0 on its components.
 *  - The solves (b200_schur_solve, b200_dense_schur_solve, b200_sparse_schur_solve, b200_schur_init) use D' = 1 on the
 *    constant components and the caller's D (0 for D == NULL) elsewhere: (E'E + D'^2)^-1 and the preconditioner blocks are
 *    identities on constant blocks, which are decoupled from the others, and every solution, b200_schur_back_substitute's
 *    included, is 0 there.  The other components are solved as in the reduced program.
 *  - Inputs on constant components are ignored: b200_plus returns x there; b200_lm_solve reads the state and returns its
 *    constant blocks bitwise unchanged, and takes |x| for parameter_tolerance over the variable blocks only
 *    (trust_region_minimizer.cc:725-742).  b200_jtj_multiply adds D^2 x there, as it does for any zero column.
 *  - The stored Jacobian's cells of the now-constant blocks are zeroed by the call, and b200_jacobian_set_values zeroes
 *    them after every upload; cells of blocks made variable keep what they held until the next evaluation with J.  The
 *    explicit S, the Schur initialisation and the preconditioner are invalidated; the resident residuals are kept.
 *  - Sharded handles: each rank passes its own points' flags and the same camera flags.
 *  - The call leaves the handle's SubsetManifolds (b200_set_subset_manifolds) alone.
 * B200_ERR_INVALID_ARGUMENT, with the handle unchanged: h == NULL, or a row whose camera and point are both constant,
 * a full SubsetManifold counting as constant (Ceres moves such a row's cost into fixed_cost; drop the row from the
 * problem, as Program::RemoveFixedBlocks does). */
int b200_set_constant_blocks(b200_handle* h, const uint8_t* camera_constant, const uint8_t* point_constant);
/* Problem::SetManifold(block, new SubsetManifold(n, S)) for every block at once: single coordinates held constant.
   camera_constant_coordinates[C]: bit k (k < 9) set = coordinate k of the camera [angle-axis | t | f, k1, k2] is
   constant, i.e. SubsetManifold(9, {k : bit k}); point_constant_coordinates[P], bits k < 3, likewise for the points of
   this shard, in the caller's order.  0 = no SubsetManifold on that block; NULL = none on any block of that kind.
 * The call replaces the handle's masks from the next evaluation on; the set of constant blocks
 * (b200_set_constant_blocks) stays as it is, and each block's effective state is the union of both, as in Ceres, where
 * SetParameterBlockConstant and SetManifold are independent.  A full mask (tangent size 0) makes its block constant
 * (ParameterBlock::IsConstant) with every consequence described above.  A masked coordinate of a variable block is held
 * as a constant block's components are -- zero Jacobian column, D' = 1 in every solve, exact zeros in every solution, x
 * kept bitwise by b200_plus and b200_lm_solve, the stored J's cells zeroed by the call and after
 * b200_jacobian_set_values -- with three differences, which follow Ceres:
 *  - Evaluation checks the ambient Jacobian before it drops the masked columns (residual_block.cc:85-159): a non-finite
 *    value in a masked column fails the evaluation, where in a constant block's column it does not.
 *  - b200_lm_solve's |x| for parameter_tolerance counts masked coordinates: Ceres' reduced x is the ambient state of the
 *    variable blocks (trust_region_minimizer.cc:725-734).
 *  - b200_covariance_cameras / _points lift the tangent covariance with the plus Jacobian (covariance_impl.cc:240-265):
 *    masked rows and columns of a block are 0, and masked coordinates take no part in the conditioning test.
 * The layout stays [3P | 9C]: S keeps 9 x 9 camera blocks, with identity rows on masked coordinates, so fixing
 * intrinsics does not make the exact solves cheaper.  Sharded handles: each rank passes its own points' masks and the
 * same camera masks.
 * B200_ERR_INVALID_ARGUMENT, with the handle unchanged: h == NULL, a camera mask with bits above 8 or a point mask with
 * bits above 2, or a row whose camera and point are then both constant. */
int b200_set_subset_manifolds(b200_handle* h, const uint16_t* camera_constant_coordinates, const uint8_t* point_constant_coordinates);
/* Evaluator::Plus (evaluator.h:146; Euclidean manifolds only): x_plus_delta = x + delta. */
int b200_plus(b200_handle* h, const double* x, const double* delta, double* x_plus_delta);

/* ---- SparseMatrix virtuals the minimizer calls on the Jacobian (internal/ceres/sparse_matrix.h:67-116) */
int b200_jacobian_squared_column_norm(b200_handle* h, double* x);            /* block_sparse_matrix.cc:351-401 */
int b200_jacobian_scale_columns(b200_handle* h, const double* scale);        /* :403-450 */
int b200_jacobian_right_multiply(b200_handle* h, const double* x, double* y);/* y += J x,  :239-274 */
int b200_jacobian_left_multiply(b200_handle* h, const double* x, double* y); /* y += J' x, :278-349 */
/* The one use the minimizer has for J*step, fused: model_cost_change = -(J step)'(r + J step / 2) with r the residuals
 * of the last b200_evaluate (still in HBM) -- trust_region_minimizer.cc:430-438 (ParallelSetZero +
 * RightMultiplyAndAccumulate + Dot) in one pass over J, returning one scalar instead of the 2N-vector J*step. */
int b200_model_cost_change(b200_handle* h, const double* step, double* model_cost_change);
int b200_jacobian_get_values(b200_handle* h, double* values);                /* BlockSparseMatrix::values(), 24N */
int b200_jacobian_set_values(b200_handle* h, const double* values);          /* mutable_values() */
/* The four single products of PartitionedMatrixView<2,3,9> (internal/ceres/partitioned_matrix_view_impl.h):
 *   B200_PMV_RIGHT_E  y[2N] += E x[3P]   (RightMultiplyAndAccumulateE, :113-137)
 *   B200_PMV_RIGHT_F  y[2N] += F x[9C]   (RightMultiplyAndAccumulateF, :140-191)
 *   B200_PMV_LEFT_E   y[3P] += E' x[2N]  (LeftMultiplyAndAccumulateE,  :194-264)
 *   B200_PMV_LEFT_F   y[9C] += F' x[2N]  (LeftMultiplyAndAccumulateF,  :267-375)
 * On the solver path these only run fused (b200_schur_multiply, b200_jtj_multiply); stand-alone they are the 2x3 / 2x9
 * block-SpMV shapes of the benchmark sweep.  Single GPU. */
enum { B200_PMV_RIGHT_E = 0, B200_PMV_RIGHT_F = 1, B200_PMV_LEFT_E = 2, B200_PMV_LEFT_F = 3 };
int b200_partitioned_multiply(b200_handle* h, int op, const double* x, double* y);
/* y = (J'J + diag(D)^2) x in one pass over J (D may be NULL).  The normal-equations product CGNR uses
 * (cgnr_solver.cc:90-115); here it is the north-star bandwidth kernel. */
int b200_jtj_multiply(b200_handle* h, const double* x, const double* D, double* y);

/* ---- LinearSolver (internal/ceres/linear_solver.h:339-342; IterativeSchurComplementSolver::SolveImpl,
 * iterative_schur_complement_solver.cc:64-157).  Solves min |J x - b|^2 + |D x|^2. */
typedef struct b200_solver_options { /* LinearSolver::Options + PerSolveOptions, linear_solver.h:150-315 */
  int32_t preconditioner_type;       /* B200_PRECOND_* */
  int32_t min_num_iterations;
  int32_t max_num_iterations;
  int32_t residual_reset_period;     /* linear_solver.h:211 (10) */
  double q_tolerance;                /* PerSolveOptions::q_tolerance (eta) */
  double r_tolerance;                /* PerSolveOptions::r_tolerance (-1 from LM) */
  int32_t max_num_spse_iterations;   /* linear_solver.h:172 (5): terms of the power series */
  int32_t use_spse_initialization;   /* :177 (0): start the PCG from the power series applied to the rhs
                                        (iterative_schur_complement_solver.cc:100-111) */
  double spse_tolerance;             /* :183 (0.1): early stop of that initialisation */
} b200_solver_options;
typedef struct b200_solver_summary { /* LinearSolver::Summary, linear_solver.h:320-326 */
  double residual_norm;
  int32_t num_iterations;
  int32_t termination_type;          /* B200_LS_* */
} b200_solver_summary;
void b200_solver_options_default(b200_solver_options* o);
/* b == NULL: b is the residual vector the last b200_evaluate produced, which is still in HBM (the minimizer passes
 * exactly that vector, trust_region_minimizer.cc:399-402 via levenberg_marquardt_strategy.cc:116; the adapter
 * compares the pointer with the one it filled in Evaluate and skips the 16N-byte upload).  Only a successful
 * b200_evaluate with residuals != NULL produces it; after one that asked for residuals and failed there is none, and
 * b == NULL returns B200_ERR_INVALID_ARGUMENT until the next successful one (as does b200_model_cost_change).  Calls
 * without residuals (cost only, Jacobian only) leave it as it was. */
int b200_schur_solve(b200_handle* h, const double* b, const double* D, const b200_solver_options* opts,
                     double* x, b200_solver_summary* summary);

/* DenseSchurComplementSolver::SolveImpl (schur_complement_solver.cc:101-159, :161-214): explicit reduced camera system
 * S (dense 9C x 9C, assembled on the device), Cholesky (cuSOLVER potrf/potrs, loaded lazily), back substitution.
 * Single GPU, 9C up to ~75k.  summary: num_iterations 1, SUCCESS or FAILURE (S not positive definite). b == NULL as above. */
int b200_dense_schur_solve(b200_handle* h, const double* b, const double* D, double* x, b200_solver_summary* summary);

/* SparseSchurComplementSolver::SolveImpl (schur_complement_solver.cc:205-335): the same explicit S, assembled block-sparse on
 * the device, factored by a supernodal Cholesky in a fill-reducing camera order (b200_plan_sparse_schur; analysed once per
 * handle, at the first call), two triangular solves and the back substitution.  Same contract as b200_dense_schur_solve:
 * num_iterations 1, residual_norm 0, FAILURE without writing x when S + D_f^2 is not positive definite (CHOLMOD_NOT_POSDEF,
 * suitesparse.cc:311-313); single GPU, factor storage up to 48 GB (B200_ERR_UNSUPPORTED otherwise); b == NULL as above. */
int b200_sparse_schur_solve(b200_handle* h, const double* b, const double* D, double* x, b200_solver_summary* summary);

/* LinearSolver::Options::use_mixed_precision_solves and max_num_refinement_iterations (linear_solver.h:226-227;
 * Solver::Options, solver.h:572-590) for the following b200_dense_schur_solve / b200_sparse_schur_solve calls on h (both 0
 * when h is created).  Mixed precision: S + D_f^2 is formed in FP64, rounded to float and factored in float; each solve
 * rounds its right-hand side to float and widens its result.  Refinement (with or without mixed precision): x_f =
 * solve(rhs_S), then k times x_f += solve(rhs_S - (S + D_f^2) x_f) with the residual in FP64, 1 + k solves per
 * factorisation as RefinedSparseCholesky / RefinedDenseCholesky do; the points follow by back substitution of the refined
 * x_f.  (Ceres' CUDA dense path with mixed precision refines 2k times; the EIGEN / LAPACK and sparse count is followed.)
 * Summary and failure as above: a non-positive pivot of the (float) factorisation is FAILURE without writing x; failures
 * of the refinement's solves are ignored.  A flag other than 0 / 1 or k < 0: B200_ERR_INVALID_ARGUMENT.  Mixed-precision
 * DENSE_SCHUR needs cusolverDnSpotrf / Spotrs in the loaded cuSOLVER (B200_ERR_UNSUPPORTED otherwise); the dense cap
 * counts the float copy, the sparse one counts the factor in the precision in use. */
int b200_set_exact_solve_options(b200_handle* h, int use_mixed_precision_solves, int max_num_refinement_iterations);

/* Solver::Options::linear_solver_ordering_type (solver.h:410) of the following b200_sparse_schur_solve calls on h (B200_AMD
 * when h is created).  A different type drops h's sparse analysis and factor storage, so the next sparse solve analyses
 * again; the same type is a no-op.  A value other than B200_AMD / B200_NESDIS: B200_ERR_INVALID_ARGUMENT. */
int b200_set_linear_solver_ordering_type(b200_handle* h, int type);

/* Finer-grained pieces of the same solve, for parity tests (each mirrors one reference class):
 *   ImplicitSchurComplement::Init / rhs / RightMultiplyAndAccumulate / BackSubstitute
 *     (implicit_schur_complement.cc:49-97, :251-276, :106-144, :208-243)
 *   SchurJacobiPreconditioner::UpdateImpl (schur_jacobi_preconditioner.cc:87-97) */
int b200_schur_init(b200_handle* h, const double* b, const double* D);
int b200_schur_rhs(b200_handle* h, double* rhs);                                /* [9C] */
int b200_schur_ete_inverse(b200_handle* h, double* out);                        /* [9P]: (E'E + D_e^2)^-1 */
int b200_schur_multiply(b200_handle* h, const double* x, double* y);            /* y = S x, [9C] */
int b200_schur_back_substitute(b200_handle* h, const double* z, double* y);     /* y [3P+9C] */
int b200_schur_jacobi_update(b200_handle* h, double* blocks, double* inverse);  /* each [81C], may be NULL */
int b200_block_jacobi_update(b200_handle* h, double* inverse);                  /* JACOBI: (F'F + D_f^2)^-1 blocks, [81C] */

/* ---- Covariance::Compute / GetCovarianceBlock (include/ceres/covariance.h, internal/ceres/covariance_impl.cc) for the
 * camera blocks and the point blocks, in the Schur form: Cov(cameras) = Z = S^-1, with S the reduced camera system at D = 0
 * (D' = 1 on constant components, as every solve uses), and Cov(p, p) = V_p^-1 + V_p^-1 (sum over rows r, s of p of
 * W_r Z_{c_r c_s} W_s') V_p^-1, V_p = E_p'E_p, W_r = E_r'F_r.  Always FP64, single GPU.
 * b200_covariance_compute evaluates J at `state` (as b200_evaluate with want_jacobian and residuals does: the stored J
 * and the resident residuals are those of `state` afterwards), forms S, factors it and keeps Z and every point block on
 * the device as a snapshot that later evaluations, solves, setters and LM runs do not change; a new compute replaces it.
 * apply_loss_function applies to this call only: the handle's own setting comes back on every exit.  The Schur
 * initialisation, the explicit S and the factor are left as the covariance's, so the next solve rebuilds them; the sparse
 * analysis is reused (the handle's linear_solver_ordering_type), and use_mixed_precision_solves and the refinement count
 * do not apply.
 *   B200_SPARSE_SCHUR: the supernodal factor and its selected inverse, Z on the pattern of L; serves every pair (i, i) and
 *                      every pair of cameras that share a point.
 *   B200_DENSE_SCHUR:  cuSOLVER potrf + potri on the dense S (cusolverDnDpotri needed); serves any pair.
 * *valid, as Covariance::Compute's bool: 0 when S or a variable point's E'E is not positive definite, or when the
 * smallest ratio d_k / A_kk over the variable components (d_k the k-th squared pivot, A_kk the diagonal of the matrix
 * factored), over S's factor and every point's 3x3 Cholesky, is below min_reciprocal_condition_number.  The return code
 * stays B200_OK then.  B200_ERR_UNSUPPORTED: B200_ITERATIVE_SCHUR, a sharded handle, or storage over the caps of the
 * solves (the sparse one counts the factor and Z).  B200_ERR_EVALUATION_FAILED: the evaluation at `state` failed. */
typedef struct b200_covariance_options { /* Covariance::Options, include/ceres/covariance.h:240-340 */
  int32_t algorithm;                       /* B200_SPARSE_SCHUR (default) or B200_DENSE_SCHUR */
  double min_reciprocal_condition_number;  /* 1e-14, covariance.h:294 */
  int32_t apply_loss_function;             /* 1, covariance.h:339 */
} b200_covariance_options;
void b200_covariance_options_default(b200_covariance_options* o);
int b200_covariance_compute(b200_handle* h, const double* state, const b200_covariance_options* o, int* valid);
/* The getters refuse with B200_ERR_INVALID_ARGUMENT before any compute and after one that set valid = 0
 * (covariance_impl.cc:137-141).  Output is row-major 9 x 9 / 3 x 3 blocks in the caller's camera and point order, as
 * GetCovarianceBlock writes them.  pairs[2 num_pairs]: Cov(c_i, c_j) of pair (i, j) in out[81 q..]; (j, i) returns its
 * transpose.  A pair with a constant camera and a constant point return exact zeros (covariance_impl.cc:143-165).  A pair
 * out of range, or (sparse) a pair of distinct cameras that share no point, is refused with nothing written. */
int b200_covariance_cameras(b200_handle* h, int num_pairs, const int32_t* pairs, double* out);
int b200_covariance_points(b200_handle* h, double* out); /* [9P] */
/* The selected inversion's task graph of the analysis b200_plan_sparse_schur_ordered describes, host-only:
 * *num_supernodes = ns; sn_first_out [ns + 1] (first position of each supernode), order_out [ns] (the factor's ticket
 * order; the selected inversion takes it in reverse) and counter_out [ns] (the initial counter of each supernode's
 * selected-inversion task: the number of supernodes owning one of its rows below, 0 for a root).  Buffers of C + 1 / C
 * entries always suffice; any may be NULL. */
int b200_plan_sparse_selinv(const b200_ba_desc* desc, int ordering_type, int32_t* num_supernodes, int32_t* sn_first_out,
                            int32_t* order_out, int32_t* counter_out);

/* ---- Device-resident trust-region loop (SURVEY §8f.3: TrustRegionMinimizer::Minimize with
 * LevenbergMarquardtStrategy, trust_region_minimizer.cc:68-137 / levenberg_marquardt_strategy.cc:69-171, or with
 * DoglegStrategy, dogleg_strategy.cc:54-717).
 * State, residuals, Jacobian, D and the step never leave HBM; only scalars cross the bus.
 * DOGLEG needs an exact solve (solver.cc:431-438): B200_DENSE_SCHUR or B200_SPARSE_SCHUR; with B200_ITERATIVE_SCHUR, or
 * an out-of-range strategy or dogleg type, b200_lm_solve returns B200_ERR_INVALID_ARGUMENT.  A rejected dogleg step
 * keeps its Gauss-Newton step and gradient and costs no solve; its record has linear_solver_iterations 0.
 * use_mixed_precision_solves / max_num_refinement_iterations apply to the call's exact solves, the Gauss-Newton solves of
 * DOGLEG included, as b200_set_exact_solve_options would; the handle's own values are restored when the call returns, also
 * on an error.  Mixed precision with B200_ITERATIVE_SCHUR is B200_ERR_INVALID_ARGUMENT (solver.cc:298-300); k is ignored
 * there.  linear_solver_ordering_type applies to the call's sparse solves in the same way, as
 * b200_set_linear_solver_ordering_type would, and the handle's own type is restored on every exit: a call whose type
 * differs from the handle's analyses once for itself, and the handle's next sparse solve analyses again. */
typedef struct b200_lm_options { /* Solver::Options subset, include/ceres/solver.h:232-632 */
  int32_t max_num_iterations;              /* bundle_adjuster.cc:121 (5) */
  int32_t jacobi_scaling;                  /* 1 */
  int32_t max_num_consecutive_invalid_steps; /* 5 */
  int32_t linear_solver_type;        /* B200_ITERATIVE_SCHUR (default), B200_DENSE_SCHUR or B200_SPARSE_SCHUR */
  double eta;                              /* 1e-2 */
  double initial_trust_region_radius;      /* 1e4 */
  double max_trust_region_radius;          /* 1e16 */
  double min_trust_region_radius;          /* 1e-32 */
  double min_relative_decrease;            /* 1e-3 */
  double min_lm_diagonal, max_lm_diagonal; /* 1e-6, 1e32 */
  double function_tolerance, gradient_tolerance, parameter_tolerance; /* 1e-16 each in bundle_adjuster */
  b200_solver_options linear_solver;
  int32_t trust_region_strategy_type;      /* B200_LEVENBERG_MARQUARDT (default) or B200_DOGLEG */
  int32_t dogleg_type;                     /* B200_TRADITIONAL_DOGLEG (default) or B200_SUBSPACE_DOGLEG */
  int32_t use_mixed_precision_solves;      /* solver.h:572-580 (0) */
  int32_t max_num_refinement_iterations;   /* :582-590 (0) */
  int32_t linear_solver_ordering_type;     /* solver.h:410: B200_AMD (default) or B200_NESDIS */
} b200_lm_options;
typedef struct b200_lm_iteration { /* IterationSummary, include/ceres/iteration_callback.h */
  int32_t iteration, linear_solver_iterations, step_is_valid, step_is_successful;
  double cost, cost_change, gradient_max_norm, gradient_norm, step_norm, relative_decrease,
      trust_region_radius, model_cost_change;
} b200_lm_iteration;
void b200_lm_options_default(b200_lm_options* o);
/* state_inout: host [3P+9C] (read at entry, best state written back at exit).  trace: up to max_records
 * IterationSummary rows; returns the number written through *num_records.  If host_boundary != 0 the loop
 * is driven through the HOST-buffer entry points above exactly as the Ceres adapters would
 * (state/D/step/residual copies every iteration); otherwise everything stays device-resident. */
int b200_lm_solve(b200_handle* h, const b200_lm_options* opts, double* state_inout, b200_lm_iteration* trace,
                  int max_records, int* num_records, int host_boundary);

/* ---- Instrumentation */
typedef struct b200_kernel_stat {
  char name[32];
  int64_t launches;       /* kernel launches */
  int64_t operations;     /* logical operations (one S*x, one evaluate ...): an operation may take several launches
                             (main kernel + the few >32-row points + ...), all billed to it */
  double device_ms;       /* sum of CUDA-event times of all launches; only filled while profiling is enabled */
  double bytes_per_operation; /* algorithmic bytes moved by ONE OPERATION (SURVEY §8d), 0 if not HBM-bound work:
                                 achieved GB/s = bytes_per_operation * operations / device_ms */
} b200_kernel_stat;
int b200_profile_enable(b200_handle* h, int on);   /* per-kernel cudaEvent timing on/off (off by default) */
int b200_stats_reset(b200_handle* h);
int b200_stats_get(b200_handle* h, b200_kernel_stat* out, int max_entries, int* num_entries);
int64_t b200_total_launches(const b200_handle* h); /* kernels launched since create / last reset */
int b200_synchronize(b200_handle* h);
/* h2d / d2h bytes moved by the host-buffer entry points since the last reset */
int b200_transfer_bytes(const b200_handle* h, int64_t* h2d, int64_t* d2h);

#ifdef __cplusplus
}
#endif
#endif /* B200BA_H_ */
