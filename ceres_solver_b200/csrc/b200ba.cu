// libb200ba.so — host side of the C ABI declared in include/b200ba.h.
//
// Owns the device-resident bundle adjustment problem (SURVEY Appendix B layout), launches the sm_90a
// kernels of kernels.cuh / vector_kernels.cuh on one stream, and implements
//   * the Evaluator-shaped entry points   (internal/ceres/evaluator.h:60-168),
//   * the SparseMatrix-shaped entry points on the device Jacobian (internal/ceres/sparse_matrix.h:67-116),
//   * the LinearSolver-shaped ITERATIVE_SCHUR solve (iterative_schur_complement_solver.cc:64-157) with the PCG
//     of conjugate_gradients_solver.h:109-306 running without host synchronisation inside the iteration,
//   * a trust-region loop (trust_region_minimizer.cc / levenberg_marquardt_strategy.cc) either through the
//     host-buffer boundary (what the Ceres adapters do) or fully device-resident.
// There is no CPU fallback: every entry point fails with B200_ERR_NO_DEVICE / B200_ERR_CUDA if the GPU path
// is unavailable.
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <numeric>
#include <string>
#include <vector>

#ifdef B200_WITH_NCCL
#include <dlfcn.h>
#include <nccl.h>  // types only: the library is resolved with dlopen at run time (see NcclApi)
#endif

#include "../../include/b200ba.h"
#include "kernels.cuh"
#include "kernels_v2.cuh"
#include "kernels_v2b.cuh"
#include "kernels_v4b.cuh"
#include "pmv_kernels.cuh"
#include "vector_kernels.cuh"
#include "cg_kernel.cuh"
#include "spse_kernels.cuh"
#include "huge_kernels.cuh"
#include "dense_schur.cuh"
#include "explicit_schur.cuh"
#include "plan.cuh"
#include "sparse_plan.cuh"
#include "sparse_schur.cuh"
#include "covariance.cuh"
#include "dogleg.h"

using namespace b200;

namespace {

thread_local std::string g_error;
constexpr int kHostThreads = 8;   // host-side vector passes of the host-boundary LM loop (the reference uses its thread pool)

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_error = buf;
  return code;
}

#define CU(expr)                                                                                   \
  do {                                                                                             \
    cudaError_t e_ = (expr);                                                                       \
    if (e_ != cudaSuccess) return fail(B200_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), \
                                       __FILE__, __LINE__);                                        \
  } while (0)
#define OK(expr)               \
  do {                         \
    int rc_ = (expr);          \
    if (rc_ != B200_OK) return rc_; \
  } while (0)

// cuSOLVER (dense Cholesky of the explicit reduced camera system, SURVEY 8f.1) is bound lazily with dlopen like NCCL: the
// library is only touched by b200_dense_schur_solve, and shares whatever libcusolver.so.11 the process already has.
struct CusolverApi {
  typedef int (*create_t)(void**);
  typedef int (*destroy_t)(void*);
  typedef int (*set_stream_t)(void*, cudaStream_t);
  typedef int (*potrf_bs_t)(void*, int, int, double*, int, int*);
  typedef int (*potrf_t)(void*, int, int, double*, int, double*, int, int*);
  typedef int (*potrs_t)(void*, int, int, int, const double*, int, double*, int, int*);
  typedef int (*spotrf_bs_t)(void*, int, int, float*, int, int*);
  typedef int (*spotrf_t)(void*, int, int, float*, int, float*, int, int*);
  typedef int (*spotrs_t)(void*, int, int, int, const float*, int, float*, int, int*);
  typedef int (*potri_bs_t)(void*, int, int, double*, int, int*);
  typedef int (*potri_t)(void*, int, int, double*, int, double*, int, int*);
  create_t Create = nullptr;
  destroy_t Destroy = nullptr;
  set_stream_t SetStream = nullptr;
  potrf_bs_t DpotrfBufferSize = nullptr;
  potrf_t Dpotrf = nullptr;
  potrs_t Dpotrs = nullptr;
  // the single-precision factorisation of use_mixed_precision_solves, bound on its own: a library without these symbols
  // fails only the mixed-precision dense solve
  spotrf_bs_t SpotrfBufferSize = nullptr;
  spotrf_t Spotrf = nullptr;
  spotrs_t Spotrs = nullptr;
  // the inverse from the factor (b200_covariance_compute with B200_DENSE_SCHUR), bound on its own as well
  potri_bs_t DpotriBufferSize = nullptr;
  potri_t Dpotri = nullptr;
  bool ok = false, float_ok = false, potri_ok = false;
};
CusolverApi g_cusolver;
bool load_cusolver() {
  if (g_cusolver.ok) return true;
  const char* name = getenv("B200_CUSOLVER_LIB");
  void* lib = dlopen(name != nullptr ? name : "libcusolver.so.11", RTLD_NOW | RTLD_GLOBAL);
  if (lib == nullptr) lib = dlopen("libcusolver.so", RTLD_NOW | RTLD_GLOBAL);
  if (lib == nullptr) return false;
  g_cusolver.Create = reinterpret_cast<CusolverApi::create_t>(dlsym(lib, "cusolverDnCreate"));
  g_cusolver.Destroy = reinterpret_cast<CusolverApi::destroy_t>(dlsym(lib, "cusolverDnDestroy"));
  g_cusolver.SetStream = reinterpret_cast<CusolverApi::set_stream_t>(dlsym(lib, "cusolverDnSetStream"));
  g_cusolver.DpotrfBufferSize = reinterpret_cast<CusolverApi::potrf_bs_t>(dlsym(lib, "cusolverDnDpotrf_bufferSize"));
  g_cusolver.Dpotrf = reinterpret_cast<CusolverApi::potrf_t>(dlsym(lib, "cusolverDnDpotrf"));
  g_cusolver.Dpotrs = reinterpret_cast<CusolverApi::potrs_t>(dlsym(lib, "cusolverDnDpotrs"));
  g_cusolver.ok = g_cusolver.Create && g_cusolver.Destroy && g_cusolver.SetStream && g_cusolver.DpotrfBufferSize &&
                  g_cusolver.Dpotrf && g_cusolver.Dpotrs;
  g_cusolver.SpotrfBufferSize = reinterpret_cast<CusolverApi::spotrf_bs_t>(dlsym(lib, "cusolverDnSpotrf_bufferSize"));
  g_cusolver.Spotrf = reinterpret_cast<CusolverApi::spotrf_t>(dlsym(lib, "cusolverDnSpotrf"));
  g_cusolver.Spotrs = reinterpret_cast<CusolverApi::spotrs_t>(dlsym(lib, "cusolverDnSpotrs"));
  g_cusolver.float_ok = g_cusolver.SpotrfBufferSize && g_cusolver.Spotrf && g_cusolver.Spotrs;
  g_cusolver.DpotriBufferSize = reinterpret_cast<CusolverApi::potri_bs_t>(dlsym(lib, "cusolverDnDpotri_bufferSize"));
  g_cusolver.Dpotri = reinterpret_cast<CusolverApi::potri_t>(dlsym(lib, "cusolverDnDpotri"));
  g_cusolver.potri_ok = g_cusolver.DpotriBufferSize && g_cusolver.Dpotri;
  return g_cusolver.ok;
}

#ifdef B200_WITH_NCCL
// NCCL is bound lazily with dlopen/dlsym, and only when world_size > 1: the library then shares whatever
// libnccl.so.2 the process already has (e.g. the one PyTorch bundles) instead of pinning its own copy, and a
// single-GPU process never needs NCCL at all.  B200_NCCL_LIB overrides the name.
struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  bool ok = false;
};
NcclApi g_nccl;
bool load_nccl() {
  if (g_nccl.ok) return true;
  const char* name = getenv("B200_NCCL_LIB");
  void* lib = dlopen(name != nullptr ? name : "libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (lib == nullptr) return false;
  g_nccl.GetUniqueId = reinterpret_cast<decltype(g_nccl.GetUniqueId)>(dlsym(lib, "ncclGetUniqueId"));
  g_nccl.CommInitRank = reinterpret_cast<decltype(g_nccl.CommInitRank)>(dlsym(lib, "ncclCommInitRank"));
  g_nccl.AllReduce = reinterpret_cast<decltype(g_nccl.AllReduce)>(dlsym(lib, "ncclAllReduce"));
  g_nccl.AllGather = reinterpret_cast<decltype(g_nccl.AllGather)>(dlsym(lib, "ncclAllGather"));
  g_nccl.CommDestroy = reinterpret_cast<decltype(g_nccl.CommDestroy)>(dlsym(lib, "ncclCommDestroy"));
  g_nccl.GetErrorString = reinterpret_cast<decltype(g_nccl.GetErrorString)>(dlsym(lib, "ncclGetErrorString"));
  g_nccl.ok = g_nccl.GetUniqueId && g_nccl.CommInitRank && g_nccl.AllReduce && g_nccl.AllGather && g_nccl.CommDestroy && g_nccl.GetErrorString;
  return g_nccl.ok;
}
#endif

// Host vector in page-locked memory (the host-buffer LM loop mirrors what an adapter with pinned buffers does).
struct PinnedVec {
  double* p = nullptr;
  size_t n = 0;
  PinnedVec() = default;
  PinnedVec(const PinnedVec&) = delete;
  ~PinnedVec() { if (p != nullptr) cudaFreeHost(p); }
  void resize(size_t m) {
    if (m == n) return;
    if (p != nullptr) cudaFreeHost(p);
    p = nullptr;
    n = m;
    if (m > 0 && cudaMallocHost(reinterpret_cast<void**>(&p), m * sizeof(double)) != cudaSuccess) { p = nullptr; n = 0; }
  }
  void assign(size_t m, double v) { resize(m); for (size_t i = 0; i < n; ++i) p[i] = v; }
  void assign(const double* b, const double* e) { resize(static_cast<size_t>(e - b)); std::memcpy(p, b, n * sizeof(double)); }
  PinnedVec& operator=(const PinnedVec& o) { resize(o.n); if (n) std::memcpy(p, o.p, n * sizeof(double)); return *this; }
  double* data() { return p; }
  double* begin() { return p; }
  double* end() { return p + n; }
};

// The host-boundary loop's vectors, kept by the handle across solves (cudaMallocHost is far too slow to sit inside a solve).
struct HostMirrors {
  PinnedVec x, cand, residuals, gradient, step, scaling, diagonal, lmD, sol, best;
  PinnedVec g, gn, ja, jb;   // DOGLEG: g, gn, J(g/diagonal), J(gn/diagonal)
};

struct EventPair {
  cudaEvent_t a, b;
  int kernel;
};

}  // namespace

struct b200_handle {
  int device = 0;
  cudaStream_t stream = nullptr;
  cudaStream_t stream2 = nullptr;   // side stream for the big-point kernel inside the PCG
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  bool own_stream = false;
  int sm_count = 132;
  int C = 0, P = 0, N = 0, num_tiles = 0;
  int np = 0;  // 3P + 9C
  // the loss of every row (b200_create's descriptor or b200_set_loss_functions): its class picks the evaluate instantiation
  // (loss.cuh); a table of more than one loss object is read per row from d_loss_table through d_row_loss
  int loss_cls = kLossTrivial;
  LossEntry loss_one{};
  int* d_row_loss = nullptr;             // [N], internal row order; allocated by the first table
  LossEntry* d_loss_table = nullptr;
  size_t loss_table_cap = 0;
  bool loss_rows = false;                // the evaluations read d_row_loss and d_loss_table
  bool apply_loss = true;   // EvaluateOptions::apply_loss_function
  // b200_set_constant_blocks and b200_set_subset_manifolds, as passed (caller's order; empty = none of that kind) ...
  std::vector<uint8_t> set_cam_const, set_pt_const, set_pt_mask;
  std::vector<uint16_t> set_cam_mask;
  // ... and their effective state (FixedState): the component states (vector_kernels.cuh kComponentMasked,
  // kComponentConstant), in the internal order on the device and in the caller's on the host, and the packed block
  // states the evaluate kernels read (kBlockConstant); fixed_any picks the evaluate instantiation that zeroes their cells
  bool fixed_any = false;
  uint8_t* d_fixed = nullptr;            // [3P+9C]; allocated by the first non-empty state
  std::vector<uint8_t> h_fixed;          // [3P+9C]
  uint16_t* d_block_state = nullptr;     // [P + C] points, then cameras
  double* d_solve_D = nullptr;           // [3P+9C] D' of the solves (solve_diagonal_kernel)
  int rank = 0, world = 1;
#ifdef B200_WITH_NCCL
  ncclComm_t comm = nullptr;
#endif
  DevKnobs knobs;
  std::vector<void*> allocs;   // every device allocation of the handle (dev_alloc), freed by b200_destroy
  ProblemView view{};
  double* d_values = nullptr;
  // evaluator state
  double *d_state = nullptr, *d_residuals = nullptr, *d_gradient = nullptr, *d_tile_partial = nullptr;
  int* d_fail = nullptr;
  double* d_scalars = nullptr;  // small device scalar block
  double* d_partial = nullptr;  // two-stage reduction partials
  // generic parameter-sized / residual-sized scratch
  double *d_vp0 = nullptr, *d_vp1 = nullptr, *d_vr0 = nullptr;
  // linear solver state
  double *d_b = nullptr, *d_D = nullptr, *d_ete_inv = nullptr, *d_rhs = nullptr, *d_ye = nullptr;
  double *d_upper45 = nullptr, *d_minv = nullptr, *d_blocks = nullptr;
  double *d_xr = nullptr, *d_p = nullptr, *d_r = nullptr, *d_z = nullptr, *d_tmp = nullptr, *d_sol = nullptr;
  CgState* d_cg = nullptr;
  // internal point order (b200_create): identity unless `permuted`
  bool permuted = false;
  int *d_pt_perm = nullptr, *d_row_perm = nullptr;   // internal block -> caller block
  std::vector<int> h_row_perm;                        // ... of the rows, for b200_set_loss_functions
  double *d_stage_p = nullptr, *d_stage_r = nullptr; // boundary staging: [3P+9C], [2N]
  std::vector<int> h_pt_perm;
  bool schur_ready = false;
  bool q_from_init = false;   // d_q3 holds the per-row blocks of the CURRENT implicit-Schur initialisation
  const double* cur_b = nullptr;  // device pointers of the current ISC Init
  const double* cur_D = nullptr;
  // LM state
  double *d_scale = nullptr, *d_sqnorm = nullptr, *d_diagonal = nullptr, *d_lmD = nullptr, *d_step = nullptr,
         *d_cand = nullptr, *d_y = nullptr;
  // DOGLEG (allocated by the first device-resident dogleg step): g, gn and the per-tile partials of dogleg_gram_kernel
  double *d_dl_g = nullptr, *d_dl_gn = nullptr, *d_dl_part = nullptr;
  // pinned host staging for scalars
  double* h_scalars = nullptr;
  CgState* h_cg = nullptr;      // two pinned slots: the host polls one batch behind the launches
  cudaEvent_t ev_cg[2] = {nullptr, nullptr};
  int* h_fail = nullptr;
  // kernel choices of the plan (plan.cuh)
  MulFamily mul = MulFamily::Tile;
  DiagPass diag = DiagPass::Tile;
  bool big_folded = false;   // S*x handles the >32-row points inside the warp-tile kernel (no extra launch)
  // warp-tile kernels (family V3 / V4): views and dynamic shared memory of jtj_v2, S*x (and the v4 kernels), the
  // evaluation and the block-diagonal pass
  V2View v2{}, v2_mul{}, v2_eval{}, v2_diag{};
  size_t v2_smem = 0, mul_smem = 0, eval_v2_smem = 0, diag_v2_smem = 0;
  int diag_v2_replicas = 0;
  ProblemView view_big{};   // CTA tiles holding only the points with more than 32 rows
  ProblemView view_chunks{};  // ... only the <= kTile-row slices of the points with more than kTile rows
  int num_big_tiles = 0;
  const int2* d_cta_big = nullptr;
  double* d_dense_s = nullptr;   // explicit reduced camera system [9C][9C] (allocated by the first dense solve)
  double* d_dense_work = nullptr;
  int dense_lwork = 0;
  int* d_dense_info = nullptr;
  float* d_dense_s32 = nullptr;  // ... its lower triangle rounded to float, then the float factor (mixed-precision solves)
  float* d_dense_work32 = nullptr;
  float* d_dense_v32 = nullptr;  // [9C] the float solve's vector
  int dense_lwork32 = 0;
  void* cusolver = nullptr;
  int num_huge = 0;           // points with more than kTile rows (huge_kernels.cuh); their rows appear as chunk tiles
  int* d_huge_pts = nullptr;
  bool residuals_resident = false;  // d_residuals holds the residuals of the last b200_evaluate(..., residuals != NULL)
  double *d_ftf_inv = nullptr, *d_spse[3] = {nullptr, nullptr, nullptr};  // general-preconditioner PCG (SPSE)
  double *d_pq_parts = nullptr, *d_seed_pq = nullptr;  // fused p.q: per-CTA partials of the product / of the vector kernel
  // camera-major block diagonal (DiagPass::CamMajor)
  int num_cam_items = 0;
  CamItem* d_cam_items = nullptr;
  int* d_cam_rows = nullptr;
  double* d_q3 = nullptr;
  // explicit S (explicit_schur.cuh), single GPU, chosen by the plan from the camera graph
  bool xs = false;
  bool xs_ready = false;        // S holds the assembly for the current implicit-Schur initialisation
  bool xs_diag_ready = false;   // ... and d_upper45 still holds its diagonal blocks
  int xs_grid = 0;
  XsView xsv{};
  int num_xs_long = 0, num_xs_short = 0;   // blocks assembled by a CTA / by a warp each
  int* d_xs_order = nullptr;   // [long blocks | short blocks]
  // resident PCG on explicit S (xs_pcg.cuh): one cooperative launch per SCHUR_JACOBI solve
  bool xs_pcg = false;
  XsPcgArgs xpa{};             // the plan's geometry and the device arrays; the solve fills in its options and vectors
  size_t xs_pcg_smem = 0;
  // SPARSE_SCHUR (sparse_plan.cuh, sparse_schur.cuh): the row structure in the internal order, kept for the symbolic analysis
  // of the first sparse solve, and what that analysis uploads
  std::vector<int> h_cam_idx, h_pt_idx, h_pt_ptr;
  bool sp_ready = false;
  bool xs_arrays = false;       // the arrays xs_assemble_dev reads exist (explicit plan, or uploaded by the sparse analysis)
  SparseView<double> spv{};
  SparseView<float> spv32{};    // the same structure with a float factor and vector (mixed-precision solves)
  long long sp_storage = 0;     // entries of factor storage
  int sp_grid = 0, sp_grid32 = 0;
  size_t sp_smem = 0, sp_smem32 = 0;
  int* d_sp_cnt_init = nullptr;
  int* d_sp_cnt_inv = nullptr;  // [ns] SparsePlan::cnt_inv
  int sp_selinv_grid = 0;
  size_t sp_selinv_smem = 0;
  double sp_selinv_flops = 0.0;
  // b200_covariance_compute (covariance.cuh): the snapshot the getters read, and the scratch that forms it
  bool cov_valid = false;
  int cov_alg = B200_SPARSE_SCHUR;
  std::vector<int> cov_row_ptr, cov_blk_col;   // S's block pattern (sparse snapshot): block row ptr, block columns
  std::vector<uint16_t> cov_cam_mask;          // [C] the constant coordinates of each camera of the snapshot (bit k)
  int* d_cov_row_ptr = nullptr;                // [C + 1]
  double* d_cov_s = nullptr;                   // sparse: Z on S's blocks [81 x blocks], row-major, S's block order
  double* d_cov_dense = nullptr;               // dense: S, its factor, then Z's lower triangle [9C][9C]
  double* d_cov_diag = nullptr;                // dense: S's diagonal before the factorisation [9C]
  double* d_cov_work = nullptr;
  int cov_lwork = 0;
  double* d_cov_z = nullptr;                   // sparse: Z in the factor's panel layout [sp_storage]
  double* d_cov_pts = nullptr;                 // [9P] Cov(p, p), caller's point order
  unsigned long long* d_cov_min = nullptr;     // the conditioning test's minimum, as bits, and the dense info
  int4* d_cov_pairs = nullptr;
  double* d_cov_out = nullptr;
  size_t cov_pairs_cap = 0;
  double* d_red = nullptr;    // per-CTA partial sums of cg_vector_kernel
  // multi-GPU exchange of the per-iteration partial products over NVLink peer memory (cg_kernel.cuh: xchg_push_kernel +
  // the gather in cg_vector_kernel); replaces the ncclAllReduce inside the PCG iteration when every peer could be mapped
  bool xchg_ok = false;
  uint4* d_xchg = nullptr;        // [2 slots][world][9C] packets {lo, epoch, hi, epoch}
  XchgPeers xpeers{};
  void* xchg_opened[kMaxXchgRanks] = {};
  unsigned xepoch = 0;
  int cg_grid = 1;
  // b200_set_exact_solve_options: LinearSolver::Options::use_mixed_precision_solves and max_num_refinement_iterations
  // (linear_solver.h:226-227) of the DENSE_SCHUR and SPARSE_SCHUR solves
  bool mixed = false;
  int refine = 0;
  int ordering = B200_AMD;    // b200_set_linear_solver_ordering_type: the camera order of the SPARSE_SCHUR analysis
  HostMirrors hm;             // host-boundary LM loop vectors
  // launch geometry
  int grid_tile[K_COUNT];
  // stats
  int64_t launches[K_COUNT];
  int64_t ops[K_COUNT];       // operations: an operation is one logical pass (e.g. one S*x); it may take several launches
  double ms[K_COUNT];
  double bytes_per_op[K_COUNT];
  int64_t h2d_bytes = 0, d2h_bytes = 0;
  bool profiling = false;
  std::vector<EventPair> pending;
  std::vector<cudaEvent_t> event_pool;
};

namespace {

// Device allocation of n elements (at least one), owned by the handle: b200_destroy frees it.
template <typename T>
int dev_alloc(b200_handle* h, T** p, size_t n) {
  if (n == 0) n = 1;
  CU(cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)));
  h->allocs.push_back(*p);
  return B200_OK;
}
// Frees one allocation of dev_alloc before the handle is destroyed.
template <typename T>
void dev_free(b200_handle* h, T*& p) {
  if (p == nullptr) return;
  void* q = const_cast<void*>(static_cast<const void*>(p));
  h->allocs.erase(std::find(h->allocs.begin(), h->allocs.end(), q));
  cudaFree(q);
  p = nullptr;
}
// dev_alloc of a device copy of `src`, uploaded on the handle's stream.
template <typename T>
int upload(b200_handle* h, const std::vector<T>& src, T** dst) {
  OK(dev_alloc(h, dst, src.size()));
  if (!src.empty()) CU(cudaMemcpyAsync(*dst, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice, h->stream));
  return B200_OK;
}
template <typename T>
int upload(b200_handle* h, const std::vector<T>& src, const T** dst) {
  T* p = nullptr;
  OK(upload(h, src, &p));
  *dst = p;
  return B200_OK;
}

int h2d(b200_handle* h, void* dst, const void* src, size_t bytes) {
  CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, h->stream));
  h->h2d_bytes += static_cast<int64_t>(bytes);
  return B200_OK;
}
int d2h(b200_handle* h, void* dst, const void* src, size_t bytes) {
  CU(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  h->d2h_bytes += static_cast<int64_t>(bytes);
  return B200_OK;
}

// ---- boundary copies in the CALLER's block order (identity order: plain copies)
int permute_blocks(b200_handle* h, bool gather, size_t nblocks, int w, const int* d_perm, const double* d_src, double* d_dst) {
  const int grid = static_cast<int>(std::max<size_t>(1, std::min<size_t>((nblocks * w + 255) / 256, static_cast<size_t>(h->sm_count) * 8)));
  if (gather) permute_gather_kernel<<<grid, 256, 0, h->stream>>>(nblocks, w, d_perm, d_src, d_dst);
  else permute_scatter_kernel<<<grid, 256, 0, h->stream>>>(nblocks, w, d_perm, d_src, d_dst);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B200_ERR_CUDA, "permute kernel: %s", cudaGetErrorString(e));
  return B200_OK;
}
// parameter-sized vector [3P | 9C]
int up_params(b200_handle* h, double* d_dst, const double* host) {
  const size_t bytes = sizeof(double) * h->np;
  if (!h->permuted) return h2d(h, d_dst, host, bytes);
  OK(h2d(h, h->d_stage_p, host, bytes));
  OK(permute_blocks(h, true, h->P, 3, h->d_pt_perm, h->d_stage_p, d_dst));
  const size_t off = 3 * static_cast<size_t>(h->P);
  CU(cudaMemcpyAsync(d_dst + off, h->d_stage_p + off, sizeof(double) * 9 * h->C, cudaMemcpyDeviceToDevice, h->stream));
  return B200_OK;
}
int down_params(b200_handle* h, double* host, const double* d_src) {
  const size_t bytes = sizeof(double) * h->np;
  if (!h->permuted) return d2h(h, host, d_src, bytes);
  OK(permute_blocks(h, false, h->P, 3, h->d_pt_perm, d_src, h->d_stage_p));
  const size_t off = 3 * static_cast<size_t>(h->P);
  CU(cudaMemcpyAsync(h->d_stage_p + off, d_src + off, sizeof(double) * 9 * h->C, cudaMemcpyDeviceToDevice, h->stream));
  return d2h(h, host, h->d_stage_p, bytes);
}
// residual-sized vector [2N]
int up_rows(b200_handle* h, double* d_dst, const double* host) {
  const size_t bytes = sizeof(double) * 2 * static_cast<size_t>(h->N);
  if (!h->permuted) return h2d(h, d_dst, host, bytes);
  OK(h2d(h, h->d_stage_r, host, bytes));
  return permute_blocks(h, true, h->N, 2, h->d_row_perm, h->d_stage_r, d_dst);
}
int down_rows(b200_handle* h, double* host, const double* d_src) {
  const size_t bytes = sizeof(double) * 2 * static_cast<size_t>(h->N);
  if (!h->permuted) return d2h(h, host, d_src, bytes);
  OK(permute_blocks(h, false, h->N, 2, h->d_row_perm, d_src, h->d_stage_r));
  return d2h(h, host, h->d_stage_r, bytes);
}

int resolve_events(b200_handle* h) {
  if (h->pending.empty()) return B200_OK;
  CU(cudaStreamSynchronize(h->stream));
  for (auto& ep : h->pending) {
    float t = 0.f;
    CU(cudaEventElapsedTime(&t, ep.a, ep.b));
    h->ms[ep.kernel] += t;
    h->event_pool.push_back(ep.a);
    h->event_pool.push_back(ep.b);
  }
  h->pending.clear();
  return B200_OK;
}

int get_event(b200_handle* h, cudaEvent_t* e) {
  if (!h->event_pool.empty()) {
    *e = h->event_pool.back();
    h->event_pool.pop_back();
    return B200_OK;
  }
  CU(cudaEventCreate(e));
  return B200_OK;
}

// Launch wrapper: counts the launch, optionally brackets it with CUDA events, checks the launch error.
// primary = false: an auxiliary launch of the same operation (the few >32-row points, the huge points, a helper pass):
// its time is billed to the operation, which is counted once.
template <typename F>
int launch(b200_handle* h, int kid, F&& f, bool primary = true) {
  EventPair ep{};
  if (h->profiling) {
    if (h->pending.size() >= 8192) OK(resolve_events(h));
    OK(get_event(h, &ep.a));
    OK(get_event(h, &ep.b));
    ep.kernel = kid;
    CU(cudaEventRecord(ep.a, h->stream));
  }
  f();
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(B200_ERR_CUDA, "launch of %s failed: %s", kKernelNames[kid], cudaGetErrorString(e));
  h->launches[kid]++;
  if (primary) h->ops[kid]++;
  if (h->profiling) {
    CU(cudaEventRecord(ep.b, h->stream));
    h->pending.push_back(ep);
  }
  return B200_OK;
}

int flat_grid(const b200_handle* h, size_t n, int block) {
  const size_t want = (n + block - 1) / block;
  const size_t cap = static_cast<size_t>(h->sm_count) * 8;
  return static_cast<int>(std::max<size_t>(1, std::min(want, cap)));
}

int allreduce_sum(b200_handle* h, double* buf, size_t n) {
#ifdef B200_WITH_NCCL
  if (h->world > 1) {
    ncclResult_t r = g_nccl.AllReduce(buf, buf, n, ncclDouble, ncclSum, h->comm, h->stream);
    if (r != ncclSuccess) return fail(B200_ERR_NCCL, "ncclAllReduce: %s", g_nccl.GetErrorString(r));
  }
#else
  (void)h; (void)buf; (void)n;
#endif
  return B200_OK;
}

template <typename K>
int tile_grid(b200_handle* h, K kernel, size_t smem) {
  int per_sm = 1;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kTile, smem) != cudaSuccess || per_sm < 1) per_sm = 1;
  return std::max(1, std::min(h->num_tiles, h->sm_count * per_sm));
}

// Point-sized entries of the huge points: zeroed before a kernel that accumulates them slice by slice.
int huge_zero(b200_handle* h, double* d_point_vec) {
  if (h->num_huge == 0) return B200_OK;
  return launch(h, K_MISC, [&] { huge_zero3_kernel<<<(3 * h->num_huge + 255) / 256, 256, 0, h->stream>>>(h->num_huge, h->d_huge_pts, d_point_vec); });
}
int huge_grid(const b200_handle* h) { return std::max(1, std::min(h->num_huge, h->sm_count * 4)); }

// ------------------------------------------------------------------------------------------------ device-pointer cores
int sqnorm_dev(b200_handle* h, double* d_out);

// The evaluate kernels of the plan for one class of loss set (loss.cuh); *num_partials = the per-tile / per-CTA cost
// partials they wrote.
template <int kLoss, bool kFixed>
int evaluate_launch(b200_handle* h, EvalArgs a, bool want_jacobian, double* d_sqnorm, bool* sqnorm_done, int* num_partials) {
  const bool with_j = want_jacobian || a.gradient != nullptr;
  const size_t coff = 3 * static_cast<size_t>(h->P);
  const size_t smem = tile_smem_bytes<3, 1>();
  *num_partials = h->num_tiles;
  if (with_j && is_v4(h->mul)) {
    EvalArgs e = a;
    e.sqnorm = d_sqnorm;   // the CTA-tile kernel below leaves them to sqnorm_kernel
    if (d_sqnorm != nullptr) CU(cudaMemsetAsync(d_sqnorm + coff, 0, sizeof(double) * 9 * h->C, h->stream));
    if (d_sqnorm != nullptr) OK(huge_zero(h, d_sqnorm));
    OK(launch(h, K_EVAL_JAC, [&] {
      if (want_jacobian) evaluate_v2_kernel<kLoss, true, kFixed><<<h->v2.num_ctas, 32 * h->v2.warps, h->eval_v2_smem, h->stream>>>(h->v2_eval, e);
      else evaluate_v2_kernel<kLoss, false, kFixed><<<h->v2.num_ctas, 32 * h->v2.warps, h->eval_v2_smem, h->stream>>>(h->v2_eval, e);
    }));
    *num_partials = h->v2.num_ctas;
    if (h->num_big_tiles > 0) {  // the few >32-row points: CTA-tile kernels on their tiles only
      a.cost_partial = h->d_tile_partial + *num_partials;
      OK(launch(h, K_EVAL_JAC, [&] {
        const int grid = std::min(h->num_big_tiles, h->sm_count * 2);
        if (want_jacobian) evaluate_kernel<kLoss, true, true, kFixed><<<grid, kTile, smem, h->stream>>>(h->view_big, a);
        else evaluate_kernel<kLoss, true, false, kFixed><<<grid, kTile, smem, h->stream>>>(h->view_big, a);
      }, false));
      *num_partials += h->num_big_tiles;
      if (d_sqnorm != nullptr)
        OK(launch(h, K_SQNORM, [&] {
          sqnorm_kernel<<<std::min(h->num_big_tiles, h->sm_count * 4), kTile, tile_smem_bytes<3, 1>(), h->stream>>>(h->view_big, d_sqnorm);
        }, false));
    }
    if (d_sqnorm != nullptr) {
      OK(allreduce_sum(h, d_sqnorm + coff, 9 * static_cast<size_t>(h->C)));
      if (sqnorm_done != nullptr) *sqnorm_done = true;
    }
  } else if (with_j) {
    OK(launch(h, K_EVAL_JAC, [&] {
      if (want_jacobian) evaluate_kernel<kLoss, true, true, kFixed><<<h->grid_tile[K_EVAL_JAC], kTile, smem, h->stream>>>(h->view, a);
      else evaluate_kernel<kLoss, true, false, kFixed><<<h->grid_tile[K_EVAL_JAC], kTile, smem, h->stream>>>(h->view, a);
    }));
  } else {
    OK(launch(h, K_EVAL_COST, [&] { evaluate_kernel<kLoss, false><<<h->grid_tile[K_EVAL_COST], kTile, smem, h->stream>>>(h->view, a); }));
  }
  return B200_OK;
}
template <int kLoss>
int evaluate_launch(b200_handle* h, EvalArgs a, bool want_jacobian, double* d_sqnorm, bool* sqnorm_done, int* num_partials) {
  if (h->fixed_any) return evaluate_launch<kLoss, true>(h, a, want_jacobian, d_sqnorm, sqnorm_done, num_partials);
  return evaluate_launch<kLoss, false>(h, a, want_jacobian, d_sqnorm, sqnorm_done, num_partials);
}

// What a write of the stored J makes stale: the explicit S and the per-row blocks Q_r of the implicit-Schur
// initialisation.  The initialisation itself stays: the b200_schur_* entry points keep using its (E'E + D^2)^-1.
void jacobian_written(b200_handle* h) {
  h->xs_ready = false;
  h->q_from_init = false;
}

// d_sqnorm (optional): squared column norms of the Jacobian as written (after the fused scaling), for free with the
// warp-tile kernel; the caller falls back to sqnorm_dev when *sqnorm_done comes back false.
// J is computed (and checked) when the Jacobian or the gradient is asked for, and stored only when want_jacobian: a
// gradient-only evaluation leaves the device-resident Jacobian as it was, as Ceres leaves it with jacobian == NULL.
int evaluate_dev(b200_handle* h, const double* d_state, double* d_residuals, double* d_gradient, bool want_jacobian,
                 const double* d_scale, double* cost_out, double* d_sqnorm = nullptr, bool* sqnorm_done = nullptr) {
  if (!want_jacobian) d_sqnorm = nullptr;   // the column norms are those of the stored Jacobian
  else jacobian_written(h);
  EvalArgs a{};
  a.state = d_state;
  a.residuals = d_residuals;
  a.gradient = d_gradient;
  a.cost_partial = h->d_tile_partial;
  a.scale = d_scale;
  a.fail_flag = h->d_fail;
  a.loss.one = h->loss_one;
  if (h->loss_rows) {
    a.loss.row_loss = h->d_row_loss;
    a.loss.table = h->d_loss_table;
  }
  a.block_state = h->d_block_state;
  if (sqnorm_done != nullptr) *sqnorm_done = false;
  CU(cudaMemsetAsync(h->d_fail, 0, sizeof(int), h->stream));
  if (d_gradient != nullptr) CU(cudaMemsetAsync(d_gradient + 3 * static_cast<size_t>(h->P), 0, sizeof(double) * 9 * h->C, h->stream));
  if (d_gradient != nullptr) OK(huge_zero(h, d_gradient));
  int num_partials = 0;
  switch (h->apply_loss ? h->loss_cls : kLossTrivial) {
    case kLossTrivial: OK(evaluate_launch<kLossTrivial>(h, a, want_jacobian, d_sqnorm, sqnorm_done, &num_partials)); break;
    case kLossHuber: OK(evaluate_launch<kLossHuber>(h, a, want_jacobian, d_sqnorm, sqnorm_done, &num_partials)); break;
    default: OK(evaluate_launch<kLossGeneral>(h, a, want_jacobian, d_sqnorm, sqnorm_done, &num_partials)); break;
  }
  OK(launch(h, K_MISC, [&] { sum_kernel<<<1, kVecThreads, 0, h->stream>>>(num_partials, h->d_tile_partial, h->d_scalars); }));
  if (d_gradient != nullptr) OK(allreduce_sum(h, d_gradient + 3 * static_cast<size_t>(h->P), 9 * static_cast<size_t>(h->C)));
  OK(allreduce_sum(h, h->d_scalars, 1));
  CU(cudaMemcpyAsync(h->h_scalars, h->d_scalars, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  if (h->world > 1) {  // a failure on any shard fails the evaluation on every rank
    OK(launch(h, K_MISC, [&] { flag_to_double_kernel<<<1, 1, 0, h->stream>>>(h->d_fail, h->d_scalars + 2); }));
#ifdef B200_WITH_NCCL
    ncclResult_t r = g_nccl.AllReduce(h->d_scalars + 2, h->d_scalars + 2, 1, ncclDouble, ncclMax, h->comm, h->stream);
    if (r != ncclSuccess) return fail(B200_ERR_NCCL, "ncclAllReduce: %s", g_nccl.GetErrorString(r));
#endif
    OK(launch(h, K_MISC, [&] { double_to_flag_kernel<<<1, 1, 0, h->stream>>>(h->d_scalars + 2, h->d_fail); }));
  }
  CU(cudaMemcpyAsync(h->h_fail, h->d_fail, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  *cost_out = h->h_scalars[0];
  if (*h->h_fail != 0 || !std::isfinite(*cost_out))
    return fail(B200_ERR_EVALUATION_FAILED, "non-finite residual, Jacobian or cost");
  return B200_OK;
}

int sqnorm_dev(b200_handle* h, double* d_out) {
  CU(cudaMemsetAsync(d_out + 3 * static_cast<size_t>(h->P), 0, sizeof(double) * 9 * h->C, h->stream));
  OK(huge_zero(h, d_out));
  OK(launch(h, K_SQNORM, [&] {
    sqnorm_kernel<<<h->grid_tile[K_SQNORM], kTile, tile_smem_bytes<3, 1>(), h->stream>>>(h->view, d_out);
  }));
  return allreduce_sum(h, d_out + 3 * static_cast<size_t>(h->P), 9 * static_cast<size_t>(h->C));
}

// Zeroes the stored Jacobian's cells of the handle's constant components (none: nothing to do).
int fixed_mask_dev(b200_handle* h) {
  if (!h->fixed_any) return B200_OK;
  jacobian_written(h);
  return launch(h, K_SCALE, [&] {
    fixed_mask_kernel<<<flat_grid(h, 12 * static_cast<size_t>(h->N), 256), 256, 0, h->stream>>>(h->view, h->d_fixed);
  }, false);
}

int scale_dev(b200_handle* h, const double* d_scale) {
  jacobian_written(h);
  return launch(h, K_SCALE, [&] {
    scale_kernel<<<flat_grid(h, 12 * static_cast<size_t>(h->N), 256), 256, 0, h->stream>>>(h->view, d_scale);
  });
}

// (Re)assembles S for the current implicit-Schur initialisation; also writes the diagonal blocks into d_upper45.
// Billed as the block-diagonal operation of the elimination, which it replaces.
int xs_assemble_dev(b200_handle* h) {
  // the blocks with long pair lists (the diagonal ones, mostly) first, one CTA each; then one warp per block
  OK(launch(h, K_DIAG_BLOCKS, [&] {
    if (h->num_xs_long > 0)
      xs_assemble_kernel<true><<<std::min(h->num_xs_long, h->sm_count * 32), kXsAsmThreads, 0, h->stream>>>(
          h->xsv, h->view, h->d_xs_order, h->num_xs_long, h->d_ete_inv, h->d_upper45);
    if (h->num_xs_short > 0)
      xs_assemble_kernel<false><<<std::min((h->num_xs_short + kXsAsmThreads / 32 - 1) / (kXsAsmThreads / 32), h->sm_count * 32),
                                  kXsAsmThreads, 0, h->stream>>>(h->xsv, h->view, h->d_xs_order + h->num_xs_long, h->num_xs_short,
                                                                 h->d_ete_inv, h->d_upper45);
  }));
  h->xs_ready = true;
  h->xs_diag_ready = true;
  return B200_OK;
}

// ImplicitSchurComplement::Init on device pointers b [2N], D [3P+9C] or null.
int schur_init_dev(b200_handle* h, const double* d_b, const double* d_D) {
  if (h->fixed_any) {   // D' = 1 on the constant components: every later stage of the solve reads cur_D
    OK(launch(h, K_LM_VEC, [&] {
      solve_diagonal_kernel<<<flat_grid(h, h->np, 256), 256, 0, h->stream>>>(h->np, d_D, h->d_fixed, h->d_solve_D);
    }, false));
    d_D = h->d_solve_D;
  }
  SchurState st{};
  st.b = d_b;
  st.D = d_D;
  st.ete_inv = h->d_ete_inv;
  st.rhs = h->d_rhs;
  st.ye = h->d_ye;
  CU(cudaMemsetAsync(h->d_rhs, 0, sizeof(double) * 9 * h->C, h->stream));
  h->q_from_init = false;
  h->xs_ready = false;
  if (is_v4(h->mul)) {
    // v4 machinery: E, F, b and the tile's D_e through the TMA slot; also writes the per-row 2x2 blocks Q_r the camera-major
    // block-diagonal pass reads (no separate pass over E for them)
    InitV4Args ia{};
    ia.b = d_b;
    ia.D = d_D;
    ia.ete_inv = h->d_ete_inv;
    ia.rhs = h->d_rhs;
    ia.ye = nullptr;   // (E'E)^-1 E'b is not consumed by anything on this path: not written
    ia.q3 = h->diag == DiagPass::CamMajor ? h->d_q3 : nullptr;
    OK(launch(h, K_SCHUR_INIT, [&] {
      V2View iv = h->v2_mul;
      iv.cta_big = h->d_cta_big;   // the kernel takes the CTA's 33..kTile-row points itself
      if (h->mul == MulFamily::V4Owned) schur_init_v4_kernel<true><<<h->v2.num_ctas, 32 * h->v2_mul.warps, h->mul_smem, h->stream>>>(iv, ia);
      else schur_init_v4_kernel<false><<<h->v2.num_ctas, 32 * h->v2_mul.warps, h->mul_smem, h->stream>>>(iv, ia);
    }));
    h->q_from_init = ia.q3 != nullptr;
  } else {
    OK(launch(h, K_SCHUR_INIT, [&] {
      schur_init_kernel<<<h->grid_tile[K_SCHUR_INIT], kTile, tile_smem_bytes<9, 3>(), h->stream>>>(h->view, st);
    }));
  }
  if (h->num_huge > 0)
    OK(launch(h, K_SCHUR_INIT, [&] {
      huge_schur_init_kernel<<<huge_grid(h), kHugeThreads, 0, h->stream>>>(h->view, h->num_huge, h->d_huge_pts, st);
    }, false));
  if (h->q_from_init && h->view_chunks.num_tiles > 0)   // Q_r of the slices of the huge points (needs their (E'E)^-1)
    OK(launch(h, K_SCHUR_INIT, [&] {
      row_q_tiles_kernel<<<std::min(h->view_chunks.num_tiles, h->sm_count * 8), kTile, 0, h->stream>>>(h->view_chunks, h->d_ete_inv, h->d_q3);
    }, false));
  OK(allreduce_sum(h, h->d_rhs, 9 * static_cast<size_t>(h->C)));
  h->cur_b = d_b;
  h->cur_D = d_D;
  h->schur_ready = true;
  return B200_OK;
}

// Launch with programmatic dependent launch allowed when `pdl`: the kernel's prologue overlaps the tail of the kernel
// before it on the stream.
template <typename... KArgs, typename... Args>
void launch_pdl(void (*kernel)(KArgs...), int grid, int block, size_t smem, cudaStream_t stream, bool pdl, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl ? 1 : 0;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  cudaLaunchKernelEx(&cfg, kernel, args...);
}

// y = D^2 x on the camera blocks (D may be null: y = 0), the seed of a product that adds into y.
int diag_sq_mul_dev(b200_handle* h, const double* d2, const double* x, double* y, const int* done_flag) {
  const int n = 9 * h->C;
  return launch(h, K_MISC, [&] { diag_sq_mul_kernel<<<flat_grid(h, n, 256), 256, 0, h->stream>>>(n, d2, x, y, done_flag); });
}

// How one S x is launched.
struct MulOpts {
  bool explicit_s = false;      // on the assembled upper triangle of S (explicit_schur.cuh) instead of the implicit product
  bool seeded = false;          // y already holds D_f^2 x (rank 0; the PCG's vector kernel wrote it): the product only adds
  bool pdl = false;             // programmatic dependent launch of the v4 and explicit-S products
  const int* done = nullptr;    // device flag: every launch is a no-op once the PCG has terminated
  double* pq_parts = nullptr;   // per-CTA partials of p.q, fused into the flush of the v4 and explicit-S products
  bool exchange = false;        // the vector kernel sums the ranks' partial products over peer memory: no all-reduce
  bool xs_columns_in_cg = false;  // explicit S: the PCG's vector kernel adds the column part from T (no gather launch)
};

// y = S x on device vectors [9C], with S = F'F + D_f^2 - F'E (E'E + D_e^2)^-1 E'F of the current initialisation.
int schur_mul_dev(b200_handle* h, const double* d_x, double* d_y, const MulOpts& o) {
  const double* Df = h->cur_D != nullptr ? h->cur_D + 3 * static_cast<size_t>(h->P) : nullptr;
  if (o.explicit_s) {
    if (!h->xs_ready) OK(xs_assemble_dev(h));
    OK(launch(h, K_SCHUR_MUL, [&] {
      launch_pdl(xs_mul_kernel, h->xs_grid, kXsThreads, 0, h->stream, o.pdl, h->xsv, d_x, d_y, o.seeded ? nullptr : Df,
                 o.seeded ? 1 : 0, o.done, o.pq_parts);
    }));
    if (o.xs_columns_in_cg) return B200_OK;
    return launch(h, K_SCHUR_MUL, [&] {
      xs_gather_kernel<<<(9 * h->C + 255) / 256, 256, 0, h->stream>>>(h->xsv, d_y);
    }, false);
  }
  const int n = 9 * h->C;
  const double* seed = (h->rank == 0) ? Df : nullptr;
  const bool direct = h->mul == MulFamily::Tile || h->v2.direct;   // the product adds into y: seeded first
  if (direct && !o.seeded) OK(diag_sq_mul_dev(h, seed, d_x, d_y, o.done));
  // The handful of >32-row points runs on a side stream, concurrently with the warp-tile kernel (both only add into the
  // pre-seeded output with REDs); outside profiling mode, where launches are bracketed by events.
  const bool big = h->num_big_tiles > 0 && !h->big_folded;
  const bool side = big && o.seeded && !h->profiling;
  auto big_points = [&](cudaStream_t s) {
    schur_mul_kernel<<<std::min(h->num_big_tiles, h->sm_count * 4), kTile, tile_smem_bytes<3, 3>(), s>>>(h->view_big, h->d_ete_inv,
                                                                                                       d_x, d_y, o.done);
  };
  if (side) {
    CU(cudaEventRecord(h->ev_fork, h->stream));
    CU(cudaStreamWaitEvent(h->stream2, h->ev_fork, 0));
    big_points(h->stream2);
    h->launches[K_SCHUR_MUL_BIG]++;
    CU(cudaEventRecord(h->ev_join, h->stream2));
  }
  OK(launch(h, K_SCHUR_MUL, [&] {
    const int ctas = h->v2.num_ctas, threads = 32 * h->v2_mul.warps;
    switch (h->mul) {
      case MulFamily::V4Owned:
        launch_pdl(schur_mul_v4_kernel<true>, ctas, threads, h->mul_smem, h->stream, o.pdl, h->v2_mul,
                   static_cast<const double*>(h->d_ete_inv), d_x, d_y, o.done, o.pq_parts);
        break;
      case MulFamily::V4:
        launch_pdl(schur_mul_v4_kernel<false>, ctas, threads, h->mul_smem, h->stream, o.pdl, h->v2_mul,
                   static_cast<const double*>(h->d_ete_inv), d_x, d_y, o.done, o.pq_parts);
        break;
      case MulFamily::V3:
        schur_mul_v3_kernel<<<ctas, threads, h->mul_smem, h->stream>>>(h->v2_mul, h->d_ete_inv, d_x, d_y, o.done);
        break;
      case MulFamily::Tile:
        schur_mul_kernel<<<h->grid_tile[K_SCHUR_MUL], kTile, tile_smem_bytes<3, 3>(), h->stream>>>(h->view, h->d_ete_inv, d_x, d_y, o.done);
        break;
    }
  }));
  if (!direct)
    OK(launch(h, K_CAM_REDUCE, [&] {
      cam_reduce_kernel<<<(n + 63) / 64, 256, h->v2.num_ctas * sizeof(int2), h->stream>>>(
          n, h->v2.num_ctas, h->v2.cta_cam, h->v2.partials, 9 * h->v2.max_cam_span, seed, d_x, d_y, 0, o.done);
    }));
  if (side) CU(cudaStreamWaitEvent(h->stream, h->ev_join, 0));
  else if (big) OK(launch(h, K_SCHUR_MUL_BIG, [&] { big_points(h->stream); }, false));
  if (h->num_huge > 0)
    OK(launch(h, K_SCHUR_MUL_BIG, [&] {
      huge_schur_mul_kernel<<<huge_grid(h), kHugeThreads, 0, h->stream>>>(h->view, h->num_huge, h->d_huge_pts, h->d_ete_inv, d_x, d_y, o.done);
    }, false));
  return o.exchange ? B200_OK : allreduce_sum(h, d_y, n);
}

// x_e = (E'E + D_e^2)^-1 E'(b - F z) (the point part of the solution) for the camera part z of the current initialisation.
int back_substitute_dev(b200_handle* h, const double* d_b, const double* d_z, double* d_x) {
  OK(launch(h, K_BACKSUB, [&] {
    backsub_kernel<<<h->grid_tile[K_BACKSUB], kTile, tile_smem_bytes<3, 1>(), h->stream>>>(h->view, h->d_ete_inv, d_b, d_z, d_x);
  }));
  if (h->num_huge > 0)
    OK(launch(h, K_BACKSUB, [&] {
      huge_backsub_kernel<<<huge_grid(h), kHugeThreads, 0, h->stream>>>(h->view, h->num_huge, h->d_huge_pts, h->d_ete_inv, d_b, d_z, d_x);
    }, false));
  return B200_OK;
}

int precond_update_dev(b200_handle* h, int type) {
  if (type == B200_PRECOND_IDENTITY) return B200_OK;
  const double* Df = h->cur_D != nullptr ? h->cur_D + 3 * static_cast<size_t>(h->P) : nullptr;
  const bool schur = type == B200_PRECOND_SCHUR_JACOBI;
  if (h->xs && schur) {
    // the diagonal blocks of the explicit S: no pass of their own
    if (!h->xs_ready || !h->xs_diag_ready) OK(xs_assemble_dev(h));
  } else {
    h->xs_diag_ready = false;
    CU(cudaMemsetAsync(h->d_upper45, 0, sizeof(double) * 45 * h->C, h->stream));
    if (h->diag == DiagPass::CamMajor) {
      if (schur && !h->q_from_init)
        OK(launch(h, K_DIAG_BLOCKS, [&] {
          row_q_kernel<<<flat_grid(h, h->N, 256), 256, 0, h->stream>>>(h->view, h->d_ete_inv, h->d_q3);
        }, false));
      OK(launch(h, K_DIAG_BLOCKS, [&] {
        const int g = std::max(1, std::min((h->num_cam_items + 3) / 4, h->sm_count * 12));
        const size_t smem = static_cast<size_t>(kCamBlkThreads / 32) * kCamBlkWarpBytes;
        if (schur) cam_blocks_v2_kernel<true><<<g, kCamBlkThreads, smem, h->stream>>>(h->view, h->num_cam_items, h->d_cam_items, h->d_cam_rows, h->d_q3, h->d_upper45);
        else cam_blocks_v2_kernel<false><<<g, kCamBlkThreads, smem, h->stream>>>(h->view, h->num_cam_items, h->d_cam_items, h->d_cam_rows, h->d_q3, h->d_upper45);
      }));
    } else if (h->diag == DiagPass::WarpTile) {
      OK(launch(h, K_DIAG_BLOCKS, [&] {
        if (schur)
          diag_blocks_v2_kernel<true><<<h->v2.num_ctas, 32 * h->v2_diag.warps, h->diag_v2_smem, h->stream>>>(h->v2_diag, h->diag_v2_replicas, h->d_ete_inv, h->d_upper45);
        else
          diag_blocks_v2_kernel<false><<<h->v2.num_ctas, 32 * h->v2_diag.warps, h->diag_v2_smem, h->stream>>>(h->v2_diag, h->diag_v2_replicas, h->d_ete_inv, h->d_upper45);
      }));
      if (h->num_big_tiles > 0)
        OK(launch(h, K_DIAG_BLOCKS, [&] {
          const int g = std::min(h->num_big_tiles, h->sm_count);
          if (schur) diag_blocks_kernel<true><<<g, kTile, tile_smem_bytes<1, 1>(), h->stream>>>(h->view_big, h->d_ete_inv, h->d_upper45);
          else diag_blocks_kernel<false><<<g, kTile, tile_smem_bytes<1, 1>(), h->stream>>>(h->view_big, h->d_ete_inv, h->d_upper45);
        }, false));
    } else {
      OK(launch(h, K_DIAG_BLOCKS, [&] {
        if (schur) diag_blocks_kernel<true><<<h->grid_tile[K_DIAG_BLOCKS], kTile, tile_smem_bytes<1, 1>(), h->stream>>>(h->view, h->d_ete_inv, h->d_upper45);
        else diag_blocks_kernel<false><<<h->grid_tile[K_DIAG_BLOCKS], kTile, tile_smem_bytes<1, 1>(), h->stream>>>(h->view, h->d_ete_inv, h->d_upper45);
      }));
    }
    OK(allreduce_sum(h, h->d_upper45, 45 * static_cast<size_t>(h->C)));
  }
  return launch(h, K_INVERT9, [&] {
    invert9_kernel<<<(h->C + kInvWarps - 1) / kInvWarps, 32 * kInvWarps, 0, h->stream>>>(h->C, h->d_upper45, Df, h->d_blocks, h->d_minv);
  });
}

int reduce_partials(b200_handle* h, int blocks, int slots, unsigned op_mask, double* host_out, bool across_ranks);
int pcg_general_dev(b200_handle* h, const b200_solver_options* o);

// IterativeSchurComplementSolver::SolveImpl on device pointers.  d_x: [3P+9C] output.
int schur_solve_dev(b200_handle* h, const double* d_b, const double* d_D, const b200_solver_options* o, double* d_x,
                    b200_solver_summary* summary) {
  OK(schur_init_dev(h, d_b, d_D));
  const bool general = o->preconditioner_type == B200_PRECOND_SCHUR_POWER_SERIES_EXPANSION || o->use_spse_initialization != 0;
  // explicit S with SCHUR_JACOBI (the configuration the reference allows use_explicit_schur_complement in): the
  // assembly in precond_update_dev yields the preconditioner's blocks too
  const bool explicit_s = h->xs && !general && o->preconditioner_type == B200_PRECOND_SCHUR_JACOBI;
  if (!general) OK(precond_update_dev(h, o->preconditioner_type));
  const int n = 9 * h->C;
  CgParams prm{};
  prm.n = n;
  prm.min_iterations = o->min_num_iterations;
  prm.max_iterations = o->max_num_iterations;
  prm.q_tolerance = o->q_tolerance;
  prm.r_tolerance = o->r_tolerance;
  const double* Df = h->cur_D != nullptr ? h->cur_D + 3 * static_cast<size_t>(h->P) : nullptr;
  const int precond = o->preconditioner_type == B200_PRECOND_IDENTITY ? 0 : 1;
  CgVecArgs va{};
  va.prm = prm;
  va.C = h->C;
  va.precond = precond;
  va.minv = h->d_minv;
  va.rhs = h->d_rhs;
  va.x = h->d_sol;
  va.r = h->d_r;
  va.z = h->d_z;
  va.p = h->d_p;
  va.red = h->d_red;
  va.st = h->d_cg;
  auto finish = [&]() -> int {
    summary->num_iterations = h->h_cg->iteration;
    summary->termination_type = h->h_cg->termination;
    summary->residual_norm = h->h_cg->norm_r;
    if (summary->termination_type != B200_LS_FAILURE && summary->termination_type != B200_LS_FATAL_ERROR) {
      OK(back_substitute_dev(h, d_b, h->d_sol, d_x));
      CU(cudaMemcpyAsync(d_x + 3 * static_cast<size_t>(h->P), h->d_sol, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
    }
    return B200_OK;
  };
  // In direct-flush mode the vector kernel pre-seeds the next product's output (D_f^2 p, rank 0 only) and the product
  // kernels RED straight into it: one product launch + one vector launch per iteration.
  const bool seeded = h->v2.direct || explicit_s;
  va.Df = (h->rank == 0) ? Df : nullptr;
  // multi-GPU: the partial products travel through peer memory instead of an NCCL all-reduce (needs the direct-flush
  // product: `out` then holds exactly this rank's partial)
  const bool xchg = h->xchg_ok && h->v2.direct && !h->knobs.no_peer_exchange;
  auto vec = [&](int mode, double* q, double* seed_target) -> int {
    va.mode = mode;
    va.q = q;
    va.seed_target = seeded ? seed_target : nullptr;
    va.xg.world = 0;
    if (xchg && mode != CG_BEGIN) {   // q of this launch is this rank's partial product: exchange + sum inside the kernel
      va.xg = h->xpeers;
      va.xg_slot = static_cast<int>(h->xepoch & 1u);
      va.xg_epoch = h->xepoch;
    }
    void* args[] = {&va};
    return launch(h, K_CG_VEC, [&] {
      cudaLaunchCooperativeKernel(reinterpret_cast<void*>(cg_vector_kernel), dim3(h->cg_grid), dim3(kCgThreads), args, 0, h->stream);
    });
  };
  // p.q fused into the product's flush (single GPU, v4 kernel, direct flush, no separate big-point launch)
  const bool fuse_pq = (explicit_s || (seeded && is_v4(h->mul) && (h->world == 1 || xchg) && h->num_huge == 0 &&
                                       (h->num_big_tiles == 0 || h->big_folded))) &&
                       !h->knobs.no_fused_pq;
  MulOpts mo;
  mo.explicit_s = explicit_s;
  mo.seeded = seeded;
  mo.pdl = !h->knobs.no_pdl && !h->profiling;
  mo.done = &h->d_cg->done;
  mo.pq_parts = fuse_pq ? h->d_pq_parts : nullptr;
  mo.exchange = xchg;
  mo.xs_columns_in_cg = explicit_s;
  va.xs_col_ptr = explicit_s ? h->xsv.col_ptr : nullptr;
  va.xs_T = explicit_s ? h->xsv.T : nullptr;
  va.pq_parts = mo.pq_parts;
  va.num_pq_parts = fuse_pq ? (explicit_s ? h->xs_grid : h->v2.num_ctas) : 0;
  va.seed_pq = fuse_pq ? h->d_seed_pq : nullptr;
  auto product = [&](const double* vin, double* out) -> int {
    OK(schur_mul_dev(h, vin, out, mo));
    if (xchg) ++h->xepoch;   // the vector kernel that consumes this product exchanges it under this epoch
    return B200_OK;
  };
  if (general) {
    // SURVEY 8f.2: power-series preconditioner / initial guess -> the general-preconditioner PCG (host-side scalars)
    OK(pcg_general_dev(h, o));
    return finish();
  }
  if (explicit_s && h->xs_pcg) {
    // the whole solve in one cooperative launch with S in shared memory (xs_pcg.cuh): no batches, no polling
    if (!h->xs_ready) OK(xs_assemble_dev(h));
    XsPcgArgs a = h->xpa;
    a.prm = prm;
    a.reset = o->residual_reset_period > 0 ? o->residual_reset_period : std::numeric_limits<int>::max();
    a.minv = h->d_minv;
    a.rhs = h->d_rhs;
    a.Df = Df;
    a.x = h->d_sol;
    a.z = h->d_z;
    a.p[0] = h->d_p;
    a.st = h->d_cg;
    void* args[] = {&a};
    OK(launch(h, K_SCHUR_PCG, [&] {
      cudaLaunchCooperativeKernel(reinterpret_cast<void*>(xs_pcg_kernel), dim3(h->sm_count), dim3(kXpThreads), args, h->xs_pcg_smem,
                                  h->stream);
    }));
    CU(cudaMemcpyAsync(h->h_cg, h->d_cg, sizeof(CgState), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    // operations: the products of the solve, one per iteration that reached it (a failed rho / beta check counts the
    // iteration it could not start) and one per residual reset
    const CgState& s = *h->h_cg;
    const int its = std::max(0, s.iteration - (s.reason == 4 || s.reason == 5 ? 1 : 0));
    h->ops[K_SCHUR_PCG] += its + its / a.reset - 1;   // launch() counted one
#ifdef B200_DEV_KNOBS
    if (a.stamps != nullptr) {
      long long t[kXpPhases];
      CU(cudaMemcpy(t, a.stamps, sizeof(t), cudaMemcpyDeviceToHost));
      fprintf(stderr, "[b200ba] xs_pcg stamps (CTA 0, cycles, cumulative): begin %lld product %lld barrier1 %lld vector %lld barrier2 %lld tests %lld\n",
              t[0], t[1], t[2], t[3], t[4], t[5]);
    }
#endif
    return finish();
  }
  OK(vec(CG_BEGIN, h->d_z, h->d_z));
  const int reset = o->residual_reset_period > 0 ? o->residual_reset_period : std::numeric_limits<int>::max();
  // Termination is decided on the device; the host only polls the state every few iterations (kernels become
  // no-ops once done is set), and it polls one batch BEHIND what it has already enqueued, so the GPU never drains
  // while the host looks at the state: batch k+1 is in the queue before the host waits for the state after batch k.
  const int max_it = std::max(o->max_num_iterations, 1);
  int it = 0;
  auto batch = [&](int count) -> int {
    for (int k = 0; k < count && it < max_it; ++k) {
      ++it;
      // q aliases z exactly like the reference (conjugate_gradients_solver.h:193): z is dead once p is updated.
      OK(product(h->d_p, h->d_z));
      if (it % reset == 0) {
        OK(vec(CG_RESET_FIRST, h->d_z, h->d_tmp));
        OK(product(h->d_sol, h->d_tmp));
        OK(vec(CG_RESET_SECOND, h->d_tmp, h->d_z));
      } else {
        OK(vec(CG_NORMAL, h->d_z, h->d_z));
      }
    }
    return B200_OK;
  };
  if (h->profiling) {
    // instrumented runs poll after every iteration: no launches after termination, they would skew the per-kernel means
    bool done = false;
    while (!done) {
      OK(batch(1));
      CU(cudaMemcpyAsync(h->h_cg, h->d_cg, sizeof(CgState), cudaMemcpyDeviceToHost, h->stream));
      CU(cudaStreamSynchronize(h->stream));
      done = h->h_cg->done != 0 || it >= max_it;
    }
    return finish();
  }
  int check_every = 2;
  int pending = 0;
  OK(batch(check_every));
  CU(cudaMemcpyAsync(h->h_cg + pending, h->d_cg, sizeof(CgState), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaEventRecord(h->ev_cg[pending], h->stream));
  for (;;) {
    const bool more = it < max_it;
    if (more) {
      check_every = std::min(check_every * 2, 8);
      OK(batch(check_every));
      CU(cudaMemcpyAsync(h->h_cg + (1 - pending), h->d_cg, sizeof(CgState), cudaMemcpyDeviceToHost, h->stream));
      CU(cudaEventRecord(h->ev_cg[1 - pending], h->stream));
    }
    CU(cudaEventSynchronize(h->ev_cg[pending]));
    if (h->h_cg[pending].done != 0 || !more) {
      if (pending != 0) h->h_cg[0] = h->h_cg[pending];
      break;
    }
    pending = 1 - pending;
  }
  return finish();
}

// r = rhs_S - (S + D_f^2) x_f of the current initialisation into v (as T, by position through pinv, see
// refine_residual_kernel): the handle's FP64 product, on the stored S when the plan keeps it, the implicit one otherwise.
template <typename T>
int refine_residual_dev(b200_handle* h, const int* pinv, T* v) {
  const int n = 9 * h->C;
  MulOpts mo;
  mo.explicit_s = h->xs;
  OK(schur_mul_dev(h, h->d_sol, h->d_tmp, mo));
  return launch(h, K_REFINE, [&] {
    refine_residual_kernel<T><<<flat_grid(h, n, 256), 256, 0, h->stream>>>(n, pinv, h->d_rhs, h->d_tmp, v);
  });
}
// x_f (h->d_sol) += v widened, or x_f = v when !add.
template <typename T>
int refine_accumulate_dev(b200_handle* h, const int* pinv, const T* v, bool add) {
  const int n = 9 * h->C;
  return launch(h, K_REFINE, [&] {
    refine_accumulate_kernel<T><<<flat_grid(h, n, 256), 256, 0, h->stream>>>(n, pinv, v, h->d_sol, add ? 1 : 0);
  });
}

// DenseSchurComplementSolver (schur_complement_solver.cc:101-159, :161-214) on device pointers: explicit S by
// dense_schur_assemble_kernel, Cholesky by cuSOLVER, back substitution by the implicit-Schur kernels.  With mixed precision
// the FP64 assembly's lower triangle is rounded to float and factored by Spotrf; the float solve rounds its rhs and widens its
// result.  Iterative refinement makes 1 + max_num_refinement_iterations solves per factorisation, as EIGEN / LAPACK's
// RefinedDenseCholesky does.  (Ceres' CUDA dense path refines 2k times with mixed precision: k times inside
// CUDADenseCholeskyMixedPrecision::Solve, dense_cholesky.cc:604-630, and k more in the RefinedDenseCholesky wrapper
// DenseCholesky::Create adds, :113-133.  That doubling is not followed.)  A failure of a refinement's solve is ignored.
int dense_schur_solve_dev(b200_handle* h, const double* d_b, const double* d_D, double* d_x, b200_solver_summary* summary) {
  if (h->world > 1) return fail(B200_ERR_UNSUPPORTED, "the explicit Schur complement is single-GPU");
  const int n = 9 * h->C;
  const bool mixed = h->mixed;
  const size_t bytes = sizeof(double) * static_cast<size_t>(n) * n;
  const size_t cap_bytes = bytes + (mixed ? sizeof(float) * static_cast<size_t>(n) * n : 0);   // and the float copy
  if (cap_bytes > (static_cast<size_t>(48) << 30))
    return fail(B200_ERR_UNSUPPORTED, "dense reduced camera system of %d cameras needs %.1f GB", h->C, cap_bytes / 1e9);
  if (!load_cusolver()) return fail(B200_ERR_UNSUPPORTED, "cannot load libcusolver.so.11: %s", dlerror());
  if (mixed && !g_cusolver.float_ok)
    return fail(B200_ERR_UNSUPPORTED, "the loaded cuSOLVER lacks cusolverDnSpotrf / cusolverDnSpotrs (mixed-precision solves)");
  if (h->cusolver == nullptr) {
    if (g_cusolver.Create(&h->cusolver) != 0) return fail(B200_ERR_CUDA, "cusolverDnCreate failed");
    if (g_cusolver.SetStream(h->cusolver, h->stream) != 0) return fail(B200_ERR_CUDA, "cusolverDnSetStream failed");
  }
  if (h->d_dense_s == nullptr) {
    OK(dev_alloc(h, &h->d_dense_s, static_cast<size_t>(n) * n));
    OK(dev_alloc(h, &h->d_dense_info, 4));
    int lwork = 0;
    if (g_cusolver.DpotrfBufferSize(h->cusolver, /*CUBLAS_FILL_MODE_LOWER*/ 0, n, h->d_dense_s, n, &lwork) != 0)
      return fail(B200_ERR_CUDA, "cusolverDnDpotrf_bufferSize failed");
    h->dense_lwork = std::max(lwork, 1);
    OK(dev_alloc(h, &h->d_dense_work, static_cast<size_t>(h->dense_lwork)));
  }
  if (mixed && h->d_dense_s32 == nullptr) {
    OK(dev_alloc(h, &h->d_dense_s32, static_cast<size_t>(n) * n));
    OK(dev_alloc(h, &h->d_dense_v32, static_cast<size_t>(n)));
    int lwork = 0;
    if (g_cusolver.SpotrfBufferSize(h->cusolver, /*CUBLAS_FILL_MODE_LOWER*/ 0, n, h->d_dense_s32, n, &lwork) != 0)
      return fail(B200_ERR_CUDA, "cusolverDnSpotrf_bufferSize failed");
    h->dense_lwork32 = std::max(lwork, 1);
    OK(dev_alloc(h, &h->d_dense_work32, static_cast<size_t>(h->dense_lwork32)));
  }
  OK(schur_init_dev(h, d_b, d_D));   // (E'E + D^2)^-1 and the reduced right-hand side
  const double* Df = h->cur_D != nullptr ? h->cur_D + 3 * static_cast<size_t>(h->P) : nullptr;
  CU(cudaMemsetAsync(h->d_dense_s, 0, bytes, h->stream));
  OK(launch(h, K_DIAG_BLOCKS, [&] {
    dense_schur_assemble_kernel<<<std::max(1, std::min(h->P, h->sm_count * 8)), kDsThreads, 0, h->stream>>>(h->view, h->d_ete_inv, h->d_dense_s, static_cast<size_t>(n));
  }));
  OK(launch(h, K_MISC, [&] { dense_schur_diagonal_kernel<<<(n + 255) / 256, 256, 0, h->stream>>>(n, Df, h->d_dense_s, static_cast<size_t>(n)); }));
  // a solve with the factor, in place: in d_dense_v32 with mixed precision, in v otherwise (the refinement's solves report to
  // info[2], which is not read)
  auto solve = [&](double* v, int* info) -> int {
    if (mixed) {
      if (g_cusolver.Spotrs(h->cusolver, 0, n, 1, h->d_dense_s32, n, h->d_dense_v32, n, info) != 0)
        return fail(B200_ERR_CUDA, "cusolverDnSpotrs failed");
    } else if (g_cusolver.Dpotrs(h->cusolver, 0, n, 1, h->d_dense_s, n, v, n, info) != 0) {
      return fail(B200_ERR_CUDA, "cusolverDnDpotrs failed");
    }
    return B200_OK;
  };
  if (mixed) {
    OK(launch(h, K_REFINE, [&] {
      dense_round_lower_kernel<<<h->sm_count * 8, 256, 0, h->stream>>>(n, h->d_dense_s, h->d_dense_s32);
    }));
    if (g_cusolver.Spotrf(h->cusolver, 0, n, h->d_dense_s32, n, h->d_dense_work32, h->dense_lwork32, h->d_dense_info) != 0)
      return fail(B200_ERR_CUDA, "cusolverDnSpotrf failed");
    OK(launch(h, K_REFINE, [&] {
      refine_residual_kernel<float><<<flat_grid(h, n, 256), 256, 0, h->stream>>>(n, nullptr, h->d_rhs, nullptr, h->d_dense_v32);
    }));
    OK(solve(nullptr, h->d_dense_info + 1));
    OK(refine_accumulate_dev(h, nullptr, h->d_dense_v32, false));
  } else {
    if (g_cusolver.Dpotrf(h->cusolver, 0, n, h->d_dense_s, n, h->d_dense_work, h->dense_lwork, h->d_dense_info) != 0)
      return fail(B200_ERR_CUDA, "cusolverDnDpotrf failed");
    CU(cudaMemcpyAsync(h->d_sol, h->d_rhs, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
    OK(solve(h->d_sol, h->d_dense_info + 1));
  }
  CU(cudaMemcpyAsync(h->h_fail, h->d_dense_info, 2 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  summary->num_iterations = 1;   // schur_complement_solver.cc:154
  summary->residual_norm = 0.0;
  if (h->h_fail[0] != 0 || h->h_fail[1] != 0) {   // not positive definite: LinearSolverTerminationType::FAILURE (:203-210)
    summary->termination_type = B200_LS_FAILURE;
    return B200_OK;
  }
  summary->termination_type = B200_LS_SUCCESS;
  for (int k = 0; k < h->refine; ++k) {
    if (mixed) {
      OK(refine_residual_dev(h, nullptr, h->d_dense_v32));
      OK(solve(nullptr, h->d_dense_info + 2));
      OK(refine_accumulate_dev(h, nullptr, h->d_dense_v32, true));
    } else {
      OK(refine_residual_dev(h, nullptr, h->d_z));
      OK(solve(h->d_z, h->d_dense_info + 2));
      OK(refine_accumulate_dev(h, nullptr, static_cast<const double*>(h->d_z), true));
    }
  }
  OK(back_substitute_dev(h, d_b, h->d_sol, d_x));
  CU(cudaMemcpyAsync(d_x + 3 * static_cast<size_t>(h->P), h->d_sol, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
  return B200_OK;
}

// The symbolic analysis of SPARSE_SCHUR (sparse_plan.cuh), once per handle: the block pattern of S from the row structure
// (the same xs_pattern b200_create ran), the plan, and its upload.  A handle whose plan kept S implicit gets the arrays
// xs_assemble_dev reads here (not those of the explicit product).
constexpr double kFactorMaxBytes = 48.0 * (1ull << 30);   // the dense path's cap
static_assert(kSpMaxCols == 9 * kSnMaxCams && kSpThreads == 32 * 8 && kSpTileRows == 64,
              "an update tile: two column blocks per warp, two rows per lane");
int sparse_analyse(b200_handle* h) {
  XsPattern xp;
  xs_pattern(h->C, h->N, h->h_cam_idx.data(), h->h_pt_idx.data(), h->h_pt_ptr.data(), &xp);
  SparsePlan sp;
  plan_sparse_schur(h->C, xp.blk_row, xp.blk_col, h->ordering, &sp);
  // the cap counts the bytes of the precision in use (sparse_factor_solve); none fits when even a float factor does not
  if (4.0 * static_cast<double>(sp.storage) > kFactorMaxBytes)
    return fail(B200_ERR_UNSUPPORTED, "sparse factor of %d cameras needs %.1f GB", h->C, 4.0 * static_cast<double>(sp.storage) / 1e9);
  if (!h->xs_arrays) {
    XsView& x = h->xsv;
    x.C = h->C;
    x.num_blocks = static_cast<int>(xp.blk_row.size());
    OK(upload(h, xp.blk_row, &x.blk_row));
    OK(upload(h, xp.blk_col, &x.blk_col));
    OK(upload(h, xp.pair_ptr, &x.pair_ptr));
    OK(upload(h, xp.pairs, &x.pairs));
    OK(dev_alloc(h, &x.S, 81 * static_cast<size_t>(x.num_blocks)));
    std::vector<int> order;
    h->num_xs_long = xs_assembly_order(xp, &order);
    h->num_xs_short = x.num_blocks - h->num_xs_long;
    OK(upload(h, order, &h->d_xs_order));
    h->xs_arrays = true;
  }
  SparseView<double>& v = h->spv;
  v.C = h->C;
  v.ns = sp.ns;
  OK(upload(h, sp.pinv, &v.pinv));
  OK(upload(h, sp.sn_first, &v.sn_first));
  OK(upload(h, sp.row_ptr, &v.row_ptr));
  OK(upload(h, sp.rows, &v.rows));
  OK(upload(h, sp.val, &v.val));
  OK(upload(h, sp.upd_ptr, &v.upd_ptr));
  OK(upload(h, sp.upd, &v.upd));
  OK(upload(h, sp.ntf_ptr, &v.ntf_ptr));
  OK(upload(h, sp.ntf, &v.ntf));
  OK(upload(h, sp.order, &v.order));
  OK(upload(h, sp.blk_off, &v.blk_off));
  OK(upload(h, sp.blk_ld, &v.blk_ld));
  OK(upload(h, sp.cnt, &h->d_sp_cnt_init));
  OK(upload(h, sp.cnt_inv, &h->d_sp_cnt_inv));
  h->sp_selinv_flops = sp.selinv_flops;
  OK(dev_alloc(h, &v.v, 9 * static_cast<size_t>(h->C)));
  OK(dev_alloc(h, &v.cnt, sp.cnt.size()));
  OK(dev_alloc(h, &v.ticket, 2));
  v.fail = v.ticket + 1;
  // the float view shares the structure, the counters, the ticket and the failure flag; each factor is allocated by the
  // first solve in its precision
  SparseView<float>& v32 = h->spv32;
  std::memcpy(static_cast<void*>(&v32), static_cast<const void*>(&v), sizeof(v));
  v32.L = nullptr;
  OK(dev_alloc(h, &v32.v, 9 * static_cast<size_t>(h->C)));
  h->sp_storage = sp.storage;
  // every CTA of a cooperative launch must be resident: the grid of each precision fits both its factor and solve-only kernels
  auto grid = [&](auto factor, auto solve_only, size_t smem, int* out) -> int {
    int a = 0, b = 0;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, factor, kSpThreads, smem));
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b, solve_only, kSpThreads, smem));
    const int per_sm = std::min(a, b);
    if (per_sm < 1) return fail(B200_ERR_UNSUPPORTED, "no CTA of the sparse factorisation fits an SM (%zu bytes of shared memory)", smem);
    *out = std::max(1, std::min(per_sm * h->sm_count, 2 * sp.ns));
    return B200_OK;
  };
  h->sp_smem = sparse_smem_bytes<double>(sp.max_width);
  h->sp_smem32 = sparse_smem_bytes<float>(sp.max_width);
  OK(grid(sparse_factor_kernel<double, true>, sparse_factor_kernel<double, false>, h->sp_smem, &h->sp_grid));
  OK(grid(sparse_factor_kernel<float, true>, sparse_factor_kernel<float, false>, h->sp_smem32, &h->sp_grid32));
  {   // the selected inversion (b200_covariance_compute): its own cooperative grid, at most one CTA per supernode
    h->sp_selinv_smem = selinv_smem_bytes(sp.max_width);
    int a = 0;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, sparse_selinv_kernel, kSpThreads, h->sp_selinv_smem));
    h->sp_selinv_grid = a < 1 ? 0 : std::max(1, std::min(a * h->sm_count, sp.ns));   // 0: no CTA fits (refused at use)
  }
  CU(cudaStreamSynchronize(h->stream));   // the host vectors above go out of scope
  if (getenv("B200_VERBOSE") != nullptr) {
    const int64_t* st = sp.stats;
    fprintf(stderr,
            "[b200ba] sparse S plan: %lld blocks of S, L %lld blocks (caller's order %lld, minimum degree %lld), flops caller %.3g / "
            "minimum degree %.3g -> %s, %d supernodes (widest %d columns), tree height %lld, factor %.1f MB, %d CTAs, "
            "critical path %lld supernodes / %.3g flops of %.3g\n",
            static_cast<long long>(st[B200_SPARSE_STAT_S_BLOCKS]), static_cast<long long>(st[B200_SPARSE_STAT_L_BLOCKS]),
            static_cast<long long>(st[B200_SPARSE_STAT_L_BLOCKS_CALLER]), static_cast<long long>(st[B200_SPARSE_STAT_L_BLOCKS_MIN_DEGREE]),
            static_cast<double>(st[B200_SPARSE_STAT_FLOPS_CALLER]), static_cast<double>(st[B200_SPARSE_STAT_FLOPS_MIN_DEGREE]),
            st[B200_SPARSE_STAT_ORDER] == 2 ? "nested dissection" : st[B200_SPARSE_STAT_ORDER] ? "minimum degree" : "caller's order",
            sp.ns, sp.max_width, static_cast<long long>(st[B200_SPARSE_STAT_TREE_HEIGHT]), 8.0 * static_cast<double>(sp.storage) / 1e6,
            h->sp_grid, static_cast<long long>(st[B200_SPARSE_STAT_CRITICAL_PATH_SUPERNODES]),
            static_cast<double>(st[B200_SPARSE_STAT_CRITICAL_PATH_FLOPS]), static_cast<double>(st[B200_SPARSE_STAT_FLOPS]));
  }
  h->sp_ready = true;
  return B200_OK;
}

// Undoes sparse_analyse: the plan's arrays and both factors (the arrays xs_assemble_dev reads stay: they do not depend on
// the camera order).
void sparse_drop(b200_handle* h) {
  if (h->stream != nullptr) cudaStreamSynchronize(h->stream);
  SparseView<double>& v = h->spv;
  dev_free(h, v.pinv);
  dev_free(h, v.sn_first);
  dev_free(h, v.row_ptr);
  dev_free(h, v.rows);
  dev_free(h, v.val);
  dev_free(h, v.upd_ptr);
  dev_free(h, v.upd);
  dev_free(h, v.ntf_ptr);
  dev_free(h, v.ntf);
  dev_free(h, v.order);
  dev_free(h, v.blk_off);
  dev_free(h, v.blk_ld);
  dev_free(h, v.L);
  dev_free(h, v.v);
  dev_free(h, v.cnt);
  dev_free(h, v.ticket);
  dev_free(h, h->spv32.L);
  dev_free(h, h->spv32.v);
  dev_free(h, h->d_sp_cnt_init);
  dev_free(h, h->d_sp_cnt_inv);
  dev_free(h, h->d_cov_z);   // Z's scratch has the factor's layout (the snapshot does not)
  h->spv = SparseView<double>{};
  h->spv32 = SparseView<float>{};
  h->sp_storage = 0;
  h->sp_ready = false;
}

// One cooperative launch of sparse_factor_kernel<T, kFactor> on v (counters and ticket set by the caller).
template <typename T, bool kFactor>
int sparse_factor_launch(b200_handle* h, SparseView<T>& v, int grid, size_t smem) {
  cudaError_t le = cudaSuccess;
  OK(launch(h, kFactor ? K_SPARSE_FACTOR : K_SPARSE_SOLVE, [&] {
    void* args[] = {&v};
    le = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(sparse_factor_kernel<T, kFactor>), dim3(grid), dim3(kSpThreads),
                                     args, smem, h->stream);
  }));
  CU(le);
  return B200_OK;
}

// S + D_f^2 scattered into v's factor storage (allocated here on first use) and factored in T, with the triangular solves of
// the current rhs in the same launch; false in *ok when a pivot is not positive.  Shared by the solves and the covariance.
template <typename T>
int sparse_factor(b200_handle* h, SparseView<T>& v, int grid, size_t smem, const double* Df, bool* ok) {
  if (v.L == nullptr) OK(dev_alloc(h, &v.L, static_cast<size_t>(h->sp_storage)));
  CU(cudaMemsetAsync(v.L, 0, sizeof(T) * static_cast<size_t>(h->sp_storage), h->stream));
  CU(cudaMemcpyAsync(v.cnt, h->d_sp_cnt_init, sizeof(int) * 2 * static_cast<size_t>(v.ns), cudaMemcpyDeviceToDevice, h->stream));
  CU(cudaMemsetAsync(v.ticket, 0, 2 * sizeof(int), h->stream));
  OK(launch(h, K_SPARSE_SCATTER, [&] {
    const int g = std::max(1, std::min((h->xsv.num_blocks + 7) / 8, h->sm_count * 8));
    sparse_scatter_kernel<T><<<g, 256, 0, h->stream>>>(v, h->xsv, Df, h->d_rhs);
  }));
  OK((sparse_factor_launch<T, true>(h, v, grid, smem)));
  CU(cudaMemcpyAsync(h->h_fail, v.fail, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  *ok = h->h_fail[0] == 0;
  return B200_OK;
}

// The factorisation of S + D_f^2 in T, its solve and the refinement's (1 + h->refine solves), into h->d_sol; false in *ok
// when a pivot is not positive (the caller's x is then not written).
template <typename T>
int sparse_factor_solve(b200_handle* h, SparseView<T>& v, int grid, size_t smem, const double* Df, bool* ok) {
  if (static_cast<double>(sizeof(T)) * static_cast<double>(h->sp_storage) > kFactorMaxBytes)
    return fail(B200_ERR_UNSUPPORTED, "sparse factor of %d cameras needs %.1f GB", h->C,
                static_cast<double>(sizeof(T)) * static_cast<double>(h->sp_storage) / 1e9);
  OK(sparse_factor(h, v, grid, smem, Df, ok));
  if (!*ok) return B200_OK;
  OK(launch(h, K_SPARSE_SCATTER, [&] {
    sparse_gather_kernel<T><<<(9 * h->C + 255) / 256, 256, 0, h->stream>>>(v, h->d_sol);
  }, false));
  for (int k = 0; k < h->refine; ++k) {
    OK(refine_residual_dev(h, v.pinv, v.v));
    CU(cudaMemcpyAsync(v.cnt, h->d_sp_cnt_init, sizeof(int) * 2 * static_cast<size_t>(v.ns), cudaMemcpyDeviceToDevice, h->stream));
    CU(cudaMemsetAsync(v.ticket, 0, sizeof(int), h->stream));
    OK((sparse_factor_launch<T, false>(h, v, grid, smem)));
    OK(refine_accumulate_dev(h, v.pinv, static_cast<const T*>(v.v), true));
  }
  return B200_OK;
}

// SparseSchurComplementSolver (schur_complement_solver.cc:205-335) on device pointers: S by xs_assemble_kernel, scattered with
// D_f^2 into the supernodal factor, factored and solved by sparse_factor_kernel, back substitution by the implicit-Schur
// kernels.  With mixed precision the factor and its solves are float (FloatSuiteSparseCholesky, suitesparse.cc:487-565); with
// refinement, RefinedSparseCholesky::Solve (sparse_cholesky.cc:160-170) on the camera block.
int sparse_schur_solve_dev(b200_handle* h, const double* d_b, const double* d_D, double* d_x, b200_solver_summary* summary) {
  if (h->world > 1) return fail(B200_ERR_UNSUPPORTED, "the explicit Schur complement is single-GPU");
  if (!h->sp_ready) OK(sparse_analyse(h));
  OK(schur_init_dev(h, d_b, d_D));   // (E'E + D^2)^-1 and the reduced right-hand side
  if (!h->xs_ready) OK(xs_assemble_dev(h));
  const double* Df = h->cur_D != nullptr ? h->cur_D + 3 * static_cast<size_t>(h->P) : nullptr;
  bool ok = false;
  if (h->mixed) OK(sparse_factor_solve(h, h->spv32, h->sp_grid32, h->sp_smem32, Df, &ok));
  else OK(sparse_factor_solve(h, h->spv, h->sp_grid, h->sp_smem, Df, &ok));
  summary->num_iterations = 1;   // schur_complement_solver.cc:154
  summary->residual_norm = 0.0;
  if (!ok) {   // not positive definite: CHOLMOD_NOT_POSDEF, suitesparse.cc:311-313 -> FAILURE
    summary->termination_type = B200_LS_FAILURE;
    return B200_OK;
  }
  summary->termination_type = B200_LS_SUCCESS;
  OK(back_substitute_dev(h, d_b, h->d_sol, d_x));
  CU(cudaMemcpyAsync(d_x + 3 * static_cast<size_t>(h->P), h->d_sol, sizeof(double) * 9 * h->C, cudaMemcpyDeviceToDevice, h->stream));
  return B200_OK;
}

int reduce_partials(b200_handle* h, int blocks, int slots, unsigned op_mask, double* host_out, bool across_ranks) {
  OK(launch(h, K_LM_VEC, [&] { reduce_final_kernel<<<1, 32, 0, h->stream>>>(blocks, slots, op_mask, h->d_partial, h->d_scalars + 8); }));
#ifdef B200_WITH_NCCL
  if (across_ranks && h->world > 1) {
    for (int i = 0; i < slots; ++i) {
      const ncclRedOp_t op = ((op_mask >> i) & 1u) ? ncclMax : ncclSum;
      ncclResult_t r = g_nccl.AllReduce(h->d_scalars + 8 + i, h->d_scalars + 8 + i, 1, ncclDouble, op, h->comm, h->stream);
      if (r != ncclSuccess) return fail(B200_ERR_NCCL, "ncclAllReduce: %s", g_nccl.GetErrorString(r));
    }
  }
#else
  (void)across_ranks;
#endif
  CU(cudaMemcpyAsync(h->h_scalars + 8, h->d_scalars + 8, sizeof(double) * slots, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  for (int i = 0; i < slots; ++i) host_out[i] = h->h_scalars[8 + i];
  return B200_OK;
}

// ConjugateGradientsSolver (conjugate_gradients_solver.h:109-306) with an arbitrary preconditioner and initial guess, for
// the configurations the fused PCG does not cover: SCHUR_POWER_SERIES_EXPANSION and use_spse_initialization
// (iterative_schur_complement_solver.cc:100-111, :178-186).  Vectors on the device, scalars on the host.
// Result in h->h_cg[0] {iteration, termination, norm_r}; the solution in h->d_sol.
int pcg_general_dev(b200_handle* h, const b200_solver_options* o) {
  const int n = 9 * h->C;
  const int g = std::min(kRedBlocks, flat_grid(h, n, 256));
  const int type = o->preconditioner_type;
  if (type < B200_PRECOND_IDENTITY || type > B200_PRECOND_SCHUR_POWER_SERIES_EXPANSION)
    return fail(B200_ERR_INVALID_ARGUMENT, "unknown preconditioner type %d", type);
  const bool need_ftf = type == B200_PRECOND_SCHUR_POWER_SERIES_EXPANSION || o->use_spse_initialization != 0;
  if (h->d_ftf_inv == nullptr) {
    OK(dev_alloc(h, &h->d_ftf_inv, 81 * static_cast<size_t>(h->C)));
    for (auto& b : h->d_spse) OK(dev_alloc(h, &b, static_cast<size_t>(n)));
  }
  if (need_ftf) {  // block_diagonal_FtF_inverse (implicit_schur_complement.cc:61-64, :90-95)
    OK(precond_update_dev(h, B200_PRECOND_JACOBI));
    CU(cudaMemcpyAsync(h->d_ftf_inv, h->d_minv, sizeof(double) * 81 * h->C, cudaMemcpyDeviceToDevice, h->stream));
  }
  if (type == B200_PRECOND_JACOBI || type == B200_PRECOND_SCHUR_JACOBI) OK(precond_update_dev(h, type));

  double *x = h->d_sol, *r = h->d_r, *z = h->d_z, *p = h->d_p, *tmp = h->d_tmp;
  const double* rhs = h->d_rhs;
  auto dots = [&](const double* a, const double* b, const double* c, const double* d, double* out2) -> int {
    OK(launch(h, K_CG_VEC, [&] { dot2_kernel<<<g, 256, 0, h->stream>>>(n, a, b, c, d, h->d_partial); }));
    return reduce_partials(h, g, 2, 0u, out2, false);
  };
  // y = power series approximation of S^-1 x   (power_series_expansion_preconditioner.cc:57-82)
  auto spse = [&](const double* xin, double* y, int max_terms, double tol) -> int {
    double *prev = h->d_spse[0], *term = h->d_spse[1], *t = h->d_spse[2];
    OK(launch(h, K_CG_VEC, [&] { block_apply_kernel<<<g, 256, 0, h->stream>>>(n, h->d_ftf_inv, xin, y); }));
    CU(cudaMemcpyAsync(prev, y, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
    double thr = 0.0;
    if (tol > 0.0) {
      double d2[2];
      OK(dots(y, y, nullptr, nullptr, d2));
      thr = tol * std::sqrt(d2[0]);
    }
    for (int i = 1;; ++i) {
      OK(schur_mul_dev(h, prev, t, MulOpts{}));   // (F'F + D^2) prev - F'E P E'F prev
      OK(launch(h, K_CG_VEC, [&] { spse_term_kernel<<<g, 256, 0, h->stream>>>(n, h->d_ftf_inv, prev, t, term, y, h->d_partial); }));
      if (i >= max_terms) break;
      if (tol > 0.0) {
        double sq[1];
        OK(reduce_partials(h, g, 1, 0u, sq, false));
        if (std::sqrt(sq[0]) < thr) break;
      }
      std::swap(prev, term);
    }
    return B200_OK;
  };
  auto precondition = [&](const double* rin, double* zout) -> int {
    switch (type) {
      case B200_PRECOND_IDENTITY:
        CU(cudaMemcpyAsync(zout, rin, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
        return B200_OK;
      case B200_PRECOND_JACOBI:
      case B200_PRECOND_SCHUR_JACOBI:
        return launch(h, K_CG_VEC, [&] { block_apply_kernel<<<g, 256, 0, h->stream>>>(n, h->d_minv, rin, zout); });
      default:  // tolerance 0 keeps the preconditioner fixed during the iterations (iterative_schur_complement_solver.cc:179-185)
        return spse(rin, zout, std::max(o->max_num_spse_iterations, 1), 0.0);
    }
  };
  CgState* st = h->h_cg;
  std::memset(st, 0, sizeof(CgState));
  st->done = 1;
  st->termination = B200_LS_NO_CONVERGENCE;
  st->iteration = 0;
  auto is_zero_or_inf = [](double v) { return v == 0.0 || std::isinf(v); };

  // initial guess
  CU(cudaMemsetAsync(x, 0, sizeof(double) * n, h->stream));
  if (o->use_spse_initialization != 0) OK(spse(rhs, x, std::max(o->max_num_spse_iterations, 1), o->spse_tolerance));

  double d2[2];
  OK(dots(rhs, rhs, nullptr, nullptr, d2));
  const double norm_rhs = std::sqrt(d2[0]);
  if (norm_rhs == 0.0) {
    CU(cudaMemsetAsync(x, 0, sizeof(double) * n, h->stream));
    st->termination = B200_LS_SUCCESS;
    return B200_OK;
  }
  const double tol_r = o->r_tolerance * norm_rhs;
  // r = rhs - S x ; Q0 = -x.(rhs + r)
  OK(schur_mul_dev(h, x, tmp, MulOpts{}));
  OK(launch(h, K_CG_VEC, [&] { cgg_update_kernel<<<g, 256, 0, h->stream>>>(n, 1, 0.0, nullptr, tmp, rhs, x, r, h->d_partial); }));
  OK(reduce_partials(h, g, 2, 0u, d2, false));
  double norm_r = std::sqrt(d2[1]);
  st->norm_r = norm_r;
  if (o->min_num_iterations == 0 && norm_r <= tol_r) {
    st->termination = B200_LS_SUCCESS;
    return B200_OK;
  }
  double rho = 1.0, Q0 = -d2[0];
  const int reset = o->residual_reset_period > 0 ? o->residual_reset_period : std::numeric_limits<int>::max();
  const int max_it = std::max(o->max_num_iterations, 1);
  for (int it = 1;; ++it) {
    st->iteration = it;
    OK(precondition(r, z));
    const double last_rho = rho;
    OK(dots(r, z, nullptr, nullptr, d2));
    rho = d2[0];
    if (is_zero_or_inf(rho) || std::isnan(rho)) {
      st->termination = B200_LS_FAILURE;
      break;
    }
    if (it == 1) {
      CU(cudaMemcpyAsync(p, z, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
    } else {
      const double beta = rho / last_rho;
      if (is_zero_or_inf(beta)) {
        st->termination = B200_LS_FAILURE;
        break;
      }
      OK(launch(h, K_CG_VEC, [&] { axpby_kernel<<<g, 256, 0, h->stream>>>(n, 1.0, z, beta, p, p); }));
    }
    double* q = z;  // conjugate_gradients_solver.h:193
    OK(schur_mul_dev(h, p, q, MulOpts{}));
    OK(dots(p, q, nullptr, nullptr, d2));
    const double pq = d2[0];
    if (!(pq > 0.0) || std::isinf(pq)) {
      st->termination = std::isnan(pq) ? B200_LS_FAILURE : B200_LS_NO_CONVERGENCE;
      break;
    }
    const double alpha = rho / pq;
    if (std::isinf(alpha)) {
      st->termination = B200_LS_FAILURE;
      break;
    }
    if (it % reset == 0) {
      OK(launch(h, K_CG_VEC, [&] { axpby_kernel<<<g, 256, 0, h->stream>>>(n, 1.0, x, alpha, p, x); }));
      OK(schur_mul_dev(h, x, tmp, MulOpts{}));
      OK(launch(h, K_CG_VEC, [&] { cgg_update_kernel<<<g, 256, 0, h->stream>>>(n, 1, 0.0, nullptr, tmp, rhs, x, r, h->d_partial); }));
    } else {
      OK(launch(h, K_CG_VEC, [&] { cgg_update_kernel<<<g, 256, 0, h->stream>>>(n, 0, alpha, p, q, rhs, x, r, h->d_partial); }));
    }
    OK(reduce_partials(h, g, 2, 0u, d2, false));
    const double Q1 = -d2[0];
    const double zeta = it * (Q1 - Q0) / Q1;
    norm_r = std::sqrt(d2[1]);
    st->norm_r = norm_r;
    if (zeta < o->q_tolerance && it >= o->min_num_iterations) {
      st->termination = B200_LS_SUCCESS;
      break;
    }
    Q0 = Q1;
    if (norm_r <= tol_r && it >= o->min_num_iterations) {
      st->termination = B200_LS_SUCCESS;
      break;
    }
    if (it >= max_it) break;
  }
  return B200_OK;
}

// Host scalars of the host-boundary LM loop on a sharded problem: vals[i] is combined across ranks (sum, or max where bit i
// of max_mask is set) through a few device words and NCCL; a no-op on one GPU.
int host_allreduce(b200_handle* h, double* vals, int n, unsigned max_mask) {
#ifdef B200_WITH_NCCL
  if (h->world <= 1) return B200_OK;
  CU(cudaMemcpyAsync(h->d_scalars + 16, vals, sizeof(double) * n, cudaMemcpyHostToDevice, h->stream));
  for (int i = 0; i < n; ++i) {
    const ncclRedOp_t op = ((max_mask >> i) & 1u) ? ncclMax : ncclSum;
    ncclResult_t r = g_nccl.AllReduce(h->d_scalars + 16 + i, h->d_scalars + 16 + i, 1, ncclDouble, op, h->comm, h->stream);
    if (r != ncclSuccess) return fail(B200_ERR_NCCL, "ncclAllReduce: %s", g_nccl.GetErrorString(r));
  }
  CU(cudaMemcpyAsync(h->h_scalars + 16, h->d_scalars + 16, sizeof(double) * n, cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  for (int i = 0; i < n; ++i) vals[i] = h->h_scalars[16 + i];
#else
  (void)h; (void)vals; (void)n; (void)max_mask;
#endif
  return B200_OK;
}

// Reduction over a [points | cameras] vector when the points are sharded across ranks and the cameras are
// replicated: the point range is reduced locally and combined across ranks, the camera range is counted once.
// run(offset, count) must launch the partial-producing kernel on that sub-range with `grid` blocks.
template <typename L>
int sharded_reduce(b200_handle* h, int grid, int slots, unsigned op_mask, double* out, L&& run) {
  const int nP = 3 * h->P, nC = 9 * h->C;
  if (h->world == 1) {
    OK(run(0, nP + nC));
    return reduce_partials(h, grid, slots, op_mask, out, false);
  }
  double pt[8], cam[8];
  OK(run(0, nP));
  OK(reduce_partials(h, grid, slots, op_mask, pt, true));
  OK(run(nP, nC));
  OK(reduce_partials(h, grid, slots, op_mask, cam, false));
  for (int i = 0; i < slots; ++i) out[i] = ((op_mask >> i) & 1u) ? std::max(pt[i], cam[i]) : pt[i] + cam[i];
  return B200_OK;
}

// The linear solver linear_solver_type selects, on device pointers (opts: ITERATIVE_SCHUR's options).
int solve_dev(b200_handle* h, int type, const double* d_b, const double* d_D, const b200_solver_options* opts, double* d_x,
              b200_solver_summary* summary) {
  if (type == B200_DENSE_SCHUR) return dense_schur_solve_dev(h, d_b, d_D, d_x, summary);
  if (type == B200_SPARSE_SCHUR) return sparse_schur_solve_dev(h, d_b, d_D, d_x, summary);
  return schur_solve_dev(h, d_b, d_D, opts, d_x, summary);
}

// Body of the public Schur solves: b (NULL: the resident residuals) and D up, the solve, x down unless it failed.
int solve_from_host(b200_handle* h, int type, const double* b, const double* D, const b200_solver_options* opts, double* x,
                    b200_solver_summary* summary) {
  if (b == nullptr && !h->residuals_resident)
    return fail(B200_ERR_INVALID_ARGUMENT, "b == NULL means the residuals of the last b200_evaluate, and there are none");
  CU(cudaSetDevice(h->device));
  if (b != nullptr) OK(up_rows(h, h->d_b, b));
  if (D != nullptr) OK(up_params(h, h->d_D, D));
  OK(solve_dev(h, type, b != nullptr ? h->d_b : h->d_residuals, D != nullptr ? h->d_D : nullptr, opts, h->d_y, summary));
  if (summary->termination_type != B200_LS_FAILURE && summary->termination_type != B200_LS_FATAL_ERROR)
    OK(down_params(h, x, h->d_y));
  return B200_OK;
}

// Change of the linearised model's cost by d_step, against the resident residuals (trust_region_minimizer.cc:430-438).
int model_cost_change_dev(b200_handle* h, const double* d_step, double* model_cost_change) {
  OK(launch(h, K_MODEL_COST, [&] {
    model_cost_kernel<<<h->grid_tile[K_MODEL_COST], kTile, tile_smem_bytes<1, 1>(), h->stream>>>(h->view, d_step, h->d_residuals, h->d_tile_partial);
  }));
  OK(launch(h, K_MISC, [&] { sum_kernel<<<1, kVecThreads, 0, h->stream>>>(h->num_tiles, h->d_tile_partial, h->d_scalars + 1); }));
  OK(allreduce_sum(h, h->d_scalars + 1, 1));
  CU(cudaMemcpyAsync(h->h_scalars + 1, h->d_scalars + 1, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  *model_cost_change = h->h_scalars[1];
  return B200_OK;
}

// Row structure checks, the SchurEliminator precondition (rows grouped by e block), and the first row of every point
// (P + 1 entries).
int validate_rows(const b200_ba_desc* desc, std::vector<int>* ptr) {
  const int C = desc->num_cameras, P = desc->num_points;
  const int N = static_cast<int>(desc->num_observations);
  ptr->assign(static_cast<size_t>(P) + 1, 0);
  for (int i = 0; i < N; ++i) {
    const int pt = desc->pt_idx[i], cam = desc->cam_idx[i];
    if (pt < 0 || pt >= P || cam < 0 || cam >= C) return fail(B200_ERR_INVALID_ARGUMENT, "row %d: block id out of range", i);
    if (i > 0 && pt < desc->pt_idx[i - 1])
      return fail(B200_ERR_INVALID_ARGUMENT, "rows are not grouped by e block at row %d (reorder_program.cc:278-359)", i);
    (*ptr)[pt + 1]++;
  }
  for (int k = 0; k < P; ++k) (*ptr)[k + 1] += (*ptr)[k];
  return B200_OK;
}

template <typename K>
int raise_smem_limit(K kernel, int bytes) {
  CU(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return B200_OK;
}
// Dynamic shared memory limits of every kernel that may take more than 48 KB.  Function attributes are process-wide:
// they are raised to the device limit, never to one handle's need.
int set_func_attributes(int smem_optin) {
  const int lim = smem_optin - 1024;
  OK(raise_smem_limit(cam_blocks_v2_kernel<true>, (kCamBlkThreads / 32) * kCamBlkWarpBytes));
  OK(raise_smem_limit(cam_blocks_v2_kernel<false>, (kCamBlkThreads / 32) * kCamBlkWarpBytes));
  OK(raise_smem_limit(jtj_v2_kernel, lim));
  OK(raise_smem_limit(schur_mul_v3_kernel, lim));
  OK(raise_smem_limit(schur_init_v4_kernel<true>, lim));
  OK(raise_smem_limit(schur_init_v4_kernel<false>, lim));
  OK(raise_smem_limit(jtj_v4_kernel<true>, lim));
  OK(raise_smem_limit(jtj_v4_kernel<false>, lim));
  OK(raise_smem_limit(schur_mul_v4_kernel<true>, lim));
  OK(raise_smem_limit(schur_mul_v4_kernel<false>, lim));
  OK(raise_smem_limit(evaluate_v2_kernel<kLossTrivial, true>, lim));
  OK(raise_smem_limit(evaluate_v2_kernel<kLossTrivial, false>, lim));
  OK(raise_smem_limit(evaluate_v2_kernel<kLossHuber, true>, lim));
  OK(raise_smem_limit(evaluate_v2_kernel<kLossHuber, false>, lim));
  OK(raise_smem_limit(evaluate_v2_kernel<kLossGeneral, true>, lim));
  OK(raise_smem_limit(evaluate_v2_kernel<kLossGeneral, false>, lim));
  OK(raise_smem_limit(evaluate_v2_kernel<kLossTrivial, true, true>, lim));
  OK(raise_smem_limit(evaluate_v2_kernel<kLossTrivial, false, true>, lim));
  OK(raise_smem_limit(evaluate_v2_kernel<kLossHuber, true, true>, lim));
  OK(raise_smem_limit(evaluate_v2_kernel<kLossHuber, false, true>, lim));
  OK(raise_smem_limit(evaluate_v2_kernel<kLossGeneral, true, true>, lim));
  OK(raise_smem_limit(evaluate_v2_kernel<kLossGeneral, false, true>, lim));
  OK(raise_smem_limit(diag_blocks_v2_kernel<true>, lim));
  OK(raise_smem_limit(diag_blocks_v2_kernel<false>, lim));
  OK(raise_smem_limit(xs_pcg_kernel, lim));
  OK(raise_smem_limit(sparse_factor_kernel<double, true>, lim));
  OK(raise_smem_limit(sparse_factor_kernel<double, false>, lim));
  OK(raise_smem_limit(sparse_factor_kernel<float, true>, lim));
  OK(raise_smem_limit(sparse_factor_kernel<float, false>, lim));
  OK(raise_smem_limit(sparse_selinv_kernel, lim));
  return B200_OK;
}

// ------------------------------------------------------------------------------------------------ trust region loop
// What a strategy's step gives the loop: the linear solver's summary, the model cost change (0 when no step was formed,
// NaN for a non-finite DOGLEG step: either makes the step invalid), |x - candidate|^2, |x|^2 and whether the step is finite.
struct StepResult {
  b200_solver_summary ls{};
  double model_cost_change = 0.0;
  double step_sq = 0.0, x_sq = 0.0;
  bool finite = true;
};

// The vectors in HBM, every pass a kernel of this library.  d_state is x, d_cand the candidate, d_vp1 the best state.
struct DeviceSide {
  b200_handle* h;
  const b200_lm_options* opt;
  int np, vgrid;
  bool have_scaling = false;
  bool sqnorm_fresh = false;    // d_sqnorm holds the squared column norms of the current device Jacobian

  DeviceSide(b200_handle* h_, const b200_lm_options* o) : h(h_), opt(o), np(h_->np), vgrid(std::min(kRedBlocks, flat_grid(h_, np, 256))) {}
  int begin(const double* state) {
    OK(up_params(h, h->d_state, state));
    OK(launch(h, K_LM_VEC, [&] { fill_kernel<<<flat_grid(h, np, 256), 256, 0, h->stream>>>(np, h->d_scale, 1.0); }));
    return keep_best();
  }
  int keep_best() {
    CU(cudaMemcpyAsync(h->d_vp1, h->d_state, sizeof(double) * np, cudaMemcpyDeviceToDevice, h->stream));
    return B200_OK;
  }
  int finish(double* state) { return down_params(h, state, h->d_vp1); }
  int accept() {
    std::swap(h->d_state, h->d_cand);
    return B200_OK;
  }
  int candidate_cost(double* cost) { return evaluate_dev(h, h->d_cand, nullptr, nullptr, false, nullptr, cost); }
  // Cost, Jacobian and gradient norms at x.  The scaling is formed on the first call and fused into the Jacobian write after.
  int evaluate(b200_lm_iteration* it) {
    OK(evaluate_dev(h, h->d_state, h->d_residuals, h->d_gradient, true, opt->jacobi_scaling && have_scaling ? h->d_scale : nullptr,
                    &it->cost, h->d_sqnorm, &sqnorm_fresh));
    if (opt->jacobi_scaling && !have_scaling) {
      if (!sqnorm_fresh) OK(sqnorm_dev(h, h->d_sqnorm));
      // scale = 1/(1+sqrt(colnorm^2)); J <- J diag(scale); and colnorm^2 of the scaled J is colnorm^2 * scale^2
      OK(launch(h, K_LM_VEC, [&] { jacobi_scale_kernel<<<flat_grid(h, np, 256), 256, 0, h->stream>>>(np, h->d_sqnorm, h->d_scale); }));
      OK(scale_dev(h, h->d_scale));
      OK(launch(h, K_LM_VEC, [&] { rescale_sq_kernel<<<flat_grid(h, np, 256), 256, 0, h->stream>>>(np, h->d_scale, h->d_sqnorm); }));
      sqnorm_fresh = true;
      have_scaling = true;
    }
    double gn[2];
    OK(sharded_reduce(h, vgrid, 2, 0x1u, gn, [&](int ofs, int cnt) {
      return launch(h, K_LM_VEC, [&] { grad_norm_kernel<<<vgrid, 256, 0, h->stream>>>(cnt, h->d_gradient + ofs, h->d_partial); });
    }));
    it->gradient_max_norm = gn[0];
    it->gradient_norm = std::sqrt(gn[1]);
    return B200_OK;
  }
  int model_cost_change(double* mcc) { return model_cost_change_dev(h, h->d_step, mcc); }

  // LM: the diagonal (refreshed from the column norms unless reused), D = sqrt(diagonal / radius) and the solve
  int lm_solve(bool reuse_diagonal, double radius, const b200_solver_options* so, b200_solver_summary* ls) {
    if (!reuse_diagonal && !sqnorm_fresh) OK(sqnorm_dev(h, h->d_sqnorm));
    OK(launch(h, K_LM_VEC, [&] {
      lm_diagonal_kernel<<<flat_grid(h, np, 256), 256, 0, h->stream>>>(np, reuse_diagonal ? 0 : 1, h->d_sqnorm, h->d_diagonal, h->d_lmD,
                                                                        opt->min_lm_diagonal, opt->max_lm_diagonal, radius);
    }));
    return solve_dev(h, opt->linear_solver_type, h->d_residuals, h->d_lmD, so, h->d_y, ls);
  }
  // step = -y, candidate = x + step * scaling and the norms, in one pass
  int lm_step(StepResult* r) {
    double red[3];
    OK(sharded_reduce(h, vgrid, 3, 0u, red, [&](int ofs, int cnt) {
      return launch(h, K_LM_VEC, [&] {
        lm_step_kernel<<<vgrid, 256, 0, h->stream>>>(cnt, h->d_y + ofs, h->d_scale + ofs, h->d_state + ofs,
                                                     h->fixed_any ? h->d_fixed + ofs : nullptr, h->d_step + ofs,
                                                     h->d_cand + ofs, h->d_partial);
      });
    }));
    r->step_sq = red[0];
    r->x_sq = red[1];
    r->finite = red[2] == 0.0;
    return B200_OK;
  }

  // DOGLEG, a new Gauss-Newton step: the column norms that D and g come from (dogleg_diagonal_kernel forms both with the
  // first solve)
  int dl_gradient(int dogleg_type) {
    if (h->d_dl_g == nullptr) {
      OK(dev_alloc(h, &h->d_dl_g, np));
      OK(dev_alloc(h, &h->d_dl_gn, np));
      OK(dev_alloc(h, &h->d_dl_part, 3 * static_cast<size_t>(h->num_tiles)));
    }
    // the subspace model's pass also reads gn
    h->bytes_per_op[K_DOGLEG_GRAM] = 196.0 * h->N + 4.0 * h->P + (dogleg_type == B200_SUBSPACE_DOGLEG ? 24.0 : 16.0) * np;
    if (!sqnorm_fresh) OK(sqnorm_dev(h, h->d_sqnorm));
    sqnorm_fresh = true;
    return B200_OK;
  }
  // D at one mu, the solve, and unless it failed gn = -diagonal * y with |g|^2, g.gn, |gn|^2; a non-finite y is reported as
  // FAILURE, as ComputeGaussNewtonStep (:517-616) treats it
  int dl_gauss_newton(bool refresh, double sqrt_mu, b200_solver_summary* ls, b200dl::Model* m) {
    // (a refresh launch is the operation; the later ones of the mu loop only rescale D: auxiliary)
    OK(launch(h, K_DOGLEG_DIAG, [&] {
      dogleg_diagonal_kernel<<<flat_grid(h, np, 256), 256, 0, h->stream>>>(np, refresh ? 1 : 0, h->d_sqnorm, h->d_gradient, h->d_scale,
                                                                            h->d_diagonal, h->d_dl_g, h->d_lmD, opt->min_lm_diagonal,
                                                                            opt->max_lm_diagonal, sqrt_mu);
    }, refresh));
    OK(solve_dev(h, opt->linear_solver_type, h->d_residuals, h->d_lmD, nullptr, h->d_y, ls));
    if (ls->termination_type == B200_LS_FAILURE || ls->termination_type == B200_LS_FATAL_ERROR) return B200_OK;
    OK(launch(h, K_DOGLEG_GN, [&] {
      dogleg_gn_kernel<<<vgrid, 256, 0, h->stream>>>(np, h->d_y, h->d_diagonal, h->d_dl_g, h->d_dl_gn, h->d_partial);
    }));
    double red[4];
    OK(reduce_partials(h, vgrid, 4, 0u, red, false));
    m->gg = red[0];
    m->ggn = red[1];
    m->gngn = red[2];
    if (red[3] != 0.0) ls->termination_type = B200_LS_FAILURE;
    return B200_OK;
  }
  // |J a|^2 (Cauchy point) and, for the subspace model, |J b|^2 and (J a).(J b): one pass over J
  int dl_gram(bool two, b200dl::Model* m) {
    OK(launch(h, K_DOGLEG_GRAM, [&] {
      dogleg_gram_kernel<<<h->grid_tile[K_DOGLEG_GRAM], kTile, tile_smem_bytes<1, 1>(), h->stream>>>(
          h->view, h->d_dl_g, two ? h->d_dl_gn : nullptr, h->d_diagonal, h->d_dl_part);
    }));
    const int nt = h->num_tiles;
    for (int k = 0; k < (two ? 3 : 1); ++k)
      OK(launch(h, K_MISC, [&] { sum_kernel<<<1, kVecThreads, 0, h->stream>>>(nt, h->d_dl_part + static_cast<size_t>(k) * nt, h->d_scalars + 16 + k); }));
    CU(cudaMemcpyAsync(h->h_scalars + 16, h->d_scalars + 16, sizeof(double) * 3, cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    m->jaja = h->h_scalars[16];
    if (two) {
      m->jbjb = h->h_scalars[17];
      m->jajb = h->h_scalars[18];
    }
    return B200_OK;
  }
  // step = (cg g + cn gn) / diagonal, candidate = x + step * scaling, the norms and |cg g + cn gn|^2, in one pass
  int dl_step(const b200dl::Step& st, StepResult* r, double* vv) {
    OK(launch(h, K_DOGLEG_STEP, [&] {
      dogleg_step_kernel<<<vgrid, 256, 0, h->stream>>>(np, st.kind, st.cg, st.cn, h->d_dl_g, h->d_dl_gn, h->d_diagonal,
                                                       h->d_scale, h->d_state, h->fixed_any ? h->d_fixed : nullptr,
                                                       h->d_step, h->d_cand, h->d_partial);
    }));
    double red[4];
    OK(reduce_partials(h, vgrid, 4, 0u, red, false));
    r->step_sq = red[0];
    r->x_sq = red[1];
    r->finite = red[2] == 0.0;
    *vv = red[3];
    return B200_OK;
  }
};

// Sum (or max, where bit k of max_mask is set) of what term(i, acc) adds into acc[k] over the parameter vector: this rank's
// points in one OpenMP pass, combined across ranks, then the replicated cameras, counted once.  On one GPU, one pass.
template <int K, typename F>
int host_reduce(b200_handle* h, unsigned max_mask, double (&out)[K], F&& term) {
  const int np = h->np, np_local = h->world > 1 ? 3 * h->P : np;
  auto pass = [&](int lo, int hi) {
#pragma omp parallel num_threads(kHostThreads)
    {
      double acc[K];
      for (int k = 0; k < K; ++k) acc[k] = ((max_mask >> k) & 1u) ? -std::numeric_limits<double>::infinity() : 0.0;
#pragma omp for schedule(static) nowait
      for (int i = lo; i < hi; ++i) term(i, acc);
#pragma omp critical
      for (int k = 0; k < K; ++k) out[k] = ((max_mask >> k) & 1u) ? std::max(out[k], acc[k]) : out[k] + acc[k];
    }
  };
  for (double& v : out) v = 0.0;
  pass(0, np_local);
  if (np_local == np) return B200_OK;
  OK(host_allreduce(h, out, K, max_mask));
  pass(np_local, np);
  return B200_OK;
}

// The vectors in the handle's pinned host mirrors, driven through the public entry points as an adapter drives them; the
// host-side passes mirror what the reference minimizer does on its Eigen vectors, adjacent ones fused so that each array
// is streamed once.  This side launches no kernel of its own and holds no device pointer.
struct HostSide {
  b200_handle* h;
  const b200_lm_options* opt;
  int np;
  size_t nr;
  HostMirrors& v;
  bool have_scaling = false;

  HostSide(b200_handle* h_, const b200_lm_options* o) : h(h_), opt(o), np(h_->np), nr(2 * static_cast<size_t>(h_->N)), v(h_->hm) {}
  int begin(const double* state) {
    v.x.assign(state, state + np);
    for (PinnedVec* p : {&v.cand, &v.gradient, &v.step, &v.diagonal, &v.lmD, &v.sol}) p->resize(np);
    v.residuals.resize(nr);
    v.scaling.assign(np, 1.0);
    return keep_best();
  }
  int keep_best() {
    v.best = v.x;
    return B200_OK;
  }
  int finish(double* state) {
    std::memcpy(state, v.best.data(), sizeof(double) * np);
    return B200_OK;
  }
  int accept() {
    v.x = v.cand;
    return B200_OK;
  }
  int candidate_cost(double* cost) { return b200_evaluate(h, v.cand.data(), cost, nullptr, nullptr, 0); }
  int evaluate(b200_lm_iteration* it) {
    OK(b200_evaluate(h, v.x.data(), &it->cost, v.residuals.data(), v.gradient.data(), 1));
    double* sc = v.scaling.data();
    if (opt->jacobi_scaling && !have_scaling) {
      OK(b200_jacobian_squared_column_norm(h, sc));
#pragma omp parallel for num_threads(kHostThreads) schedule(static)
      for (int i = 0; i < np; ++i) sc[i] = 1.0 / (1.0 + std::sqrt(sc[i]));
      have_scaling = true;
    }
    if (opt->jacobi_scaling) OK(b200_jacobian_scale_columns(h, sc));
    const double* gr = v.gradient.data();
    double n[2];
    OK(host_reduce(h, 0x1u, n, [&](int i, double* a) {
      a[0] = std::max(a[0], std::fabs(gr[i]));
      a[1] += gr[i] * gr[i];
    }));
    it->gradient_max_norm = n[0];
    it->gradient_norm = std::sqrt(n[1]);
    return B200_OK;
  }
  int model_cost_change(double* mcc) { return b200_model_cost_change(h, v.step.data(), mcc); }
  // the solve at D = lmD of the configured solver, on the residuals of the last evaluate, still in HBM
  int solve(const b200_solver_options* so, b200_solver_summary* ls) {
    if (opt->linear_solver_type == B200_DENSE_SCHUR) return b200_dense_schur_solve(h, nullptr, v.lmD.data(), v.sol.data(), ls);
    if (opt->linear_solver_type == B200_SPARSE_SCHUR) return b200_sparse_schur_solve(h, nullptr, v.lmD.data(), v.sol.data(), ls);
    return b200_schur_solve(h, nullptr, v.lmD.data(), so, v.sol.data(), ls);
  }

  int lm_solve(bool reuse_diagonal, double radius, const b200_solver_options* so, b200_solver_summary* ls) {
    double *dg = v.diagonal.data(), *ld = v.lmD.data();
    const double lo = opt->min_lm_diagonal, hi = opt->max_lm_diagonal;
    if (!reuse_diagonal) OK(b200_jacobian_squared_column_norm(h, dg));
#pragma omp parallel for num_threads(kHostThreads) schedule(static)
    for (int i = 0; i < np; ++i) {
      if (!reuse_diagonal) dg[i] = std::min(std::max(dg[i], lo), hi);
      ld[i] = std::sqrt(dg[i] / radius);
    }
    return solve(so, ls);
  }
  // step = -sol, delta = step * scaling, candidate = x + delta (Evaluator::Plus on Euclidean blocks) and the norms
  int lm_step(StepResult* r) {
    const double *sl = v.sol.data(), *xx = v.x.data(), *sc = v.scaling.data();
    const uint8_t* fx = h->fixed_any ? h->h_fixed.data() : nullptr;
    double *stp = v.step.data(), *cd = v.cand.data();
    double s[3];
    OK(host_reduce(h, 0u, s, [&](int i, double* a) {
      const double si = -sl[i];
      stp[i] = si;
      // constant: x unchanged; |x| over the reduced x, which holds masked coordinates and no constant block
      const uint8_t fixed = fx != nullptr ? fx[i] : 0;
      const double ci = fixed != 0 ? xx[i] : xx[i] + si * sc[i];
      cd[i] = ci;
      a[0] += (xx[i] - ci) * (xx[i] - ci);
      if (fixed != kComponentConstant) a[1] += xx[i] * xx[i];
      a[2] += (si - si);   // NaN/Inf - itself is NaN, finite - itself is 0
    }));
    r->step_sq = s[0];
    r->x_sq = s[1];
    r->finite = s[2] == 0.0;
    return B200_OK;
  }

  // DOGLEG, a new Gauss-Newton step: diagonal = sqrt(clamped column norms), g = J'r / diagonal
  int dl_gradient(int) {
    for (PinnedVec* p : {&v.g, &v.gn}) p->resize(np);
    for (PinnedVec* p : {&v.ja, &v.jb}) p->resize(nr);
    double *d = v.diagonal.data(), *gp = v.g.data();
    OK(b200_jacobian_squared_column_norm(h, d));
    const double lo = opt->min_lm_diagonal, hi = opt->max_lm_diagonal;
#pragma omp parallel for num_threads(kHostThreads) schedule(static)
    for (int i = 0; i < np; ++i) d[i] = std::sqrt(std::min(std::max(d[i], lo), hi));
    std::fill(v.g.begin(), v.g.end(), 0.0);
    OK(b200_jacobian_left_multiply(h, v.residuals.data(), gp));
#pragma omp parallel for num_threads(kHostThreads) schedule(static)
    for (int i = 0; i < np; ++i) gp[i] /= d[i];
    return B200_OK;
  }
  int dl_gauss_newton(bool, double sqrt_mu, b200_solver_summary* ls, b200dl::Model* m) {
    const double *dg = v.diagonal.data(), *sl = v.sol.data(), *gp = v.g.data();
    double *ld = v.lmD.data(), *gnp = v.gn.data();
#pragma omp parallel for num_threads(kHostThreads) schedule(static)
    for (int i = 0; i < np; ++i) ld[i] = dg[i] * sqrt_mu;
    OK(solve(nullptr, ls));
    if (ls->termination_type == B200_LS_FAILURE || ls->termination_type == B200_LS_FATAL_ERROR) return B200_OK;
    double s[4];
    OK(host_reduce(h, 0u, s, [&](int i, double* a) {
      const double x = sl[i] * -dg[i];
      gnp[i] = x;
      a[0] += gp[i] * gp[i];
      a[1] += gp[i] * x;
      a[2] += x * x;
      if (!std::isfinite(sl[i])) a[3] += 1.0;
    }));
    m->gg = s[0];
    m->ggn = s[1];
    m->gngn = s[2];
    if (s[3] != 0.0) ls->termination_type = B200_LS_FAILURE;
    return B200_OK;
  }
  int dl_gram(bool two, b200dl::Model* m) {
    const double *dg = v.diagonal.data(), *ja = v.ja.data(), *jb = v.jb.data();
    double* sl = v.sol.data();
    auto jmul = [&](const double* src, PinnedVec& dst) -> int {   // dst = J (src / diagonal)
#pragma omp parallel for num_threads(kHostThreads) schedule(static)
      for (int i = 0; i < np; ++i) sl[i] = src[i] / dg[i];
      std::fill(dst.begin(), dst.end(), 0.0);
      return b200_jacobian_right_multiply(h, sl, dst.data());
    };
    OK(jmul(v.g.data(), v.ja));
    double aa = 0.0;
#pragma omp parallel for num_threads(kHostThreads) schedule(static) reduction(+ : aa)
    for (size_t i = 0; i < nr; ++i) aa += ja[i] * ja[i];
    m->jaja = aa;
    if (!two) return B200_OK;
    OK(jmul(v.gn.data(), v.jb));
    double bb = 0.0, ab = 0.0;
#pragma omp parallel for num_threads(kHostThreads) schedule(static) reduction(+ : bb, ab)
    for (size_t i = 0; i < nr; ++i) {
      bb += jb[i] * jb[i];
      ab += ja[i] * jb[i];
    }
    m->jbjb = bb;
    m->jajb = ab;
    return B200_OK;
  }
  int dl_step(const b200dl::Step& st, StepResult* r, double* vv) {
    const double *gp = v.g.data(), *gnp = v.gn.data(), *dg = v.diagonal.data(), *xx = v.x.data(), *sc = v.scaling.data();
    const uint8_t* fx = h->fixed_any ? h->h_fixed.data() : nullptr;
    double *stp = v.step.data(), *cd = v.cand.data();
    const int kind = st.kind;
    const double cg = st.cg, cn = st.cn;
    double s[4];
    OK(host_reduce(h, 0u, s, [&](int i, double* a) {
      const double x = kind == b200dl::kGaussNewton ? gnp[i] : kind == b200dl::kGradient ? cg * gp[i] : cg * gp[i] + cn * gnp[i];
      const double si = x / dg[i];
      stp[i] = si;
      const uint8_t fixed = fx != nullptr ? fx[i] : 0;
      const double ci = fixed != 0 ? xx[i] : xx[i] + si * sc[i];
      cd[i] = ci;
      a[0] += (xx[i] - ci) * (xx[i] - ci);
      if (fixed != kComponentConstant) a[1] += xx[i] * xx[i];
      if (!std::isfinite(si)) a[2] += 1.0;
      a[3] += x * x;
    }));
    r->step_sq = s[0];
    r->x_sq = s[1];
    r->finite = s[2] == 0.0;
    *vv = s[3];
    return B200_OK;
  }
};

// LevenbergMarquardtStrategy (levenberg_marquardt_strategy.cc): the radius and its updates.
struct LmStrategy {
  double radius, max_radius;
  b200_solver_options so;   // ITERATIVE_SCHUR's options: q_tolerance = eta, no r_tolerance
  double decrease_factor = 2.0;
  bool reuse_diagonal = false;

  explicit LmStrategy(const b200_lm_options* o) : radius(o->initial_trust_region_radius), max_radius(o->max_trust_region_radius), so(o->linear_solver) {
    so.q_tolerance = o->eta;
    so.r_tolerance = -1.0;
  }
  template <class Side>
  int compute_step(Side& side, StepResult* r) {
    // (levenberg_marquardt_strategy.cc:108 pre-fills the step with NaN so that a solver that silently writes nothing is
    //  caught; here the solve either fills its output or reports FAILURE / FATAL_ERROR, which is checked below)
    OK(side.lm_solve(reuse_diagonal, radius, &so, &r->ls));
    reuse_diagonal = true;
    if (r->ls.termination_type == B200_LS_FATAL_ERROR) return fail(B200_ERR_CUDA, "linear solver fatal error");
    if (r->ls.termination_type == B200_LS_FAILURE) return B200_OK;
    OK(side.lm_step(r));
    return r->finite ? side.model_cost_change(&r->model_cost_change) : B200_OK;
  }
  void accepted(double relative_decrease) {
    radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * relative_decrease - 1.0, 3));
    radius = std::min(max_radius, radius);
    decrease_factor = 2.0;
    reuse_diagonal = false;
  }
  void rejected() {
    radius = radius / decrease_factor;
    decrease_factor *= 2.0;
    reuse_diagonal = true;
  }
  void invalid() { rejected(); }
};

// DoglegStrategy (dogleg_strategy.cc:54-717): the state and its updates are dogleg.h's (accepted() has no clamp to
// max_trust_region_radius, :618-634; invalid() keeps the radius, :641-644); ComputeStep (:79-167) is here.
struct DoglegStrategy : b200dl::Strategy {
  b200dl::Model dm;

  explicit DoglegStrategy(const b200_lm_options* o) {
    type = o->dogleg_type;
    radius = o->initial_trust_region_radius;
  }
  template <class Side>
  int compute_step(Side& side, StepResult* r) {
    b200_solver_summary* ls = &r->ls;
    if (!reuse) {
      reuse = true;
      ls->num_iterations = -1;   // LinearSolver::Summary's defaults (linear_solver.h:320-326) when no solve runs
      ls->termination_type = B200_LS_FAILURE;
      OK(side.dl_gradient(type));
      // ComputeGaussNewtonStep (:517-616): raise mu tenfold after each FAILURE or non-finite solution, while mu < 1
      for (bool refresh = true; mu < b200dl::kMaxMu; refresh = false) {
        OK(side.dl_gauss_newton(refresh, std::sqrt(mu), ls, &dm));
        if (ls->termination_type == B200_LS_FATAL_ERROR) return fail(B200_ERR_CUDA, "linear solver fatal error");
        if (ls->termination_type != B200_LS_FAILURE) break;
        mu *= b200dl::kMuIncreaseFactor;
      }
      if (ls->termination_type == B200_LS_FAILURE) return B200_OK;
      const bool two = type == b200dl::kSubspace;
      OK(side.dl_gram(two, &dm));
      b200dl::cauchy_point(&dm);
      if (two) b200dl::subspace_model(&dm);
      if (two && dm.rank == 0) {   // ComputeSubspaceModel fails (:656-664): the strategy reports FAILURE
        ls->termination_type = B200_LS_FAILURE;
        return B200_OK;
      }
    } else {   // a rejected step: same GN step, gradient and model, new radius (:89-106)
      ls->num_iterations = 0;
      ls->termination_type = B200_LS_SUCCESS;
    }
    const b200dl::Step st = step(dm);
    double vv = 0.0;
    OK(side.dl_step(st, r, &vv));
    step_norm = st.measure_norm ? std::sqrt(vv) : st.norm;
    // a non-finite step has a NaN model cost change in the reference, which makes the step invalid
    r->model_cost_change = std::numeric_limits<double>::quiet_NaN();
    return r->finite ? side.model_cost_change(&r->model_cost_change) : B200_OK;
  }
};

// TrustRegionMinimizer::Minimize (trust_region_minimizer.cc): the iteration records, the exits, the relative decrease with
// the step evaluator's non-monotonic history, accept / reject and the best state, over either side and either strategy.
template <class Side, class Strategy>
int minimize(Side side, Strategy strategy, const b200_lm_options* opt, double* state_inout, b200_lm_iteration* trace,
             int max_records, int* num_records) {
  OK(side.begin(state_inout));
  b200_lm_iteration it{};
  OK(side.evaluate(&it));
  double x_cost = it.cost, minimum_cost = std::numeric_limits<double>::max();
  it.step_is_valid = 1;
  it.step_is_successful = 1;
  double se_minimum = x_cost, se_current = x_cost, se_reference = x_cost, se_candidate = x_cost, se_acc_ref = 0, se_acc_cand = 0;
  int num_consecutive_invalid = 0;
  bool at_least_one_successful = false;

  for (;;) {
    if (it.step_is_successful && x_cost < minimum_cost) {
      minimum_cost = x_cost;
      OK(side.keep_best());
    }
    it.trust_region_radius = strategy.radius;
    if (*num_records < max_records) trace[(*num_records)++] = it;
    if (it.iteration >= opt->max_num_iterations) break;
    if (it.step_is_successful && it.gradient_max_norm <= opt->gradient_tolerance) break;
    if (it.trust_region_radius <= opt->min_trust_region_radius) break;

    const b200_lm_iteration prev = it;
    it = b200_lm_iteration{};
    it.iteration = prev.iteration + 1;

    StepResult r;
    OK(strategy.compute_step(side, &r));
    const double model_cost_change = r.model_cost_change;
    it.linear_solver_iterations = r.ls.num_iterations;
    it.model_cost_change = model_cost_change;
    it.step_is_valid = model_cost_change > 0.0;
    if (!it.step_is_valid) {
      if (++num_consecutive_invalid >= opt->max_num_consecutive_invalid_steps) break;
      strategy.invalid();
      it.cost = x_cost;
      it.cost_change = 0.0;
      it.gradient_max_norm = prev.gradient_max_norm;
      it.gradient_norm = prev.gradient_norm;
      it.step_norm = 0.0;
      it.relative_decrease = 0.0;
      continue;
    }
    num_consecutive_invalid = 0;

    // ---- ComputeCandidatePointAndEvaluateCost
    double candidate_cost = 0.0;
    const int rc = side.candidate_cost(&candidate_cost);
    if (rc == B200_ERR_EVALUATION_FAILED) candidate_cost = std::numeric_limits<double>::max();
    else if (rc != B200_OK) return rc;

    // (assigned only once a step has been accepted, like the reference: trust_region_minimizer.cc:113, :730)
    it.step_norm = at_least_one_successful ? std::sqrt(r.step_sq) : 0.0;
    if (at_least_one_successful && it.step_norm <= opt->parameter_tolerance * (std::sqrt(r.x_sq) + opt->parameter_tolerance)) break;
    it.cost_change = x_cost - candidate_cost;
    if (std::fabs(it.cost_change) <= opt->function_tolerance * x_cost) break;

    if (candidate_cost >= std::numeric_limits<double>::max()) {
      it.relative_decrease = std::numeric_limits<double>::lowest();
    } else {
      const double rd = (se_current - candidate_cost) / model_cost_change;
      const double hist = (se_reference - candidate_cost) / (se_acc_ref + model_cost_change);
      it.relative_decrease = std::max(rd, hist);
    }
    if (it.relative_decrease > opt->min_relative_decrease) {
      at_least_one_successful = true;
      OK(side.accept());
      OK(side.evaluate(&it));
      x_cost = it.cost;
      it.step_is_successful = 1;
      strategy.accepted(it.relative_decrease);
      se_current = candidate_cost;
      se_acc_cand += model_cost_change;
      se_acc_ref += model_cost_change;
      if (se_current < se_minimum) {
        se_minimum = se_current;
        se_candidate = se_current;
        se_acc_cand = 0.0;
        se_reference = se_candidate;
        se_acc_ref = se_acc_cand;
      } else if (se_current > se_candidate) {
        se_candidate = se_current;
        se_acc_cand = 0.0;
      }
    } else {
      it.step_is_successful = 0;
      it.cost = candidate_cost;
      it.gradient_norm = prev.gradient_norm;
      it.gradient_max_norm = prev.gradient_max_norm;
      strategy.rejected();
    }
  }
  return side.finish(state_inout);
}

}  // namespace

// ================================================================================================ C ABI
// Covariance (b200_covariance_compute)
namespace {

// b200_covariance_compute's apply_loss_function holds for that call only: the handle's own setting comes back on every exit.
struct ApplyLossGuard {
  b200_handle* h;
  bool saved;
  ~ApplyLossGuard() { h->apply_loss = saved; }
};

// S's block pattern on the host and its block row pointers on the device, once per handle (it depends on the rows only).
int cov_pattern(b200_handle* h) {
  if (h->d_cov_row_ptr != nullptr) return B200_OK;
  XsPattern xp;
  xs_pattern(h->C, h->N, h->h_cam_idx.data(), h->h_pt_idx.data(), h->h_pt_ptr.data(), &xp);
  h->cov_row_ptr = xp.row_ptr;
  h->cov_blk_col = xp.blk_col;
  OK(upload(h, h->cov_row_ptr, &h->d_cov_row_ptr));
  CU(cudaStreamSynchronize(h->stream));
  return B200_OK;
}

// SPARSE_SCHUR: S with D = 0 (D' = 1 on constant components) factored by sparse_factor_kernel, Z on L's pattern by
// sparse_selinv_kernel, copied to S's blocks (h->d_cov_s).  *factored = false when a pivot is not positive.
int cov_sparse_dev(b200_handle* h, bool* factored) {
  if (!h->sp_ready) OK(sparse_analyse(h));
  SparseView<double>& v = h->spv;
  if (h->sp_selinv_grid < 1)
    return fail(B200_ERR_UNSUPPORTED, "no CTA of the selected inversion fits an SM (%zu bytes of shared memory)", h->sp_selinv_smem);
  OK(cov_pattern(h));
  // what is resident at once: the FP64 factor, Z, Z on S's blocks, and a float factor a mixed-precision solve left
  const double bytes = 16.0 * static_cast<double>(h->sp_storage) + 648.0 * static_cast<double>(h->cov_blk_col.size()) +
                       (h->spv32.L != nullptr ? 4.0 * static_cast<double>(h->sp_storage) : 0.0);
  if (bytes > kFactorMaxBytes) return fail(B200_ERR_UNSUPPORTED, "covariance of %d cameras needs %.1f GB of factor and inverse", h->C, bytes / 1e9);
  if (h->d_cov_z == nullptr) OK(dev_alloc(h, &h->d_cov_z, static_cast<size_t>(h->sp_storage)));
  if (h->d_cov_s == nullptr) OK(dev_alloc(h, &h->d_cov_s, 81 * h->cov_blk_col.size()));
  OK(schur_init_dev(h, h->d_residuals, nullptr));   // (E'E)^-1, identity on constant points
  OK(xs_assemble_dev(h));
  const double* Df = h->cur_D != nullptr ? h->cur_D + 3 * static_cast<size_t>(h->P) : nullptr;
  OK(sparse_factor(h, v, h->sp_grid, h->sp_smem, Df, factored));
  if (!*factored) return B200_OK;
  cudaError_t le = cudaSuccess;
  const uint8_t* fixed_f = h->fixed_any ? h->d_fixed + 3 * static_cast<size_t>(h->P) : nullptr;
  OK(launch(h, K_MISC, [&] {
    selinv_pivots_kernel<<<flat_grid(h, 9 * static_cast<size_t>(h->C), 256), 256, 0, h->stream>>>(v, h->xsv, h->d_cov_row_ptr, Df,
                                                                                                 fixed_f, h->d_cov_min);
  }));
  CU(cudaMemcpyAsync(v.cnt, h->d_sp_cnt_inv, sizeof(int) * static_cast<size_t>(v.ns), cudaMemcpyDeviceToDevice, h->stream));
  CU(cudaMemsetAsync(v.ticket, 0, sizeof(int), h->stream));
  OK(launch(h, K_SELINV, [&] {
    void* args[] = {&v, &h->d_cov_z};
    le = cudaLaunchCooperativeKernel(reinterpret_cast<void*>(sparse_selinv_kernel), dim3(h->sp_selinv_grid), dim3(kSpThreads), args,
                                     h->sp_selinv_smem, h->stream);
  }));
  CU(le);
  const int nb = static_cast<int>(h->cov_blk_col.size());
  return launch(h, K_SELINV, [&] {
    selinv_blocks_kernel<<<std::max(1, std::min((nb + 7) / 8, h->sm_count * 8)), 256, 0, h->stream>>>(v, nb, h->d_cov_z, h->d_cov_s);
  }, false);
}

// DENSE_SCHUR: the FP64 dense assembly of the solves into h->d_cov_dense, cusolverDnDpotrf, then cusolverDnDpotri: Z's lower
// triangle.  *factored = false when potrf finds a non-positive pivot.
int cov_dense_dev(b200_handle* h, bool* factored) {
  const int n = 9 * h->C;
  const size_t bytes = sizeof(double) * static_cast<size_t>(n) * n;
  // what is resident at once: the covariance's matrix and workspace, and whatever dense solves left allocated (their FP64
  // matrix and workspace, and the float copy of mixed precision)
  auto resident = [&](size_t cov_work) {
    size_t b = bytes + sizeof(double) * cov_work;
    if (h->d_dense_s != nullptr) b += bytes + sizeof(double) * static_cast<size_t>(h->dense_lwork);
    if (h->d_dense_s32 != nullptr) b += bytes / 2 + sizeof(float) * static_cast<size_t>(h->dense_lwork32);
    return b;
  };
  const size_t cap = static_cast<size_t>(48) << 30;
  if (resident(0) > cap)
    return fail(B200_ERR_UNSUPPORTED, "dense covariance of %d cameras needs %.1f GB", h->C, resident(0) / 1e9);
  if (!load_cusolver()) return fail(B200_ERR_UNSUPPORTED, "cannot load libcusolver.so.11: %s", dlerror());
  if (!g_cusolver.potri_ok) return fail(B200_ERR_UNSUPPORTED, "the loaded cuSOLVER lacks cusolverDnDpotri (covariance)");
  if (h->cusolver == nullptr) {
    if (g_cusolver.Create(&h->cusolver) != 0) return fail(B200_ERR_CUDA, "cusolverDnCreate failed");
    if (g_cusolver.SetStream(h->cusolver, h->stream) != 0) return fail(B200_ERR_CUDA, "cusolverDnSetStream failed");
  }
  if (h->d_cov_dense == nullptr) {
    OK(dev_alloc(h, &h->d_cov_dense, static_cast<size_t>(n) * n));
    OK(dev_alloc(h, &h->d_cov_diag, static_cast<size_t>(n)));
    int a = 0, b = 0;
    if (g_cusolver.DpotrfBufferSize(h->cusolver, /*CUBLAS_FILL_MODE_LOWER*/ 0, n, h->d_cov_dense, n, &a) != 0)
      return fail(B200_ERR_CUDA, "cusolverDnDpotrf_bufferSize failed");
    if (g_cusolver.DpotriBufferSize(h->cusolver, 0, n, h->d_cov_dense, n, &b) != 0)
      return fail(B200_ERR_CUDA, "cusolverDnDpotri_bufferSize failed");
    h->cov_lwork = std::max(1, std::max(a, b));
    if (resident(static_cast<size_t>(h->cov_lwork)) > cap) {   // refused with nothing left half-allocated
      dev_free(h, h->d_cov_dense);
      dev_free(h, h->d_cov_diag);
      return fail(B200_ERR_UNSUPPORTED, "dense covariance of %d cameras needs %.1f GB with its workspace", h->C,
                  resident(static_cast<size_t>(h->cov_lwork)) / 1e9);
    }
    OK(dev_alloc(h, &h->d_cov_work, static_cast<size_t>(h->cov_lwork)));
  }
  OK(schur_init_dev(h, h->d_residuals, nullptr));
  const double* Df = h->cur_D != nullptr ? h->cur_D + 3 * static_cast<size_t>(h->P) : nullptr;
  CU(cudaMemsetAsync(h->d_cov_dense, 0, bytes, h->stream));
  OK(launch(h, K_DIAG_BLOCKS, [&] {
    dense_schur_assemble_kernel<<<std::max(1, std::min(h->P, h->sm_count * 8)), kDsThreads, 0, h->stream>>>(h->view, h->d_ete_inv, h->d_cov_dense, static_cast<size_t>(n));
  }));
  OK(launch(h, K_MISC, [&] {
    dense_schur_diagonal_kernel<<<(n + 255) / 256, 256, 0, h->stream>>>(n, Df, h->d_cov_dense, static_cast<size_t>(n));
    dense_diagonal_copy_kernel<<<flat_grid(h, n, 256), 256, 0, h->stream>>>(n, h->d_cov_dense, h->d_cov_diag);
  }));
  int* info = reinterpret_cast<int*>(h->d_cov_min + 1);
  if (g_cusolver.Dpotrf(h->cusolver, 0, n, h->d_cov_dense, n, h->d_cov_work, h->cov_lwork, info) != 0)
    return fail(B200_ERR_CUDA, "cusolverDnDpotrf failed");
  CU(cudaMemcpyAsync(h->h_fail, info, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  *factored = h->h_fail[0] == 0;
  if (!*factored) return B200_OK;
  const uint8_t* fixed_f = h->fixed_any ? h->d_fixed + 3 * static_cast<size_t>(h->P) : nullptr;
  OK(launch(h, K_MISC, [&] {
    dense_pivots_kernel<<<flat_grid(h, n, 256), 256, 0, h->stream>>>(n, h->d_cov_dense, h->d_cov_diag, fixed_f, h->d_cov_min);
  }));
  int potri = 0;
  OK(launch(h, K_SELINV, [&] { potri = g_cusolver.Dpotri(h->cusolver, 0, n, h->d_cov_dense, n, h->d_cov_work, h->cov_lwork, info); }));
  if (potri != 0) return fail(B200_ERR_CUDA, "cusolverDnDpotri failed");
  return launch(h, K_SELINV, [&] {
    dense_symmetrize_kernel<<<h->sm_count * 8, 256, 0, h->stream>>>(static_cast<long long>(n), h->d_cov_dense);
  }, false);
}

// The effective state of the constant blocks and SubsetManifolds a handle holds, as Ceres' ParameterBlock sees it: a block
// is constant when it is set constant or when its SubsetManifold holds every coordinate (IsConstant: is_set_constant_ ||
// TangentSize() == 0); otherwise the coordinates its SubsetManifold holds are masked.  This is the one place that decides
// between a masked coordinate and a constant block: the component states in the caller's and the internal order, and the
// packed block states of the evaluate kernels.
struct FixedState {
  std::vector<uint8_t> caller, internal;   // [3P+9C] 0, kComponentMasked, kComponentConstant
  std::vector<uint16_t> blocks;            // [P + C] internal order: kBlockConstant, or the masked coordinates' bits
  bool any = false;
};

// From the setters' inputs (caller's order; empty = none).  B200_ERR_INVALID_ARGUMENT for a row whose camera and point are
// both constant: Program::RemoveFixedBlocks drops it (its cost goes to fixed_cost), which the caller does by not passing it.
int fixed_state(const b200_handle* h, const std::vector<uint8_t>& cam_const, const std::vector<uint8_t>& pt_const,
                const std::vector<uint16_t>& cam_mask, const std::vector<uint8_t>& pt_mask, FixedState* st) {
  const size_t coff = 3 * static_cast<size_t>(h->P);
  st->caller.assign(h->np, 0);
  st->internal.assign(h->np, 0);
  st->blocks.assign(static_cast<size_t>(h->P) + h->C, 0);
  st->any = false;
  // one block of n coordinates: its packed state, and its component states at caller[c0..] and internal[i0..]
  auto block = [&](bool constant, unsigned mask, int n, size_t c0, size_t i0, size_t b) {
    const unsigned full = (1u << n) - 1;
    constant = constant || (mask & full) == full;
    st->blocks[b] = constant ? kBlockConstant : static_cast<uint16_t>(mask & full);
    for (int j = 0; j < n; ++j) {
      const uint8_t f = constant ? kComponentConstant : (mask >> j) & 1u ? kComponentMasked : 0;
      st->caller[c0 + j] = st->internal[i0 + j] = f;
      st->any = st->any || f != 0;
    }
  };
  for (int k = 0; k < h->P; ++k) {
    const int c = h->permuted ? h->h_pt_perm[k] : k;   // internal point k is the caller's point c
    block(!pt_const.empty() && pt_const[c] != 0, pt_mask.empty() ? 0u : pt_mask[c], 3, 3 * static_cast<size_t>(c),
          3 * static_cast<size_t>(k), static_cast<size_t>(k));
  }
  for (int k = 0; k < h->C; ++k)
    block(!cam_const.empty() && cam_const[k] != 0, cam_mask.empty() ? 0u : cam_mask[k], 9, coff + 9 * static_cast<size_t>(k),
          coff + 9 * static_cast<size_t>(k), static_cast<size_t>(h->P) + k);
  for (int i = 0; i < h->N; ++i) {
    const int pt = h->h_pt_idx[i], cam = h->h_cam_idx[i];
    if (st->blocks[pt] == kBlockConstant && st->blocks[static_cast<size_t>(h->P) + cam] == kBlockConstant)
      return fail(B200_ERR_INVALID_ARGUMENT,
                  "row %d: camera %d and point %d are both constant; drop the row, as Program::RemoveFixedBlocks does",
                  h->permuted ? h->h_row_perm[i] : i, cam, h->permuted ? h->h_pt_perm[pt] : pt);
  }
  return B200_OK;
}

// Validates and applies the setters' inputs; the handle is unchanged when they are refused.  The new state applies from
// the next evaluation on: the stored J's constant cells are zeroed now, and everything formed from J is invalidated.
int set_fixed(b200_handle* h, std::vector<uint8_t> cam_const, std::vector<uint8_t> pt_const, std::vector<uint16_t> cam_mask,
              std::vector<uint8_t> pt_mask) {
  FixedState st;
  OK(fixed_state(h, cam_const, pt_const, cam_mask, pt_mask, &st));
  CU(cudaSetDevice(h->device));
  if (st.any) {
    if (h->d_fixed == nullptr) OK(dev_alloc(h, &h->d_fixed, h->np));
    if (h->d_solve_D == nullptr) OK(dev_alloc(h, &h->d_solve_D, h->np));
    if (h->d_block_state == nullptr) OK(dev_alloc(h, &h->d_block_state, st.blocks.size()));
    CU(cudaMemcpyAsync(h->d_fixed, st.internal.data(), st.internal.size(), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_block_state, st.blocks.data(), sizeof(uint16_t) * st.blocks.size(), cudaMemcpyHostToDevice, h->stream));
  }
  h->set_cam_const = std::move(cam_const);
  h->set_pt_const = std::move(pt_const);
  h->set_cam_mask = std::move(cam_mask);
  h->set_pt_mask = std::move(pt_mask);
  h->h_fixed = std::move(st.caller);
  h->fixed_any = st.any;
  OK(fixed_mask_dev(h));
  CU(cudaStreamSynchronize(h->stream));   // (the uploads read st, which goes out of scope)
  // everything formed from J is stale, the Schur initialisation and the preconditioner built on it included
  jacobian_written(h);
  h->xs_diag_ready = false;
  h->schur_ready = false;
  return B200_OK;
}

template <bool kDense>
ZAccess<kDense> cov_access(const b200_handle* h) {
  ZAccess<kDense> z{};
  z.Z = kDense ? h->d_cov_dense : h->d_cov_s;
  z.blk_row_ptr = h->d_cov_row_ptr;
  z.blk_col = h->xsv.blk_col;
  z.n = 9LL * h->C;
  return z;
}

}  // namespace

extern "C" {

const char* b200_last_error(void) { return g_error.c_str(); }

int b200_nccl_unique_id(void* out128) {
#ifdef B200_WITH_NCCL
  if (!load_nccl()) return fail(B200_ERR_NCCL, "cannot load libnccl.so.2: %s", dlerror());
  ncclUniqueId id;
  ncclResult_t r = g_nccl.GetUniqueId(&id);
  if (r != ncclSuccess) return fail(B200_ERR_NCCL, "ncclGetUniqueId: %s", g_nccl.GetErrorString(r));
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
  std::memcpy(out128, &id, 128);
  return B200_OK;
#else
  (void)out128;
  return fail(B200_ERR_UNSUPPORTED, "built without NCCL");
#endif
}

int b200_plan_point_order(const b200_ba_desc* desc, int num_chunks, int32_t* perm_out, int64_t metrics_out[4], int* choice_out) {
  if (desc == nullptr || desc->cam_idx == nullptr || desc->pt_idx == nullptr || num_chunks < 1)
    return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  const int C = desc->num_cameras, P = desc->num_points;
  const int N = static_cast<int>(desc->num_observations);
  if (C <= 0 || P <= 0 || N <= 0) return fail(B200_ERR_INVALID_ARGUMENT, "empty problem");
  std::vector<int> ptr;
  OK(validate_rows(desc, &ptr));
  std::vector<int> perm;
  long m[4];
  const int choice = choose_point_order(C, P, N, desc->cam_idx, ptr.data(), num_chunks, &perm, m);
  if (perm_out != nullptr)
    for (int k = 0; k < P; ++k) perm_out[k] = perm[k];
  if (metrics_out != nullptr)
    for (int k = 0; k < 4; ++k) metrics_out[k] = m[k];
  if (choice_out != nullptr) *choice_out = choice;
  return B200_OK;
}

int b200_plan_sparse_schur(const b200_ba_desc* desc, int32_t* cam_perm_out, int64_t stats_out[B200_SPARSE_STATS]) {
  return b200_plan_sparse_schur_ordered(desc, B200_AMD, cam_perm_out, stats_out);
}

int b200_plan_sparse_schur_ordered(const b200_ba_desc* desc, int ordering_type, int32_t* cam_perm_out,
                                   int64_t stats_out[B200_SPARSE_STATS]) {
  if (ordering_type != B200_AMD && ordering_type != B200_NESDIS)
    return fail(B200_ERR_INVALID_ARGUMENT, "linear_solver_ordering_type must be B200_AMD or B200_NESDIS, not %d", ordering_type);
  if (desc == nullptr || desc->cam_idx == nullptr || desc->pt_idx == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  const int C = desc->num_cameras, P = desc->num_points;
  const int N = static_cast<int>(desc->num_observations);
  if (C <= 0 || P <= 0 || N <= 0) return fail(B200_ERR_INVALID_ARGUMENT, "empty problem");
  std::vector<int> ptr;
  OK(validate_rows(desc, &ptr));
  XsPattern xp;   // the block pattern of S does not depend on the point order: the caller's rows give the handle's pattern
  xs_pattern(C, N, desc->cam_idx, desc->pt_idx, ptr.data(), &xp);
  SparsePlan sp;
  plan_sparse_schur(C, xp.blk_row, xp.blk_col, ordering_type, &sp);
  if (cam_perm_out != nullptr)
    for (int k = 0; k < C; ++k) cam_perm_out[k] = sp.perm[k];
  if (stats_out != nullptr)
    for (int k = 0; k < B200_SPARSE_STATS; ++k) stats_out[k] = sp.stats[k];
  return B200_OK;
}

int b200_plan_sparse_selinv(const b200_ba_desc* desc, int ordering_type, int32_t* num_supernodes, int32_t* sn_first_out,
                            int32_t* order_out, int32_t* counter_out) {
  if (ordering_type != B200_AMD && ordering_type != B200_NESDIS)
    return fail(B200_ERR_INVALID_ARGUMENT, "linear_solver_ordering_type must be B200_AMD or B200_NESDIS, not %d", ordering_type);
  if (desc == nullptr || desc->cam_idx == nullptr || desc->pt_idx == nullptr || num_supernodes == nullptr)
    return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  const int C = desc->num_cameras, P = desc->num_points;
  const int N = static_cast<int>(desc->num_observations);
  if (C <= 0 || P <= 0 || N <= 0) return fail(B200_ERR_INVALID_ARGUMENT, "empty problem");
  std::vector<int> ptr;
  OK(validate_rows(desc, &ptr));
  XsPattern xp;
  xs_pattern(C, N, desc->cam_idx, desc->pt_idx, ptr.data(), &xp);
  SparsePlan sp;
  plan_sparse_schur(C, xp.blk_row, xp.blk_col, ordering_type, &sp);
  *num_supernodes = sp.ns;
  for (int s = 0; s <= sp.ns; ++s)
    if (sn_first_out != nullptr) sn_first_out[s] = sp.sn_first[s];
  for (int s = 0; s < sp.ns; ++s) {
    if (order_out != nullptr) order_out[s] = sp.order[s];
    if (counter_out != nullptr) counter_out[s] = sp.cnt_inv[s];
  }
  return B200_OK;
}

void b200_solver_options_default(b200_solver_options* o) {
  o->preconditioner_type = B200_PRECOND_SCHUR_JACOBI;
  o->min_num_iterations = 0;
  o->max_num_iterations = 500;  // examples/bundle_adjuster.cc:122
  o->residual_reset_period = 10;
  o->q_tolerance = 0.0;
  o->r_tolerance = 0.0;
  o->max_num_spse_iterations = 5;   // linear_solver.h:172
  o->use_spse_initialization = 0;   // :177
  o->spse_tolerance = 0.1;          // :183
}

void b200_lm_options_default(b200_lm_options* o) {
  o->max_num_iterations = 5;
  o->jacobi_scaling = 1;
  o->max_num_consecutive_invalid_steps = 5;
  o->linear_solver_type = B200_ITERATIVE_SCHUR;
  o->eta = 1e-2;
  o->initial_trust_region_radius = 1e4;
  o->max_trust_region_radius = 1e16;
  o->min_trust_region_radius = 1e-32;
  o->min_relative_decrease = 1e-3;
  o->min_lm_diagonal = 1e-6;
  o->max_lm_diagonal = 1e32;
  o->function_tolerance = 1e-16;
  o->gradient_tolerance = 1e-16;
  o->parameter_tolerance = 1e-16;
  b200_solver_options_default(&o->linear_solver);
  o->trust_region_strategy_type = B200_LEVENBERG_MARQUARDT;   // bundle_adjuster.cc:79-81
  o->dogleg_type = B200_TRADITIONAL_DOGLEG;
  o->use_mixed_precision_solves = 0;     // solver.h:572-580
  o->max_num_refinement_iterations = 0;  // :582-590
  o->linear_solver_ordering_type = B200_AMD;   // solver.h:410
}

int b200_create(const b200_ba_desc* desc, b200_handle** out) {
  if (desc == nullptr || out == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  if (desc->num_cameras <= 0 || desc->num_points <= 0 || desc->num_observations <= 0)
    return fail(B200_ERR_INVALID_ARGUMENT, "empty problem (C=%d P=%d N=%lld)", desc->num_cameras, desc->num_points,
                static_cast<long long>(desc->num_observations));
  if (desc->num_observations > 2000000000LL) return fail(B200_ERR_UNSUPPORTED, "more than 2e9 row blocks");
  if (desc->cam_idx == nullptr || desc->pt_idx == nullptr || desc->obs == nullptr)
    return fail(B200_ERR_INVALID_ARGUMENT, "null structure array");
  if (desc->loss_type != B200_LOSS_TRIVIAL && desc->loss_type != B200_LOSS_HUBER)
    return fail(B200_ERR_INVALID_ARGUMENT, "loss_type %d: the descriptor takes B200_LOSS_TRIVIAL or B200_LOSS_HUBER, other losses "
                "go through b200_set_loss_functions", desc->loss_type);
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(B200_ERR_NO_DEVICE, "no CUDA device visible: libb200ba has no CPU fallback");
  }
  if (desc->device < 0 || desc->device >= ndev) return fail(B200_ERR_INVALID_ARGUMENT, "device %d of %d", desc->device, ndev);
  CU(cudaSetDevice(desc->device));
  cudaDeviceProp prop;
  CU(cudaGetDeviceProperties(&prop, desc->device));
  if (prop.major != 9 || prop.minor != 0)   // sm_90a code loads on sm_90 devices only
    return fail(B200_ERR_NO_DEVICE, "device %s is sm_%d%d; this library is built for sm_90a (H100) only", prop.name, prop.major, prop.minor);

  const int C = desc->num_cameras, P = desc->num_points;
  const int N = static_cast<int>(desc->num_observations);
  std::vector<int> caller_ptr;
  OK(validate_rows(desc, &caller_ptr));
  int l2_bytes = 0;
  CU(cudaDeviceGetAttribute(&l2_bytes, cudaDevAttrL2CacheSize, desc->device));
  int xs_per_sm = 0;   // the explicit-S product's grid is one wave of these (plan.cuh)
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&xs_per_sm, xs_mul_kernel, kXsThreads, 0));
  int xs_pcg_per_sm = 0;   // the resident PCG needs one CTA per SM at the most shared memory it may plan
  OK(set_func_attributes(static_cast<int>(prop.sharedMemPerBlockOptin)));
  CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&xs_pcg_per_sm, xs_pcg_kernel, kXpThreads, prop.sharedMemPerBlockOptin - 1024));
  const DevLimits lim{prop.multiProcessorCount, prop.sharedMemPerBlockOptin, l2_bytes, xs_per_sm, xs_pcg_per_sm};
  const DevKnobs knobs = DevKnobs::from_env();
  const int world = desc->world_size > 1 ? desc->world_size : 1;
  KernelPlan pl;
  plan_kernels(C, P, N, desc->cam_idx, desc->obs, caller_ptr, world, lim, knobs, &pl);
  if (!pl.huge_pts.empty() && pl.has_dups)
    return fail(B200_ERR_UNSUPPORTED,
                "a point with more than %d observations together with duplicate (camera, point) observations is not supported", kTile);
  print_plan(pl, C, P, N, world, lim, knobs);

  b200_handle* h = new b200_handle;
  h->device = desc->device;
  h->sm_count = prop.multiProcessorCount;
  h->C = C;
  h->P = P;
  h->N = N;
  h->np = 3 * P + 9 * C;
  h->num_tiles = static_cast<int>(pl.tiles.size());
  h->loss_one.type = desc->loss_type;
  h->loss_one.p = desc->loss_a;
  h->loss_one.q = desc->loss_a * desc->loss_a;
  h->loss_one.scale = 1.0;
  h->loss_cls = desc->loss_type == B200_LOSS_HUBER ? kLossHuber : kLossTrivial;
  h->rank = world > 1 ? desc->rank : 0;
  h->world = world;
  h->knobs = knobs;
  h->mul = pl.mul;
  h->diag = pl.diag;
  h->big_folded = pl.big_folded;
  h->xs = pl.xs;
  std::memset(h->launches, 0, sizeof(h->launches));
  std::memset(h->ms, 0, sizeof(h->ms));
  std::memset(h->ops, 0, sizeof(h->ops));
  std::copy(pl.bytes_per_op, pl.bytes_per_op + K_COUNT, h->bytes_per_op);
  *out = h;  // from here on the caller owns the handle even on failure (b200_destroy is safe on partial state)
  if (desc->stream != nullptr) {
    h->stream = static_cast<cudaStream_t>(desc->stream);
  } else {
    CU(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    h->own_stream = true;
  }
  CU(cudaStreamCreateWithFlags(&h->stream2, cudaStreamNonBlocking));
  CU(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&h->ev_join, cudaEventDisableTiming));

  // ---- device arrays: the problem, the solver state, and what the plan's kernels read
  const size_t n = static_cast<size_t>(N), nc = 9 * static_cast<size_t>(C);
  ProblemView& v = h->view;
  v.C = C;
  v.P = P;
  v.N = N;
  v.num_tiles = h->num_tiles;
  OK(upload(h, pl.tiles, &v.tiles));
  OK(upload(h, pl.cam_idx, &v.cam_idx));
  OK(upload(h, pl.pt_ptr, &v.pt_ptr));
  OK(upload(h, pl.pt_idx, &v.pt_of_row));
  OK(upload(h, pl.obs, &v.obs));
  OK(dev_alloc(h, &h->d_values, 24 * n));
  CU(cudaMemsetAsync(h->d_values, 0, 24 * n * sizeof(double), h->stream));
  v.values = h->d_values;
  for (double** p : {&h->d_state, &h->d_gradient, &h->d_vp0, &h->d_vp1, &h->d_D, &h->d_scale, &h->d_sqnorm, &h->d_diagonal,
                     &h->d_lmD, &h->d_step, &h->d_cand, &h->d_y})
    OK(dev_alloc(h, p, h->np));
  for (double** p : {&h->d_residuals, &h->d_vr0, &h->d_b}) OK(dev_alloc(h, p, 2 * n));
  for (double** p : {&h->d_rhs, &h->d_xr, &h->d_p, &h->d_r, &h->d_z, &h->d_tmp, &h->d_sol}) OK(dev_alloc(h, p, nc));
  OK(dev_alloc(h, &h->d_tile_partial, pl.tiles.size() + pl.num_ctas + pl.num_plain_big + pl.chunk_tiles.size() + 8));
  OK(dev_alloc(h, &h->d_fail, 4));
  OK(dev_alloc(h, &h->d_scalars, 64));
  OK(dev_alloc(h, &h->d_partial, kRedBlocks * 4));
  OK(dev_alloc(h, &h->d_ete_inv, 6 * static_cast<size_t>(P)));
  OK(dev_alloc(h, &h->d_ye, 3 * static_cast<size_t>(P)));
  OK(dev_alloc(h, &h->d_upper45, 45 * static_cast<size_t>(C)));
  OK(dev_alloc(h, &h->d_minv, 81 * static_cast<size_t>(C)));
  OK(dev_alloc(h, &h->d_blocks, 81 * static_cast<size_t>(C)));
  OK(dev_alloc(h, &h->d_cg, 1));
  CU(cudaMemsetAsync(h->d_cg, 0, sizeof(CgState), h->stream));
  CU(cudaMallocHost(reinterpret_cast<void**>(&h->h_scalars), 64 * sizeof(double)));
  CU(cudaMallocHost(reinterpret_cast<void**>(&h->h_cg), 2 * sizeof(CgState)));
  CU(cudaEventCreateWithFlags(&h->ev_cg[0], cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&h->ev_cg[1], cudaEventDisableTiming));
  CU(cudaMallocHost(reinterpret_cast<void**>(&h->h_fail), 4 * sizeof(int)));
  if (pl.order_choice != 0) {
    OK(upload(h, pl.pt_perm, &h->d_pt_perm));
    OK(upload(h, pl.row_perm, &h->d_row_perm));
    OK(dev_alloc(h, &h->d_stage_p, h->np));
    OK(dev_alloc(h, &h->d_stage_r, 2 * n));
    h->h_pt_perm = pl.pt_perm;
    h->h_row_perm = pl.row_perm;
    h->permuted = true;
  }
  if (h->diag == DiagPass::CamMajor) {
    h->num_cam_items = static_cast<int>(pl.cam_items.size());
    OK(upload(h, pl.cam_items, &h->d_cam_items));
    OK(upload(h, pl.cam_rows, &h->d_cam_rows));
    OK(dev_alloc(h, &h->d_q3, kQStride * n + 8));
  }
  h->num_huge = static_cast<int>(pl.huge_pts.size());
  if (h->num_huge > 0) OK(upload(h, pl.huge_pts, &h->d_huge_pts));
  if (h->mul != MulFamily::Tile) {
    TileDesc* d_big = nullptr;
    OK(upload(h, pl.big_tiles, &d_big));
    h->num_big_tiles = static_cast<int>(pl.big_tiles.size());
    h->view_big = h->view;
    h->view_big.tiles = d_big;
    h->view_big.num_tiles = h->num_big_tiles;
    h->view_chunks = h->view;
    h->view_chunks.tiles = d_big + pl.num_plain_big;
    h->view_chunks.num_tiles = static_cast<int>(pl.chunk_tiles.size());
    V2View dv{};   // the device arrays every warp-tile view reads
    OK(upload(h, pl.wtiles, &dv.wtiles));
    OK(upload(h, pl.row_meta, &dv.row_meta));
    OK(upload(h, pl.cta_part, &dv.cta_part));
    OK(upload(h, pl.cta_cam, &dv.cta_cam));
    OK(upload(h, pl.cta_cams, &dv.cta_cams));
    OK(upload(h, pl.cta_big, &dv.cta_big));
    OK(dev_alloc(h, &dv.partials, static_cast<size_t>(pl.num_ctas) * 9 * pl.max_cam_span));
    auto bind = [&](V2View g) {
      g.p = h->view;
      g.wtiles = dv.wtiles;
      g.row_meta = dv.row_meta;
      g.cta_part = dv.cta_part;
      g.cta_cam = dv.cta_cam;
      g.cta_cams = dv.cta_cams;
      g.cta_big = dv.cta_big;
      g.big_tiles = d_big;
      g.partials = dv.partials;
      return g;
    };
    h->d_cta_big = dv.cta_big;
    h->v2 = bind(pl.v2);
    h->v2_eval = bind(pl.v2_eval);
    h->v2_diag = bind(pl.v2_diag);
    h->v2_mul = bind(pl.v2_mul);
    if (is_v4(h->mul)) OK(upload(h, pl.tile_meta, &h->v2_mul.tile_meta));
    if (!h->big_folded) {
      // the S*x kernel must not take the >32-row points itself when they are handled by a separate launch
      OK(upload(h, std::vector<int2>(pl.num_ctas, make_int2(0, 0)), &h->v2_mul.cta_big));
    }
    h->v2_smem = pl.v2_smem;
    h->mul_smem = pl.mul_smem;
    h->eval_v2_smem = pl.eval_smem;
    h->diag_v2_smem = pl.diag_smem;
    h->diag_v2_replicas = pl.diag_replicas;
  }
  if (h->xs) {
    const XsPattern& xp = pl.xp;
    XsView& x = h->xsv;
    x.C = C;
    x.num_blocks = static_cast<int>(xp.blk_row.size());
    OK(upload(h, xp.blk_row, &x.blk_row));
    OK(upload(h, xp.blk_col, &x.blk_col));
    OK(upload(h, xp.pair_ptr, &x.pair_ptr));
    OK(upload(h, xp.pairs, &x.pairs));
    OK(upload(h, xp.cols, &x.cols));
    OK(upload(h, xp.col_ptr, &x.col_ptr));
    OK(upload(h, pl.xs_steps, &x.steps));
    OK(upload(h, pl.xs_warp_step, &x.warp_step));
    OK(dev_alloc(h, &x.S, 81 * static_cast<size_t>(x.num_blocks)));
    OK(dev_alloc(h, &x.T, 9 * static_cast<size_t>(xp.off_blocks)));
    OK(upload(h, pl.xs_order, &h->d_xs_order));
    h->num_xs_long = pl.num_xs_long;
    h->num_xs_short = x.num_blocks - pl.num_xs_long;
    h->xs_grid = pl.xs_grid;
    h->xs_pcg = pl.xs_pcg;
    if (h->xs_pcg) {
      XsPcgArgs& a = h->xpa;
      a.v = x;
      OK(upload(h, pl.xs_pcg_cta, &a.cta));
      OK(upload(h, pl.xs_pcg_warp_step, &a.warp_step));
      OK(upload(h, pl.xs_pcg_fptr, &a.fptr));
      OK(upload(h, pl.xs_pcg_fcol, &a.fcol));
      OK(upload(h, pl.xs_pcg_cols, &a.v.cols));   // the kernel's blocks address their columns CTA-locally
      a.max_blocks = pl.xs_pcg_max_blocks;
      a.max_cams = pl.xs_pcg_max_cams;
      a.max_foreign = pl.xs_pcg_max_foreign;
      a.max_steps = pl.xs_pcg_max_cta_steps;
      a.stage_slots = pl.xs_pcg_stage_slots;
      OK(dev_alloc(h, &a.p[1], nc));   // the second p buffer; the first is d_p
      OK(dev_alloc(h, &a.red, static_cast<size_t>(prop.multiProcessorCount) * 4));
      h->xs_pcg_smem = pl.xs_pcg_smem;
#ifdef B200_DEV_KNOBS
      a.stamps = nullptr;
      if (dev_env("B200_XS_STAMPS") != nullptr) {
        OK(dev_alloc(h, &a.stamps, kXpPhases));
        CU(cudaMemsetAsync(a.stamps, 0, sizeof(long long) * kXpPhases, h->stream));
      }
#endif
    }
  }
  CU(cudaStreamSynchronize(h->stream));
  h->xs_arrays = h->xs;
  // the uploads above are complete: the plan's host copies can move (the row structure also serves
  // b200_set_constant_blocks' check of the rows)
  h->h_cam_idx = std::move(pl.cam_idx);
  h->h_pt_idx = std::move(pl.pt_idx);
  if (world == 1) h->h_pt_ptr = std::move(pl.pt_ptr);

  for (int k = 0; k < K_COUNT; ++k) h->grid_tile[k] = std::max(1, std::min(h->num_tiles, h->sm_count * 4));
  // (from the Huber instantiations, which use the most registers of the trivial and Huber ones; the persistent tile loop
  // is correct at any grid)
  h->grid_tile[K_EVAL_JAC] = tile_grid(h, evaluate_kernel<kLossHuber, true>, tile_smem_bytes<3, 1>());
  h->grid_tile[K_EVAL_COST] = tile_grid(h, evaluate_kernel<kLossHuber, false>, tile_smem_bytes<3, 1>());
  h->grid_tile[K_SQNORM] = tile_grid(h, sqnorm_kernel, tile_smem_bytes<3, 1>());
  h->grid_tile[K_JMUL] = tile_grid(h, jmul_kernel, tile_smem_bytes<1, 1>());
  h->grid_tile[K_JTMUL] = tile_grid(h, jtmul_kernel<false>, tile_smem_bytes<3, 1>());
  h->grid_tile[K_JTJ] = tile_grid(h, jtmul_kernel<true>, tile_smem_bytes<3, 1>());
  h->grid_tile[K_SCHUR_INIT] = tile_grid(h, schur_init_kernel, tile_smem_bytes<9, 3>());
  h->grid_tile[K_SCHUR_MUL] = tile_grid(h, schur_mul_kernel, tile_smem_bytes<3, 3>());
  h->grid_tile[K_DIAG_BLOCKS] = tile_grid(h, diag_blocks_kernel<true>, tile_smem_bytes<1, 1>());
  h->grid_tile[K_BACKSUB] = tile_grid(h, backsub_kernel, tile_smem_bytes<3, 1>());
  h->grid_tile[K_MODEL_COST] = tile_grid(h, model_cost_kernel, tile_smem_bytes<1, 1>());
  h->grid_tile[K_DOGLEG_GRAM] = tile_grid(h, dogleg_gram_kernel, tile_smem_bytes<1, 1>());
  {
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cg_vector_kernel, kCgThreads, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
    const int nblocks = (C + kCgCamsPerCta - 1) / kCgCamsPerCta;
    h->cg_grid = std::max(1, std::min(nblocks, per_sm * h->sm_count));
  }
  OK(dev_alloc(h, &h->d_red, static_cast<size_t>(h->cg_grid) * 4));
  OK(dev_alloc(h, &h->d_seed_pq, static_cast<size_t>(h->cg_grid)));
  const int num_pq_parts = std::max(prop.multiProcessorCount, h->xs_grid);   // v4 or explicit-S product CTAs
  OK(dev_alloc(h, &h->d_pq_parts, static_cast<size_t>(num_pq_parts)));
  CU(cudaMemsetAsync(h->d_seed_pq, 0, sizeof(double) * h->cg_grid, h->stream));
  CU(cudaMemsetAsync(h->d_pq_parts, 0, sizeof(double) * num_pq_parts, h->stream));

  if (h->world > 1) {
#ifdef B200_WITH_NCCL
    if (desc->nccl_unique_id == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "world_size > 1 needs nccl_unique_id");
    if (!load_nccl()) return fail(B200_ERR_NCCL, "cannot load libnccl.so.2: %s", dlerror());
    ncclUniqueId id;
    std::memcpy(&id, desc->nccl_unique_id, 128);
    ncclResult_t r = g_nccl.CommInitRank(&h->comm, h->world, id, h->rank);
    if (r != ncclSuccess) return fail(B200_ERR_NCCL, "ncclCommInitRank: %s", g_nccl.GetErrorString(r));
    if (h->world <= kMaxXchgRanks && !h->knobs.no_peer_exchange) {
      // Peer exchange buffers: allocated with cudaMalloc, exported with CUDA IPC, the handles all-gathered through the NCCL
      // communicator (the only plumbing the ranks share), every peer's buffer mapped into this process.  Any failure
      // (no P2P path, IPC unavailable in the launch mode) leaves the NCCL all-reduce in place -- decided jointly.
      OK(dev_alloc(h, &h->d_xchg, 2 * static_cast<size_t>(h->world) * (nc + 1)));
      CU(cudaMemsetAsync(h->d_xchg, 0, sizeof(uint4) * 2 * h->world * (nc + 1), h->stream));   // epoch 0 is never used
      unsigned char* d_handles = nullptr;
      CU(cudaMalloc(reinterpret_cast<void**>(&d_handles), static_cast<size_t>(h->world) * 64));
      std::vector<unsigned char> hh(static_cast<size_t>(h->world) * 64, 0);
      cudaIpcMemHandle_t mine;
      bool ok = cudaIpcGetMemHandle(&mine, h->d_xchg) == cudaSuccess;
      if (!ok) cudaGetLastError();
      static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
      std::memcpy(hh.data() + 64 * h->rank, &mine, 64);
      CU(cudaMemcpyAsync(d_handles + 64 * h->rank, hh.data() + 64 * h->rank, 64, cudaMemcpyHostToDevice, h->stream));
      r = g_nccl.AllGather(d_handles + 64 * h->rank, d_handles, 64, ncclChar, h->comm, h->stream);
      if (r != ncclSuccess) return fail(B200_ERR_NCCL, "ncclAllGather: %s", g_nccl.GetErrorString(r));
      CU(cudaMemcpyAsync(hh.data(), d_handles, hh.size(), cudaMemcpyDeviceToHost, h->stream));
      CU(cudaStreamSynchronize(h->stream));
      h->xpeers.world = h->world;
      h->xpeers.rank = h->rank;
      for (int p = 0; p < h->world && ok; ++p) {
        if (p == h->rank) {
          h->xpeers.buf[p] = h->d_xchg;
          continue;
        }
        cudaIpcMemHandle_t theirs;
        std::memcpy(&theirs, hh.data() + 64 * p, 64);
        void* pb = nullptr;
        if (cudaIpcOpenMemHandle(&pb, theirs, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
          cudaGetLastError();
          ok = false;
          break;
        }
        h->xchg_opened[p] = pb;
        h->xpeers.buf[p] = static_cast<uint4*>(pb);
      }
      // all ranks or none
      double flag = ok ? 1.0 : 0.0;
      CU(cudaMemcpyAsync(h->d_scalars + 4, &flag, sizeof(double), cudaMemcpyHostToDevice, h->stream));
      r = g_nccl.AllReduce(h->d_scalars + 4, h->d_scalars + 4, 1, ncclDouble, ncclMin, h->comm, h->stream);
      if (r != ncclSuccess) return fail(B200_ERR_NCCL, "ncclAllReduce: %s", g_nccl.GetErrorString(r));
      CU(cudaMemcpyAsync(&flag, h->d_scalars + 4, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
      CU(cudaStreamSynchronize(h->stream));
      cudaFree(d_handles);
      h->xchg_ok = flag == 1.0;
      if (getenv("B200_VERBOSE") != nullptr)
        fprintf(stderr, "[b200ba] rank %d/%d: peer exchange over NVLink %s\n", h->rank, h->world, h->xchg_ok ? "enabled" : "unavailable (NCCL all-reduce per CG iteration)");
    }
#else
    return fail(B200_ERR_UNSUPPORTED, "built without NCCL");
#endif
  }
  return B200_OK;
}

void b200_destroy(b200_handle* h) {
  if (h == nullptr) return;
  cudaSetDevice(h->device);
  if (h->stream != nullptr) cudaStreamSynchronize(h->stream);
#ifdef B200_WITH_NCCL
  if (h->comm != nullptr && g_nccl.ok) g_nccl.CommDestroy(h->comm);
#endif
  for (void* p : h->xchg_opened)
    if (p != nullptr) cudaIpcCloseMemHandle(p);
  for (void* p : h->allocs) cudaFree(p);
  if (h->h_scalars) cudaFreeHost(h->h_scalars);
  if (h->cusolver != nullptr && g_cusolver.ok) g_cusolver.Destroy(h->cusolver);
  if (h->h_cg) cudaFreeHost(h->h_cg);
  for (cudaEvent_t e : h->ev_cg)
    if (e != nullptr) cudaEventDestroy(e);
  if (h->h_fail) cudaFreeHost(h->h_fail);
  for (auto& ep : h->pending) {
    cudaEventDestroy(ep.a);
    cudaEventDestroy(ep.b);
  }
  for (auto e : h->event_pool) cudaEventDestroy(e);
  if (h->stream2 != nullptr) { cudaStreamSynchronize(h->stream2); cudaStreamDestroy(h->stream2); }
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  if (h->ev_join) cudaEventDestroy(h->ev_join);
  if (h->own_stream && h->stream != nullptr) cudaStreamDestroy(h->stream);
  delete h;
}

int b200_num_parameters(const b200_handle* h) { return h->np; }
int64_t b200_num_residuals(const b200_handle* h) { return 2 * static_cast<int64_t>(h->N); }

int b200_synchronize(b200_handle* h) {
  CU(cudaStreamSynchronize(h->stream));
  return B200_OK;
}

// ------------------------------------------------------------------------------------------------ Evaluator
int b200_evaluate(b200_handle* h, const double* state, double* cost, double* residuals, double* gradient,
                  int want_jacobian) {
  if (h == nullptr || state == nullptr || cost == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(h->device));
  OK(up_params(h, h->d_state, state));
  // an evaluation that asks for residuals overwrites d_residuals: they are the resident residuals again only if it succeeds
  if (residuals != nullptr) h->residuals_resident = false;
  OK(evaluate_dev(h, h->d_state, residuals != nullptr ? h->d_residuals : nullptr,
                  gradient != nullptr ? h->d_gradient : nullptr, want_jacobian != 0, nullptr, cost));
  if (residuals != nullptr) {
    OK(down_rows(h, residuals, h->d_residuals));
    h->residuals_resident = true;  // the copy in HBM stays valid until the next evaluation that asks for residuals
  }
  if (gradient != nullptr) OK(down_params(h, gradient, h->d_gradient));
  return B200_OK;
}

int b200_set_apply_loss_function(b200_handle* h, int apply) {
  if (h == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
  h->apply_loss = apply != 0;
  return B200_OK;
}

namespace {
// A loss object as the kernels read it (loss.cuh LossEntry), with the checks of its constructor; false if it is refused.
bool make_loss_entry(const b200_loss& l, LossEntry* e) {
  const double a = l.a, b = l.b;
  *e = LossEntry{};
  e->type = l.type;
  e->scale = l.scale;
  if (!std::isfinite(l.scale) || l.scale <= 0.0) return false;
  switch (l.type) {
    case B200_LOSS_TRIVIAL:
      return true;
    case B200_LOSS_TOLERANT:
      if (!std::isfinite(a) || !std::isfinite(b) || a < 0.0 || b <= 0.0) return false;
      e->p = a;
      e->q = b;
      e->r = b * std::log(1.0 + std::exp(-a / b));
      return true;
    case B200_LOSS_HUBER: case B200_LOSS_SOFT_L_ONE: case B200_LOSS_CAUCHY: case B200_LOSS_ARCTAN: case B200_LOSS_TUKEY:
      if (!std::isfinite(a) || a <= 0.0) return false;
      e->p = a;
      e->q = l.type == B200_LOSS_ARCTAN ? 1.0 / (a * a) : a * a;
      e->r = 1.0 / (a * a);
      return true;
    default:
      return false;
  }
}
}  // namespace

int b200_set_loss_functions(b200_handle* h, const b200_loss* losses, int num_losses, const int32_t* row_loss) {
  if (h == nullptr || losses == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  if (num_losses < 1) return fail(B200_ERR_INVALID_ARGUMENT, "num_losses %d < 1", num_losses);
  if (row_loss == nullptr && num_losses != 1) return fail(B200_ERR_INVALID_ARGUMENT, "row_loss == NULL needs one loss, not %d", num_losses);
  std::vector<LossEntry> table(num_losses);
  for (int k = 0; k < num_losses; ++k)
    if (!make_loss_entry(losses[k], &table[k]))
      return fail(B200_ERR_INVALID_ARGUMENT, "loss %d: type %d, a %g, b %g, scale %g refused", k, losses[k].type, losses[k].a,
                  losses[k].b, losses[k].scale);
  if (row_loss != nullptr)
    for (int i = 0; i < h->N; ++i)
      if (row_loss[i] < 0 || row_loss[i] >= num_losses)
        return fail(B200_ERR_INVALID_ARGUMENT, "row %d: loss index %d outside [0, %d)", i, row_loss[i], num_losses);
  CU(cudaSetDevice(h->device));
  const bool rows = num_losses > 1;   // one loss object, indexed or not, is every row's: no per-row array
  if (rows) {
    std::vector<int> internal(h->N);
    for (int i = 0; i < h->N; ++i) internal[i] = row_loss[h->permuted ? h->h_row_perm[i] : i];
    if (h->d_row_loss == nullptr) OK(dev_alloc(h, &h->d_row_loss, h->N));
    if (h->loss_table_cap < table.size()) {
      dev_free(h, h->d_loss_table);
      OK(dev_alloc(h, &h->d_loss_table, table.size()));
      h->loss_table_cap = table.size();
    }
    CU(cudaMemcpyAsync(h->d_row_loss, internal.data(), sizeof(int) * internal.size(), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_loss_table, table.data(), sizeof(LossEntry) * table.size(), cudaMemcpyHostToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));
  }
  const LossEntry& one = table[0];
  h->loss_rows = rows;
  h->loss_one = one;
  if (rows || one.scale != 1.0) h->loss_cls = kLossGeneral;
  else h->loss_cls = one.type == B200_LOSS_TRIVIAL ? kLossTrivial : one.type == B200_LOSS_HUBER ? kLossHuber : kLossGeneral;
  h->residuals_resident = false;   // they were corrected by the previous losses
  return B200_OK;
}

int b200_set_constant_blocks(b200_handle* h, const uint8_t* camera_constant, const uint8_t* point_constant) {
  if (h == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
  std::vector<uint8_t> cam, pts;
  if (camera_constant != nullptr) cam.assign(camera_constant, camera_constant + h->C);
  if (point_constant != nullptr) pts.assign(point_constant, point_constant + h->P);
  return set_fixed(h, std::move(cam), std::move(pts), h->set_cam_mask, h->set_pt_mask);
}

int b200_set_subset_manifolds(b200_handle* h, const uint16_t* camera_constant_coordinates, const uint8_t* point_constant_coordinates) {
  if (h == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
  std::vector<uint16_t> cam;
  std::vector<uint8_t> pts;
  if (camera_constant_coordinates != nullptr) {
    cam.assign(camera_constant_coordinates, camera_constant_coordinates + h->C);
    for (int k = 0; k < h->C; ++k)
      if (cam[k] >> 9 != 0) return fail(B200_ERR_INVALID_ARGUMENT, "camera %d: mask 0x%x has bits above 8 (9 coordinates)", k, cam[k]);
  }
  if (point_constant_coordinates != nullptr) {
    pts.assign(point_constant_coordinates, point_constant_coordinates + h->P);
    for (int k = 0; k < h->P; ++k)
      if (pts[k] >> 3 != 0) return fail(B200_ERR_INVALID_ARGUMENT, "point %d: mask 0x%x has bits above 2 (3 coordinates)", k, pts[k]);
  }
  return set_fixed(h, h->set_cam_const, h->set_pt_const, std::move(cam), std::move(pts));
}

int b200_plus(b200_handle* h, const double* x, const double* delta, double* x_plus_delta) {
  if (h == nullptr || x == nullptr || delta == nullptr || x_plus_delta == nullptr)
    return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  const uint8_t* fx = h->fixed_any ? h->h_fixed.data() : nullptr;
  // Euclidean blocks: program.cc:114-142; constant blocks are not in the reduced x, and SubsetManifold::Plus returns x on
  // the coordinates it holds (manifold.cc:154-166)
  for (int i = 0; i < h->np; ++i)
    x_plus_delta[i] = fx != nullptr && fx[i] != 0 ? x[i] : x[i] + delta[i];
  return B200_OK;
}

// ------------------------------------------------------------------------------------------------ SparseMatrix
int b200_jacobian_squared_column_norm(b200_handle* h, double* x) {
  if (h == nullptr || x == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(h->device));
  OK(sqnorm_dev(h, h->d_vp0));
  return down_params(h, x, h->d_vp0);
}

int b200_jacobian_scale_columns(b200_handle* h, const double* scale) {
  if (h == nullptr || scale == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(h->device));
  OK(up_params(h, h->d_vp0, scale));
  OK(scale_dev(h, h->d_vp0));
  CU(cudaStreamSynchronize(h->stream));
  return B200_OK;
}

int b200_jacobian_right_multiply(b200_handle* h, const double* x, double* y) {
  if (h == nullptr || x == nullptr || y == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(h->device));
  OK(up_params(h, h->d_vp0, x));
  OK(up_rows(h, h->d_vr0, y));
  OK(launch(h, K_JMUL, [&] {
    jmul_kernel<<<h->grid_tile[K_JMUL], kTile, tile_smem_bytes<1, 1>(), h->stream>>>(h->view, h->d_vp0, h->d_vr0);
  }));
  return down_rows(h, y, h->d_vr0);
}

int b200_model_cost_change(b200_handle* h, const double* step, double* model_cost_change) {
  if (h == nullptr || step == nullptr || model_cost_change == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  if (!h->residuals_resident) return fail(B200_ERR_INVALID_ARGUMENT, "needs the residuals of a previous b200_evaluate");
  CU(cudaSetDevice(h->device));
  OK(up_params(h, h->d_vp0, step));
  return model_cost_change_dev(h, h->d_vp0, model_cost_change);
}

int b200_jacobian_left_multiply(b200_handle* h, const double* x, double* y) {
  if (h == nullptr || x == nullptr || y == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(h->device));
  OK(up_rows(h, h->d_vr0, x));
  // camera part accumulates across ranks: only rank 0 carries the incoming y there
  OK(up_params(h, h->d_vp0, y));
  if (h->rank != 0) CU(cudaMemsetAsync(h->d_vp0 + 3 * static_cast<size_t>(h->P), 0, sizeof(double) * 9 * h->C, h->stream));
  OK(launch(h, K_JTMUL, [&] {
    jtmul_kernel<false><<<h->grid_tile[K_JTMUL], kTile, tile_smem_bytes<3, 1>(), h->stream>>>(h->view, h->d_vr0, nullptr, h->d_vp0);
  }));
  OK(allreduce_sum(h, h->d_vp0 + 3 * static_cast<size_t>(h->P), 9 * static_cast<size_t>(h->C)));
  return down_params(h, y, h->d_vp0);
}

int b200_partitioned_multiply(b200_handle* h, int op, const double* x, double* y) {
  if (h == nullptr || x == nullptr || y == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  if (op < B200_PMV_RIGHT_E || op > B200_PMV_LEFT_F) return fail(B200_ERR_INVALID_ARGUMENT, "unknown partitioned product %d", op);
  if (h->world > 1) return fail(B200_ERR_UNSUPPORTED, "partitioned products are single-GPU");
  CU(cudaSetDevice(h->device));
  const size_t nE = 3 * static_cast<size_t>(h->P), nF = 9 * static_cast<size_t>(h->C);
  double* d_par = h->d_vp0;   // [points | cameras] scratch
  double* d_row = h->d_vr0;   // [2N] scratch
  // point-sized vectors cross the boundary in the caller's point order, row-sized ones in its row order
  auto up_e = [&](const double* host) -> int {
    if (!h->permuted) return h2d(h, d_par, host, sizeof(double) * nE);
    OK(h2d(h, h->d_stage_p, host, sizeof(double) * nE));
    return permute_blocks(h, true, h->P, 3, h->d_pt_perm, h->d_stage_p, d_par);
  };
  auto down_e = [&](double* host) -> int {
    if (!h->permuted) return d2h(h, host, d_par, sizeof(double) * nE);
    OK(permute_blocks(h, false, h->P, 3, h->d_pt_perm, d_par, h->d_stage_p));
    return d2h(h, host, h->d_stage_p, sizeof(double) * nE);
  };
  switch (op) {
    case B200_PMV_RIGHT_E:
      OK(up_e(x));
      OK(up_rows(h, d_row, y));
      OK(launch(h, K_PMV_RIGHT_E, [&] { pmv_right_e_kernel<<<flat_grid(h, h->N, 256), 256, 0, h->stream>>>(h->view, d_par, d_row); }));
      return down_rows(h, y, d_row);
    case B200_PMV_RIGHT_F:
      OK(h2d(h, d_par + nE, x, sizeof(double) * nF));
      OK(up_rows(h, d_row, y));
      OK(launch(h, K_PMV_RIGHT_F, [&] { pmv_right_f_kernel<<<flat_grid(h, h->N, 256), 256, 0, h->stream>>>(h->view, d_par + nE, d_row); }));
      return down_rows(h, y, d_row);
    case B200_PMV_LEFT_E:
      OK(up_rows(h, d_row, x));
      OK(up_e(y));
      OK(launch(h, K_PMV_LEFT_E, [&] { pmv_left_e_kernel<<<flat_grid(h, h->P, 256), 256, 0, h->stream>>>(h->view, d_row, d_par); }));
      return down_e(y);
    default:
      OK(up_rows(h, d_row, x));
      OK(h2d(h, d_par + nE, y, sizeof(double) * nF));
      if (h->diag == DiagPass::CamMajor)
        OK(launch(h, K_PMV_LEFT_F, [&] {
          pmv_left_f_kernel<<<std::max(1, std::min((h->num_cam_items + 7) / 8, h->sm_count * 8)), 256, 0, h->stream>>>(
              h->view, h->num_cam_items, h->d_cam_items, h->d_cam_rows, d_row, d_par + nE);
        }));
      else
        OK(launch(h, K_PMV_LEFT_F, [&] { pmv_left_f_rows_kernel<<<flat_grid(h, h->N, 256), 256, 0, h->stream>>>(h->view, d_row, d_par + nE); }));
      return d2h(h, y, d_par + nE, sizeof(double) * nF);
  }
}

int b200_jtj_multiply(b200_handle* h, const double* x, const double* D, double* y) {
  if (h == nullptr || x == nullptr || y == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(h->device));
  OK(up_params(h, h->d_vp0, x));
  if (D != nullptr) OK(up_params(h, h->d_D, D));
  const double* dD = D != nullptr ? h->d_D : nullptr;
  const size_t off = 3 * static_cast<size_t>(h->P);
  const double* seedD = (dD != nullptr && h->rank == 0) ? dD + off : nullptr;
  const int nc = 9 * h->C;
  OK(huge_zero(h, h->d_vp1));  // point entries of huge points are accumulated slice by slice
  // The camera part of y is seeded with D_c^2 x_c when the product adds into it; the v4 kernel takes the CTA's
  // 33..kTile-row points itself and only the slices of >kTile-row points need a second launch.
  if (h->mul == MulFamily::Tile || h->v2.direct) OK(diag_sq_mul_dev(h, seedD, h->d_vp0 + off, h->d_vp1 + off, nullptr));
  const ProblemView* rest = &h->view_big;   // CTA tiles beside the warp-tile kernel
  if (is_v4(h->mul)) {
    V2View jv = h->v2_mul;
    jv.cta_big = h->d_cta_big;
    OK(launch(h, K_JTJ, [&] {
      if (h->mul == MulFamily::V4Owned) jtj_v4_kernel<true><<<h->v2.num_ctas, 32 * h->v2_mul.warps, h->mul_smem, h->stream>>>(jv, h->d_vp0, dD, h->d_vp1);
      else jtj_v4_kernel<false><<<h->v2.num_ctas, 32 * h->v2_mul.warps, h->mul_smem, h->stream>>>(jv, h->d_vp0, dD, h->d_vp1);
    }));
    rest = &h->view_chunks;
  } else if (h->mul == MulFamily::V3) {
    OK(launch(h, K_JTJ, [&] {
      jtj_v2_kernel<<<h->v2.num_ctas, 32 * h->v2.warps, h->v2_smem, h->stream>>>(h->v2, h->d_vp0, dD, h->d_vp1);
    }));
    if (!h->v2.direct)
      OK(launch(h, K_CAM_REDUCE, [&] {
        cam_reduce_kernel<<<(nc + 63) / 64, 256, h->v2.num_ctas * sizeof(int2), h->stream>>>(
            nc, h->v2.num_ctas, h->v2.cta_cam, h->v2.partials, 9 * h->v2.max_cam_span, seedD, h->d_vp0 + off, h->d_vp1 + off, 0, nullptr);
      }));
  } else {
    OK(launch(h, K_JTJ, [&] {
      jtmul_kernel<true><<<h->grid_tile[K_JTJ], kTile, tile_smem_bytes<3, 1>(), h->stream>>>(h->view, h->d_vp0, dD, h->d_vp1);
    }));
  }
  if (rest->num_tiles > 0)
    OK(launch(h, K_JTJ, [&] {
      jtmul_kernel<true><<<std::min(rest->num_tiles, h->sm_count * 4), kTile, tile_smem_bytes<3, 1>(), h->stream>>>(*rest, h->d_vp0, dD, h->d_vp1);
    }, false));
  OK(allreduce_sum(h, h->d_vp1 + off, 9 * static_cast<size_t>(h->C)));
  return down_params(h, y, h->d_vp1);
}

int b200_jacobian_get_values(b200_handle* h, double* values) {
  if (h == nullptr || values == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(h->device));
  const size_t n = static_cast<size_t>(h->N);
  if (!h->permuted) return d2h(h, values, h->d_values, sizeof(double) * 24 * n);
  // cold path (dumps, CPU consumers of the Jacobian): rows back into the caller's order through a temporary
  double* tmp = nullptr;
  CU(cudaMalloc(reinterpret_cast<void**>(&tmp), sizeof(double) * 24 * n));
  int rc = permute_blocks(h, false, n, 6, h->d_row_perm, h->d_values, tmp);
  if (rc == B200_OK) rc = permute_blocks(h, false, n, 18, h->d_row_perm, h->d_values + 6 * n, tmp + 6 * n);
  if (rc == B200_OK) rc = d2h(h, values, tmp, sizeof(double) * 24 * n);
  cudaFree(tmp);
  return rc;
}
int b200_jacobian_set_values(b200_handle* h, const double* values) {
  if (h == nullptr || values == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(h->device));
  jacobian_written(h);
  const size_t n = static_cast<size_t>(h->N);
  if (!h->permuted) {
    OK(h2d(h, h->d_values, values, sizeof(double) * 24 * n));
    OK(fixed_mask_dev(h));
    CU(cudaStreamSynchronize(h->stream));
    return B200_OK;
  }
  double* tmp = nullptr;
  CU(cudaMalloc(reinterpret_cast<void**>(&tmp), sizeof(double) * 24 * n));
  int rc = h2d(h, tmp, values, sizeof(double) * 24 * n);
  if (rc == B200_OK) rc = permute_blocks(h, true, n, 6, h->d_row_perm, tmp, h->d_values);
  if (rc == B200_OK) rc = permute_blocks(h, true, n, 18, h->d_row_perm, tmp + 6 * n, h->d_values + 6 * n);
  if (rc == B200_OK) rc = fixed_mask_dev(h);
  cudaStreamSynchronize(h->stream);
  cudaFree(tmp);
  return rc;
}

// ------------------------------------------------------------------------------------------------ LinearSolver
int b200_schur_solve(b200_handle* h, const double* b, const double* D, const b200_solver_options* opts, double* x,
                     b200_solver_summary* summary) {
  if (h == nullptr || opts == nullptr || x == nullptr || summary == nullptr)
    return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  return solve_from_host(h, B200_ITERATIVE_SCHUR, b, D, opts, x, summary);
}

int b200_dense_schur_solve(b200_handle* h, const double* b, const double* D, double* x, b200_solver_summary* summary) {
  if (h == nullptr || x == nullptr || summary == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  return solve_from_host(h, B200_DENSE_SCHUR, b, D, nullptr, x, summary);
}

int b200_sparse_schur_solve(b200_handle* h, const double* b, const double* D, double* x, b200_solver_summary* summary) {
  if (h == nullptr || x == nullptr || summary == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  return solve_from_host(h, B200_SPARSE_SCHUR, b, D, nullptr, x, summary);
}

int b200_set_exact_solve_options(b200_handle* h, int use_mixed_precision_solves, int max_num_refinement_iterations) {
  if (h == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
  if (use_mixed_precision_solves != 0 && use_mixed_precision_solves != 1)
    return fail(B200_ERR_INVALID_ARGUMENT, "use_mixed_precision_solves must be 0 or 1, not %d", use_mixed_precision_solves);
  if (max_num_refinement_iterations < 0)
    return fail(B200_ERR_INVALID_ARGUMENT, "max_num_refinement_iterations must be >= 0, not %d", max_num_refinement_iterations);
  h->mixed = use_mixed_precision_solves != 0;
  h->refine = max_num_refinement_iterations;
  return B200_OK;
}

int b200_set_linear_solver_ordering_type(b200_handle* h, int type) {
  if (h == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
  if (type != B200_AMD && type != B200_NESDIS)
    return fail(B200_ERR_INVALID_ARGUMENT, "linear_solver_ordering_type must be B200_AMD or B200_NESDIS, not %d", type);
  if (type == h->ordering) return B200_OK;
  CU(cudaSetDevice(h->device));
  sparse_drop(h);
  h->ordering = type;
  return B200_OK;
}

// ------------------------------------------------------------------------------------------------ Covariance
void b200_covariance_options_default(b200_covariance_options* o) {
  o->algorithm = B200_SPARSE_SCHUR;
  o->min_reciprocal_condition_number = 1e-14;   // covariance.h:294
  o->apply_loss_function = 1;                   // covariance.h:339
}

int b200_covariance_compute(b200_handle* h, const double* state, const b200_covariance_options* o, int* valid) {
  if (h == nullptr || state == nullptr || o == nullptr || valid == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  if (o->algorithm == B200_ITERATIVE_SCHUR)
    return fail(B200_ERR_UNSUPPORTED, "covariance needs an exact factorisation: B200_SPARSE_SCHUR or B200_DENSE_SCHUR");
  if (o->algorithm != B200_SPARSE_SCHUR && o->algorithm != B200_DENSE_SCHUR)
    return fail(B200_ERR_INVALID_ARGUMENT, "covariance algorithm must be B200_SPARSE_SCHUR or B200_DENSE_SCHUR, not %d", o->algorithm);
  if (!std::isfinite(o->min_reciprocal_condition_number) || o->min_reciprocal_condition_number < 0.0)
    return fail(B200_ERR_INVALID_ARGUMENT, "min_reciprocal_condition_number %g", o->min_reciprocal_condition_number);
  if (h->world > 1) return fail(B200_ERR_UNSUPPORTED, "covariance needs the explicit Schur complement, which is single-GPU");
  *valid = 0;
  CU(cudaSetDevice(h->device));
  h->cov_valid = false;   // a new compute replaces the snapshot, also when it fails
  ApplyLossGuard guard{h, h->apply_loss};
  h->apply_loss = o->apply_loss_function != 0;
  OK(up_params(h, h->d_state, state));
  h->residuals_resident = false;
  double cost = 0.0;
  OK(evaluate_dev(h, h->d_state, h->d_residuals, nullptr, true, nullptr, &cost));
  h->residuals_resident = true;
  if (h->d_cov_min == nullptr) OK(dev_alloc(h, &h->d_cov_min, 2));
  if (h->d_cov_pts == nullptr) OK(dev_alloc(h, &h->d_cov_pts, 9 * static_cast<size_t>(h->P)));
  const double inf = std::numeric_limits<double>::infinity();
  CU(cudaMemcpyAsync(h->d_cov_min, &inf, sizeof(double), cudaMemcpyHostToDevice, h->stream));
  const bool dense = o->algorithm == B200_DENSE_SCHUR;
  bool factored = false;
  int rc = dense ? cov_dense_dev(h, &factored) : cov_sparse_dev(h, &factored);
  // the Schur initialisation, S and the factor now hold the covariance's: the next solve rebuilds them
  jacobian_written(h);
  h->schur_ready = false;
  h->xs_diag_ready = false;
  OK(rc);
  if (!factored) {
    if (getenv("B200_VERBOSE") != nullptr) fprintf(stderr, "[b200ba] covariance: S is not positive definite\n");
    return B200_OK;
  }
  const int* perm = h->permuted ? h->d_pt_perm : nullptr;
  OK(launch(h, K_COV_POINTS, [&] {
    const int g = std::max(1, std::min((h->P + 7) / 8, h->sm_count * 16));
    if (dense) covariance_point_kernel<true><<<g, 256, 0, h->stream>>>(h->view, cov_access<true>(h), h->d_fixed, perm, h->d_cov_pts, h->d_cov_min);
    else covariance_point_kernel<false><<<g, 256, 0, h->stream>>>(h->view, cov_access<false>(h), h->d_fixed, perm, h->d_cov_pts, h->d_cov_min);
  }));
  unsigned long long bits = 0;
  CU(cudaMemcpyAsync(&bits, h->d_cov_min, sizeof(bits), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  double rcond = 0.0;
  std::memcpy(&rcond, &bits, sizeof(rcond));
  if (getenv("B200_VERBOSE") != nullptr)
    fprintf(stderr, "[b200ba] covariance: %s, selected inversion %.3g flops, min pivot / diagonal %.3e (threshold %.3e)\n",
            dense ? "dense potri" : "sparse", dense ? 0.0 : h->sp_selinv_flops, rcond, o->min_reciprocal_condition_number);
  if (!(rcond >= o->min_reciprocal_condition_number)) return B200_OK;
  h->cov_alg = o->algorithm;
  h->cov_cam_mask.assign(static_cast<size_t>(h->C), 0);
  if (h->fixed_any)
    for (int c = 0; c < h->C; ++c)
      for (int j = 0; j < 9; ++j)
        h->cov_cam_mask[c] |= (h->h_fixed[3 * static_cast<size_t>(h->P) + 9 * static_cast<size_t>(c) + j] != 0) << j;
  h->cov_valid = true;
  *valid = 1;
  return B200_OK;
}

int b200_covariance_cameras(b200_handle* h, int num_pairs, const int32_t* pairs, double* out) {
  if (h == nullptr || num_pairs < 0 || (num_pairs > 0 && (pairs == nullptr || out == nullptr)))
    return fail(B200_ERR_INVALID_ARGUMENT, "null argument or num_pairs < 0");
  if (!h->cov_valid) return fail(B200_ERR_INVALID_ARGUMENT, "no valid covariance: b200_covariance_compute first (CHECK(is_valid_))");
  const bool dense = h->cov_alg == B200_DENSE_SCHUR;
  std::vector<int4> desc(static_cast<size_t>(num_pairs));
  for (int q = 0; q < num_pairs; ++q) {
    const int i = pairs[2 * q], j = pairs[2 * q + 1];
    if (i < 0 || i >= h->C || j < 0 || j >= h->C)
      return fail(B200_ERR_INVALID_ARGUMENT, "pair %d: cameras (%d, %d) outside [0, %d)", q, i, j, h->C);
    int b = -1;
    if (!dense) {
      const int a = std::min(i, j), c = std::max(i, j);
      auto first = h->cov_blk_col.begin() + h->cov_row_ptr[a], last = h->cov_blk_col.begin() + h->cov_row_ptr[a + 1];
      auto it = std::lower_bound(first, last, c);
      if (it == last || *it != c)
        return fail(B200_ERR_INVALID_ARGUMENT, "pair %d: cameras (%d, %d) share no point, so SPARSE_SCHUR does not compute their block "
                    "(DENSE_SCHUR does)", q, i, j);
      b = static_cast<int>(it - h->cov_blk_col.begin());
    }
    desc[q] = make_int4(i, j, b, h->cov_cam_mask[i] | h->cov_cam_mask[j] << 9);
  }
  if (num_pairs == 0) return B200_OK;
  CU(cudaSetDevice(h->device));
  if (h->cov_pairs_cap < desc.size()) {
    dev_free(h, h->d_cov_pairs);
    dev_free(h, h->d_cov_out);
    OK(dev_alloc(h, &h->d_cov_pairs, desc.size()));
    OK(dev_alloc(h, &h->d_cov_out, 81 * desc.size()));
    h->cov_pairs_cap = desc.size();
  }
  CU(cudaMemcpyAsync(h->d_cov_pairs, desc.data(), sizeof(int4) * desc.size(), cudaMemcpyHostToDevice, h->stream));
  OK(launch(h, K_COV_GATHER, [&] {
    const int g = flat_grid(h, 81 * desc.size(), 256);
    if (dense) covariance_gather_kernel<true><<<g, 256, 0, h->stream>>>(cov_access<true>(h), num_pairs, h->d_cov_pairs, h->d_cov_out);
    else covariance_gather_kernel<false><<<g, 256, 0, h->stream>>>(cov_access<false>(h), num_pairs, h->d_cov_pairs, h->d_cov_out);
  }));
  CU(cudaMemcpyAsync(out, h->d_cov_out, sizeof(double) * 81 * desc.size(), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  return B200_OK;
}

int b200_covariance_points(b200_handle* h, double* out) {
  if (h == nullptr || out == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  if (!h->cov_valid) return fail(B200_ERR_INVALID_ARGUMENT, "no valid covariance: b200_covariance_compute first (CHECK(is_valid_))");
  CU(cudaSetDevice(h->device));
  CU(cudaMemcpyAsync(out, h->d_cov_pts, sizeof(double) * 9 * static_cast<size_t>(h->P), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  return B200_OK;
}

int b200_schur_init(b200_handle* h, const double* b, const double* D) {
  if (h == nullptr || b == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(h->device));
  OK(up_rows(h, h->d_b, b));
  if (D != nullptr) OK(up_params(h, h->d_D, D));
  OK(schur_init_dev(h, h->d_b, D != nullptr ? h->d_D : nullptr));
  CU(cudaStreamSynchronize(h->stream));
  return B200_OK;
}
int b200_schur_rhs(b200_handle* h, double* rhs) {
  if (h == nullptr || rhs == nullptr || !h->schur_ready) return fail(B200_ERR_INVALID_ARGUMENT, "b200_schur_init first");
  return d2h(h, rhs, h->d_rhs, sizeof(double) * 9 * h->C);
}
int b200_schur_ete_inverse(b200_handle* h, double* out) {
  if (h == nullptr || out == nullptr || !h->schur_ready) return fail(B200_ERR_INVALID_ARGUMENT, "b200_schur_init first");
  std::vector<double> packed(6 * static_cast<size_t>(h->P));
  OK(d2h(h, packed.data(), h->d_ete_inv, sizeof(double) * packed.size()));
  for (int k = 0; k < h->P; ++k) {
    const double* s = &packed[6 * static_cast<size_t>(k)];
    double* o = out + 9 * static_cast<size_t>(h->permuted ? h->h_pt_perm[k] : k);
    o[0] = s[0]; o[1] = s[1]; o[2] = s[2];
    o[3] = s[1]; o[4] = s[3]; o[5] = s[4];
    o[6] = s[2]; o[7] = s[4]; o[8] = s[5];
  }
  return B200_OK;
}
int b200_schur_multiply(b200_handle* h, const double* x, double* y) {
  if (h == nullptr || x == nullptr || y == nullptr || !h->schur_ready) return fail(B200_ERR_INVALID_ARGUMENT, "b200_schur_init first");
  CU(cudaSetDevice(h->device));
  OK(h2d(h, h->d_xr, x, sizeof(double) * 9 * h->C));
  MulOpts mo;
  mo.explicit_s = h->xs;
  OK(schur_mul_dev(h, h->d_xr, h->d_tmp, mo));
  return d2h(h, y, h->d_tmp, sizeof(double) * 9 * h->C);
}
int b200_schur_back_substitute(b200_handle* h, const double* z, double* y) {
  if (h == nullptr || z == nullptr || y == nullptr || !h->schur_ready) return fail(B200_ERR_INVALID_ARGUMENT, "b200_schur_init first");
  CU(cudaSetDevice(h->device));
  OK(h2d(h, h->d_xr, z, sizeof(double) * 9 * h->C));
  OK(back_substitute_dev(h, h->cur_b, h->d_xr, h->d_y));
  if (h->permuted) {
    OK(permute_blocks(h, false, h->P, 3, h->d_pt_perm, h->d_y, h->d_stage_p));
    OK(d2h(h, y, h->d_stage_p, sizeof(double) * 3 * static_cast<size_t>(h->P)));
  } else {
    OK(d2h(h, y, h->d_y, sizeof(double) * 3 * static_cast<size_t>(h->P)));
  }
  std::memcpy(y + 3 * static_cast<size_t>(h->P), z, sizeof(double) * 9 * h->C);
  if (h->fixed_any)
    for (size_t i = 3 * static_cast<size_t>(h->P); i < static_cast<size_t>(h->np); ++i)
      if (h->h_fixed[i] != 0) y[i] = 0.0;
  return B200_OK;
}
int b200_schur_jacobi_update(b200_handle* h, double* blocks, double* inverse) {
  if (h == nullptr || !h->schur_ready) return fail(B200_ERR_INVALID_ARGUMENT, "b200_schur_init first");
  CU(cudaSetDevice(h->device));
  OK(precond_update_dev(h, B200_PRECOND_SCHUR_JACOBI));
  if (blocks != nullptr) OK(d2h(h, blocks, h->d_blocks, sizeof(double) * 81 * static_cast<size_t>(h->C)));
  if (inverse != nullptr) OK(d2h(h, inverse, h->d_minv, sizeof(double) * 81 * static_cast<size_t>(h->C)));
  return B200_OK;
}
int b200_block_jacobi_update(b200_handle* h, double* inverse) {
  if (h == nullptr || !h->schur_ready) return fail(B200_ERR_INVALID_ARGUMENT, "b200_schur_init first");
  CU(cudaSetDevice(h->device));
  OK(precond_update_dev(h, B200_PRECOND_JACOBI));
  if (inverse != nullptr) OK(d2h(h, inverse, h->d_minv, sizeof(double) * 81 * static_cast<size_t>(h->C)));
  return B200_OK;
}

// ------------------------------------------------------------------------------------------------ trust region loop
// `host_boundary` selects whether the vectors cross the bus through the public entry points (adapter behaviour) or stay
// in HBM.
int b200_lm_solve(b200_handle* h, const b200_lm_options* opt, double* state_inout, b200_lm_iteration* trace,
                  int max_records, int* num_records, int host_boundary) {
  if (h == nullptr || opt == nullptr || state_inout == nullptr || trace == nullptr || num_records == nullptr)
    return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  if (opt->trust_region_strategy_type != B200_LEVENBERG_MARQUARDT && opt->trust_region_strategy_type != B200_DOGLEG)
    return fail(B200_ERR_INVALID_ARGUMENT, "unknown trust_region_strategy_type %d", opt->trust_region_strategy_type);
  const bool dogleg = opt->trust_region_strategy_type == B200_DOGLEG;
  if (dogleg && opt->dogleg_type != B200_TRADITIONAL_DOGLEG && opt->dogleg_type != B200_SUBSPACE_DOGLEG)
    return fail(B200_ERR_INVALID_ARGUMENT, "unknown dogleg_type %d", opt->dogleg_type);
  if (dogleg && opt->linear_solver_type == B200_ITERATIVE_SCHUR)   // solver.cc:431-438
    return fail(B200_ERR_INVALID_ARGUMENT,
                "DOGLEG only supports exact factorization based linear solvers. If you want to use an iterative solver "
                "please use LEVENBERG_MARQUARDT as the trust_region_strategy_type");
  if (opt->use_mixed_precision_solves != 0 && opt->linear_solver_type == B200_ITERATIVE_SCHUR)   // solver.cc:298-300
    return fail(B200_ERR_INVALID_ARGUMENT, "use_mixed_precision_solves does not make sense with ITERATIVE_SCHUR");
  // the exact solves of this call (the host-boundary loop's public calls included) use the call's options; the handle's
  // own are restored on every exit
  const bool mixed0 = h->mixed;
  const int refine0 = h->refine, ordering0 = h->ordering;
  OK(b200_set_exact_solve_options(h, opt->use_mixed_precision_solves, opt->max_num_refinement_iterations));
  struct Restore {
    b200_handle* h;
    bool mixed;
    int refine, ordering;
    ~Restore() {
      h->mixed = mixed;
      h->refine = refine;
      b200_set_linear_solver_ordering_type(h, ordering);
    }
  } restore{h, mixed0, refine0, ordering0};
  OK(b200_set_linear_solver_ordering_type(h, opt->linear_solver_ordering_type));
  CU(cudaSetDevice(h->device));
  *num_records = 0;
  auto run = [&](auto side) {
    if (dogleg) return minimize(side, DoglegStrategy(opt), opt, state_inout, trace, max_records, num_records);
    return minimize(side, LmStrategy(opt), opt, state_inout, trace, max_records, num_records);
  };
  return host_boundary ? run(HostSide(h, opt)) : run(DeviceSide(h, opt));
}

// ------------------------------------------------------------------------------------------------ instrumentation
int b200_profile_enable(b200_handle* h, int on) {
  if (h == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
  OK(resolve_events(h));
  h->profiling = on != 0;
  return B200_OK;
}
int b200_stats_reset(b200_handle* h) {
  if (h == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
  OK(resolve_events(h));
  std::memset(h->launches, 0, sizeof(h->launches));
  std::memset(h->ops, 0, sizeof(h->ops));
  std::memset(h->ms, 0, sizeof(h->ms));
  h->h2d_bytes = 0;
  h->d2h_bytes = 0;
  return B200_OK;
}
int b200_stats_get(b200_handle* h, b200_kernel_stat* out, int max_entries, int* num_entries) {
  if (h == nullptr || out == nullptr || num_entries == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  OK(resolve_events(h));
  int n = 0;
  for (int k = 0; k < K_COUNT && n < max_entries; ++k) {
    std::memset(&out[n], 0, sizeof(out[n]));
    std::strncpy(out[n].name, kKernelNames[k], sizeof(out[n].name) - 1);
    out[n].launches = h->launches[k];
    out[n].operations = h->ops[k];
    out[n].device_ms = h->ms[k];
    out[n].bytes_per_operation = h->bytes_per_op[k];
    ++n;
  }
  *num_entries = n;
  return B200_OK;
}
int64_t b200_total_launches(const b200_handle* h) {
  int64_t t = 0;
  for (int k = 0; k < K_COUNT; ++k) t += h->launches[k];
  return t;
}
int b200_transfer_bytes(const b200_handle* h, int64_t* h2d_out, int64_t* d2h_out) {
  if (h == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null handle");
  if (h2d_out) *h2d_out = h->h2d_bytes;
  if (d2h_out) *d2h_out = h->d2h_bytes;
  return B200_OK;
}

}  // extern "C"
