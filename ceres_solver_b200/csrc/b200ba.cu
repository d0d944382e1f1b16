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

using namespace b200;

namespace {

thread_local std::string g_error;
constexpr int kHostThreads = 8;   // host-side vector passes of the host-boundary LM loop (the reference uses its thread pool)
// Share of the L2 the S*x residency plan may fill (b200_create).  On an H100 (50 MB L2) the product got faster up to
// ~24 MB resident and slower again from 32 MB on (DESIGN §3.2).
constexpr double kL2ResidentShare = 0.5;
// Explicit S (explicit_schur.cuh) when the implicit product's stream is at least kXsByteRatio times the bytes of a
// product on the explicit upper triangle (each off-diagonal block read twice), does not fit the L2 residency budget
// (then the implicit product is served from L2 and the assembly cannot pay for itself), and S with its row-pair list
// fits kXsMaxBytes (the assembly time grows with the row pairs, and a solve of few CG iterations cannot repay it).
// Measured on one H100 (DESIGN §3): Ladybug-1723 (ratio 3.3, 40 MB) is faster explicit; ladybug-1723-random (ratio 0.47),
// C16 (stream within the L2 budget) and Venice-1778 (186 MB, 3-10 CG iterations per solve) are faster implicit.
constexpr double kXsByteRatio = 2.0;
constexpr double kXsMaxBytes = 128.0 * (1 << 20);

// Development switches (A/B measurements of kernel variants and tuning knobs) exist only in builds with
// -DB200_DEV_KNOBS; the product library has a single code path per problem class and reads no such variable.
#ifdef B200_DEV_KNOBS
inline const char* dev_env(const char* name) { return getenv(name); }
#else
inline const char* dev_env(const char*) { return nullptr; }
#endif

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

enum KernelId {
  K_EVAL_JAC = 0,
  K_EVAL_COST,
  K_SQNORM,
  K_SCALE,
  K_JMUL,
  K_JTMUL,
  K_JTJ,
  K_SCHUR_INIT,
  K_SCHUR_MUL,
  K_SCHUR_MUL_BIG,
  K_CAM_REDUCE,
  K_DIAG_BLOCKS,
  K_INVERT9,
  K_BACKSUB,
  K_MODEL_COST,
  K_CG_VEC,
  K_LM_VEC,
  K_PMV_RIGHT_E,
  K_PMV_RIGHT_F,
  K_PMV_LEFT_E,
  K_PMV_LEFT_F,
  K_MISC,
  K_COUNT
};
const char* kKernelNames[K_COUNT] = {"evaluate_jacobian", "evaluate_cost", "squared_column_norm", "scale_columns",
                                     "jacobian_multiply", "jacobian_t_multiply", "jtj_multiply", "schur_init",
                                     "schur_multiply", "schur_multiply_big_points", "camera_reduce", "schur_diag_blocks", "invert_9x9", "back_substitute",
                                     "model_cost", "cg_vector", "lm_vector", "pmv_right_e", "pmv_right_f", "pmv_left_e", "pmv_left_f", "misc"};

// cuSOLVER (dense Cholesky of the explicit reduced camera system, SURVEY 8f.1) is bound lazily with dlopen like NCCL: the
// library is only touched by b200_dense_schur_solve, and shares whatever libcusolver.so.11 the process already has.
struct CusolverApi {
  typedef int (*create_t)(void**);
  typedef int (*destroy_t)(void*);
  typedef int (*set_stream_t)(void*, cudaStream_t);
  typedef int (*potrf_bs_t)(void*, int, int, double*, int, int*);
  typedef int (*potrf_t)(void*, int, int, double*, int, double*, int, int*);
  typedef int (*potrs_t)(void*, int, int, int, const double*, int, double*, int, int*);
  create_t Create = nullptr;
  destroy_t Destroy = nullptr;
  set_stream_t SetStream = nullptr;
  potrf_bs_t DpotrfBufferSize = nullptr;
  potrf_t Dpotrf = nullptr;
  potrs_t Dpotrs = nullptr;
  bool ok = false;
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
  double& operator[](size_t i) { return p[i]; }
  size_t size() const { return n; }
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
  int loss_type = 0;
  double loss_a = 1.0;
  bool apply_loss = true;   // EvaluateOptions::apply_loss_function
  int rank = 0, world = 1;
#ifdef B200_WITH_NCCL
  ncclComm_t comm = nullptr;
#endif
  ProblemView view{};
  // structure
  TileDesc* d_tiles = nullptr;
  int *d_cam_idx = nullptr, *d_pt_ptr = nullptr, *d_pt_of_row = nullptr;
  double* d_obs = nullptr;
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
  double *d_stage_p = nullptr, *d_stage_r = nullptr; // boundary staging: [3P+9C], [2N]
  std::vector<int> h_pt_perm;
  bool schur_ready = false;
  bool q_from_init = false;   // d_q3 holds the per-row blocks of the CURRENT implicit-Schur initialisation
  const double* cur_b = nullptr;  // device pointers of the current ISC Init
  const double* cur_D = nullptr;
  // LM state
  double *d_scale = nullptr, *d_sqnorm = nullptr, *d_diagonal = nullptr, *d_lmD = nullptr, *d_step = nullptr,
         *d_cand = nullptr, *d_y = nullptr;
  // pinned host staging for scalars
  double* h_scalars = nullptr;
  CgState* h_cg = nullptr;      // two pinned slots: the host polls one batch behind the launches
  cudaEvent_t ev_cg[2] = {nullptr, nullptr};
  int* h_fail = nullptr;
  // v2 (warp-tile, shared-memory-privatised camera vector) path
  bool v2_ok = false;
  V2View v2{};
  ProblemView view_big{};   // CTA tiles holding only the points with more than 32 rows
  ProblemView view_chunks{};  // ... only the <= kTile-row slices of the points with more than kTile rows
  int num_big_tiles = 0;
  double* d_dense_s = nullptr;   // explicit reduced camera system [9C][9C] (allocated by the first dense solve)
  double* d_dense_work = nullptr;
  int dense_lwork = 0;
  int* d_dense_info = nullptr;
  void* cusolver = nullptr;
  int num_huge = 0;           // points with more than kTile rows (huge_kernels.cuh); their rows appear as chunk tiles
  int* d_huge_pts = nullptr;
  bool big_folded = false;   // S*x handles them inside schur_mul_v3_kernel (no extra launch)
  int2* d_cta_big = nullptr;
  int2* d_cta_big_none = nullptr;
  uint32_t* d_tile_meta = nullptr;
  bool mul_v4 = false, mul_v4_owned = false;
  bool residuals_resident = false;  // d_residuals holds the residuals of the last b200_evaluate(..., residuals != NULL)
  double *d_ftf_inv = nullptr, *d_spse[3] = {nullptr, nullptr, nullptr};  // general-preconditioner PCG (SPSE)
  double *d_pq_parts = nullptr, *d_seed_pq = nullptr;  // fused p.q: per-CTA partials of the product / of the vector kernel
  WarpTile* d_wtiles = nullptr;
  uint32_t* d_row_meta = nullptr;
  int2 *d_cta_part = nullptr, *d_cta_cam = nullptr;
  int* d_cta_cams = nullptr;
  double* d_partials = nullptr;
  size_t v2_smem = 0;
  bool v2b_ok = false;        // warp-tile versions of evaluate / schur_init / diag_blocks usable (narrow camera ranges)
  V2View v2_init{}, v2_diag{}, v2_eval{}, v2_mul{};
  size_t mul_smem = 0;
  bool mul_v3 = false;
  size_t eval_v2_smem = 0, init_v2_smem = 0, diag_v2_smem = 0;
  int diag_v2_replicas = 0;
  // camera-major block diagonal (used when no camera sees a point twice)
  bool cam_major_ok = false;
  int num_cam_items = 0;
  CamItem* d_cam_items = nullptr;
  int* d_cam_rows = nullptr;
  double* d_q3 = nullptr;
  // explicit S (explicit_schur.cuh), single GPU, chosen by b200_create from the camera graph
  bool xs = false;
  bool xs_ready = false;        // S holds the assembly for the current implicit-Schur initialisation
  bool xs_diag_ready = false;   // ... and d_upper45 still holds its diagonal blocks
  int xs_grid = 0;
  XsView xsv{};
  int num_xs_long = 0, num_xs_short = 0;   // blocks assembled by a CTA / by a warp each
  int *d_xs_blk_row = nullptr, *d_xs_blk_col = nullptr, *d_xs_pair_ptr = nullptr, *d_xs_list_ptr = nullptr, *d_xs_warp_cam = nullptr;
  int* d_xs_order = nullptr;   // [long blocks | short blocks]
  int2 *d_xs_pairs = nullptr, *d_xs_list = nullptr;
  double* d_xs_S = nullptr;
  double* d_ybig = nullptr;  // RED target of the big-point kernel inside the PCG (consumed + zeroed by cg_vector_kernel)
  double* d_red = nullptr;    // per-CTA partial sums of cg_vector_kernel
  // multi-GPU exchange of the per-iteration partial products over NVLink peer memory (cg_kernel.cuh: xchg_push_kernel +
  // the gather in cg_vector_kernel); replaces the ncclAllReduce inside the PCG iteration when every peer could be mapped
  bool xchg_ok = false;
  uint4* d_xchg = nullptr;        // [2 slots][world][9C] packets {lo, epoch, hi, epoch}
  XchgPeers xpeers{};
  void* xchg_opened[kMaxXchgRanks] = {};
  unsigned xepoch = 0;
  int cg_grid = 1;
  PinnedVec hv[12];           // host-boundary LM loop vectors
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

template <typename T>
int dev_alloc(T** p, size_t n) {
  if (n == 0) n = 1;
  CU(cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)));
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

// d_sqnorm (optional): squared column norms of the Jacobian as written (after the fused scaling), for free with the
// warp-tile kernel; the caller falls back to sqnorm_dev when *sqnorm_done comes back false.
// J is computed (and checked) when the Jacobian or the gradient is asked for, and stored only when want_jacobian: a
// gradient-only evaluation leaves the device-resident Jacobian as it was, as Ceres leaves it with jacobian == NULL.
int evaluate_dev(b200_handle* h, const double* d_state, double* d_residuals, double* d_gradient, bool want_jacobian,
                 const double* d_scale, double* cost_out, double* d_sqnorm = nullptr, bool* sqnorm_done = nullptr) {
  if (!want_jacobian) d_sqnorm = nullptr;   // the column norms are those of the stored Jacobian
  else h->xs_ready = false;                 // S is a function of J
  EvalArgs a{};
  a.state = d_state;
  a.residuals = d_residuals;
  a.gradient = d_gradient;
  a.cost_partial = h->d_tile_partial;
  a.scale = d_scale;
  a.fail_flag = h->d_fail;
  a.loss_type = h->apply_loss ? h->loss_type : B200_LOSS_TRIVIAL;
  a.loss_a = h->loss_a;
  if (sqnorm_done != nullptr) *sqnorm_done = false;
  CU(cudaMemsetAsync(h->d_fail, 0, sizeof(int), h->stream));
  const bool with_j = want_jacobian || d_gradient != nullptr;
  const size_t coff = 3 * static_cast<size_t>(h->P);
  if (d_gradient != nullptr) CU(cudaMemsetAsync(d_gradient + coff, 0, sizeof(double) * 9 * h->C, h->stream));
  if (d_gradient != nullptr) OK(huge_zero(h, d_gradient));
  const size_t smem = tile_smem_bytes<3, 1>();
  int num_partials = h->num_tiles;
  if (with_j && h->v2b_ok) {
    EvalV2Args e{};
    e.state = d_state;
    e.residuals = d_residuals;
    e.gradient = d_gradient;
    e.sqnorm = d_sqnorm;
    e.cost_partial = h->d_tile_partial;
    e.scale = d_scale;
    e.fail_flag = h->d_fail;
    e.loss_type = a.loss_type;
    e.loss_a = h->loss_a;
    if (d_sqnorm != nullptr) CU(cudaMemsetAsync(d_sqnorm + coff, 0, sizeof(double) * 9 * h->C, h->stream));
    if (d_sqnorm != nullptr) OK(huge_zero(h, d_sqnorm));
    OK(launch(h, K_EVAL_JAC, [&] {
      if (want_jacobian) evaluate_v2_kernel<true><<<h->v2.num_ctas, 32 * h->v2.warps, h->eval_v2_smem, h->stream>>>(h->v2_eval, e);
      else evaluate_v2_kernel<false><<<h->v2.num_ctas, 32 * h->v2.warps, h->eval_v2_smem, h->stream>>>(h->v2_eval, e);
    }));
    num_partials = h->v2.num_ctas;
    if (h->num_big_tiles > 0) {  // the few >32-row points: CTA-tile kernels on their tiles only
      a.cost_partial = h->d_tile_partial + num_partials;
      OK(launch(h, K_EVAL_JAC, [&] {
        const int grid = std::min(h->num_big_tiles, h->sm_count * 2);
        if (want_jacobian) evaluate_kernel<true><<<grid, kTile, smem, h->stream>>>(h->view_big, a);
        else evaluate_kernel<true, false><<<grid, kTile, smem, h->stream>>>(h->view_big, a);
      }, false));
      num_partials += h->num_big_tiles;
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
      if (want_jacobian) evaluate_kernel<true><<<h->grid_tile[K_EVAL_JAC], kTile, smem, h->stream>>>(h->view, a);
      else evaluate_kernel<true, false><<<h->grid_tile[K_EVAL_JAC], kTile, smem, h->stream>>>(h->view, a);
    }));
  } else {
    OK(launch(h, K_EVAL_COST, [&] { evaluate_kernel<false><<<h->grid_tile[K_EVAL_COST], kTile, smem, h->stream>>>(h->view, a); }));
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

int scale_dev(b200_handle* h, const double* d_scale) {
  h->xs_ready = false;   // S is a function of J
  return launch(h, K_SCALE, [&] {
    scale_kernel<<<flat_grid(h, 12 * static_cast<size_t>(h->N), 256), 256, 0, h->stream>>>(h->view, d_scale);
  });
}

// Block pattern of the upper triangle of S and what its assembly and product read (explicit_schur.cuh), built from the
// row structure in the internal order.  Block row i: the diagonal block first (also for a camera without rows), then
// the cameras j > i sharing a point with i in increasing order; every block lists its row pairs (r, s) in the order
// (row r of camera i in row order, row s of r's point in row order) -- a fixed summation order.
struct XsPattern {
  long long off_blocks = 0;   // distinct camera pairs i < j that share a point
  std::vector<int> blk_row, blk_col, pair_ptr, list_ptr;
  std::vector<int2> pairs, list;
};
void xs_pattern(int C, int N, const int* cam_idx, const int* pt_idx, const int* pt_ptr, XsPattern* xp) {
  std::vector<int> cptr(static_cast<size_t>(C) + 1, 0), crow(static_cast<size_t>(N));
  for (int r = 0; r < N; ++r) cptr[cam_idx[r] + 1]++;
  for (int c = 0; c < C; ++c) cptr[c + 1] += cptr[c];
  {
    std::vector<int> fill(cptr.begin(), cptr.end() - 1);
    for (int r = 0; r < N; ++r) crow[fill[cam_idx[r]]++] = r;
  }
  std::vector<int> stamp(static_cast<size_t>(C), -1), slot(static_cast<size_t>(C), 0), js, start;
  std::vector<int> row_start(static_cast<size_t>(C) + 1, 0);
  std::vector<int3> tup;
  for (int i = 0; i < C; ++i) {
    js.clear();
    tup.clear();
    stamp[i] = i;   // the diagonal block exists even for a camera without rows
    js.push_back(i);
    for (int k = cptr[i]; k < cptr[i + 1]; ++k) {
      const int r = crow[k], p = pt_idx[r];
      for (int s = pt_ptr[p]; s < pt_ptr[p + 1]; ++s) {
        const int j = cam_idx[s];
        if (j < i) continue;
        if (stamp[j] != i) {
          stamp[j] = i;
          js.push_back(j);
        }
        tup.push_back(make_int3(j, r, s));
      }
    }
    std::sort(js.begin(), js.end());
    xp->off_blocks += static_cast<long long>(js.size()) - 1;
    row_start[i] = static_cast<int>(xp->blk_row.size());
    start.assign(js.size() + 1, 0);
    for (size_t t = 0; t < js.size(); ++t) {
      slot[js[t]] = static_cast<int>(t);
      xp->blk_row.push_back(i);
      xp->blk_col.push_back(js[t]);
    }
    for (const int3& t : tup) start[slot[t.x] + 1]++;
    for (size_t t = 0; t < js.size(); ++t) start[t + 1] += start[t];
    const size_t base = xp->pairs.size();
    for (size_t t = 0; t < js.size(); ++t) xp->pair_ptr.push_back(static_cast<int>(base + start[t]));
    xp->pairs.resize(base + tup.size());
    for (const int3& t : tup) xp->pairs[base + start[slot[t.x]]++] = make_int2(t.y, t.z);
  }
  const int nb = static_cast<int>(xp->blk_row.size());
  row_start[C] = nb;
  xp->pair_ptr.push_back(static_cast<int>(xp->pairs.size()));
  // product lists: block row i, then the blocks (j, i) above the diagonal of column i, in order of j
  std::vector<int> tcnt(static_cast<size_t>(C) + 1, 0);
  for (int b = 0; b < nb; ++b)
    if (xp->blk_col[b] != xp->blk_row[b]) tcnt[xp->blk_col[b] + 1]++;
  for (int c = 0; c < C; ++c) tcnt[c + 1] += tcnt[c];
  std::vector<int2> tr(static_cast<size_t>(tcnt[C]));
  {
    std::vector<int> fill(tcnt.begin(), tcnt.end() - 1);
    for (int b = 0; b < nb; ++b)
      if (xp->blk_col[b] != xp->blk_row[b])
        tr[fill[xp->blk_col[b]]++] = make_int2(b, static_cast<int>(static_cast<uint32_t>(xp->blk_row[b]) | kXsTransposed));
  }
  xp->list_ptr.assign(static_cast<size_t>(C) + 1, 0);
  xp->list.reserve(static_cast<size_t>(nb) + tr.size());
  for (int i = 0; i < C; ++i) {
    xp->list_ptr[i] = static_cast<int>(xp->list.size());
    for (int b = row_start[i]; b < row_start[i + 1]; ++b) xp->list.push_back(make_int2(b, xp->blk_col[b]));
    xp->list.insert(xp->list.end(), tr.begin() + tcnt[i], tr.begin() + tcnt[i + 1]);
  }
  xp->list_ptr[C] = static_cast<int>(xp->list.size());
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

// y = S x (+ D_f^2 x) on the explicit S, assembled first if it is stale; y is overwritten.
int xs_mul_dev(b200_handle* h, const double* d_x, double* d_y) {
  if (!h->xs_ready) OK(xs_assemble_dev(h));
  const double* Df = h->cur_D != nullptr ? h->cur_D + 3 * static_cast<size_t>(h->P) : nullptr;
  return launch(h, K_SCHUR_MUL, [&] {
    xs_mul_kernel<<<h->xs_grid, kXsThreads, 0, h->stream>>>(h->xsv, d_x, d_y, Df, 0, nullptr, nullptr);
  });
}

// ImplicitSchurComplement::Init on device pointers b [2N], D [3P+9C] or null.
int schur_init_dev(b200_handle* h, const double* d_b, const double* d_D) {
  SchurState st{};
  st.b = d_b;
  st.D = d_D;
  st.ete_inv = h->d_ete_inv;
  st.rhs = h->d_rhs;
  st.ye = h->d_ye;
  CU(cudaMemsetAsync(h->d_rhs, 0, sizeof(double) * 9 * h->C, h->stream));
  h->q_from_init = false;
  h->xs_ready = false;
  if (h->mul_v4) {
    // v4 machinery: E, F, b and the tile's D_e through the TMA slot; also writes the per-row 2x2 blocks Q_r the camera-major
    // block-diagonal pass reads (no separate pass over E for them)
    InitV4Args ia{};
    ia.b = d_b;
    ia.D = d_D;
    ia.ete_inv = h->d_ete_inv;
    ia.rhs = h->d_rhs;
    ia.ye = nullptr;   // (E'E)^-1 E'b is not consumed by anything on this path: not written
    ia.q3 = h->cam_major_ok ? h->d_q3 : nullptr;
    OK(launch(h, K_SCHUR_INIT, [&] {
      V2View iv = h->v2_mul;
      iv.cta_big = h->d_cta_big;   // the kernel takes the CTA's 33..kTile-row points itself
      if (h->mul_v4_owned) schur_init_v4_kernel<true><<<h->v2.num_ctas, 32 * h->v2_mul.warps, h->mul_smem, h->stream>>>(iv, ia);
      else schur_init_v4_kernel<false><<<h->v2.num_ctas, 32 * h->v2_mul.warps, h->mul_smem, h->stream>>>(iv, ia);
    }));
    h->q_from_init = ia.q3 != nullptr;
  } else if (h->v2b_ok) {
    OK(launch(h, K_SCHUR_INIT, [&] {
      schur_init_v2_kernel<<<h->v2.num_ctas, 32 * h->v2_init.warps, h->init_v2_smem, h->stream>>>(h->v2_init, st);
    }));
    if (h->num_big_tiles > 0)
      OK(launch(h, K_SCHUR_INIT, [&] {
        schur_init_kernel<<<std::min(h->num_big_tiles, h->sm_count * 4), kTile, tile_smem_bytes<9, 3>(), h->stream>>>(h->view_big, st);
      }, false));
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

// y = S x on device vectors [9C]; y is overwritten.  done_flag (device int*, may be null) turns every launch into a
// no-op once the PCG has terminated.
int schur_mul_dev(b200_handle* h, const double* d_x, double* d_y, const int* done_flag) {
  const double* Df = h->cur_D != nullptr ? h->cur_D + 3 * static_cast<size_t>(h->P) : nullptr;
  const double* seed = (h->rank == 0) ? Df : nullptr;
  const int n = 9 * h->C;
  if (h->v2_ok) {
    if (h->v2.direct)
      OK(launch(h, K_MISC, [&] {
        diag_sq_mul_kernel<<<flat_grid(h, n, 256), 256, 0, h->stream>>>(n, seed, d_x, d_y, done_flag);
      }));
    OK(launch(h, K_SCHUR_MUL, [&] {
      if (h->mul_v4 && h->mul_v4_owned) schur_mul_v4_kernel<true><<<h->v2.num_ctas, 32 * h->v2_mul.warps, h->mul_smem, h->stream>>>(h->v2_mul, h->d_ete_inv, d_x, d_y, done_flag, nullptr);
      else if (h->mul_v4) schur_mul_v4_kernel<false><<<h->v2.num_ctas, 32 * h->v2_mul.warps, h->mul_smem, h->stream>>>(h->v2_mul, h->d_ete_inv, d_x, d_y, done_flag, nullptr);
      else schur_mul_v3_kernel<<<h->v2.num_ctas, 32 * h->v2_mul.warps, h->mul_smem, h->stream>>>(h->v2_mul, h->d_ete_inv, d_x, d_y, done_flag);
    }));
    if (!h->v2.direct)
      OK(launch(h, K_CAM_REDUCE, [&] {
        cam_reduce_kernel<<<(n + 63) / 64, 256, h->v2.num_ctas * sizeof(int2), h->stream>>>(
            n, h->v2.num_ctas, h->d_cta_cam, h->d_partials, 9 * h->v2.max_cam_span, seed, d_x, d_y, 0, done_flag);
      }));
    if (h->num_big_tiles > 0 && !h->big_folded)
      OK(launch(h, K_SCHUR_MUL_BIG, [&] {
        schur_mul_kernel<<<std::min(h->num_big_tiles, h->sm_count * 4), kTile, tile_smem_bytes<3, 3>(), h->stream>>>(
            h->view_big, h->d_ete_inv, d_x, d_y, done_flag);
      }, false));
  } else {
    OK(launch(h, K_MISC, [&] {
      diag_sq_mul_kernel<<<flat_grid(h, n, 256), 256, 0, h->stream>>>(n, seed, d_x, d_y, done_flag);
    }));
    OK(launch(h, K_SCHUR_MUL, [&] {
      schur_mul_kernel<<<h->grid_tile[K_SCHUR_MUL], kTile, tile_smem_bytes<3, 3>(), h->stream>>>(h->view, h->d_ete_inv, d_x, d_y, done_flag);
    }));
  }
  if (h->num_huge > 0)
    OK(launch(h, K_SCHUR_MUL_BIG, [&] {
      huge_schur_mul_kernel<<<huge_grid(h), kHugeThreads, 0, h->stream>>>(h->view, h->num_huge, h->d_huge_pts, h->d_ete_inv, d_x, d_y, done_flag);
    }, false));
  return allreduce_sum(h, d_y, n);
}

int precond_update_dev(b200_handle* h, int type) {
  if (type == B200_PRECOND_IDENTITY) return B200_OK;
  const double* Df = h->cur_D != nullptr ? h->cur_D + 3 * static_cast<size_t>(h->P) : nullptr;
  if (h->xs && type == B200_PRECOND_SCHUR_JACOBI) {
    // the diagonal blocks of the explicit S: no pass of their own
    if (!h->xs_ready || !h->xs_diag_ready) OK(xs_assemble_dev(h));
    return launch(h, K_INVERT9, [&] {
      invert9_kernel<<<(h->C + kInvWarps - 1) / kInvWarps, 32 * kInvWarps, 0, h->stream>>>(h->C, h->d_upper45, Df, h->d_blocks, h->d_minv);
    });
  }
  h->xs_diag_ready = false;
  CU(cudaMemsetAsync(h->d_upper45, 0, sizeof(double) * 45 * h->C, h->stream));
  if (h->cam_major_ok) {
    const bool schur = type == B200_PRECOND_SCHUR_JACOBI;
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
  } else if (h->v2b_ok && h->diag_v2_replicas > 0) {
    const bool schur = type == B200_PRECOND_SCHUR_JACOBI;
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
  } else if (type == B200_PRECOND_SCHUR_JACOBI) {
    OK(launch(h, K_DIAG_BLOCKS, [&] {
      diag_blocks_kernel<true><<<h->grid_tile[K_DIAG_BLOCKS], kTile, tile_smem_bytes<1, 1>(), h->stream>>>(h->view, h->d_ete_inv, h->d_upper45);
    }));
  } else {
    OK(launch(h, K_DIAG_BLOCKS, [&] {
      diag_blocks_kernel<false><<<h->grid_tile[K_DIAG_BLOCKS], kTile, tile_smem_bytes<1, 1>(), h->stream>>>(h->view, h->d_ete_inv, h->d_upper45);
    }));
  }
  OK(allreduce_sum(h, h->d_upper45, 45 * static_cast<size_t>(h->C)));
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
  const double* Df = d_D != nullptr ? d_D + 3 * static_cast<size_t>(h->P) : nullptr;
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
      OK(launch(h, K_BACKSUB, [&] {
        backsub_kernel<<<h->grid_tile[K_BACKSUB], kTile, tile_smem_bytes<3, 1>(), h->stream>>>(h->view, h->d_ete_inv, d_b, h->d_sol, d_x);
      }));
      if (h->num_huge > 0)
        OK(launch(h, K_BACKSUB, [&] {
          huge_backsub_kernel<<<huge_grid(h), kHugeThreads, 0, h->stream>>>(h->view, h->num_huge, h->d_huge_pts, h->d_ete_inv, d_b, h->d_sol, d_x);
        }, false));
      CU(cudaMemcpyAsync(d_x + 3 * static_cast<size_t>(h->P), h->d_sol, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
    }
    return B200_OK;
  };
  // In direct-flush mode the vector kernel pre-seeds the next product's output (D_f^2 p, rank 0 only) and the product
  // kernels RED straight into it: one product launch + one vector launch per iteration.
  const bool seeded = (h->v2_ok && h->v2.direct) || explicit_s;
  va.Df = (h->rank == 0) ? Df : nullptr;
  // multi-GPU: the partial products travel through peer memory instead of an NCCL all-reduce (needs the direct-flush
  // product: `out` then holds exactly this rank's partial)
  const bool xchg = h->xchg_ok && h->v2_ok && h->v2.direct && dev_env("B200_NO_PEER_EXCHANGE") == nullptr;
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
  const bool fuse_pq = (explicit_s || (seeded && h->mul_v4 && (h->world == 1 || xchg) && h->num_huge == 0 &&
                                       (h->num_big_tiles == 0 || h->big_folded))) &&
                       dev_env("B200_NO_FUSED_PQ") == nullptr;
  double* pq_parts = fuse_pq ? h->d_pq_parts : nullptr;
  va.pq_parts = pq_parts;
  va.num_pq_parts = fuse_pq ? (explicit_s ? h->xs_grid : h->v2.num_ctas) : 0;
  va.seed_pq = fuse_pq ? h->d_seed_pq : nullptr;
  const bool use_pdl = dev_env("B200_NO_PDL") == nullptr && !h->profiling;
  auto product = [&](const double* vin, double* out) -> int {
    if (explicit_s) {
      // adds S vin onto the seeded output; programmatic dependent launch like the v4 product
      return launch(h, K_SCHUR_MUL, [&] {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(h->xs_grid);
        cfg.blockDim = dim3(kXsThreads);
        cfg.dynamicSmemBytes = 0;
        cfg.stream = h->stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = use_pdl ? 1 : 0;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        cudaLaunchKernelEx(&cfg, xs_mul_kernel, h->xsv, vin, out, static_cast<const double*>(nullptr), 1,
                           static_cast<const int*>(&h->d_cg->done), pq_parts);
      });
    }
    if (seeded) {
      // The handful of >32-row points runs on a side stream, concurrently with the warp-tile kernel (both only add
      // into the pre-seeded output with REDs); outside profiling mode, where launches are bracketed by events.
      const bool side = h->num_big_tiles > 0 && !h->profiling && !h->big_folded;
      if (side) {
        CU(cudaEventRecord(h->ev_fork, h->stream));
        CU(cudaStreamWaitEvent(h->stream2, h->ev_fork, 0));
        schur_mul_kernel<<<std::min(h->num_big_tiles, h->sm_count * 4), kTile, tile_smem_bytes<3, 3>(), h->stream2>>>(
            h->view_big, h->d_ete_inv, vin, out, &h->d_cg->done);
        h->launches[K_SCHUR_MUL_BIG]++;
        CU(cudaEventRecord(h->ev_join, h->stream2));
      }
      OK(launch(h, K_SCHUR_MUL, [&] {
        if (h->mul_v4) {
          // programmatic dependent launch: the product's prologue overlaps the tail of the vector kernel before it
          cudaLaunchConfig_t cfg{};
          cfg.gridDim = dim3(h->v2.num_ctas);
          cfg.blockDim = dim3(32 * h->v2_mul.warps);
          cfg.dynamicSmemBytes = h->mul_smem;
          cfg.stream = h->stream;
          cudaLaunchAttribute attr[1];
          attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
          attr[0].val.programmaticStreamSerializationAllowed = use_pdl ? 1 : 0;
          cfg.attrs = attr;
          cfg.numAttrs = 1;
          const int* done_ptr = &h->d_cg->done;
          if (h->mul_v4_owned) cudaLaunchKernelEx(&cfg, schur_mul_v4_kernel<true>, h->v2_mul, static_cast<const double*>(h->d_ete_inv), vin, out, done_ptr, pq_parts);
          else cudaLaunchKernelEx(&cfg, schur_mul_v4_kernel<false>, h->v2_mul, static_cast<const double*>(h->d_ete_inv), vin, out, done_ptr, pq_parts);
        }
        else schur_mul_v3_kernel<<<h->v2.num_ctas, 32 * h->v2_mul.warps, h->mul_smem, h->stream>>>(h->v2_mul, h->d_ete_inv, vin, out, &h->d_cg->done);
      }));
      if (side) {
        CU(cudaStreamWaitEvent(h->stream, h->ev_join, 0));
      } else if (h->num_big_tiles > 0 && !h->big_folded) {
        OK(launch(h, K_SCHUR_MUL_BIG, [&] {
          schur_mul_kernel<<<std::min(h->num_big_tiles, h->sm_count * 4), kTile, tile_smem_bytes<3, 3>(), h->stream>>>(
              h->view_big, h->d_ete_inv, vin, out, &h->d_cg->done);
        }, false));
      }
      if (h->num_huge > 0)
        OK(launch(h, K_SCHUR_MUL_BIG, [&] {
          huge_schur_mul_kernel<<<huge_grid(h), kHugeThreads, 0, h->stream>>>(h->view, h->num_huge, h->d_huge_pts, h->d_ete_inv, vin, out, &h->d_cg->done);
        }, false));
      if (!xchg) return allreduce_sum(h, out, n);
      ++h->xepoch;   // the vector kernel that consumes this product exchanges it under this epoch
      return B200_OK;
    }
    return schur_mul_dev(h, vin, out, &h->d_cg->done);
  };
  if (general) {
    // SURVEY 8f.2: power-series preconditioner / initial guess -> the general-preconditioner PCG (host-side scalars)
    OK(pcg_general_dev(h, o));
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

// DenseSchurComplementSolver (schur_complement_solver.cc:101-159, :161-214) on device pointers: explicit S by
// dense_schur_assemble_kernel, Cholesky by cuSOLVER, back substitution by the implicit-Schur kernels.
int dense_schur_solve_dev(b200_handle* h, const double* d_b, const double* d_D, double* d_x, b200_solver_summary* summary) {
  if (h->world > 1) return fail(B200_ERR_UNSUPPORTED, "the explicit Schur complement is single-GPU");
  const int n = 9 * h->C;
  const size_t bytes = sizeof(double) * static_cast<size_t>(n) * n;
  if (bytes > (static_cast<size_t>(48) << 30))
    return fail(B200_ERR_UNSUPPORTED, "dense reduced camera system of %d cameras needs %.1f GB", h->C, bytes / 1e9);
  if (!load_cusolver()) return fail(B200_ERR_UNSUPPORTED, "cannot load libcusolver.so.11: %s", dlerror());
  if (h->cusolver == nullptr) {
    if (g_cusolver.Create(&h->cusolver) != 0) return fail(B200_ERR_CUDA, "cusolverDnCreate failed");
    if (g_cusolver.SetStream(h->cusolver, h->stream) != 0) return fail(B200_ERR_CUDA, "cusolverDnSetStream failed");
  }
  if (h->d_dense_s == nullptr) {
    OK(dev_alloc(&h->d_dense_s, static_cast<size_t>(n) * n));
    OK(dev_alloc(&h->d_dense_info, 4));
    int lwork = 0;
    if (g_cusolver.DpotrfBufferSize(h->cusolver, /*CUBLAS_FILL_MODE_LOWER*/ 0, n, h->d_dense_s, n, &lwork) != 0)
      return fail(B200_ERR_CUDA, "cusolverDnDpotrf_bufferSize failed");
    h->dense_lwork = std::max(lwork, 1);
    OK(dev_alloc(&h->d_dense_work, static_cast<size_t>(h->dense_lwork)));
  }
  OK(schur_init_dev(h, d_b, d_D));   // (E'E + D^2)^-1 and the reduced right-hand side
  const double* Df = d_D != nullptr ? d_D + 3 * static_cast<size_t>(h->P) : nullptr;
  CU(cudaMemsetAsync(h->d_dense_s, 0, bytes, h->stream));
  OK(launch(h, K_DIAG_BLOCKS, [&] {
    dense_schur_assemble_kernel<<<std::max(1, std::min(h->P, h->sm_count * 8)), kDsThreads, 0, h->stream>>>(h->view, h->d_ete_inv, h->d_dense_s, static_cast<size_t>(n));
  }));
  OK(launch(h, K_MISC, [&] { dense_schur_diagonal_kernel<<<(n + 255) / 256, 256, 0, h->stream>>>(n, Df, h->d_dense_s, static_cast<size_t>(n)); }));
  if (g_cusolver.Dpotrf(h->cusolver, 0, n, h->d_dense_s, n, h->d_dense_work, h->dense_lwork, h->d_dense_info) != 0)
    return fail(B200_ERR_CUDA, "cusolverDnDpotrf failed");
  CU(cudaMemcpyAsync(h->d_sol, h->d_rhs, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
  if (g_cusolver.Dpotrs(h->cusolver, 0, n, 1, h->d_dense_s, n, h->d_sol, n, h->d_dense_info + 1) != 0)
    return fail(B200_ERR_CUDA, "cusolverDnDpotrs failed");
  CU(cudaMemcpyAsync(h->h_fail, h->d_dense_info, 2 * sizeof(int), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  summary->num_iterations = 1;   // schur_complement_solver.cc:154
  summary->residual_norm = 0.0;
  if (h->h_fail[0] != 0 || h->h_fail[1] != 0) {   // not positive definite: LinearSolverTerminationType::FAILURE (:203-210)
    summary->termination_type = B200_LS_FAILURE;
    return B200_OK;
  }
  summary->termination_type = B200_LS_SUCCESS;
  OK(launch(h, K_BACKSUB, [&] {
    backsub_kernel<<<h->grid_tile[K_BACKSUB], kTile, tile_smem_bytes<3, 1>(), h->stream>>>(h->view, h->d_ete_inv, d_b, h->d_sol, d_x);
  }));
  if (h->num_huge > 0)
    OK(launch(h, K_BACKSUB, [&] {
      huge_backsub_kernel<<<huge_grid(h), kHugeThreads, 0, h->stream>>>(h->view, h->num_huge, h->d_huge_pts, h->d_ete_inv, d_b, h->d_sol, d_x);
    }, false));
  CU(cudaMemcpyAsync(d_x + 3 * static_cast<size_t>(h->P), h->d_sol, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream));
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
    OK(dev_alloc(&h->d_ftf_inv, 81 * static_cast<size_t>(h->C)));
    for (auto& b : h->d_spse) OK(dev_alloc(&b, static_cast<size_t>(n)));
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
      OK(schur_mul_dev(h, prev, t, nullptr));   // (F'F + D^2) prev - F'E P E'F prev
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
  OK(schur_mul_dev(h, x, tmp, nullptr));
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
    OK(schur_mul_dev(h, p, q, nullptr));
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
      OK(schur_mul_dev(h, x, tmp, nullptr));
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

// ---- Internal point order.  The fast kernels give every persistent CTA a contiguous run of points and keep the cameras
// those points see in shared memory, so they want neighbouring points to see the same few cameras.  The caller's e-block
// order is whatever Ceres' ordering produced (first use in the residual list); the library is free to keep its own: points
// (with all their rows, in the caller's relative order) are re-ordered privately, and every vector / matrix that crosses the
// ABI is permuted at the boundary (up_* / down_*), so the layout contract of the header (block_jacobian_writer.cc:68-167,
// reorder_program.cc:262-273) is untouched.  Candidates: 0 the caller's order; 1 by the start of the point's camera ARC (its
// cameras seen as a set on the circle of camera ids, the arc being the complement of the largest gap: the smallest camera
// unless the set wraps around -- keeps the seam of a loop closure together), then the arc's length; 2 by mean camera id; 3 by
// smallest, then largest camera id.  Score: distinct cameras per 1/chunks-th of the rows, summed; the best wins, the caller's
// order whenever it is within 10 % of the best (no boundary permutation then).  Pure host code (tests/test_host.py).
const char* const kOrderNames[4] = {"caller's order kept", "by camera arc", "by mean camera", "by smallest camera"};
int choose_point_order(int C, int P, int N, const int32_t* cam_of_row, const int* caller_ptr, int chunks, std::vector<int>* perm,
                       long metrics[4]) {
  std::vector<int> ident(static_cast<size_t>(P));
  std::iota(ident.begin(), ident.end(), 0);
  auto metric = [&](const std::vector<int>& ord) -> long {
    std::vector<int> stamp(static_cast<size_t>(C), -1);
    long total = 0, rows = 0;
    int chunk = 0;
    const long target = N / chunks + 1;
    for (int k = 0; k < P; ++k) {
      const int q = ord[k];
      for (int r = caller_ptr[q]; r < caller_ptr[q + 1]; ++r) {
        const int c = cam_of_row[r];
        if (stamp[c] != chunk) {
          stamp[c] = chunk;
          ++total;
        }
      }
      rows += caller_ptr[q + 1] - caller_ptr[q];
      while (rows >= static_cast<long>(chunk + 1) * target) ++chunk;
    }
    return total;
  };
  std::vector<long long> key[3];
  for (auto& k : key) k.resize(static_cast<size_t>(P));
  {
    std::vector<int> cams;
    for (int q = 0; q < P; ++q) {
      const int deg = caller_ptr[q + 1] - caller_ptr[q];
      long long sum = 0;
      cams.clear();
      for (int r = caller_ptr[q]; r < caller_ptr[q + 1]; ++r) {
        cams.push_back(cam_of_row[r]);
        sum += cam_of_row[r];
      }
      std::sort(cams.begin(), cams.end());
      long long start = C, len = 0, lo = C, hi = C;
      if (deg > 0) {
        int best_gap = cams[0] + C - cams[deg - 1];   // the gap that wraps around
        start = cams[0];
        for (int i = 1; i < deg; ++i)
          if (cams[i] - cams[i - 1] > best_gap) {
            best_gap = cams[i] - cams[i - 1];
            start = cams[i];
          }
        len = C - best_gap;
        lo = cams[0];
        hi = cams[deg - 1];
      }
      key[0][q] = start * (static_cast<long long>(C) + 1) + len;
      key[1][q] = deg > 0 ? (sum * 64) / deg : static_cast<long long>(C) * 64;
      key[2][q] = lo * (static_cast<long long>(C) + 1) + hi;
    }
  }
  metrics[0] = metric(ident);
  std::vector<int> cand[3];
  int best = 0;
  for (int c = 0; c < 3; ++c) {
    cand[c] = ident;
    std::stable_sort(cand[c].begin(), cand[c].end(), [&](int a, int b) { return key[c][a] < key[c][b]; });
    metrics[c + 1] = metric(cand[c]);
    if (metrics[c + 1] < metrics[best + 1]) best = c;
  }
  if (static_cast<double>(metrics[0]) > 1.10 * static_cast<double>(metrics[best + 1])) {
    *perm = cand[best];
    return best + 1;
  }
  *perm = ident;
  return 0;
}

}  // namespace

// ================================================================================================ C ABI
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
  std::vector<int> ptr(static_cast<size_t>(P) + 1, 0);
  for (int i = 0; i < N; ++i) {
    const int pt = desc->pt_idx[i], cam = desc->cam_idx[i];
    if (pt < 0 || pt >= P || cam < 0 || cam >= C) return fail(B200_ERR_INVALID_ARGUMENT, "row %d: block id out of range", i);
    if (i > 0 && pt < desc->pt_idx[i - 1]) return fail(B200_ERR_INVALID_ARGUMENT, "rows are not grouped by e block at row %d", i);
    ptr[pt + 1]++;
  }
  for (int k = 0; k < P; ++k) ptr[k + 1] += ptr[k];
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
  // Row structure checks: the SchurEliminator precondition (rows grouped by e block).
  std::vector<int> caller_ptr(static_cast<size_t>(P) + 1, 0);
  for (int i = 0; i < N; ++i) {
    const int pt = desc->pt_idx[i], cam = desc->cam_idx[i];
    if (pt < 0 || pt >= P || cam < 0 || cam >= C) return fail(B200_ERR_INVALID_ARGUMENT, "row %d: block id out of range", i);
    if (i > 0 && pt < desc->pt_idx[i - 1])
      return fail(B200_ERR_INVALID_ARGUMENT, "rows are not grouped by e block at row %d (reorder_program.cc:278-359)", i);
    caller_ptr[pt + 1]++;
  }
  for (int k = 0; k < P; ++k) caller_ptr[k + 1] += caller_ptr[k];

  // ---- Internal point order (choose_point_order above): private to the library, undone at the ABI boundary.
  std::vector<int> pt_perm;   // internal point k = caller point pt_perm[k]
  long order_metrics[4];
  const int order_choice = dev_env("B200_KEEP_ORDER") != nullptr
                               ? (pt_perm.resize(static_cast<size_t>(P)), std::iota(pt_perm.begin(), pt_perm.end(), 0), 0)
                               : choose_point_order(C, P, N, desc->cam_idx, caller_ptr.data(), prop.multiProcessorCount, &pt_perm, order_metrics);
  const bool identity_order = order_choice == 0;
  if (getenv("B200_VERBOSE") != nullptr && dev_env("B200_KEEP_ORDER") == nullptr)
    fprintf(stderr, "[b200ba] point order: distinct cameras per 1/%d of the rows, summed: caller %ld, by camera arc %ld, by mean camera %ld, by smallest camera %ld -> %s\n",
            prop.multiProcessorCount, order_metrics[0], order_metrics[1], order_metrics[2], order_metrics[3], kOrderNames[order_choice]);
  // internal copies of the row structure
  std::vector<int> cam_i(static_cast<size_t>(N)), pt_i(static_cast<size_t>(N)), row_perm(static_cast<size_t>(N));
  std::vector<double> obs_i(2 * static_cast<size_t>(N));
  std::vector<int> pt_ptr(static_cast<size_t>(P) + 1, 0);
  {
    int r = 0;
    for (int k = 0; k < P; ++k) {
      const int q = pt_perm[k];
      for (int j = caller_ptr[q]; j < caller_ptr[q + 1]; ++j, ++r) {
        row_perm[r] = j;                     // internal row r = caller row j
        cam_i[r] = desc->cam_idx[j];
        pt_i[r] = k;
        obs_i[2 * static_cast<size_t>(r)] = desc->obs[2 * static_cast<size_t>(j)];
        obs_i[2 * static_cast<size_t>(r) + 1] = desc->obs[2 * static_cast<size_t>(j) + 1];
      }
      pt_ptr[k + 1] = r;
    }
  }
  const int* const cam_idx = cam_i.data();   // from here on: INTERNAL order
  const int* const pt_idx = pt_i.data();
  // Tiles: whole points, <= kTile rows and <= kTile points each; a point with more rows becomes chunk tiles.
  std::vector<TileDesc> tiles, chunk_tiles;
  std::vector<int> huge_pts;
  {
    int k = 0;
    while (k < P) {
      TileDesc t;
      t.pt_begin = k;
      t.obs_begin = pt_ptr[k];
      int rows = 0, pts = 0;
      bool huge = false;
      while (k < P && pts < kTile - 1) {  // pt_count + 1 chunk boundaries are loaded by one thread each
        const int deg = pt_ptr[k + 1] - pt_ptr[k];
        if (deg > kTile) {
          huge = pts == 0;
          break;
        }
        if (rows + deg > kTile) break;
        rows += deg;
        ++pts;
        ++k;
      }
      if (huge) {  // more than kTile rows: <= kTile-row slices of the one point (TileDesc::chunk)
        huge_pts.push_back(k);
        for (int r = pt_ptr[k]; r < pt_ptr[k + 1]; r += kTile) {
          TileDesc c;
          c.pt_begin = k;
          c.pt_count = 1;
          c.obs_begin = r;
          c.obs_count = std::min(kTile, pt_ptr[k + 1] - r);
          c.chunk = 1;
          tiles.push_back(c);
          chunk_tiles.push_back(c);
        }
        ++k;
        continue;
      }
      t.obs_count = rows;
      t.pt_count = pts;
      tiles.push_back(t);
    }
  }
  // Camera-major row lists (the reference's transpose block structure) for the block-diagonal kernels, cut into
  // slices of a few thousand rows so that small-C problems still fill the machine; unusable if a camera sees a
  // point twice (cross terms between the two rows), which is detected here.
  std::vector<int> cam_rows(static_cast<size_t>(N));
  std::vector<CamItem> cam_items;
  bool has_dups = false;
  {
    std::vector<int> cptr(static_cast<size_t>(C) + 1, 0);
    for (int i = 0; i < N; ++i) cptr[cam_idx[i] + 1]++;
    for (int c = 0; c < C; ++c) cptr[c + 1] += cptr[c];
    std::vector<int> fill(cptr.begin(), cptr.end() - 1);
    for (int i = 0; i < N; ++i) cam_rows[fill[cam_idx[i]]++] = i;
    for (int c = 0; c < C && !has_dups; ++c)
      for (int j = cptr[c] + 1; j < cptr[c + 1]; ++j)
        if (pt_idx[cam_rows[j]] == pt_idx[cam_rows[j - 1]]) { has_dups = true; break; }
    // ~3 items per resident warp (12 warps per SM): short enough to balance, long enough to amortise the final reduction
    const int slice = std::max(64, std::min(4096, N / (prop.multiProcessorCount * 36) + 1));
    for (int c = 0; c < C; ++c)
      for (int b = cptr[c]; b < cptr[c + 1]; b += slice) cam_items.push_back(CamItem{c, b, std::min(b + slice, cptr[c + 1])});
  }
  // v2 structures: warp tiles (whole points, <= 32 rows) for the points with <= 32 rows; points with 33..kTile
  // rows stay on the CTA-tile kernels (one tile each).  Needs every point to have at least one row.
  std::vector<WarpTile> wtiles;
  std::vector<TileDesc> big_tiles;
  std::vector<uint32_t> row_meta(static_cast<size_t>(N));
  bool v2_possible = dev_env("B200_DISABLE_V2") == nullptr;
  for (int k = 0; k < P && v2_possible; ++k)
    if (pt_ptr[k + 1] == pt_ptr[k]) v2_possible = false;
  if (v2_possible) {
    for (int k = 0; k < P; ++k)
      for (int r = pt_ptr[k]; r < pt_ptr[k + 1]; ++r)
        row_meta[r] = static_cast<uint32_t>(cam_idx[r]) | (r == pt_ptr[k] ? 0x80000000u : 0u);
    int k = 0;
    while (k < P) {
      const int deg0 = pt_ptr[k + 1] - pt_ptr[k];
      if (deg0 > kTile) {  // huge point: chunk tiles (appended to the big tiles below) + huge_kernels.cuh
        ++k;
        continue;
      }
      if (deg0 > 32) {
        TileDesc t;
        t.pt_begin = k;
        t.obs_begin = pt_ptr[k];
        t.obs_count = deg0;
        t.pt_count = 1;
        big_tiles.push_back(t);
        ++k;
        continue;
      }
      WarpTile t;
      t.row_begin = pt_ptr[k];
      t.pt_begin = k;
      int rows = 0, pts = 0;
      while (k < P) {
        const int deg = pt_ptr[k + 1] - pt_ptr[k];
        if (deg > 32 || rows + deg > 32) break;
        rows += deg;
        ++pts;
        ++k;
      }
      t.row_count = static_cast<unsigned short>(rows);
      t.pt_count = static_cast<unsigned short>(pts);
      wtiles.push_back(t);
    }
  }
  const int num_ctas_v2 = prop.multiProcessorCount;
  std::vector<int2> cta_part(num_ctas_v2), cta_cam(num_ctas_v2), cta_big(num_ctas_v2, make_int2(0, 0));
  std::vector<int> cta_cams;   // direct mode: concatenated per-CTA camera lists
  bool direct_mode = false;
  int max_cam_span = 1, v2_warps = 0, v2_stages = 0, v2_replicas = 1, mul_warps = 0, mul_stages = 0, mul_replicas = 1;
  if (v2_possible && !wtiles.empty()) {
    // Static partition by position in the row order, balanced by cost: a warp tile costs about the same whatever its
    // fill (the kernels are bound by warp-instruction issue / LSU work, not by bytes), and a >32-row point, which the
    // whole CTA processes serially, costs as much as ~20 tiles (in-kernel time stamps).
    // CTA b owns the items whose cumulative cost starts in [total * b / n, total * (b + 1) / n): neighbouring CTAs stream
    // neighbouring HBM ranges and touch neighbouring cameras.
    const int T = static_cast<int>(wtiles.size());
    {
      double big_cost = 22.0;
      if (const char* e = dev_env("B200_BIG_COST")) big_cost = std::max(0.0, atof(e));
      const double total_cost = T + big_cost * big_tiles.size();
      int t = 0, g = 0, b = 0;
      double cum = 0.0;
      std::vector<int> t_end(num_ctas_v2, 0), g_end(num_ctas_v2, 0);
      const int G = static_cast<int>(big_tiles.size());
      while (t < T || g < G) {
        const bool take_big = g < G && (t >= T || big_tiles[g].obs_begin < wtiles[t].row_begin);
        const int owner = std::min(num_ctas_v2 - 1, static_cast<int>(cum * num_ctas_v2 / std::max(total_cost, 1.0)));
        while (b < owner) {
          t_end[b] = t;
          g_end[b] = g;
          ++b;
        }
        if (take_big) {
          ++g;
          cum += big_cost;
        } else {
          ++t;
          cum += 1.0;
        }
      }
      for (; b < num_ctas_v2; ++b) {
        t_end[b] = T;
        g_end[b] = G;
      }
      for (int k = 0; k < num_ctas_v2; ++k) {
        cta_part[k] = make_int2(k == 0 ? 0 : t_end[k - 1], t_end[k]);
        cta_big[k] = make_int2(k == 0 ? 0 : g_end[k - 1], g_end[k]);
      }
    }
    // Cameras each CTA touches.  Direct mode (camera locality): every CTA gets the sorted LIST of its distinct cameras --
    // a row addresses its camera by the position in that list (packed into the row word), x of the listed cameras is
    // staged in shared memory and the private result is flushed with REDs.  What matters is the NUMBER of distinct
    // cameras per CTA, not their ids (a point that sees cameras 0, 1 and C-1 costs three entries).  Otherwise: id ranges,
    // per-CTA partial vectors and a fixed-order reduction.
    {
      std::vector<int> stamp(static_cast<size_t>(C), -1), local_of(static_cast<size_t>(C), 0);
      std::vector<int> lo_v(num_ctas_v2, 0), hi_v(num_ctas_v2, 0);
      std::vector<std::vector<int>> lists(num_ctas_v2);
      long list_total = 0;
      int max_list = 1, max_range = 1;
      for (int b = 0; b < num_ctas_v2; ++b) {
        int lo = C, hi = 0;
        auto visit = [&](int r0, int r1) {
          for (int r = r0; r < r1; ++r) {
            const int c = cam_idx[r];
            lo = std::min(lo, c);
            hi = std::max(hi, c + 1);
            if (stamp[c] != b) {
              stamp[c] = b;
              lists[b].push_back(c);
            }
          }
        };
        for (int t = cta_part[b].x; t < cta_part[b].y; ++t) visit(wtiles[t].row_begin, wtiles[t].row_begin + wtiles[t].row_count);
        for (int g = cta_big[b].x; g < cta_big[b].y; ++g) visit(big_tiles[g].obs_begin, big_tiles[g].obs_begin + big_tiles[g].obs_count);
        if (hi <= lo) { lo = 0; hi = 0; }
        std::sort(lists[b].begin(), lists[b].end());
        lo_v[b] = lo;
        hi_v[b] = hi;
        list_total += static_cast<long>(lists[b].size());
        max_list = std::max(max_list, static_cast<int>(lists[b].size()));
        max_range = std::max(max_range, hi - lo);
      }
      // list positions must fit the row word
      long direct_limit = 700000;   // REDs of the flush: a few microseconds, still far cheaper than partial vectors
      if (const char* e = dev_env("B200_DIRECT_LIMIT")) direct_limit = atol(e);
      direct_mode = 9 * list_total <= direct_limit && max_list <= static_cast<int>(kMetaLocalMask) && C <= static_cast<int>(kMetaCamMask);
      if (C > static_cast<int>(kMetaCamMask)) v2_possible = false;   // camera ids do not fit the row word: CTA-tile kernels
      if (direct_mode) {
        max_cam_span = max_list;
        for (int b = 0; b < num_ctas_v2; ++b) {
          cta_cam[b] = make_int2(static_cast<int>(cta_cams.size()), static_cast<int>(lists[b].size()));
          for (size_t i = 0; i < lists[b].size(); ++i) local_of[lists[b][i]] = static_cast<int>(i);
          auto pack = [&](int r0, int r1) {
            for (int r = r0; r < r1; ++r) row_meta[r] |= static_cast<uint32_t>(local_of[cam_idx[r]]) << kMetaLocalShift;
          };
          for (int t = cta_part[b].x; t < cta_part[b].y; ++t) pack(wtiles[t].row_begin, wtiles[t].row_begin + wtiles[t].row_count);
          for (int g = cta_big[b].x; g < cta_big[b].y; ++g) pack(big_tiles[g].obs_begin, big_tiles[g].obs_begin + big_tiles[g].obs_count);
          cta_cams.insert(cta_cams.end(), lists[b].begin(), lists[b].end());
        }
      } else {
        max_cam_span = max_range;
        for (int b = 0; b < num_ctas_v2; ++b) cta_cam[b] = make_int2(lo_v[b], hi_v[b]);
      }
    }
    // Shared memory budget: `replicas` private camera vectors + per-warp {TMA ring of F cells, exchange scratch}.
    // Prefer one replica per warp (no cross-warp contention) when the camera span of a CTA is small.
    const long total = static_cast<long>(prop.sharedMemPerBlockOptin) - 2048;
    const long sy1 = static_cast<long>(v2_sy_bytes(max_cam_span, 1));
    auto choose = [&](long cap, int max_stages, int* warps, int* stages_out, int* replicas) {
      *warps = 0;
      for (int stages = max_stages; stages >= 1 && *warps == 0; --stages) {
        const long pw = v2_per_warp_bytes(stages, kV2Scratch);
        long w = (total - sy1) / pw;                       // warps with a single shared copy
        long wr = total / (pw + sy1);                      // warps with one copy each
        if (wr >= cap) {                                    // everything fits with per-warp copies
          *warps = static_cast<int>(cap);
          *replicas = *warps;
          *stages_out = stages;
        } else if (w >= (stages >= 2 ? 8 : 4)) {
          *warps = static_cast<int>(std::min(w, cap));
          *stages_out = stages;
          *replicas = static_cast<int>(std::max<long>(1, std::min<long>(*warps, (total - *warps * pw) / sy1)));
        }
      }
    };
    choose(kV2MaxThreads / 32, 3, &v2_warps, &v2_stages, &v2_replicas);
    // the S*x kernel runs under 128 registers: up to 16 warps, 2-deep ring
    choose(kV3MaxThreads / 32, 2, &mul_warps, &mul_stages, &mul_replicas);
    if (const char* e = dev_env("B200_V3_WARPS")) {  // tuning knob
      const int w = atoi(e);
      if (w >= 1 && w <= mul_warps) { mul_warps = w; mul_replicas = std::min(mul_replicas, w); }
    }
    if (const char* e = dev_env("B200_V3_REPLICAS")) {
      const int r = atoi(e);
      if (r >= 1 && r <= mul_replicas) mul_replicas = r;
    }
    if (v2_warps == 0 || mul_warps == 0) v2_possible = false;  // camera vector does not fit next to the tile buffers: v1 kernels
  } else {
    v2_possible = false;
  }

  b200_handle* h = new b200_handle;
  h->device = desc->device;
  h->sm_count = prop.multiProcessorCount;
  h->C = C;
  h->P = P;
  h->N = N;
  h->np = 3 * P + 9 * C;
  h->num_tiles = static_cast<int>(tiles.size());
  h->loss_type = desc->loss_type;
  h->loss_a = desc->loss_a;
  h->rank = desc->world_size > 1 ? desc->rank : 0;
  h->world = desc->world_size > 1 ? desc->world_size : 1;
  std::memset(h->launches, 0, sizeof(h->launches));
  std::memset(h->ms, 0, sizeof(h->ms));
  std::memset(h->ops, 0, sizeof(h->ops));
  std::memset(h->bytes_per_op, 0, sizeof(h->bytes_per_op));
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
  if (h->world > 1) {
#ifdef B200_WITH_NCCL
    if (desc->nccl_unique_id == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "world_size > 1 needs nccl_unique_id");
    if (!load_nccl()) return fail(B200_ERR_NCCL, "cannot load libnccl.so.2: %s", dlerror());
    ncclUniqueId id;
    std::memcpy(&id, desc->nccl_unique_id, 128);
    ncclResult_t r = g_nccl.CommInitRank(&h->comm, h->world, id, h->rank);
    if (r != ncclSuccess) return fail(B200_ERR_NCCL, "ncclCommInitRank: %s", g_nccl.GetErrorString(r));
#else
    return fail(B200_ERR_UNSUPPORTED, "built without NCCL");
#endif
  }
  const size_t n = static_cast<size_t>(N);
  std::vector<int> pt_of_row(n);
  for (size_t i = 0; i < n; ++i) pt_of_row[i] = pt_idx[i];
  OK(dev_alloc(&h->d_tiles, tiles.size()));
  OK(dev_alloc(&h->d_cam_idx, n));
  OK(dev_alloc(&h->d_pt_ptr, static_cast<size_t>(P) + 1));
  OK(dev_alloc(&h->d_pt_of_row, n));
  OK(dev_alloc(&h->d_obs, 2 * n));
  OK(dev_alloc(&h->d_values, 24 * n));
  OK(dev_alloc(&h->d_state, h->np));
  OK(dev_alloc(&h->d_residuals, 2 * n));
  OK(dev_alloc(&h->d_gradient, h->np));
  OK(dev_alloc(&h->d_tile_partial, tiles.size() + num_ctas_v2 + big_tiles.size() + chunk_tiles.size() + 8));
  OK(dev_alloc(&h->d_fail, 4));
  OK(dev_alloc(&h->d_scalars, 64));
  OK(dev_alloc(&h->d_partial, kRedBlocks * 4));
  OK(dev_alloc(&h->d_vp0, h->np));
  OK(dev_alloc(&h->d_vp1, h->np));
  OK(dev_alloc(&h->d_vr0, 2 * n));
  OK(dev_alloc(&h->d_b, 2 * n));
  OK(dev_alloc(&h->d_D, h->np));
  OK(dev_alloc(&h->d_ete_inv, 6 * static_cast<size_t>(P)));
  OK(dev_alloc(&h->d_rhs, 9 * static_cast<size_t>(C)));
  OK(dev_alloc(&h->d_ye, 3 * static_cast<size_t>(P)));
  OK(dev_alloc(&h->d_upper45, 45 * static_cast<size_t>(C)));
  OK(dev_alloc(&h->d_minv, 81 * static_cast<size_t>(C)));
  OK(dev_alloc(&h->d_blocks, 81 * static_cast<size_t>(C)));
  OK(dev_alloc(&h->d_xr, 9 * static_cast<size_t>(C)));
  OK(dev_alloc(&h->d_p, 9 * static_cast<size_t>(C)));
  OK(dev_alloc(&h->d_r, 9 * static_cast<size_t>(C)));
  OK(dev_alloc(&h->d_z, 9 * static_cast<size_t>(C)));
  OK(dev_alloc(&h->d_tmp, 9 * static_cast<size_t>(C)));
  OK(dev_alloc(&h->d_sol, 9 * static_cast<size_t>(C)));
  OK(dev_alloc(&h->d_cg, 1));
  OK(dev_alloc(&h->d_ybig, 9 * static_cast<size_t>(C)));
  CU(cudaMemsetAsync(h->d_ybig, 0, sizeof(double) * 9 * C, h->stream));
  CU(cudaMemsetAsync(h->d_cg, 0, sizeof(CgState), h->stream));
  OK(dev_alloc(&h->d_scale, h->np));
  OK(dev_alloc(&h->d_sqnorm, h->np));
  OK(dev_alloc(&h->d_diagonal, h->np));
  OK(dev_alloc(&h->d_lmD, h->np));
  OK(dev_alloc(&h->d_step, h->np));
  OK(dev_alloc(&h->d_cand, h->np));
  OK(dev_alloc(&h->d_y, h->np));
  CU(cudaMallocHost(reinterpret_cast<void**>(&h->h_scalars), 64 * sizeof(double)));
  CU(cudaMallocHost(reinterpret_cast<void**>(&h->h_cg), 2 * sizeof(CgState)));
  CU(cudaEventCreateWithFlags(&h->ev_cg[0], cudaEventDisableTiming));
  CU(cudaEventCreateWithFlags(&h->ev_cg[1], cudaEventDisableTiming));
  CU(cudaMallocHost(reinterpret_cast<void**>(&h->h_fail), 4 * sizeof(int)));
  CU(cudaMemcpyAsync(h->d_tiles, tiles.data(), tiles.size() * sizeof(TileDesc), cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(h->d_cam_idx, cam_idx, n * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(h->d_pt_ptr, pt_ptr.data(), pt_ptr.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(h->d_pt_of_row, pt_of_row.data(), n * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemcpyAsync(h->d_obs, obs_i.data(), 2 * n * sizeof(double), cudaMemcpyHostToDevice, h->stream));
  CU(cudaMemsetAsync(h->d_values, 0, 24 * n * sizeof(double), h->stream));
  if (!identity_order) {
    OK(dev_alloc(&h->d_pt_perm, static_cast<size_t>(P)));
    OK(dev_alloc(&h->d_row_perm, n));
    OK(dev_alloc(&h->d_stage_p, h->np));
    OK(dev_alloc(&h->d_stage_r, 2 * n));
    CU(cudaMemcpyAsync(h->d_pt_perm, pt_perm.data(), sizeof(int) * P, cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_row_perm, row_perm.data(), sizeof(int) * n, cudaMemcpyHostToDevice, h->stream));
    h->h_pt_perm = pt_perm;
    h->permuted = true;
  }
  CU(cudaStreamSynchronize(h->stream));
  h->view.C = C;
  h->view.P = P;
  h->view.N = N;
  h->view.num_tiles = h->num_tiles;
  h->view.tiles = h->d_tiles;
  h->view.cam_idx = h->d_cam_idx;
  h->view.pt_ptr = h->d_pt_ptr;
  h->view.pt_of_row = h->d_pt_of_row;
  h->view.obs = h->d_obs;
  h->view.values = h->d_values;

  CU(cudaFuncSetAttribute(cam_blocks_v2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (kCamBlkThreads / 32) * kCamBlkWarpBytes));
  CU(cudaFuncSetAttribute(cam_blocks_v2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (kCamBlkThreads / 32) * kCamBlkWarpBytes));
  if (!has_dups && dev_env("B200_DISABLE_CAM_MAJOR") == nullptr) {
    h->num_cam_items = static_cast<int>(cam_items.size());
    OK(dev_alloc(&h->d_cam_items, cam_items.size()));
    OK(dev_alloc(&h->d_cam_rows, n));
    OK(dev_alloc(&h->d_q3, kQStride * n + 8));
    CU(cudaMemcpyAsync(h->d_cam_items, cam_items.data(), cam_items.size() * sizeof(CamItem), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_cam_rows, cam_rows.data(), n * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->cam_major_ok = true;
  }
  h->num_huge = static_cast<int>(huge_pts.size());
  if (h->num_huge > 0) {
    if (has_dups)
      return fail(B200_ERR_UNSUPPORTED,
                  "a point with more than %d observations together with duplicate (camera, point) observations is not supported", kTile);
    OK(dev_alloc(&h->d_huge_pts, huge_pts.size()));
    CU(cudaMemcpyAsync(h->d_huge_pts, huge_pts.data(), huge_pts.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
  }
  if (v2_possible) {
    // the slices of the huge points ride along with the >32-row points in every kernel that has no coupling between the
    // rows of a point (the partition above only covers the plain ones: cta_big indexes the first part of the array)
    const int num_plain_big = static_cast<int>(big_tiles.size());
    big_tiles.insert(big_tiles.end(), chunk_tiles.begin(), chunk_tiles.end());
    h->num_big_tiles = static_cast<int>(big_tiles.size());
    TileDesc* d_big = nullptr;
    OK(dev_alloc(&d_big, big_tiles.size()));
    h->view_big = h->view;
    h->view_big.tiles = d_big;
    h->view_big.num_tiles = h->num_big_tiles;
    h->view_chunks = h->view;
    h->view_chunks.tiles = d_big + num_plain_big;
    h->view_chunks.num_tiles = static_cast<int>(chunk_tiles.size());
    OK(dev_alloc(&h->d_wtiles, wtiles.size()));
    OK(dev_alloc(&h->d_row_meta, n));
    OK(dev_alloc(&h->d_cta_part, cta_part.size()));
    OK(dev_alloc(&h->d_cta_cam, cta_cam.size()));
    OK(dev_alloc(&h->d_partials, static_cast<size_t>(num_ctas_v2) * 9 * max_cam_span));
    if (!big_tiles.empty())
      CU(cudaMemcpyAsync(d_big, big_tiles.data(), big_tiles.size() * sizeof(TileDesc), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_wtiles, wtiles.data(), wtiles.size() * sizeof(WarpTile), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_row_meta, row_meta.data(), n * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_cta_part, cta_part.data(), cta_part.size() * sizeof(int2), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_cta_cam, cta_cam.data(), cta_cam.size() * sizeof(int2), cudaMemcpyHostToDevice, h->stream));
    OK(dev_alloc(&h->d_cta_big, cta_big.size()));
    CU(cudaMemcpyAsync(h->d_cta_big, cta_big.data(), cta_big.size() * sizeof(int2), cudaMemcpyHostToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->v2.p = h->view;
    h->v2.cta_big = h->d_cta_big;
    h->v2.big_tiles = d_big;
    h->v2.wtiles = h->d_wtiles;
    h->v2.row_meta = h->d_row_meta;
    h->v2.cta_part = h->d_cta_part;
    h->v2.cta_cam = h->d_cta_cam;
    h->v2.partials = h->d_partials;
    h->v2.num_ctas = num_ctas_v2;
    h->v2.max_cam_span = max_cam_span;
    h->v2.warps = v2_warps;
    h->v2.stages = v2_stages;
    h->v2.replicas = v2_replicas;
    h->v2.direct = direct_mode ? 1 : 0;
    OK(dev_alloc(&h->d_cta_cams, cta_cams.size()));
    if (!cta_cams.empty())
      CU(cudaMemcpyAsync(h->d_cta_cams, cta_cams.data(), cta_cams.size() * sizeof(int), cudaMemcpyHostToDevice, h->stream));
    h->v2.cta_cams = h->d_cta_cams;
    h->v2.per_warp_bytes = v2_per_warp_bytes(v2_stages, kV2Scratch);
    h->v2_smem = v2_sy_bytes(max_cam_span, v2_replicas) + static_cast<size_t>(v2_warps) * h->v2.per_warp_bytes;
    h->v2_mul = h->v2;
    {
      h->v2_mul.warps = mul_warps;
      h->v2_mul.stages = mul_stages;
      h->v2_mul.replicas = mul_replicas;
      h->v2_mul.per_warp_bytes = v2_per_warp_bytes(mul_stages, kV2Scratch);
      h->mul_smem = v2_sy_bytes(max_cam_span, mul_replicas) + static_cast<size_t>(mul_warps) * h->v2_mul.per_warp_bytes;
      h->mul_v3 = true;
      // the S*x kernel takes the >32-row points itself when its TMA rings can stage a kTile-row point
      h->big_folded = mul_warps >= kTile / 32 &&
                      static_cast<size_t>(mul_warps) * h->v2_mul.per_warp_bytes >= kTile * 192 + 160 &&
                      dev_env("B200_DISABLE_BIG_FOLD") == nullptr;
      CU(cudaFuncSetAttribute(schur_mul_v3_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
    }
    // v4 (all operands through the TMA ring, x staged in shared memory): needs the narrow camera ranges of the
    // direct-flush mode; up to 16 warps with a one-slot ring each, one private camera vector per warp when they fit.
    if (h->mul_v3 && h->v2.direct && dev_env("B200_MUL_V3") == nullptr) {
      const long total = static_cast<long>(prop.sharedMemPerBlockOptin) - 2048;
      const long sy1 = static_cast<long>(v2_sy_bytes(max_cam_span, 1));
      int w4 = kV4MaxThreads / 32;
      if (const char* e = dev_env("B200_V4_WARPS")) w4 = std::max(4, std::min(w4, atoi(e)));
      int st4 = 1;  // the slot is refilled as soon as its contents are in registers: one stage per warp, more warps
      if (const char* e = dev_env("B200_V4_STAGES")) st4 = std::max(1, std::min(3, atoi(e)));
      for (; w4 >= 8; --w4) {
        const long rem = total - static_cast<long>(w4) * v4_per_warp_bytes(st4) - sy1 /* staged x */;
        if (rem < sy1) continue;
        int rep4 = static_cast<int>(std::min<long>(w4, rem / sy1));
        if (const char* e = dev_env("B200_V4_REPLICAS")) rep4 = std::max(1, std::min(rep4, atoi(e)));
        std::vector<uint32_t> meta(static_cast<size_t>(wtiles.size()) * kV4MetaWords, 0u);
        for (int b = 0; b < num_ctas_v2; ++b)
          for (int t = cta_part[b].x; t < cta_part[b].y; ++t) {
            uint32_t* m = meta.data() + static_cast<size_t>(t) * kV4MetaWords;
            const WarpTile& wt = wtiles[t];
            for (int r = 0; r < wt.row_count; ++r) m[r] = row_meta[wt.row_begin + r];
            m[32] = static_cast<uint32_t>(wt.row_begin);
            m[33] = static_cast<uint32_t>(wt.pt_begin);
            m[34] = static_cast<uint32_t>(wt.row_count) | (static_cast<uint32_t>(wt.pt_count) << 16);
            {
              int maxdeg = 1;   // longest point of the tile (rows): bounds the segmented reductions
              for (int k = 0; k < wt.pt_count; ++k) maxdeg = std::max(maxdeg, pt_ptr[wt.pt_begin + k + 1] - pt_ptr[wt.pt_begin + k]);
              m[35] = static_cast<uint32_t>(maxdeg);
            }
            const int tn = t + w4 * st4;
            if (tn < cta_part[b].y) {
              m[36] = static_cast<uint32_t>(wtiles[tn].row_begin);
              m[37] = static_cast<uint32_t>(wtiles[tn].pt_begin);
              m[38] = static_cast<uint32_t>(wtiles[tn].row_count) | (static_cast<uint32_t>(wtiles[tn].pt_count) << 16);
            }
          }
        OK(dev_alloc(&h->d_tile_meta, meta.size()));
        CU(cudaMemcpyAsync(h->d_tile_meta, meta.data(), meta.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, h->stream));
        CU(cudaStreamSynchronize(h->stream));
        h->v2_mul.warps = w4;
        h->v2_mul.stages = st4;
        h->v2_mul.replicas = rep4;
        h->v2_mul.per_warp_bytes = v4_per_warp_bytes(st4);
        h->v2_mul.tile_meta = h->d_tile_meta;
        h->v2_mul.stage_x = 1;
        if (const char* e = dev_env("B200_VARIANT")) h->v2_mul.variant = atoi(e);
        h->mul_smem = v2_sy_bytes(max_cam_span, rep4) + v4_sx_bytes(max_cam_span, 1) + static_cast<size_t>(w4) * h->v2_mul.per_warp_bytes;
        h->mul_v4 = true;
        h->big_folded = dev_env("B200_DISABLE_BIG_FOLD") == nullptr;
        h->mul_v4_owned = rep4 == w4;
        CU(cudaFuncSetAttribute(schur_init_v4_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
        CU(cudaFuncSetAttribute(schur_init_v4_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
        CU(cudaFuncSetAttribute(jtj_v4_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
        CU(cudaFuncSetAttribute(jtj_v4_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
        CU(cudaFuncSetAttribute(schur_mul_v4_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
        CU(cudaFuncSetAttribute(schur_mul_v4_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
        break;
      }
    }
    // function attributes are process-wide: always raise them to the device limit, never to this handle's need
    CU(cudaFuncSetAttribute(jtj_v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
    if (!h->big_folded) {
      // the S*x kernel must not take the >32-row points itself when they are handled by a separate launch
      int2* none = nullptr;
      OK(dev_alloc(&none, static_cast<size_t>(num_ctas_v2)));
      CU(cudaMemsetAsync(none, 0, sizeof(int2) * num_ctas_v2, h->stream));
      h->d_cta_big_none = none;
      h->v2_mul.cta_big = none;
    }
    h->v2_ok = true;
    if (h->v2.direct && dev_env("B200_DISABLE_V2B") == nullptr) {
      const size_t lim = prop.sharedMemPerBlockOptin - 2048;
      // Each kernel gets as many replicas of its private accumulators as fit next to its per-warp buffers
      // (one per warp at best), and a shallower TMA ring if even a single replica would not fit.
      const size_t sy1 = v2_sy_bytes(max_cam_span, 1);
      auto fit = [&](size_t per_warp, size_t acc1, int* replicas) -> size_t {
        const size_t fixed = per_warp * v2_warps;
        if (fixed + acc1 > lim) return lim + 1;
        *replicas = static_cast<int>(std::min<size_t>(v2_warps, (lim - fixed) / acc1));
        return fixed + acc1 * *replicas;
      };
      // evaluate: two accumulators (gradient, column norms) + per-warp staging
      h->v2_eval = h->v2;
      h->eval_v2_smem = fit(eval_v2_per_warp_bytes(), 2 * sy1, &h->v2_eval.replicas);
      // schur_init: same ring as S*x with a 9-double exchange scratch
      h->v2_init = h->v2;
      h->init_v2_smem = lim + 1;
      for (int st = v2_stages; st >= 1 && h->init_v2_smem > lim; --st) {
        h->v2_init.stages = st;
        h->v2_init.per_warp_bytes = v2_per_warp_bytes(st, kInitScratch);
        h->init_v2_smem = fit(h->v2_init.per_warp_bytes, sy1, &h->v2_init.replicas);
      }
      // diag blocks: 45 doubles per camera
      h->v2_diag = h->v2;
      h->diag_v2_smem = lim + 1;
      h->diag_v2_replicas = 0;
      for (int st = v2_stages; st >= 1 && h->diag_v2_smem > lim; --st) {
        h->v2_diag.stages = st;
        h->diag_v2_smem = fit(diag_v2_per_warp_bytes(st), diag_v2_acc_stride(max_cam_span) * 8, &h->diag_v2_replicas);
      }
      if (h->diag_v2_smem > lim) h->diag_v2_replicas = 0;  // falls back to the CTA-tile kernel
      if (h->eval_v2_smem <= lim && h->init_v2_smem <= lim) {
        CU(cudaFuncSetAttribute(evaluate_v2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
        CU(cudaFuncSetAttribute(evaluate_v2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
        CU(cudaFuncSetAttribute(schur_init_v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
        CU(cudaFuncSetAttribute(diag_blocks_v2_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
        CU(cudaFuncSetAttribute(diag_blocks_v2_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(prop.sharedMemPerBlockOptin) - 1024));
        h->v2b_ok = true;
      }
    }
  }

  if (h->mul_v4) {
    // L2 residency plan of S*x.  J does not change during a PCG, and every product streams the same bytes (F, E,
    // (E'E+D^2)^-1 blocks, descriptors: 141 MB on Ladybug-1723); under the default policy a stream larger than L2 leaves
    // nothing behind for the next product.  So a fixed share of the tiles, spread evenly through every CTA's tile range
    // (HBM keeps streaming while the resident tiles are read from L2), is copied with evict_normal and the rest with
    // evict_first: the resident share then survives from one product to the next.  The budget is kL2ResidentShare of the
    // L2 minus the working set of the CG loop, which is read with the default policy; a stream within the budget is all
    // resident.  Whole tiles: the four copies of a tile share one policy.
    int l2_bytes = 0;
    CU(cudaDeviceGetAttribute(&l2_bytes, cudaDevAttrL2CacheSize, h->device));
    double stream_bytes = 0.0;
    for (int b = 0; b < num_ctas_v2; ++b) {
      for (int t = cta_part[b].x; t < cta_part[b].y; ++t) stream_bytes += 192.0 * wtiles[t].row_count + 48.0 * wtiles[t].pt_count + 4 * kV4MetaWords;
      for (int t = cta_big[b].x; t < cta_big[b].y; ++t) stream_bytes += 192.0 * big_tiles[t].obs_count;
    }
    const double working_set = 8.0 * (8 * 9 + 81) * C                                  // rhs x r z p q seed D_f, minv
                               + (h->world > 1 ? 2.0 * h->world * 16 * 9 * C : 0.0);    // peer exchange slots
    double budget = std::max(0.0, kL2ResidentShare * l2_bytes - working_set);
    const char* dev_mb = dev_env("B200_L2_RESIDENT_MB");   // 0: no plan, every copy with the default policy
    if (dev_mb != nullptr) budget = atof(dev_mb) * (1 << 20);
    if (const char* e = dev_env("B200_L2_RESIDENT_POLICY")) h->v2_mul.l2_last = strcmp(e, "last") == 0 ? 1 : 0;
    const bool no_plan = dev_mb != nullptr && budget <= 0.0;
    h->v2_mul.l2_stream = (budget >= stream_bytes || no_plan) ? 0u : static_cast<uint32_t>(std::ceil(65536.0 * (1.0 - budget / stream_bytes)));
    if (getenv("B200_VERBOSE") != nullptr) {
      // what the plan marks, counted the way the kernel decides it
      const uint64_t s = h->v2_mul.l2_stream;
      auto streamed = [&](int i) { return ((static_cast<uint64_t>(i) + 1) * s >> 16) != (static_cast<uint64_t>(i) * s >> 16); };
      double res = 0.0;
      for (int b = 0; b < num_ctas_v2; ++b) {
        for (int t = cta_part[b].x; t < cta_part[b].y; ++t)
          if (!streamed(t - cta_part[b].x)) res += 192.0 * wtiles[t].row_count + 48.0 * wtiles[t].pt_count + 4 * kV4MetaWords;
        for (int t = cta_big[b].x; t < cta_big[b].y; ++t)
          if (!streamed(t - cta_big[b].x)) res += 192.0 * big_tiles[t].obs_count;
      }
      fprintf(stderr, "[b200ba] S*x L2 plan (L2 %d MiB, budget %.1f MiB): resident %.1f MiB, streamed %.1f MiB, stride %.2f tiles (%s)\n",
              l2_bytes >> 20, budget / (1 << 20), res / (1 << 20), (stream_bytes - res) / (1 << 20), s < 65536 ? 65536.0 / (65536 - s) : 0.0,
              h->v2_mul.l2_last ? "evict_last" : "evict_normal");
    }
  }
  if (getenv("B200_VERBOSE") != nullptr)
    // mul: the S*x family (tile = the CTA-tile kernels everywhere); diag: the block-diagonal pass precond_update_dev runs
    fprintf(stderr,
            "[b200ba] C=%d P=%d N=%d wtiles=%zu big(+slices)=%zu huge=%d span=%d direct=%d v2(w=%d,s=%d,r=%d) mul(%s w=%d,s=%d,r=%d,smem=%zu) folded=%d v2b=%d cam_major=%d diag=%s\n",
            C, P, N, wtiles.size(), big_tiles.size(), h->num_huge, max_cam_span, h->v2.direct, h->v2.warps, h->v2.stages, h->v2.replicas,
            !h->v2_ok ? "tile" : h->mul_v4 ? (h->mul_v4_owned ? "v4-owned" : "v4") : "v3", h->v2_mul.warps, h->v2_mul.stages, h->v2_mul.replicas, h->mul_smem,
            h->big_folded ? 1 : 0, h->v2b_ok ? 1 : 0, h->cam_major_ok ? 1 : 0,
            h->cam_major_ok ? "cam_major" : (h->v2b_ok && h->diag_v2_replicas > 0) ? "v2" : "tile");
  // Explicit or implicit S (DESIGN §1): explicit when the product on the stored upper triangle reads clearly fewer bytes
  // than the implicit product streams and the storage fits; sharded handles stay implicit.
  XsPattern xp;
  double xs_mul_bytes = 0.0, xs_asm_bytes = 0.0;
  if (h->world == 1) {
    int l2_bytes = 0;
    CU(cudaDeviceGetAttribute(&l2_bytes, cudaDevAttrL2CacheSize, h->device));
    const double l2_budget = kL2ResidentShare * l2_bytes - 8.0 * (8 * 9 + 81) * C;   // as the S*x residency plan
    xs_pattern(C, N, cam_idx, pt_idx, pt_ptr.data(), &xp);
    const double nb = static_cast<double>(xp.blk_row.size()), npairs = static_cast<double>(xp.pairs.size());
    const double implicit_bytes = 196.0 * N + 52.0 * P + 216.0 * C;
    xs_mul_bytes = 648.0 * xp.list.size() + 8.0 * xp.list.size() + 216.0 * C;   // blocks as listed (off-diagonal twice), list, x, y
    const double storage = 648.0 * nb + 8.0 * npairs + 12.0 * nb;
    h->xs = implicit_bytes >= kXsByteRatio * xs_mul_bytes && implicit_bytes > l2_budget && storage <= kXsMaxBytes && npairs < 2.0e9;
    if (const char* e = dev_env("B200_EXPLICIT_S")) h->xs = atoi(e) != 0 && npairs < 2.0e9;
    // J, point of each row, (E'E+D^2)^-1, row pairs, block table; S and the diagonal upper triangles written
    xs_asm_bytes = 196.0 * N + 48.0 * P + 8.0 * npairs + 12.0 * nb + 648.0 * nb + 360.0 * C;
    if (getenv("B200_VERBOSE") != nullptr)
      fprintf(stderr, "[b200ba] S plan: %s, %lld pairs, %.1f MB\n", h->xs ? "explicit" : "implicit", xp.off_blocks, 648.0 * nb / 1e6);
  } else if (getenv("B200_VERBOSE") != nullptr) {
    fprintf(stderr, "[b200ba] S plan: implicit, sharded\n");
  }
  if (h->xs) {
    const int nb = static_cast<int>(xp.blk_row.size());
    // product warp groups: contiguous camera ranges balanced by list length (+ a per-camera overhead)
    const int groups_want = std::max(1, std::min(C, 4 * h->sm_count * kXsGroups));
    h->xs_grid = (groups_want + kXsGroups - 1) / kXsGroups;
    const int nw = h->xs_grid * kXsGroups;
    std::vector<int> warp_cam(static_cast<size_t>(nw) + 1, C);
    {
      const double per_cam = 4.0;
      const double total = static_cast<double>(xp.list.size()) + per_cam * C;
      double cum = 0.0;
      int w = 0;
      for (int i = 0; i < C; ++i) {
        const int owner = std::min(nw - 1, static_cast<int>(cum * nw / total));
        while (w <= owner) warp_cam[w++] = i;
        cum += (xp.list_ptr[i + 1] - xp.list_ptr[i]) + per_cam;
      }
      // warps past the last owner start (and end) at C
    }
    OK(dev_alloc(&h->d_xs_blk_row, static_cast<size_t>(nb)));
    OK(dev_alloc(&h->d_xs_blk_col, static_cast<size_t>(nb)));
    OK(dev_alloc(&h->d_xs_pair_ptr, static_cast<size_t>(nb) + 1));
    OK(dev_alloc(&h->d_xs_pairs, xp.pairs.size()));
    OK(dev_alloc(&h->d_xs_list_ptr, static_cast<size_t>(C) + 1));
    OK(dev_alloc(&h->d_xs_list, xp.list.size()));
    OK(dev_alloc(&h->d_xs_warp_cam, warp_cam.size()));
    OK(dev_alloc(&h->d_xs_S, 81 * static_cast<size_t>(nb)));
    std::vector<int> order;
    order.reserve(static_cast<size_t>(nb));
    for (int b = 0; b < nb; ++b)
      if (xp.pair_ptr[b + 1] - xp.pair_ptr[b] > kXsLongPairs) order.push_back(b);
    h->num_xs_long = static_cast<int>(order.size());
    for (int b = 0; b < nb; ++b)
      if (xp.pair_ptr[b + 1] - xp.pair_ptr[b] <= kXsLongPairs) order.push_back(b);
    h->num_xs_short = nb - h->num_xs_long;
    OK(dev_alloc(&h->d_xs_order, static_cast<size_t>(nb)));
    CU(cudaMemcpyAsync(h->d_xs_order, order.data(), sizeof(int) * nb, cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_xs_blk_row, xp.blk_row.data(), sizeof(int) * nb, cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_xs_blk_col, xp.blk_col.data(), sizeof(int) * nb, cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_xs_pair_ptr, xp.pair_ptr.data(), sizeof(int) * (nb + 1), cudaMemcpyHostToDevice, h->stream));
    if (!xp.pairs.empty())
      CU(cudaMemcpyAsync(h->d_xs_pairs, xp.pairs.data(), sizeof(int2) * xp.pairs.size(), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_xs_list_ptr, xp.list_ptr.data(), sizeof(int) * (C + 1), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_xs_list, xp.list.data(), sizeof(int2) * xp.list.size(), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync(h->d_xs_warp_cam, warp_cam.data(), sizeof(int) * warp_cam.size(), cudaMemcpyHostToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    h->xsv.C = C;
    h->xsv.num_blocks = nb;
    h->xsv.blk_row = h->d_xs_blk_row;
    h->xsv.blk_col = h->d_xs_blk_col;
    h->xsv.pair_ptr = h->d_xs_pair_ptr;
    h->xsv.pairs = h->d_xs_pairs;
    h->xsv.list_ptr = h->d_xs_list_ptr;
    h->xsv.list = h->d_xs_list;
    h->xsv.warp_cam = h->d_xs_warp_cam;
    h->xsv.S = h->d_xs_S;
  }
  for (int k = 0; k < K_COUNT; ++k) h->grid_tile[k] = std::max(1, std::min(h->num_tiles, h->sm_count * 4));
  h->grid_tile[K_EVAL_JAC] = tile_grid(h, evaluate_kernel<true>, tile_smem_bytes<3, 1>());
  h->grid_tile[K_EVAL_COST] = tile_grid(h, evaluate_kernel<false>, tile_smem_bytes<3, 1>());
  h->grid_tile[K_SQNORM] = tile_grid(h, sqnorm_kernel, tile_smem_bytes<3, 1>());
  h->grid_tile[K_JMUL] = tile_grid(h, jmul_kernel, tile_smem_bytes<1, 1>());
  h->grid_tile[K_JTMUL] = tile_grid(h, jtmul_kernel<false>, tile_smem_bytes<3, 1>());
  h->grid_tile[K_JTJ] = tile_grid(h, jtmul_kernel<true>, tile_smem_bytes<3, 1>());
  h->grid_tile[K_SCHUR_INIT] = tile_grid(h, schur_init_kernel, tile_smem_bytes<9, 3>());
  h->grid_tile[K_SCHUR_MUL] = tile_grid(h, schur_mul_kernel, tile_smem_bytes<3, 3>());
  h->grid_tile[K_DIAG_BLOCKS] = tile_grid(h, diag_blocks_kernel<true>, tile_smem_bytes<1, 1>());
  h->grid_tile[K_BACKSUB] = tile_grid(h, backsub_kernel, tile_smem_bytes<3, 1>());
  h->grid_tile[K_MODEL_COST] = tile_grid(h, model_cost_kernel, tile_smem_bytes<1, 1>());
  {
    int per_sm = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cg_vector_kernel, kCgThreads, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
    const int nblocks = (C + kCgCamsPerCta - 1) / kCgCamsPerCta;
    h->cg_grid = std::max(1, std::min(nblocks, per_sm * h->sm_count));
    OK(dev_alloc(&h->d_red, static_cast<size_t>(h->cg_grid) * 4));
    OK(dev_alloc(&h->d_seed_pq, static_cast<size_t>(h->cg_grid)));
    const int num_pq_parts = std::max(prop.multiProcessorCount, h->xs_grid);   // v4 or explicit-S product CTAs
    OK(dev_alloc(&h->d_pq_parts, static_cast<size_t>(num_pq_parts)));
#ifdef B200_WITH_NCCL
    if (h->world > 1 && h->world <= kMaxXchgRanks && dev_env("B200_NO_PEER_EXCHANGE") == nullptr) {
      // Peer exchange buffers: allocated with cudaMalloc, exported with CUDA IPC, the handles all-gathered through the NCCL
      // communicator (the only plumbing the ranks share), every peer's buffer mapped into this process.  Any failure
      // (no P2P path, IPC unavailable in the launch mode) leaves the NCCL all-reduce in place -- decided jointly.
      const size_t nC = 9 * static_cast<size_t>(C);
      OK(dev_alloc(&h->d_xchg, 2 * static_cast<size_t>(h->world) * (nC + 1)));
      CU(cudaMemsetAsync(h->d_xchg, 0, sizeof(uint4) * 2 * h->world * (nC + 1), h->stream));   // epoch 0 is never used
      unsigned char* d_handles = nullptr;
      OK(dev_alloc(&d_handles, static_cast<size_t>(h->world) * 64));
      std::vector<unsigned char> hh(static_cast<size_t>(h->world) * 64, 0);
      cudaIpcMemHandle_t mine;
      bool ok = cudaIpcGetMemHandle(&mine, h->d_xchg) == cudaSuccess;
      if (!ok) cudaGetLastError();
      static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
      std::memcpy(hh.data() + 64 * h->rank, &mine, 64);
      CU(cudaMemcpyAsync(d_handles + 64 * h->rank, hh.data() + 64 * h->rank, 64, cudaMemcpyHostToDevice, h->stream));
      ncclResult_t r = g_nccl.AllGather(d_handles + 64 * h->rank, d_handles, 64, ncclChar, h->comm, h->stream);
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
#endif
    CU(cudaMemsetAsync(h->d_seed_pq, 0, sizeof(double) * h->cg_grid, h->stream));
    CU(cudaMemsetAsync(h->d_pq_parts, 0, sizeof(double) * num_pq_parts, h->stream));
  }

  // Algorithmic (compulsory) bytes per launch, SURVEY §8d with this layout: J values 192 B/row + 4 B camera
  // index per row + 4 B chunk boundary per point, plus the vectors each kernel must read/write once.
  const double Nn = N, Pp = P, Cc = C;
  h->bytes_per_op[K_JTJ] = 196 * Nn + 4 * Pp + 24.0 * (3 * Pp + 9 * Cc);
  h->bytes_per_op[K_SCHUR_MUL] = 196 * Nn + 52 * Pp + 216 * Cc;
  h->bytes_per_op[K_SCHUR_INIT] = 196 * Nn + 16 * Nn + 4 * Pp + 24 * Pp + 48 * Pp + 72 * Cc;   // J, b, chunk ids, D_e, (E'E)^-1 out, rhs out
  h->bytes_per_op[K_DIAG_BLOCKS] = 196 * Nn + 52 * Pp + 360 * Cc;
  h->bytes_per_op[K_BACKSUB] = 196 * Nn + 16 * Nn + 52 * Pp + 24 * Pp + 72 * Cc;
  h->bytes_per_op[K_EVAL_JAC] = 192 * Nn + 16 * Nn + 16 * Nn + 4 * Nn + 4 * Pp + 2 * 8.0 * (3 * Pp + 9 * Cc);
  h->bytes_per_op[K_EVAL_COST] = 16 * Nn + 4 * Nn + 4 * Pp + 8.0 * (3 * Pp + 9 * Cc);
  h->bytes_per_op[K_SQNORM] = 196 * Nn + 4 * Pp + 8.0 * (3 * Pp + 9 * Cc);
  h->bytes_per_op[K_SCALE] = 2 * 192 * Nn + 8 * Nn + 8.0 * (3 * Pp + 9 * Cc);
  h->bytes_per_op[K_JMUL] = 196 * Nn + 32 * Nn + 4 * Pp + 8.0 * (3 * Pp + 9 * Cc);
  h->bytes_per_op[K_JTMUL] = 196 * Nn + 16 * Nn + 4 * Pp + 16.0 * (3 * Pp + 9 * Cc);
  h->bytes_per_op[K_PMV_RIGHT_E] = 48 * Nn + 4 * Nn + 32 * Nn + 24 * Pp;            // E cells, point id, y read + written, x_e
  h->bytes_per_op[K_PMV_RIGHT_F] = 144 * Nn + 4 * Nn + 32 * Nn + 72 * Cc;           // F cells, camera id, y read + written, x_f
  h->bytes_per_op[K_PMV_LEFT_E] = 48 * Nn + 16 * Nn + 4 * Pp + 48 * Pp;             // E cells, y, chunk boundaries, x_e read + written
  h->bytes_per_op[K_PMV_LEFT_F] = 144 * Nn + 16 * Nn + 4 * Nn + 144 * Cc;           // F cells, y, row list, x_f read + written
  h->bytes_per_op[K_MODEL_COST] = 196 * Nn + 16 * Nn + 4 * Pp + 8.0 * (3 * Pp + 9 * Cc);
  if (h->xs) {   // explicit S: the product and the assembly that replaces the block-diagonal pass
    h->bytes_per_op[K_SCHUR_MUL] = xs_mul_bytes;
    h->bytes_per_op[K_DIAG_BLOCKS] = xs_asm_bytes;
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
  void* dev_ptrs[] = {h->d_xchg, h->d_tiles, h->d_cam_idx, h->d_pt_ptr, h->d_pt_of_row, h->d_obs, h->d_values, h->d_state,
                      h->d_residuals, h->d_gradient, h->d_tile_partial, h->d_fail, h->d_scalars, h->d_partial,
                      h->d_vp0, h->d_vp1, h->d_vr0, h->d_b, h->d_D, h->d_ete_inv, h->d_rhs, h->d_ye, h->d_upper45,
                      h->d_minv, h->d_blocks, h->d_xr, h->d_p, h->d_r, h->d_z, h->d_tmp, h->d_sol, h->d_cg,
                      h->d_scale, h->d_sqnorm, h->d_diagonal, h->d_lmD, h->d_step, h->d_cand, h->d_y, h->d_wtiles,
                      h->d_row_meta, h->d_cta_part, h->d_cta_cam, h->d_cta_cams, h->d_cta_big, h->d_cta_big_none, h->d_tile_meta, h->d_pq_parts, h->d_seed_pq, h->d_huge_pts, h->d_dense_s, h->d_dense_work, h->d_dense_info, h->d_ftf_inv, h->d_spse[0], h->d_spse[1], h->d_spse[2], h->d_partials, h->d_ybig, h->d_red, h->d_cam_items, h->d_cam_rows, h->d_q3, h->d_pt_perm, h->d_row_perm, h->d_stage_p, h->d_stage_r,
                      h->d_xs_blk_row, h->d_xs_blk_col, h->d_xs_pair_ptr, h->d_xs_list_ptr, h->d_xs_warp_cam, h->d_xs_order, h->d_xs_pairs, h->d_xs_list, h->d_xs_S,
                      const_cast<TileDesc*>(h->view_big.tiles)};
  for (void* p : dev_ptrs)
    if (p != nullptr) cudaFree(p);
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

int b200_plus(b200_handle* h, const double* x, const double* delta, double* x_plus_delta) {
  if (h == nullptr || x == nullptr || delta == nullptr || x_plus_delta == nullptr)
    return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  for (int i = 0; i < h->np; ++i) x_plus_delta[i] = x[i] + delta[i];  // Euclidean blocks: program.cc:114-142
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
  const size_t nr = 2 * static_cast<size_t>(h->N);
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
  OK(launch(h, K_MODEL_COST, [&] {
    model_cost_kernel<<<h->grid_tile[K_MODEL_COST], kTile, tile_smem_bytes<1, 1>(), h->stream>>>(h->view, h->d_vp0, h->d_residuals, h->d_tile_partial);
  }));
  OK(launch(h, K_MISC, [&] { sum_kernel<<<1, kVecThreads, 0, h->stream>>>(h->num_tiles, h->d_tile_partial, h->d_scalars + 1); }));
  OK(allreduce_sum(h, h->d_scalars + 1, 1));
  CU(cudaMemcpyAsync(h->h_scalars + 1, h->d_scalars + 1, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  CU(cudaStreamSynchronize(h->stream));
  *model_cost_change = h->h_scalars[1];
  return B200_OK;
}

int b200_jacobian_left_multiply(b200_handle* h, const double* x, double* y) {
  if (h == nullptr || x == nullptr || y == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(h->device));
  const size_t nr = 2 * static_cast<size_t>(h->N);
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
      if (h->cam_major_ok)
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
  if (h->mul_v4 && h->v2.direct) {
    // one launch (jtj_v4_kernel): the camera part of y is seeded with D_c^2 x_c (9C elements), the tile kernel writes the
    // point part and adds J'(J x) into the camera part; only the slices of >kTile-row points need a second launch
    OK(launch(h, K_MISC, [&] {
      diag_sq_mul_kernel<<<flat_grid(h, nc, 256), 256, 0, h->stream>>>(nc, seedD, h->d_vp0 + off, h->d_vp1 + off, nullptr);
    }));
    OK(huge_zero(h, h->d_vp1));  // the chunk tiles of huge points add their own D^2 x
    V2View jv = h->v2_mul;
    jv.cta_big = h->d_cta_big;   // the kernel takes the CTA's 33..kTile-row points itself
    OK(launch(h, K_JTJ, [&] {
      if (h->mul_v4_owned) jtj_v4_kernel<true><<<h->v2.num_ctas, 32 * h->v2_mul.warps, h->mul_smem, h->stream>>>(jv, h->d_vp0, dD, h->d_vp1);
      else jtj_v4_kernel<false><<<h->v2.num_ctas, 32 * h->v2_mul.warps, h->mul_smem, h->stream>>>(jv, h->d_vp0, dD, h->d_vp1);
    }));
    if (h->view_chunks.num_tiles > 0)
      OK(launch(h, K_JTJ, [&] {
        jtmul_kernel<true><<<std::min(h->view_chunks.num_tiles, h->sm_count * 4), kTile, tile_smem_bytes<3, 1>(), h->stream>>>(h->view_chunks, h->d_vp0, dD, h->d_vp1);
      }, false));
    OK(allreduce_sum(h, h->d_vp1 + off, 9 * static_cast<size_t>(h->C)));
    return down_params(h, y, h->d_vp1);
  }
  OK(huge_zero(h, h->d_vp1));  // point entries of huge points are accumulated slice by slice
  if (h->v2_ok) {
    if (h->v2.direct)
      OK(launch(h, K_MISC, [&] {
        diag_sq_mul_kernel<<<flat_grid(h, nc, 256), 256, 0, h->stream>>>(nc, seedD, h->d_vp0 + off, h->d_vp1 + off, nullptr);
      }));
    OK(launch(h, K_JTJ, [&] {
      jtj_v2_kernel<<<h->v2.num_ctas, 32 * h->v2.warps, h->v2_smem, h->stream>>>(h->v2, h->d_vp0, dD, h->d_vp1);
    }));
    if (!h->v2.direct)
      OK(launch(h, K_CAM_REDUCE, [&] {
        cam_reduce_kernel<<<(nc + 63) / 64, 256, h->v2.num_ctas * sizeof(int2), h->stream>>>(
            nc, h->v2.num_ctas, h->d_cta_cam, h->d_partials, 9 * h->v2.max_cam_span, seedD, h->d_vp0 + off, h->d_vp1 + off, 0, nullptr);
      }));
    if (h->num_big_tiles > 0)
      OK(launch(h, K_JTJ, [&] {
        jtmul_kernel<true><<<std::min(h->num_big_tiles, h->sm_count * 4), kTile, tile_smem_bytes<3, 1>(), h->stream>>>(h->view_big, h->d_vp0, dD, h->d_vp1);
      }, false));
  } else {
    OK(launch(h, K_MISC, [&] {
      diag_sq_mul_kernel<<<flat_grid(h, nc, 256), 256, 0, h->stream>>>(nc, seedD, h->d_vp0 + off, h->d_vp1 + off, nullptr);
    }));
    OK(launch(h, K_JTJ, [&] {
      jtmul_kernel<true><<<h->grid_tile[K_JTJ], kTile, tile_smem_bytes<3, 1>(), h->stream>>>(h->view, h->d_vp0, dD, h->d_vp1);
    }));
  }
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
  OK(dev_alloc(&tmp, 24 * n));
  int rc = permute_blocks(h, false, n, 6, h->d_row_perm, h->d_values, tmp);
  if (rc == B200_OK) rc = permute_blocks(h, false, n, 18, h->d_row_perm, h->d_values + 6 * n, tmp + 6 * n);
  if (rc == B200_OK) rc = d2h(h, values, tmp, sizeof(double) * 24 * n);
  cudaFree(tmp);
  return rc;
}
int b200_jacobian_set_values(b200_handle* h, const double* values) {
  if (h == nullptr || values == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(h->device));
  h->xs_ready = false;   // S is a function of J
  const size_t n = static_cast<size_t>(h->N);
  if (!h->permuted) {
    OK(h2d(h, h->d_values, values, sizeof(double) * 24 * n));
    CU(cudaStreamSynchronize(h->stream));
    return B200_OK;
  }
  double* tmp = nullptr;
  OK(dev_alloc(&tmp, 24 * n));
  int rc = h2d(h, tmp, values, sizeof(double) * 24 * n);
  if (rc == B200_OK) rc = permute_blocks(h, true, n, 6, h->d_row_perm, tmp, h->d_values);
  if (rc == B200_OK) rc = permute_blocks(h, true, n, 18, h->d_row_perm, tmp + 6 * n, h->d_values + 6 * n);
  cudaStreamSynchronize(h->stream);
  cudaFree(tmp);
  return rc;
}

// ------------------------------------------------------------------------------------------------ LinearSolver
int b200_schur_solve(b200_handle* h, const double* b, const double* D, const b200_solver_options* opts, double* x,
                     b200_solver_summary* summary) {
  if (h == nullptr || opts == nullptr || x == nullptr || summary == nullptr)
    return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  if (b == nullptr && !h->residuals_resident)
    return fail(B200_ERR_INVALID_ARGUMENT, "b == NULL means the residuals of the last b200_evaluate, and there are none");
  CU(cudaSetDevice(h->device));
  const double* d_b = h->d_residuals;
  if (b != nullptr) {
    OK(up_rows(h, h->d_b, b));
    d_b = h->d_b;
  }
  if (D != nullptr) OK(up_params(h, h->d_D, D));
  OK(schur_solve_dev(h, d_b, D != nullptr ? h->d_D : nullptr, opts, h->d_y, summary));
  if (summary->termination_type != B200_LS_FAILURE && summary->termination_type != B200_LS_FATAL_ERROR)
    OK(down_params(h, x, h->d_y));
  return B200_OK;
}

int b200_dense_schur_solve(b200_handle* h, const double* b, const double* D, double* x, b200_solver_summary* summary) {
  if (h == nullptr || x == nullptr || summary == nullptr) return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  if (b == nullptr && !h->residuals_resident)
    return fail(B200_ERR_INVALID_ARGUMENT, "b == NULL means the residuals of the last b200_evaluate, and there are none");
  CU(cudaSetDevice(h->device));
  const double* d_b = h->d_residuals;
  if (b != nullptr) {
    OK(up_rows(h, h->d_b, b));
    d_b = h->d_b;
  }
  if (D != nullptr) OK(up_params(h, h->d_D, D));
  OK(dense_schur_solve_dev(h, d_b, D != nullptr ? h->d_D : nullptr, h->d_y, summary));
  if (summary->termination_type == B200_LS_SUCCESS) OK(down_params(h, x, h->d_y));
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
  if (h->xs) OK(xs_mul_dev(h, h->d_xr, h->d_tmp));
  else OK(schur_mul_dev(h, h->d_xr, h->d_tmp, nullptr));
  return d2h(h, y, h->d_tmp, sizeof(double) * 9 * h->C);
}
int b200_schur_back_substitute(b200_handle* h, const double* z, double* y) {
  if (h == nullptr || z == nullptr || y == nullptr || !h->schur_ready) return fail(B200_ERR_INVALID_ARGUMENT, "b200_schur_init first");
  CU(cudaSetDevice(h->device));
  OK(h2d(h, h->d_xr, z, sizeof(double) * 9 * h->C));
  OK(launch(h, K_BACKSUB, [&] {
    backsub_kernel<<<h->grid_tile[K_BACKSUB], kTile, tile_smem_bytes<3, 1>(), h->stream>>>(h->view, h->d_ete_inv, h->cur_b, h->d_xr, h->d_y);
  }));
  if (h->num_huge > 0)
    OK(launch(h, K_BACKSUB, [&] {
      huge_backsub_kernel<<<huge_grid(h), kHugeThreads, 0, h->stream>>>(h->view, h->num_huge, h->d_huge_pts, h->d_ete_inv, h->cur_b, h->d_xr, h->d_y);
    }, false));
  if (h->permuted) {
    OK(permute_blocks(h, false, h->P, 3, h->d_pt_perm, h->d_y, h->d_stage_p));
    OK(d2h(h, y, h->d_stage_p, sizeof(double) * 3 * static_cast<size_t>(h->P)));
  } else {
    OK(d2h(h, y, h->d_y, sizeof(double) * 3 * static_cast<size_t>(h->P)));
  }
  std::memcpy(y + 3 * static_cast<size_t>(h->P), z, sizeof(double) * 9 * h->C);
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
// One implementation of TrustRegionMinimizer::Minimize's control flow; `host_boundary` selects whether the vectors
// cross the bus through the public entry points (adapter behaviour) or stay in HBM.
int b200_lm_solve(b200_handle* h, const b200_lm_options* opt, double* state_inout, b200_lm_iteration* trace,
                  int max_records, int* num_records, int host_boundary) {
  if (h == nullptr || opt == nullptr || state_inout == nullptr || trace == nullptr || num_records == nullptr)
    return fail(B200_ERR_INVALID_ARGUMENT, "null argument");
  CU(cudaSetDevice(h->device));
  *num_records = 0;
  const int np = h->np;
  const size_t nr = 2 * static_cast<size_t>(h->N);
  const size_t off = 3 * static_cast<size_t>(h->P);
  // host mirrors (host_boundary only)
  // page-locked host mirrors, allocated once per handle (cudaMallocHost is far too slow to sit inside a solve)
  PinnedVec &x = h->hv[0], &cand = h->hv[1], &residuals = h->hv[2], &gradient = h->hv[3], &step = h->hv[4], &delta = h->hv[5],
            &scaling = h->hv[6], &diagonal = h->hv[7], &lmD = h->hv[8], &model_res = h->hv[9], &sol = h->hv[10], &best = h->hv[11];
  if (host_boundary) {
    x.assign(state_inout, state_inout + np);
    cand.resize(np); residuals.resize(nr); gradient.resize(np); step.resize(np); delta.resize(np);
    scaling.assign(np, 1.0); diagonal.resize(np); lmD.resize(np); model_res.resize(nr); sol.resize(np);
    best = x;
  } else {
    OK(up_params(h, h->d_state, state_inout));
    OK(launch(h, K_LM_VEC, [&] { fill_kernel<<<flat_grid(h, np, 256), 256, 0, h->stream>>>(np, h->d_scale, 1.0); }));
    CU(cudaMemcpyAsync(h->d_vp1, h->d_state, sizeof(double) * np, cudaMemcpyDeviceToDevice, h->stream));  // best
  }
  double x_cost = std::numeric_limits<double>::max(), candidate_cost = 0.0, model_cost_change = 0.0;
  double minimum_cost = x_cost;
  double radius = opt->initial_trust_region_radius, decrease_factor = 2.0;
  bool reuse_diagonal = false;
  double se_minimum = 0, se_current = 0, se_reference = 0, se_candidate = 0, se_acc_ref = 0, se_acc_cand = 0;
  b200_lm_iteration it{};
  int iteration = 0;
  bool have_scaling = false;
  bool sqnorm_fresh = false;  // d_sqnorm holds the squared column norms of the current device Jacobian
  const int vgrid = std::min(kRedBlocks, flat_grid(h, np, 256));

  auto evaluate_gradient_and_jacobian = [&]() -> int {
    if (host_boundary) {
      OK(b200_evaluate(h, x.data(), &x_cost, residuals.data(), gradient.data(), 1));
      it.cost = x_cost;
      if (opt->jacobi_scaling) {
        if (iteration == 0) {
          OK(b200_jacobian_squared_column_norm(h, scaling.data()));
          double* sc = scaling.data();
#pragma omp parallel for num_threads(kHostThreads) schedule(static)
          for (int i = 0; i < np; ++i) sc[i] = 1.0 / (1.0 + std::sqrt(sc[i]));
        }
        OK(b200_jacobian_scale_columns(h, scaling.data()));
      }
      double mx = 0, sq = 0;
      const double* gr = gradient.data();
      const int np_local = h->world > 1 ? static_cast<int>(off) : np;   // sharded: points are this rank's, cameras replicated
#pragma omp parallel for num_threads(kHostThreads) schedule(static) reduction(max : mx) reduction(+ : sq)
      for (int i = 0; i < np_local; ++i) {
        mx = std::max(mx, std::fabs(gr[i]));
        sq += gr[i] * gr[i];
      }
      if (h->world > 1) {
        double v[2] = {mx, sq};
        OK(host_allreduce(h, v, 2, 0x1u));
        mx = v[0];
        sq = v[1];
        for (int i = np_local; i < np; ++i) {   // the camera part, counted once
          mx = std::max(mx, std::fabs(gr[i]));
          sq += gr[i] * gr[i];
        }
      }
      it.gradient_max_norm = mx;
      it.gradient_norm = std::sqrt(sq);
      return B200_OK;
    }
    // device-resident: scaling is fused into the Jacobian write once it is known
    const bool fuse = opt->jacobi_scaling && have_scaling;
    OK(evaluate_dev(h, h->d_state, h->d_residuals, h->d_gradient, true, fuse ? h->d_scale : nullptr, &x_cost, h->d_sqnorm,
                    &sqnorm_fresh));
    it.cost = x_cost;
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
    it.gradient_max_norm = gn[0];
    it.gradient_norm = std::sqrt(gn[1]);
    return B200_OK;
  };

  it.iteration = 0;
  OK(evaluate_gradient_and_jacobian());
  it.step_is_valid = 1;
  it.step_is_successful = 1;
  se_minimum = se_current = se_reference = se_candidate = x_cost;
  int num_consecutive_invalid = 0;
  bool at_least_one_successful = false;

  for (;;) {
    if (it.step_is_successful && x_cost < minimum_cost) {
      minimum_cost = x_cost;
      if (host_boundary) best = x;
      else CU(cudaMemcpyAsync(h->d_vp1, h->d_state, sizeof(double) * np, cudaMemcpyDeviceToDevice, h->stream));
    }
    it.trust_region_radius = radius;
    if (*num_records < max_records) trace[(*num_records)++] = it;
    if (it.iteration >= opt->max_num_iterations) break;
    if (it.step_is_successful && it.gradient_max_norm <= opt->gradient_tolerance) break;
    if (it.trust_region_radius <= opt->min_trust_region_radius) break;

    const double prev_gn = it.gradient_norm, prev_gmax = it.gradient_max_norm;
    const int prev_iteration = it.iteration;
    it = b200_lm_iteration{};
    it.iteration = prev_iteration + 1;
    iteration = it.iteration;

    // ---- LevenbergMarquardtStrategy::ComputeStep
    b200_solver_options so = opt->linear_solver;
    so.q_tolerance = opt->eta;
    so.r_tolerance = -1.0;
    b200_solver_summary ls{};
    bool step_finite = true;
    double host_x_sq = 0.0, host_step_sq = 0.0;
    if (host_boundary) {
      // (the host-side vector passes mirror what the reference minimizer does on its Eigen vectors; adjacent ones are
      // fused so that each array is streamed once)
      if (!reuse_diagonal) {
        OK(b200_jacobian_squared_column_norm(h, diagonal.data()));
        double *dg = diagonal.data(), *ld = lmD.data();
        const double lo = opt->min_lm_diagonal, hi = opt->max_lm_diagonal;
#pragma omp parallel for num_threads(kHostThreads) schedule(static)
        for (int i = 0; i < np; ++i) {
          dg[i] = std::min(std::max(dg[i], lo), hi);
          ld[i] = std::sqrt(dg[i] / radius);
        }
      } else {
        const double* dg = diagonal.data();
        double* ld = lmD.data();
#pragma omp parallel for num_threads(kHostThreads) schedule(static)
        for (int i = 0; i < np; ++i) ld[i] = std::sqrt(dg[i] / radius);
      }
      // (levenberg_marquardt_strategy.cc:108 pre-fills the step with NaN so that a solver that silently writes nothing is
      //  caught; here the solve either fills sol or reports FAILURE / FATAL_ERROR, which the code below checks)
      if (opt->linear_solver_type == B200_DENSE_SCHUR) OK(b200_dense_schur_solve(h, nullptr, lmD.data(), sol.data(), &ls));
      else OK(b200_schur_solve(h, nullptr /* residuals of the last evaluate, still in HBM */, lmD.data(), &so, sol.data(), &ls));
      if (ls.termination_type != B200_LS_FAILURE && ls.termination_type != B200_LS_FATAL_ERROR) {
        // step = -sol, delta = step * scaling, candidate = x + delta (Evaluator::Plus on Euclidean blocks) and the two
        // norms the minimizer needs, in one pass
        double acc_x = 0.0, acc_s = 0.0, bad = 0.0;
        const double *sl = sol.data(), *xx = x.data(), *sc = scaling.data();
        double *stp = step.data(), *cd = cand.data();
        double cam_x = 0.0, cam_s = 0.0;   // camera part (replicated when sharded: counted once)
        const int np_local = h->world > 1 ? static_cast<int>(off) : np;
#pragma omp parallel for num_threads(kHostThreads) schedule(static) reduction(+ : acc_x, acc_s, bad, cam_x, cam_s)
        for (int i = 0; i < np; ++i) {
          const double si = -sl[i];
          stp[i] = si;
          const double ci = xx[i] + si * sc[i];
          cd[i] = ci;
          const double ax = xx[i] * xx[i], as = (xx[i] - ci) * (xx[i] - ci);
          if (i < np_local) {
            acc_x += ax;
            acc_s += as;
          } else {
            cam_x += ax;
            cam_s += as;
          }
          bad += (si - si);  // NaN/Inf - itself is NaN, finite - itself is 0
        }
        if (h->world > 1) {
          double v[3] = {acc_x, acc_s, bad};
          OK(host_allreduce(h, v, 3, 0u));
          acc_x = v[0];
          acc_s = v[1];
          bad = v[2];
        }
        acc_x += cam_x;
        acc_s += cam_s;
        step_finite = (bad == 0.0);
        host_x_sq = acc_x;
        host_step_sq = acc_s;
      }
    } else {
      if (!reuse_diagonal && !sqnorm_fresh) OK(sqnorm_dev(h, h->d_sqnorm));
      OK(launch(h, K_LM_VEC, [&] {
        lm_diagonal_kernel<<<flat_grid(h, np, 256), 256, 0, h->stream>>>(np, reuse_diagonal ? 0 : 1, h->d_sqnorm, h->d_diagonal, h->d_lmD,
                                                                          opt->min_lm_diagonal, opt->max_lm_diagonal, radius);
      }));
      if (opt->linear_solver_type == B200_DENSE_SCHUR) OK(dense_schur_solve_dev(h, h->d_residuals, h->d_lmD, h->d_y, &ls));
      else OK(schur_solve_dev(h, h->d_residuals, h->d_lmD, &so, h->d_y, &ls));
    }
    reuse_diagonal = true;
    it.linear_solver_iterations = ls.num_iterations;
    if (ls.termination_type == B200_LS_FATAL_ERROR) return fail(B200_ERR_CUDA, "linear solver fatal error");
    bool solver_ok = ls.termination_type != B200_LS_FAILURE && step_finite;

    double step_sq = 0.0, x_sq = 0.0;
    if (solver_ok) {
      if (host_boundary) {
        OK(b200_model_cost_change(h, step.data(), &model_cost_change));
      } else {
        // step = -y, delta = step * scaling, candidate = x + delta and the norms, in one pass
        double red[3];
        OK(sharded_reduce(h, vgrid, 3, 0u, red, [&](int ofs, int cnt) {
          return launch(h, K_LM_VEC, [&] {
            lm_step_kernel<<<vgrid, 256, 0, h->stream>>>(cnt, h->d_y + ofs, h->d_scale + ofs, h->d_state + ofs, h->d_step + ofs,
                                                         h->d_cand + ofs, h->d_partial);
          });
        }));
        step_sq = red[0];
        x_sq = red[1];
        if (red[2] != 0.0) solver_ok = false;
        if (solver_ok) {
          OK(launch(h, K_MODEL_COST, [&] {
            model_cost_kernel<<<h->grid_tile[K_MODEL_COST], kTile, tile_smem_bytes<1, 1>(), h->stream>>>(h->view, h->d_step, h->d_residuals, h->d_tile_partial);
          }));
          OK(launch(h, K_MISC, [&] { sum_kernel<<<1, kVecThreads, 0, h->stream>>>(h->num_tiles, h->d_tile_partial, h->d_scalars + 1); }));
          OK(allreduce_sum(h, h->d_scalars + 1, 1));
          CU(cudaMemcpyAsync(h->h_scalars + 1, h->d_scalars + 1, sizeof(double), cudaMemcpyDeviceToHost, h->stream));
          CU(cudaStreamSynchronize(h->stream));
          model_cost_change = h->h_scalars[1];
        }
      }
      if (solver_ok) {
        it.model_cost_change = model_cost_change;
        it.step_is_valid = model_cost_change > 0.0;
      }
    }
    if (!it.step_is_valid) {
      if (++num_consecutive_invalid >= opt->max_num_consecutive_invalid_steps) break;
      radius = radius / decrease_factor;
      decrease_factor *= 2.0;
      reuse_diagonal = true;
      it.cost = x_cost;
      it.cost_change = 0.0;
      it.gradient_max_norm = prev_gmax;
      it.gradient_norm = prev_gn;
      it.step_norm = 0.0;
      it.relative_decrease = 0.0;
      continue;
    }
    num_consecutive_invalid = 0;

    // ---- ComputeCandidatePointAndEvaluateCost
    int rc;
    if (host_boundary) {
      rc = b200_evaluate(h, cand.data(), &candidate_cost, nullptr, nullptr, 0);
      x_sq = host_x_sq;
      step_sq = host_step_sq;
    } else {
      rc = evaluate_dev(h, h->d_cand, nullptr, nullptr, false, nullptr, &candidate_cost);
    }
    if (rc == B200_ERR_EVALUATION_FAILED) candidate_cost = std::numeric_limits<double>::max();
    else if (rc != B200_OK) return rc;

    // (assigned only once a step has been accepted, like the reference: trust_region_minimizer.cc:113, :730)
    it.step_norm = at_least_one_successful ? std::sqrt(step_sq) : 0.0;
    if (at_least_one_successful && it.step_norm <= opt->parameter_tolerance * (std::sqrt(x_sq) + opt->parameter_tolerance)) break;
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
      if (host_boundary) x = cand;
      else std::swap(h->d_state, h->d_cand);
      OK(evaluate_gradient_and_jacobian());
      it.step_is_successful = 1;
      radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * it.relative_decrease - 1.0, 3));
      radius = std::min(opt->max_trust_region_radius, radius);
      decrease_factor = 2.0;
      reuse_diagonal = false;
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
      it.gradient_norm = prev_gn;
      it.gradient_max_norm = prev_gmax;
      radius = radius / decrease_factor;
      decrease_factor *= 2.0;
      reuse_diagonal = true;
    }
  }
  if (host_boundary) std::memcpy(state_inout, best.data(), sizeof(double) * np);
  else OK(down_params(h, state_inout, h->d_vp1));
  return B200_OK;
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
