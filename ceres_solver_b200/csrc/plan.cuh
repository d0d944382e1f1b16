// Kernel plan of one problem: everything b200_create decides before it touches the device.  From the validated rows, the
// device limits and the development knobs it chooses the internal point order, cuts the tiles, partitions them over the
// persistent CTAs, picks the kernel family of every operation and the shared-memory geometry of each warp-tile kernel,
// plans the L2 residency of S*x, decides explicit or implicit S and counts the algorithmic bytes of each operation.
// Host code only, no CUDA runtime call: b200_create allocates and uploads what the plan holds, and every entry point
// dispatches from its enums.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <vector>

#include "explicit_schur.cuh"
#include "kernels_v4b.cuh"
#include "xs_pcg.cuh"

namespace b200 {

// Share of the L2 the S*x residency plan may fill.  On an H100 (50 MB L2) the product got faster up to ~24 MB resident
// and slower again from 32 MB on (DESIGN §3.2).
constexpr double kL2ResidentShare = 0.5;
// Explicit S (explicit_schur.cuh) when the implicit product's stream is at least kXsByteRatio times 656 (C + 2 pairs) +
// 216 C bytes (the cost of a product that reads every off-diagonal block twice, the yardstick the thresholds were
// measured against; the product now reads each block once), does not fit the L2 residency budget
// (then the implicit product is served from L2 and the assembly cannot pay for itself), and S with its row-pair list
// fits kXsMaxBytes (the assembly time grows with the row pairs, and a solve of few CG iterations cannot repay it).
// Measured on one H100 (DESIGN §3): Ladybug-1723 (ratio 3.3, 40 MB) is faster explicit; ladybug-1723-random (ratio 0.47),
// C16 (stream within the L2 budget) and Venice-1778 (186 MB, 3-10 CG iterations per solve) are faster implicit.
constexpr double kXsByteRatio = 2.0;
constexpr double kXsMaxBytes = 128.0 * (1 << 20);

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
  K_SCHUR_PCG,
  K_SPARSE_SCATTER,
  K_SPARSE_FACTOR,
  K_SPARSE_SOLVE,
  K_DOGLEG_GRAM,
  K_DOGLEG_DIAG,
  K_DOGLEG_GN,
  K_DOGLEG_STEP,
  K_REFINE,
  K_SELINV,
  K_COV_POINTS,
  K_COV_GATHER,
  K_MISC,
  K_COUNT
};
const char* const kKernelNames[K_COUNT] = {"evaluate_jacobian", "evaluate_cost", "squared_column_norm", "scale_columns",
                                           "jacobian_multiply", "jacobian_t_multiply", "jtj_multiply", "schur_init",
                                           "schur_multiply", "schur_multiply_big_points", "camera_reduce", "schur_diag_blocks", "invert_9x9", "back_substitute",
                                           "model_cost", "cg_vector", "lm_vector", "pmv_right_e", "pmv_right_f", "pmv_left_e", "pmv_left_f", "schur_pcg",
                                           "sparse_scatter", "sparse_factor", "sparse_solve", "dogleg_gram", "dogleg_diagonal", "dogleg_gn", "dogleg_step",
                                           "refine_convert", "selected_inversion", "covariance_points",
                                           "covariance_gather", "misc"};

// Development switches (A/B measurements of kernel variants and tuning knobs) exist only in builds with
// -DB200_DEV_KNOBS; the product library has a single code path per problem class and reads no such variable.
#ifdef B200_DEV_KNOBS
inline const char* dev_env(const char* name) { return getenv(name); }
#else
inline const char* dev_env(const char*) { return nullptr; }
#endif

// The development knobs of the DESIGN appendix, read once per handle.  Every field holds its default in the product library.
struct DevKnobs {
  bool keep_order = false;           // B200_KEEP_ORDER
  bool disable_v2 = false;           // B200_DISABLE_V2: CTA-tile kernels everywhere
  bool disable_cam_major = false;    // B200_DISABLE_CAM_MAJOR
  bool disable_big_fold = false;     // B200_DISABLE_BIG_FOLD: the >32-row points in a launch of their own
  double big_cost = 22.0;            // B200_BIG_COST: a >32-row point costs this many warp tiles in the CTA partition
  long direct_limit = 700000;        // B200_DIRECT_LIMIT: REDs of the direct-mode flush
  int v3_warps = 0, v3_replicas = 0; // B200_V3_WARPS, B200_V3_REPLICAS (0: as planned)
  int v4_warps = kV4MaxThreads / 32; // B200_V4_WARPS: the most warps the v4 geometry tries
  int v4_stages = 1;                 // B200_V4_STAGES
  int v4_replicas = 0;               // B200_V4_REPLICAS (0: as planned)
  bool l2_mb_set = false;            // B200_L2_RESIDENT_MB: this residency budget instead of the planned one
  double l2_mb = 0.0;
  bool l2_last = false;              // B200_L2_RESIDENT_POLICY=last
  int explicit_s = -1;               // B200_EXPLICIT_S (-1: as planned)
  bool no_pdl = false;               // B200_NO_PDL
  bool no_fused_pq = false;          // B200_NO_FUSED_PQ
  bool no_peer_exchange = false;     // B200_NO_PEER_EXCHANGE
  int xs_resident = -1;              // B200_XS_RESIDENT (-1: as planned; 0: the two-kernel explicit-S PCG)

  static DevKnobs from_env() {
    DevKnobs k;
    k.keep_order = dev_env("B200_KEEP_ORDER") != nullptr;
    k.disable_v2 = dev_env("B200_DISABLE_V2") != nullptr;
    k.disable_cam_major = dev_env("B200_DISABLE_CAM_MAJOR") != nullptr;
    k.disable_big_fold = dev_env("B200_DISABLE_BIG_FOLD") != nullptr;
    if (const char* e = dev_env("B200_BIG_COST")) k.big_cost = std::max(0.0, atof(e));
    if (const char* e = dev_env("B200_DIRECT_LIMIT")) k.direct_limit = atol(e);
    if (const char* e = dev_env("B200_V3_WARPS")) k.v3_warps = atoi(e);
    if (const char* e = dev_env("B200_V3_REPLICAS")) k.v3_replicas = atoi(e);
    if (const char* e = dev_env("B200_V4_WARPS")) k.v4_warps = std::max(4, std::min(k.v4_warps, atoi(e)));
    if (const char* e = dev_env("B200_V4_STAGES")) k.v4_stages = std::max(1, std::min(3, atoi(e)));
    if (const char* e = dev_env("B200_V4_REPLICAS")) k.v4_replicas = std::max(1, atoi(e));
    if (const char* e = dev_env("B200_L2_RESIDENT_MB")) {
      k.l2_mb_set = true;
      k.l2_mb = atof(e);
    }
    if (const char* e = dev_env("B200_L2_RESIDENT_POLICY")) k.l2_last = strcmp(e, "last") == 0;
    if (const char* e = dev_env("B200_EXPLICIT_S")) k.explicit_s = atoi(e) != 0 ? 1 : 0;
    k.no_pdl = dev_env("B200_NO_PDL") != nullptr;
    k.no_fused_pq = dev_env("B200_NO_FUSED_PQ") != nullptr;
    k.no_peer_exchange = dev_env("B200_NO_PEER_EXCHANGE") != nullptr;
    if (const char* e = dev_env("B200_XS_RESIDENT")) k.xs_resident = atoi(e) != 0 ? 1 : 0;
    return k;
  }
};

struct DevLimits {
  int sm_count;
  size_t smem_optin;   // cudaDeviceProp::sharedMemPerBlockOptin
  int l2_bytes;
  int xs_ctas_per_sm;  // resident CTAs of xs_mul_kernel per SM (cudaOccupancyMaxActiveBlocksPerMultiprocessor)
  int xs_pcg_ctas_per_sm;  // ... of xs_pcg_kernel with the most dynamic shared memory a CTA may take
};

// Kernel family of S*x, and with it of the Schur initialisation, J'J x and the evaluation.  Tile: the CTA-tile kernels
// everywhere.  V3: schur_mul_v3_kernel and jtj_v2_kernel on warp tiles, CTA-tile evaluate and initialisation.  V4 / V4Owned:
// the v4 kernels (every operand through the TMA ring, x staged in shared memory; V4Owned: one private camera vector per
// warp) and the warp-tile evaluate.
enum class MulFamily { Tile, V3, V4, V4Owned };
// The block-diagonal pass of the preconditioners: camera-major row lists (no camera sees a point twice), the warp-tile
// kernel, or the CTA-tile kernel.
enum class DiagPass { CamMajor, WarpTile, Tile };

inline bool is_v4(MulFamily m) { return m == MulFamily::V4 || m == MulFamily::V4Owned; }

// Block pattern of the upper triangle of S and what its assembly and product read (explicit_schur.cuh), built from the
// row structure in the internal order.  Block row i: the diagonal block first (also for a camera without rows), then
// the cameras j > i sharing a point with i in increasing order; every block lists its row pairs (r, s) in the order
// (row r of camera i in row order, row s of r's point in row order) -- a fixed summation order.  T slots: the
// off-diagonal blocks ordered by column, then by row.
struct XsPattern {
  long long off_blocks = 0;   // distinct camera pairs i < j that share a point
  std::vector<int> blk_row, blk_col, pair_ptr, row_ptr, col_ptr;
  std::vector<int2> pairs, cols;
};

struct KernelPlan {
  // internal point order and the rows in it
  int order_choice = 0;
  long order_metrics[4] = {0, 0, 0, 0};
  std::vector<int> pt_perm;    // internal point k = caller point pt_perm[k]
  std::vector<int> row_perm;   // internal row r = caller row row_perm[r]
  std::vector<int> cam_idx, pt_idx, pt_ptr;
  std::vector<double> obs;
  // tiles
  std::vector<TileDesc> tiles;         // whole points, <= kTile rows and points each, then the slices of the huge points
  std::vector<TileDesc> chunk_tiles;   // the <= kTile-row slices of the points with more than kTile rows
  std::vector<int> huge_pts;           // the points with more than kTile rows
  std::vector<WarpTile> wtiles;        // whole points, <= 32 rows
  std::vector<TileDesc> big_tiles;     // the 33..kTile-row points, one each; then, unless MulFamily::Tile, the chunk tiles
  int num_plain_big = 0;               // big tiles before the chunk tiles
  std::vector<uint32_t> row_meta;
  std::vector<int> cam_rows;           // camera-major row lists
  std::vector<CamItem> cam_items;
  bool has_dups = false;               // a camera sees a point twice
  // per-CTA work of the warp-tile kernels
  int num_ctas = 0;
  std::vector<int2> cta_part, cta_cam, cta_big;
  std::vector<int> cta_cams;           // direct mode: the CTAs' sorted camera lists, concatenated
  int max_cam_span = 1;
  // kernel choices
  MulFamily mul = MulFamily::Tile;
  DiagPass diag = DiagPass::Tile;
  bool big_folded = false;             // S*x, J'J x and the v4 initialisation take the >32-row points themselves
  // warp-tile geometry; b200_create binds the device pointers
  V2View v2{}, v2_mul{}, v2_eval{}, v2_diag{};
  size_t v2_smem = 0, mul_smem = 0, eval_smem = 0, diag_smem = 0;
  int diag_replicas = 0;
  std::vector<uint32_t> tile_meta;     // v4: [warp tiles][kV4MetaWords]
  double l2_budget = 0.0, l2_stream_bytes = 0.0, l2_resident_bytes = 0.0;
  // explicit S
  bool xs = false;
  XsPattern xp;
  std::vector<int> xs_order;           // [long blocks | short blocks]
  std::vector<int2> xs_steps;         // product steps (XsView::steps), warp by warp
  std::vector<int> xs_warp_step;
  int num_xs_long = 0, xs_grid = 0, xs_resident = 0, xs_max_steps = 0;
  // resident PCG on explicit S (xs_pcg.cuh): one CTA per SM, its block rows, their steps over its warps
  bool xs_pcg = false;
  std::vector<int2> xs_pcg_cta;        // [sm_count + 1] {first block row, first block}
  std::vector<int> xs_pcg_warp_step;   // [sm_count * kXpWarps + 1] first step of each warp (into xs_steps)
  std::vector<int> xs_pcg_fptr;        // [sm_count + 1] each CTA's foreign columns in xs_pcg_fcol
  std::vector<int> xs_pcg_fcol;        // per CTA, ascending: the columns past its last row that its blocks touch
  std::vector<int2> xs_pcg_cols;       // [blocks] {CTA-local column, T slot}: l < owned cameras n: camera first row + l,
                                       // else foreign column l - n of the block's CTA
  int xs_pcg_max_blocks = 0, xs_pcg_max_cams = 0, xs_pcg_max_steps = 0, xs_pcg_max_foreign = 0;
  int xs_pcg_max_cta_steps = 0;        // the most product steps of a CTA
  int xs_pcg_walk_max = 0;             // the most steps of a warp, counting one per row segment for its sum
  int xs_pcg_split_rows = 0;           // rows whose steps are cut over two or more warps, all CTAs together
  int xs_pcg_max_slots = 0;            // the most T slots of a CTA's owned columns
  int xs_pcg_stage_slots = 0;          // ... that fit the shared memory left: a CTA with at most these stages them
  size_t xs_pcg_smem = 0;
  const char* xs_pcg_why = "";         // why the PCG is not resident
  double bytes_per_op[K_COUNT] = {};
};

inline void xs_pattern(int C, int N, const int* cam_idx, const int* pt_idx, const int* pt_ptr, XsPattern* xp) {
  std::vector<int> cptr(static_cast<size_t>(C) + 1, 0), crow(static_cast<size_t>(N));
  for (int r = 0; r < N; ++r) cptr[cam_idx[r] + 1]++;
  for (int c = 0; c < C; ++c) cptr[c + 1] += cptr[c];
  {
    std::vector<int> fill(cptr.begin(), cptr.end() - 1);
    for (int r = 0; r < N; ++r) crow[fill[cam_idx[r]]++] = r;
  }
  std::vector<int> stamp(static_cast<size_t>(C), -1), slot(static_cast<size_t>(C), 0), js, start;
  std::vector<int>& row_start = xp->row_ptr;
  row_start.assign(static_cast<size_t>(C) + 1, 0);
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
  // T slots by column, each column's blocks in order of their row
  xp->col_ptr.assign(static_cast<size_t>(C) + 1, 0);
  for (int b = 0; b < nb; ++b)
    if (xp->blk_col[b] != xp->blk_row[b]) xp->col_ptr[xp->blk_col[b] + 1]++;
  for (int c = 0; c < C; ++c) xp->col_ptr[c + 1] += xp->col_ptr[c];
  std::vector<int> fill(xp->col_ptr.begin(), xp->col_ptr.end() - 1);
  xp->cols.resize(static_cast<size_t>(nb));
  for (int b = 0; b < nb; ++b)
    xp->cols[b] = make_int2(xp->blk_col[b], xp->blk_col[b] != xp->blk_row[b] ? fill[xp->blk_col[b]]++ : -1);
}

// The order xs_assemble_dev assembles the blocks in: the blocks with long pair lists (the diagonal ones, mostly) first, one
// CTA each; then one warp per block.  Returns the number of long blocks.
inline int xs_assembly_order(const XsPattern& xp, std::vector<int>* order) {
  const int nb = static_cast<int>(xp.blk_row.size());
  order->clear();
  order->reserve(static_cast<size_t>(nb));
  for (int b = 0; b < nb; ++b)
    if (xp.pair_ptr[b + 1] - xp.pair_ptr[b] > kXsLongPairs) order->push_back(b);
  const int num_long = static_cast<int>(order->size());
  for (int b = 0; b < nb; ++b)
    if (xp.pair_ptr[b + 1] - xp.pair_ptr[b] <= kXsLongPairs) order->push_back(b);
  return num_long;
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
inline int choose_point_order(int C, int P, int N, const int32_t* cam_of_row, const int* caller_ptr, int chunks, std::vector<int>* perm,
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

// The plan of a problem with C cameras, P points and N rows grouped by point (caller_ptr: first row of each point, P + 1
// entries) on `world` ranks.
inline void plan_kernels(int C, int P, int N, const int* caller_cam, const double* caller_obs, const std::vector<int>& caller_ptr,
                  int world, const DevLimits& lim, const DevKnobs& knobs, KernelPlan* out) {
  KernelPlan& pl = *out;
  if (knobs.keep_order) {
    pl.pt_perm.resize(static_cast<size_t>(P));
    std::iota(pl.pt_perm.begin(), pl.pt_perm.end(), 0);
  } else {
    pl.order_choice = choose_point_order(C, P, N, caller_cam, caller_ptr.data(), lim.sm_count, &pl.pt_perm, pl.order_metrics);
  }
  // internal copies of the row structure
  pl.cam_idx.resize(static_cast<size_t>(N));
  pl.pt_idx.resize(static_cast<size_t>(N));
  pl.row_perm.resize(static_cast<size_t>(N));
  pl.obs.resize(2 * static_cast<size_t>(N));
  pl.pt_ptr.assign(static_cast<size_t>(P) + 1, 0);
  {
    int r = 0;
    for (int k = 0; k < P; ++k) {
      const int q = pl.pt_perm[k];
      for (int j = caller_ptr[q]; j < caller_ptr[q + 1]; ++j, ++r) {
        pl.row_perm[r] = j;
        pl.cam_idx[r] = caller_cam[j];
        pl.pt_idx[r] = k;
        pl.obs[2 * static_cast<size_t>(r)] = caller_obs[2 * static_cast<size_t>(j)];
        pl.obs[2 * static_cast<size_t>(r) + 1] = caller_obs[2 * static_cast<size_t>(j) + 1];
      }
      pl.pt_ptr[k + 1] = r;
    }
  }
  const int* const cam_idx = pl.cam_idx.data();   // from here on: INTERNAL order
  const int* const pt_idx = pl.pt_idx.data();
  const std::vector<int>& pt_ptr = pl.pt_ptr;
  // CTA tiles: whole points, <= kTile rows and <= kTile points each; a point with more rows becomes chunk tiles.
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
        pl.huge_pts.push_back(k);
        for (int r = pt_ptr[k]; r < pt_ptr[k + 1]; r += kTile) {
          TileDesc c;
          c.pt_begin = k;
          c.pt_count = 1;
          c.obs_begin = r;
          c.obs_count = std::min(kTile, pt_ptr[k + 1] - r);
          c.chunk = 1;
          pl.tiles.push_back(c);
          pl.chunk_tiles.push_back(c);
        }
        ++k;
        continue;
      }
      t.obs_count = rows;
      t.pt_count = pts;
      pl.tiles.push_back(t);
    }
  }
  // Camera-major row lists (the reference's transpose block structure) for the block-diagonal kernels, cut into
  // slices of a few thousand rows so that small-C problems still fill the machine; unusable if a camera sees a
  // point twice (cross terms between the two rows), which is detected here.
  pl.cam_rows.resize(static_cast<size_t>(N));
  {
    std::vector<int> cptr(static_cast<size_t>(C) + 1, 0);
    for (int i = 0; i < N; ++i) cptr[cam_idx[i] + 1]++;
    for (int c = 0; c < C; ++c) cptr[c + 1] += cptr[c];
    std::vector<int> fill(cptr.begin(), cptr.end() - 1);
    for (int i = 0; i < N; ++i) pl.cam_rows[fill[cam_idx[i]]++] = i;
    for (int c = 0; c < C && !pl.has_dups; ++c)
      for (int j = cptr[c] + 1; j < cptr[c + 1]; ++j)
        if (pt_idx[pl.cam_rows[j]] == pt_idx[pl.cam_rows[j - 1]]) { pl.has_dups = true; break; }
    // ~3 items per resident warp (12 warps per SM): short enough to balance, long enough to amortise the final reduction
    const int slice = std::max(64, std::min(4096, N / (lim.sm_count * 36) + 1));
    for (int c = 0; c < C; ++c)
      for (int b = cptr[c]; b < cptr[c + 1]; b += slice) pl.cam_items.push_back(CamItem{c, b, std::min(b + slice, cptr[c + 1])});
  }
  pl.diag = !pl.has_dups && !knobs.disable_cam_major ? DiagPass::CamMajor : DiagPass::Tile;
  // Warp tiles (whole points, <= 32 rows) for the points with <= 32 rows; points with 33..kTile rows stay on the CTA-tile
  // kernels (one tile each).  Needs every point to have at least one row.
  pl.row_meta.resize(static_cast<size_t>(N));
  bool v2_possible = !knobs.disable_v2;
  for (int k = 0; k < P && v2_possible; ++k)
    if (pt_ptr[k + 1] == pt_ptr[k]) v2_possible = false;
  if (v2_possible) {
    for (int k = 0; k < P; ++k)
      for (int r = pt_ptr[k]; r < pt_ptr[k + 1]; ++r)
        pl.row_meta[r] = static_cast<uint32_t>(cam_idx[r]) | (r == pt_ptr[k] ? 0x80000000u : 0u);
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
        pl.big_tiles.push_back(t);
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
      pl.wtiles.push_back(t);
    }
  }
  pl.num_plain_big = static_cast<int>(pl.big_tiles.size());
  const int num_ctas = lim.sm_count;
  const std::vector<WarpTile>& wtiles = pl.wtiles;
  const std::vector<TileDesc>& big_tiles = pl.big_tiles;
  std::vector<int2> &cta_part = pl.cta_part, &cta_cam = pl.cta_cam, &cta_big = pl.cta_big;
  cta_part.resize(num_ctas);
  cta_cam.resize(num_ctas);
  cta_big.assign(num_ctas, make_int2(0, 0));
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
      const double big_cost = knobs.big_cost;
      const double total_cost = T + big_cost * big_tiles.size();
      int t = 0, g = 0, b = 0;
      double cum = 0.0;
      std::vector<int> t_end(num_ctas, 0), g_end(num_ctas, 0);
      const int G = static_cast<int>(big_tiles.size());
      while (t < T || g < G) {
        const bool take_big = g < G && (t >= T || big_tiles[g].obs_begin < wtiles[t].row_begin);
        const int owner = std::min(num_ctas - 1, static_cast<int>(cum * num_ctas / std::max(total_cost, 1.0)));
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
      for (; b < num_ctas; ++b) {
        t_end[b] = T;
        g_end[b] = G;
      }
      for (int k = 0; k < num_ctas; ++k) {
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
      std::vector<int> lo_v(num_ctas, 0), hi_v(num_ctas, 0);
      std::vector<std::vector<int>> lists(num_ctas);
      long list_total = 0;
      int max_list = 1, max_range = 1;
      for (int b = 0; b < num_ctas; ++b) {
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
      // list positions must fit the row word; REDs of the flush: a few microseconds, still far cheaper than partial vectors
      direct_mode = 9 * list_total <= knobs.direct_limit && max_list <= static_cast<int>(kMetaLocalMask) && C <= static_cast<int>(kMetaCamMask);
      if (C > static_cast<int>(kMetaCamMask)) v2_possible = false;   // camera ids do not fit the row word: CTA-tile kernels
      if (direct_mode) {
        max_cam_span = max_list;
        for (int b = 0; b < num_ctas; ++b) {
          cta_cam[b] = make_int2(static_cast<int>(pl.cta_cams.size()), static_cast<int>(lists[b].size()));
          for (size_t i = 0; i < lists[b].size(); ++i) local_of[lists[b][i]] = static_cast<int>(i);
          auto pack = [&](int r0, int r1) {
            for (int r = r0; r < r1; ++r) pl.row_meta[r] |= static_cast<uint32_t>(local_of[cam_idx[r]]) << kMetaLocalShift;
          };
          for (int t = cta_part[b].x; t < cta_part[b].y; ++t) pack(wtiles[t].row_begin, wtiles[t].row_begin + wtiles[t].row_count);
          for (int g = cta_big[b].x; g < cta_big[b].y; ++g) pack(big_tiles[g].obs_begin, big_tiles[g].obs_begin + big_tiles[g].obs_count);
          pl.cta_cams.insert(pl.cta_cams.end(), lists[b].begin(), lists[b].end());
        }
      } else {
        max_cam_span = max_range;
        for (int b = 0; b < num_ctas; ++b) cta_cam[b] = make_int2(lo_v[b], hi_v[b]);
      }
    }
    // Shared memory budget: `replicas` private camera vectors + per-warp {TMA ring of F cells, exchange scratch}.
    // Prefer one replica per warp (no cross-warp contention) when the camera span of a CTA is small.
    const long total = static_cast<long>(lim.smem_optin) - 2048;
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
    if (knobs.v3_warps >= 1 && knobs.v3_warps <= mul_warps) {
      mul_warps = knobs.v3_warps;
      mul_replicas = std::min(mul_replicas, mul_warps);
    }
    if (knobs.v3_replicas >= 1 && knobs.v3_replicas <= mul_replicas) mul_replicas = knobs.v3_replicas;
    if (v2_warps == 0 || mul_warps == 0) v2_possible = false;  // camera vector does not fit next to the tile buffers: v1 kernels
  } else {
    v2_possible = false;
  }
  pl.num_ctas = num_ctas;
  pl.max_cam_span = max_cam_span;

  if (v2_possible) {
    // the slices of the huge points ride along with the >32-row points in every kernel that has no coupling between the
    // rows of a point (the partition above only covers the plain ones: cta_big indexes the first part of the array)
    pl.big_tiles.insert(pl.big_tiles.end(), pl.chunk_tiles.begin(), pl.chunk_tiles.end());
    V2View& v = pl.v2;
    v.num_ctas = num_ctas;
    v.max_cam_span = max_cam_span;
    v.warps = v2_warps;
    v.stages = v2_stages;
    v.replicas = v2_replicas;
    v.direct = direct_mode ? 1 : 0;
    v.per_warp_bytes = v2_per_warp_bytes(v2_stages, kV2Scratch);
    pl.v2_smem = v2_sy_bytes(max_cam_span, v2_replicas) + static_cast<size_t>(v2_warps) * v.per_warp_bytes;
    pl.mul = MulFamily::V3;
    V2View& m = pl.v2_mul;
    m = v;
    m.warps = mul_warps;
    m.stages = mul_stages;
    m.replicas = mul_replicas;
    m.per_warp_bytes = v2_per_warp_bytes(mul_stages, kV2Scratch);
    pl.mul_smem = v2_sy_bytes(max_cam_span, mul_replicas) + static_cast<size_t>(mul_warps) * m.per_warp_bytes;
    // the S*x kernel takes the >32-row points itself when its TMA rings can stage a kTile-row point
    pl.big_folded = mul_warps >= kTile / 32 && static_cast<size_t>(mul_warps) * m.per_warp_bytes >= kTile * 192 + 160 &&
                    !knobs.disable_big_fold;
    if (direct_mode) {
      // v4 (all operands through the TMA ring, x staged in shared memory) needs the narrow camera ranges of the
      // direct-flush mode: up to 16 warps with a one-slot ring each (the slot is refilled as soon as its contents are in
      // registers), one private camera vector per warp when they fit.
      const long total = static_cast<long>(lim.smem_optin) - 2048;
      const long sy1 = static_cast<long>(v2_sy_bytes(max_cam_span, 1));
      const int st4 = knobs.v4_stages;
      int w4 = knobs.v4_warps, rep4 = 0;
      for (; w4 >= 8; --w4) {
        const long rem = total - static_cast<long>(w4) * v4_per_warp_bytes(st4) - sy1 /* staged x */;
        if (rem < sy1) continue;
        rep4 = static_cast<int>(std::min<long>(w4, rem / sy1));
        if (knobs.v4_replicas > 0) rep4 = std::max(1, std::min(rep4, knobs.v4_replicas));
        break;
      }
      // The warp-tile evaluate and block-diagonal pass: each gets as many replicas of its private accumulators as fit
      // next to its per-warp buffers (one per warp at best), and the diagonal pass a shallower TMA ring if even a single
      // replica would not fit.
      const size_t lim2 = lim.smem_optin - 2048;
      auto fit = [&](size_t per_warp, size_t acc1, int* replicas) -> size_t {
        const size_t fixed = per_warp * v2_warps;
        if (fixed + acc1 > lim2) return lim2 + 1;
        *replicas = static_cast<int>(std::min<size_t>(v2_warps, (lim2 - fixed) / acc1));
        return fixed + acc1 * *replicas;
      };
      // evaluate: two accumulators (gradient, column norms) + per-warp staging
      pl.v2_eval = v;
      pl.eval_smem = fit(eval_v2_per_warp_bytes(), 2 * static_cast<size_t>(sy1), &pl.v2_eval.replicas);
      // diag blocks: 45 doubles per camera
      pl.v2_diag = v;
      pl.diag_smem = lim2 + 1;
      for (int st = v2_stages; st >= 1 && pl.diag_smem > lim2; --st) {
        pl.v2_diag.stages = st;
        pl.diag_smem = fit(diag_v2_per_warp_bytes(st), diag_v2_acc_stride(max_cam_span) * 8, &pl.diag_replicas);
      }
      if (pl.diag_smem > lim2) pl.diag_replicas = 0;
      // On sm_90 (232,448 B per CTA) the v4 ring fits exactly when the warp-tile evaluate does; V4 asks for both.
      if (w4 >= 8 && pl.eval_smem <= lim2) {
        pl.mul = rep4 == w4 ? MulFamily::V4Owned : MulFamily::V4;
        m.warps = w4;
        m.stages = st4;
        m.replicas = rep4;
        m.per_warp_bytes = v4_per_warp_bytes(st4);
        pl.mul_smem = v2_sy_bytes(max_cam_span, rep4) + v4_sx_bytes(max_cam_span) + static_cast<size_t>(w4) * m.per_warp_bytes;
        pl.big_folded = !knobs.disable_big_fold;
        pl.tile_meta.assign(wtiles.size() * kV4MetaWords, 0u);
        for (int b = 0; b < num_ctas; ++b)
          for (int t = cta_part[b].x; t < cta_part[b].y; ++t) {
            uint32_t* mt = pl.tile_meta.data() + static_cast<size_t>(t) * kV4MetaWords;
            const WarpTile& wt = wtiles[t];
            for (int r = 0; r < wt.row_count; ++r) mt[r] = pl.row_meta[wt.row_begin + r];
            mt[32] = static_cast<uint32_t>(wt.row_begin);
            mt[33] = static_cast<uint32_t>(wt.pt_begin);
            mt[34] = static_cast<uint32_t>(wt.row_count) | (static_cast<uint32_t>(wt.pt_count) << 16);
            int maxdeg = 1;   // longest point of the tile (rows): bounds the segmented reductions
            for (int k = 0; k < wt.pt_count; ++k) maxdeg = std::max(maxdeg, pt_ptr[wt.pt_begin + k + 1] - pt_ptr[wt.pt_begin + k]);
            mt[35] = static_cast<uint32_t>(maxdeg);
            const int tn = t + w4 * st4;
            if (tn < cta_part[b].y) {
              mt[36] = static_cast<uint32_t>(wtiles[tn].row_begin);
              mt[37] = static_cast<uint32_t>(wtiles[tn].pt_begin);
              mt[38] = static_cast<uint32_t>(wtiles[tn].row_count) | (static_cast<uint32_t>(wtiles[tn].pt_count) << 16);
            }
          }
        if (pl.diag == DiagPass::Tile && pl.diag_replicas > 0) pl.diag = DiagPass::WarpTile;
      }
    }
  }

  if (is_v4(pl.mul)) {
    // L2 residency plan of S*x.  J does not change during a PCG, and every product streams the same bytes (F, E,
    // (E'E+D^2)^-1 blocks, descriptors: 141 MB on Ladybug-1723); under the default policy a stream larger than L2 leaves
    // nothing behind for the next product.  So a fixed share of the tiles, spread evenly through every CTA's tile range
    // (HBM keeps streaming while the resident tiles are read from L2), is copied with evict_normal and the rest with
    // evict_first: the resident share then survives from one product to the next.  The budget is kL2ResidentShare of the
    // L2 minus the working set of the CG loop, which is read with the default policy; a stream within the budget is all
    // resident.  Whole tiles: the four copies of a tile share one policy.
    auto wbytes = [&](int t) { return 192.0 * wtiles[t].row_count + 48.0 * wtiles[t].pt_count + 4 * kV4MetaWords; };
    auto bbytes = [&](int t) { return 192.0 * big_tiles[t].obs_count; };
    double stream_bytes = 0.0;
    for (int b = 0; b < num_ctas; ++b) {
      for (int t = cta_part[b].x; t < cta_part[b].y; ++t) stream_bytes += wbytes(t);
      for (int t = cta_big[b].x; t < cta_big[b].y; ++t) stream_bytes += bbytes(t);
    }
    const double working_set = 8.0 * (8 * 9 + 81) * C                               // rhs x r z p q seed D_f, minv
                               + (world > 1 ? 2.0 * world * 16 * 9 * C : 0.0);    // peer exchange slots
    double budget = std::max(0.0, kL2ResidentShare * lim.l2_bytes - working_set);
    if (knobs.l2_mb_set) budget = knobs.l2_mb * (1 << 20);   // 0: no plan, every copy with the default policy
    const bool no_plan = knobs.l2_mb_set && budget <= 0.0;
    V2View& m = pl.v2_mul;
    m.l2_last = knobs.l2_last ? 1 : 0;
    m.l2_stream = (budget >= stream_bytes || no_plan) ? 0u : static_cast<uint32_t>(std::ceil(65536.0 * (1.0 - budget / stream_bytes)));
    // what the plan marks, counted the way the kernel decides it
    const uint64_t s = m.l2_stream;
    auto streamed = [&](int i) { return ((static_cast<uint64_t>(i) + 1) * s >> 16) != (static_cast<uint64_t>(i) * s >> 16); };
    double res = 0.0;
    for (int b = 0; b < num_ctas; ++b) {
      for (int t = cta_part[b].x; t < cta_part[b].y; ++t)
        if (!streamed(t - cta_part[b].x)) res += wbytes(t);
      for (int t = cta_big[b].x; t < cta_big[b].y; ++t)
        if (!streamed(t - cta_big[b].x)) res += bbytes(t);
    }
    pl.l2_budget = budget;
    pl.l2_stream_bytes = stream_bytes;
    pl.l2_resident_bytes = res;
  }

  // Explicit or implicit S (DESIGN §1): explicit when the product on the stored upper triangle reads clearly fewer bytes
  // than the implicit product streams and the storage fits; sharded handles stay implicit.
  double xs_mul_bytes = 0.0, xs_asm_bytes = 0.0;
  if (world == 1) {
    const double l2_budget = kL2ResidentShare * lim.l2_bytes - 8.0 * (8 * 9 + 81) * C;   // as the S*x residency plan
    XsPattern& xp = pl.xp;
    xs_pattern(C, N, cam_idx, pt_idx, pt_ptr.data(), &xp);
    const double nb = static_cast<double>(xp.blk_row.size()), npairs = static_cast<double>(xp.pairs.size());
    const double implicit_bytes = 196.0 * N + 52.0 * P + 216.0 * C;
    const double off = static_cast<double>(xp.off_blocks);
    const double two_pass_bytes = 656.0 * (nb + off) + 216.0 * C;   // the decision's yardstick (kXsByteRatio)
    const double storage = 648.0 * nb + 8.0 * npairs + 12.0 * nb;
    pl.xs = implicit_bytes >= kXsByteRatio * two_pass_bytes && implicit_bytes > l2_budget && storage <= kXsMaxBytes && npairs < 2.0e9;
    // S read once, its column entries, T written, x read, y written
    xs_mul_bytes = 656.0 * nb + 72.0 * off + 144.0 * C;
    if (knobs.explicit_s >= 0) pl.xs = knobs.explicit_s != 0 && npairs < 2.0e9;
    // J, point of each row, (E'E+D^2)^-1, row pairs, block table; S and the diagonal upper triangles written
    xs_asm_bytes = 196.0 * N + 48.0 * P + 8.0 * npairs + 12.0 * nb + 648.0 * nb + 360.0 * C;
  }
  if (pl.xs) {
    const XsPattern& xp = pl.xp;
    const int nb = static_cast<int>(xp.blk_row.size());
    // One wave: at most the CTAs that are resident together, and no more warps than block rows.  Each warp owns a
    // contiguous range of block rows, balanced by its steps (kXsStep blocks each) plus one per row for the row's sum.
    pl.xs_resident = std::max(1, lim.xs_ctas_per_sm) * lim.sm_count;
    pl.xs_grid = std::max(1, std::min(pl.xs_resident, (C + kXsWarps - 1) / kXsWarps));
    const int nw = pl.xs_grid * kXsWarps;
    auto row_steps = [&](int i) { return (xp.row_ptr[i + 1] - xp.row_ptr[i] + kXsStep - 1) / kXsStep; };
    double total = 0.0;
    for (int i = 0; i < C; ++i) total += row_steps(i) + 1;
    pl.xs_warp_step.assign(static_cast<size_t>(nw) + 1, 0);
    double cum = 0.0;
    int w = 0;
    for (int i = 0; i < C; ++i) {
      const int owner = std::min(nw - 1, static_cast<int>(cum * nw / total));
      while (w < owner) pl.xs_warp_step[++w] = static_cast<int>(pl.xs_steps.size());   // warps before the owner end here
      const int r0 = xp.row_ptr[i], r1 = xp.row_ptr[i + 1];
      for (int b = r0; b < r1; b += kXsStep) {
        const int n = std::min(kXsStep, r1 - b);
        pl.xs_steps.push_back(make_int2(b, i | (n << kXsStepCountShift) | (b == r0 ? kXsStepFirst : 0) |
                                               (b + kXsStep >= r1 ? kXsStepLast : 0)));
      }
      cum += row_steps(i) + 1;
    }
    while (w < nw) pl.xs_warp_step[++w] = static_cast<int>(pl.xs_steps.size());
    for (int k = 0; k < nw; ++k) pl.xs_max_steps = std::max(pl.xs_max_steps, pl.xs_warp_step[k + 1] - pl.xs_warp_step[k]);
    // Resident PCG (xs_pcg.cuh): the block rows in G contiguous ranges with the smallest possible largest range in blocks
    // (the share of S a CTA holds in shared memory): the least capacity K at which filling the CTAs in row order, each up
    // to K blocks, needs at most G of them.  Within a CTA its steps go to the warps in contiguous
    // ranges that may cut rows (below).  Every CTA also gets the sorted list of its foreign columns (j past its last row: its blocks are in the upper
    // triangle, so j below that is an owned camera) and every block its column as an index into [owned cameras | foreign
    // columns].  Resident when the largest CTA's blocks (with their column entries), M^-1 blocks and vectors, the most
    // foreign columns and the most product steps of a CTA fit one CTA's shared memory next to the static scratch, and
    // one CTA of the kernel fits each SM.
    {
      const int G = lim.sm_count;
      std::vector<int> first_step(static_cast<size_t>(C) + 1, 0);
      for (int i = 0; i < C; ++i) first_step[i + 1] = first_step[i] + row_steps(i);
      auto row_blocks = [&](int i) { return xp.row_ptr[i + 1] - xp.row_ptr[i]; };
      auto ctas_at = [&](int K) {
        int g = 1, cur = 0;
        for (int i = 0; i < C; ++i) {
          if (cur + row_blocks(i) > K) {
            ++g;
            cur = 0;
          }
          cur += row_blocks(i);
        }
        return g;
      };
      int lo = (nb + G - 1) / G, hi = nb;
      for (int i = 0; i < C; ++i) lo = std::max(lo, row_blocks(i));
      while (lo < hi) {
        const int mid = lo + (hi - lo) / 2;
        if (ctas_at(mid) <= G) hi = mid;
        else lo = mid + 1;
      }
      pl.xs_pcg_cta.assign(static_cast<size_t>(G) + 1, make_int2(C, nb));
      pl.xs_pcg_cta[0] = make_int2(0, 0);
      for (int i = 0, g = 0, cur = 0; i < C; ++i) {
        if (cur + row_blocks(i) > lo) {
          pl.xs_pcg_cta[++g] = make_int2(i, xp.row_ptr[i]);
          cur = 0;
        }
        cur += row_blocks(i);
      }
      pl.xs_pcg_warp_step.assign(static_cast<size_t>(G) * kXpWarps + 1, first_step[C]);
      pl.xs_pcg_fptr.assign(static_cast<size_t>(G) + 1, 0);
      pl.xs_pcg_cols.resize(static_cast<size_t>(nb));
      for (int b = 0; b < G; ++b) {
        const int i0 = pl.xs_pcg_cta[b].x, i1 = pl.xs_pcg_cta[b + 1].x;
        const int b0 = pl.xs_pcg_cta[b].y, b1 = pl.xs_pcg_cta[b + 1].y;
        pl.xs_pcg_max_blocks = std::max(pl.xs_pcg_max_blocks, b1 - b0);
        pl.xs_pcg_max_cams = std::max(pl.xs_pcg_max_cams, i1 - i0);
        pl.xs_pcg_max_cta_steps = std::max(pl.xs_pcg_max_cta_steps, first_step[i1] - first_step[i0]);
        pl.xs_pcg_max_slots = std::max(pl.xs_pcg_max_slots, xp.col_ptr[i1] - xp.col_ptr[i0]);
        std::vector<int> fc;
        for (int k = b0; k < b1; ++k)
          if (xp.blk_col[k] >= i1) fc.push_back(xp.blk_col[k]);
        std::sort(fc.begin(), fc.end());
        fc.erase(std::unique(fc.begin(), fc.end()), fc.end());
        for (int k = b0; k < b1; ++k) {
          const int j = xp.blk_col[k];
          const int l = j < i1 ? j - i0 : (i1 - i0) + static_cast<int>(std::lower_bound(fc.begin(), fc.end(), j) - fc.begin());
          pl.xs_pcg_cols[k] = make_int2(l, xp.cols[k].y);
        }
        pl.xs_pcg_fcol.insert(pl.xs_pcg_fcol.end(), fc.begin(), fc.end());
        pl.xs_pcg_fptr[b + 1] = static_cast<int>(pl.xs_pcg_fcol.size());
        pl.xs_pcg_max_foreign = std::max(pl.xs_pcg_max_foreign, static_cast<int>(fc.size()));
        // the CTA's steps in kXpWarps contiguous ranges, cut anywhere, with the least largest cost: a range costs its steps
        // plus one per row segment in it (the segment's butterfly).  Filling the warps in order, each up to K, is optimal
        // for a given K (extending a range never lowers its cost); K is the least that needs at most kXpWarps of them.
        const int s0 = first_step[i0], s1 = first_step[i1];
        auto fill = [&](int K, int* ws) {
          int g = 0, cost = 0;
          if (ws != nullptr) ws[0] = s0;
          for (int k = s0; k < s1; ++k) {
            const bool row_start = (pl.xs_steps[k].y & kXsStepFirst) != 0;
            if (cost + 1 + (row_start || cost == 0) > K) {
              if (++g == kXpWarps) return g + 1;
              if (ws != nullptr) ws[g] = k;
              cost = 0;
            }
            cost += 1 + (row_start || cost == 0);
          }
          if (ws != nullptr)
            while (g < kXpWarps - 1) ws[++g] = s1;
          return g + 1;
        };
        int klo = 2, khi = std::max(2, 2 * (s1 - s0));
        while (klo < khi) {
          const int mid = klo + (khi - klo) / 2;
          if (fill(mid, nullptr) <= kXpWarps) khi = mid;
          else klo = mid + 1;
        }
        int* ws = pl.xs_pcg_warp_step.data() + static_cast<size_t>(b) * kXpWarps;
        fill(klo, ws);
        for (int wv = 0; wv < kXpWarps; ++wv) {
          const int ka = ws[wv], kb = wv + 1 < kXpWarps ? ws[wv + 1] : s1;   // ws[kXpWarps]: the next CTA's, not set yet
          if (ka == kb) continue;
          int cost = kb - ka + 1;
          for (int k = ka + 1; k < kb; ++k) cost += (pl.xs_steps[k].y & kXsStepFirst) != 0;
          pl.xs_pcg_walk_max = std::max(pl.xs_pcg_walk_max, cost);
          const int df = pl.xs_steps[ka].y, dl = pl.xs_steps[kb - 1].y;
          // the range ends inside a row that begins in it
          if (!(dl & kXsStepLast) && ((df & kXsStepFirst) || (df & kXsStepRowMask) != (dl & kXsStepRowMask))) ++pl.xs_pcg_split_rows;
        }
      }
      for (int k = 0; k < G * kXpWarps; ++k)
        pl.xs_pcg_max_steps = std::max(pl.xs_pcg_max_steps, pl.xs_pcg_warp_step[k + 1] - pl.xs_pcg_warp_step[k]);
      // the T slots of the owned columns are staged in what shared memory is left, up to the most any CTA has; a CTA
      // with more sums its columns from T in L2
      const size_t base = xs_pcg_smem_bytes(pl.xs_pcg_max_blocks, pl.xs_pcg_max_cams, pl.xs_pcg_max_foreign, pl.xs_pcg_max_cta_steps, 0);
      const size_t room = lim.smem_optin > base + 1024 ? lim.smem_optin - base - 1024 : 0;
      pl.xs_pcg_stage_slots = static_cast<int>(std::min<size_t>(pl.xs_pcg_max_slots, room / (9 * sizeof(double))));
      pl.xs_pcg_smem = xs_pcg_smem_bytes(pl.xs_pcg_max_blocks, pl.xs_pcg_max_cams, pl.xs_pcg_max_foreign, pl.xs_pcg_max_cta_steps,
                                         pl.xs_pcg_stage_slots);
      if (pl.xs_pcg_smem + 1024 > lim.smem_optin) pl.xs_pcg_why = "largest CTA's shared memory exceeds the limit";
      else if (lim.xs_pcg_ctas_per_sm < 1) pl.xs_pcg_why = "no CTA of the kernel fits an SM";
      else if (knobs.xs_resident == 0) pl.xs_pcg_why = "B200_XS_RESIDENT=0";
      else pl.xs_pcg = true;
    }
    pl.num_xs_long = xs_assembly_order(xp, &pl.xs_order);
  }

  // Algorithmic (compulsory) bytes per launch, SURVEY §8d with this layout: J values 192 B/row + 4 B camera
  // index per row + 4 B chunk boundary per point, plus the vectors each kernel must read/write once.
  const double Nn = N, Pp = P, Cc = C;
  double* bpo = pl.bytes_per_op;
  bpo[K_JTJ] = 196 * Nn + 4 * Pp + 24.0 * (3 * Pp + 9 * Cc);
  bpo[K_SCHUR_MUL] = 196 * Nn + 52 * Pp + 216 * Cc;
  bpo[K_SCHUR_INIT] = 196 * Nn + 16 * Nn + 4 * Pp + 24 * Pp + 48 * Pp + 72 * Cc;   // J, b, chunk ids, D_e, (E'E)^-1 out, rhs out
  bpo[K_DIAG_BLOCKS] = 196 * Nn + 52 * Pp + 360 * Cc;
  bpo[K_BACKSUB] = 196 * Nn + 16 * Nn + 52 * Pp + 24 * Pp + 72 * Cc;
  bpo[K_EVAL_JAC] = 192 * Nn + 16 * Nn + 16 * Nn + 4 * Nn + 4 * Pp + 2 * 8.0 * (3 * Pp + 9 * Cc);
  bpo[K_EVAL_COST] = 16 * Nn + 4 * Nn + 4 * Pp + 8.0 * (3 * Pp + 9 * Cc);
  bpo[K_SQNORM] = 196 * Nn + 4 * Pp + 8.0 * (3 * Pp + 9 * Cc);
  bpo[K_SCALE] = 2 * 192 * Nn + 8 * Nn + 8.0 * (3 * Pp + 9 * Cc);
  bpo[K_JMUL] = 196 * Nn + 32 * Nn + 4 * Pp + 8.0 * (3 * Pp + 9 * Cc);
  bpo[K_JTMUL] = 196 * Nn + 16 * Nn + 4 * Pp + 16.0 * (3 * Pp + 9 * Cc);
  bpo[K_PMV_RIGHT_E] = 48 * Nn + 4 * Nn + 32 * Nn + 24 * Pp;            // E cells, point id, y read + written, x_e
  bpo[K_PMV_RIGHT_F] = 144 * Nn + 4 * Nn + 32 * Nn + 72 * Cc;           // F cells, camera id, y read + written, x_f
  bpo[K_PMV_LEFT_E] = 48 * Nn + 16 * Nn + 4 * Pp + 48 * Pp;             // E cells, y, chunk boundaries, x_e read + written
  bpo[K_PMV_LEFT_F] = 144 * Nn + 16 * Nn + 4 * Nn + 144 * Cc;           // F cells, y, row list, x_f read + written
  bpo[K_MODEL_COST] = 196 * Nn + 16 * Nn + 4 * Pp + 8.0 * (3 * Pp + 9 * Cc);
  // J, chunk ids, g and the diagonal; the subspace variant also reads gn (b200_lm_solve sets that figure for its run)
  bpo[K_DOGLEG_GRAM] = 196 * Nn + 4 * Pp + 16.0 * (3 * Pp + 9 * Cc);
  bpo[K_DOGLEG_DIAG] = 48.0 * (3 * Pp + 9 * Cc);   // refresh: colnorm^2, gradient, scale read; diagonal, g, D written
  bpo[K_DOGLEG_GN] = 32.0 * (3 * Pp + 9 * Cc);     // y, diagonal, g read; gn written
  bpo[K_DOGLEG_STEP] = 56.0 * (3 * Pp + 9 * Cc);   // g, gn, diagonal, scale, x read; step, cand written
  if (pl.xs) {   // explicit S: the product and the assembly that replaces the block-diagonal pass
    bpo[K_SCHUR_MUL] = xs_mul_bytes;
    bpo[K_DIAG_BLOCKS] = xs_asm_bytes;
    // one iteration of the resident PCG (xs_pcg.cuh): S and its column entries, T written and read, M^-1, and p, x, r, z
    // read and written
    const double nb = static_cast<double>(pl.xp.blk_row.size()), off = static_cast<double>(pl.xp.off_blocks);
    if (pl.xs_pcg) bpo[K_SCHUR_PCG] = 656.0 * nb + 144.0 * off + 648.0 * Cc + 8 * 72.0 * Cc;
  }
}

// The B200_VERBOSE lines of a plan: the point order, the L2 residency plan of S*x (v4), the kernel configuration and the
// S plan.
inline void print_plan(const KernelPlan& pl, int C, int P, int N, int world, const DevLimits& lim, const DevKnobs& knobs) {
  if (getenv("B200_VERBOSE") == nullptr) return;
  if (!knobs.keep_order)
    fprintf(stderr, "[b200ba] point order: distinct cameras per 1/%d of the rows, summed: caller %ld, by camera arc %ld, by mean camera %ld, by smallest camera %ld -> %s\n",
            lim.sm_count, pl.order_metrics[0], pl.order_metrics[1], pl.order_metrics[2], pl.order_metrics[3], kOrderNames[pl.order_choice]);
  const V2View &v = pl.v2, &m = pl.v2_mul;
  if (is_v4(pl.mul)) {
    const uint32_t s = m.l2_stream;
    fprintf(stderr, "[b200ba] S*x L2 plan (L2 %d MiB, budget %.1f MiB): resident %.1f MiB, streamed %.1f MiB, stride %.2f tiles (%s)\n",
            lim.l2_bytes >> 20, pl.l2_budget / (1 << 20), pl.l2_resident_bytes / (1 << 20), (pl.l2_stream_bytes - pl.l2_resident_bytes) / (1 << 20),
            s < 65536 ? 65536.0 / (65536 - s) : 0.0, m.l2_last ? "evict_last" : "evict_normal");
  }
  // mul: the S*x family; v2b: the warp-tile evaluate (family v4); diag: the block-diagonal pass precond_update_dev runs
  const char* const mul_names[] = {"tile", "v3", "v4", "v4-owned"};
  const char* const diag_names[] = {"cam_major", "v2", "tile"};
  fprintf(stderr,
          "[b200ba] C=%d P=%d N=%d wtiles=%zu big(+slices)=%zu huge=%d span=%d direct=%d v2(w=%d,s=%d,r=%d) mul(%s w=%d,s=%d,r=%d,smem=%zu) folded=%d v2b=%d cam_major=%d diag=%s\n",
          C, P, N, pl.wtiles.size(), pl.big_tiles.size(), static_cast<int>(pl.huge_pts.size()), pl.max_cam_span, v.direct, v.warps, v.stages,
          v.replicas, mul_names[static_cast<int>(pl.mul)], m.warps, m.stages, m.replicas, pl.mul_smem, pl.big_folded ? 1 : 0,
          is_v4(pl.mul) ? 1 : 0, pl.diag == DiagPass::CamMajor ? 1 : 0, diag_names[static_cast<int>(pl.diag)]);
  if (world == 1) {
    fprintf(stderr, "[b200ba] S plan: %s, %lld pairs, %.1f MB\n", pl.xs ? "explicit" : "implicit", pl.xp.off_blocks,
            648.0 * static_cast<double>(pl.xp.blk_row.size()) / 1e6);
    if (pl.xs)
      fprintf(stderr, "[b200ba] S product: grid %d of %d resident CTAs (%d per SM), %d warps, at most %d steps per warp\n",
              pl.xs_grid, pl.xs_resident, lim.xs_ctas_per_sm, pl.xs_grid * kXsWarps, pl.xs_max_steps);
    if (pl.xs) {
      const double share = 648.0 * pl.xs_pcg_max_blocks / 1024.0, limit = static_cast<double>(lim.smem_optin) / 1024.0;
      const double cta = static_cast<double>(pl.xs_pcg_smem) / 1024.0;
      if (pl.xs_pcg) {
        fprintf(stderr, "[b200ba] S PCG: resident, %d CTAs, largest S share %.2f KiB of %.2f KiB (%.2f KiB with M^-1, vectors and staging), %d warps, at most %d steps per warp, at most %d foreign columns, at most %d column slots per CTA (%d staged)\n",
                lim.sm_count, share, limit, cta, lim.sm_count * kXpWarps, pl.xs_pcg_max_steps, pl.xs_pcg_max_foreign, pl.xs_pcg_max_slots,
                pl.xs_pcg_stage_slots);
        fprintf(stderr, "[b200ba] S PCG walk: at most %d steps per warp (one per row segment included), %d split rows\n",
                pl.xs_pcg_walk_max, pl.xs_pcg_split_rows);
      } else {
        fprintf(stderr, "[b200ba] S PCG: two-kernel (%s: largest S share %.2f KiB, %.2f KiB with M^-1, vectors and staging, of %.2f KiB)\n",
                pl.xs_pcg_why, share, cta, limit);
      }
    }
  } else
    fprintf(stderr, "[b200ba] S plan: implicit, sharded\n");
}

}  // namespace b200
