// Symbolic analysis of the sparse Cholesky factorisation of the reduced camera system (SPARSE_SCHUR,
// SparseSchurComplementSolver, schur_complement_solver.cc:205-335), at the level of 9x9 camera blocks.  Host code only, no
// CUDA runtime call: b200_plan_sparse_schur runs it without a GPU, and the first b200_sparse_schur_solve of a handle runs it
// once and uploads the result (sparse_schur.cuh).
//
// Input: the block pattern of the upper triangle of S (XsPattern, plan.cuh), in the caller's camera ids.  Cameras are
// eliminated in a fill-reducing order: the caller's order or a minimum-degree order, whichever needs fewer factor flops (the
// caller's on a tie).  The reference lets CHOLMOD's AMD choose (suitesparse.cc:167-183); an exact solve does not depend on the
// order, and on a video sequence the caller's order is already a band with no fill, which minimum degree can make worse.
//
// Supernodes: consecutive columns j, j+1, ... of the chosen order whose elimination-tree parent is the next column, merged
// while the supernode has at most kSnMaxCams cameras and the explicit zero blocks the merge adds stay within kSnRelax of its
// storage (relaxed amalgamation).  A supernode [f, l] stores, column-major, the dense panel of its rows: its own columns f..l
// (the diagonal block; only its lower triangle is meaningful) then the rows of column l below l, which contain the rows of
// every other column of the supernode below l.  Positions below are camera positions in the chosen order.
#pragma once
#include <algorithm>
#include <cstdint>
#include <set>
#include <vector>

#include "../../include/b200ba.h"
#include "plan.cuh"

namespace b200 {

constexpr int kSnMaxCams = 16;            // widest supernode (cameras): its 144 x 144 update stage fits one CTA's shared memory
constexpr double kSnRelax = 0.25;         // share of a supernode's storage that merges may spend on explicit zero blocks
constexpr int kMinDegreeMaxCams = 32768;  // the minimum-degree elimination graph is a C x C bit matrix (128 MB at this size)
constexpr int kSpAlign = 16;              // panels start on 128-byte boundaries: no cache line holds two supernodes' values

// Factor flops of one block column with k blocks below the diagonal: Cholesky of the 9x9 diagonal block (9^3 / 3), the
// triangular solve of k blocks (k 9^3) and the k (k + 1) / 2 block products of the update (2 x 9^3 each).
inline double column_flops(double k) { return 243.0 + 729.0 * k + 729.0 * k * (k + 1.0); }

struct Elimination {
  long long l_blocks = 0;                // blocks of L, diagonal included
  double flops = 0.0;
  int height = 0;                        // nodes on the longest root-to-leaf path of the elimination tree
  std::vector<int> parent;               // by position; -1 for a root
  std::vector<std::vector<int>> below;   // positions of the blocks below the diagonal of each column (kept on request)
};

// Block-level symbolic elimination of the camera graph `adj` (off-diagonal neighbours of each camera) in the order with
// positions pinv[camera]: the row structure of column j is its own lower neighbours and its children's rows, minus j.
inline void eliminate(int C, const std::vector<std::vector<int>>& adj, const std::vector<int>& pinv, bool keep_rows, Elimination* e) {
  std::vector<std::vector<int>> lower(static_cast<size_t>(C)), rows(static_cast<size_t>(C)), kids(static_cast<size_t>(C));
  for (int i = 0; i < C; ++i)
    for (int j : adj[i])
      if (pinv[i] < pinv[j]) lower[pinv[i]].push_back(pinv[j]);
  e->parent.assign(static_cast<size_t>(C), -1);
  std::vector<int> mark(static_cast<size_t>(C), -1);
  for (int j = 0; j < C; ++j) {
    std::vector<int>& s = rows[j];
    auto add = [&](int x) {
      if (x != j && mark[x] != j) {
        mark[x] = j;
        s.push_back(x);
      }
    };
    for (int x : lower[j]) add(x);
    for (int c : kids[j]) {
      for (int x : rows[c]) add(x);
      if (!keep_rows) std::vector<int>().swap(rows[c]);
    }
    std::sort(s.begin(), s.end());
    e->l_blocks += 1 + static_cast<long long>(s.size());
    e->flops += column_flops(static_cast<double>(s.size()));
    if (!s.empty()) {
      e->parent[j] = s[0];
      kids[s[0]].push_back(j);
    }
  }
  std::vector<int> depth(static_cast<size_t>(C), 1);
  e->height = 0;
  for (int j = C - 1; j >= 0; --j) {
    if (e->parent[j] >= 0) depth[j] = depth[e->parent[j]] + 1;
    e->height = std::max(e->height, depth[j]);
  }
  if (keep_rows) e->below = std::move(rows);
}

// Minimum-degree order on the explicit elimination graph (a bit matrix): repeatedly eliminate the camera of least degree,
// the smallest id on a tie, and join its neighbours into a clique.
inline std::vector<int> minimum_degree_order(int C, const std::vector<std::vector<int>>& adj) {
  const size_t W = (static_cast<size_t>(C) + 63) / 64;
  std::vector<uint64_t> g(W * static_cast<size_t>(C), 0);
  std::vector<int> deg(static_cast<size_t>(C));
  std::set<std::pair<int, int>> queue;
  for (int i = 0; i < C; ++i) {
    for (int j : adj[i]) g[i * W + j / 64] |= 1ull << (j % 64);
    deg[i] = static_cast<int>(adj[i].size());
    queue.insert({deg[i], i});
  }
  std::vector<int> order, nb;
  order.reserve(static_cast<size_t>(C));
  while (!queue.empty()) {
    const int v = queue.begin()->second;
    queue.erase(queue.begin());
    order.push_back(v);
    const uint64_t* gv = g.data() + v * W;
    nb.clear();
    for (size_t w = 0; w < W; ++w)
      for (uint64_t m = gv[w]; m != 0; m &= m - 1) nb.push_back(static_cast<int>(w * 64 + __builtin_ctzll(m)));
    for (int u : nb) {
      uint64_t* gu = g.data() + u * W;
      for (size_t w = 0; w < W; ++w) gu[w] |= gv[w];
      gu[u / 64] &= ~(1ull << (u % 64));
      gu[v / 64] &= ~(1ull << (v % 64));
      int d = 0;
      for (size_t w = 0; w < W; ++w) d += __builtin_popcountll(gu[w]);
      queue.erase({deg[u], u});
      deg[u] = d;
      queue.insert({d, u});
    }
  }
  return order;
}

struct SparsePlan {
  int C = 0, ns = 0;
  int64_t stats[B200_SPARSE_STATS] = {};
  std::vector<int> perm, pinv;              // position k holds camera perm[k]; pinv[camera] = position
  std::vector<int> sn_first;                // [ns + 1] first column (position) of each supernode
  std::vector<int> row_ptr, rows;           // [ns + 1] / positions: the supernode's columns, then its rows below, ascending
  std::vector<long long> val;               // [ns] offset of each panel in the factor storage (doubles)
  long long storage = 0;                    // doubles of factor storage
  std::vector<int> upd_ptr;                 // [ns + 1]
  std::vector<int4> upd;                    // {d, k0, k1, 0}: rows k0..k1-1 of descendant d lie in this supernode's columns
  std::vector<int> ntf_ptr, ntf;            // [ns + 1] / the supernodes each supernode updates, ascending
  std::vector<int> cnt;                     // [2 ns] initial dependency counters of the forward and backward tasks
  std::vector<long long> blk_off;           // per S block: offset of its 9x9 block in the factor storage
  std::vector<int> blk_ld;                  // ... and the panel's leading dimension, negated when the block goes in transposed
  int max_width = 0;                        // widest supernode (scalar columns)
};

// The plan of S's block pattern (upper triangle, blocks (i, j >= i), every diagonal block present) for C cameras.
inline void plan_sparse_schur(int C, const std::vector<int>& blk_row, const std::vector<int>& blk_col, SparsePlan* out) {
  SparsePlan& sp = *out;
  sp.C = C;
  std::vector<std::vector<int>> adj(static_cast<size_t>(C));
  for (size_t b = 0; b < blk_row.size(); ++b)
    if (blk_row[b] != blk_col[b]) {
      adj[blk_row[b]].push_back(blk_col[b]);
      adj[blk_col[b]].push_back(blk_row[b]);
    }
  std::vector<int> ident(static_cast<size_t>(C));
  for (int i = 0; i < C; ++i) ident[i] = i;
  Elimination caller, md;
  eliminate(C, adj, ident, false, &caller);
  std::vector<int> md_perm;
  if (C <= kMinDegreeMaxCams) {
    md_perm = minimum_degree_order(C, adj);
    std::vector<int> md_pinv(static_cast<size_t>(C));
    for (int k = 0; k < C; ++k) md_pinv[md_perm[k]] = k;
    eliminate(C, adj, md_pinv, false, &md);
  } else {
    md = caller;   // not tried: reported with the caller's counts
  }
  const bool use_md = C <= kMinDegreeMaxCams && md.flops < caller.flops;
  sp.perm = use_md ? md_perm : ident;
  sp.pinv.assign(static_cast<size_t>(C), 0);
  for (int k = 0; k < C; ++k) sp.pinv[sp.perm[k]] = k;
  Elimination e;
  eliminate(C, adj, sp.pinv, true, &e);

  // relaxed supernodes
  sp.sn_first.clear();
  sp.sn_first.push_back(0);
  long long true_blocks = 1 + static_cast<long long>(e.below[0].size());
  for (int j = 1; j < C; ++j) {
    const int f = sp.sn_first.back();
    bool merge = e.parent[j - 1] == j && j - f < kSnMaxCams;
    if (merge) {
      const long long w = j - f + 1, tb = true_blocks + 1 + static_cast<long long>(e.below[j].size());
      const long long stored = w * (w + 1) / 2 + w * static_cast<long long>(e.below[j].size());
      merge = static_cast<double>(stored - tb) <= kSnRelax * static_cast<double>(stored);
      if (merge) true_blocks = tb;
    }
    if (!merge) {
      sp.sn_first.push_back(j);
      true_blocks = 1 + static_cast<long long>(e.below[j].size());
    }
  }
  sp.ns = static_cast<int>(sp.sn_first.size());
  sp.sn_first.push_back(C);
  const int ns = sp.ns;
  std::vector<int> sn_of(static_cast<size_t>(C));
  sp.row_ptr.assign(1, 0);
  sp.val.resize(static_cast<size_t>(ns));
  sp.storage = 0;
  for (int s = 0; s < ns; ++s) {
    const int f = sp.sn_first[s], l = sp.sn_first[s + 1] - 1;
    for (int c = f; c <= l; ++c) {
      sn_of[c] = s;
      sp.rows.push_back(c);
    }
    sp.rows.insert(sp.rows.end(), e.below[l].begin(), e.below[l].end());
    sp.row_ptr.push_back(static_cast<int>(sp.rows.size()));
    const long long R = sp.row_ptr[s + 1] - sp.row_ptr[s], w = l - f + 1;
    sp.val[s] = sp.storage;
    sp.storage += (81 * R * w + kSpAlign - 1) / kSpAlign * kSpAlign;
    sp.max_width = std::max(sp.max_width, static_cast<int>(9 * w));
  }
  // update lists: descendant d updates the supernode owning each run of its rows below its own columns
  std::vector<std::vector<int4>> upd(static_cast<size_t>(ns));
  sp.ntf_ptr.assign(1, 0);
  for (int d = 0; d < ns; ++d) {
    const int r0 = sp.row_ptr[d], w = sp.sn_first[d + 1] - sp.sn_first[d], R = sp.row_ptr[d + 1] - r0;
    for (int k = w; k < R;) {
      const int s = sn_of[sp.rows[r0 + k]];
      int k1 = k;
      while (k1 < R && sn_of[sp.rows[r0 + k1]] == s) ++k1;
      upd[s].push_back(make_int4(d, k, k1, 0));
      sp.ntf.push_back(s);
      k = k1;
    }
    sp.ntf_ptr.push_back(static_cast<int>(sp.ntf.size()));
  }
  sp.upd_ptr.assign(1, 0);
  for (int s = 0; s < ns; ++s) {
    sp.upd.insert(sp.upd.end(), upd[s].begin(), upd[s].end());
    sp.upd_ptr.push_back(static_cast<int>(sp.upd.size()));
  }
  // forward task of s: after every descendant that updates it; backward task: after every supernode it updates (a root: after
  // its own forward task)
  sp.cnt.assign(2 * static_cast<size_t>(ns), 0);
  for (int s = 0; s < ns; ++s) {
    sp.cnt[s] = sp.upd_ptr[s + 1] - sp.upd_ptr[s];
    const int n = sp.ntf_ptr[s + 1] - sp.ntf_ptr[s];
    sp.cnt[ns + s] = n > 0 ? n : 1;
  }
  // where each block of S (and its transpose) goes
  sp.blk_off.resize(blk_row.size());
  sp.blk_ld.resize(blk_row.size());
  for (size_t b = 0; b < blk_row.size(); ++b) {
    const int a = sp.pinv[blk_row[b]], c = sp.pinv[blk_col[b]];
    const int lo = std::min(a, c), hi = std::max(a, c), s = sn_of[lo];
    const int f = sp.sn_first[s], r0 = sp.row_ptr[s], R = sp.row_ptr[s + 1] - r0;
    const int idx = static_cast<int>(std::lower_bound(sp.rows.begin() + r0, sp.rows.begin() + r0 + R, hi) - (sp.rows.begin() + r0));
    const int ld = 9 * R;
    sp.blk_off[b] = sp.val[s] + 9LL * idx + 9LL * (lo - f) * ld;
    sp.blk_ld[b] = a < c ? -ld : ld;   // S_ij with i eliminated first lands in L as S_ij'
  }
  int64_t* st = sp.stats;
  st[B200_SPARSE_STAT_S_BLOCKS] = static_cast<int64_t>(blk_row.size());
  st[B200_SPARSE_STAT_L_BLOCKS] = e.l_blocks;
  st[B200_SPARSE_STAT_L_BLOCKS_CALLER] = caller.l_blocks;
  st[B200_SPARSE_STAT_L_BLOCKS_MIN_DEGREE] = md.l_blocks;
  st[B200_SPARSE_STAT_FLOPS_CALLER] = static_cast<int64_t>(caller.flops);
  st[B200_SPARSE_STAT_FLOPS_MIN_DEGREE] = static_cast<int64_t>(md.flops);
  st[B200_SPARSE_STAT_SUPERNODES] = ns;
  st[B200_SPARSE_STAT_TREE_HEIGHT] = e.height;
  st[B200_SPARSE_STAT_ORDER] = use_md ? 1 : 0;
  st[B200_SPARSE_STAT_FACTOR_BYTES] = 8 * sp.storage;
}

}  // namespace b200
