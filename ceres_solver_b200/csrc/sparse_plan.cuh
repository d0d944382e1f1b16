// Symbolic analysis of the sparse Cholesky factorisation of the reduced camera system (SPARSE_SCHUR,
// SparseSchurComplementSolver, schur_complement_solver.cc:205-335), at the level of 9x9 camera blocks.  Host code only, no
// CUDA runtime call: b200_plan_sparse_schur runs it without a GPU, and the first b200_sparse_schur_solve of a handle runs it
// once and uploads the result (sparse_schur.cuh).
//
// Input: the block pattern of the upper triangle of S (XsPattern, plan.cuh), in the caller's camera ids, and Ceres'
// linear_solver_ordering_type.  With B200_AMD, cameras are eliminated in a fill-reducing order: the caller's order or a
// minimum-degree order, whichever needs fewer factor flops (the caller's on a tie).  The reference lets CHOLMOD's AMD choose
// (suitesparse.cc:167-183); an exact solve does not depend on the order, and on a video sequence the caller's order is already
// a band with no fill, which minimum degree can make worse.  With B200_NESDIS the order is always nested dissection (below),
// as Ceres orders by METIS then (suitesparse.cc:53-66).
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

// ---- Nested dissection (linear_solver_ordering_type = NESDIS, solver.h:410; for the Schur solvers the reduced camera system
// is what is ordered, nnls_solving.rst:1160-1172).  The graph is split by a small vertex separator into two parts, which are
// ordered first (recursively), and the separator is numbered last (George, "Nested dissection of a regular finite element
// mesh", SIAM J. Numer. Anal. 10, 1973): the two parts never fill into each other, so their subtrees of the elimination tree
// are independent and the tree is shallow where the caller's or a minimum-degree order of a band graph gives a chain.
//
// Each separator comes from a multilevel bisection (Hendrickson and Leland, "A multilevel algorithm for partitioning
// graphs", Supercomputing 1995; Karypis and Kumar, "A fast and high quality multilevel scheme for partitioning irregular
// graphs", SIAM J. Sci. Comput. 20, 1998): the graph is coarsened by heavy-edge matching, the coarsest graph is split by
// greedy graph growing from a few start vertices, the best split is projected back level by level and refined at each by
// Fiduccia-Mattheyses passes ("A linear-time heuristic for improving network partitions", DAC 1982) under the balance bound
// kNdImbalance.  The edge cut becomes a vertex separator by a minimum vertex cover of the bipartite graph of the cut edges
// (Konig's theorem, from a Hopcroft-Karp maximum matching, SIAM J. Comput. 2, 1973).  No random number is drawn, and every
// tie goes to the smallest camera id (local vertex ids keep the camera ids' order; a coarse vertex is numbered by its
// smallest member), so a structure always gets the same order.
constexpr int kNdLeafCams = 64;        // parts of at most this many cameras are ordered by minimum degree (DESIGN §3.5)
constexpr int kNdCoarsest = 100;       // coarsening stops at this many vertices ...
constexpr double kNdMinShrink = 0.9;   // ... or when a level keeps more than this share of the vertices
constexpr double kNdImbalance = 1.1;   // the heavier part weighs at most 1.1 x half the graph (55%)
constexpr int kNdFmPasses = 8;         // Fiduccia-Mattheyses passes per level, fewer when a pass gains nothing
constexpr int kNdFmStall = 64;         // a pass ends after this many moves without a better partition

struct NdGraph {                       // CSR, neighbours ascending, with vertex and edge weights
  std::vector<int> ptr, adj, ew, vw;
  int n() const { return static_cast<int>(vw.size()); }
};

// One level of heavy-edge matching: each unmatched vertex, in ascending order, is matched with the unmatched neighbour of
// the heaviest edge (the smallest on a tie) or stays alone.  false when the level would not shrink the graph enough.
inline bool nd_coarsen(const NdGraph& g, NdGraph* c, std::vector<int>* cmap) {
  const int n = g.n();
  std::vector<int> match(static_cast<size_t>(n), -1);
  for (int v = 0; v < n; ++v) {
    if (match[v] >= 0) continue;
    int best = v, bw = 0;
    for (int k = g.ptr[v]; k < g.ptr[v + 1]; ++k)
      if (match[g.adj[k]] < 0 && g.ew[k] > bw) {
        bw = g.ew[k];
        best = g.adj[k];
      }
    match[v] = best;
    match[best] = v;
  }
  std::vector<int>& m = *cmap;
  m.assign(static_cast<size_t>(n), -1);
  int nc = 0;
  for (int v = 0; v < n; ++v)
    if (m[v] < 0) m[v] = m[match[v]] = nc++;
  if (nc > kNdMinShrink * n) return false;
  c->ptr.assign(1, 0);
  c->adj.clear();
  c->ew.clear();
  c->vw.assign(static_cast<size_t>(nc), 0);
  std::vector<int> slot(static_cast<size_t>(nc), -1);
  std::vector<std::pair<int, int>> row;
  for (int v = 0; v < n; ++v) {   // coarse vertices in the order of their smaller member
    if (match[v] < v) continue;
    const int cv = m[v];
    row.clear();
    for (int x : {v, match[v]}) {
      c->vw[cv] += g.vw[x];
      for (int k = g.ptr[x]; k < g.ptr[x + 1]; ++k) {
        const int cu = m[g.adj[k]];
        if (cu == cv) continue;
        if (slot[cu] < 0) {
          slot[cu] = static_cast<int>(row.size());
          row.push_back({cu, 0});
        }
        row[slot[cu]].second += g.ew[k];
      }
      if (match[v] == v) break;
    }
    std::sort(row.begin(), row.end());
    for (const auto& r : row) {
      c->adj.push_back(r.first);
      c->ew.push_back(r.second);
      slot[r.first] = -1;
    }
    c->ptr.push_back(static_cast<int>(c->adj.size()));
  }
  return true;
}

// The last vertex (smallest id among the farthest) of a breadth-first search from `s`; *ecc its distance.
inline int nd_farthest(const NdGraph& g, int s, int* ecc) {
  std::vector<int> dist(static_cast<size_t>(g.n()), -1), q{s};
  dist[s] = 0;
  int far = s;
  for (size_t h = 0; h < q.size(); ++h) {
    const int v = q[h];
    if (dist[v] > dist[far] || (dist[v] == dist[far] && v < far)) far = v;
    for (int k = g.ptr[v]; k < g.ptr[v + 1]; ++k)
      if (dist[g.adj[k]] < 0) {
        dist[g.adj[k]] = dist[v] + 1;
        q.push_back(g.adj[k]);
      }
  }
  *ecc = dist[far];
  return far;
}

// A pseudo-peripheral vertex (Gibbs, Poole and Stockmeyer, SIAM J. Numer. Anal. 13, 1976): repeated farthest-vertex searches
// from `s` while the eccentricity grows.
inline int nd_peripheral(const NdGraph& g, int s) {
  int ecc = -1;
  for (int it = 0; it < 8; ++it) {
    int e = 0;
    const int f = nd_farthest(g, s, &e);
    if (e <= ecc) break;
    ecc = e;
    s = f;
  }
  return s;
}

struct NdCut {   // comparison key of a bisection: weight above the bound, then cut, then imbalance
  long long over, cut, diff;
  bool operator<(const NdCut& o) const {
    return over != o.over ? over < o.over : cut != o.cut ? cut < o.cut : diff < o.diff;
  }
};

inline NdCut nd_key(long long w0, long long w1, long long maxw, long long cut) {
  return {std::max(0LL, std::max(w0, w1) - maxw), cut, w0 > w1 ? w0 - w1 : w1 - w0};
}

// Fiduccia-Mattheyses refinement of `part` (0 / 1 per vertex): each pass moves boundary vertices one at a time, the move of
// largest gain first (the heavier side's, then the smallest id, on a tie), each vertex at most once, while the receiving
// side stays within maxw (or the giving side is above it), and keeps the best prefix of its moves.  Returns the final key.
inline NdCut nd_refine(const NdGraph& g, std::vector<char>* part_io, long long maxw) {
  std::vector<char>& part = *part_io;
  const int n = g.n();
  std::vector<long long> ext(static_cast<size_t>(n)), in(static_cast<size_t>(n));
  std::vector<char> locked(static_cast<size_t>(n));
  NdCut key{};
  for (int pass = 0; pass < kNdFmPasses; ++pass) {
    long long w[2] = {0, 0}, cut = 0;
    for (int v = 0; v < n; ++v) {
      w[part[v]] += g.vw[v];
      ext[v] = in[v] = 0;
      for (int k = g.ptr[v]; k < g.ptr[v + 1]; ++k) (part[g.adj[k]] == part[v] ? in[v] : ext[v]) += g.ew[k];
      cut += ext[v];
    }
    cut /= 2;
    key = nd_key(w[0], w[1], maxw, cut);
    std::set<std::pair<long long, int>> q[2];   // (-gain, vertex) of the unlocked boundary vertices of each side
    for (int v = 0; v < n; ++v) {
      locked[v] = 0;
      if (ext[v] > 0) q[part[v]].insert({in[v] - ext[v], v});
    }
    NdCut best = key;
    std::vector<int> moves;
    size_t best_len = 0;
    int stall = 0;
    while (stall < kNdFmStall) {
      int pick = -1, from = -1;
      for (int s = 0; s < 2; ++s) {
        if (q[s].empty()) continue;
        const int v = q[s].begin()->second;
        if (w[1 - s] + g.vw[v] > maxw && w[s] <= maxw) continue;
        if (pick < 0) {
          pick = v;
          from = s;
          continue;
        }
        const long long gv = -q[s].begin()->first, gp = ext[pick] - in[pick];
        if (gv > gp || (gv == gp && (w[s] > w[from] || (w[s] == w[from] && v < pick)))) {
          pick = v;
          from = s;
        }
      }
      if (pick < 0) break;
      const int v = pick, to = 1 - from;
      q[from].erase({in[v] - ext[v], v});
      locked[v] = 1;
      cut -= ext[v] - in[v];
      part[v] = static_cast<char>(to);
      std::swap(ext[v], in[v]);
      w[from] -= g.vw[v];
      w[to] += g.vw[v];
      for (int k = g.ptr[v]; k < g.ptr[v + 1]; ++k) {
        const int u = g.adj[k];
        if (!locked[u] && ext[u] > 0) q[part[u]].erase({in[u] - ext[u], u});
        if (part[u] == to) { ext[u] -= g.ew[k]; in[u] += g.ew[k]; }
        else { ext[u] += g.ew[k]; in[u] -= g.ew[k]; }
        if (!locked[u] && ext[u] > 0) q[part[u]].insert({in[u] - ext[u], u});
      }
      moves.push_back(v);
      const NdCut k = nd_key(w[0], w[1], maxw, cut);
      if (k < best) {
        best = k;
        best_len = moves.size();
        stall = 0;
      } else {
        ++stall;
      }
    }
    for (size_t i = best_len; i < moves.size(); ++i) part[moves[i]] ^= 1;
    key = best;
    if (best_len == 0) break;
  }
  return key;
}

// Greedy graph growing (Karypis and Kumar, 1998, section 4.1): side 0 grows from `seed` by the boundary vertex whose move
// lowers the cut most (the smallest id on a tie) until it holds half the weight.
inline std::vector<char> nd_grow(const NdGraph& g, int seed) {
  const int n = g.n();
  long long total = 0, w0 = 0;
  for (int v = 0; v < n; ++v) total += g.vw[v];
  std::vector<char> part(static_cast<size_t>(n), 1);
  std::vector<long long> to0(static_cast<size_t>(n), 0), deg(static_cast<size_t>(n), 0);
  for (int v = 0; v < n; ++v)
    for (int k = g.ptr[v]; k < g.ptr[v + 1]; ++k) deg[v] += g.ew[k];
  std::set<std::pair<long long, int>> front;   // (-gain, vertex) of side-1 vertices next to side 0
  int v = seed;
  while (2 * w0 < total) {
    part[v] = 0;
    w0 += g.vw[v];
    for (int k = g.ptr[v]; k < g.ptr[v + 1]; ++k) {
      const int u = g.adj[k];
      if (part[u] == 0) continue;
      if (to0[u] > 0) front.erase({deg[u] - 2 * to0[u], u});
      to0[u] += g.ew[k];
      front.insert({deg[u] - 2 * to0[u], u});
    }
    if (front.empty()) break;   // only for a disconnected graph, which is never bisected
    v = front.begin()->second;
    front.erase(front.begin());
  }
  return part;
}

// The multilevel bisection of a connected graph of more than one vertex: 0 / 1 per vertex, both sides non-empty.
inline std::vector<char> nd_bisect(const NdGraph& g) {
  std::vector<NdGraph> lv(1, g);
  std::vector<std::vector<int>> maps;
  while (lv.back().n() > kNdCoarsest) {
    NdGraph c;
    std::vector<int> m;
    if (!nd_coarsen(lv.back(), &c, &m)) break;
    lv.push_back(std::move(c));
    maps.push_back(std::move(m));
  }
  long long total = 0;
  for (int w : g.vw) total += w;
  const long long maxw = std::max((total + 1) / 2, static_cast<long long>(kNdImbalance * static_cast<double>(total) / 2.0));
  // starts: pseudo-peripheral vertices found from the first, middle and last vertex, and the middle vertex itself
  const NdGraph& cg = lv.back();
  const int nc = cg.n();
  std::vector<int> starts{nd_peripheral(cg, 0), nd_peripheral(cg, nc / 2), nd_peripheral(cg, nc - 1), nc / 2};
  std::vector<char> part;
  NdCut best{};
  for (size_t i = 0; i < starts.size(); ++i) {
    if (std::find(starts.begin(), starts.begin() + i, starts[i]) != starts.begin() + i) continue;
    std::vector<char> p = nd_grow(cg, starts[i]);
    const NdCut k = nd_refine(cg, &p, maxw);
    if (part.empty() || k < best) {
      best = k;
      part = std::move(p);
    }
  }
  for (size_t l = maps.size(); l-- > 0;) {
    std::vector<char> fine(maps[l].size());
    for (size_t v = 0; v < fine.size(); ++v) fine[v] = part[maps[l][v]];
    part = std::move(fine);
    nd_refine(lv[l], &part, maxw);
  }
  return part;
}

// The vertex separator of a bisection: a minimum vertex cover of the bipartite graph of its cut edges (Konig: from a maximum
// matching, the side-0 boundary vertices not reachable from an unmatched side-0 vertex by an alternating path, and the side-1
// boundary vertices that are).  Returns 0 / 1 for the two parts, 2 for the separator.
inline std::vector<char> nd_separator(const NdGraph& g, const std::vector<char>& part) {
  const int n = g.n();
  std::vector<int> id(static_cast<size_t>(n), -1), L, R;
  for (int v = 0; v < n; ++v)
    for (int k = g.ptr[v]; k < g.ptr[v + 1]; ++k)
      if (part[g.adj[k]] != part[v]) {
        std::vector<int>& side = part[v] == 0 ? L : R;
        id[v] = static_cast<int>(side.size());
        side.push_back(v);
        break;
      }
  const int nl = static_cast<int>(L.size()), nr = static_cast<int>(R.size());
  std::vector<int> bptr(1, 0), badj;   // cut edges from each side-0 boundary vertex, ascending
  for (int v : L) {
    for (int k = g.ptr[v]; k < g.ptr[v + 1]; ++k)
      if (part[g.adj[k]] == 1) badj.push_back(id[g.adj[k]]);
    bptr.push_back(static_cast<int>(badj.size()));
  }
  // Hopcroft-Karp
  std::vector<int> mateL(static_cast<size_t>(nl), -1), mateR(static_cast<size_t>(nr), -1), dist(static_cast<size_t>(nl));
  const int kInf = 1 << 30;
  auto bfs = [&]() {
    std::vector<int> q;
    bool found = false;
    for (int l = 0; l < nl; ++l) {
      dist[l] = mateL[l] < 0 ? 0 : kInf;
      if (mateL[l] < 0) q.push_back(l);
    }
    for (size_t h = 0; h < q.size(); ++h) {
      const int l = q[h];
      for (int k = bptr[l]; k < bptr[l + 1]; ++k) {
        const int m = mateR[badj[k]];
        if (m < 0) found = true;
        else if (dist[m] == kInf) {
          dist[m] = dist[l] + 1;
          q.push_back(m);
        }
      }
    }
    return found;
  };
  struct Dfs {
    const std::vector<int>&bptr, &badj;
    std::vector<int>&mateL, &mateR, &dist;
    bool operator()(int l) {
      for (int k = bptr[l]; k < bptr[l + 1]; ++k) {
        const int r = badj[k], m = mateR[r];
        if (m < 0 || (dist[m] == dist[l] + 1 && (*this)(m))) {
          mateL[l] = r;
          mateR[r] = l;
          return true;
        }
      }
      dist[l] = 1 << 30;
      return false;
    }
  } dfs{bptr, badj, mateL, mateR, dist};
  while (bfs())
    for (int l = 0; l < nl; ++l)
      if (mateL[l] < 0) dfs(l);
  // alternating reachability from the unmatched side-0 vertices
  std::vector<char> zl(static_cast<size_t>(nl), 0), zr(static_cast<size_t>(nr), 0);
  std::vector<int> q;
  for (int l = 0; l < nl; ++l)
    if (mateL[l] < 0) {
      zl[l] = 1;
      q.push_back(l);
    }
  for (size_t h = 0; h < q.size(); ++h)
    for (int k = bptr[q[h]]; k < bptr[q[h] + 1]; ++k) {
      const int r = badj[k];
      if (zr[r]) continue;
      zr[r] = 1;
      const int m = mateR[r];   // matched: a maximum matching leaves no augmenting path
      if (m >= 0 && !zl[m]) {
        zl[m] = 1;
        q.push_back(m);
      }
    }
  std::vector<char> lab(part.begin(), part.end());
  for (int l = 0; l < nl; ++l)
    if (!zl[l]) lab[L[l]] = 2;
  for (int r = 0; r < nr; ++r)
    if (zr[r]) lab[R[r]] = 2;
  return lab;
}

// Appends the nested-dissection order of the cameras `vs` (ascending) of the graph `adj` to *out.  loc: -1 for every camera
// on entry and on return (the local ids of the induced subgraph while it is built).
inline void nd_order(const std::vector<std::vector<int>>& adj, const std::vector<int>& vs, std::vector<int>* loc, std::vector<int>* out) {
  const int n = static_cast<int>(vs.size());
  if (n == 0) return;
  std::vector<int>& lc = *loc;
  for (int i = 0; i < n; ++i) lc[vs[i]] = i;
  std::vector<std::vector<int>> sub(static_cast<size_t>(n));
  for (int i = 0; i < n; ++i) {
    for (int j : adj[vs[i]])
      if (lc[j] >= 0) sub[i].push_back(lc[j]);
    std::sort(sub[i].begin(), sub[i].end());
  }
  for (int v : vs) lc[v] = -1;
  // connected components, in the order of their smallest camera, each ordered on its own
  std::vector<int> comp(static_cast<size_t>(n), -1), q;
  int ncomp = 0;
  for (int s = 0; s < n; ++s) {
    if (comp[s] >= 0) continue;
    comp[s] = ncomp;
    q.assign(1, s);
    for (size_t h = 0; h < q.size(); ++h)
      for (int u : sub[q[h]])
        if (comp[u] < 0) {
          comp[u] = ncomp;
          q.push_back(u);
        }
    ++ncomp;
  }
  if (ncomp > 1) {
    std::vector<std::vector<int>> parts(static_cast<size_t>(ncomp));
    for (int i = 0; i < n; ++i) parts[comp[i]].push_back(vs[i]);
    for (const auto& p : parts) nd_order(adj, p, loc, out);
    return;
  }
  if (n <= kNdLeafCams) {
    for (int k : minimum_degree_order(n, sub)) out->push_back(vs[k]);
    return;
  }
  NdGraph g;
  g.ptr.assign(1, 0);
  g.vw.assign(static_cast<size_t>(n), 1);
  for (int i = 0; i < n; ++i) {
    g.adj.insert(g.adj.end(), sub[i].begin(), sub[i].end());
    g.ptr.push_back(static_cast<int>(g.adj.size()));
  }
  g.ew.assign(g.adj.size(), 1);
  std::vector<std::vector<int>>().swap(sub);
  const std::vector<char> lab = nd_separator(g, nd_bisect(g));
  std::vector<int> part[3];
  for (int i = 0; i < n; ++i) part[lab[i]].push_back(vs[i]);
  nd_order(adj, part[0], loc, out);
  nd_order(adj, part[1], loc, out);
  out->insert(out->end(), part[2].begin(), part[2].end());
}

struct SparsePlan {
  int C = 0, ns = 0;
  int64_t stats[B200_SPARSE_STATS] = {};
  std::vector<int> perm, pinv;              // position k holds camera perm[k]; pinv[camera] = position
  std::vector<int> order;                   // [ns] the supernodes in the order the factor kernel's tickets take them
  std::vector<int> sn_first;                // [ns + 1] first column (position) of each supernode
  std::vector<int> row_ptr, rows;           // [ns + 1] / positions: the supernode's columns, then its rows below, ascending
  std::vector<long long> val;               // [ns] offset of each panel in the factor storage (doubles)
  long long storage = 0;                    // doubles of factor storage
  std::vector<int> upd_ptr;                 // [ns + 1]
  std::vector<int4> upd;                    // {d, k0, k1, 0}: rows k0..k1-1 of descendant d lie in this supernode's columns
  std::vector<int> ntf_ptr, ntf;            // [ns + 1] / the supernodes each supernode updates, ascending
  std::vector<int> cnt;                     // [2 ns] initial dependency counters of the forward and backward tasks
  std::vector<int> cnt_inv;                 // [ns] ... of the selected-inversion tasks (covariance.cuh): the supernodes
                                            // each supernode updates, 0 for a root
  double selinv_flops = 0.0;                // flops of the selected inversion (covariance.cuh) on this factor
  std::vector<long long> blk_off;           // per S block: offset of its 9x9 block in the factor storage
  std::vector<int> blk_ld;                  // ... and the panel's leading dimension, negated when the block goes in transposed
  int max_width = 0;                        // widest supernode (scalar columns)
};

// The plan of S's block pattern (upper triangle, blocks (i, j >= i), every diagonal block present) for C cameras, in the
// order of `ordering_type` (B200_AMD or B200_NESDIS).
inline void plan_sparse_schur(int C, const std::vector<int>& blk_row, const std::vector<int>& blk_col, int ordering_type,
                              SparsePlan* out) {
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
  const bool nesdis = ordering_type == B200_NESDIS;
  std::vector<int> md_perm;
  if (!nesdis && C <= kMinDegreeMaxCams) {
    md_perm = minimum_degree_order(C, adj);
    std::vector<int> md_pinv(static_cast<size_t>(C));
    for (int k = 0; k < C; ++k) md_pinv[md_perm[k]] = k;
    eliminate(C, adj, md_pinv, false, &md);
  } else {
    md = caller;   // not tried: reported with the caller's counts
  }
  const bool use_md = !nesdis && C <= kMinDegreeMaxCams && md.flops < caller.flops;
  if (nesdis) {
    std::vector<int> loc(static_cast<size_t>(C), -1);
    sp.perm.clear();
    sp.perm.reserve(static_cast<size_t>(C));
    nd_order(adj, ident, &loc, &sp.perm);
  } else {
    sp.perm = use_md ? md_perm : ident;
  }
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
  // the selected inversion has no forward tasks: a root starts at once
  sp.cnt_inv.assign(static_cast<size_t>(ns), 0);
  for (int s = 0; s < ns; ++s) sp.cnt_inv[s] = sp.ntf_ptr[s + 1] - sp.ntf_ptr[s];
  // its flops per supernode of W columns and n rows below: L_ss^-1 and L_ss^-T L_ss^-1 (W^3 / 3 each), U = L_Rs L_ss^-1
  // (n W^2), Z_Rs = -Z_RR U (2 n^2 W) and U' Z_Rs (2 n W^2)
  sp.selinv_flops = 0.0;
  for (int s = 0; s < ns; ++s) {
    const double W = 9.0 * (sp.sn_first[s + 1] - sp.sn_first[s]), n = 9.0 * (sp.row_ptr[s + 1] - sp.row_ptr[s]) - W;
    sp.selinv_flops += 2.0 * W * W * W / 3.0 + n * W * W + 2.0 * n * n * W + 2.0 * n * W * W;
  }
  // the supernodal tree (the parent of s owns the elimination-tree parent of s's last column; every descendant has a smaller
  // index), its critical paths from a leaf to a root, in supernodes and in the flops of the columns (those of the `flops`
  // statistic), and the task order: the identity with B200_AMD; with B200_NESDIS by ascending height above the leaves, then
  // index, so that the independent subtrees of the dissection are taken before the separators that wait on them.  Either is
  // topological: every descendant comes before its ancestors (sparse_schur.cuh relies on it).
  std::vector<int> up_n(static_cast<size_t>(ns), 0), kid_n(static_cast<size_t>(ns), 0);
  std::vector<double> up_f(static_cast<size_t>(ns), 0.0), kid_f(static_cast<size_t>(ns), 0.0);
  int path_n = 0;
  double path_f = 0.0;
  for (int s = 0; s < ns; ++s) {
    double f = 0.0;
    for (int c = sp.sn_first[s]; c < sp.sn_first[s + 1]; ++c) f += column_flops(static_cast<double>(e.below[c].size()));
    up_n[s] = kid_n[s] + 1;
    up_f[s] = kid_f[s] + f;
    path_n = std::max(path_n, up_n[s]);
    path_f = std::max(path_f, up_f[s]);
    const int pc = e.parent[sp.sn_first[s + 1] - 1];
    if (pc >= 0) {
      kid_n[sn_of[pc]] = std::max(kid_n[sn_of[pc]], up_n[s]);
      kid_f[sn_of[pc]] = std::max(kid_f[sn_of[pc]], up_f[s]);
    }
  }
  sp.order.resize(static_cast<size_t>(ns));
  for (int s = 0; s < ns; ++s) sp.order[s] = s;
  if (nesdis)
    std::stable_sort(sp.order.begin(), sp.order.end(), [&](int a, int b) { return up_n[a] < up_n[b]; });
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
  st[B200_SPARSE_STAT_ORDER] = nesdis ? 2 : use_md ? 1 : 0;
  st[B200_SPARSE_STAT_FACTOR_BYTES] = 8 * sp.storage;
  st[B200_SPARSE_STAT_FLOPS] = static_cast<int64_t>(e.flops);
  st[B200_SPARSE_STAT_CRITICAL_PATH_SUPERNODES] = path_n;
  st[B200_SPARSE_STAT_CRITICAL_PATH_FLOPS] = static_cast<int64_t>(path_f);
}

}  // namespace b200
