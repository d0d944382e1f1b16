"""b200_plan_sparse_schur (the host-only symbolic analysis of SPARSE_SCHUR) against an independent block-level elimination of
the permuted camera graph in numpy.  No GPU needed."""
import numpy as np
import pytest


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


def column_flops(k):
    """Flops of one block column with k blocks below the diagonal (the count the library reports)."""
    return 243 + 729 * k + 729 * k * (k + 1)


def camera_edges(C, cam_idx, pt_idx):
    """Camera pairs i < j that share a point: the off-diagonal blocks of the upper triangle of S."""
    edges = set()
    cam_idx = np.asarray(cam_idx)
    pt_idx = np.asarray(pt_idx)
    starts = np.flatnonzero(np.r_[True, pt_idx[1:] != pt_idx[:-1]])
    ends = np.r_[starts[1:], len(pt_idx)]
    for a, b in zip(starts, ends):
        cams = np.unique(cam_idx[a:b])
        for x in range(len(cams)):
            for y in range(x + 1, len(cams)):
                edges.add((int(cams[x]), int(cams[y])))
    return edges


def eliminate(C, edges, perm, structure=False):
    """Block-level symbolic Cholesky in the order perm (perm[k] = camera eliminated k-th): (blocks of L, flops, tree height),
    and with `structure` also the elimination tree (parent by position) and the positions below the diagonal of each
    column."""
    pinv = np.empty(C, dtype=int)
    pinv[perm] = np.arange(C)
    A = np.zeros((C, C), dtype=bool)
    for i, j in edges:
        A[pinv[i], pinv[j]] = A[pinv[j], pinv[i]] = True
    blocks, flops, parent, below = C, 0, np.full(C, -1), []
    for k in range(C):
        nz = np.flatnonzero(A[k, k + 1:]) + k + 1
        below.append(nz)
        blocks += len(nz)
        flops += column_flops(len(nz))
        A[np.ix_(nz, nz)] = True
        if len(nz):
            parent[k] = nz[0]
    depth = np.ones(C, dtype=int)
    for k in range(C - 1, -1, -1):
        if parent[k] >= 0:
            depth[k] = depth[parent[k]] + 1
    if structure:
        return blocks, flops, int(depth.max()), parent, below
    return blocks, flops, int(depth.max())


SN_MAX_CAMS = 16   # widest supernode, in cameras
SN_RELAX = 0.25    # share of a supernode's stored blocks that merges may spend on explicit zero blocks


class Layout:
    """The supernodal layout of the factor, recounted from the elimination tree: relaxed amalgamation (merge column j into
    the supernode of j - 1 while parent[j - 1] == j, the supernode has at most SN_MAX_CAMS cameras and its explicit zero
    blocks stay within SN_RELAX of its stored blocks), each supernode's rows (its own columns, then the rows below its last
    column) and each supernode's update list: (descendant d, k0, k1) for every run of d's rows below its own columns that
    lies in the supernode's columns."""

    def __init__(self, parent, below):
        C = len(parent)
        first, true_blocks = [0], 1 + len(below[0])
        for j in range(1, C):
            f = first[-1]
            merge = parent[j - 1] == j and j - f < SN_MAX_CAMS
            if merge:
                w = j - f + 1
                tb = true_blocks + 1 + len(below[j])
                stored = w * (w + 1) // 2 + w * len(below[j])
                merge = stored - tb <= SN_RELAX * stored
                if merge:
                    true_blocks = tb
            if not merge:
                first.append(j)
                true_blocks = 1 + len(below[j])
        first.append(C)
        self.first = np.array(first)
        self.ns = ns = len(first) - 1
        self.width = np.diff(self.first)
        sn_of = np.repeat(np.arange(ns), self.width)
        self.rows = [np.r_[np.arange(self.first[s], self.first[s + 1]), below[self.first[s + 1] - 1]].astype(int)
                     for s in range(ns)]
        self.R = np.array([len(r) for r in self.rows])
        self.updates = [[] for _ in range(ns)]
        for d in range(ns):
            k = self.width[d]
            while k < self.R[d]:
                s = sn_of[self.rows[d][k]]
                k1 = k
                while k1 < self.R[d] and sn_of[self.rows[d][k1]] == s:
                    k1 += 1
                self.updates[s].append((d, k, k1))
                k = k1
        self.factor_bytes = 8 * sum((81 * int(R) * int(w) + 15) // 16 * 16 for R, w in zip(self.R, self.width))
        self.roots = int(sum(1 for s in range(ns) if self.R[s] == self.width[s]))

    def all_updates(self):
        """(s, d, k0, k1, ncb, Wd, Rd) of every update."""
        return [(s, d, k0, k1, k1 - k0, 9 * self.width[d], self.R[d]) for s in range(self.ns) for d, k0, k1 in self.updates[s]]


def check_plan(cs, C, P, cam_idx, pt_idx):
    perm, st = cs.plan_sparse_schur(C, P, cam_idx, pt_idx)
    assert sorted(perm.tolist()) == list(range(C))
    edges = camera_edges(C, cam_idx, pt_idx)
    assert st["s_blocks"] == C + len(edges)
    blocks, flops, height, parent, below = eliminate(C, edges, perm, structure=True)
    blocks_c, flops_c, _ = eliminate(C, edges, np.arange(C))
    assert st["l_blocks"] == blocks
    assert st["l_blocks_caller"] == blocks_c
    assert st["flops_caller"] == flops_c
    assert st["tree_height"] == height
    assert flops <= flops_c
    assert st["order"] in (0, 1)
    if st["order"] == 0:
        assert np.array_equal(perm, np.arange(C))
    else:
        assert st["flops_min_degree"] == flops < flops_c
        assert st["l_blocks_min_degree"] == blocks
    lay = Layout(parent, below)
    assert st["supernodes"] == lay.ns
    assert st["factor_bytes"] == lay.factor_bytes >= 648 * blocks
    return perm, st, lay


def random_structure(rng, C, components=1, empty_camera=False):
    """Points that see 2..5 distinct cameras of one component (cameras split into contiguous groups)."""
    usable = C - 1 if empty_camera else C
    bounds = np.linspace(0, usable, components + 1).astype(int)
    cam_idx, pt_idx = [], []
    P = int(rng.randint(2 * C, 6 * C))
    for p in range(P):
        g = rng.randint(components)
        lo, hi = bounds[g], bounds[g + 1]
        deg = min(hi - lo, int(rng.randint(2, 6)))
        cams = rng.choice(np.arange(lo, hi), size=deg, replace=False)
        cam_idx += [int(c) for c in cams]
        pt_idx += [p] * deg
    return P, np.array(cam_idx, dtype=np.int32), np.array(pt_idx, dtype=np.int32)


@pytest.mark.parametrize("seed", range(8))
def test_random_camera_graphs(cs, seed):
    rng = np.random.RandomState(1000 + seed)
    C = int(rng.randint(5, 81))
    P, cam, pt = random_structure(rng, C, components=1 + seed % 3, empty_camera=seed % 2 == 1)
    check_plan(cs, C, P, cam, pt)


def test_edge_graphs(cs):
    # C = 5 with a camera that sees nothing; an arrow (camera 0 shares a point with every other camera: the caller's order
    # fills everything, minimum degree leaves it last)
    check_plan(cs, 5, 3, np.array([0, 1, 1, 2, 2, 3], np.int32), np.array([0, 0, 1, 1, 2, 2], np.int32))
    C = 40
    cam = np.array([c for k in range(1, C) for c in (0, k)], np.int32)
    pt = np.repeat(np.arange(C - 1), 2).astype(np.int32)
    perm, st, _ = check_plan(cs, C, C - 1, cam, pt)
    assert st["order"] == 1 and list(perm).index(0) >= C - 2 and st["l_blocks"] == st["s_blocks"]


@pytest.mark.parametrize("name", ["tiny", "trafalgar-257", "sequence"])
def test_synthetic_shapes(cs, name):
    from ceres_solver_b200 import bal as B
    b = B.synthetic_sequence(240, 20000, 90000) if name == "sequence" else B.synthetic(name)
    rp = B.ReducedProgram(b)
    perm, st, _ = check_plan(cs, rp.C, rp.P, rp.row_cam, rp.row_pt)
    if name == "sequence":
        # a video sequence is a band in the caller's order: kept, no fill
        assert st["order"] == 0 and st["l_blocks"] == st["s_blocks"]
        assert st["supernodes"] < rp.C // 4


# ---- camera graphs built to reach each path of the device factorisation (csrc/sparse_schur.cuh); tests/test_gpu_sparse_factor.py
# solves on them.  Every camera also gets SOLO_POINTS points that it alone sees twice (duplicate rows): they add to the
# diagonal blocks of S only, leave the camera graph as built, and make S positive definite for any generic Jacobian values.
SOLO_POINTS = 10


def _rows(C, tracks, rng, solo=SOLO_POINTS):
    """(C, P, cam_idx, pt_idx) of points with the given camera tracks, rows grouped by point, plus the solo points."""
    tracks = [list(t) for t in tracks] + [[c, c] for c in range(C) for _ in range(solo)]
    order = rng.permutation(len(tracks))   # points in no particular order
    tracks = [tracks[i] for i in order]
    cam = np.concatenate([np.asarray(t) for t in tracks]).astype(np.int32)
    pt = np.repeat(np.arange(len(tracks)), [len(t) for t in tracks]).astype(np.int32)
    return C, len(tracks), cam, pt


def _clique(cams, rng, extra=None):
    """Tracks under which every pair of `cams` shares a point, plus `extra` points seeing 3..5 of them."""
    cams = list(cams)
    t = [[a, b] for i, a in enumerate(cams) for b in cams[i + 1:]]
    for _ in range(len(cams) if extra is None else extra):
        t.append(list(rng.choice(cams, size=min(len(cams), int(rng.randint(3, 6))), replace=False)))
    return t


def _band(C, rng, points, lo=20, hi=40):
    """Video tracks: each point seen by lo..hi consecutive frames."""
    t = []
    for _ in range(points):
        n = int(rng.randint(lo, hi + 1))
        s = int(rng.randint(0, C - n + 1))
        t.append(list(range(s, s + n)))
    t += [[c, c + 1] for c in range(C - 1)]   # consecutive frames always share a point
    return t


def _binary_tree(first, n):
    """Tracks whose camera graph is a complete binary tree of n cameras numbered first.. in post-order (children first)."""
    edges = []

    def post(size):   # numbers a subtree of `size` nodes in post-order, returns its root
        if size == 0:
            return None
        left = post((size - 1) // 2)
        right = post(size - 1 - (size - 1) // 2)
        post.next += 1
        root = post.next - 1
        edges.extend([(c, root) for c in (left, right) if c is not None])
        return root
    post.next = first
    post(n)
    return [[a, b] for a, b in edges for _ in range(2)]


def structure(name, seed=7):
    """(C, P, cam_idx, pt_idx) of one camera graph of STRUCTURES, camera ids in the caller's order."""
    rng = np.random.RandomState(seed)
    if name == "one":
        return _rows(1, [[0, 0]] * 30, rng)
    if name == "two":
        return _rows(2, [[0, 1]] * 30, rng)
    if name == "clique16":
        return _rows(16, _clique(range(16), rng), rng)
    if name == "cliques":
        t, f = [], 0
        for n in (17, 31, 33, 40):
            t += _clique(range(f, f + n), rng)
            f += n
        # a 31-clique whose last 15 cameras also see camera f + 32 (camera f + 31 sees none): the supernode of those 15
        # (135 columns) updates that camera's
        t += _clique(range(f, f + 31), rng) + [[f + 32, c] for c in range(f + 16, f + 31)]
        return _rows(f + 33, t, rng)
    if name == "hub":   # camera 0 sees every other camera; the others in pairs
        C = 121
        t = [[0, c] for c in range(1, C)]
        t += [[a, a + 1] for a in range(1, C, 2) for _ in range(3)]
        return _rows(C, t, rng)
    if name == "band":
        return _rows(160, _band(160, rng, 600), rng)
    if name == "loop":   # the band, and tracks that run from its last frames into its first ones
        C = 160
        t = _band(C, rng, 600)
        t += [[C - 1 - k, k % 8] for k in range(64)]
        return _rows(C, t, rng)
    if name == "forest":   # 400 small components, and a binary-tree camera graph
        t, f = [], 0
        for _ in range(400):
            n = int(rng.randint(2, 6))
            t += _clique(range(f, f + n), rng, extra=1)
            f += n
        t += _binary_tree(f, 127)
        return _rows(f + 127, t, rng)
    if name == "random400":   # synthetic_bal's camera graph with tracks of up to 100 cameras (Ladybug-1723-random, scaled)
        from ceres_solver_b200 import bal as B
        b = B.synthetic_bal(400, 3000, 30000, seed=seed, max_degree=100)
        return 400, b.P, b.cam_idx, b.pt_idx
    if name == "shuffled":   # the loop closures with the camera ids shuffled and two duplicate (camera, point) rows
        C, P, cam, pt = structure("loop", seed)
        cam = rng.permutation(C).astype(np.int32)[cam]
        for p in (5, 77):
            j = int(np.flatnonzero(pt == p)[0])
            cam = np.insert(cam, j, cam[j])
            pt = np.insert(pt, j, p)
        return C, P, cam, pt
    raise KeyError(name)


STRUCTURES = ("one", "two", "clique16", "cliques", "hub", "band", "loop", "forest", "random400", "shuffled")


def structure_properties(name, perm, lay):
    """Asserts the property each structure of STRUCTURES is built for, from the recounted layout."""
    ups = lay.all_updates()
    identity = np.array_equal(perm, np.arange(len(perm)))
    if name in ("one", "two", "clique16"):
        assert lay.ns == 1 and not ups and lay.width[0] == {"one": 1, "two": 2, "clique16": 16}[name]
    elif name == "cliques":
        assert identity and lay.width.max() == SN_MAX_CAMS
        kinds = {(ncb, Wd) for _, _, _, _, ncb, Wd, _ in ups}
        assert {(16, 144), (15, 144), (1, 135)} <= kinds, kinds   # warp g takes blocks g and g + 8; a stage tail of 7
        assert any(9 * (Rd - k0) % 64 for _, _, k0, _, _, _, Rd in ups)   # a row tile ends part-way
        assert any(k0 > lay.width[d] for _, d, k0, _, _, _, _ in ups)      # a descendant that updates two supernodes
    elif name == "hub":
        assert not identity and list(perm).index(0) >= len(perm) - 3       # minimum degree: the hub in the last supernode
        assert max(len(u) for u in lay.updates) >= 59
    elif name == "band":
        assert identity and all(len(u) >= 1 for u in lay.updates[1:])
        parents = {s: {t for t in range(lay.ns) for d, _, _ in lay.updates[t] if d == s} for s in range(lay.ns)}
        assert all(min(p) == s + 1 for s, p in parents.items() if p)       # a chain: each supernode's first ancestor is the next
        assert any(k0 > lay.width[d] for _, d, k0, _, _, _, _ in ups)
    elif name == "loop":
        assert lay.R.max() >= 64 and max(-(-9 * (Rd - k0) // 64) for _, _, k0, _, _, _, Rd in ups) >= 8
        assert max(lay.R[s] - lay.width[s] for s in range(lay.ns)) >= 48   # rows below searched by bisection
    elif name == "forest":
        assert lay.ns >= 264 and lay.roots >= 300                          # 2 ns >= 4 x 132 CTAs on an H100 SXM
    elif name == "random400":
        assert lay.R[lay.width == SN_MAX_CAMS].max() >= 200
    elif name == "shuffled":
        assert not identity and lay.ns > 1 and ups


@pytest.mark.parametrize("name", STRUCTURES)
def test_structures(cs, name):
    """The supernode partition and factor size of every camera graph the device factorisation is tested on, and the
    property each is built for."""
    C, P, cam, pt = structure(name)
    perm, _, lay = check_plan(cs, C, P, cam, pt)
    structure_properties(name, perm, lay)
