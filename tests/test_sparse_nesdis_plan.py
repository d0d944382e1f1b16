"""b200_plan_sparse_schur_ordered with B200_NESDIS (nested dissection of the camera graph, csrc/sparse_plan.cuh) against an
independent elimination, supernode layout and supernodal-tree recount in numpy.  No GPU needed.

What the order must be is not fixed here (any permutation is a valid fill-reducing order); what is checked is that every
statistic the library reports for the order it returns is what that order gives, that the tree is shallow where the order
matters, and that degenerate graphs, graphs above the minimum-degree cap and repeated calls behave."""
import ctypes
import time

import numpy as np
import pytest
import scipy.sparse as sps

from tests.test_sparse_schur_plan import (STRUCTURES, Layout, camera_edges, column_flops, eliminate, random_structure,
                                          structure)


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


def fast_edges(C, cam_idx, pt_idx):
    """camera_edges through a sparse product: the pairs i < j of cameras that share a point."""
    cam, pt = np.asarray(cam_idx), np.asarray(pt_idx)
    M = sps.csr_matrix((np.ones(len(cam)), (pt, cam)), shape=(int(pt.max()) + 1, C))
    G = (M.T @ M).tocoo()
    keep = G.row < G.col
    return set(zip(G.row[keep].tolist(), G.col[keep].tolist()))


def tree_paths(lay, parent, below):
    """(most supernodes, most flops) on one leaf-to-root path of the supernodal tree, and each supernode's height above the
    leaves (1 for a leaf): the parent of supernode s owns the elimination-tree parent of s's last column, and a supernode's
    flops are those of its columns."""
    ns, first = lay.ns, lay.first
    sn_of = np.repeat(np.arange(ns), lay.width)
    sn_parent = [int(sn_of[parent[first[s + 1] - 1]]) if parent[first[s + 1] - 1] >= 0 else -1 for s in range(ns)]
    flops = [sum(column_flops(len(below[c])) for c in range(first[s], first[s + 1])) for s in range(ns)]
    kids = [[] for _ in range(ns)]
    for s, p in enumerate(sn_parent):
        if p >= 0:
            assert p > s
            kids[p].append(s)
    up_n, up_f = [0] * ns, [0] * ns
    for s in range(ns):
        up_n[s] = 1 + max((up_n[k] for k in kids[s]), default=0)
        up_f[s] = flops[s] + max((up_f[k] for k in kids[s]), default=0)
    return max(up_n), max(up_f), up_n


def check_ordered(cs, C, P, cam, pt, ordering, edges=None):
    """The plan under `ordering`, every statistic of its order recounted; returns (perm, stats, layout, heights)."""
    perm, st = cs.plan_sparse_schur(C, P, cam, pt, ordering)
    assert sorted(perm.tolist()) == list(range(C))
    edges = camera_edges(C, cam, pt) if edges is None else edges
    assert st["s_blocks"] == C + len(edges)
    blocks, flops, height, parent, below = eliminate(C, edges, perm, structure=True)
    assert st["l_blocks"] == blocks
    assert st["flops"] == flops
    assert st["tree_height"] == height
    lay = Layout(parent, below)
    assert st["supernodes"] == lay.ns
    assert st["factor_bytes"] == lay.factor_bytes
    path_n, path_f, heights = tree_paths(lay, parent, below)
    assert st["critical_path_supernodes"] == path_n
    assert st["critical_path_flops"] == path_f
    assert st["order"] == 2 if ordering == cs.NESDIS else st["order"] in (0, 1)
    return perm, st, lay, heights


@pytest.mark.parametrize("name", STRUCTURES)
def test_structures(cs, name):
    C, P, cam, pt = structure(name)
    check_ordered(cs, C, P, cam, pt, cs.NESDIS)
    check_ordered(cs, C, P, cam, pt, cs.AMD)


@pytest.mark.parametrize("seed", range(8))
def test_random_camera_graphs(cs, seed):
    """Random graphs of 1..3 components, every other one with a camera that sees no other."""
    rng = np.random.RandomState(2000 + seed)
    C = int(rng.randint(5, 200))
    P, cam, pt = random_structure(rng, C, components=1 + seed % 3, empty_camera=seed % 2 == 1)
    check_ordered(cs, C, P, cam, pt, cs.NESDIS)


@pytest.mark.parametrize("name", ["ladybug-1723", "trafalgar-257", "venice-1778", "ladybug-1723-random"])
def test_synthetic_problems(cs, name, record_property):
    from ceres_solver_b200 import bal as B
    rp = B.ReducedProgram(B.synthetic(name))
    edges = fast_edges(rp.C, rp.row_cam, rp.row_pt)
    _, nd, _, _ = check_ordered(cs, rp.C, rp.P, rp.row_cam, rp.row_pt, cs.NESDIS, edges)
    _, amd, _, _ = check_ordered(cs, rp.C, rp.P, rp.row_cam, rp.row_pt, cs.AMD, edges)
    keys = ("flops", "l_blocks", "supernodes", "tree_height", "critical_path_supernodes", "critical_path_flops")
    record_property(name, "amd %s / nesdis %s" % ({k: amd[k] for k in keys}, {k: nd[k] for k in keys}))
    if name == "ladybug-1723":
        assert_shallower(nd, amd)


def assert_shallower(nd, amd):
    """The tree of a band graph under nested dissection: at most a quarter of AMD's height and at most half of AMD's
    critical-path flops (observed on ladybug-1723: height 121 against 1723, critical path 9.4e7 flops against 4.8e8 and 13
    supernodes against 148)."""
    assert 4 * nd["tree_height"] <= amd["tree_height"], (nd, amd)
    assert 2 * nd["critical_path_flops"] <= amd["critical_path_flops"], (nd, amd)
    assert nd["critical_path_supernodes"] < amd["critical_path_supernodes"], (nd, amd)


def test_band_tree_shape(cs, record_property):
    """The `band` structure is 160 frames with tracks of up to 40: only four bandwidths long, so every separator is a
    quarter of the graph.  Nested dissection shortens its elimination tree (113 against 160 columns) but not its critical
    path, which is 9 supernodes against AMD's 10 and 2.3 times AMD's flops (3.2e8 against 1.4e8): the columns of the
    second-level separators see the whole top separator below them.  Asserted: a tree at most 3/4 as high, no more
    supernodes on the critical path, and at most 3 times its flops."""
    C, P, cam, pt = structure("band")
    _, nd, _, _ = check_ordered(cs, C, P, cam, pt, cs.NESDIS)
    _, amd, _, _ = check_ordered(cs, C, P, cam, pt, cs.AMD)
    record_property("band", "amd height %d cp %d / %d flops; nesdis height %d cp %d / %d flops" % (
        amd["tree_height"], amd["critical_path_supernodes"], amd["critical_path_flops"], nd["tree_height"],
        nd["critical_path_supernodes"], nd["critical_path_flops"]))
    assert 4 * nd["tree_height"] <= 3 * amd["tree_height"]
    assert nd["critical_path_supernodes"] <= amd["critical_path_supernodes"]
    assert nd["critical_path_flops"] <= 3 * amd["critical_path_flops"]


def _tracks(C, tracks, solo=2):
    t = [list(x) for x in tracks] + [[c] for c in range(C) for _ in range(solo)]
    cam = np.concatenate([np.asarray(x) for x in t]).astype(np.int32)
    pt = np.repeat(np.arange(len(t)), [len(x) for x in t]).astype(np.int32)
    return C, len(t), cam, pt


@pytest.mark.parametrize("name", ["one", "two", "clique80", "hub200", "isolated100", "path3"])
def test_degenerate(cs, name):
    """One camera, two, a clique above the leaf size (no separator but a whole side), a hub above the leaf size, cameras
    that share nothing, a path of three."""
    if name == "one":
        args = _tracks(1, [])
    elif name == "two":
        args = _tracks(2, [[0, 1]])
    elif name == "clique80":
        args = _tracks(80, [[a, b] for a in range(80) for b in range(a + 1, 80)])
    elif name == "hub200":
        args = _tracks(200, [[0, c] for c in range(1, 200)] + [[c, c + 1] for c in range(1, 199, 2)])
    elif name == "isolated100":
        args = _tracks(100, [])
    else:
        args = _tracks(3, [[0, 1], [1, 2]])
    perm, st, lay, _ = check_ordered(cs, *args, cs.NESDIS)
    if name == "isolated100":
        assert st["l_blocks"] == 100 and st["critical_path_supernodes"] == 1


def test_deterministic(cs):
    for name in ("loop", "random400", "shuffled"):
        C, P, cam, pt = structure(name)
        a = cs.plan_sparse_schur(C, P, cam, pt, cs.NESDIS)
        b = cs.plan_sparse_schur(C, P, cam, pt, cs.NESDIS)
        assert np.array_equal(a[0], b[0]) and a[1] == b[1], name


def test_above_minimum_degree_cap(cs, record_property):
    """A band of 40000 cameras, above the 32768 the whole-graph minimum degree is tried to: nested dissection still orders
    it (minimum degree runs on its leaves only) and its tree is shallow."""
    C = 40000
    tracks = [[c, c + 1, c + 2] for c in range(C - 2)]
    C, P, cam, pt = _tracks(C, tracks, solo=1)
    t = time.perf_counter()
    perm, st = cs.plan_sparse_schur(C, P, cam, pt, cs.NESDIS)
    dt = time.perf_counter() - t
    _, amd = cs.plan_sparse_schur(C, P, cam, pt, cs.AMD)
    record_property("band40000", "nesdis analysis %.2f s, height %d (amd %d), critical path %d supernodes (amd %d)" % (
        dt, st["tree_height"], amd["tree_height"], st["critical_path_supernodes"], amd["critical_path_supernodes"]))
    assert sorted(perm.tolist()) == list(range(C))
    assert st["order"] == 2 and amd["order"] == 0
    assert st["s_blocks"] == amd["s_blocks"] == C + 2 * (C - 1) - 1
    assert 100 * st["tree_height"] <= amd["tree_height"]
    assert 10 * st["critical_path_supernodes"] <= amd["critical_path_supernodes"]


def _raw_plan(cs, fn, C, P, cam, pt, *extra):
    from ceres_solver_b200 import binding as Bd
    cam = np.ascontiguousarray(cam, dtype=np.int32)
    pt = np.ascontiguousarray(pt, dtype=np.int32)
    d = Bd.BaDesc()
    d.num_cameras, d.num_points, d.num_observations = C, P, len(cam)
    d.cam_idx = cam.ctypes.data_as(Bd._ip)
    d.pt_idx = pt.ctypes.data_as(Bd._ip)
    perm = np.full(C, -1, dtype=np.int32)
    stats = (ctypes.c_int64 * len(Bd.SPARSE_STATS))()
    rc = getattr(cs.lib(), fn)(ctypes.byref(d), *extra, perm.ctypes.data_as(Bd._ip), stats)
    return rc, perm, list(stats)


def test_amd_unchanged(cs):
    """b200_plan_sparse_schur is the AMD case of b200_plan_sparse_schur_ordered, statistics and order."""
    for name in STRUCTURES:
        C, P, cam, pt = structure(name)
        a = _raw_plan(cs, "b200_plan_sparse_schur", C, P, cam, pt)
        b = _raw_plan(cs, "b200_plan_sparse_schur_ordered", C, P, cam, pt, cs.AMD)
        assert a[0] == b[0] == 0 and np.array_equal(a[1], b[1]) and a[2] == b[2], name
        assert a[2][cs.SPARSE_STATS.index("order")] in (0, 1)


def test_invalid_ordering_type(cs):
    C, P, cam, pt = structure("two")
    for bad in (2, -1, 7):
        rc, _, _ = _raw_plan(cs, "b200_plan_sparse_schur_ordered", C, P, cam, pt, bad)
        assert rc == -1, bad   # B200_ERR_INVALID_ARGUMENT
    with pytest.raises(cs.B200Error):
        cs.plan_sparse_schur(C, P, cam, pt, 2)
