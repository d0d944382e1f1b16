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


def eliminate(C, edges, perm):
    """Block-level symbolic Cholesky in the order perm (perm[k] = camera eliminated k-th): (blocks of L, flops, tree height)."""
    pinv = np.empty(C, dtype=int)
    pinv[perm] = np.arange(C)
    A = np.zeros((C, C), dtype=bool)
    for i, j in edges:
        A[pinv[i], pinv[j]] = A[pinv[j], pinv[i]] = True
    blocks, flops, parent = C, 0, np.full(C, -1)
    for k in range(C):
        nz = np.flatnonzero(A[k, k + 1:]) + k + 1
        blocks += len(nz)
        flops += column_flops(len(nz))
        A[np.ix_(nz, nz)] = True
        if len(nz):
            parent[k] = nz[0]
    depth = np.ones(C, dtype=int)
    for k in range(C - 1, -1, -1):
        if parent[k] >= 0:
            depth[k] = depth[parent[k]] + 1
    return blocks, flops, int(depth.max())


def check_plan(cs, C, P, cam_idx, pt_idx):
    perm, st = cs.plan_sparse_schur(C, P, cam_idx, pt_idx)
    assert sorted(perm.tolist()) == list(range(C))
    edges = camera_edges(C, cam_idx, pt_idx)
    assert st["s_blocks"] == C + len(edges)
    blocks, flops, height = eliminate(C, edges, perm)
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
    assert 1 <= st["supernodes"] <= C
    assert st["factor_bytes"] >= 648 * blocks
    return perm, st


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
    perm, st = check_plan(cs, C, C - 1, cam, pt)
    assert st["order"] == 1 and list(perm).index(0) >= C - 2 and st["l_blocks"] == st["s_blocks"]


@pytest.mark.parametrize("name", ["tiny", "trafalgar-257", "sequence"])
def test_synthetic_shapes(cs, name):
    from ceres_solver_b200 import bal as B
    b = B.synthetic_sequence(240, 20000, 90000) if name == "sequence" else B.synthetic(name)
    rp = B.ReducedProgram(b)
    perm, st = check_plan(cs, rp.C, rp.P, rp.row_cam, rp.row_pt)
    if name == "sequence":
        # a video sequence is a band in the caller's order: kept, no fill
        assert st["order"] == 0 and st["l_blocks"] == st["s_blocks"]
        assert st["supernodes"] < rp.C // 4
