"""CPU-only checks of the product's host side: the C-ABI library loads and exports every declared symbol, fails
loudly without a GPU (no CPU fallback), and the host-side problem preparation (BAL reader, Normalize, reduced
program order, synthetic regeneration) agrees with the oracle's restatement of the reference."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def cs():
    import __graft_entry__ as g
    g.build()
    import ceres_solver_b200 as m
    return m


def test_library_exports_every_declared_symbol(cs):
    header = open(os.path.join(ROOT, "include", "b200ba.h")).read()
    declared = set(re.findall(r"\b(b200_[a-z0-9_]+)\s*\(", header))
    declared -= {"b200_handle"}
    assert declared, "no declarations parsed"
    lib = cs.lib()
    for name in sorted(declared):
        assert hasattr(lib, name), "libb200ba.so does not export %s" % name
    assert declared == set(cs.SYMBOLS), (declared ^ set(cs.SYMBOLS))


def test_struct_layouts_match_header(cs):
    from ceres_solver_b200 import binding as b
    o = b.SolverOptions()
    cs.lib().b200_solver_options_default(ctypes.byref(o))
    assert (o.preconditioner_type, o.max_num_iterations, o.residual_reset_period) == (2, 500, 10)
    lm = b.LmOptions()
    cs.lib().b200_lm_options_default(ctypes.byref(lm))
    assert lm.max_num_iterations == 5 and lm.eta == 1e-2 and lm.initial_trust_region_radius == 1e4
    assert lm.min_lm_diagonal == 1e-6 and lm.max_lm_diagonal == 1e32 and lm.linear_solver.max_num_iterations == 500


def test_struct_sizes_match_a_c_compiler(cs, tmp_path):
    """sizeof of every ABI struct as gcc sees include/b200ba.h against the ctypes mirrors in binding.py, plus the new
    option fields' defaults (a silent layout mismatch would corrupt options, not crash)."""
    import subprocess
    from ceres_solver_b200 import binding as b
    src = tmp_path / "sizes.c"
    src.write_text('#include <stdio.h>\n#include "b200ba.h"\nint main(void){printf("%zu %zu %zu %zu %zu %zu\\n", '
                   'sizeof(b200_ba_desc), sizeof(b200_solver_options), sizeof(b200_solver_summary), sizeof(b200_lm_options), '
                   'sizeof(b200_lm_iteration), sizeof(b200_kernel_stat)); return 0;}\n')
    exe = tmp_path / "sizes"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    sizes = [int(t) for t in subprocess.check_output([str(exe)]).split()]
    mirrors = [b.BaDesc, b.SolverOptions, b.SolverSummary, b.LmOptions, b.LmIteration, b.KernelStat]
    assert sizes == [ctypes.sizeof(m) for m in mirrors]
    o = b.SolverOptions()
    cs.lib().b200_solver_options_default(ctypes.byref(o))
    assert (o.max_num_spse_iterations, o.use_spse_initialization, o.spse_tolerance) == (5, 0, 0.1)
    lm = b.LmOptions()
    cs.lib().b200_lm_options_default(ctypes.byref(lm))
    assert lm.linear_solver_type == cs.ITERATIVE_SCHUR and lm.linear_solver.spse_tolerance == 0.1


def test_no_gpu_means_loud_failure_not_fallback(cs):
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible here")
    with pytest.raises(cs.B200Error) as e:
        cs.Problem(2, 3, [0, 1, 0], [0, 1, 2], np.zeros(6))
    assert e.value.code == -4  # B200_ERR_NO_DEVICE
    assert "no CPU fallback" in str(e.value)


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "ceres_solver_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cc")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"import\s+oracle|from\s+oracle|oracle/|libceres_oracle|pyoracle", text), \
                    "%s reaches into the oracle" % os.path.join(dirpath, f)


def test_bal_reader_and_normalize(oracle, c16_raw, c16):
    from ceres_solver_b200 import bal as B
    b = B.read_bal(os.path.join(ROOT, "tests", "golden", "problem-16-22106-pre.txt.bz2"))
    assert (b.C, b.P, b.N) == (16, 22106, 83718)
    assert np.array_equal(b.cam_idx, c16_raw.cam_idx) and np.array_equal(b.pt_idx, c16_raw.pt_idx)
    assert np.array_equal(b.obs.ravel(), c16_raw.obs)
    assert np.array_equal(b.cameras.ravel(), c16_raw.cameras) and np.array_equal(b.points.ravel(), c16_raw.points)
    n = B.normalize(b)
    assert np.allclose(n.points.ravel(), c16.points, rtol=1e-14, atol=1e-12)
    assert np.allclose(n.cameras.ravel(), c16.cameras, rtol=1e-13, atol=1e-12)


def test_reduced_program_order(oracle, c16):
    from ceres_solver_b200 import bal as B
    b = B.Bal(c16.cam_idx, c16.pt_idx, c16.obs, c16.cameras, c16.points)
    rp = B.ReducedProgram(b)
    op = oracle.BaProgram(c16.C, c16.P, c16.cam_idx, c16.pt_idx, c16.obs)
    for k in ("point_of_eblock", "camera_of_fblock", "obs_of_row", "row_pt", "row_cam"):
        assert np.array_equal(getattr(rp, k), getattr(op, k)), k
    assert np.array_equal(rp.row_obs.ravel(), op.row_obs)
    assert np.array_equal(rp.state(b), op.state_from_parameters(c16.cameras, c16.points))
    # unordered input (shuffled observations): still the reference's rule
    rng = np.random.RandomState(0)
    perm = rng.permutation(b.N)[:5000]
    sb = B.Bal(b.cam_idx[perm], b.pt_idx[perm], b.obs[perm], b.cameras, b.points)
    rp = B.ReducedProgram(sb)
    op = oracle.BaProgram(sb.C, sb.P, sb.cam_idx, sb.pt_idx, sb.obs.ravel())
    for k in ("point_of_eblock", "camera_of_fblock", "obs_of_row", "row_pt", "row_cam"):
        assert np.array_equal(getattr(rp, k), getattr(op, k)), k


def test_synthetic_is_seeded_and_well_formed():
    from ceres_solver_b200 import bal as B
    a = B.synthetic("tiny")
    b = B.synthetic("tiny")
    assert np.array_equal(a.obs, b.obs) and np.array_equal(a.cam_idx, b.cam_idx)
    C, P, N = B.SHAPES["tiny"]
    assert (a.C, a.P, a.N) == (C, P, N)
    deg = np.bincount(a.pt_idx, minlength=P)
    assert deg.min() >= 2
    key = a.pt_idx.astype(np.int64) * C + a.cam_idx
    assert np.unique(key).size == N  # a camera sees a point at most once
    assert np.all(np.diff(a.pt_idx) >= 0)
    # every point is in front of its cameras (Snavely convention: p_z < 0)
    cam = a.cameras[a.cam_idx]
    p = B.angle_axis_rotate(cam[:, 0:3], a.points[a.pt_idx]) + cam[:, 3:6]
    assert np.all(p[:, 2] < 0)
    proj = B.snavely_project(a.cameras, a.points, a.cam_idx, a.pt_idx)
    assert np.abs(proj - a.obs).max() < 200.0


def test_shard_partition_covers_all_rows():
    from ceres_solver_b200 import bal as B
    rp = B.ReducedProgram(B.synthetic("tiny"))
    for world in (1, 2, 3, 8):
        rows = 0
        prev_hi = 0
        for r in range(world):
            lo, hi, rlo, rhi = rp.shard(r, world)
            assert lo == prev_hi
            prev_hi = hi
            assert np.all(rp.row_pt[rlo:rhi] >= lo) and np.all(rp.row_pt[rlo:rhi] < hi)
            rows += rhi - rlo
        assert prev_hi == rp.P and rows == rp.N


def _random_bal(rng, C, P, max_deg):
    from ceres_solver_b200 import bal as B
    cam, pt = [], []
    for k in range(P):
        d = rng.randint(1, min(max_deg, C) + 1)
        cs_k = rng.choice(C, size=d, replace=False)
        cam.extend(cs_k.tolist())
        pt.extend([k] * d)
    order = rng.permutation(len(cam))               # BAL files are not required to be grouped by point
    cam = np.asarray(cam, dtype=np.int32)[order]
    pt = np.asarray(pt, dtype=np.int32)[order]
    obs = rng.normal(0.0, 100.0, (cam.size, 2))
    cameras = rng.normal(0.0, 1.0, (C, 9))
    points = rng.normal(0.0, 1.0, (P, 3))
    return B.Bal(cam, pt, obs, cameras, points)


@pytest.mark.parametrize("seed", range(8))
def test_reduced_program_invariants_on_random_structures(seed, tmp_path):
    """Whatever the observation order of the input: rows grouped by point (the SchurEliminator precondition), points in
    first-use order, a bijection between input observations and rows, BAL write/read round trip, and a shard partition
    that is contiguous, complete and balanced to within one point's worth of rows."""
    from ceres_solver_b200 import bal as B
    rng = np.random.RandomState(100 + seed)
    bal = _random_bal(rng, C=int(rng.randint(2, 12)), P=int(rng.randint(1, 60)), max_deg=int(rng.randint(1, 9)))
    path = str(tmp_path / "p.txt")
    B.write_bal(bal, path)
    back = B.read_bal(path)
    assert np.array_equal(back.cam_idx, bal.cam_idx) and np.array_equal(back.pt_idx, bal.pt_idx)
    assert np.allclose(back.obs, bal.obs, rtol=1e-15, atol=0) and np.allclose(back.cameras, bal.cameras, rtol=1e-15, atol=0)
    rp = B.ReducedProgram(bal)
    # parameter blocks nobody observes are not part of the reduced program (Program::RemoveFixedBlocks drops them)
    assert rp.N == bal.N and rp.P == np.unique(bal.pt_idx).size and rp.C == np.unique(bal.cam_idx).size
    assert np.all(np.diff(rp.row_pt) >= 0)                       # grouped by (reduced) point
    deg = np.bincount(rp.row_pt, minlength=rp.P)
    assert deg.min() >= 1 and deg.sum() == rp.N
    # every row is one input observation: same (original camera, original point, observation)
    o = rp.obs_of_row
    assert np.array_equal(np.sort(o), np.arange(bal.N))
    assert np.array_equal(rp.camera_of_fblock[rp.row_cam], bal.cam_idx[o])
    assert np.array_equal(rp.point_of_eblock[rp.row_pt], bal.pt_idx[o])
    assert np.array_equal(rp.row_obs, bal.obs[o])
    # parameter blocks in first-use order, rows of a point in reverse input order (SURVEY Appendix A)
    first_pt = [int(np.flatnonzero(bal.pt_idx == p)[0]) for p in rp.point_of_eblock]
    assert first_pt == sorted(first_pt)
    first_cam = [int(np.flatnonzero(bal.cam_idx == c)[0]) for c in rp.camera_of_fblock]
    assert first_cam == sorted(first_cam)
    for k in range(rp.P):
        rows = o[rp.row_pt == k]
        assert np.all(np.diff(rows) < 0) or rows.size == 1
    st = rp.state(bal)
    assert st.size == 3 * rp.P + 9 * rp.C
    for world in (1, 2, 3, 5):
        covered_pts, covered_rows, sizes = 0, 0, []
        for r in range(world):
            lo, hi, rlo, rhi = rp.shard(r, world)
            assert lo == covered_pts and rlo == covered_rows
            covered_pts, covered_rows = hi, rhi
            sizes.append(rhi - rlo)
        assert covered_pts == rp.P and covered_rows == rp.N
        assert max(sizes) - min(sizes) <= 2 * deg.max() + rp.N // world


def test_internal_point_order_plan():
    """b200_plan_point_order (host-only part of b200_create): the chosen order is a permutation, its score is what numpy
    computes for it, a capture whose points already follow the frames keeps the caller's order, the SURVEY 8d I2 recipe
    (points in random order) is re-ordered to a several times better score."""
    import ceres_solver_b200 as cs
    from ceres_solver_b200 import bal as B

    def score(cam, pt, P, C, order, chunks):
        newid = np.empty(P, dtype=np.int64)
        newid[order] = np.arange(P)
        rows = np.argsort(newid[pt], kind="stable")
        deg = np.bincount(pt, minlength=P)
        # chunk of a row = chunk of the point it belongs to: a point moves to the next chunk once the rows before it reach
        # chunk * (N / chunks + 1)  (same rule as the library)
        N = len(cam)
        target = N // chunks + 1
        ends = np.cumsum(deg[order])                  # rows up to and including each point, in the new order
        starts = ends - deg[order]
        chunk_of_point = starts // target
        chunk_of_row = np.repeat(chunk_of_point, deg[order])
        return int(np.unique(chunk_of_row * C + cam[rows]).size)

    for bal, expect_identity in ((B.synthetic_sequence(300, 9000, 40000, seed=3), True), (B.synthetic("tiny"), None)):
        rp = B.ReducedProgram(bal)
        perm, metrics, choice = cs.plan_point_order(rp.C, rp.P, rp.row_cam, rp.row_pt, 132)
        assert sorted(perm.tolist()) == list(range(rp.P))
        if expect_identity:
            assert choice == 0 and np.array_equal(perm, np.arange(rp.P))
        assert metrics[0] == score(rp.row_cam.astype(np.int64), rp.row_pt.astype(np.int64), rp.P, rp.C, np.arange(rp.P), 132)
    bal = B.synthetic_bal(400, 12000, 52000, seed=11)   # points in random order
    rp = B.ReducedProgram(bal)
    perm, metrics, choice = cs.plan_point_order(rp.C, rp.P, rp.row_cam, rp.row_pt, 132)
    assert choice != 0 and sorted(perm.tolist()) == list(range(rp.P))
    assert metrics[choice] * 2 < metrics[0]
    assert metrics[choice] == score(rp.row_cam.astype(np.int64), rp.row_pt.astype(np.int64), rp.P, rp.C, perm.astype(np.int64), 132)
    assert metrics[choice] == min(metrics[1:])
