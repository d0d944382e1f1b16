"""b200_create picks its kernels from the problem's structure (the shared-memory arithmetic on the per-CTA camera span
in plan_kernels, csrc/plan.cuh), and each choice is a different kernel, or a different combination of kernels writing into the same
output.  One fixture per configuration, each checked through every entry point and three LM iterations against the
oracle (tests/entry_points.py), and each asserting the configuration it got from the `[b200ba] C=...` line
(B200_VERBOSE), so that a change of the planning heuristics fails here instead of quietly moving coverage.

  id_range       cameras drawn uniformly from 2000: id ranges, schur_mul_v3 + jtj_v2 + cam_reduce_kernel, CTA-tile
                 evaluate / init; one 33..128-row point (folded into the v3 product) and one >128-row point (huge
                 kernels next to the id-range ones)
  direct_v3      circle geometry with camera locality, except that the points in the middle of the order holding
                 ~2/132 of the rows see cameras from all 1800: camera lists of ~1200 cameras, too many for v4, so
                 schur_mul_v3 in direct mode, jtj_v2, CTA-tile evaluate / init, and the seeded PCG without the fused p.q
  v4_narrow      the same with the middle rows over a 900-camera window: camera lists of ~800 cameras, v4 with fewer
                 than 16 warps and one shared camera vector
  dups_direct    v4_narrow plus one duplicated (camera, point) row: no camera-major pass, and 45 doubles per camera
                 of ~800 do not fit for diag_blocks_v2_kernel, so the CTA-tile diag_blocks_kernel runs beside the
                 warp-tile kernels
  dups_id_range  id_range without its >128-row point, plus one duplicate: CTA-tile diag_blocks_kernel with id ranges
  tile           every point sees cameras drawn uniformly from 3000 (the scatter problem of tests/test_gpu_orders.py)
                 plus one >128-row point: no camera vector fits, CTA-tile kernels everywhere

The remaining configurations are covered by fixtures of other modules, whose plans test_configuration_table reads too:
C16 (v4 with one camera vector per warp), circle (v4 with shared vectors, 16 warps) and the ragged problem with a
duplicate (diag_blocks_v2_kernel).
"""
import numpy as np
import pytest

from tests.entry_points import Case, check_every_entry_point, check_lm_trajectory, oracle_lm_traces, parse_plan

pytestmark = pytest.mark.gpu

# Three LM iterations with the CG capped at 40 iterations: from the second iteration on the solves of these problems
# run 50..200 iterations to the eta stop, which sits on a plateau where the oracle's own count moves by up to 5 between
# runs (52 or 57 on `tile`).  Capped, every solve of GPU and oracle runs the same count, and cost and step norm are held
# to 1e-6 on every iteration.
LM_ITERATIONS, LM_MAX_CG = 3, 40


def _uniform_cameras(C, P, N, seed):
    """synthetic_bal geometry (every point is in front of every camera), each observation re-assigned to a camera drawn
    uniformly from all of them (distinct within a point)."""
    from ceres_solver_b200 import bal as B
    base = B.synthetic_bal(C, P, N, seed=seed)
    rng = np.random.RandomState(seed)
    deg = np.bincount(base.pt_idx, minlength=P)
    cam = np.concatenate([rng.choice(C, size=d, replace=False) for d in deg]).astype(np.int32)
    obs = B.snavely_project(base.cameras, base.points, cam, base.pt_idx) + rng.normal(0.0, 0.5, (N, 2))
    return B.Bal(cam, base.pt_idx, obs, base.cameras, base.points)


def _add_rows(bal, point, cams, seed):
    """bal with extra observations of `point` by `cams` (projection of the initial parameters + noise)."""
    from ceres_solver_b200 import bal as B
    rng = np.random.RandomState(seed)
    cams = np.asarray(cams, dtype=np.int32)
    pts = np.full(cams.size, point, dtype=np.int32)
    obs = B.snavely_project(bal.cameras, bal.points, cams, pts) + rng.normal(0.0, 0.5, (cams.size, 2))
    return B.Bal(np.concatenate([bal.cam_idx, cams]), np.concatenate([bal.pt_idx, pts]), np.concatenate([bal.obs, obs]),
                 bal.cameras, bal.points)


def _grow_point(bal, point, degree, seed):
    """Adds observations of `point` by cameras it is not seen by yet, up to `degree` rows."""
    rng = np.random.RandomState(seed)
    have = set(bal.cam_idx[bal.pt_idx == point].tolist())
    extra = [c for c in rng.permutation(bal.C) if c not in have][:degree - len(have)]
    return _add_rows(bal, point, sorted(extra), seed)


def _duplicate_row(bal, point):
    """A second observation of `point` by the first camera that sees it (a duplicate (camera, point) pair)."""
    j = np.flatnonzero(bal.pt_idx == point)[0]
    return _add_rows(bal, point, [bal.cam_idx[j]], 17)


def _local_with_wide_middle(share, window, seed=23):
    """synthetic_bal(1800, 60000, 260000) with the points relabelled in order of their smallest camera (camera
    locality in the caller's order); the points in the middle of that order that hold `share` of the rows see distinct
    cameras drawn uniformly from `window` cameras centred on camera 900 instead of their azimuth window.  Every point
    is in front of every camera of this geometry."""
    from ceres_solver_b200 import bal as B
    bal = B.synthetic_bal(1800, 60000, 260000, seed=seed)
    rng = np.random.RandomState(seed)
    C, P, N = bal.C, bal.P, bal.N
    kmin = np.full(P, C, dtype=np.int64)
    np.minimum.at(kmin, bal.pt_idx, bal.cam_idx)
    order = np.argsort(kmin, kind="stable")
    new_id = np.empty(P, dtype=np.int64)
    new_id[order] = np.arange(P)
    pt = new_id[bal.pt_idx]
    rows = np.argsort(pt, kind="stable")
    cam, pt, points = bal.cam_idx[rows], pt[rows].astype(np.int32), bal.points[order]
    deg = np.bincount(pt, minlength=P)
    ptr = np.concatenate([[0], np.cumsum(deg)])
    mid = np.flatnonzero((ptr[:-1] >= N * (0.5 - share / 2)) & (ptr[1:] <= N * (0.5 + share / 2)))
    lo = C // 2 - window // 2
    for k in mid:
        cam[ptr[k]:ptr[k + 1]] = lo + rng.choice(window, size=deg[k], replace=False)
    obs = B.snavely_project(bal.cameras, points, cam, pt) + rng.normal(0.0, 0.5, (N, 2))
    return B.Bal(cam, pt, obs, bal.cameras, points)


def _id_range(huge=True):
    bal = _grow_point(_uniform_cameras(2000, 30000, 130000, seed=7), 100, 100, seed=1)
    return _grow_point(bal, 200, 200, seed=2) if huge else bal


def _make(name):
    from tests.test_gpu_orders import _make as make_orders
    if name == "id_range":
        return _id_range()
    if name == "direct_v3":
        return _local_with_wide_middle(2.0 / 132, 1800)
    if name == "v4_narrow":
        return _local_with_wide_middle(2.0 / 132, 900)
    if name == "dups_direct":
        return _duplicate_row(_local_with_wide_middle(2.0 / 132, 900), 5)
    if name == "dups_id_range":
        return _duplicate_row(_id_range(huge=False), 5)
    if name == "tile":
        return _grow_point(make_orders("scatter"), 300, 200, seed=3)
    raise KeyError(name)


# The fields that define each fixture's configuration, and the rows of the configuration table (see configurations)
# it falls in: exactly these, so a fixture that drifts into another configuration fails test_configuration_table.
EXPECT = {
    "id_range": (dict(direct=0, mul="v3", v2b=0, folded=1, cam_major=1, diag="cam_major", huge=1), {"id_range", "huge_without_v4"}),
    "direct_v3": (dict(direct=1, mul="v3", v2b=0, cam_major=1, diag="cam_major", huge=0), {"direct_v3"}),
    "v4_narrow": (dict(direct=1, mul="v4", mul_r=1, v2b=1, cam_major=1, diag="cam_major", huge=0), {"direct_v4_fewer_warps"}),
    "dups_direct": (dict(direct=1, mul="v4", mul_r=1, cam_major=0, diag="tile", huge=0),
                    {"direct_v4_fewer_warps", "diag_tile_beside_warp_tiles"}),
    "dups_id_range": (dict(direct=0, mul="v3", cam_major=0, diag="tile", huge=0), {"id_range", "diag_tile_beside_warp_tiles"}),
    "tile": (dict(mul="tile", cam_major=1, diag="cam_major", huge=1), {"tile_everywhere", "huge_without_v4"}),
}


def configurations(plan):
    """The rows of the configuration table a plan falls in."""
    rows = set()
    mul = plan["mul"]
    if mul == "v4-owned":
        rows.add("direct_v4_owned")
    elif mul == "v4":
        rows.add("direct_v4_shared_16_warps" if plan["mul_w"] == 16 else "direct_v4_fewer_warps")
    elif mul == "v3":
        rows.add("direct_v3" if plan["direct"] else "id_range")
    elif mul == "tile":
        rows.add("tile_everywhere")
    if plan["diag"] == "v2":
        rows.add("diag_v2")
    elif plan["diag"] == "tile" and mul != "tile":
        rows.add("diag_tile_beside_warp_tiles")
    if plan["huge"] > 0 and mul in ("v3", "tile"):
        rows.add("huge_without_v4")
    return rows


TABLE = {"direct_v4_owned", "direct_v4_shared_16_warps", "direct_v4_fewer_warps", "direct_v3", "id_range", "tile_everywhere",
         "diag_v2", "diag_tile_beside_warp_tiles", "huge_without_v4"}


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.fixture
def problem_plan(monkeypatch, capfd):
    """plan(C, P, row_cam, row_pt, row_obs) -> dict: creates a Problem with B200_VERBOSE set (the library reads it in
    b200_create), closes it again and returns the configuration line as parsed by parse_plan."""
    def plan(C, P, row_cam, row_pt, row_obs):
        import ceres_solver_b200 as cs
        monkeypatch.setenv("B200_VERBOSE", "1")
        capfd.readouterr()
        gpu = cs.Problem(C, P, row_cam, row_pt, row_obs)
        gpu.close()
        monkeypatch.delenv("B200_VERBOSE")
        return parse_plan(capfd.readouterr().err)
    return plan


_bals = {}


def _bal(name):
    if name not in _bals:
        _bals[name] = _make(name)
    return _bals[name]


def _plan_of(problem_plan, bal):
    from ceres_solver_b200 import bal as B
    rp = B.ReducedProgram(bal)
    return problem_plan(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs)


@pytest.mark.parametrize("name", sorted(EXPECT))
def test_plan(name, cs, problem_plan):
    plan = _plan_of(problem_plan, _bal(name))
    fields, _ = EXPECT[name]
    assert {k: plan[k] for k in fields} == fields, plan
    if name == "v4_narrow":
        assert 8 <= plan["mul_w"] < 16, plan


@pytest.fixture(scope="module", params=sorted(EXPECT))
def case(request, cs, oracle):
    c = Case(cs, oracle, _bal(request.param))
    yield c
    c.close()


def test_every_entry_point(case, oracle):
    check_every_entry_point(case, oracle)


@pytest.fixture(scope="module")
def oracle_traces(case):
    return oracle_lm_traces(case, LM_ITERATIONS, max_cg=LM_MAX_CG)


@pytest.mark.parametrize("host_boundary", [False, True])
def test_lm_trajectory(case, oracle_traces, host_boundary):
    check_lm_trajectory(case, oracle_traces, LM_ITERATIONS, host_boundary, max_cg=LM_MAX_CG)


def test_huge_point_with_duplicates_is_refused(cs):
    """b200_create refuses a point with more than 128 rows together with a duplicate (camera, point) row."""
    from ceres_solver_b200 import bal as B
    bal = _duplicate_row(_bal("id_range"), 5)
    rp = B.ReducedProgram(bal)
    with pytest.raises(cs.B200Error) as e:
        cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs)
    assert e.value.code == cs.binding.ERR_UNSUPPORTED


def test_configuration_table(cs, problem_plan, c16):
    """The fixtures of this module, with the ones of other modules that cover the remaining configurations, fall in
    exactly the configurations they are meant for, and together cover every row of the table."""
    from ceres_solver_b200 import bal as B
    from tests.test_gpu_orders import _make as make_orders
    from tests.test_gpu_parity import ragged_bal
    bals = {name: _bal(name) for name in EXPECT}
    bals["c16"] = B.Bal(c16.cam_idx, c16.pt_idx, c16.obs, c16.cameras, c16.points)
    bals["circle"] = make_orders("circle")
    bals["ragged"] = ragged_bal()
    expect = {name: rows for name, (_, rows) in EXPECT.items()}
    expect.update(c16={"direct_v4_owned"}, circle={"direct_v4_shared_16_warps"}, ragged={"direct_v4_owned", "diag_v2"})
    got = {name: configurations(_plan_of(problem_plan, bal)) for name, bal in bals.items()}
    assert got == expect
    assert set().union(*got.values()) == TABLE
