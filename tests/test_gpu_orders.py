"""The library keeps its own point order and per-CTA camera lists (b200_create); what crosses the ABI stays in the
caller's order.  Three structures exercise the three orders, each against the oracle through every entry point
(tests/entry_points.py):

  circle   SURVEY 8d I2 recipe (cameras on a circle, each point seen by cameras spread over a window around its
           azimuth), points in RANDOM order  -> internal re-ordering + boundary permutations + camera lists with
           wrap-around at camera 0 / C-1
  scatter  every point sees cameras drawn uniformly from all 3000 of them: no order has locality.  Its per-CTA camera
           span is all 3000 cameras, and one camera vector of that size does not fit in shared memory next to the tile
           buffers, so every operation runs on the CTA-tile kernels.  The id-range kernels (schur_mul_v3, jtj_v2,
           cam_reduce_kernel) are tested on their own fixture in tests/test_gpu_dispatch.py.
  sorted   the circle problem with the points already sorted by azimuth -> the caller's order is kept (identity)
"""
import numpy as np
import pytest

from tests.entry_points import Case, check_every_entry_point, check_lm_trajectory, oracle_lm_traces

pytestmark = pytest.mark.gpu


def _scatter_problem(C=3000, P=35000, N=150000, seed=5):
    from ceres_solver_b200 import bal as B
    base = B.synthetic_bal(C, P, N, seed=seed)
    rng = np.random.RandomState(seed)
    # same geometry, but every observation re-assigned to a uniformly random camera (distinct within a point)
    deg = np.bincount(base.pt_idx, minlength=P)
    cam = np.concatenate([rng.choice(C, size=d, replace=False) for d in deg]).astype(np.int32)
    obs = B.snavely_project(base.cameras, base.points, cam, base.pt_idx) + rng.normal(0.0, 0.5, (N, 2))
    return B.Bal(cam, base.pt_idx, obs, base.cameras, base.points)


def _make(kind):
    from ceres_solver_b200 import bal as B
    if kind == "scatter":
        return _scatter_problem()
    bal = B.synthetic_bal(400, 12000, 52000, seed=11)
    if kind == "sorted":
        # relabel the points in order of their smallest camera (what an incremental reconstruction would produce)
        P = bal.P
        kmin = np.full(P, bal.C, dtype=np.int64)
        np.minimum.at(kmin, bal.pt_idx, bal.cam_idx)
        order = np.argsort(kmin, kind="stable")
        new_id = np.empty(P, dtype=np.int64)
        new_id[order] = np.arange(P)
        pt = new_id[bal.pt_idx]
        rows = np.argsort(pt, kind="stable")
        bal = B.Bal(bal.cam_idx[rows], pt[rows].astype(np.int32), bal.obs[rows], bal.cameras, bal.points[order])
    return bal


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.fixture(scope="module", params=["circle", "scatter", "sorted"])
def case(request, cs, oracle):
    c = Case(cs, oracle, _make(request.param))
    yield c
    c.close()


def test_every_entry_point_in_caller_order(case, oracle):
    check_every_entry_point(case, oracle)


@pytest.fixture(scope="module")
def oracle_traces(case):
    return oracle_lm_traces(case, 4)


@pytest.mark.parametrize("host_boundary", [False, True])
def test_lm_trajectory(case, oracle_traces, host_boundary):
    check_lm_trajectory(case, oracle_traces, 4, host_boundary)
