"""What the resident PCG on the explicit S (csrc/xs_pcg.cuh) stages in shared memory besides S: p (or, in a residual
reset, x) of every foreign column -- a column past the CTA's last block row that its blocks touch -- and the T slots of
its owned columns, where they fit.

  plan     the largest number of foreign columns and of owned-column T slots of any CTA that b200_create prints equal a
           count made here from the block pattern and the CTA split, the problems stay resident, and the slots are
           staged in every CTA except where a 160-camera point leaves no room
  parity   solves against the oracle's IterativeSchurComplementSolver, across residual resets, on two layouts the video
           sequences of test_gpu_xs_pcg.py do not have -- a loop closure (CTA 0's blocks reach into the last CTA's
           cameras), and fewer cameras than SMs (CTAs that own no rows, and a last CTA with rows but no foreign
           column) -- and on big_points, where some CTAs' T slots are staged and some are not
"""
import re

import numpy as np
import pytest

from tests.entry_points import Case, relerr
from tests.test_gpu_xs_pcg import RESET_PERIOD, _inputs, _make, _solve_both, plan_lines, sm_count

pytestmark = pytest.mark.gpu


def _loop_closure(C=1000, P=100000, N=450000, seed=43, tracks=40):
    """A video sequence whose end sees the start again: `tracks` points first seen by cameras 0..2 are also seen by the
    last three cameras."""
    from ceres_solver_b200 import bal as B
    from tests.test_gpu_dispatch import _add_rows
    bal = B.synthetic_sequence(C, P, N, seed=seed)
    first = np.full(bal.P, C, dtype=np.int64)
    np.minimum.at(first, bal.pt_idx, bal.cam_idx)
    for k in np.flatnonzero(first <= 2)[:tracks]:
        bal = _add_rows(bal, int(k), [C - 3, C - 2, C - 1], seed + int(k))
    return bal


def _problem(name):
    from ceres_solver_b200 import bal as B
    if name == "loop_closure":
        return _loop_closure()
    if name == "few_cameras":
        # 100 cameras on 132 SMs, still explicit: the implicit stream (29 MB) exceeds the L2 budget
        return B.synthetic_sequence(100, 30000, 150000, seed=47)
    return _make(name)


def block_pairs(cam, pt):
    """The off-diagonal blocks (i, j), i < j, of the upper triangle of S: camera pairs that share a point."""
    cam = np.asarray(cam, dtype=np.int64)
    pt = np.asarray(pt, dtype=np.int64)
    order = np.argsort(pt, kind="stable")
    cam, pt = cam[order], pt[order]
    deg = np.bincount(pt)
    ptr = np.concatenate([[0], np.cumsum(deg)])
    cnt = deg[pt]
    a = np.repeat(np.arange(cam.size), cnt)
    b = ptr[pt[a]] + np.arange(a.size) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    m = cam[a] < cam[b]
    C = int(cam.max()) + 1
    pairs = np.unique(cam[a][m] * C + cam[b][m])
    return pairs // C, pairs % C


def cta_rows(nb, G):
    """First block row of each of the G CTAs, and C after the last: the split of largest_share_kib (test_gpu_xs_pcg.py),
    filling CTAs in row order up to the least capacity that needs at most G of them; CTAs past the last one that gets
    rows own none."""
    nb = [int(n) for n in nb]

    def fill(K):
        starts, cur = [0], 0
        for i, n in enumerate(nb):
            if cur + n > K:
                starts.append(i)
                cur = 0
            cur += n
        return starts

    lo, hi = max(max(nb), -(-sum(nb) // G)), sum(nb)
    while lo < hi:
        mid = (lo + hi) // 2
        if len(fill(mid)) <= G:
            hi = mid
        else:
            lo = mid + 1
    starts = fill(lo)
    return starts + [len(nb)] * (G + 1 - len(starts))


def staging(cam, pt, C, G):
    """Per CTA: its sorted foreign columns, and the T slots of its owned columns (blocks (i, j), i < j, j owned)."""
    bi, bj = block_pairs(cam, pt)
    nb = 1 + np.bincount(bi, minlength=C)
    starts = cta_rows(nb, G)
    foreign, slots = [], []
    for g in range(G):
        i0, i1 = starts[g], starts[g + 1]
        foreign.append(np.unique(bj[(bi >= i0) & (bi < i1) & (bj >= i1)]))
        slots.append(int(np.count_nonzero((bj >= i0) & (bj < i1))))
    return starts, foreign, slots


PLAN_RE = (r"^\[b200ba\] S PCG: resident, (\d+) CTAs, .*, at most (\d+) foreign columns, at most (\d+) column slots "
           r"per CTA \((\d+) staged\)$")


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.mark.parametrize("name", ["seq_dups", "big_points", "ladybug-1723", "loop_closure", "few_cameras"])
def test_plan_staging_maxima(name, cs, monkeypatch, capfd):
    from ceres_solver_b200 import bal as B
    rp = B.ReducedProgram(_problem(name))
    err = plan_lines(cs, rp, monkeypatch, capfd)
    assert "[b200ba] S plan: explicit," in err, err
    m = re.search(PLAN_RE, err, re.M)
    assert m, err
    G = int(m.group(1))
    assert G == sm_count()
    starts, foreign, slots = staging(rp.row_cam, rp.row_pt, rp.C, G)
    assert int(m.group(2)) == max(f.size for f in foreign)
    assert int(m.group(3)) == max(slots)
    # every CTA's slots are staged, except on big_points: its 160-camera point gives the CTAs around it more T slots
    # than the shared memory S leaves, and those CTAs sum from T in L2
    staged = int(m.group(4))
    assert staged < max(slots) if name == "big_points" else staged == max(slots)
    if name == "loop_closure":
        last = max(g for g in range(G) if starts[g] < starts[g + 1])
        assert np.any(foreign[0] >= starts[last]), (foreign[0], starts[last])
    if name == "few_cameras":
        owning = [g for g in range(G) if starts[g] < starts[g + 1]]
        assert len(owning) < G
        assert foreign[owning[-1]].size == 0


# 25 iterations cross two residual resets.  few_cameras: 100 cameras that each see ~1500 points make block Jacobi
# nearly exact; the CG reaches rounding level within about 5 iterations, after which the zeta test stops it at a
# rounding-dependent iteration (5 here, 11 in the oracle, with this change and without it), so it is held to 4.
ITERATIONS = {"loop_closure": 25, "big_points": 25, "few_cameras": 4}


@pytest.mark.parametrize("name", sorted(ITERATIONS))
def test_staged_solve(name, cs, oracle, monkeypatch, capfd):
    """big_points mixes CTAs that sum their columns from staged T slots with CTAs that sum them from T in L2."""
    iterations = ITERATIONS[name]
    assert name == "few_cameras" or iterations > 2 * RESET_PERIOD
    c = Case(cs, oracle, _problem(name))
    try:
        err = plan_lines(cs, c.rp, monkeypatch, capfd)
        assert re.search(PLAN_RE, err, re.M), err
        _inputs(c)
        x, its, term, xo, its_o, term_o = _solve_both(c, c.res, c.res_o, iterations)
        assert (its, term) == (its_o, term_o) == (iterations, term_o)
        assert relerr(x, xo) < 1e-7
    finally:
        c.close()
