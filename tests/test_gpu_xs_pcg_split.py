"""The resident PCG's product walk (csrc/xs_pcg.cuh) with block rows split over warps: each CTA's steps are cut into 16
contiguous warp ranges balanced by steps plus one per row segment, and a range may begin and end inside a row.

the most steps of a warp (one per row segment included) and the number of split rows that b200_create prints equal a
count made here from the block pattern with the same rule, and Ladybug-1723's longest warp walks at most 8.

The parity of solves on problems with split rows (Ladybug-1723, big_points, loop_closure; across residual resets and at
every exit) is held by test_gpu_xs_pcg.py and test_gpu_xs_pcg_staging.py; the plan test here asserts that those
problems do split rows.
"""
import re

import numpy as np
import pytest

from tests.test_gpu_xs_pcg import plan_lines, row_blocks, sm_count
from tests.test_gpu_xs_pcg_staging import _problem, cta_rows

pytestmark = pytest.mark.gpu

WARPS = 16    # kXpWarps
STEP = 3      # kXsStep: blocks per step

WALK_RE = r"^\[b200ba\] S PCG walk: at most (\d+) steps per warp \(one per row segment included\), (\d+) split rows$"


def _cut(starts, K):
    """Fill ranges in order, each up to cost K (a step costs 1, and 1 more when it begins a row segment); the range
    starts, or None when more than WARPS ranges are needed."""
    cuts, cost = [0], 0
    for k, first in enumerate(starts):
        add = 1 + (first or cost == 0)
        if cost + add > K:
            if len(cuts) == WARPS:
                return None
            cuts.append(k)
            cost, add = 0, 2
        cost += add
    return cuts


def walk_split(nb, G):
    """Per the plan: the largest warp cost over all CTAs, and the rows split over two or more warps."""
    steps = -(-np.asarray(nb) // STEP)
    rows = cta_rows(nb, G)
    worst, split = 0, 0
    for g in range(G):
        row_of, first, last = [], [], []
        for i in range(rows[g], rows[g + 1]):
            n = int(steps[i])
            row_of += [i] * n
            first += [True] + [False] * (n - 1)
            last += [False] * (n - 1) + [True]
        if not row_of:
            continue
        K = 2
        while _cut(first, K) is None:
            K += 1
        cuts = _cut(first, K) + [len(row_of)]
        for a, b in zip(cuts[:-1], cuts[1:]):
            if a == b:
                continue
            worst = max(worst, (b - a) + 1 + sum(first[a + 1:b]))
            if not last[b - 1] and (first[a] or row_of[a] != row_of[b - 1]):
                split += 1
    return worst, split


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.mark.parametrize("name", ["seq_dups", "big_points", "ladybug-1723", "loop_closure"])
def test_walk_balance(name, cs, monkeypatch, capfd):
    from ceres_solver_b200 import bal as B
    rp = B.ReducedProgram(_problem(name))
    err = plan_lines(cs, rp, monkeypatch, capfd)
    m = re.search(WALK_RE, err, re.M)
    assert m, err
    worst, split = walk_split(row_blocks(rp.row_cam, rp.row_pt, rp.C), sm_count())
    assert (int(m.group(1)), int(m.group(2))) == (worst, split)
    if name != "seq_dups":
        assert split > 0
    if name == "ladybug-1723":
        assert worst <= 8

