"""The resident PCG on the explicit S (csrc/xs_pcg.cuh): one cooperative launch per SCHUR_JACOBI solve, S in the shared
memory of one CTA per SM.

  plan      on the explicit sequences of test_gpu_explicit_schur.py and on Ladybug-1723 the PCG is resident on every SM,
            and the largest CTA's share of S that b200_create prints equals a count made here from the block pattern
  fallback  a sequence about twice Ladybug-1723's size is still explicit, but its S does not fit: the two-kernel loop runs
            and matches the oracle
  parity    25- and 60-iteration solves across residual resets, and every exit the oracle can reach (zeta, |r| tolerance,
            the iteration cap, min_iterations, b = 0), against the oracle's IterativeSchurComplementSolver: the same
            iteration counts and terminations, solutions within 1e-7
"""
import re

import numpy as np
import pytest

from tests.entry_points import Case, relerr

pytestmark = pytest.mark.gpu

RESET_PERIOD = 10


def _make(name):
    from ceres_solver_b200 import bal as B
    from tests.test_gpu_explicit_schur import _sequence_with_big_points, _sequence_with_duplicates
    if name == "seq_dups":
        return _sequence_with_duplicates()
    if name == "big_points":
        return _sequence_with_big_points()
    if name == "seq_large":
        # about twice Ladybug-1723's cameras, points and rows: S is ~43 MB, ~330 KiB per SM
        return B.synthetic_sequence(3446, 313000, 1357000)
    return B.synthetic(name)


def row_blocks(cam, pt, C):
    """Stored blocks of each block row of the upper triangle of S: the diagonal block and one per camera j > i that
    shares a point with camera i."""
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
    pairs = np.unique(cam[a][m] * C + cam[b][m])
    return 1 + np.bincount(pairs // C, minlength=C)


def largest_share_kib(nb, G):
    """The block rows in G contiguous ranges with the smallest largest range: the least capacity at which filling
    ranges in row order, each up to that many blocks, needs at most G ranges."""
    nb = [int(n) for n in nb]

    def fill(K):
        shares, cur = [], 0
        for n in nb:
            if cur + n > K:
                shares.append(cur)
                cur = 0
            cur += n
        return shares + [cur]

    lo, hi = max(max(nb), -(-sum(nb) // G)), sum(nb)
    while lo < hi:
        mid = (lo + hi) // 2
        if len(fill(mid)) <= G:
            hi = mid
        else:
            lo = mid + 1
    return max(fill(lo)) * 648.0 / 1024.0


def plan_lines(cs, rp, monkeypatch, capfd):
    monkeypatch.setenv("B200_VERBOSE", "1")
    capfd.readouterr()
    cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs).close()
    monkeypatch.delenv("B200_VERBOSE")
    return capfd.readouterr().err


def sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.mark.parametrize("name", ["seq_dups", "big_points", "ladybug-1723"])
def test_plan_is_resident(name, cs, monkeypatch, capfd):
    from ceres_solver_b200 import bal as B
    rp = B.ReducedProgram(_make(name))
    err = plan_lines(cs, rp, monkeypatch, capfd)
    assert "[b200ba] S plan: explicit," in err, err
    m = re.search(r"^\[b200ba\] S PCG: resident, (\d+) CTAs, largest S share ([\d.]+) KiB of ([\d.]+) KiB", err, re.M)
    assert m, err
    G, share, limit = int(m.group(1)), float(m.group(2)), float(m.group(3))
    assert G == sm_count()
    assert share == pytest.approx(largest_share_kib(row_blocks(rp.row_cam, rp.row_pt, rp.C), G), abs=0.006)
    assert share <= limit


def _inputs(c):
    """Jacobi-scaled J and the LM diagonal of the first iteration, on GPU and oracle alike."""
    gpu, orc = c.gpu, c.orc
    ok, _, res, _ = gpu.evaluate(c.state)
    ok_o, _, res_o, _ = orc.evaluate(c.state, nt=8)
    assert ok and ok_o
    J = orc.jacobian()
    s = 1.0 / (1.0 + np.sqrt(J.squared_column_norm()))
    gpu.scale_columns(s)
    J.scale_columns(s, nt=8)
    c.J, c.res, c.res_o = J, res, res_o
    c.D = np.sqrt(np.clip(J.squared_column_norm(), 1e-6, 1e32) / 1e4)


def _solve_both(c, res, res_o, max_iter, min_iter=0, q_tol=0.0, r_tol=-1.0):
    gpu = c.gpu
    o = gpu.solver_options(preconditioner_type=2, max_num_iterations=max_iter, min_num_iterations=min_iter,
                           residual_reset_period=RESET_PERIOD, q_tolerance=q_tol, r_tolerance=r_tol)
    x, its, term = gpu.schur_solve(res, c.D, o)
    xo, its_o, term_o = c.J.linear_solve(gpu.P, res_o, c.D, solver=0, preconditioner=2, min_iter=min_iter,
                                         max_iter=max_iter, reset_period=RESET_PERIOD, q_tolerance=q_tol,
                                         r_tolerance=r_tol, nt=8)
    return x, its, term, xo, its_o, term_o


def test_fallback_two_kernel(cs, oracle, monkeypatch, capfd):
    c = Case(cs, oracle, _make("seq_large"))
    try:
        err = plan_lines(cs, c.rp, monkeypatch, capfd)
        assert "[b200ba] S plan: explicit," in err, err
        assert re.search(r"^\[b200ba\] S PCG: two-kernel \(", err, re.M), err
        _inputs(c)
        x, its, term, xo, its_o, term_o = _solve_both(c, c.res, c.res_o, 25)
        assert (its, term) == (its_o, term_o) == (25, term_o)
        assert relerr(x, xo) < 1e-7
    finally:
        c.close()


@pytest.fixture(scope="module")
def lcase(cs, oracle):
    c = Case(cs, oracle, _make("ladybug-1723"))
    _inputs(c)
    yield c
    c.close()


@pytest.mark.parametrize("iterations", [25, 60])
def test_resident_across_residual_resets(lcase, iterations):
    x, its, term, xo, its_o, term_o = _solve_both(lcase, lcase.res, lcase.res_o, iterations)
    assert (its, term) == (its_o, term_o) == (iterations, term_o)
    assert relerr(x, xo) < 1e-7


# each exit: (max iterations, min iterations, q_tolerance, r_tolerance)
EXITS = {"zeta": (200, 0, 0.1, -1.0), "residual": (200, 0, 0.0, 0.5), "max_iterations": (7, 0, 0.0, -1.0),
         "min_iterations": (200, 23, 0.1, -1.0)}


@pytest.mark.parametrize("exit_name", sorted(EXITS))
def test_resident_exits(lcase, exit_name):
    max_iter, min_iter, q_tol, r_tol = EXITS[exit_name]
    x, its, term, xo, its_o, term_o = _solve_both(lcase, lcase.res, lcase.res_o, max_iter, min_iter, q_tol, r_tol)
    assert (its, term) == (its_o, term_o), exit_name
    assert its < max_iter if exit_name != "max_iterations" else its == max_iter
    if exit_name == "min_iterations":
        assert its >= min_iter
        zeta_its = _solve_both(lcase, lcase.res, lcase.res_o, max_iter, 0, q_tol, r_tol)[1]
        assert zeta_its < min_iter   # without the floor the zeta test would have stopped earlier
    assert relerr(x, xo) < 1e-7, exit_name


def test_resident_zero_rhs(lcase):
    zero, zero_o = np.zeros_like(lcase.res), np.zeros_like(lcase.res_o)
    x, its, term, xo, its_o, term_o = _solve_both(lcase, zero, zero_o, 25)
    assert (its, term) == (its_o, term_o) == (0, 0)
    assert not np.any(x) and not np.any(xo)
