"""The explicit block-sparse Schur complement (csrc/explicit_schur.cuh).  b200_create stores S when its camera graph is
sparse enough (DESIGN §1); the PCG, b200_schur_multiply and b200_schur_jacobi_update then run on the stored S.

  plan      which problems go explicit, and the pair count and size b200_create prints against a count made here
  columns   S rebuilt column by column through schur_multiply on unit vectors (every column of a few cameras) against the
            oracle's ImplicitSchurComplement: a video sequence with duplicate (camera, point) rows, and one with a
            33..128-row and a >128-row point
  jacobi    the SCHUR_JACOBI blocks against the oracle
  lm        three LM iterations against the oracle at two thread counts, device-resident and through the host buffers
"""
import re

import numpy as np
import pytest

from tests.entry_points import Case, check_lm_trajectory, oracle_lm_traces, relerr

pytestmark = pytest.mark.gpu

# Three LM iterations with the CG capped at 10 iterations.  With 40, the second solve on big_points moves its step norm by
# up to 1.5e-5 between runs of the same GPU build (implicit and explicit S alike: last-bit differences of the reductions,
# amplified by the solve), more than the oracle's spread over two thread counts; 10 keeps every solve where GPU and oracle
# agree to 1e-6.
LM_ITERATIONS, LM_MAX_CG = 3, 10


def camera_pairs(cam, pt):
    """Number of distinct camera pairs i < j that share a point (the off-diagonal blocks of the upper triangle of S)."""
    cam = np.asarray(cam, dtype=np.int64)
    pt = np.asarray(pt, dtype=np.int64)
    C = int(cam.max()) + 1
    order = np.argsort(pt, kind="stable")
    cam, pt = cam[order], pt[order]
    deg = np.bincount(pt)
    ptr = np.concatenate([[0], np.cumsum(deg)])
    cnt = deg[pt]
    a = np.repeat(np.arange(cam.size), cnt)
    b = ptr[pt[a]] + np.arange(a.size) - np.repeat(np.cumsum(cnt) - cnt, cnt)
    m = cam[a] < cam[b]
    return int(np.unique(cam[a][m] * C + cam[b][m]).size)


def parse_s_plan(text):
    lines = [ln for ln in text.splitlines() if ln.startswith("[b200ba] S plan:")]
    assert len(lines) == 1, text
    m = re.fullmatch(r"\[b200ba\] S plan: (explicit|implicit), (\d+) pairs, ([\d.]+) MB", lines[0])
    assert m, lines[0]
    return m.group(1), int(m.group(2)), float(m.group(3))


def _sequence_with_big_points(C=1000, P=100000, N=450000, seed=29):
    """A video-sequence capture with one point seen by 60 more consecutive cameras (a 33..128-row point) and one by 160
    more (a >128-row point)."""
    from ceres_solver_b200 import bal as B
    from tests.test_gpu_dispatch import _add_rows
    bal = B.synthetic_sequence(C, P, N, seed=seed)
    for k, (lo, hi) in ((10, (C // 2, C // 2 + 60)), (20, (C // 2 - 80, C // 2 + 80))):
        have = set(bal.cam_idx[bal.pt_idx == k].tolist())
        bal = _add_rows(bal, k, [c for c in range(lo, hi) if c not in have], seed + k)
    return bal


def _sequence_with_duplicates(C=1000, P=100000, N=450000, seed=31):
    """A video-sequence capture with two duplicate (camera, point) rows."""
    from ceres_solver_b200 import bal as B
    from tests.test_gpu_dispatch import _duplicate_row
    return _duplicate_row(_duplicate_row(B.synthetic_sequence(C, P, N, seed=seed), 5), 77)


def _make(name, c16):
    from ceres_solver_b200 import bal as B
    from tests.test_gpu_dispatch import _make as make_dispatch
    if name == "c16":
        return B.Bal(c16.cam_idx, c16.pt_idx, c16.obs, c16.cameras, c16.points)
    if name == "seq_dups":
        return _sequence_with_duplicates()
    if name == "big_points":
        return _sequence_with_big_points()
    if name in ("tile", "dups_direct"):
        return make_dispatch(name)
    return B.synthetic(name)


# C16: its implicit stream fits the L2 residency budget; venice-1778: S with its row-pair list exceeds the size cap
# (both measured faster implicit); the others: the explicit product would read more than half of the implicit stream.
PLAN = {"seq_dups": "explicit", "big_points": "explicit", "ladybug-1723": "explicit", "c16": "implicit",
        "venice-1778": "implicit", "ladybug-1723-random": "implicit", "tile": "implicit", "dups_direct": "implicit"}


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.mark.parametrize("name", sorted(PLAN))
def test_plan(name, cs, c16, monkeypatch, capfd):
    from ceres_solver_b200 import bal as B
    rp = B.ReducedProgram(_make(name, c16))
    monkeypatch.setenv("B200_VERBOSE", "1")
    capfd.readouterr()
    cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs).close()
    monkeypatch.delenv("B200_VERBOSE")
    kind, pairs, mb = parse_s_plan(capfd.readouterr().err)
    expect_pairs = camera_pairs(rp.row_cam, rp.row_pt)
    assert (kind, pairs) == (PLAN[name], expect_pairs)
    assert mb == pytest.approx(648.0 * (expect_pairs + rp.C) / 1e6, abs=0.051)


@pytest.fixture(scope="module", params=["seq_dups", "big_points"])
def case(request, cs, oracle, c16):
    c = Case(cs, oracle, _make(request.param, c16))
    c.name = request.param
    yield c
    c.close()


def _schur_inputs(case):
    """Jacobi-scaled J and the LM diagonal of the first iteration, on GPU and oracle alike; returns (J, D, res)."""
    gpu, orc = case.gpu, case.orc
    ok, _, res, _ = gpu.evaluate(case.state)
    ok_o, _, res_o, _ = orc.evaluate(case.state, nt=8)
    assert ok and ok_o
    J = orc.jacobian()
    s = 1.0 / (1.0 + np.sqrt(J.squared_column_norm()))
    gpu.scale_columns(s)
    J.scale_columns(s, nt=8)
    D = np.sqrt(np.clip(J.squared_column_norm(), 1e-6, 1e32) / 1e4)
    gpu.schur_init(res, D)
    return J, D, res_o


def _unit(n, k):
    e = np.zeros(n)
    e[k] = 1.0
    return e


def test_columns_of_s(case, oracle):
    gpu = case.gpu
    C, P = gpu.C, gpu.P
    J, D, res_o = _schur_inputs(case)
    # every column of a few cameras: both ends of the sequence, the middle (the big points), and the cameras of the
    # duplicated rows
    rp = case.rp
    dup_cams = [int(rp.row_cam[np.flatnonzero(rp.row_pt == k)[0]]) for k in (5, 77)] if case.name == "seq_dups" else []
    cams = sorted({0, 1, C // 2, C // 2 + 30, C // 2 - 70, C - 1, *dup_cams})
    cols = np.concatenate([np.arange(9 * c, 9 * c + 9) for c in cams])
    isc = oracle.ImplicitSchur(J, P, want_ftf=False, nt=8)
    isc.init(D, res_o)
    expect = np.stack([isc.right_multiply(_unit(9 * C, k)) for k in cols], axis=1)
    got = np.stack([gpu.schur_multiply(_unit(9 * C, k)) for k in cols], axis=1)
    for t in range(len(cols)):
        assert relerr(got[:, t], expect[:, t]) < 1e-9, (case.name, cols[t])
    # S is symmetric: the blocks among the chosen cameras, read from both sides (the transposed half of the product)
    sub = got[cols, :]
    assert relerr(sub, sub.T) < 1e-12


def test_schur_jacobi_blocks(case, oracle):
    gpu = case.gpu
    C, P = gpu.C, gpu.P
    J, D, _ = _schur_inputs(case)
    diag, _ = J.schur_eliminate(P, None, D, diagonal_only=True, diag_len=81 * C, nt=8, n_f=9 * C)
    blocks, inv = gpu.schur_jacobi_update()
    assert relerr(blocks, diag) < 1e-9
    assert relerr(inv, np.linalg.inv(diag.reshape(-1, 9, 9)).ravel()) < 1e-7
    # the product after the preconditioner: S itself is unchanged by it
    u = np.random.RandomState(1).randn(9 * C)
    ref = gpu.schur_multiply(u)
    gpu.schur_jacobi_update()
    assert np.array_equal(gpu.schur_multiply(u), ref)


@pytest.fixture(scope="module")
def oracle_traces(case):
    return oracle_lm_traces(case, LM_ITERATIONS, max_cg=LM_MAX_CG)


@pytest.mark.parametrize("host_boundary", [False, True])
def test_lm_trajectory(case, oracle_traces, host_boundary):
    check_lm_trajectory(case, oracle_traces, LM_ITERATIONS, host_boundary, max_cg=LM_MAX_CG)
