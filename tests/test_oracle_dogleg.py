"""The DOGLEG reference (tests/dogleg_reference.py) against known answers, the library's host-only scalar logic
(ceres_solver_b200/csrc/dogleg.h, compiled with g++) against the reference, and the guard of tests/dogleg_cases.py: the
option sets the GPU tests run take every branch they are chosen for, on the reference's own traces."""
import os
import subprocess

import numpy as np
import pytest

from tests import dogleg_cases as K
from tests import dogleg_reference as R
from tests import lm_cases as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------- polynomial_test.cc: quartics with known roots
@pytest.mark.parametrize("roots", [(1.0, 2.0, 3.0, 4.0), (-42.0, 1e-3, 1.23e5, -9.0), (0.5, 0.5, -2.0, 7.0)])
def test_quartic_real_roots(roots):
    poly = np.poly(roots)
    ok, re, im = R.find_polynomial_roots(poly)
    assert ok and np.allclose(np.sort(re), np.sort(roots), rtol=1e-6, atol=1e-9) and np.allclose(im, 0.0, atol=1e-6)


def test_quartic_complex_roots_give_real_parts():
    poly = np.real(np.poly([1 + 2j, 1 - 2j, -3 + 0.5j, -3 - 0.5j]))
    ok, re, im = R.find_polynomial_roots(poly)
    assert ok and np.allclose(np.sort(re), [-3, -3, 1, 1]) and np.allclose(np.sort(np.abs(im)), [0.5, 0.5, 2, 2])


def test_leading_zeros_and_low_degrees():
    assert np.allclose(R.find_polynomial_roots([0.0, 0.0, 2.0, -4.0])[1], [2.0])
    assert np.allclose(np.sort(R.find_polynomial_roots([1.0, -3.0, 2.0])[1]), [1.0, 2.0])
    assert R.find_polynomial_roots([0.0, 0.0, 5.0])[0] and R.find_polynomial_roots([0.0, 0.0, 5.0])[1].size == 0
    assert not R.find_polynomial_roots([1.0, np.nan, 0.0, 1.0, 2.0])[0]


# ---------------------------------------------------------------- dogleg_strategy_test.cc, its six cases
def _fixture(name):
    from tests.golden import dogleg_fixtures as F
    d = np.array(F.DDIAG)
    if name == "ellipse":
        J = np.diag(np.sqrt(d)) @ np.array(F.BASIS)
        r = -J @ np.array(F.ELLIPSE_MINIMUM)
    else:
        J = np.diag(d)
        r = -J @ np.array(F.VALLEY_MINIMUM)
    return J, r


@pytest.mark.parametrize("case", list(range(6)))
def test_ceres_dogleg_strategy_cases(case):
    from tests.golden import dogleg_fixtures as F
    name, fixture, kind, radius, expected = F.CASES[case]
    J, r = _fixture(fixture)
    s = R.DoglegStrategy(R.TRADITIONAL if kind == "traditional" else R.SUBSPACE, radius, F.MIN_LM_DIAGONAL,
                         F.MAX_LM_DIAGONAL)
    x, _, term = s.compute_step(R.DenseOps(J, r), r)
    assert term != R.LS_FAILURE, name
    if expected == "obeyed":
        assert np.linalg.norm(x) <= radius * (1.0 + 4.0 * R.EPS), name
        # the constraint is active on the ellipse: both variants end on the boundary, in its two-dimensional cases
        if kind == "traditional":
            assert s.branch == "interpolated", name
        else:
            assert s.branch == "boundary" and s.rank == 2, name
    elif expected == "basis":
        B = s.basis
        assert abs(np.linalg.norm(B[:, 0]) - 1.0) <= F.K_TOLERANCE and abs(np.linalg.norm(B[:, 1]) - 1.0) <= F.K_TOLERANCE
        assert abs(B[:, 0] @ B[:, 1]) <= F.K_TOLERANCE
        for v in (s.gradient, s.gauss_newton_step):   # both project onto themselves
            assert np.linalg.norm(v - B @ (B.T @ v)) <= F.K_TOLERANCE, name
    else:
        assert np.all(np.abs(x - np.array(expected)) <= F.K_TOLERANCE_LOOSE), (name, x)


# ---------------------------------------------------------------- dogleg.h against the reference
@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("dogleg") / "dogleg_driver")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "dogleg_driver.cc")])
    return exe


def _run_driver(driver, lines):
    out = subprocess.run([driver], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True).stdout
    return [ln.split() for ln in out.strip().splitlines()]


def _model_line(s, dogleg_type, J):
    g, gn, d = s.gradient, s.gauss_newton_step, s.diagonal
    ja, jb = J @ (g / d), J @ (gn / d)
    vals = [g @ g, g @ gn, gn @ gn, ja @ ja, ja @ jb, jb @ jb]
    return "%d %.17g " % (dogleg_type, s.radius) + " ".join("%.17g" % v for v in vals)


def _strategy(dogleg_type, radius):
    return R.DoglegStrategy(dogleg_type, radius, 1e-6, 1e32)


BRANCHES = ["gauss_newton", "one_dimensional", "root_failure", "cosine_fallback", "boundary"]


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("dogleg_type", [R.TRADITIONAL, R.SUBSPACE])
def test_scalar_logic_matches_reference(driver, seed, dogleg_type):
    """Random dense problems at radii that take each step: the step dogleg.h describes equals the reference's step."""
    rng = np.random.RandomState(seed)
    J = rng.randn(8, 4) * rng.uniform(0.1, 10, size=4)
    r = rng.randn(8)
    for radius in (1e-3, 1e-1, 1.0, 1e3):
        s = _strategy(dogleg_type, radius)
        step, _, _ = s.compute_step(R.DenseOps(J, r), r)
        rank, kind, cg, cn, norm, branch = _run_driver(driver, [_model_line(s, dogleg_type, J)])[0]
        v = s.gauss_newton_step if int(kind) == 0 else float(cg) * s.gradient + float(cn) * s.gauss_newton_step
        assert np.linalg.norm(v / s.diagonal - step) <= 1e-9 * np.linalg.norm(step), (radius, s.branch)
        if dogleg_type == R.SUBSPACE:
            assert BRANCHES[int(branch)] == s.branch
            assert int(rank) == s.rank


def _reference_from_scalars(dogleg_type, radius, g, gn, G):
    """The reference's strategy on a two-dimensional model given as g, gn (diagonal 1) and G, the Gram matrix of J g and
    J gn: its basis from the Householder QR of [g gn], B = C^-T G C^-1 with C = Q' [g gn].  Returns (strategy, step),
    step None when ComputeSubspaceModel fails."""
    s = R.DoglegStrategy(dogleg_type, radius, 1.0, 1.0)
    s.diagonal = np.ones(2)
    s.gradient, s.gauss_newton_step = np.array(g, float), np.array(gn, float)
    G = np.array(G, float)
    with np.errstate(all="ignore"):
        s.alpha = (s.gradient @ s.gradient) / G[0, 0]
        if dogleg_type == R.SUBSPACE:
            Q, s.rank, _, _ = R.col_piv_householder_qr(np.stack([s.gradient, s.gauss_newton_step], 1))
            if s.rank == 0:
                return s, None
            s.subspace_is_one_dimensional = s.rank == 1
            if s.rank == 2:
                C = Q.T @ np.stack([s.gradient, s.gauss_newton_step], 1)
                Ci = np.linalg.inv(C)
                s.basis, s.sg, s.B = Q, Q.T @ s.gradient, Ci.T @ G @ Ci
        return s, s._step()


def _scalar_line(dogleg_type, radius, g, gn, G):
    g, gn = np.array(g, float), np.array(gn, float)
    vals = [g @ g, g @ gn, gn @ gn, G[0][0], G[0][1], G[1][1]]
    return "%d %.17g " % (dogleg_type, radius) + " ".join("%.17g" % v for v in vals)


# Branches no BA trace reaches, on two-dimensional models: g parallel to gn (rank 1), both zero (rank 0), a NaN in the
# Gram matrix (the roots cannot be found: traditional step), and a model whose boundary minimum fails the 0.99 cosine test
# (G is not the Gram matrix that made gn, which only scalar inputs allow: traditional step).
SCALAR_CASES = [
    ("one_dimensional", 0.5, [1.0, 2.0], [-3.0, -6.0], [[5.0, -15.0], [-15.0, 45.0]]),
    ("rank_zero", 1.0, [0.0, 0.0], [0.0, 0.0], [[0.0, 0.0], [0.0, 0.0]]),
    ("root_failure", 0.1, [1.0, 0.0], [0.3, 2.0], [[2.0, float("nan")], [float("nan"), 3.0]]),
    ("cosine_fallback", 0.5, [-0.25, -0.78], [-5.06, 0.91], [[1.47, 1.11], [1.11, 2.67]]),
]


@pytest.mark.parametrize("case", SCALAR_CASES, ids=[c[0] for c in SCALAR_CASES])
def test_scalar_logic_unreachable_branches(driver, case):
    branch, radius, g, gn, G = case
    s, step = _reference_from_scalars(R.SUBSPACE, radius, g, gn, G)
    rank, kind, cg, cn, norm, br = _run_driver(driver, [_scalar_line(R.SUBSPACE, radius, g, gn, G)])[0]
    if branch == "rank_zero":
        assert step is None and s.rank == 0 and int(rank) == 0   # the strategy reports FAILURE on both sides
        return
    assert s.branch == branch and BRANCHES[int(br)] == branch
    assert int(rank) == s.rank
    gv, gnv = np.array(g, float), np.array(gn, float)
    v = gnv if int(kind) == 0 else (float(cg) * gv if int(kind) == 1 else float(cg) * gv + float(cn) * gnv)
    assert np.linalg.norm(v - step) <= 1e-12 * np.linalg.norm(step), (v, step)
    if branch == "one_dimensional":   # (an interpolated traditional step's norm is measured by the pass that forms it)
        assert abs(float(norm) - s.dogleg_step_norm) <= 1e-12 * s.dogleg_step_norm


# ---------------------------------------------------------------- the guard of tests/dogleg_cases.py
@pytest.fixture(scope="module")
def problems(oracle, c16):
    from ceres_solver_b200 import bal as B
    out = {}
    for name, bal in (("tiny", L.tiny_bal()), ("c16", L.c16_bal(c16)), ("zero_focal", L.zero_focal_bal())):
        rp = B.ReducedProgram(bal)
        orc = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())
        out[name] = (orc, rp.state(bal))
    return out


def test_option_sets_take_every_branch(problems):
    seen = set()
    for problem, option_set in K.TRACES:
        orc, state = problems[problem]
        options = K.OPTIONS[option_set]
        for dogleg_type in (R.TRADITIONAL, R.SUBSPACE):
            _, recs, info = R.minimize(orc, state, dogleg_type, **options)
            L.assert_decisions_have_margin(recs, options.get("min_relative_decrease", 1e-3))
            for (n, b, thresholds), r in zip(info[1:], recs[1:]):
                # |gn| and alpha |g| against the radius, and an accepted step's quality against StepAccepted's 0.25 / 0.75
                for key, ratio in thresholds.items():
                    assert abs(ratio - 1.0) >= K.MARGIN, (problem, option_set, dogleg_type, r["iteration"], key, ratio)
                if r["step_is_successful"]:
                    for t in (0.25, 0.75):
                        assert abs(r["tr_ratio"] - t) >= K.MARGIN * t, (problem, option_set, r["iteration"], r["tr_ratio"])
            seen.update(b for _, b, _ in info[1:] if b)
            reused = [i for i, (n, b, _) in enumerate(info) if i > 0 and n == 0 and b]
            if reused:
                seen.add("reused")
                assert all(recs[i - 1]["step_is_successful"] == 0 for i in reused)
    assert {"gauss_newton", "cauchy", "interpolated", "boundary", "reused"} <= seen, seen
    orc, state = problems["zero_focal"]
    _, recs, info = R.minimize(orc, state, R.TRADITIONAL, **K.INVALID)
    assert info[1][0] == 8 and all(r["step_is_valid"] == 0 for r in recs[1:])   # the mu retry loop, 1e-8 .. 1e-1
