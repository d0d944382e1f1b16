import bz2
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (sm_90) CUDA device (select with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import pyoracle
    pyoracle.build()
    return pyoracle


@pytest.fixture(scope="session")
def c16_path(tmp_path_factory):
    """data/problem-16-22106-pre.txt of the reference, shipped bz2-compressed under tests/golden/."""
    dst = tmp_path_factory.mktemp("bal") / "problem-16-22106-pre.txt"
    with bz2.open(os.path.join(GOLDEN, "problem-16-22106-pre.txt.bz2"), "rb") as f:
        dst.write_bytes(f.read())
    return str(dst)


@pytest.fixture(scope="session")
def c16(oracle, c16_path):
    """C16 after BALProblem::Normalize(), as the bundle_adjuster example feeds it to Ceres."""
    bal = oracle.BalProblem(c16_path)
    bal.normalize()
    return bal


@pytest.fixture(scope="session")
def c16_raw(oracle, c16_path):
    return oracle.BalProblem(c16_path)


def rel_err(a, b):
    a = np.asarray(a, dtype=float)
    b = np.asarray(b, dtype=float)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def compare_lm_traces(recs, recs_o, *recs_alt, keys=("cost", "step_norm", "gradient_max_norm", "tr_radius")):
    """GPU trace against the oracle's, with the oracle's OWN sensitivity as the yardstick.

    recs_o / recs_alt: the same oracle solve with different thread counts (different summation orders of its products); the
    spread of a value is its largest deviation over recs_alt.  The inexact
    Schur solve stops on a threshold after k CG iterations; while k is small the trajectory is reproducible to 1e-10 and
    north_star's 1e-6 is asserted.  Once a solve runs for 50+ iterations on the ill-conditioned reduced system, last-bit
    differences are amplified to the 1e-5 level in the step (measured: 2e-5 between oracle thread counts at 117 iterations
    on ladybug-1723) and the stopping test may fire one iteration earlier or later; from there on the tolerance is
    max(10 x oracle spread, 1e-4 -- 2e-3 after a 100+-iteration solve), a difference of up to max(2, 5 %) in the CG count is accepted (with 1e-2 on that iteration), and the
    comparison ends where the trajectories fork (different counts or accept/reject decisions)."""
    assert recs_alt and all(len(recs) == len(recs_o) == len(r) for r in recs_alt)
    loose = 0.0     # sticky: the state after a long solve carries its deviation into every later iteration
    for i, (a, b) in enumerate(zip(recs, recs_o)):
        alts = [r[i] for r in recs_alt]
        ko, kg = int(b["ls_iterations"]), int(a["ls_iterations"])
        if any(int(b2["ls_iterations"]) != ko or int(b2["step_is_successful"]) != int(b["step_is_successful"]) for b2 in alts):
            return   # the oracle forks against itself here
        long_solve = ko >= 50
        # 50-99 CG iterations: 1e-4; 100+ (observed on the I2-recipe problem: a 143-iteration solve that ends in a REJECTED
        # step, GPU and oracle 1e-4..1e-3 apart, two oracle runs 1e-5..1e-4 apart): 2e-3
        loose = max(loose, 2e-3 if ko >= 100 else (1e-4 if long_solve else 0.0))
        # (the stopping test zeta < eta fires on a plateau of a long solve: observed +-2 at ~50 iterations)
        assert abs(kg - ko) <= (max(2, ko // 20) if long_solve else 0), (a, b)
        assert a["step_is_successful"] == int(b["step_is_successful"]), (a, b)
        for key in keys:
            ref = float(b[key])
            spread = max(abs(float(b2[key]) - ref) for b2 in alts) / max(abs(ref), 1e-300)
            tol = max(1e-6, 10.0 * spread, loose)
            if kg != ko:
                tol = max(tol, 1e-2)   # one CG iteration more or less on a 50+-iteration solve: a percent-level change of the step
            assert abs(a[key] - ref) <= tol * max(abs(ref), 1e-300), (key, a[key], ref, spread, a["iteration"])
        if kg != ko:
            return   # forked by one CG iteration: later iterations are different problems
