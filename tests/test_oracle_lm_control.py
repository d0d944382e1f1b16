"""The constructions of tests/lm_cases.py on the oracle alone: each does what the GPU tests built on it
(tests/test_gpu_lm_control.py, tests/test_gpu_robust_loss.py) rely on, so that a change to a generator or to the oracle
fails here on a CPU machine instead of quietly testing something else on an H100."""
import numpy as np
import pytest

from tests import lm_cases as L


def _program(oracle, bal):
    from ceres_solver_b200 import bal as B
    orc = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())
    return orc, B.ReducedProgram(bal).state(bal)


@pytest.fixture(scope="module")
def programs(oracle, c16):
    return {"tiny": _program(oracle, L.tiny_bal()), "c16": _program(oracle, L.c16_bal(c16))}


@pytest.mark.parametrize("problem,name,k", L.EXITS)
def test_exit_fires_where_intended(problem, name, k, programs):
    """place_exit finds its threshold with the margin (it asserts that), and the exit then ends the solve at iteration k,
    before max_num_iterations and with every accept / reject decision clear of min_relative_decrease.

    The oracle runs on one thread here.  Threaded, its Schur elimination adds into shared blocks in the order the threads
    take their locks, as Ceres' does, so two runs differ in the last bits; past `tiny`'s convergence, where the cost
    changes by a few ulps, that decides whether a step is accepted and whether the free solve reaches its last
    iteration."""
    orc, state = programs[problem]
    options, num_records = L.place_exit(orc, state, name, k, L.REJECTION if name == "min_trust_region_radius" else None,
                                        nt=1)
    _, recs, _ = L.oracle_solve(orc, state, nt=1, **options)
    assert len(recs) == num_records < options["max_num_iterations"]
    L.assert_decisions_have_margin(recs, options.get("min_relative_decrease", 1e-3))
    # without the option the same solve runs on past the exit
    del options[name]
    _, recs_free, _ = L.oracle_solve(orc, state, nt=1, **options)
    assert len(recs_free) == options["max_num_iterations"] + 1


def test_rejection_chain(programs):
    orc, state = programs["c16"]
    _, recs, _ = L.oracle_solve(orc, state, **L.REJECTION)
    assert [int(r["step_is_successful"]) for r in recs] == [1, 1, 0, 0, 0, 0, 1, 0]
    assert all(r["step_is_valid"] for r in recs)
    L.assert_decisions_have_margin(recs, L.REJECTION["min_relative_decrease"])
    first, last = L.REJECTED_RUN
    assert [recs[j]["tr_radius"] / recs[j - 1]["tr_radius"] for j in range(first, last + 1)] == [0.5, 0.25, 0.125, 0.0625]


def test_zero_focal_length_makes_every_dense_solve_fail(oracle):
    orc, state = _program(oracle, L.zero_focal_bal())
    ok, _, res, _ = orc.evaluate(state, nt=8)
    assert ok
    J = orc.jacobian()
    colnorm = J.squared_column_norm()
    fblock = int(np.flatnonzero(orc.camera_of_fblock == 0)[0])
    assert np.flatnonzero(colnorm == 0.0).tolist() == [3 * orc.P + 9 * fblock + i for i in range(9) if i != 6]
    # each point keeps a camera with f != 0, so each E'E block stays positive definite without the diagonal
    assert np.unique(orc.row_pt[orc.row_cam != fblock]).size == orc.P
    for radius in L.INVALID_RADII:
        D = np.sqrt(colnorm / radius)   # min_lm_diagonal = 0, Jacobi scaling leaves zero columns zero
        _, its, term = J.linear_solve(orc.P, res, D, solver=L.DENSE_SCHUR, nt=8)
        assert (its, term) == (1, 2)   # FAILURE after one iteration
    for limit in (1, 3, 5):
        out, recs, _ = L.oracle_solve(orc, state, **dict(L.INVALID, max_num_consecutive_invalid_steps=limit))
        assert len(recs) == limit and np.array_equal(out, state)
        assert [r["tr_radius"] for r in recs] == list(L.INVALID_RADII[:limit])
        assert not any(r["step_is_valid"] for r in recs[1:])
    _, recs, _ = L.oracle_solve(orc, state, **dict(L.INVALID, min_trust_region_radius=1250.0))
    assert len(recs) == 3


def test_huber_branches(oracle):
    """Every class of rows of every problem of tests/test_gpu_robust_loss.py has inliers and outliers under Huber(a)
    with a = the median row norm, and the row classes each problem is meant to have are there."""
    from tests.test_gpu_dispatch import EXPECT, _bal
    from tests.test_gpu_parity import huge_bal
    problems = {name: _bal(name) for name in EXPECT}
    problems["huge"] = huge_bal()
    for name, bal in problems.items():
        orc, state = _program(oracle, bal)
        a = L.huber_scale(orc, state)
        branches = L.huber_branches(orc, state, a)
        for key, (inliers, outliers) in branches.items():
            assert inliers > 0 and outliers > 0, (name, key, inliers, outliers)
        if name in ("id_range", "tile", "huge"):
            assert len(branches) == 3, (name, branches)


def test_huber_branches_c16(oracle, c16):
    orc, state = _program(oracle, L.c16_bal(c16))
    a = L.huber_scale(orc, state)
    ((inliers, outliers),) = L.huber_branches(orc, state, a).values()
    assert inliers > 0 and outliers > 0
