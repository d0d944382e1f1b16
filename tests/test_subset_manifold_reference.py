"""CPU guard of tests/subset_manifold_reference.py, the tangent-space reference the GPU tests of
b200_set_subset_manifolds compare against, and of the Python packing of the masks."""
import numpy as np
import pytest

from tests import constant_blocks_reference as R
from tests import lm_cases as L
from tests import subset_manifold_reference as S
from tests.entry_points import compare_lm_traces_exact
from tests.test_constant_blocks_reference import c16_sets


@pytest.fixture(scope="module")
def c16_state(c16):
    from ceres_solver_b200 import bal as B
    bal = L.c16_bal(c16)
    return bal, B.ReducedProgram(bal).state(bal)


def _full(oracle, bal):
    return R.ReducedProgram(oracle, bal)


@pytest.mark.parametrize("solver", ["iterative", "dense"])
def test_empty_masks_are_the_oracle_transcript(oracle, c16_state, solver):
    """With empty masks the tangent program is the oracle's program: its LM loop reproduces the oracle's C16 transcript."""
    bal, state = c16_state
    sp = S.SubsetProgram(oracle, bal, camera_mask=np.zeros((bal.C, 9), bool), point_mask=np.zeros((bal.P, 3), bool))
    o = sp.default_options()
    o.num_threads, o.max_num_iterations = 8, 5
    o.linear_solver = 0 if solver == "iterative" else 1
    best_o, recs_o, _ = sp.base.solve(state, o)
    best, recs = sp.solve(state, o)
    compare_lm_traces_exact(recs, recs_o)
    assert np.linalg.norm(best - best_o) <= 1e-9 * np.linalg.norm(best_o)


@pytest.mark.parametrize("name", ["gauge_points", "points"])
def test_full_masks_are_constant_blocks(oracle, c16_state, name):
    """A full mask is a constant block (ParameterBlock::IsConstant): the same records as the reduced program with those
    blocks constant (to the multithreaded oracle's summation order)."""
    bal, state = c16_state
    full = _full(oracle, bal)
    cam, pts = c16_sets(full.P, full.C, full.base.row_cam, full.base.row_pt)[name]
    cm = np.zeros((bal.C, 9), bool)
    pm = np.zeros((bal.P, 3), bool)
    if cam is not None:
        cm[cam] = True
    pm[pts] = True
    sp = S.SubsetProgram(oracle, bal, camera_mask=cm, point_mask=pm)
    rp = R.ReducedProgram(oracle, bal, cam, pts)
    assert np.array_equal(sp.fixed, rp.fixed) and not sp.masked.any()
    o = rp.default_options()
    o.num_threads, o.max_num_iterations, o.linear_solver = 8, 3, 1
    best_r, recs_r = rp.solve(state, o)
    best_s, recs_s = sp.solve(state, o)
    compare_lm_traces_exact(recs_s, recs_r)
    assert np.linalg.norm(best_s - best_r) <= 1e-9 * np.linalg.norm(best_r)
    assert np.array_equal(best_s[sp.fixed], state[sp.fixed])


@pytest.mark.parametrize("name", ["intrinsics", "mixed", "heights", "combined"])
def test_tangent_solve_is_the_reduced_solve(oracle, c16_state, name):
    """The oracle's dynamic-size Schur solve on the tangent Jacobian (column blocks of mixed sizes) equals a direct solve
    of the reduced normal equations with the masked components removed."""
    bal, state = c16_state
    full = _full(oracle, bal)
    cam, pts, cm, pm = S.c16_mask_sets(full.P, full.C, full.base.row_cam, full.base.row_pt)[name]
    sp = S.SubsetProgram(oracle, bal, cam, pts, cm, pm)
    assert sp.masked.any() and len(set(sp.col_sizes)) > (1 if name == "intrinsics" else 2) - (name == "heights")
    full.state0 = state
    ok, _, r, _ = full.evaluate(state)
    assert ok
    J = full.base.jacobian().values()
    Jf = R.jacobian_matrix(J, full.base.row_cam, full.base.row_pt, full.P, full.C)
    D = np.random.RandomState(4).uniform(0.5, 1.0, full.num_parameters)
    x_ref = R.reduced_solve(Jf, r, D, sp.fixed)
    x, _, term = sp.tangent_solve(J, r, D)
    assert term == 0
    assert np.all(x[sp.fixed] == 0.0)
    assert np.linalg.norm(x - x_ref) <= 1e-8 * np.linalg.norm(x_ref)


def test_reduced_solve_dense_guard(oracle):
    """On a problem small enough for a dense solve: reduced_solve with masked components equals the dense solve, and the
    tangent solve equals both."""
    from ceres_solver_b200 import bal as B
    bal = B.synthetic("tiny")
    rp = B.ReducedProgram(bal)
    state = rp.state(bal)
    full = _full(oracle, bal)
    full.state0 = state
    ok, _, r, _ = full.evaluate(state)
    assert ok
    J = full.base.jacobian().values()
    Jf = R.jacobian_matrix(J, full.base.row_cam, full.base.row_pt, full.P, full.C)
    cm, pm = S.mask_sets(full.base.row_cam, full.base.row_pt, full.P, full.C, per_class=3)
    pm[:3, 2] = True
    sp = S.SubsetProgram(oracle, bal, camera_mask=cm, point_mask=pm)
    D = np.random.RandomState(5).uniform(0.3, 1.0, full.num_parameters)
    x = R.reduced_solve(Jf, r, D, sp.fixed)
    xd = R.reduced_dense_solve(Jf, r, D, sp.fixed)
    xt, _, term = sp.tangent_solve(J, r, D)
    assert term == 0
    assert np.linalg.norm(x - xd) <= 1e-10 * np.linalg.norm(xd)
    assert np.linalg.norm(xt - xd) <= 1e-9 * np.linalg.norm(xd)


@pytest.mark.parametrize("name", ["intrinsics", "combined"])
def test_loop_keeps_masked_coordinates(oracle, c16_state, name):
    """The tangent loop converges, returns every constant component bitwise and moves the others."""
    bal, state = c16_state
    full = _full(oracle, bal)
    cam, pts, cm, pm = S.c16_mask_sets(full.P, full.C, full.base.row_cam, full.base.row_pt)[name]
    sp = S.SubsetProgram(oracle, bal, cam, pts, cm, pm)
    o = sp.default_options()
    o.num_threads, o.max_num_iterations, o.linear_solver = 8, 3, 1
    best, recs = sp.solve(state, o)
    assert np.array_equal(best[sp.fixed].view(np.int64), state[sp.fixed].view(np.int64))
    assert np.any(best[~sp.fixed] != state[~sp.fixed])
    assert recs[-1]["cost"] < recs[0]["cost"]


def test_effective_state():
    """A full mask makes its block constant; set-constant and masks combine as a union."""
    cc, pc, fixed, masked = S.effective(2, 2, camera_constant=[False, True], point_constant=None,
                                        camera_mask=[[True] * 9, [True] + [False] * 8], point_mask=[[0, 0, 1], [1, 1, 1]])
    assert list(cc) == [True, True] and list(pc) == [False, True]
    assert list(fixed) == [False, False, True, True, True, True] + [True] * 18
    assert list(masked) == [False, False, True] + [False] * 21


def test_python_packing():
    from ceres_solver_b200 import subset_manifold_masks
    cm = np.zeros((3, 9), bool)
    cm[0, [6, 7, 8]] = True
    cm[2, 0] = True
    pm = np.zeros((2, 3), bool)
    pm[1, 2] = True
    c, p = subset_manifold_masks(3, 2, cm, pm)
    assert c.dtype == np.uint16 and list(c) == [0x1c0, 0, 1]
    assert p.dtype == np.uint8 and list(p) == [0, 4]
    assert subset_manifold_masks(3, 2, None, None) == (None, None)
    for bad in (np.zeros((3, 8), bool), np.zeros((2, 9), bool), np.zeros(27, bool)):
        with pytest.raises(ValueError):
            subset_manifold_masks(3, 2, bad, None)
    for bad in (np.zeros((2, 2), bool), np.zeros((3, 3), bool), np.zeros(6, bool)):
        with pytest.raises(ValueError):
            subset_manifold_masks(3, 2, None, bad)
