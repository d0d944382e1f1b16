"""The one-pass product on the explicit S (csrc/explicit_schur.cuh): xs_mul_kernel reads each stored block once, writes
the row part of S x and leaves the transposed half in T, which xs_gather_kernel (b200_schur_multiply) or the PCG's
vector kernel adds to the output.  On the two explicit video sequences of test_gpu_explicit_schur.py and on Ladybug-1723:

  product   S x on random vectors against the oracle's ImplicitSchurComplement, and bitwise-identical repeats
  pcg       a 25-iteration SCHUR_JACOBI solve (two residual resets, at iterations 10 and 20) against the oracle's
  grid      the product's grid, as b200_create prints it, is one wave: at most the CTAs that are resident together
"""
import re

import numpy as np
import pytest

from tests.entry_points import Case, relerr

pytestmark = pytest.mark.gpu

CG_ITERATIONS, RESET_PERIOD = 25, 10


def _make(name):
    from ceres_solver_b200 import bal as B
    from tests.test_gpu_explicit_schur import _sequence_with_big_points, _sequence_with_duplicates
    if name == "seq_dups":
        return _sequence_with_duplicates()
    if name == "big_points":
        return _sequence_with_big_points()
    return B.synthetic(name)


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.fixture(scope="module", params=["seq_dups", "big_points", "ladybug-1723"])
def xcase(request, cs, oracle):
    c = Case(cs, oracle, _make(request.param))
    c.name = request.param
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
    yield c
    c.close()


def test_products_match_oracle_and_repeat_bitwise(xcase, oracle):
    gpu, J, D = xcase.gpu, xcase.J, xcase.D
    isc = oracle.ImplicitSchur(J, gpu.P, want_ftf=False, nt=8)
    isc.init(D, xcase.res_o)
    gpu.schur_init(xcase.res, D)
    rng = np.random.RandomState(11)
    for _ in range(3):
        u = rng.randn(9 * gpu.C)
        got = gpu.schur_multiply(u)
        assert relerr(got, isc.right_multiply(u)) < 1e-9, xcase.name
        assert np.array_equal(gpu.schur_multiply(u), got), xcase.name


def test_pcg_across_two_residual_resets(xcase):
    gpu, J, D = xcase.gpu, xcase.J, xcase.D
    o = gpu.solver_options(preconditioner_type=2, max_num_iterations=CG_ITERATIONS, residual_reset_period=RESET_PERIOD,
                           q_tolerance=0.0, r_tolerance=-1.0)
    x, its, term = gpu.schur_solve(xcase.res, D, o)
    xo, its_o, term_o = J.linear_solve(gpu.P, xcase.res_o, D, solver=0, preconditioner=2, max_iter=CG_ITERATIONS,
                                       reset_period=RESET_PERIOD, q_tolerance=0.0, r_tolerance=-1.0, nt=8)
    assert (its, term) == (its_o, term_o) == (CG_ITERATIONS, term_o), xcase.name
    assert relerr(x, xo) < 1e-7, xcase.name


def test_product_grid_is_one_wave(xcase, cs, monkeypatch, capfd):
    rp = xcase.rp
    monkeypatch.setenv("B200_VERBOSE", "1")
    capfd.readouterr()
    cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs).close()
    monkeypatch.delenv("B200_VERBOSE")
    err = capfd.readouterr().err
    assert "[b200ba] S plan: explicit," in err, err
    m = re.search(r"^\[b200ba\] S product: grid (\d+) of (\d+) resident CTAs \((\d+) per SM\), (\d+) warps", err, re.M)
    assert m, err
    grid, resident, per_sm, warps = (int(g) for g in m.groups())
    assert 1 <= grid <= resident and per_sm >= 1 and warps == 8 * grid
    assert warps <= rp.C + 7   # no more warps than block rows (up to the last CTA's)
