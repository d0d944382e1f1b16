"""Oracle parity ON THE BENCHMARKED WORKLOADS (BASELINE.json configs[2], configs[3] and SURVEY 8d's I2 recipe):
the CUDA path through the C ABI against the CPU oracle at full size -- evaluate, S*x, the SCHUR_JACOBI blocks, J'J x and
the first LM iterations (cost and step norm to north_star's 1e-6; the later iterations of bench.py hit the
500-iteration cap of the inexact solver, where the trajectory is no longer a parity statement).
`-m gpu`; the oracle side takes a few seconds per workload on the box's host cores."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def relerr(a, b):
    a = np.asarray(a, dtype=float)
    b = np.asarray(b, dtype=float)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


class Headline:
    def __init__(self, cs, oracle, name):
        from ceres_solver_b200 import bal as B
        bal = B.synthetic(name)
        self.rp = B.ReducedProgram(bal)
        self.orc = oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())
        assert np.array_equal(self.rp.row_pt, self.orc.row_pt) and np.array_equal(self.rp.row_cam, self.orc.row_cam)
        self.gpu = cs.Problem(self.rp.C, self.rp.P, self.rp.row_cam, self.rp.row_pt, self.rp.row_obs)
        self.state = self.rp.state(bal)
        self.nt = oracle.max_threads()


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.fixture(scope="module", params=["ladybug-1723", "ladybug-1723-random", "venice-1778"])
def case(request, cs, oracle):
    c = Headline(cs, oracle, request.param)
    yield c
    c.gpu.close()


def test_components_match_oracle(case, oracle):
    gpu, orc, nt = case.gpu, case.orc, case.nt
    ok, cost, res, grad = gpu.evaluate(case.state)
    ok_o, cost_o, res_o, grad_o = orc.evaluate(case.state, nt=nt)
    assert ok and ok_o
    assert abs(cost - cost_o) <= 1e-12 * cost_o
    assert relerr(res, res_o) < 1e-12                       # north_star: residuals to 1e-6
    assert np.abs(res - res_o).max() <= 1e-9 * np.abs(res_o).max()
    assert relerr(grad, grad_o) < 1e-10
    J = orc.jacobian()
    assert relerr(gpu.jacobian_values(), J.values()) < 1e-12
    # Jacobi scaling + LM diagonal as the first iteration sees them
    s = 1.0 / (1.0 + np.sqrt(J.squared_column_norm()))
    assert relerr(gpu.squared_column_norm(), J.squared_column_norm()) < 1e-12
    gpu.scale_columns(s)
    J.scale_columns(s, nt=nt)
    D = np.sqrt(np.clip(J.squared_column_norm(), 1e-6, 1e32) / 1e4)
    rng = np.random.RandomState(5)
    # J'J x + D^2 x
    x = rng.randn(gpu.num_parameters)
    expect = J.left_multiply(J.right_multiply(x, nt=nt), nt=nt) + D * D * x
    assert relerr(gpu.jtj_multiply(x, D), expect) < 1e-11
    # implicit Schur complement: rhs, (E'E + D^2)^-1, S x, back substitution
    isc = oracle.ImplicitSchur(J, gpu.P, want_ftf=False, nt=nt)
    isc.init(D, res_o)
    gpu.schur_init(res, D)
    assert relerr(gpu.schur_rhs(), isc.rhs()) < 1e-9
    assert relerr(gpu.schur_ete_inverse(), isc.ete_inverse()) < 1e-9
    u = rng.randn(9 * gpu.C)
    assert relerr(gpu.schur_multiply(u), isc.right_multiply(u)) < 1e-9
    assert relerr(gpu.schur_back_substitute(u), isc.back_substitute(u)) < 1e-9
    # SCHUR_JACOBI blocks = diagonal blocks of the eliminator's S
    C = gpu.C
    diag, _ = J.schur_eliminate(gpu.P, None, D, diagonal_only=True, diag_len=81 * C, nt=nt, n_f=9 * C)
    blocks, inv = gpu.schur_jacobi_update()
    assert relerr(blocks, diag) < 1e-9


@pytest.fixture(scope="module")
def oracle_traces(case):
    """The oracle's first three LM iterations with all host threads and with 7, 5 and 3 -- different summation orders in
    its own products.  The inexact solver amplifies last-bit differences once it runs for 100+ CG iterations on an
    ill-conditioned reduced system: on ladybug-1723 the oracle's step norm at LM iteration 3 (117 CG iterations) moves by
    2e-5 between thread counts while iterations 1-2 (4 and 34 CG iterations) agree to 1e-10, and its |g|_inf there spans
    5e-3 over 1, 2, 3, 5, 7 and 16 threads although some pairs agree to 2e-4.  The spread over several oracle runs is
    therefore the resolution of the comparison."""
    out = []
    for nt in dict.fromkeys((case.nt, 7, 5, 3)):
        o = case.orc.default_options()
        o.num_threads = nt
        o.max_num_iterations = 3
        _, recs, _ = case.orc.solve(case.state, o)
        out.append(recs)
    return out


@pytest.mark.parametrize("host_boundary", [False, True])
def test_first_lm_iterations_match_oracle(case, oracle_traces, host_boundary):
    """Three LM iterations of bundle_adjuster's configuration from the bench's initial point: same CG iteration counts and
    accept/reject sequence; cost, step norm, gradient norm and radius to north_star's 1e-6 -- or, where the oracle itself
    cannot reproduce its own numbers to 1e-6 under a change of summation order, measured against the oracle's own spread
    (tests/conftest.py: compare_lm_traces)."""
    from tests.conftest import compare_lm_traces
    _, recs = case.gpu.lm_solve(case.state, case.gpu.lm_options(max_num_iterations=3), host_boundary=host_boundary)
    assert len(recs) == 4
    compare_lm_traces(recs, *oracle_traces)
