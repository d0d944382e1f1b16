"""The Huber loss (bundle_adjuster --robustify) in every evaluate kernel, against the oracle.

The loss and its corrector are applied by one row function (evaluate_row) in two kernels: evaluate_v2_kernel (warp
tiles, points of up to 32 rows, Jacobian wanted) and evaluate_kernel<kWantJ> (CTA tiles: every cost-only evaluate,
points of more than 32 rows, and every row in the configurations without warp-tile evaluate).  Each problem here sets
the Huber parameter a to its median row norm at the initial state, so that every class of rows (points of <= 32,
33..128 and > 128 rows) has inliers and outliers and both branches run in both kernels; tests/test_oracle_lm_control.py
asserts that on a CPU machine.

  - every entry point (tests/entry_points.py) on the fixtures of tests/test_gpu_dispatch.py, C16 and the huge-point
    problem of tests/test_gpu_parity.py: evaluate with and without the Jacobian against the oracle (cost 1e-12, Jacobian
    1e-12), then every product and solve on the GPU's Jacobian and residuals, which the loss has corrected;
  - b200_set_apply_loss_function(0) against the trivial-loss oracle and (1) against Huber again, on the CTA-tile
    configurations (`id_range`, `tile`);
  - LM trajectories with Huber, device-resident and through the host-buffer boundary.
"""
import numpy as np
import pytest

from tests import lm_cases as L
from tests.entry_points import Case, check_every_entry_point, check_lm_trajectory, compare_lm_traces_exact, oracle_lm_traces, relerr
from tests.test_gpu_dispatch import EXPECT, LM_ITERATIONS, LM_MAX_CG

pytestmark = pytest.mark.gpu

PROBLEMS = sorted(EXPECT) + ["c16", "huge"]


def problem_bal(name, c16):
    from tests.test_gpu_dispatch import _bal
    from tests.test_gpu_parity import huge_bal
    if name == "c16":
        return L.c16_bal(c16)
    if name == "huge":
        return huge_bal()
    return _bal(name)


def trivial_oracle(oracle, bal):
    return oracle.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())


@pytest.fixture(scope="module")
def cs():
    import ceres_solver_b200 as m
    m.lib()
    return m


@pytest.fixture(scope="module")
def huber_cases(cs, oracle, c16):
    """name -> (Case with Huber(a), the trivial-loss oracle of the same problem), created on first use."""
    made = {}

    def get(name):
        if name not in made:
            bal = problem_bal(name, c16)
            from ceres_solver_b200 import bal as B
            orc0 = trivial_oracle(oracle, bal)
            state = B.ReducedProgram(bal).state(bal)
            a = L.huber_scale(orc0, state)
            for (lo, hi), (inliers, outliers) in L.huber_branches(orc0, state, a).items():
                assert inliers > 0 and outliers > 0, (name, lo, hi, inliers, outliers)
            made[name] = (Case(cs, oracle, bal, loss_type=cs.LOSS_HUBER, loss_a=a), orc0)
        return made[name]
    yield get
    for case, _ in made.values():
        case.close()


@pytest.mark.parametrize("name", PROBLEMS)
def test_every_entry_point(name, huber_cases, oracle):
    case, _ = huber_cases(name)
    check_every_entry_point(case, oracle, shared_inputs=True)


@pytest.mark.parametrize("name", ["id_range", "tile"])
def test_apply_loss_function(name, huber_cases):
    """Off: the trivial-loss oracle's cost, residuals, gradient and Jacobian (cost-only evaluate too).  On again: Huber's."""
    case, orc0 = huber_cases(name)
    gpu = case.gpu
    for apply, orc in ((False, orc0), (True, case.orc)):
        gpu.set_apply_loss_function(apply)
        ok, cost, res, grad = gpu.evaluate(case.state)
        ok_o, cost_o, res_o, grad_o = orc.evaluate(case.state, nt=8)
        assert ok and ok_o and abs(cost - cost_o) <= 1e-12 * cost_o, apply
        assert relerr(res, res_o) < 1e-12 and relerr(grad, grad_o) < 1e-10, apply
        assert relerr(gpu.jacobian_values(), orc.jacobian().values()) < 1e-12, apply
        ok, cost2, _, _ = gpu.evaluate(case.state, want_residuals=False, want_gradient=False, want_jacobian=False)
        assert ok and abs(cost2 - cost_o) <= 1e-12 * cost_o, apply
    ok0, cost0, _, _ = orc0.evaluate(case.state, want_gradient=False, want_jacobian=False, nt=8)
    assert ok0 and cost0 > cost_o   # the loss is on, and lowers the cost of the outliers


@pytest.mark.parametrize("host_boundary", [False, True])
def test_lm_trajectory_c16(host_boundary, cs, oracle, c16):
    """C16 with Huber(1.0) (bundle_adjuster --robustify), five iterations, every field of every record."""
    case = Case(cs, oracle, L.c16_bal(c16), loss_type=cs.LOSS_HUBER, loss_a=1.0)
    try:
        state_o, recs_o, _ = L.oracle_solve(case.orc, case.state, max_num_iterations=5)
        state, recs = L.gpu_solve(case.gpu, case.state, host_boundary, max_num_iterations=5)
        compare_lm_traces_exact(recs, recs_o)
        assert len(recs) == 6
        assert relerr(state, state_o) < 1e-9
    finally:
        case.close()


_traces = {}


@pytest.mark.parametrize("host_boundary", [False, True])
@pytest.mark.parametrize("name", ["id_range", "tile"])
def test_lm_trajectory(name, host_boundary, huber_cases):
    """The CTA-tile configurations with Huber(median row norm), as tests/test_gpu_dispatch.py runs them without."""
    case, _ = huber_cases(name)
    if name not in _traces:
        _traces[name] = oracle_lm_traces(case, LM_ITERATIONS, max_cg=LM_MAX_CG)
    check_lm_trajectory(case, _traces[name], LM_ITERATIONS, host_boundary, max_cg=LM_MAX_CG)
