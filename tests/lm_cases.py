"""Problems and option sets that drive the trust-region loop and the Huber loss down specific paths, shared by the GPU
tests (tests/test_gpu_lm_control.py, tests/test_gpu_robust_loss.py) and by their CPU guard on the oracle alone
(tests/test_oracle_lm_control.py), which fails if a change here stops a construction from doing what it is built for.

Every exit of the loop compares one value with one option.  Each threshold is placed from the oracle's own trace with
default options, between the value at the iteration where the exit is meant to fire and the values before it, at least
MARGIN (relative) away from all of them: summation-order differences between GPU and oracle are ~1e-10, so no exit can
move by an iteration.
"""
import math

import numpy as np

MARGIN = 1e-4

# b200_lm_options field names; the oracle's SolveOptions uses the same names except for the solver type
_ORACLE_NAME = {"linear_solver_type": "linear_solver"}

ITERATIVE_SCHUR, DENSE_SCHUR = 0, 1

# (problem, exit, iteration at which it fires): each exit on problems whose first iterations run short CG solves
EXITS = [
    ("tiny", "gradient_tolerance", 2),
    ("tiny", "function_tolerance", 3),
    ("tiny", "parameter_tolerance", 3),
    ("c16", "gradient_tolerance", 4),
    ("c16", "function_tolerance", 3),
    ("c16", "parameter_tolerance", 3),
    ("c16", "min_trust_region_radius", 5),   # at the end of the rejection chain of REJECTION
]

# C16 from a radius of 1e6 with min_relative_decrease 0.9: iteration 1 is accepted, 2..5 are rejected in a row (radius
# /2, /4, /8, /16), 6 is accepted, 7 is rejected again.  The step qualities are -4.5, -4.4, -3.6, -0.6, 0.97 and 0.75.
REJECTION = dict(min_relative_decrease=0.9, initial_trust_region_radius=1e6, max_num_iterations=7)
REJECTED_RUN = (2, 5)   # first and last iteration of the chain

# Every step invalid (tests/test_gpu_lm_control.py explains the construction): DENSE_SCHUR without the LM diagonal's
# floor, on `tiny` with the focal length of camera 0 set to 0.
INVALID = dict(linear_solver_type=DENSE_SCHUR, min_lm_diagonal=0.0, max_num_iterations=50)
# radius of record i: 1e4, then / 2, / 4, / 8, / 16 (exact in binary)
INVALID_RADII = (1e4, 5000.0, 1250.0, 156.25, 9.765625)


def tiny_bal():
    from ceres_solver_b200 import bal as B
    return B.synthetic("tiny")


def c16_bal(c16):
    from ceres_solver_b200 import bal as B
    return B.Bal(c16.cam_idx, c16.pt_idx, c16.obs, c16.cameras, c16.points)


def zero_focal_bal(camera=0):
    """`tiny` with camera `camera`'s focal length 0: 8 of its 9 Jacobian columns (all but d r / d f) are exactly zero.
    Every point of `tiny` is seen by at least two distinct cameras, so each point keeps a camera with f != 0."""
    from ceres_solver_b200 import bal as B
    bal = tiny_bal()
    cams = np.array(bal.cameras, dtype=float, copy=True)
    cams[camera, 6] = 0.0
    return B.Bal(bal.cam_idx, bal.pt_idx, bal.obs, cams, bal.points)


def oracle_solve(orc, state, nt=8, **options):
    o = orc.default_options()
    o.num_threads = nt
    for key, value in options.items():
        setattr(o, _ORACLE_NAME.get(key, key), value)
    return orc.solve(state, o)


def gpu_solve(gpu, state, host_boundary, **options):
    return gpu.lm_solve(state, gpu.lm_options(**options), host_boundary=host_boundary)


def threshold_between(fire, before):
    """Threshold t for an exit that fires once a value is <= t: `fire`, the value where it must fire, lies MARGIN below t
    and every value of `before` (where it must not) MARGIN above."""
    lo = min(before)
    t = math.sqrt(fire * lo)
    assert fire <= t * (1.0 - MARGIN) and lo >= t * (1.0 + MARGIN), (fire, before)
    return t


def exit_values(orc, state, recs, name, nt=8):
    """{iteration: value} of what the exit `name` compares with its option at each iteration of the oracle trace `recs`
    (trust_region_minimizer.cc: the gradient and radius tests on every record, :316-361; the parameter and function
    tolerances on every valid candidate, :726-769).  nt: the oracle's threads for the solves it runs."""
    if name == "gradient_tolerance":
        return {int(r["iteration"]): r["gradient_max_norm"] for r in recs if r["step_is_successful"]}
    if name == "min_trust_region_radius":
        return {int(r["iteration"]): r["tr_radius"] for r in recs}
    out = {}
    x_cost, accepted = recs[0]["cost"], False
    for r in recs[1:]:
        j = int(r["iteration"])
        if r["step_is_valid"]:
            if name == "function_tolerance":
                out[j] = abs(r["cost_change"]) / x_cost
            elif accepted:   # parameter_tolerance: |step| / |x|, tested once a step has been accepted
                x, _, _ = oracle_solve(orc, state, nt=nt, max_num_iterations=j - 1)   # x at iteration j (the best so far)
                out[j] = r["step_norm"] / np.linalg.norm(x)
        if r["step_is_successful"]:
            x_cost, accepted = r["cost"], True
    return out


def place_exit(orc, state, name, k, base=None, nt=8):
    """(options, number of records) of a solve on which exit `name` fires at iteration k: the threshold comes from the
    oracle's run with `base` options (default ones if None) and no exit before iteration k + 1.  The gradient and radius
    exits end the loop after record k is written, the parameter and function tolerances before it.  nt: the oracle's
    threads."""
    base = dict(base or {})
    base["max_num_iterations"] = k + 1
    _, recs, _ = oracle_solve(orc, state, nt=nt, **base)
    values = exit_values(orc, state, recs, name, nt)
    t = threshold_between(values[k], [v for j, v in values.items() if j < k])
    if name == "parameter_tolerance":
        # the test is |step| <= t (|x| + t): t^2 against t |x| moves the threshold by t / |x|, a tenth of MARGIN at most
        assert t < 0.1 * MARGIN * np.linalg.norm(state)
    base["max_num_iterations"] = k + 5
    base[name] = t
    return base, (k + 1 if name in ("gradient_tolerance", "min_trust_region_radius") else k)


def assert_decisions_have_margin(recs, min_relative_decrease):
    """Every accept / reject decision of a trace is at least MARGIN (relative) away from min_relative_decrease."""
    for r in recs[1:]:
        if r["step_is_valid"]:
            rho = r["tr_ratio"]
            assert abs(rho - min_relative_decrease) >= MARGIN * max(abs(rho), min_relative_decrease), r


def huber_scale(orc, state):
    """The Huber parameter a of a problem: the median row norm |(r0, r1)| at `state`, from the oracle's trivial-loss
    evaluate, so that about half the rows are inliers (s <= a^2) and half outliers."""
    ok, _, res, _ = orc.evaluate(state, want_gradient=False, want_jacobian=False, nt=8)
    assert ok
    return float(np.median(np.hypot(res[0::2], res[1::2])))


ROW_CLASSES = ((1, 32), (33, 128), (129, 1 << 30))   # rows per point: warp-tile evaluate, chunk tiles, huge points


def huber_branches(orc, state, a):
    """{(lo, hi): (inliers, outliers)} over the row classes present, by the degree of each row's point."""
    ok, _, res, _ = orc.evaluate(state, want_gradient=False, want_jacobian=False, nt=8)
    assert ok
    s = res[0::2] ** 2 + res[1::2] ** 2
    degree = np.bincount(orc.row_pt)[orc.row_pt]
    out = {}
    for lo, hi in ROW_CLASSES:
        rows = (degree >= lo) & (degree <= hi)
        if rows.any():
            out[(lo, hi)] = (int((s[rows] <= a * a).sum()), int((s[rows] > a * a).sum()))
    return out
