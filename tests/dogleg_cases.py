"""Option sets that drive the DOGLEG strategy down each of its branches, shared by the GPU tests (tests/test_gpu_dogleg.py)
and by their CPU guard on the reference alone (tests/test_oracle_dogleg.py), which fails if a change here stops a set from
taking the branches it is chosen for, or puts a decision within MARGIN of its threshold.
"""
MARGIN = 1e-4

OPTIONS = {
    # a small radius: the Cauchy point scaled to the region (traditional), the boundary minimum (subspace), then the
    # Gauss-Newton step once the radius has grown past it
    "small_radius": dict(initial_trust_region_radius=0.1, max_num_iterations=8),
    # a demanding min_relative_decrease: rejected steps in a row, each reusing the Gauss-Newton step at half the radius
    "rejections": dict(initial_trust_region_radius=10.0, min_relative_decrease=0.97, max_num_iterations=8),
}

# (problem, option set) pairs the GPU test runs
TRACES = [("tiny", "small_radius"), ("tiny", "rejections"), ("c16", "small_radius"), ("c16", "rejections")]

# every factorisation fails: `tiny` with camera 0's focal length 0 and no LM diagonal floor (tests/lm_cases.py)
INVALID = dict(min_lm_diagonal=0.0, max_num_iterations=5, max_num_consecutive_invalid_steps=5)
