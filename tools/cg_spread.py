"""Spread of the inexact Schur solve under rounding, implicit against explicit S (DESIGN §3.4, §3.2).

Solves the reduced system of the fourth LM iteration of a benchmark workload (the first solve that runs for ~300 CG
iterations on Ladybug-1723) repeatedly from IDENTICAL inputs, once with the implicit product and once with the explicit
S, and prints the CG iteration counts and how far the solutions lie from the first implicit one.  The only differences
between repeats of one operator are the summation orders of the reductions; what the two operators show against each
other should be no more than what each shows against itself.  Needs the development build (tools/build_dev.sh), which
honours B200_EXPLICIT_S:

    B200BA_LIB=ceres_solver_b200/libb200ba_dev.so python tools/cg_spread.py [workload] [repeats]
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import ceres_solver_b200 as cs  # noqa: E402
from ceres_solver_b200 import bal as B  # noqa: E402

workload = sys.argv[1] if len(sys.argv) > 1 else "ladybug-1723"
repeats = int(sys.argv[2]) if len(sys.argv) > 2 else 30
bal = B.synthetic(workload)
rp = B.ReducedProgram(bal)
state = rp.state(bal)
handles = {}
for name, flag in (("implicit", "0"), ("explicit", "1")):
    os.environ["B200_EXPLICIT_S"] = flag
    handles[name] = cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs)
os.environ.pop("B200_EXPLICIT_S")
# the state and trust region radius the fourth LM iteration starts from
state3, recs = handles["implicit"].lm_solve(state, handles["implicit"].lm_options(max_num_iterations=3))
radius = recs[-1]["tr_radius"]
scale = D = res0 = None
results = {}
for name, gpu in handles.items():
    ok, _, res, _ = gpu.evaluate(state3)
    assert ok
    if scale is None:   # Jacobi scaling and LM diagonal as the solver forms them
        scale = 1.0 / (1.0 + np.sqrt(gpu.squared_column_norm()))
        gpu.scale_columns(scale)
        D = np.sqrt(np.clip(gpu.squared_column_norm(), 1e-6, 1e32) / radius)
        res0 = res
    else:
        gpu.scale_columns(scale)
    assert np.array_equal(res, res0)
    opts = gpu.solver_options(preconditioner_type=2, q_tolerance=1e-2, r_tolerance=-1.0, max_num_iterations=500)
    results[name] = [gpu.schur_solve(res, D, opts)[:2] for _ in range(repeats)]
ref = results["implicit"][0][0]
for name, runs in results.items():
    err = [np.linalg.norm(x - ref) / np.linalg.norm(ref) for x, _ in runs]
    print("%s: CG iterations %s; solution vs the first implicit one: median %.1e, max %.1e"
          % (name, sorted(its for _, its in runs), np.median(err), np.max(err)))
for gpu in handles.values():
    gpu.close()
