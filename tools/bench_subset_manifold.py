"""Cost of SubsetManifolds (b200_set_subset_manifolds) on the device, on Ladybug-1723 (the synthetic video sequence of
ceres_solver_b200.bal).

For each setup: the evaluate kernels' device time per evaluation with the Jacobian (CUDA-event stats, profiling on, in a
pass of its own), and b200_lm_solve's iterations per second (device-resident, profiling off) with ITERATIVE_SCHUR and
with SPARSE_SCHUR under NESDIS.  Setups: nothing constant; camera 0 and 1 % of the points constant (blocks); focal length
and distortion held on every camera, SubsetManifold(9, {6, 7, 8}); and mixed masks (a seeded random non-empty, non-full
subset on every camera, one or two coordinates on 10 % of the points).  S keeps its 9 x 9 camera blocks, so the exact
solves are expected to cost what they cost without masks.

    python tools/bench_subset_manifold.py [--runs 3] [--reps 20] [--lm-iterations 10] [--out results.json]

One JSON line per (run, setup) and a summary line (medians and run-to-run spread) on stdout, each with the card's name and
power limit.  Needs an H100; nothing is written unless --out is given.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SETUPS = ("none", "constant_blocks", "intrinsics", "mixed")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True)
    except OSError:
        return "unknown"
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def setup_of(setup, C, P, row_cam, row_pt):
    """(camera_constant, point_constant, camera_mask, point_mask) of a setup."""
    rng = np.random.RandomState(0)
    if setup == "none":
        return None, None, None, None
    if setup == "constant_blocks":
        cam = np.zeros(C, dtype=bool)
        cam[0] = True
        seen = np.zeros(P, dtype=bool)
        seen[row_pt[row_cam == 0]] = True
        pts = np.zeros(P, dtype=bool)
        pts[rng.choice(np.flatnonzero(~seen), size=P // 100, replace=False)] = True
        return cam, pts, None, None
    cm = np.zeros((C, 9), dtype=bool)
    if setup == "intrinsics":
        cm[:, 6:] = True
        return None, None, cm, None
    for c in range(C):
        cm[c, rng.choice(9, size=rng.randint(1, 9), replace=False)] = True
    pm = np.zeros((P, 3), dtype=bool)
    for p in rng.choice(P, size=P // 10, replace=False):
        pm[p, rng.choice(3, size=rng.randint(1, 3), replace=False)] = True
    return None, None, cm, pm


def lm_rate(cs, gpu, state, lm_iterations, **kw):
    gpu.lm_solve(state, gpu.lm_options(max_num_iterations=1, **kw))   # warm-up (and the sparse analysis)
    gpu.synchronize()
    t = time.perf_counter()
    _, recs = gpu.lm_solve(state, gpu.lm_options(max_num_iterations=lm_iterations, **kw))
    dt = time.perf_counter() - t
    return round((len(recs) - 1) / dt, 3), recs[-1]["cost"]


def worker(problem_path, setups, reps, lm_iterations):
    import ceres_solver_b200 as cs
    d = np.load(problem_path)
    C, P, row_cam, row_pt, row_obs, state = (int(d["C"]), int(d["P"]), d["row_cam"], d["row_pt"], d["row_obs"], d["state"])
    out = []
    for setup in setups:
        gpu = cs.Problem(C, P, row_cam, row_pt, row_obs)
        cam, pts, cm, pm = setup_of(setup, C, P, row_cam, row_pt)
        gpu.set_constant_blocks(cam, pts)
        gpu.set_subset_manifolds(cm, pm)
        ok, cost, _, _ = gpu.evaluate(state, want_residuals=False, want_gradient=False, want_jacobian=False)
        assert ok
        for _ in range(3):
            gpu.evaluate(state, want_residuals=False, want_gradient=True, want_jacobian=True)
        gpu.synchronize()
        gpu.stats_reset()
        gpu.profile(True)
        for _ in range(reps):
            gpu.evaluate(state, want_residuals=False, want_gradient=True, want_jacobian=True)
        gpu.synchronize()
        st = gpu.stats()
        gpu.profile(False)
        eval_jac = st["evaluate_jacobian"]["ms"] / reps
        it_iter, cost_iter = lm_rate(cs, gpu, state, lm_iterations)
        gpu.set_linear_solver_ordering_type(cs.NESDIS)
        it_sparse, cost_sparse = lm_rate(cs, gpu, state, lm_iterations, linear_solver_type=cs.SPARSE_SCHUR,
                                         linear_solver_ordering_type=cs.NESDIS)
        out.append(dict(setup=setup, cost=float(cost).hex(), eval_jacobian_ms=round(eval_jac, 4),
                        lm_iterative_it_per_s=it_iter, lm_sparse_nesdis_it_per_s=it_sparse,
                        lm_iterative_final_cost=cost_iter, lm_sparse_final_cost=cost_sparse))
        gpu.close()
    print("WORKER " + json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--lm-iterations", type=int, default=10)
    ap.add_argument("--out", default=None)
    ap.add_argument("--worker", nargs=4, default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        path, setups, reps, its = args.worker
        worker(path, setups.split(","), int(reps), int(its))
        return
    from ceres_solver_b200 import bal as B
    bal = B.synthetic("ladybug-1723")
    rp = B.ReducedProgram(bal)
    state = rp.state(bal)
    name = card()
    results = []
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "ladybug-1723.npz")
        np.savez(path, C=rp.C, P=rp.P, row_cam=rp.row_cam, row_pt=rp.row_pt, row_obs=rp.row_obs, state=state)
        for run in range(args.runs):
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", path, ",".join(SETUPS), str(args.reps),
                   str(args.lm_iterations)]
            r = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT)
            lines = [ln for ln in r.stdout.splitlines() if ln.startswith("WORKER ")]
            if r.returncode != 0 or not lines:
                sys.stderr.write(r.stdout[-2000:] + r.stderr[-4000:])
                raise SystemExit("worker failed")
            for rec in json.loads(lines[0][len("WORKER "):]):
                rec.update(run=run, card=name, problem="ladybug-1723")
                results.append(rec)
                print(json.dumps(rec), flush=True)
    summary = dict(card=name, problem="ladybug-1723", rows=int(rp.N), setups={})
    for setup in SETUPS:
        recs = [r for r in results if r["setup"] == setup]
        entry = {}
        for key in ("eval_jacobian_ms", "lm_iterative_it_per_s", "lm_sparse_nesdis_it_per_s"):
            v = [r[key] for r in recs]
            entry[key] = dict(median=float(np.median(v)), min=min(v), max=max(v))
        summary["setups"][setup] = entry
    print("SUMMARY " + json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(results=results, summary=summary), f, indent=1)


if __name__ == "__main__":
    main()
