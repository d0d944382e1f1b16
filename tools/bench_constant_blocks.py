"""Cost of constant parameter blocks (b200_set_constant_blocks) on the device, on Ladybug-1723 (the synthetic video
sequence of ceres_solver_b200.bal).

For each setup: the evaluate kernels' device time per evaluation with the Jacobian (CUDA-event stats, profiling on, in a
pass of its own), the wall time of one ITERATIVE_SCHUR solve on the resident residuals (default options, D = 1e-2), and
b200_lm_solve's iterations per second (device-resident, ITERATIVE_SCHUR, profiling off).  Setups: nothing constant, also
with the library of another build (--baseline-lib, e.g. the parent commit's) in the same call, the two libraries
alternating run by run so that both see the same machine, and their costs compared to the last bit; then camera 0
constant (the gauge), and camera 0 plus 1 % of the points (seeded, none seen by camera 0) constant.

    python tools/bench_constant_blocks.py [--baseline-lib build/parent/libb200ba.so] [--runs 3] [--reps 20]
                                          [--lm-iterations 10] [--out results.json]

One JSON line per (run, library, setup) and a summary line (medians and run-to-run spread) on stdout, each with the
card's name and power limit.  Needs an H100; nothing is written unless --out is given.
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

BASE_SETUPS = ("none",)
NEW_SETUPS = ("camera0", "camera0_points1pct")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True)
    except OSError:
        return "unknown"
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def constant_of(setup, C, P, row_cam, row_pt):
    """(camera_constant, point_constant) of a setup."""
    if setup == "none":
        return None, None
    cam = np.zeros(C, dtype=bool)
    cam[0] = True
    if setup == "camera0":
        return cam, None
    seen = np.zeros(P, dtype=bool)
    seen[row_pt[row_cam == 0]] = True
    free = np.flatnonzero(~seen)
    pts = np.zeros(P, dtype=bool)
    pts[np.random.RandomState(0).choice(free, size=P // 100, replace=False)] = True
    return cam, pts


def worker(problem_path, setups, reps, lm_iterations):
    """One library (the B200BA_LIB the process was started with): every setup on the problem saved at problem_path."""
    import ceres_solver_b200 as cs
    d = np.load(problem_path)
    C, P, row_cam, row_pt, row_obs, state = (int(d["C"]), int(d["P"]), d["row_cam"], d["row_pt"], d["row_obs"], d["state"])
    out = []
    for setup in setups:
        gpu = cs.Problem(C, P, row_cam, row_pt, row_obs)
        cam, pts = constant_of(setup, C, P, row_cam, row_pt)
        if cam is not None:
            gpu.set_constant_blocks(cam, pts)
        ok, cost, _, _ = gpu.evaluate(state, want_residuals=False, want_gradient=False, want_jacobian=False)
        assert ok
        for _ in range(3):
            gpu.evaluate(state, want_residuals=False, want_gradient=True, want_jacobian=True)
        gpu.synchronize()
        gpu.stats_reset()
        gpu.profile(True)
        for _ in range(reps):
            gpu.evaluate(state, want_residuals=False, want_gradient=True, want_jacobian=True)
            gpu.evaluate(state, want_residuals=False, want_gradient=False, want_jacobian=False)
        gpu.synchronize()
        st = gpu.stats()
        gpu.profile(False)
        eval_jac = st["evaluate_jacobian"]["ms"] / reps
        eval_cost = st["evaluate_cost"]["ms"] / reps
        gpu.evaluate(state)
        D = np.full(gpu.num_parameters, 1e-2)
        gpu.schur_solve(None, D)   # warm-up
        gpu.synchronize()
        t = time.perf_counter()
        for _ in range(reps):
            gpu.schur_solve(None, D)
        gpu.synchronize()
        solve_ms = (time.perf_counter() - t) * 1e3 / reps
        o = gpu.lm_options(max_num_iterations=1)
        gpu.lm_solve(state, o)   # warm-up
        o = gpu.lm_options(max_num_iterations=lm_iterations)
        gpu.synchronize()
        t = time.perf_counter()
        _, recs = gpu.lm_solve(state, o)
        dt = time.perf_counter() - t
        out.append(dict(setup=setup, cost=float(cost).hex(), eval_jacobian_ms=round(eval_jac, 4),
                        eval_cost_ms=round(eval_cost, 4), solve_ms=round(solve_ms, 3), lm_it_per_s=round((len(recs) - 1) / dt, 3),
                        lm_final_cost=recs[-1]["cost"], lm_iterations=len(recs) - 1))
        gpu.close()
    print("WORKER " + json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--baseline-lib", default=None, help="libb200ba.so of another build, measured alternately")
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
    from ceres_solver_b200.binding import LIB_PATH
    bal = B.synthetic("ladybug-1723")
    rp = B.ReducedProgram(bal)
    state = rp.state(bal)
    name = card()
    libs = [("this", LIB_PATH)] + ([("baseline", os.path.abspath(args.baseline_lib))] if args.baseline_lib else [])
    results = []
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "ladybug-1723.npz")
        np.savez(path, C=rp.C, P=rp.P, row_cam=rp.row_cam, row_pt=rp.row_pt, row_obs=rp.row_obs, state=state)
        for run in range(args.runs):
            order = libs if run % 2 == 0 else libs[::-1]
            for label, lib in order:
                setups = BASE_SETUPS + (NEW_SETUPS if label == "this" else ())
                env = dict(os.environ, B200BA_LIB=lib)
                cmd = [sys.executable, os.path.abspath(__file__), "--worker", path, ",".join(setups), str(args.reps),
                       str(args.lm_iterations)]
                r = subprocess.run(cmd, capture_output=True, text=True, env=env, cwd=ROOT)
                lines = [ln for ln in r.stdout.splitlines() if ln.startswith("WORKER ")]
                if r.returncode != 0 or not lines:
                    sys.stderr.write(r.stdout[-2000:] + r.stderr[-4000:])
                    raise SystemExit("worker for %s failed" % label)
                for rec in json.loads(lines[0][len("WORKER "):]):
                    rec.update(run=run, library=label, card=name, problem="ladybug-1723")
                    results.append(rec)
                    print(json.dumps(rec), flush=True)
    summary = dict(card=name, problem="ladybug-1723", rows=int(rp.N), setups={})
    for label, _ in libs:
        for setup in BASE_SETUPS + NEW_SETUPS:
            recs = [r for r in results if r["library"] == label and r["setup"] == setup]
            if not recs:
                continue
            entry = {}
            for key in ("eval_jacobian_ms", "eval_cost_ms", "solve_ms", "lm_it_per_s"):
                v = [r[key] for r in recs]
                entry[key] = dict(median=float(np.median(v)), min=min(v), max=max(v))
            entry["costs"] = sorted({r["cost"] for r in recs})
            entry["lm_final_cost"] = dict(min=min(r["lm_final_cost"] for r in recs), max=max(r["lm_final_cost"] for r in recs))
            summary["setups"]["%s/%s" % (label, setup)] = entry
    if args.baseline_lib:
        # (the evaluate's cost is reproducible to the bit; the LM's final cost is not even between runs of one build: the
        # PCG sums with atomics)
        summary["same_cost_bits"] = {setup: summary["setups"]["this/" + setup]["costs"] == summary["setups"]["baseline/" + setup]["costs"]
                                     for setup in BASE_SETUPS}
    print("SUMMARY " + json.dumps(summary), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(results=results, summary=summary), f, indent=1)


if __name__ == "__main__":
    main()
