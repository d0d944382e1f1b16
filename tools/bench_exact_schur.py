"""The two exact LM-step solvers, DENSE_SCHUR (b200_dense_schur_solve: dense S, cuSOLVER Cholesky) and SPARSE_SCHUR
(b200_sparse_schur_solve: block-sparse S, supernodal Cholesky), on the same handle of each problem: time per solve from a host
clock around synchronised calls and from the CUDA-event stats of a profiled pass; b200_lm_solve with each solver type and each
trust-region strategy (LM, traditional and subspace DOGLEG): iterations per second, factorisations per iteration, the cost
after K iterations and the rejected steps; the symbolic statistics and the host analysis time, and the card's name and power
limit.

With --precision, the precision / refinement axis of the exact solves instead (b200_set_exact_solve_options and the matching
b200_lm_options fields): FP64, FP64 with 2 refinements, and mixed precision (float factorisation) with k = 0, 1 and 3, each with
SPARSE_SCHUR: the factor kernel's time and the solve's, its termination, b200_lm_solve's iterations per second over
--lm-iterations LM iterations, its factorisation FAILUREs (invalid steps) and rejected steps, and the cost reached relative
to FP64's.

With --ordering amd,nesdis, the linear_solver_ordering_type axis of SPARSE_SCHUR instead (b200_set_linear_solver_ordering_type
and b200_lm_options.linear_solver_ordering_type), --runs times with the orderings alternating on one handle: the plan's
statistics and host analysis time, the factor kernel's time and the solve's, LM and traditional DOGLEG iterations per second,
and |dx| / |x| against the AMD solve; DENSE_SCHUR's LM rate once per problem for comparison.

    python tools/bench_exact_schur.py [--reps 5] [--lm-iterations 5] [--problems ladybug-1723,...]
                                      [--strategies lm,traditional_dogleg,subspace_dogleg] [--precision]
                                      [--ordering amd,nesdis [--runs 3]] [--out results.json]

One JSON line per problem on stdout.  Needs an H100; nothing is written unless --out is given.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import ceres_solver_b200 as cs  # noqa: E402
from ceres_solver_b200 import bal as B  # noqa: E402

PROBLEMS = ["ladybug-1723", "venice-1778", "trafalgar-257", "ladybug-1723-random", "c16"]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def load(name):
    if name == "c16":
        return B.normalize(B.read_bal(os.path.join(ROOT, "tests", "golden", "problem-16-22106-pre.txt.bz2")))
    return B.synthetic(name)


def timed_solves(gpu, solve, b, D, reps):
    solve(b, D)   # warm-up (the sparse analysis runs at the first call)
    gpu.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        x, _, term = solve(b, D)
    ms = 1e3 * (time.perf_counter() - t) / reps
    gpu.stats_reset()
    gpu.profile(True)
    for _ in range(reps):
        solve(b, D)
    gpu.synchronize()
    gpu.profile(False)
    kernels = {k: round(v["ms"] / reps, 3) for k, v in gpu.stats().items() if v["launches"] > 0}
    return x, term, ms, kernels


# trust-region strategy axis: (name, trust_region_strategy_type, dogleg_type)
STRATEGIES = [("lm", cs.LEVENBERG_MARQUARDT, cs.TRADITIONAL_DOGLEG), ("traditional_dogleg", cs.DOGLEG, cs.TRADITIONAL_DOGLEG),
              ("subspace_dogleg", cs.DOGLEG, cs.SUBSPACE_DOGLEG)]


def lm_rate(gpu, state, solver_type, iterations, strategy=cs.LEVENBERG_MARQUARDT, dogleg_type=cs.TRADITIONAL_DOGLEG, **extra):
    """b200_lm_solve for `iterations` iterations: iterations per second, the cost reached, factorisations per iteration
    (launches of the dense assembly or of the sparse factor kernel: a rejected DOGLEG step reuses its factorisation, a
    rejected LM step does not) and the rejected and invalid steps of the run."""
    kw = dict(linear_solver_type=solver_type, trust_region_strategy_type=strategy, dogleg_type=dogleg_type, **extra)
    gpu.lm_solve(state, gpu.lm_options(max_num_iterations=1, **kw))   # warm-up
    gpu.synchronize()
    gpu.stats_reset()
    t = time.perf_counter()
    _, recs = gpu.lm_solve(state, gpu.lm_options(max_num_iterations=iterations, **kw))
    dt = time.perf_counter() - t
    its = len(recs) - 1
    factor = gpu.stats()["schur_diag_blocks" if solver_type == cs.DENSE_SCHUR else "sparse_factor"]["launches"]
    return dict(its_per_s=its / dt, cost=recs[-1]["cost"], iterations=its, factorisations_per_iteration=factor / max(its, 1),
                rejected=sum(1 for r in recs[1:] if r["step_is_valid"] and not r["step_is_successful"]),
                invalid=sum(1 for r in recs[1:] if not r["step_is_valid"]))


# precision / refinement axis: (name, use_mixed_precision_solves, max_num_refinement_iterations)
PRECISIONS = [("fp64", 0, 0), ("fp64_k2", 0, 2), ("mixed_k0", 1, 0), ("mixed_k1", 1, 1), ("mixed_k3", 1, 3)]


def precision_axis(gpu, state, res, D, reps, iterations):
    out = {}
    for name, mixed, k in PRECISIONS:   # every solve before any LM run: b200_lm_solve leaves its own Jacobian on the handle
        gpu.set_exact_solve_options(mixed, k)
        x, term, ms, kernels = timed_solves(gpu, gpu.sparse_schur_solve, res, D, reps)
        out[name] = dict(solve_ms=round(ms, 3), factor_ms=kernels.get("sparse_factor"), solve_only_ms=kernels.get("sparse_solve"),
                         termination=int(term), x=x)
    gpu.set_exact_solve_options(0, 0)
    for name, mixed, k in PRECISIONS:
        kw = dict(linear_solver_type=cs.SPARSE_SCHUR, use_mixed_precision_solves=mixed, max_num_refinement_iterations=k)
        gpu.lm_solve(state, gpu.lm_options(max_num_iterations=1, **kw))   # warm-up
        gpu.synchronize()
        t = time.perf_counter()
        _, recs = gpu.lm_solve(state, gpu.lm_options(max_num_iterations=iterations, **kw))
        dt = time.perf_counter() - t
        its = len(recs) - 1
        out[name].update(lm_its_per_s=its / dt, lm_iterations=its, lm_cost=recs[-1]["cost"],
                         lm_failures=sum(1 for r in recs[1:] if not r["step_is_valid"]),
                         lm_rejected=sum(1 for r in recs[1:] if r["step_is_valid"] and not r["step_is_successful"]))
    x64 = out["fp64"]["x"]
    for v in out.values():
        x = v.pop("x")
        v["relerr_vs_fp64"] = float(np.linalg.norm(x - x64) / np.linalg.norm(x64))
        v["lm_cost_vs_fp64"] = v["lm_cost"] / out["fp64"]["lm_cost"] - 1.0
    return out


ORDERINGS = {"amd": cs.AMD, "nesdis": cs.NESDIS}
ORDER_STATS = ("flops", "l_blocks", "supernodes", "tree_height", "critical_path_supernodes", "critical_path_flops",
               "factor_bytes", "order")


def ordering_axis(gpu, rp, state, res, D, names, runs, reps, iterations):
    """Per ordering: the statistics, then per run (orderings alternating) the analysis time, the factor and solve times, the
    LM and traditional DOGLEG rates with SPARSE_SCHUR and |dx| / |x| against the AMD solve of the same run."""
    out = {n: dict(runs=[]) for n in names}
    for n in names:
        _, st = cs.plan_sparse_schur(rp.C, rp.P, rp.row_cam, rp.row_pt, ORDERINGS[n])
        out[n].update({k: st[k] for k in ORDER_STATS})
    for run in range(runs):
        xs = {}
        for n in names:   # every solve of the run before its LM runs: b200_lm_solve leaves its own Jacobian on the handle
            t = time.perf_counter()
            cs.plan_sparse_schur(rp.C, rp.P, rp.row_cam, rp.row_pt, ORDERINGS[n])
            analysis_ms = 1e3 * (time.perf_counter() - t)
            gpu.set_linear_solver_ordering_type(ORDERINGS[n])
            x, term, ms, kernels = timed_solves(gpu, gpu.sparse_schur_solve, res, D, reps)
            xs[n] = x
            out[n]["runs"].append(dict(analysis_ms=round(analysis_ms, 2), solve_ms=round(ms, 3),
                                       factor_ms=kernels.get("sparse_factor"), termination=int(term)))
        for n in names:
            r = out[n]["runs"][-1]
            if "amd" in xs:
                r["relerr_vs_amd"] = float(np.linalg.norm(xs[n] - xs["amd"]) / np.linalg.norm(xs["amd"]))
            # the handle at the call's type: a b200_lm_solve call of another type would analyse again at each call
            gpu.set_linear_solver_ordering_type(ORDERINGS[n])
            lm = lm_rate(gpu, state, cs.SPARSE_SCHUR, iterations, linear_solver_ordering_type=ORDERINGS[n])
            dl = lm_rate(gpu, state, cs.SPARSE_SCHUR, iterations, cs.DOGLEG, cs.TRADITIONAL_DOGLEG,
                         linear_solver_ordering_type=ORDERINGS[n])
            r.update(lm_its_per_s=round(lm["its_per_s"], 2), lm_cost=lm["cost"],
                     dogleg_its_per_s=round(dl["its_per_s"], 2), dogleg_cost=dl["cost"])
    gpu.set_linear_solver_ordering_type(cs.AMD)
    for n in names:
        for key in ("analysis_ms", "solve_ms", "factor_ms", "lm_its_per_s", "dogleg_its_per_s"):
            v = [r[key] for r in out[n]["runs"] if r.get(key) is not None]
            if v:
                out[n][key] = dict(median=float(np.median(v)), min=min(v), max=max(v))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--lm-iterations", type=int, default=5)
    ap.add_argument("--problems", default=",".join(PROBLEMS))
    ap.add_argument("--strategies", default=",".join(n for n, _, _ in STRATEGIES))
    ap.add_argument("--precision", action="store_true")
    ap.add_argument("--ordering", default=None)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    device = card()
    results = []
    for name in a.problems.split(","):
        bal = load(name)
        rp = B.ReducedProgram(bal)
        state = rp.state(bal)
        t = time.perf_counter()
        _, st = cs.plan_sparse_schur(rp.C, rp.P, rp.row_cam, rp.row_pt)
        analysis_ms = 1e3 * (time.perf_counter() - t)
        gpu = cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs)
        ok, _, res, _ = gpu.evaluate(state)
        assert ok
        s = 1.0 / (1.0 + np.sqrt(gpu.squared_column_norm()))
        gpu.scale_columns(s)
        D = np.sqrt(np.clip(gpu.squared_column_norm(), 1e-6, 1e32) / 1e4)
        row = dict(problem=name, device=device, C=rp.C, P=rp.P, N=rp.N, analysis_ms=round(analysis_ms, 2), **st)
        if a.ordering:
            row["ordering"] = ordering_axis(gpu, rp, state, res, D, a.ordering.split(","), a.runs, a.reps, a.lm_iterations)
            row["lm_its_per_s_dense"] = round(lm_rate(gpu, state, cs.DENSE_SCHUR, a.lm_iterations)["its_per_s"], 2)
            gpu.close()
            print(json.dumps(row), flush=True)
            results.append(row)
            continue
        if a.precision:
            row["precision"] = precision_axis(gpu, state, res, D, a.reps, a.lm_iterations)
            gpu.close()
            print(json.dumps(row), flush=True)
            results.append(row)
            continue
        xs, ts, row["sparse_ms"], row["sparse_kernels_ms"] = timed_solves(gpu, gpu.sparse_schur_solve, res, D, a.reps)
        xd, td, row["dense_ms"], row["dense_kernels_ms"] = timed_solves(gpu, gpu.dense_schur_solve, res, D, a.reps)
        row["terminations"] = [int(ts), int(td)]
        row["relerr_sparse_dense"] = float(np.linalg.norm(xs - xd) / np.linalg.norm(xd))
        for sname, solver in (("sparse", cs.SPARSE_SCHUR), ("dense", cs.DENSE_SCHUR)):
            for name_s, strategy, dogleg_type in STRATEGIES:
                if name_s not in a.strategies.split(","):
                    continue
                rate = lm_rate(gpu, state, solver, a.lm_iterations, strategy, dogleg_type)
                if name_s == "lm":
                    row["lm_its_per_s_" + sname], row["lm_cost_" + sname] = rate["its_per_s"], rate["cost"]
                row.setdefault("strategies", {})["%s/%s" % (name_s, sname)] = rate
        gpu.close()
        print(json.dumps(row), flush=True)
        results.append(row)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
