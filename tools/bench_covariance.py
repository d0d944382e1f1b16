"""Cost of b200_covariance_compute and its getters on the synthetic BAL shapes of ceres_solver_b200.bal, with camera 0 and
1 % of the points (seeded, none seen by camera 0) constant.

For each workload and algorithm (sparse AMD, sparse NESDIS, dense): the wall time of one compute, split by the CUDA-event
stats of its launches (evaluate, assembly = schur_init + schur_diag_blocks + sparse_scatter, factor, selected inversion or
potri, points; the dense path's cuSOLVER potrf is not bracketed by the stats and is not split out); the wall time of the
getters (the C diagonal camera blocks and all points); and the wall time of one LM iteration of the same exact solver
under the same ordering, for scale.

    python tools/bench_covariance.py [--workloads ladybug-1723,venice-1778,trafalgar-257,ladybug-1723-random]
                                     [--algorithms amd,nesdis,dense]

One JSON line per (workload, algorithm) on stdout, each with the card's name and power limit.  Needs an H100; writes
nothing.
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True)
    except OSError:
        return "unknown"
    return out.stdout.strip().splitlines()[0] if out.returncode == 0 and out.stdout.strip() else "unknown"


def gauge(C, P, row_cam, row_pt):
    cam = np.zeros(C, dtype=bool)
    cam[0] = True
    seen = np.zeros(P, dtype=bool)
    seen[row_pt[row_cam == 0]] = True
    pts = np.zeros(P, dtype=bool)
    pts[np.random.RandomState(0).choice(np.flatnonzero(~seen), size=P // 100, replace=False)] = True
    return cam, pts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="ladybug-1723,venice-1778,trafalgar-257,ladybug-1723-random")
    ap.add_argument("--algorithms", default="amd,nesdis,dense")
    args = ap.parse_args()
    import ceres_solver_b200 as cs
    from ceres_solver_b200 import bal as B
    gpu_card = card()
    for name in args.workloads.split(","):
        bal = B.synthetic(name)
        rp = B.ReducedProgram(bal)
        state = rp.state(bal)
        row_cam, row_pt = np.asarray(rp.row_cam), np.asarray(rp.row_pt)
        cam, pts = gauge(rp.C, rp.P, row_cam, row_pt)
        for alg in args.algorithms.split(","):
            gpu = cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs)
            try:
                gpu.set_constant_blocks(cam, pts)
                algorithm = cs.DENSE_SCHUR if alg == "dense" else cs.SPARSE_SCHUR
                gpu.set_linear_solver_ordering_type(cs.NESDIS if alg == "nesdis" else cs.AMD)
                gpu.covariance_compute(state, algorithm=algorithm)   # warm-up: analysis, allocations, cuSOLVER
                gpu.stats_reset()
                gpu.profile(True)
                t0 = time.perf_counter()
                valid = gpu.covariance_compute(state, algorithm=algorithm)
                gpu.synchronize()
                wall = time.perf_counter() - t0
                st = gpu.stats()
                gpu.profile(False)
                ms = lambda *k: round(sum(st.get(x, {}).get("ms", 0.0) for x in k), 3)
                rec = dict(card=gpu_card, workload=name, algorithm=alg, valid=valid, compute_ms=round(1e3 * wall, 3),
                           evaluate_ms=ms("evaluate_jacobian"), assembly_ms=ms("schur_init", "schur_diag_blocks", "sparse_scatter"),
                           factor_ms=ms("sparse_factor") if alg != "dense" else "not measured",
                           inverse_ms=ms("selected_inversion"), points_ms=ms("covariance_points"))
                if valid:
                    pairs = [(i, i) for i in range(rp.C)]
                    t0 = time.perf_counter()
                    gpu.covariance_cameras(pairs)
                    gpu.covariance_points()
                    rec["getters_ms"] = round(1e3 * (time.perf_counter() - t0), 3)
                gpu.set_constant_blocks(cam, pts)
                t0 = time.perf_counter()
                gpu.lm_solve(state, gpu.lm_options(max_num_iterations=1, linear_solver_type=algorithm,
                                                   linear_solver_ordering_type=cs.NESDIS if alg == "nesdis" else cs.AMD))
                rec["lm_iteration_ms"] = round(1e3 * (time.perf_counter() - t0), 3)
            except Exception as e:   # a refusal (e.g. a cap) is a result too
                rec = dict(card=gpu_card, workload=name, algorithm=alg, error=str(e))
            finally:
                gpu.close()
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
