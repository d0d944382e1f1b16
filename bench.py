#!/usr/bin/env python
"""bench.py — LM iterations/sec of the ITERATIVE_SCHUR + SCHUR_JACOBI bundle-adjustment hot path.

  python bench.py --gpus N --steps K --warmup W [--workload NAME] [--impl b200|reference] [--dump-outputs DIR]

A "step" is one Levenberg-Marquardt iteration (ComputeTrustRegionStep: LM diagonal, implicit-Schur PCG solve,
model cost; candidate cost evaluation; on acceptance a Jacobian evaluation + column scaling) of the configuration
BASELINE.json names: bundle_adjuster defaults (eta 1e-2, <=500 CG iterations, SCHUR_JACOBI, Jacobi scaling, user
ordering, no robust loss) on a BAL problem.  K steps are timed from the problem's initial point after W warm-up
steps on the same problem (the state is reset in between, so every timed run does identical work).

  value      K / device time of the device-resident loop (inputs already in HBM)
  e2e        the same K iterations driven through the host-buffer C ABI the Ceres adapters use
             (state/D/residual/step copies inside the timed region)
  roofline   dominant kernel: algorithmic bytes per launch / mean CUDA-event time per launch, vs measured HBM peak
  cpu_baseline / --impl reference: the CPU restatement of the reference path (oracle/) on the host cores

--dump-outputs DIR writes what the timed run returned to its caller as DIR/<name>.npy (float64): the final state
(points then cameras, reduced-program order; rank 0's shard when sharded) and the per-iteration trace, so that two
builds can be compared output for output on identical seeded inputs.  For spmv-sweep: the products of the largest size.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

DUMP_BYTES = 60_000_000   # --dump-outputs budget over all arrays


def dump_outputs(path, arrays):
    """Writes every array as path/<name>.npy in float64.  When they exceed DUMP_BYTES together, each array larger than
    an equal share is replaced by a fixed sample of that share (indices from RandomState(0), sorted), the same for every
    build and run."""
    os.makedirs(path, exist_ok=True)
    arrays = {k: np.ascontiguousarray(v, dtype=np.float64).ravel() for k, v in arrays.items()}
    share = DUMP_BYTES // (8 * len(arrays))
    sample = 8 * sum(a.size for a in arrays.values()) > DUMP_BYTES
    for name, a in arrays.items():
        if sample and a.size > share:
            a = a[np.sort(np.random.RandomState(0).randint(0, a.size, share))]
        np.save(os.path.join(path, name + ".npy"), a)


def trace_arrays(recs):
    return {k: np.array([float(r[k]) for r in recs]) for k in ("cost", "step_norm", "gradient_max_norm", "ls_iterations")}


def op_rate(v, peak):
    """GB/s of an operation class: bytes of ONE operation x operations / event time of ALL its launches."""
    if not v or v.get("ms", 0) <= 0 or v.get("operations", 0) <= 0 or v.get("bytes_per_operation", 0) <= 0:
        return None
    gbps = v["bytes_per_operation"] * v["operations"] / (v["ms"] * 1e-3) / 1e9
    return {"GBps": round(gbps, 1), "frac": round(gbps / peak, 4), "operations": v["operations"],
            "launches": v["launches"], "mean_op_ms": round(v["ms"] / v["operations"], 5),
            "bytes_per_operation": v["bytes_per_operation"]}

METRIC = "lm_iterations_per_sec"
UNIT = "LM iterations/s"


def load_peaks():
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            p = json.load(f)
        return float(p["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
    except Exception:
        return 3350.0, "H100 SXM data sheet (HBM3 3.35 TB/s)"


def make_problem(workload):
    from ceres_solver_b200 import bal as B
    if workload == "c16":
        path = os.path.join(ROOT, "tests", "golden", "problem-16-22106-pre.txt.bz2")
        bal = B.normalize(B.read_bal(path))
        desc = "BAL problem-16-22106-pre (real, Normalize()d): 16 cameras / 22106 points / 83718 observations"
    else:
        bal = B.synthetic(workload)
        desc = "synthetic-regen %s: %d cameras / %d points / %d observations (seed 38401)" % (
            workload, bal.C, bal.P, bal.N)
    return bal, desc


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled during the timed region."""

    def __init__(self, device=0):
        self.device = device
        self.rows = []
        self.proc = None

    def start(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.device), "--query-gpu=" + q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        time.sleep(0.15)
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            try:
                sm.append(float(r[0]))
                mx.append(float(r[1]))
                for n, v in zip(names, r[3:7]):
                    if v.lower().startswith("active"):
                        reasons.add(n)
            except Exception:
                pass
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None,
                "reasons": sorted(reasons), "samples": len(sm)}


def make_config(desc, num_obs):
    """The workload description both arms print (identical dicts: the driver compares them)."""
    jb = 192 * num_obs
    return {"workload": desc, "linear_solver": "ITERATIVE_SCHUR", "preconditioner": "SCHUR_JACOBI", "eta": 1e-2,
            "max_linear_solver_iterations": 500, "jacobian_bytes": jb,
            "l2": "inputs larger than L2 (J alone is %.0f MB)" % (jb / 1e6) if jb > 50e6
            else "working set fits L2: roofline fraction is vs HBM peak and may exceed 1"}


def run_reference(args, bal, desc, rank0=True):
    """The reference's own CPU path (restated in oracle/: the real Ceres cannot be built in this image — Eigen is
    absent) on all host threads, same problem, same options."""
    from oracle import pyoracle as po
    nt = po.max_threads()
    prog = po.BaProgram(bal.C, bal.P, bal.cam_idx, bal.pt_idx, np.ascontiguousarray(bal.obs).ravel())
    state = prog.state_from_parameters(np.ascontiguousarray(bal.cameras).ravel(), np.ascontiguousarray(bal.points).ravel())
    o = prog.default_options()
    o.num_threads = nt
    o.max_num_iterations = args.steps
    if args.warmup > 0:  # touch memory / spin up the thread pool
        ow = prog.default_options()
        ow.num_threads = nt
        ow.max_num_iterations = 1
        prog.solve(state, ow)
    t0 = time.perf_counter()
    state_out, recs, times = prog.solve(state, o, max_records=args.steps + 1)
    dt = time.perf_counter() - t0
    iters = max(1, len(recs) - 1)
    return {"value": iters / dt, "seconds": dt, "iterations": iters, "cores": nt, "trace": recs, "times": times,
            "state": state_out}


def run_spmv_sweep(args):
    """BASELINE.json configs[4] / SURVEY 8d I4: synthetic block-SpMV sweep, N residual blocks of shape (2x3 + 2x9), P = N/4
    points, C = max(16, N/400) cameras, rows point-sorted, cameras uniform random, values and x ~ N(0,1) from MT19937 with
    its default seed (the set-up of the reference's own spmv_benchmark.cc:70-80 / evaluation_benchmark.cc:147-153).  Per size:
    the 2x3-only products (E x, E'y), the 2x9-only ones (F x, F'y), both shapes (J x, J'y) and (J'J + D^2) x in one pass, as
    GB/s of algorithmic bytes over CUDA-event kernel time and as a fraction of the measured HBM peak."""
    import torch
    import ceres_solver_b200 as cs
    peak, peak_src = load_peaks()
    sizes = [int(float(v)) for v in (args.sizes.split(",") if args.sizes else ["1e5", "3e5", "1e6", "3e6", "1e7", "3e7"])]
    rows = []
    names = {"pmv_right_e": "E x (2x3)", "pmv_left_e": "E'y (2x3)", "pmv_right_f": "F x (2x9)", "pmv_left_f": "F'y (2x9)",
             "jacobian_multiply": "J x (both)", "jacobian_t_multiply": "J'y (both)", "jtj_multiply": "(J'J + D^2) x"}
    for N in sizes:
        N -= N % 4
        P, C = N // 4, max(16, N // 400)
        rng = np.random.RandomState(5489)
        pt = np.repeat(np.arange(P, dtype=np.int32), 4)
        base = rng.randint(0, C, P).astype(np.int64)
        step = rng.randint(1, max(2, C // 4), P).astype(np.int64)
        cam = ((base[:, None] + step[:, None] * np.arange(4)[None, :]) % C).astype(np.int32).ravel()   # 4 distinct cameras
        gpu = cs.Problem(C, P, cam, pt, np.zeros(2 * N))
        vals = rng.standard_normal(24 * N)
        gpu.set_jacobian_values(vals)
        del vals
        x = rng.standard_normal(gpu.num_parameters)
        D = np.abs(rng.standard_normal(gpu.num_parameters)) + 0.1
        y = rng.standard_normal(gpu.num_residuals)
        reps = 5 if N <= 3_000_000 else 2

        def ops():
            return {"pmv_right_e": gpu.partitioned_multiply(0, x[:3 * P]), "pmv_left_e": gpu.partitioned_multiply(2, y),
                    "pmv_right_f": gpu.partitioned_multiply(1, x[3 * P:]), "pmv_left_f": gpu.partitioned_multiply(3, y),
                    "jacobian_multiply": gpu.right_multiply(x), "jacobian_t_multiply": gpu.left_multiply(y),
                    "jtj_multiply": gpu.jtj_multiply(x, D)}
        ops()   # warm-up
        gpu.stats_reset()
        gpu.profile(True)
        for _ in range(reps):
            out = ops()
        st = gpu.stats()
        gpu.profile(False)
        row = {"N": N, "P": P, "C": C, "jacobian_bytes": 192 * N, "ops": {}}
        for k, label in names.items():
            r = op_rate(st.get(k), peak)
            if r:
                row["ops"][label] = {"GBps": r["GBps"], "frac": r["frac"], "mean_op_ms": r["mean_op_ms"]}
        rows.append(row)
        if args.dump_outputs and N == sizes[-1] - sizes[-1] % 4:
            dump_outputs(args.dump_outputs, out)
        del out
        gpu.close()
        torch.cuda.empty_cache()
    last = rows[-1]["ops"].get("(J'J + D^2) x", {})
    line = {"metric": "block_spmv_GBps", "value": last.get("GBps"), "unit": "GB/s", "n_gpus": 1, "higher_is_better": True,
            "dtype": "f64", "data": "synthetic", "config": {"workload": "spmv-sweep: N residual blocks (2x3 + 2x9), P = N/4, "
            "C = max(16, N/400), point-sorted rows, uniform random cameras, values ~ N(0,1) MT19937(5489)"},
            "peak": peak, "peak_source": peak_src, "sweep": rows}
    print(json.dumps(line))
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--workload", default=None)
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--sizes", default=None, help="spmv-sweep: comma separated N list (default 1e5..3e7; 1e8 needs ~60 GB host RAM)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the outputs of the last timed run as DIR/<name>.npy (float64, <= 60 MB in all)")
    args = ap.parse_args()
    if args.steps < 1 or args.warmup < 0:
        ap.error("--steps must be >= 1 and --warmup >= 0")

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if os.environ.get("NCCL_DEBUG", "").upper() in ("", "VERSION"):
        os.environ["NCCL_DEBUG"] = "WARN"  # keep stdout to the one JSON line (NCCL prints its version banner there)
    workload = args.workload or "ladybug-1723"
    if workload == "spmv-sweep":
        return run_spmv_sweep(args) if rank == 0 and args.impl == "b200" else 0

    if args.impl == "reference":
        if rank != 0:
            return 0
        bal, desc = make_problem(workload)
        r = run_reference(args, bal, desc)
        line = {"impl": "reference", "metric": METRIC, "value": r["value"], "unit": UNIT, "n_gpus": args.gpus,
                "steps": r["iterations"], "warmup": args.warmup, "ms_per_step": 1e3 * r["seconds"] / r["iterations"],
                "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f64",
                "data": "synthetic" if workload != "c16" else "real BAL file shipped with the reference",
                "config": make_config(desc, bal.N),
                "cg_iterations": [int(t["ls_iterations"]) for t in r["trace"][1:]],
                "costs": [float(t["cost"]) for t in r["trace"]], "final_cost": float(r["trace"][-1]["cost"]),
                "step_norms": [float(t["step_norm"]) for t in r["trace"]],
                "cpu_baseline": {"value": r["value"], "unit": UNIT, "cores": r["cores"], "kind": "port",
                                 "sample": "%d LM iterations from the initial point, %d CG iterations" % (
                                     r["iterations"], sum(int(t["ls_iterations"]) for t in r["trace"]))},
                "e2e": {"value": r["value"], "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}}
        if args.dump_outputs:
            dump_outputs(args.dump_outputs, dict(state=r["state"], **trace_arrays(r["trace"])))
        print(json.dumps(line))
        return 0

    import torch
    import torch.distributed as dist
    import ceres_solver_b200 as cs
    from ceres_solver_b200 import bal as B

    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local_rank)
    nccl_id = None
    if world > 1:
        dist.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
        # the library runs its own communicator (one all-reduce of the camera-sized vector per CG iteration);
        # torch.distributed is only the plumbing that hands the NCCL id to every rank and synchronises the timing
        idt = torch.zeros(128, dtype=torch.uint8, device="cuda")
        if rank == 0:
            idt.copy_(torch.frombuffer(bytearray(cs.nccl_unique_id()), dtype=torch.uint8))
        dist.broadcast(idt, 0)
        nccl_id = bytes(idt.cpu().numpy().tobytes())

    bal, desc = make_problem(workload)
    rp = B.ReducedProgram(bal)
    full_state = rp.state(bal)
    stream = torch.cuda.current_stream()
    if world > 1:
        # SURVEY §8e: points (and all their rows) are sharded by observation count, cameras are replicated
        plo, phi, rlo, rhi = rp.shard(rank, world)
        gpu = cs.Problem(rp.C, phi - plo, rp.row_cam[rlo:rhi], rp.row_pt[rlo:rhi] - plo, rp.row_obs[rlo:rhi],
                         device=local_rank, stream=stream.cuda_stream, rank=rank, world_size=world, nccl_id=nccl_id)
        state0 = np.concatenate([full_state[3 * plo:3 * phi], full_state[3 * rp.P:]])
    else:
        gpu = cs.Problem(rp.C, rp.P, rp.row_cam, rp.row_pt, rp.row_obs, device=local_rank, stream=stream.cuda_stream)
        state0 = full_state

    def timed_solve(iters, host_boundary):
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(stream)
        state, recs = gpu.lm_solve(state0, gpu.lm_options(max_num_iterations=iters), host_boundary=host_boundary,
                                   max_records=iters + 1)
        e1.record(stream)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        dev = e0.elapsed_time(e1) / 1e3
        if world > 1:
            dist.barrier()
            t = torch.tensor([dev, wall], dtype=torch.float64, device="cuda")
            dist.all_reduce(t, op=dist.ReduceOp.MAX)   # max over ranks
            dev, wall = float(t[0]), float(t[1])
        return dev, wall, recs, state

    # warm-up
    single = world == 1
    if args.warmup > 0:
        timed_solve(args.warmup, False)
        timed_solve(min(args.warmup, 2), True)
    sampler = ClockSampler(local_rank)
    sampler.start()
    gpu.stats_reset()
    dev_s, wall_s, recs, state_out = timed_solve(args.steps, False)
    launches = gpu.total_launches()
    clocks = sampler.stop()
    iters = max(1, len(recs) - 1)
    # end to end through the host-buffer boundary (N > 1: every rank drives its shard through the same entry points with its
    # own host buffers; the few host-side scalars of the loop are combined across ranks; wall clock, max over ranks)
    gpu.stats_reset()
    e2e_dev_s, e2e_wall_s, recs_e2e, _ = timed_solve(args.steps, True)
    h2d, d2h = gpu.transfer_bytes()
    e2e_iters = max(1, len(recs_e2e) - 1)
    # per-kernel event timing for the roofline (same steps, instrumented)
    gpu.stats_reset()
    gpu.profile(True)
    timed_solve(args.steps, False)
    stats = gpu.stats()
    gpu.profile(False)
    peak, peak_src = load_peaks()
    # the other kernel BASELINE.json's metric names, J'J x (+ D^2 x) in one pass (not on the ITERATIVE_SCHUR path, so it
    # is timed on its own: a few launches through the public entry point, kernel time from the same CUDA-event stats)
    jtj = None
    if world == 1:
        try:
            rng = np.random.RandomState(1)
            xj = rng.randn(gpu.num_parameters)
            Dj = np.abs(rng.randn(gpu.num_parameters)) + 0.1
            gpu.jtj_multiply(xj, Dj)
            gpu.stats_reset()
            gpu.profile(True)
            for _ in range(5):
                gpu.jtj_multiply(xj, Dj)
            sj = gpu.stats().get("jtj_multiply")
            jtj = op_rate(sj, peak)
        except Exception as e:  # never let the extra measurement take the bench line down
            jtj = {"error": str(e)[:200]}
        finally:
            try:
                gpu.profile(False)
            except Exception:
                pass
    total_ms = sum(v["ms"] for v in stats.values())
    # S*x: the product's own launch plus, where a problem needs them, the >32-row-point launch and the fixed-order
    # reduction of per-CTA partials -- all billed to the one operation
    sx = dict(stats.get("schur_multiply", {"ms": 0.0, "operations": 0, "launches": 0, "bytes_per_operation": 0.0}))
    for extra in ("schur_multiply_big_points", "camera_reduce"):
        if extra in stats:
            sx["ms"] += stats[extra]["ms"]
            sx["launches"] += stats[extra]["launches"]
    rates = {k: op_rate(v, peak) for k, v in stats.items() if v["operations"] > 0 and v["bytes_per_operation"] > 0}
    rates["schur_multiply"] = op_rate(sx, peak)
    by_time = max(((k, v) for k, v in stats.items() if v["bytes_per_operation"] > 0), key=lambda kv: kv[1]["ms"])[0]
    # the roofline line is about the kernel north_star names (the implicit-Schur product feeding CG), which is also
    # the dominant kernel on the default workload; `dominant_kernel_by_time` says which HBM kernel took most time here
    dom_name = "schur_multiply" if sx["operations"] > 0 else by_time
    dom = rates[dom_name]
    kernels = {k: {"launches": v["launches"], "operations": v["operations"], "ms": round(v["ms"], 4),
                   "share": round(v["ms"] / total_ms, 4) if total_ms > 0 else 0.0,
                   "GBps": rates[k]["GBps"] if k in rates and rates[k] else None}
               for k, v in stats.items() if v["launches"] > 0}

    # "Schur-eliminate" of the metric = (E'E + D^2)^-1, reduced rhs and the block diagonal of S (SCHUR_JACOBI):
    # two passes over J here (point-major, then camera-major); `frac` bills each pass its own algorithmic bytes,
    # `frac_single_pass` bills the whole elimination SURVEY 8d's one-pass figure (216 N + vectors)
    elim = None
    parts = [stats[k] for k in ("schur_init", "schur_diag_blocks") if stats.get(k, {}).get("operations", 0) > 0 and stats[k]["ms"] > 0]
    if len(parts) == 2:
        n_ops = min(v["operations"] for v in parts)
        eb = sum(v["bytes_per_operation"] * v["operations"] for v in parts)
        et = sum(v["ms"] for v in parts) * 1e-3
        one_pass = (216.0 * rp.N + 8.0 * (3 * rp.P + 9 * rp.C) + 720.0 * rp.C) * n_ops
        elim = {"GBps": round(eb / et / 1e9, 1), "frac": round(eb / et / 1e9 / peak, 4), "operations": n_ops,
                "mean_op_ms": round(1e3 * et / n_ops, 4), "frac_single_pass": round(one_pass / et / 1e9 / peak, 4)}
    line = {"metric": METRIC, "value": iters / dev_s, "unit": UNIT, "n_gpus": world, "steps": iters,
            "warmup": args.warmup, "ms_per_step": 1e3 * dev_s / iters, "higher_is_better": True, "scaling": "strong",
            "vs_baseline": None, "dtype": "f64",
            "data": "synthetic" if workload != "c16" else "real BAL file shipped with the reference",
            "config": make_config(desc, rp.N),
            "cg_iterations": [r["ls_iterations"] for r in recs[1:]],
            "costs": [r["cost"] for r in recs], "step_norms": [r["step_norm"] for r in recs],
            "e2e": {"value": e2e_iters / e2e_wall_s, "unit": UNIT, "h2d_bytes_per_step": h2d // e2e_iters,
                    "d2h_bytes_per_step": d2h // e2e_iters, "device_seconds": e2e_dev_s, "wall_seconds": e2e_wall_s},
            "gpu_launches": launches, "clocks": clocks, "wall_seconds": wall_s,
            "roofline": {"bound": "hbm", "kernel": dom_name, "achieved": dom["GBps"], "peak": peak, "unit": "GB/s",
                         "frac": dom["frac"], "peak_source": peak_src,
                         "bytes_per_operation": dom["bytes_per_operation"], "operations": dom["operations"],
                         "launches": dom["launches"], "dominant_kernel_by_time": by_time,
                         "mean_op_ms": dom["mean_op_ms"],
                         "note": "achieved = algorithmic bytes of one operation x operations / sum of CUDA-event time "
                                 "of all launches of those operations"},
            "kernels": kernels,
            "rates": {k: v for k, v in rates.items() if v},
            "jtj_multiply": jtj,
            "schur_eliminate": elim,
            "final_cost": recs[-1]["cost"]}
    if world > 1:
        line["sharding"] = "points sharded over %d ranks by observation count, cameras replicated; one NCCL all-reduce of the %d-double camera vector per CG iteration" % (world, 9 * rp.C)
        if rank != 0:
            gpu.close()
            dist.destroy_process_group()
            return 0
    if not args.no_cpu_baseline and world == 1:
        r = run_reference(args, bal, desc)
        line["cpu_baseline"] = {"value": r["value"], "unit": UNIT, "cores": r["cores"], "kind": "port",
                                "sample": "%d LM iterations from the same initial point (%d CG iterations), %.1f s" % (
                                    r["iterations"], sum(int(t["ls_iterations"]) for t in r["trace"]), r["seconds"])}
    if args.dump_outputs:
        dump_outputs(args.dump_outputs, dict(state=state_out, **trace_arrays(recs)))
    print(json.dumps(line))
    gpu.close()
    if world > 1:
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
