"""Hybrid A* warm starts of a parking sweep: the host planner on every host CPU (native.plan_batch) against the GPU planner
(device.plan_batch, obca_plan_parking_warmstart_batch) on the same seeded start poses, in alternating runs; the outputs of both are
compared in the same run.  Then the end-to-end plan + solve time of examples/sweep_parking.py with each planner.  Prints one JSON line
per measurement (and appends them to --out); the card's name and power limit are read in the same call.

usage: python tools/bench_plan.py [--B 512 4096] [--reps 3] [--out FILE.jsonl]          (needs a CUDA device)
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
sys.path.insert(0, os.path.join(ROOT, "examples"))

from obca_b200 import scenarios                                     # noqa: E402
from obca_b200.planner import device, native                        # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception as e:      # the measurement still stands; say that the card was not read
        return f"not read ({e})"


def compare(a, b):
    """(# poses with a different status or N, max |a - b| over the paths and warm starts of the others)"""
    diff, worst = 0, 0.0
    for w, v in zip(a, b):
        if (w is None) != (v is None) or (w is not None and w["N"] != v["N"]):
            diff += 1
        elif w is not None:
            worst = max(worst, max(float(np.abs(w[k] - v[k]).max()) for k in ("rx", "ry", "ryaw", "xWS", "uWS")))
    return diff, worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, nargs="+", default=[512, 4096])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = card()
    rows = []

    def emit(r):
        r["card"] = gpu
        print(json.dumps(r), flush=True)
        rows.append(r)

    device.plan_batch(np.array([[-6.0, 9.5, 0.0]]), (0.0, 1.3, np.pi / 2), "backwards")      # module load, first allocation
    for scenario in ("backwards", "parallel"):
        sc = scenarios.reverse_parking_scenario() if scenario == "backwards" else scenarios.parallel_parking_scenario(4)
        for B in a.B:
            rng = np.random.default_rng(a.seed)
            x0 = np.column_stack([rng.uniform(-9, 9, B), rng.uniform(6.8, 9.3, B), np.zeros(B)])
            t_host, t_gpu, k_gpu = [], [], []
            for _ in range(a.reps):
                t0 = time.perf_counter(); h = native.plan_batch(x0, sc["xF"], scenario); t_host.append(time.perf_counter() - t0)
                ox, oy = native.obstacle_points(scenario)
                t0 = time.perf_counter()
                o = device.plan_raw(x0, sc["xF"], ox, oy, (0.6 if scenario == "backwards" else 0.9))
                t_gpu.append(time.perf_counter() - t0); k_gpu.append(o["seconds"])
            g = device.plan_batch(x0, sc["xF"], scenario)
            diff, worst = compare(h, g)
            emit(dict(what="plan", scenario=scenario, B=B, host_threads=os.cpu_count(), host_s=t_host, gpu_call_s=t_gpu, gpu_kernel_s=k_gpu,
                      planned=sum(w is not None for w in g), max_expansions=int(o["expansions"].max()),
                      status_or_N_differs=diff, max_abs_diff=worst))
    import sweep_parking
    for planner in ("host", "gpu", "host", "gpu"):
        t0 = time.perf_counter()
        o = sweep_parking.sweep(512, "backwards", 0, planner=planner)
        emit(dict(what="plan+solve", scenario="backwards", B=512, planner=planner, wall_s=time.perf_counter() - t0, plan_s=o["t_plan"],
                  solve_device_s=o["t_solve"], converged=o["converged"], feasible=o["feasible"]))
    if a.out:
        with open(a.out, "a") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
