"""3-D A* warm starts of the quadcopter flow: the host library on every host CPU (native.astar3d_raw, obca_astar3d_batch) against the GPU
planner (device.plan_quadcopter_raw, obca_plan_quadcopter_warmstart_batch) on the config-4 pairs of scenarios.quadcopter_batch(B, seed),
in alternating runs; the two must agree pair for pair (status, N, path, expansions), which is checked in the same run.  Then the
plan + solve time of examples/sweep_quadcopter.py with each planner.  Prints one JSON line per measurement (and appends them to --out);
the card's name and power limit are read in the same call.

usage: python tools/bench_plan_quad.py [--B 512 2048] [--reps 3] [--sweep 512] [--out FILE.jsonl]          (needs a CUDA device)
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "examples"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_plan import card                                         # noqa: E402
from obca_b200 import scenarios                                     # noqa: E402
from obca_b200.planner import device, native                        # noqa: E402

OUT = ("rx", "ry", "rz", "N", "status", "expansions")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, nargs="+", default=[512, 2048])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=2)
    ap.add_argument("--sweep", type=int, default=512, help="pairs of the plan + solve sweep (0: skip)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = card()
    rows = []

    def emit(r):
        r["card"] = gpu
        print(json.dumps(r), flush=True)
        rows.append(r)

    sc = scenarios.quadcopter_batch(4, seed=a.seed)
    device.plan_quadcopter_raw(*native.quadcopter_problem(sc["x0"], sc["xF"]))      # module load, first allocation
    for B in a.B:
        sc = scenarios.quadcopter_batch(B, seed=a.seed)
        args = native.quadcopter_problem(sc["x0"], sc["xF"])
        t_host, t_gpu, k_gpu, differs = [], [], [], []
        for _ in range(a.reps):
            t0 = time.perf_counter(); h = native.astar3d_raw(*args); t_host.append(time.perf_counter() - t0)
            t0 = time.perf_counter(); g = device.plan_quadcopter_raw(*args); t_gpu.append(time.perf_counter() - t0)
            k_gpu.append(g["seconds"])
            differs.append(sum(any(not np.array_equal(g[k][i], h[k][i], equal_nan=True) for k in OUT) for i in range(B)))
        emit(dict(what="plan3d", B=B, seed=a.seed, host_threads=os.cpu_count(), host_s=t_host, gpu_call_s=t_gpu, gpu_kernel_s=k_gpu,
                  status_counts=np.bincount(g["status"], minlength=5).tolist(), expansions_sum=int(g["expansions"].sum()),
                  expansions_max=int(g["expansions"].max()), pairs_differing=differs))
    if a.sweep:
        import sweep_quadcopter
        for planner in ("host", "gpu", "host", "gpu"):
            t0 = time.perf_counter()
            o = sweep_quadcopter.sweep(a.sweep, a.seed, 1, None, planner)
            emit(dict(what="plan+solve", B=a.sweep, planner=planner, wall_s=time.perf_counter() - t0, plan_s=o["t_plan"],
                      solve_device_s=o["t_solve"], planned=o["planned"], converged=o["converged"], feasible=o["feasible"]))
    if a.out:
        with open(a.out, "a") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
