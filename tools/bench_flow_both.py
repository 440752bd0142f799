"""Run the reference's flows with both formulations two ways, alternating in one process: (a) two one-formulation flow calls on the same
inputs, Dist then SD (obca_parking_plan_solve_goals / obca_quadcopter_plan_solve, which plan twice), against (b) one call that plans
once and solves and checks with both (obca_parking_plan_solve_both / obca_quadcopter_plan_solve_both).  Wall clock around each path (every
call ends in a stream synchronise), plus the device times of the search and the two solves.  Workloads: the parking workloads of
tools/bench_flow.py at B = 4096 (backwards sweep with one goal, free-slot car park with a goal per pose) and the config-4 quadcopter
pairs of tools/bench_quad_flow.py at B = 512 and 2048.  In every timed run the two paths' status and N, and each formulation's exitflag,
iters and checker value, are compared.  Prints one JSON line per workload (and appends them to --out); the card's name, power limit and
maximum SM clock are read in the same call.

usage: python tools/bench_flow_both.py [--reps 3] [--out FILE.jsonl]          (needs a CUDA device)
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench_flow                                                   # noqa: E402
import bench_quad_flow                                              # noqa: E402
from bench_plan import card                                         # noqa: E402
from obca_b200 import scenarios                                     # noqa: E402
from obca_b200.planner import device                                # noqa: E402
from obca_b200.planner.a_star_3d import quadcopter_environment      # noqa: E402

CHECKED = ("exitflag", "iters", "feasible")


def parking_paths(name, B):
    x0, xF, ox, oy, sc = bench_flow.workload(name, B)
    args = (x0, xF, ox, oy, sc["Ts"], sc["nOb"], sc["vOb"], sc["A"], sc["b"], bench_flow.EGO, bench_flow.XYB, sc["L"], 3, bench_flow.NCAP)

    def two_calls():
        o = [device.plan_solve_goals_raw(*args, signed_dist=f) for f in (0, 1)]
        return dict(o[1], dist=o[0], sd=o[1], plan_s=[o[0]["plan_seconds"], o[1]["plan_seconds"]])

    def one_call():
        o = device.plan_solve_goals_both_raw(*args)
        return dict(o, plan_s=[o["plan_seconds"]])
    return two_calls, one_call, ("status", "N")


def quadcopter_paths(B):
    sc = scenarios.quadcopter_batch(B, seed=2)
    env = quadcopter_environment()
    args = (sc["x0"], sc["xF"], *env, 1.0, sc["Ts80"], sc["R"], sc["obs"], 1.0)

    def two_calls():
        o = [device.plan_solve_quadcopter_raw(*args, signed_dist=f, Ncap=bench_quad_flow.NCAP) for f in (0, 1)]
        return dict(o[1], dist=o[0], sd=o[1], plan_s=[o[0]["plan_seconds"], o[1]["plan_seconds"]])

    def one_call():
        o = device.plan_solve_quadcopter_both_raw(*args, Ncap=bench_quad_flow.NCAP)
        return dict(o, plan_s=[o["plan_seconds"]])
    return two_calls, one_call, ("status", "N", "Tsb")


def same(a, b, shared):
    """Equal shared outputs, and per formulation equal exitflag, iters and checker value on the solved problems."""
    if not all(np.array_equal(a[k], b[k], equal_nan=True) for k in shared):
        return False
    ok = a["status"] == 0
    return all(np.array_equal(a[f][k][ok], b[f][k][ok]) for f in ("dist", "sd") for k in CHECKED)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    gpu = card()
    runs = [(f"parking_{n}", 4096, parking_paths(n, 4096)) for n in ("backwards", "lot_free_slots")] + \
        [("quadcopter_config4", B, quadcopter_paths(B)) for B in (512, 2048)]
    for name, B, (two_calls, one_call, shared) in runs:
        two_calls(); one_call()      # warm-up: module loads, workspace growth
        ta, tb, dev_a, dev_b, eq = [], [], [], [], []
        for _ in range(a.reps):
            t, ra = bench_flow.timed(two_calls); ta.append(t)
            dev_a.append([round(p, 4) for p in ra["plan_s"]] + [round(ra[f]["time"], 4) for f in ("dist", "sd")])
            t, rb = bench_flow.timed(one_call); tb.append(t)
            dev_b.append([round(p, 4) for p in rb["plan_s"]] + [round(rb[f]["time"], 4) for f in ("dist", "sd")])
            eq.append(same(ra, rb, shared))
        ok = rb["status"] == 0
        rec = dict(bench="plan_solve_both", gpu=gpu, workload=name, B=B, reps=a.reps, solved=int(ok.sum()),
                   converged={f: int((rb[f]["exitflag"][ok] == 1).sum()) for f in ("dist", "sd")},
                   feasible={f: int((rb[f]["feasible"][ok] == 1).sum()) for f in ("dist", "sd")},
                   same_outputs_every_run=all(eq), two_calls_s=[round(t, 4) for t in ta], both_call_s=[round(t, 4) for t in tb],
                   two_calls_mean_s=round(float(np.mean(ta)), 4), both_call_mean_s=round(float(np.mean(tb)), 4),
                   two_calls_device_plan_plan_dist_sd_s=dev_a, both_call_device_plan_dist_sd_s=dev_b)
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
