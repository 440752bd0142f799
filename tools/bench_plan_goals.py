"""Hybrid A* warm starts with a goal per start pose (obca_plan_parking_warmstart_goals) in the car-park row with free slots
(scenarios.parking_lot_free_slots), for three goal sets: one shared goal (the target slot), the free slots (pose i -> slot i mod n_slots)
and a distinct goal per pose (a random pose in the lane, heading within 0.25 rad of the lane's direction).  For each: the device time of the heuristic maps
(k_plan_hmap, one CTA per distinct goal cell, read through obca_plan_parking_heuristic_maps), the device time of the search (k_plan), the
whole GPU call, and the host twin (native.plan_cloud_raw) on every host CPU, in alternating runs; the outputs of both are compared in
the same run.  Prints one JSON line per measurement (and appends them to --out); the card's name and power limit are read in the same
call.

usage: python tools/bench_plan_goals.py [--B 512 4096] [--reps 2] [--out FILE.jsonl]          (needs a CUDA device)
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_plan import card                                         # noqa: E402
from obca_b200 import scenarios                                     # noqa: E402
from obca_b200.planner import device, native                        # noqa: E402


def goal_sets(lot, B, seed):
    rng = np.random.default_rng(seed + 1)
    lane = np.column_stack([rng.uniform(-9, 9, B), rng.uniform(6.8, 9.3, B), rng.choice([0.0, np.pi], B) + rng.uniform(-0.25, 0.25, B)])
    return {"shared": np.tile(lot["goals"][0][:3], (B, 1)), "free_slots": lot["goals"][np.arange(B) % len(lot["goals"])][:, :3],
            "distinct": lane}


def compare(o, h):
    """(# poses with a different status, N or expansion count, max |o - h| over the paths and warm starts of the others)"""
    diff = int(((o["status"] != h["status"]) | (o["N"] != h["N"]) | (o["expansions"] != h["expansions"])).sum())
    worst = 0.0
    for i in np.nonzero((o["status"] == 0) & (h["status"] == 0))[0]:
        n = int(o["N"][i])
        for k, m in (("rx", n + 1), ("ry", n + 1), ("ryaw", n + 1), ("xWS", 4 * (n + 1)), ("uWS", 2 * n)):
            worst = max(worst, float(np.abs(o[k][i, :m] - h[k][i, :m]).max()))
    return diff, worst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, nargs="+", default=[512, 4096])
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    gpu = card()
    rows = []
    lot = scenarios.parking_lot_free_slots()
    ox, oy, Ts = lot["ox"], lot["oy"], 0.6
    device.plan_goals_raw(np.array([[-6.0, 9.5, 0.0]]), lot["goals"][0], ox, oy, Ts)      # module load, first allocation
    for B in a.B:
        rng = np.random.default_rng(a.seed)
        x0 = np.column_stack([rng.uniform(-9, 9, B), rng.uniform(6.8, 9.3, B), np.zeros(B)])
        for name, xF in goal_sets(lot, B, a.seed).items():
            cells = np.unique(np.round(xF[:, :2] / 0.3), axis=0)
            t_host, t_call, t_map, t_search = [], [], [], []
            for _ in range(a.reps):
                t0 = time.perf_counter(); h = native.plan_cloud_raw(x0, xF, ox, oy, Ts); t_host.append(time.perf_counter() - t0)
                t0 = time.perf_counter(); o = device.plan_goals_raw(x0, xF, ox, oy, Ts); t_call.append(time.perf_counter() - t0)
                t_search.append(o["seconds"])
                t_map.append(device.heuristic_maps(cells * 0.3, ox, oy)[2])
            diff, worst = compare(o, h)
            r = dict(what="plan_goals", goals=name, B=B, goal_cells=int(len(cells)), host_threads=os.cpu_count(), host_s=t_host,
                     gpu_call_s=t_call, gpu_map_s=t_map, gpu_search_s=t_search, planned=int((o["status"] == 0).sum()),
                     pool_full=int((o["status"] == device.POOL_FULL).sum()), max_expansions=int(o["expansions"].max()),
                     status_N_or_expansions_differ=diff, max_abs_diff=worst, card=gpu)
            print(json.dumps(r), flush=True)
            rows.append(r)
    if a.out:
        with open(a.out, "a") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
