"""Throughput of the car-park scene (obca_b200.scenarios.parking_lot_batch: n_cars parked cars + the far wall, N = 80) next to
config 2 in the same process: device time of the solve (median of --reps timed calls after one warm-up), problems/s, converged
and checker-clean fractions, and per-kernel event times of one more call with OBCA_PHASE_TIMING=1 (kernel_ms slots of
obca_last_schedule: k_pk_eval, k_pk_sweep, k_pk_step, k_pk_tail).  Prints the card's name and power limit, read in the same run,
and one JSON line per workload.

usage: python tools/bench_lot.py [--B 4096] [--reps 3] [--workloads config2 lot10 lot15] [--out results.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import obca_b200                          # noqa: E402
from obca_b200 import parking, scenarios  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    except OSError:
        return "unknown"
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def one(sc, sd, reps):
    run = lambda: parking.parking_solve_batch(sc["x0"], sc["xF"], sc["N"], sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"],
                                              sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], 0, sc["xWS"], sc["uWS"], sd)
    r = run()                                   # warm-up: module load, workspace allocation
    times = []
    for _ in range(reps):
        r = run()
        times.append(r["time"])
    feas, _, _ = parking.check_parking_batch(sc["x0"], sc["xF"], sc["N"], sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"],
                                             sc["A"], sc["b"], r["xp"], r["up"], r["lp"], r["np"], r["ts"], 0, sd, r["sl"])
    conv = r["exitflag"] == 1
    os.environ["OBCA_PHASE_TIMING"] = "1"
    try:
        run()
    finally:
        os.environ.pop("OBCA_PHASE_TIMING", None)
    rnd, hand = C.c_int(), C.c_int()
    kms = (C.c_double * 5)()
    obca_b200.lib().obca_last_schedule(C.c_int(0), C.byref(rnd), C.byref(hand), kms)
    t = float(np.median(times))
    return dict(B=sc["B"], N=sc["N"], nOb=int(sc["nOb"]), V=int(np.sum(sc["vOb"])), formulation="SD" if sd else "Dist",
                solve_ms=round(t * 1e3, 2), solve_ms_all=[round(x * 1e3, 2) for x in times], problems_per_s=round(sc["B"] / t, 1),
                converged=round(float(conv.mean()), 4), checker_clean=round(float((np.asarray(feas)[conv] == 1).mean()) if conv.any() else 0.0, 4),
                mean_iters=round(float(r["iters"].mean()), 2), rounds=rnd.value, handed_to_tail=hand.value,
                kernel_ms=dict(eval=round(kms[0], 2), sweep=round(kms[1], 2), step=round(kms[2], 2), tail=round(kms[3], 2)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--workloads", nargs="*", default=["config2", "lot10"], help="config2 and / or lot<n_cars>")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = card()
    print("card:", info, flush=True)
    rows = []
    for name in a.workloads:
        sc = scenarios.reverse_parking_batch(a.B, 80, 0) if name == "config2" else scenarios.parking_lot_batch(a.B, 80, 0, int(name[3:]))
        for sd in (1, 0):
            row = dict(workload=name, card=info, **one(sc, sd, a.reps))
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
