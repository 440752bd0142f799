"""Parking problems with horizons past 127 steps.  Prints the card's name and power limit, read in the same run, and one JSON line
per measurement:

  sweep      the backwards sweep of examples/sweep_parking.py (B start poses, seed 0) planned by libobca_planner.so at each
             --sampleN (main.jl:46-57: Ts = 0.6 / 3 * sampleN) and solved in ONE obca_parking_solve_mixed call: device time of the
             solve (median of --reps after one warm-up), trajectories/s, converged share, share of the converged that pass
             ParkingConstraints (one obca_check_parking_mixed call).
  split      the same problems of the first sampleN as two mixed calls, N <= 127 and N > 127, against the one call: what a long
             layout costs the short problems (the stage slots of N + 1 > 127 leave fewer CTAs per SM).
  horizon    uniform config-2 poses (reverse_parking_batch's ranges, Ts = 48 / N) at each --horizons N: device time and per-kernel
             event times of one more call with OBCA_PHASE_TIMING=1 (kernel_ms of obca_last_schedule: k_pk_eval, k_pk_sweep,
             k_pk_step, k_pk_tail), rounds and problems handed to the tail kernel.

usage: python tools/bench_long_parking.py [--B 4096] [--reps 3] [--sampleN 1 3] [--horizons 80 127 128 192 319] [--out results.json]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import obca_b200                          # noqa: E402
from obca_b200 import parking, scenarios  # noqa: E402
from obca_b200.planner import native      # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    except OSError:
        return "unknown"
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def schedule():
    rnd, hand = C.c_int(), C.c_int()
    kms = (C.c_double * 5)()
    obca_b200.lib().obca_last_schedule(C.c_int(0), C.byref(rnd), C.byref(hand), kms)
    return rnd.value, hand.value, dict(eval=round(kms[0], 2), sweep=round(kms[1], 2), step=round(kms[2], 2), tail=round(kms[3], 2))


def timed(run, reps):
    r = run()                                   # warm-up: module load, workspace allocation
    times = []
    for _ in range(reps):
        r = run()
        times.append(r["time"])
    return r, float(np.median(times)), times


def sweep_problems(B, sampleN):
    sc = scenarios.reverse_parking_scenario()
    rng = np.random.default_rng(0)
    x0 = np.column_stack([rng.uniform(-9, 9, B), rng.uniform(6.8, 9.3, B), np.zeros(B), np.zeros(B)])      # examples/sweep_parking.py
    t0 = time.time()
    plans = native.plan_batch(x0, sc["xF"], "backwards", 0, sampleN=sampleN)
    t_plan = time.time() - t0
    ok = [i for i, w in enumerate(plans) if w is not None]
    g = lambda k: [plans[i][k] for i in ok]
    return dict(sc=sc, x0=x0[ok], Ns=np.array(g("N")), Ts=plans[ok[0]]["Ts"], rx=g("rx"), ry=g("ry"), ryaw=g("ryaw"), xWS=g("xWS"),
                uWS=g("uWS"), planned=len(ok), t_plan=t_plan)


def solve_mixed(p, idx):
    sc = p["sc"]
    pick = lambda k: [p[k][i] for i in idx]
    return parking.parking_solve_mixed(p["x0"][idx], sc["xF"], p["Ns"][idx], p["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"],
                                       sc["vOb"], sc["A"], sc["b"], pick("rx"), pick("ry"), pick("ryaw"), 0, pick("xWS"), pick("uWS"))


def sweep_row(p, B, sampleN, reps):
    idx = np.arange(p["planned"])
    r, t, times = timed(lambda: solve_mixed(p, idx), reps)
    sc = p["sc"]
    feas, _, _ = parking.check_parking_mixed(p["x0"], sc["xF"], p["Ns"], p["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"],
                                             sc["A"], sc["b"], r["xp"], r["up"], r["lp"], r["np"], r["ts"], 0, 1, r["sl"])
    conv = r["exitflag"] == 1
    rnd, hand, _ = schedule()
    return dict(kind="sweep", B=B, sampleN=sampleN, Ts=round(p["Ts"], 4), planned=p["planned"], plan_s=round(p["t_plan"], 2),
                N_min=int(p["Ns"].min()), N_max=int(p["Ns"].max()), share_long=round(float((p["Ns"] > 127).mean()), 4),
                solve_ms=round(t * 1e3, 2), solve_ms_all=[round(x * 1e3, 2) for x in times], traj_per_s=round(p["planned"] / t, 1),
                converged=round(float(conv.mean()), 4), checker_pass=round(float((np.asarray(feas)[conv] == 1).mean()) if conv.any() else 0.0, 4),
                mean_iters=round(float(r["iters"].mean()), 2), rounds=rnd, handed_to_tail=hand)


def split_row(p, reps):
    short = np.flatnonzero(p["Ns"] <= 127); long_ = np.flatnonzero(p["Ns"] > 127)
    _, t_one, one_all = timed(lambda: solve_mixed(p, np.arange(p["planned"])), reps)
    _, t_s, s_all = timed(lambda: solve_mixed(p, short), reps)
    _, t_l, l_all = timed(lambda: solve_mixed(p, long_), reps)
    return dict(kind="split", problems=p["planned"], n_short=int(short.size), n_long=int(long_.size), one_call_ms=round(t_one * 1e3, 2),
                one_call_ms_all=[round(x * 1e3, 2) for x in one_all], short_call_ms=round(t_s * 1e3, 2),
                short_call_ms_all=[round(x * 1e3, 2) for x in s_all], long_call_ms=round(t_l * 1e3, 2),
                long_call_ms_all=[round(x * 1e3, 2) for x in l_all], two_calls_ms=round((t_s + t_l) * 1e3, 2))


def horizon_batch(B, N):
    sc = scenarios.reverse_parking_scenario()
    rng = np.random.default_rng(0)
    x0 = np.stack([rng.uniform(-10, 10, B), rng.uniform(6.5, 9.5, B), np.zeros(B), np.zeros(B)], 1)
    Ts = 48.0 / N
    w = [scenarios.warmstart_reverse(x0[i], sc["xF"], N, Ts, sc["L"]) for i in range(B)]
    sc.update(B=B, N=N, Ts=Ts, x0=x0, rx=np.stack([a[0] for a in w]), ry=np.stack([a[1] for a in w]), ryaw=np.stack([a[2] for a in w]),
              xWS=np.stack([a[3] for a in w]), uWS=np.stack([a[4] for a in w]))
    return sc


def horizon_row(B, N, reps):
    sc = horizon_batch(B, N)
    run = lambda: parking.parking_solve_batch(sc["x0"], sc["xF"], N, sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"],
                                              sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], 0, sc["xWS"], sc["uWS"])
    r, t, times = timed(run, reps)
    rnd, hand, _ = schedule()
    os.environ["OBCA_PHASE_TIMING"] = "1"
    try:
        run()
    finally:
        os.environ.pop("OBCA_PHASE_TIMING", None)
    _, _, kms = schedule()
    return dict(kind="horizon", B=B, N=N, Ts=round(sc["Ts"], 4), solve_ms=round(t * 1e3, 2), solve_ms_all=[round(x * 1e3, 2) for x in times],
                problems_per_s=round(B / t, 1), converged=round(float((r["exitflag"] == 1).mean()), 4), mean_iters=round(float(r["iters"].mean()), 2),
                rounds=rnd, handed_to_tail=hand, kernel_ms=kms)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--sampleN", type=int, nargs="*", default=[1, 3])
    ap.add_argument("--horizons", type=int, nargs="*", default=[80, 127, 128, 192, 319])
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if obca_b200.lib().obca_device_count() < 1:
        sys.exit("bench_long_parking.py needs a CUDA device")
    info = card()
    print("card:", info, flush=True)
    rows = []

    def emit(row):
        row["card"] = info
        rows.append(row)
        print(json.dumps(row), flush=True)
    for k, sn in enumerate(a.sampleN):
        p = sweep_problems(a.B, sn)
        emit(sweep_row(p, a.B, sn, a.reps))
        if k == 0 and (p["Ns"] <= 127).any() and (p["Ns"] > 127).any():
            emit(split_row(p, a.reps))
    for N in a.horizons:
        emit(horizon_row(a.B, N, a.reps))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
