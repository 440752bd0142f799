"""Plan, solve and check a parking batch two ways, alternating in one process: the composed path -- device.plan_goals_raw
(obca_plan_parking_warmstart_goals), the host cutting and padding of the planned poses, parking.parking_solve_mixed, parking.check_parking_mixed --
against the one call obca_parking_plan_solve_goals (device.plan_solve_goals_raw), which keeps everything on the device.  Wall clock around
the whole path (both end in a stream synchronise), plus the device times of the search and the solve.  Workloads: the backwards sweep of
main.jl:165-168 with one goal at B = 512 and 4096, and the free-slot car park (scenarios.parking_lot_free_slots, pose i -> slot
i mod n_slots) at B = 4096.  The two paths' outputs (status, N, exitflag, iters, feasible) are compared in the same run.  Prints one JSON
line per workload (and appends them to --out); the card's name and power limit are read in the same call.

usage: python tools/bench_flow.py [--reps 3] [--out FILE.jsonl]          (needs a CUDA device)
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
from obca_b200 import parking, scenarios                            # noqa: E402
from obca_b200.planner import device, native                        # noqa: E402

EGO = np.array([3.7, 1.0, 1.0, 1.0]); XYB = np.array([-15.0, 15.0, 1.0, 10.0]); NCAP = 319


def workload(name, B, seed=0):
    rng = np.random.default_rng(seed)
    x0 = np.column_stack([rng.uniform(-9, 9, B), rng.uniform(6.8, 9.3, B), np.zeros(B), np.zeros(B)])
    if name == "backwards":
        sc = scenarios.reverse_parking_scenario()
        ox, oy = native.obstacle_points("backwards")
        return x0, np.tile(sc["xF"], (B, 1)), ox, oy, sc
    sc = scenarios.parking_lot_free_slots()
    return x0, sc["goals"][np.arange(B) % len(sc["goals"])], sc["ox"], sc["oy"], sc


def composed(x0, xF, ox, oy, sc):
    o = device.plan_goals_raw(x0, xF, ox, oy, sc["Ts"], sc["L"], 3)
    o["status"][(o["status"] == 0) & ((o["N"] < 2) | (o["N"] > NCAP))] = 2      # the one call's OBCA_PLAN_CAPACITY
    idx = np.flatnonzero(o["status"] == 0)
    Ns = o["N"][idx]
    rx = [o["rx"][i, :n + 1] for i, n in zip(idx, Ns)]; ry = [o["ry"][i, :n + 1] for i, n in zip(idx, Ns)]
    ryaw = [o["ryaw"][i, :n + 1] for i, n in zip(idx, Ns)]
    xWS = [o["xWS"][i, :4 * (n + 1)].reshape(4, n + 1).T for i, n in zip(idx, Ns)]
    uWS = [o["uWS"][i, :2 * n].reshape(2, n).T for i, n in zip(idx, Ns)]
    r = parking.parking_solve_mixed(x0[idx], xF[idx], Ns, sc["Ts"], sc["L"], EGO, XYB, sc["nOb"], sc["vOb"], sc["A"], sc["b"], rx, ry,
                                    ryaw, 0, xWS, uWS, 1)
    feas, _, _ = parking.check_parking_mixed(x0[idx], xF[idx], Ns, sc["Ts"], sc["L"], EGO, XYB, sc["nOb"], sc["vOb"], sc["A"], sc["b"],
                                             r["xp"], r["up"], r["lp"], r["np"], r["ts"], 0, 1, r["sl"])
    out = dict(status=o["status"], N=o["N"], exitflag=np.zeros(len(x0), np.int32), iters=np.zeros(len(x0), np.int32),
               feasible=np.zeros(len(x0), np.int32), plan_s=o["seconds"], solve_s=r["time"])
    out["exitflag"][idx] = r["exitflag"]; out["iters"][idx] = r["iters"]; out["feasible"][idx] = feas
    return out


def one_call(x0, xF, ox, oy, sc):
    g = device.plan_solve_goals_raw(x0, xF, ox, oy, sc["Ts"], sc["nOb"], sc["vOb"], sc["A"], sc["b"], EGO, XYB, sc["L"], 3, NCAP)
    ok = g["status"] == 0
    return dict(status=g["status"], N=g["N"], exitflag=np.where(ok, g["exitflag"], 0), iters=np.where(ok, g["iters"], 0),
                feasible=np.where(ok, g["feasible"], 0), plan_s=g["plan_seconds"], solve_s=g["time"])


def timed(f, *a):
    t0 = time.perf_counter()
    r = f(*a)
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    gpu = card()
    for name, B in (("backwards", 512), ("backwards", 4096), ("lot_free_slots", 4096)):
        x0, xF, ox, oy, sc = workload(name, B)
        composed(x0, xF, ox, oy, sc); one_call(x0, xF, ox, oy, sc)      # warm-up: module loads, workspace growth
        tc, t1, dev_c, dev_1 = [], [], [], []
        for _ in range(a.reps):
            t, rc = timed(composed, x0, xF, ox, oy, sc); tc.append(t); dev_c.append((rc["plan_s"], rc["solve_s"]))
            t, r1 = timed(one_call, x0, xF, ox, oy, sc); t1.append(t); dev_1.append((r1["plan_s"], r1["solve_s"]))
        same = all(np.array_equal(rc[k], r1[k]) for k in ("status", "N", "exitflag", "iters", "feasible"))
        ok = r1["status"] == 0
        rec = dict(bench="plan_solve_flow", gpu=gpu, workload=name, B=B, Ncap=NCAP, reps=a.reps, solved=int(ok.sum()),
                   converged=int((r1["exitflag"] == 1).sum()), feasible=int((r1["feasible"] == 1).sum()), same_outputs=same,
                   composed_s=[round(t, 4) for t in tc], one_call_s=[round(t, 4) for t in t1],
                   composed_mean_s=round(float(np.mean(tc)), 4), one_call_mean_s=round(float(np.mean(t1)), 4),
                   composed_device_plan_solve_s=[[round(p, 4), round(s, 4)] for p, s in dev_c],
                   one_call_device_plan_solve_s=[[round(p, 4), round(s, 4)] for p, s in dev_1])
        line = json.dumps(rec)
        print(line, flush=True)
        if a.out:
            with open(a.out, "a") as f:
                f.write(line + "\n")


if __name__ == "__main__":
    main()
