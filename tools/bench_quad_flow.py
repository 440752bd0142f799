"""Plan, build the warm starts, solve and check a quadcopter batch two ways, alternating in one process: the composed path --
device.plan_quadcopter_raw (obca_plan_quadcopter_warmstart_batch), native.quadcopter_warm_start on every path (host), the host padding of
quadcopter.quadcopter_solve_mixed and quadcopter.check_quadcopter_mixed -- against the one call obca_quadcopter_plan_solve
(device.plan_solve_quadcopter_raw), which keeps everything on the device.  Wall clock around the whole path (both end in a stream
synchronise), plus the device times of the search and the solve.  Workload: config-4 start / goal pairs (scenarios.quadcopter_batch,
seed 2, mainQuadcopter.jl:48-51), SignedDist, at B = 512 and 2048.  The two paths' outputs (status, N, Ts, exitflag, iters, feasible, and
xp, lp over every solved pair's horizon) are compared in every run.  Prints one JSON line per batch size (and appends them to --out);
the card's name and power limit are read in the same call.

usage: python tools/bench_quad_flow.py [--reps 3] [--B 512 2048] [--out FILE.jsonl]          (needs a CUDA device)
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
from obca_b200 import quadcopter, scenarios                         # noqa: E402
from obca_b200.planner import device, native                        # noqa: E402
from obca_b200.planner.a_star_3d import quadcopter_environment      # noqa: E402

NCAP = 511


def composed(sc, env):
    s, g = sc["x0"][:, :3] * 10.0, sc["xF"][:, :3] * 10.0
    o = device.plan_quadcopter_raw(s, g, *env, 1.0, cap=NCAP + 1)
    st = o["status"].copy()
    st[(st == 0) & (o["N"] < 2)] = 2                                 # the one call's OBCA_PLAN_CAPACITY
    idx = np.flatnonzero(st == 0)
    Ns = o["N"][idx]
    ws = [native.quadcopter_warm_start(o["rx"][i, :n + 1].copy(), o["ry"][i, :n + 1].copy(), o["rz"][i, :n + 1].copy(), sc["Ts80"])
          for i, n in zip(idx, Ns)]
    Tsb = np.array([w["Ts"] for w in ws])
    x0, xF = sc["x0"][idx], sc["xF"][idx]
    r = quadcopter.quadcopter_solve_mixed(x0, xF, Ns, Tsb, sc["R"], sc["obs"], [w["xWS"] for w in ws], 1.0, 1)
    feas, _ = quadcopter.check_quadcopter_mixed(r["xp"], r["up"], r["ts"], x0, xF, Ns, Tsb, r["lp"], sc["obs"], sc["R"])
    B = len(st)
    out = dict(status=st, N=o["N"], Ts=np.full(B, np.nan), exitflag=np.zeros(B, np.int32), iters=np.zeros(B, np.int32),
               feasible=np.zeros(B, np.int32), xp=[None] * B, lp=[None] * B, plan_s=o["seconds"], solve_s=r["time"])
    out["Ts"][idx] = Tsb; out["exitflag"][idx] = r["exitflag"]; out["iters"][idx] = r["iters"]; out["feasible"][idx] = feas
    for q, i in enumerate(idx):
        out["xp"][i], out["lp"][i] = r["xp"][q], r["lp"][q]
    return out


def one_call(sc, env):
    g = device.plan_solve_quadcopter_raw(sc["x0"], sc["xF"], *env, 1.0, sc["Ts80"], sc["R"], sc["obs"], 1.0, 1, NCAP)
    ok = g["status"] == 0
    B = len(ok)
    out = dict(status=g["status"], N=g["N"], Ts=np.where(ok, g["Tsb"], np.nan), exitflag=np.where(ok, g["exitflag"], 0),
               iters=np.where(ok, g["iters"], 0), feasible=np.where(ok, g["feasible"], 0), xp=[None] * B, lp=[None] * B,
               plan_s=g["plan_seconds"], solve_s=g["time"])
    for i in np.flatnonzero(ok):
        n = int(g["N"][i])
        out["xp"][i], out["lp"][i] = g["xp"][i, :n + 1].T, g["lp"][i, :n + 1].T
    return out


def same(a, b):
    if not all(np.array_equal(a[k], b[k], equal_nan=True) for k in ("status", "N", "Ts", "exitflag", "iters", "feasible")):
        return False
    return all((u is None and v is None) or (u is not None and v is not None and np.array_equal(u, v))
               for k in ("xp", "lp") for u, v in zip(a[k], b[k]))


def timed(f, *a):
    t0 = time.perf_counter()
    r = f(*a)
    return time.perf_counter() - t0, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--B", type=int, nargs="+", default=[512, 2048])
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    gpu = card()
    env = quadcopter_environment()
    for B in a.B:
        sc = scenarios.quadcopter_batch(B, seed=2)
        composed(sc, env); one_call(sc, env)      # warm-up: module loads, workspace growth
        tc, t1, dev_c, dev_1, eq = [], [], [], [], []
        for _ in range(a.reps):
            t, rc = timed(composed, sc, env); tc.append(t); dev_c.append((rc["plan_s"], rc["solve_s"]))
            t, r1 = timed(one_call, sc, env); t1.append(t); dev_1.append((r1["plan_s"], r1["solve_s"]))
            eq.append(same(rc, r1))
        ok = r1["status"] == 0
        rec = dict(bench="quad_plan_solve_flow", gpu=gpu, workload="config4_sd", B=B, Ncap=NCAP, reps=a.reps, solved=int(ok.sum()),
                   converged=int((r1["exitflag"] == 1).sum()), feasible=int((r1["feasible"] == 1).sum()), same_outputs_every_run=all(eq),
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
