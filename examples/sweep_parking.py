"""The randomised sweep of the reference's AutonomousParking/main.jl:165-168 (many start poses, each planned by Hybrid A* and then
solved) as a batch: plan every pose on the host threads (libobca_planner.so), solve all planned problems -- each with the horizon
N the planner gave it -- in ONE GPU call (obca_parking_solve_mixed), run the reference's acceptance test on every result in one
more call.  With planner="gpu" (4th argument `gpu`) the poses are planned on the GPU as well, with the host planner's search
decisions, and planned, solved and checked in ONE call (obca_parking_plan_solve_goals) that keeps everything on the device.  With
planner="both" the poses are planned once on the GPU and solved and checked with ParkingDist and then ParkingSignedDist in the same call
(obca_parking_plan_solve_both), as main.jl:258-269 does for one pose; it prints one line per formulation.  sampleN (5th argument, default 3) is the
warm-start sampling of main.jl:46-57: Ts = 0.6 / 3 * sampleN ("backwards", 0.9 for "parallel"); sampleN = 1 gives horizons past 127
steps (the solver takes N <= 319), still solved in one call.

usage: python examples/sweep_parking.py [B] [backwards|parallel] [seed] [host|gpu|both] [sampleN]      (needs a CUDA device for the solves)
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import obca_b200                                            # noqa: E402
from obca_b200 import parking, scenarios                    # noqa: E402
from obca_b200.planner import device, native, warmstart     # noqa: E402


def batch(B, scenario, seed):
    sc = scenarios.reverse_parking_scenario() if scenario == "backwards" else scenarios.parallel_parking_scenario(4)
    rng = np.random.default_rng(seed)
    x0 = np.column_stack([rng.uniform(-9, 9, B), rng.uniform(6.8, 9.3, B), np.zeros(B), np.zeros(B)])      # start poses in the lane, v = 0
    return sc, x0, np.array([3.7, 1.0, 1.0, 1.0]), np.array([-15.0, 15.0, 1.0, 10.0]), 2.7      # sc, x0, ego, XYbounds, L


def sweep(B=256, scenario="backwards", seed=0, signed_dist=1, workers=0, planner="host", sampleN=3):
    sc, x0, ego, XYbounds, L = batch(B, scenario, seed)
    if planner == "gpu":
        r = device.plan_solve_batch(x0, sc["xF"], sc["nOb"], sc["vOb"], sc["A"], sc["b"], ego, XYbounds, scenario, sampleN=sampleN, L=L,
                                    signed_dist=signed_dist, host_fallback=True)
        ok = r["status"] == 0
        return dict(B=B, planned=int(ok.sum()), groups=len(set(r["N"][ok].tolist())), t_plan=r["plan_seconds"], t_solve=r["time"],
                    converged=int((r["exitflag"] == 1).sum()), feasible=int((r["feasible"][ok] == 1).sum()),
                    exitflag=r["exitflag"].astype(int), N=np.where(ok, r["N"], -1))
    t0 = time.time()
    plans = native.plan_batch(x0, sc["xF"], scenario, workers, sampleN=sampleN)
    t_plan = time.time() - t0
    groups = warmstart.group_by_horizon(plans)
    out = dict(B=B, planned=sum(w is not None for w in plans), groups=len(groups), t_plan=t_plan, t_solve=0.0, converged=0, feasible=0,
               exitflag=np.zeros(B, int), N=np.array([w["N"] if w else -1 for w in plans]))
    idx = [i for i, w in enumerate(plans) if w is not None]
    if not idx:
        return out
    Ts = plans[idx[0]]["Ts"]
    g = lambda k: [plans[i][k] for i in idx]
    Ns = out["N"][idx]
    r = parking.parking_solve_mixed(x0[idx], sc["xF"], Ns, Ts, L, ego, XYbounds, sc["nOb"], sc["vOb"], sc["A"], sc["b"], g("rx"), g("ry"),
                                    g("ryaw"), 0, g("xWS"), g("uWS"), signed_dist)
    feas, _, _ = parking.check_parking_mixed(x0[idx], sc["xF"], Ns, Ts, L, ego, XYbounds, sc["nOb"], sc["vOb"], sc["A"], sc["b"], r["xp"],
                                             r["up"], r["lp"], r["np"], r["ts"], 0, signed_dist, r["sl"])
    out["t_solve"] = float(r["time"])
    out["converged"] = int((r["exitflag"] == 1).sum()); out["feasible"] = int(np.asarray(feas).sum())
    out["exitflag"][idx] = r["exitflag"]
    return out


def sweep_both(B=256, scenario="backwards", seed=0, sampleN=3):
    """Every pose planned once on the GPU (POOL_FULL poses on the host), then solved and checked with both formulations."""
    sc, x0, ego, XYbounds, L = batch(B, scenario, seed)
    ox, oy = native.obstacle_points(scenario)
    Ts = (0.6 if scenario == "backwards" else 0.9) / 3 * sampleN
    r = device.plan_solve_goals_both(x0, sc["xF"], ox, oy, Ts, sc["nOb"], sc["vOb"], sc["A"], sc["b"], ego, XYbounds, L, sampleN,
                                     host_fallback=True)
    ok = r["status"] == 0
    return dict(B=B, planned=int(ok.sum()), N=np.where(ok, r["N"], -1), t_plan=r["plan_seconds"],
                sets={f: dict(converged=int((r[f]["exitflag"] == 1).sum()), feasible=int((r[f]["feasible"][ok] == 1).sum()),
                              t_solve=r[f]["time"]) for f in ("dist", "sd")})


if __name__ == "__main__":
    a = sys.argv
    if len(a) > 4 and a[4] == "both":
        try:
            o = sweep_both(int(a[1]) if len(a) > 1 else 256, a[2] if len(a) > 2 else "backwards", int(a[3]) if len(a) > 3 else 0,
                           int(a[5]) if len(a) > 5 else 3)
        except obca_b200.ObcaError as e:
            print("solve not run:", e); sys.exit(2)
        n = o["N"][o["N"] >= 0]
        print(f"{o['B']} start poses: {o['planned']} planned once in {o['t_plan']:.2f} s GPU device time, N = {n.min()}..{n.max()}")
        for f, name in (("dist", "ParkingDist"), ("sd", "ParkingSignedDist")):
            s = o["sets"][f]
            print(f"{name}: {o['planned']} planned, {s['converged']} converged, {s['feasible']} pass ParkingConstraints, "
                  f"solve {s['t_solve'] * 1e3:.0f} ms device time")
        sys.exit(0)
    try:
        planner = a[4] if len(a) > 4 else "host"
        o = sweep(int(a[1]) if len(a) > 1 else 256, a[2] if len(a) > 2 else "backwards", int(a[3]) if len(a) > 3 else 0, planner=planner,
                  sampleN=int(a[5]) if len(a) > 5 else 3)
    except obca_b200.ObcaError as e:
        print("solve not run:", e); sys.exit(2)
    print(f"{o['B']} start poses: {o['planned']} planned in {o['t_plan']:.2f} s ({'host threads' if planner == 'host' else 'GPU device time'}), "
          f"{o['groups']} horizons N = {o['N'][o['N'] >= 0].min()}..{o['N'].max()}; solved in {'one' if planner == 'host' else 'the same'} GPU "
          f"call in {o['t_solve'] * 1e3:.0f} ms device time: "
          f"{o['converged']} converged, {o['feasible']} pass ParkingConstraints")
