"""The quadcopter flow of the reference's QuadcopterNavigation/mainQuadcopter.jl:122-154 (each start / goal pair planned by the 3-D A*,
then solved) as a batch: plan K config-4 pairs -- planner "python": the Python restatement obca_b200.planner.a_star_3d on host
processes (8-11 s per pair); "host": the same search in C++ on host threads (native.plan_quadcopter_batch); "gpu": on the GPU in one
call (device.plan_quadcopter_batch); all three give the same plans --, solve all planned
pairs -- each with the horizon N = path length - 1 and the sampling time Ts = round(0.25 * 80 / N, 2) the planner gave it -- in ONE
GPU call (obca_quadcopter_solve_mixed), run the reference's constrSatisfaction on every result in one more call.  Pairs whose
horizon exceeds the solver's limit (N + 1 <= 512; the planner gives N = 80..147 over the config-4 box) are counted and listed
as skipped.  Planner "flow" does all of it -- plan, warm start, solve, check -- in one call that keeps everything on the GPU
(device.plan_solve_quadcopter, obca_quadcopter_plan_solve), with the pairs whose search outgrew the device's scratch planned on the host;
it prints the same counts as "gpu".  Planner "both" plans once in one call and solves and checks with QuadcopterDist and then
QuadcopterSignedDist in the same call (device.plan_solve_quadcopter_both, obca_quadcopter_plan_solve_both), as mainQuadcopter.jl:145-154
does for one pair; it prints one line per formulation.

usage: python examples/sweep_quadcopter.py [K] [seed] [workers] [python|host|gpu|flow|both]      (needs a CUDA device for the solves)
"""
import os
import sys
import time
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import obca_b200                                                   # noqa: E402
from obca_b200 import quadcopter, scenarios                        # noqa: E402
from obca_b200.planner import device, native                        # noqa: E402
from obca_b200.planner.a_star_3d import plan_quadcopter_warm_start  # noqa: E402

N_LIMIT = 511      # the quadcopter solver's longest horizon (N + 1 <= 512 stages, at most four per thread of a 128-thread CTA)


def sweep(K=32, seed=2, signed_dist=1, workers=None, planner="python"):
    sc = scenarios.quadcopter_batch(K, seed=seed)          # config-4 start / goal pairs (mainQuadcopter.jl:48-51)
    t0 = time.time()
    if planner == "flow":
        return flow(sc, K, signed_dist, t0)
    if planner == "python":
        with ProcessPoolExecutor(workers) as ex:
            plans = list(ex.map(plan_quadcopter_warm_start, sc["x0"], sc["xF"], [sc["Ts80"]] * K))
    elif planner == "host":
        plans = native.plan_quadcopter_batch(sc["x0"], sc["xF"], sc["Ts80"], nthreads=workers or 0)
    elif planner == "gpu":
        plans = device.plan_quadcopter_batch(sc["x0"], sc["xF"], sc["Ts80"])
    else:
        raise ValueError(f"planner must be python, host, gpu or flow, not {planner!r}")
    t_plan = time.time() - t0
    N = np.array([p["N"] if p else -1 for p in plans])
    idx = [i for i in range(K) if 2 <= N[i] <= N_LIMIT]
    out = dict(K=K, planner=planner, planned=int((N >= 0).sum()), skipped=[(i, int(N[i])) for i in range(K) if N[i] > N_LIMIT], t_plan=t_plan,
               t_solve=0.0, converged=0, feasible=0, N=N, Ts=np.array([p["Ts"] if p else np.nan for p in plans]))
    if not idx:
        return out
    Ns, Ts = N[idx], out["Ts"][idx]
    r = quadcopter.quadcopter_solve_mixed(sc["x0"][idx], sc["xF"][idx], Ns, Ts, sc["R"], sc["obs"], [plans[i]["xWS"] for i in idx],
                                          1.0, signed_dist)
    feas, _ = quadcopter.check_quadcopter_mixed(r["xp"], r["up"], r["ts"], sc["x0"][idx], sc["xF"][idx], Ns, Ts, r["lp"], sc["obs"], sc["R"])
    out.update(t_solve=float(r["time"]), converged=int((r["exitflag"] == 1).sum()), feasible=int(np.asarray(feas).sum()),
               solved=len(idx), exitflag=r["exitflag"])
    return out


def flow(sc, K, signed_dist, t0):
    o = device.plan_solve_quadcopter(sc["x0"], sc["xF"], sc["R"], sc["obs"], sc["Ts80"], signed_dist, Ncap=N_LIMIT, host_fallback=True)
    t_all = time.time() - t0
    N, ok = o["N"], o["status"] == 0
    out = dict(K=K, planner="flow", planned=int((N >= 0).sum()), skipped=[(i, int(N[i])) for i in range(K) if N[i] > N_LIMIT],
               t_plan=t_all, t_solve=o["time"], converged=int((o["exitflag"][ok] == 1).sum()), feasible=int(o["feasible"][ok].sum()),
               N=N, Ts=o["Ts"])
    if ok.any():
        out.update(solved=int(ok.sum()), exitflag=o["exitflag"][ok])
    return out


def both(K=32, seed=2):
    """Every pair planned once on the GPU (POOL_FULL pairs on the host), then solved and checked with both formulations."""
    sc = scenarios.quadcopter_batch(K, seed=seed)
    o = device.plan_solve_quadcopter_both(sc["x0"], sc["xF"], sc["R"], sc["obs"], sc["Ts80"], Ncap=N_LIMIT, host_fallback=True)
    ok = o["status"] == 0
    return dict(K=K, planned=int(ok.sum()), N=np.where(ok, o["N"], -1), t_plan=o["plan_seconds"],
                sets={f: dict(converged=int((o[f]["exitflag"][ok] == 1).sum()), feasible=int(o[f]["feasible"][ok].sum()),
                              t_solve=o[f]["time"]) for f in ("dist", "sd")})


if __name__ == "__main__":
    a = sys.argv
    if len(a) > 4 and a[4] == "both":
        try:
            o = both(int(a[1]) if len(a) > 1 else 32, int(a[2]) if len(a) > 2 else 2)
        except obca_b200.ObcaError as e:
            print("solve not run:", e); sys.exit(2)
        n = o["N"][o["N"] >= 0]
        print(f"{o['K']} start / goal pairs: {o['planned']} planned once in {o['t_plan']:.2f} s GPU device time, N = {n.min()}..{n.max()}")
        for f, name in (("dist", "QuadcopterDist"), ("sd", "QuadcopterSignedDist")):
            s = o["sets"][f]
            print(f"{name}: {o['planned']} planned, {s['converged']} converged, {s['feasible']} pass constrSatisfaction, "
                  f"solve {s['t_solve'] * 1e3:.0f} ms device time")
        sys.exit(0)
    try:
        o = sweep(int(a[1]) if len(a) > 1 else 32, int(a[2]) if len(a) > 2 else 2, 1, int(a[3]) if len(a) > 3 and int(a[3]) > 0 else None,
                  a[4] if len(a) > 4 else "python")
    except obca_b200.ObcaError as e:
        print("solve not run:", e); sys.exit(2)
    ok = o["N"][o["N"] >= 0]
    how = "planned, solved and checked in one call" if o["planner"] == "flow" else "planned"
    print(f"{o['K']} start / goal pairs: {o['planned']} {how} in {o['t_plan']:.1f} s ({o['planner']} planner), N = {ok.min()}..{ok.max()} "
          f"({len(set(ok.tolist()))} distinct), Ts = {np.nanmin(o['Ts']):.2f}..{np.nanmax(o['Ts']):.2f}")
    if o["skipped"]:
        print(f"skipped {len(o['skipped'])} pair(s) with N > {N_LIMIT} (pair, N): {o['skipped']}")
    if o.get("solved"):
        print(f"solved {o['solved']} in one GPU call in {o['t_solve'] * 1e3:.0f} ms device time: {o['converged']} converged, "
              f"{o['feasible']} pass constrSatisfaction")
