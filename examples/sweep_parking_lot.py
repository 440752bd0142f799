"""The reverse-parking sweep in a row of a car park (obca_b200.scenarios.parking_lot_scenario: n_cars parked cars + the far wall,
nOb = n_cars + 1 obstacles), in ONE GPU call that keeps everything on the device (obca_parking_plan_solve_goals): plan every start pose
with the GPU Hybrid A* against the lot's point cloud, solve every pose planned OK -- each with the horizon the planner gave it -- and
run the reference's acceptance test on every result.  Poses whose search outgrew the device's scratch are planned by the host twin
(obca_plan_warmstart_cloud_batch) and solved and checked after the call; poses without a path are reported.

--free-slots: the row of scenarios.parking_lot_free_slots instead -- some parked cars left out -- and each car is sent to one of the
free slots (car i to slot i mod the number of slots): the planner takes a goal per pose, the solve and the check xF of shape (B, 4).

sampleN (4th argument, default 3) is the warm-start sampling of main.jl:46-57: Ts = 0.6 / 3 * sampleN; sampleN = 1 gives horizons
past 127 steps (the solver takes N <= 319), still solved in one call.

usage: python examples/sweep_parking_lot.py [B] [n_cars] [seed] [sampleN] [--free-slots]      (needs a CUDA device)
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import obca_b200                                 # noqa: E402
from obca_b200 import scenarios                  # noqa: E402
from obca_b200.planner import device             # noqa: E402


def run(B=64, seed=0, n_cars=10, signed_dist=1, sampleN=3, free_slots=False):
    sc = scenarios.parking_lot_free_slots(n_cars) if free_slots else scenarios.parking_lot_scenario(n_cars)
    rng = np.random.default_rng(seed)
    x0 = np.column_stack([rng.uniform(-9, 9, B), rng.uniform(6.8, 9.3, B), np.zeros(B), np.zeros(B)])      # start poses in the lane, v = 0
    if free_slots:
        ox, oy = sc["ox"], sc["oy"]
        xF = sc["goals"][np.arange(B) % len(sc["goals"])]                                           # car i -> free slot i mod n_slots
    else:
        ox, oy = scenarios.parking_lot_points(n_cars)
        xF = np.tile(sc["xF"], (B, 1))
    Ts = sc["Ts"] / 3 * sampleN
    t0 = time.time()
    r = device.plan_solve_goals(x0, xF, ox, oy, Ts, sc["nOb"], sc["vOb"], sc["A"], sc["b"], sc["ego"], sc["XYbounds"], sc["L"], sampleN,
                                signed_dist=signed_dist, host_fallback=True)
    ok = r["status"] == 0
    conv = ok & (r["exitflag"] == 1)
    return dict(B=B, n_planned=int(ok.sum()), status=r["status"].copy(), t_call=time.time() - t0, t_plan=r["plan_seconds"], t_solve=r["time"],
                n_converged=int(conv.sum()), n_clean=int((r["feasible"][conv] == 1).sum()), exitflag=r["exitflag"].astype(int), N=r["N"].copy(),
                per_slot=np.bincount(np.arange(B) % len(sc["goals"])).tolist() if free_slots else None)


if __name__ == "__main__":
    free = "--free-slots" in sys.argv
    a = [v for v in sys.argv if v != "--free-slots"]
    try:
        o = run(int(a[1]) if len(a) > 1 else 64, int(a[3]) if len(a) > 3 else 0, int(a[2]) if len(a) > 2 else 10,
                sampleN=int(a[4]) if len(a) > 4 else 3, free_slots=free)
    except obca_b200.ObcaError as e:
        print("not run:", e); sys.exit(2)
    miss = np.flatnonzero(o["status"] != 0)
    print(f"{o['B']} start poses: {o['n_planned']} planned on the GPU in {o['t_plan']:.2f} s device time"
          + (f" (not planned: poses {miss.tolist()}, status {o['status'][miss].tolist()})" if miss.size else "")
          + f"; solved in the same GPU call in {o['t_solve'] * 1e3:.0f} ms device time ({o['t_call']:.2f} s wall clock for the call): "
          f"{o['n_converged']} converged, "
          f"{o['n_clean']} of them pass ParkingConstraints" + (f"; cars per free slot {o['per_slot']}" if free else ""))
