"""The flow of the reference's AutonomousParking/main.jl with this repository's pieces (host side in Python because the image
has no Julia; julia/OBCA.jl holds the equivalent ccall shims for the reference tree):

    scenario constants (main.jl:36-108, 207-213)  ->  Hybrid A* path (main.jl:215-219)  ->  speed / steering profile and
    down-sampling (main.jl:222-248)  ->  obstHrep (main.jl:252)  ->  ParkingDist and ParkingSignedDist (main.jl:258, 269) on the GPU
    ->  ParkingConstraints (the reference's acceptance test)

sampleN (last argument, default 3) is the warm-start sampling of main.jl:46-57: Ts = 0.6 / 3 * sampleN ("backwards", 0.9 for
"parallel").  The reference's own pose at sampleN = 1 gives N = 192.

usage: python examples/main_parking.py [backwards|parallel] [x0 y0 yaw0] [sampleN]          (needs a CUDA device for the two solves)
"""
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import obca_b200                                            # noqa: E402
from obca_b200 import scenarios                             # noqa: E402
from obca_b200.planner import warmstart                     # noqa: E402


def main(argv):
    scenario = argv[1] if len(argv) > 1 else "backwards"
    sc = scenarios.reverse_parking_scenario() if scenario == "backwards" else scenarios.parallel_parking_scenario(4)
    x0 = np.array([float(v) for v in argv[2:5]] + [0.0]) if len(argv) >= 5 else np.array([-6.0, 9.5, 0.0, 0.0])       # main.jl:213
    sampleN = int(argv[-1]) if len(argv) in (3, 6) else 3                                                             # main.jl:46
    xF, L, fixTime = sc["xF"], 2.7, 0
    ego = np.array([3.7, 1.0, 1.0, 1.0])                     # main.jl:72-73
    XYbounds = np.array([-15.0, 15.0, 1.0, 10.0])            # main.jl:209-210
    t0 = time.time()
    w = warmstart.plan_warm_start(x0, xF, scenario, sampleN=sampleN)      # Hybrid A* + main.jl:222-248
    if w is None:
        print("Hybrid A*: no path found"); return 1
    N, Ts = w["N"], w["Ts"]
    print(f"Hybrid A*: {len(w['path'][0])} path points, N = {N}, Ts = {Ts:.3f} ({time.time() - t0:.2f} s)")
    args = (x0[None], xF[None], N, Ts, L, ego, XYbounds, sc["nOb"], sc["vOb"], sc["A"], sc["b"], w["rx"], w["ry"], w["ryaw"], fixTime,
            w["xWS"], w["uWS"][:N])
    try:
        for name, fn, sd in (("Distance Approach", obca_b200.ParkingDist, 0), ("Signed Distance Approach", obca_b200.ParkingSignedDist, 1)):
            xp, up, ts, exitflag, t, lp, np_ = fn(*args)
            ok = obca_b200.ParkingConstraints(x0[None], xF[None], N, Ts, L, ego, XYbounds, sc["nOb"], sc["vOb"], sc["A"], sc["b"], xp, up, lp, np_, ts,
                                              fixTime, sd)
            print(f"Parking using {name}: exitflag {exitflag}, solve time {t * 1e3:.1f} ms, ParkingConstraints {'passed' if ok else 'FAILED'}, "
                  f"final pose ({xp[0, -1]:.3f}, {xp[1, -1]:.3f}, {xp[2, -1]:.3f}), time scale {ts.ravel()[0]:.3f}")
    except obca_b200.ObcaError as e:
        print("solve not run:", e)
        return 2
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv))
