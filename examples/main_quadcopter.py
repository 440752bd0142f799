"""The flow of the reference's QuadcopterNavigation/mainQuadcopter.jl: environment and 3-D A* (mainQuadcopter.jl:36-128), warm
start (:130-137), QuadcopterDist and QuadcopterSignedDist on the GPU (:145, :152), constrSatisfaction (:147, :154).

usage: python examples/main_quadcopter.py [Y0 Z0 YF ZF]                            (needs a CUDA device for the two solves)

Y0 Z0 YF ZF: the start (1, Y0, Z0) and the goal (9, YF, ZF) the reference asks its user to edit (mainQuadcopter.jl:48-51);
by default the reference's (1, 1, 3) -> (9, 3, 2).  Corners of the box, e.g. 9.5 4.5 9.5 4.5, plan horizons up to N = 147.
"""
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import obca_b200                                            # noqa: E402
from obca_b200 import scenarios                             # noqa: E402
from obca_b200.planner import a_star_3d                     # noqa: E402


def main(argv):
    sc = scenarios.quadcopter_scenario()
    x0, xF, R = sc["x0"].copy(), sc["xF"].copy(), sc["R"]
    if argv:
        if len(argv) != 4:
            print(__doc__); return 2
        x0[1], x0[2], xF[1], xF[2] = (float(a) for a in argv)
    t0 = time.time()
    w = a_star_3d.plan_quadcopter_warm_start(x0, xF, sc["Ts80"])
    if w is None:
        print("A*: no path found"); return 1
    N, Ts = w["N"], w["Ts"]
    print(f"A*: N = {N}, Ts = {Ts:.2f} ({time.time() - t0:.1f} s)")
    obs = sc["obs"]
    try:
        for name, fn in (("Distance Approach", obca_b200.QuadcopterDist), ("Signed Distance Approach", obca_b200.QuadcopterSignedDist)):
            xp, up, ts, exitflag, t, lp, status = fn(x0[None], xF[None], N, Ts, R, *obs, w["xWS"], w["uWS"], w["timeWS"])
            feas = obca_b200.constrSatisfaction(xp, up, ts, x0[None], xF[None], Ts, lp, *obs, R)
            print(f"Trajectory using {name}: exitflag {exitflag} ({status}), solve time {t * 1e3:.1f} ms, constrSatisfaction {feas}, "
                  f"flight time {float(np.sum(ts[:-1]) * Ts):.2f} s")
    except obca_b200.ObcaError as e:
        print("solve not run:", e)
        return 2
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
