"""Golden solutions of a parking problem with a horizon past 127 steps: the start pose of the reference's main.jl
(x0 = [-6, 9.5, 0], "backwards") planned by Hybrid A* (libobca_planner.so) at sampleN = 1, which gives N = 192 and Ts = 0.2
(main.jl:46-57: Ts = 0.6 / 3 * sampleN), solved with the ORACLE solver (oracle/ipm_ref.py with the sparse LDL' on the restated
reference NLP).

Run in the build container:  PYTHONPATH=. python tests/golden/make_long_parking_golden.py [case ...]
Stored in tests/golden/long_park/<case>.npz.  Each file holds the warm start (rx, ry, ryaw, xWS, uWS) and the DualMultWS result
(lWS, nWS, dWS) next to the solution, so that the tests do not depend on re-planning.
"""
import sys
import time

import numpy as np

from obca_b200 import scenarios
from obca_b200.planner import native
from oracle import ipm_ref
from oracle.dualmultws_ref import dualmultws
from oracle.parking_solve import solve_parking

X0 = np.array([-6.0, 9.5, 0.0, 0.0])      # main.jl:213
SAMPLE_N = 1
CASES = {
    "main_sd_n1": "sd",      # name: variant (variable time, fixTime = 0)
    "main_d_n1": "d",
}


def main(names):
    sc = scenarios.reverse_parking_scenario()
    w = native.plan_warm_start(X0[:3], sc["xF"], "backwards", None, sc["L"], SAMPLE_N)
    N, Ts = int(w["N"]), float(w["Ts"])
    xWS = np.asarray(w["xWS"], float)[:N + 1]
    uWS = np.asarray(w["uWS"], float)[:N]
    lWS, nWS, d = dualmultws(N, sc["nOb"], sc["vOb"], sc["A"], sc["b"], w["rx"], w["ry"], w["ryaw"], sc["ego"])
    for name in names:
        variant = CASES[name]
        t0 = time.time()
        out, res, nlp = solve_parking(X0, sc["xF"], N, Ts, sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"], sc["b"],
                                      w["rx"], w["ry"], w["ryaw"], 0, xWS, uWS, variant, lWS, nWS, ipm_ref.IpmOptions(linsolve="sparse"))
        xp, up, ts, exitflag, dt, lp, npp = out
        sl = nlp.lay.unpack(res.z)[5]
        print(name, "N", N, "Ts", Ts, "status", res.status, "iters", res.iters, "err", res.err, "f", nlp.f(res.z),
              "time", round(time.time() - t0, 1), flush=True)
        np.savez_compressed(f"tests/golden/long_park/{name}.npz", scenario="reverse", variant=variant, fixTime=0, sampleN=SAMPLE_N,
                            N=N, Ts=Ts, x0=X0, rx=w["rx"], ry=w["ry"], ryaw=w["ryaw"], xWS=xWS, uWS=uWS, lWS=lWS, nWS=nWS, dWS=d,
                            xp=xp, up=up, ts=ts, lp=lp, np=npp, sl=sl if sl is not None else np.zeros(0), f=nlp.f(res.z),
                            status=res.status, iters=res.iters, err=res.err)


if __name__ == "__main__":
    main(sys.argv[1:] or list(CASES))
