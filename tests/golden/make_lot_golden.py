"""Golden solutions of the car-park scene (obca_b200.scenarios.parking_lot_batch: 10 parked cars + the far wall, 11 obstacles,
41 half-spaces, N = 80, seed 0) with the ORACLE solver (oracle/ipm_ref.py with the sparse LDL' on the restated reference NLP).

Run in the build container:  PYTHONPATH=. python tests/golden/make_lot_golden.py [case ...]
Stored in tests/golden/lot/<case>.npz in the format of make_golden.py (scenario = "lot10"), so that the GPU test
(tests/test_gpu_many_obstacles.py) compares them the way test_gpu_parking.test_matches_oracle_golden compares the others.
"""
import sys
import time

import numpy as np

from obca_b200.scenarios import parking_lot_batch
from oracle import ipm_ref
from oracle.dualmultws_ref import dualmultws
from oracle.parking_solve import solve_parking

N_CARS = 10
CASES = {
    "lot_sd_var_p0": (0, "sd", 0),      # name: (problem index, variant, fixTime)
    "lot_d_var_p1": (1, "d", 0),
}


def main(names):
    sc = parking_lot_batch(8, 80, 0, N_CARS)
    for name in names:
        i, variant, fix = CASES[name]
        Ts = sc["Ts_fix"] if fix else sc["Ts"]
        t0 = time.time()
        lWS, nWS, d = dualmultws(80, sc["nOb"], sc["vOb"], sc["A"], sc["b"], sc["rx"][i], sc["ry"][i], sc["ryaw"][i], sc["ego"])
        out, res, nlp = solve_parking(sc["x0"][i], sc["xF"], 80, Ts, sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"],
                                      sc["vOb"], sc["A"], sc["b"], sc["rx"][i], sc["ry"][i], sc["ryaw"][i], fix,
                                      sc["xWS"][i], sc["uWS"][i], variant, lWS, nWS, ipm_ref.IpmOptions(linsolve="sparse"))
        xp, up, ts, exitflag, dt, lp, npp = out
        sl = nlp.lay.unpack(res.z)[5]
        print(name, "status", res.status, "iters", res.iters, "err", res.err, "f", nlp.f(res.z), "time", time.time() - t0, flush=True)
        np.savez_compressed(f"tests/golden/lot/{name}.npz", scenario=f"lot{N_CARS}", index=i, variant=variant, fixTime=fix, seed=0,
                            N=80, lWS=lWS, nWS=nWS, dWS=d, xp=xp, up=up, ts=ts, lp=lp, np=npp,
                            sl=sl if sl is not None else np.zeros(0), f=nlp.f(res.z), status=res.status, iters=res.iters, err=res.err)


if __name__ == "__main__":
    main(sys.argv[1:] or list(CASES))
