"""Writes tests/golden/quad_astar_long_pairs.npz: A*-planned config-4 start / goal pairs whose horizon exceeds 127 stages,
the range that needs more than one stage per thread in the quadcopter solver.  The pairs are

  - those of scenarios.quadcopter_batch(64, seed=2) that the 3-D A* of obca_b200/planner/a_star_3d.py plans with N > 127, and
  - the corners (1, Y, Z0) -> (9, Y, ZF) of the start / goal box of mainQuadcopter.jl:48-51, Y in {0.5, 9.5}, Z0 and ZF in
    {0.5, 4.5}, that the planner gives N > 127.

Arrays: x0, xF (P, 12), N (P,), Ts (P,), the position warm starts xWS padded with NaN to (P, 12, max N + 1), and src (P,):
the index of the pair in quadcopter_batch(64, seed=2), -1 for a corner.  Planning takes 8-11 s per pair on host processes;
tests/test_quad_long.py re-plans two of the pairs and requires the stored values exactly.

    python tests/golden/make_quad_astar_long.py
"""
import itertools
import os
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from obca_b200 import scenarios                                   # noqa: E402
from obca_b200.planner.a_star_3d import plan_quadcopter_warm_start  # noqa: E402

N_BATCH = 64
N_SHORT = 127      # longest horizon that fits one stage per thread


def corners():
    x0, xF = [], []
    for Y, Z0, ZF in itertools.product((0.5, 9.5), (0.5, 4.5), (0.5, 4.5)):
        a = np.zeros(12); a[:3] = (1.0, Y, Z0)
        b = np.zeros(12); b[:3] = (9.0, Y, ZF)
        x0.append(a); xF.append(b)
    return np.array(x0), np.array(xF)


def candidates():
    sc = scenarios.quadcopter_batch(N_BATCH, seed=2)
    cx0, cxF = corners()
    src = np.concatenate([np.arange(N_BATCH), np.full(len(cx0), -1)])
    return np.concatenate([sc["x0"], cx0]), np.concatenate([sc["xF"], cxF]), src, sc["Ts80"]


def main():
    x0, xF, src, Ts80 = candidates()
    with ProcessPoolExecutor() as ex:
        plans = list(ex.map(plan_quadcopter_warm_start, x0, xF, [Ts80] * len(x0)))
    keep = [i for i, p in enumerate(plans) if p is not None and p["N"] > N_SHORT]
    N = np.array([plans[i]["N"] for i in keep], np.int32)
    xWS = np.full((len(keep), 12, int(N.max()) + 1), np.nan)
    for k, i in enumerate(keep):
        xWS[k, :, :plans[i]["N"] + 1] = plans[i]["xWS"]
    np.savez_compressed(os.path.join(HERE, "quad_astar_long_pairs.npz"), x0=x0[keep], xF=xF[keep], N=N,
                        Ts=np.array([plans[i]["Ts"] for i in keep]), xWS=xWS, src=src[keep].astype(np.int32))
    print("all N", [p["N"] if p else None for p in plans])
    print("kept src", src[keep].tolist(), "N", N.tolist(), "Ts", [plans[i]["Ts"] for i in keep])


if __name__ == "__main__":
    main()
