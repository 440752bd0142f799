"""Writes tests/golden/quad_astar_pairs.npz: the first 8 config-4 start / goal pairs of scenarios.quadcopter_batch(12, seed=2),
each planned by the 3-D A* of obca_b200/planner/a_star_3d.py (mainQuadcopter.jl:114-137): x0, xF (8, 12), N (8,), Ts (8,),
and the position warm starts xWS padded with NaN to (8, 12, max N + 1).  The fixture keeps the slow host-side planner (8-11 s
per pair) out of the GPU tests; tests/test_quad_mixed.py re-plans two of the pairs and requires the stored values exactly.

    python tests/golden/make_quad_astar.py
"""
import os
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from obca_b200 import scenarios                                   # noqa: E402
from obca_b200.planner.a_star_3d import plan_quadcopter_warm_start  # noqa: E402

N_PAIRS = 8


def pairs():
    sc = scenarios.quadcopter_batch(12, seed=2)
    return sc["x0"][:N_PAIRS], sc["xF"][:N_PAIRS], sc["Ts80"]


def main():
    x0, xF, Ts80 = pairs()
    with ProcessPoolExecutor() as ex:
        plans = list(ex.map(plan_quadcopter_warm_start, x0, xF, [Ts80] * N_PAIRS))
    assert all(p is not None for p in plans)
    N = np.array([p["N"] for p in plans], np.int32)
    xWS = np.full((N_PAIRS, 12, int(N.max()) + 1), np.nan)
    for i, p in enumerate(plans):
        xWS[i, :, :p["N"] + 1] = p["xWS"]
    np.savez_compressed(os.path.join(HERE, "quad_astar_pairs.npz"), x0=x0, xF=xF, N=N,
                        Ts=np.array([p["Ts"] for p in plans]), xWS=xWS)
    print("N", N.tolist(), "Ts", [p["Ts"] for p in plans])


if __name__ == "__main__":
    main()
