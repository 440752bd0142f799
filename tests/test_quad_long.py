"""A*-planned quadcopter pairs whose horizon exceeds 127 stages, CPU side: the fixture of the GPU tests
(tests/golden/quad_astar_long_pairs.npz) is what the planner gives, and the kernel sources, run through the development
emulation, solve every pair of it to a KKT point of the reference NLP that the verbatim constrSatisfaction accepts."""
import os

import numpy as np
import pytest

import emul
import emul_quad_mixed
from obca_b200 import scenarios
from oracle import checkers, kkt_check
from oracle.quadcopter_nlp import build_quadcopter_nlp

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "quad_astar_long_pairs.npz")


def test_long_fixture_is_what_the_planner_gives():
    """The pairs are the long ones of quadcopter_batch(64, seed=2) and corners of the start / goal box; one of each re-planned by
    the 3-D A* gives exactly the stored N, Ts and warm start."""
    from obca_b200.planner.a_star_3d import plan_quadcopter_warm_start
    g = np.load(GOLDEN)
    sc = scenarios.quadcopter_batch(64, seed=2)
    src = g["src"]
    assert (g["N"] > 127).all() and (src >= 0).any() and (src < 0).any()
    assert np.array_equal(g["x0"][src >= 0], sc["x0"][src[src >= 0]]) and np.array_equal(g["xF"][src >= 0], sc["xF"][src[src >= 0]])
    for i in (int(np.argmax(src >= 0)), int(np.argmax(g["N"]))):
        p = plan_quadcopter_warm_start(g["x0"][i], g["xF"][i], sc["Ts80"])
        N = int(g["N"][i])
        assert p["N"] == N and p["Ts"] == g["Ts"][i]
        assert np.array_equal(p["xWS"], g["xWS"][i][:, :N + 1]) and np.isnan(g["xWS"][i][:, N + 1:]).all()


@pytest.mark.parametrize("variant", ["sd", "d"])
def test_emulated_solve_of_long_planned_pairs(variant):
    """Every fixture pair, in one emulated batch laid out for its longest horizon, converges; the result passes the verbatim
    constrSatisfaction and its reference-formulation KKT error is below 1e-4."""
    g = np.load(GOLDEN)
    sc = scenarios.quadcopter_scenario()
    Ns = g["N"]
    sc.update(Ns=Ns, Ts=g["Ts"], x0=g["x0"], xF=g["xF"], xWS=[g["xWS"][i][:, :int(n) + 1] for i, n in enumerate(Ns)], timeWS=1.0)
    o = emul.default_opts(); o.max_iter = 3000
    r = emul_quad_mixed.quad_solve_mixed(sc, int(Ns.max()), variant, o)
    assert (r["status"] == 1).all(), r["status"]
    for i, n in enumerate(Ns):
        n = int(n)
        xp, up, ts, lp, sl = r["xp"][i][:, :n + 1], r["up"][i][:, :n], r["ts"][i][:n + 1], r["lp"][i][:, :n + 1], r["slack"][i][:, :n + 1]
        assert checkers.constrSatisfaction(xp, up, ts, g["x0"][i], g["xF"][i], g["Ts"][i], lp, *sc["obs"], sc["R"]), i
        nlp = build_quadcopter_nlp(g["x0"][i], g["xF"][i], n, float(g["Ts"][i]), sc["R"], sc["obs"], variant)
        e = kkt_check.kkt_certificate(nlp, nlp.lay.pack(xp, up, ts, lp, sl if variant == "sd" else None))
        assert e["E0"] < 1e-4, (i, n, e["E0"])
