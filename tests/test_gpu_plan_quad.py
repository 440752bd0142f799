"""The GPU 3-D A* planner (obca_plan_quadcopter_warmstart_batch) against the host library obca_astar3d_batch: the same status, N, path
(exact) and expansion count for the planned fixture pairs and 512 config-4 pairs, the right outcomes and untouched outputs in a batch that
mixes paths, NO_PATH and POOL_FULL, and GPU-planned warm starts that the quadcopter solver converges from."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import emul_plan3d                                                      # noqa: E402
from obca_b200 import scenarios                                         # noqa: E402
from obca_b200.planner import device, native                            # noqa: E402

pytestmark = pytest.mark.gpu
OUT = ("rx", "ry", "rz", "N", "status", "expansions")


def _pairs():
    x0, xF = [], []
    for f in ("quad_astar_pairs", "quad_astar_long_pairs"):
        z = np.load(os.path.join(ROOT, "tests", "golden", f + ".npz"))
        x0.append(z["x0"]); xF.append(z["xF"])
    sc = scenarios.quadcopter_batch(512, seed=2)
    return np.concatenate(x0 + [sc["x0"]]), np.concatenate(xF + [sc["xF"]])


def test_gpu_plans_equal_host_library():
    x0, xF = _pairs()
    args = native.quadcopter_problem(x0, xF)
    g = device.plan_quadcopter_raw(*args)
    h = native.astar3d_raw(*args)
    bad = [i for i in range(len(x0)) if any(not np.array_equal(g[k][i], h[k][i], equal_nan=True) for k in OUT)]
    assert not bad, [(i, int(g["status"][i]), int(h["status"][i]), int(g["expansions"][i]), int(h["expansions"][i])) for i in bad[:10]]
    assert (g["status"] == 0).all()
    print(f"{len(x0)} pairs: identical to the host library, kernel {g['seconds']:.3f} s, expansions {g['expansions'].min()}.."
          f"{g['expansions'].max()}")
    plans = device.plan_quadcopter_batch(x0[:16], xF[:16])
    ref = native.plan_quadcopter_batch(x0[:16], xF[:16])
    for a, b in zip(plans, ref):
        assert a["N"] == b["N"] and a["Ts"] == b["Ts"] and np.array_equal(a["xWS"], b["xWS"])


def test_gpu_mixed_outcomes_keep_unwritten_entries():
    from test_plan_quad_native import mixed_world
    args = mixed_world()
    h = native.astar3d_raw(*args, cap=256)
    e = emul_plan3d.plan_raw(*args, max_nodes=1 << 16, max_queue=1 << 14, cap=256)
    small = int(np.sort(e["nodes"])[-2]) - 1
    for max_nodes in (0, small):
        g = device.plan_quadcopter_raw(*args, cap=256, max_nodes=max_nodes)
        ref = emul_plan3d.plan_raw(*args, max_nodes=max_nodes or (1 << 18), max_queue=max(max_nodes // 4, 64) if max_nodes else 1 << 16,
                                   cap=256)
        for k in OUT:
            assert np.array_equal(g[k], ref[k], equal_nan=True), (max_nodes, k)
        full = g["status"] == device.POOL_FULL
        assert (full.sum() >= 2) == bool(max_nodes), (max_nodes, g["status"])
        assert set(g["status"][~full].tolist()) == {0, 1}
        for k in OUT:
            assert np.array_equal(g[k][~full], h[k][~full], equal_nan=True), (max_nodes, k)
        bad = g["status"] != 0
        assert np.isnan(g["rx"][bad]).all() and np.isnan(g["rz"][bad]).all() and (g["N"][bad] == -1).all()
        for i in np.nonzero(~bad)[0]:
            assert np.isnan(g["rx"][i, g["N"][i] + 1:]).all()


def test_gpu_plan_batch_plans_pool_full_pairs_on_the_host():
    sc = scenarios.quadcopter_batch(8, seed=4)
    args = native.quadcopter_problem(sc["x0"], sc["xF"])
    small = int(np.median(emul_plan3d.plan_raw(*args)["nodes"]))
    st = device.plan_quadcopter_raw(*args, max_nodes=small)["status"]
    assert (st == device.POOL_FULL).any() and (st == 0).any(), st
    got, ref = device.plan_quadcopter_batch(sc["x0"], sc["xF"], max_nodes=small), native.plan_quadcopter_batch(sc["x0"], sc["xF"])
    for a, b in zip(got, ref):
        assert a["N"] == b["N"] and a["Ts"] == b["Ts"] and np.array_equal(a["xWS"], b["xWS"])
        assert all(np.array_equal(u, v) for u, v in zip(a["path"], b["path"]))


def test_gpu_planned_pairs_solve_and_pass_constr_satisfaction():
    from obca_b200 import quadcopter
    sc = scenarios.quadcopter_batch(64, seed=2)
    plans = device.plan_quadcopter_batch(sc["x0"], sc["xF"], sc["Ts80"])
    assert all(p is not None for p in plans)
    Ns = np.array([p["N"] for p in plans]); Ts = np.array([p["Ts"] for p in plans])
    r = quadcopter.quadcopter_solve_mixed(sc["x0"], sc["xF"], Ns, Ts, sc["R"], sc["obs"], [p["xWS"] for p in plans], 1.0, 1)
    feas, _ = quadcopter.check_quadcopter_mixed(r["xp"], r["up"], r["ts"], sc["x0"], sc["xF"], Ns, Ts, r["lp"], sc["obs"], sc["R"])
    print(f"64 GPU-planned pairs, N = {Ns.min()}..{Ns.max()}: {(r['exitflag'] == 1).sum()} converged, {np.asarray(feas).sum()} feasible")
    assert (r["exitflag"] == 1).all(), r["exitflag"]
    assert np.asarray(feas).all()
