"""The GPU Hybrid A* planner (obca_plan_parking_warmstart_batch) on the 512-pose sweeps of examples/sweep_parking.py: the host planner's
status and horizon for every pose, the emulation's expansion count, paths and warm starts within 1e-9 of the host's (the device's
sin / cos / atan2 / acos / tan / atan differ from glibc's in the last bits), untouched output padding, and warm starts the solver
accepts as often as the host-planned ones."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
import emul_plan                                                        # noqa: E402
from obca_b200.planner import device, native                            # noqa: E402

pytestmark = pytest.mark.gpu
GOAL = {"backwards": (0.0, 1.3, math.pi / 2), "parallel": (-1.35, 4.0, 0.0)}
TS = {"backwards": 0.6, "parallel": 0.9}


def sweep_poses(B, seed=0):
    rng = np.random.default_rng(seed)
    return np.column_stack([rng.uniform(-9, 9, B), rng.uniform(6.8, 9.3, B), np.zeros(B)])


def _decisions(o, e, plans):
    """Poses where the device decided differently from the host planner / the emulation (reported, never tolerated)."""
    bad = []
    for i, w in enumerate(plans):
        st, n = (1, -1) if w is None else (0, w["N"])
        if o["status"][i] != st or (st == 0 and o["N"][i] != n) or o["expansions"][i] != e["expansions"][i]:
            bad.append((i, "status/N/expansions", (int(o["status"][i]), int(o["N"][i]), int(o["expansions"][i])),
                        (st, n, int(e["expansions"][i]))))
    return bad


@pytest.mark.parametrize("scenario", ["backwards", "parallel"])
def test_gpu_plans_match_host_planner(scenario):
    x0 = sweep_poses(512)
    ox, oy = native.obstacle_points(scenario)
    o = device.plan_raw(x0, GOAL[scenario], ox, oy, TS[scenario])
    e = emul_plan.plan_raw(x0, GOAL[scenario], ox, oy, TS[scenario])
    plans = native.plan_batch(x0, GOAL[scenario], scenario)
    bad = _decisions(o, e, plans)
    assert not bad, bad[:10]
    worst = 0.0
    for i, w in enumerate(plans):
        if w is None:
            assert np.isnan(o["rx"][i]).all() and np.isnan(o["xWS"][i]).all()
            continue
        n = w["N"]
        got = dict(rx=o["rx"][i, :n + 1], ry=o["ry"][i, :n + 1], ryaw=o["ryaw"][i, :n + 1],
                   xWS=o["xWS"][i, :4 * (n + 1)].reshape(4, n + 1).T, uWS=o["uWS"][i, :2 * n].reshape(2, n).T)
        for k, v in got.items():
            d = float(np.abs(v - w[k]).max())
            worst = max(worst, d)
            assert d <= 1e-9, (i, k, d)
        assert np.isnan(o["rx"][i, n + 1:]).all() and np.isnan(o["ryaw"][i, n + 1:]).all()
        assert np.isnan(o["xWS"][i, 4 * (n + 1):]).all() and np.isnan(o["uWS"][i, 2 * n:]).all()
    print(f"{scenario}: 512 poses, same decisions, max |device - host| = {worst:.2e}, kernel {o['seconds'] * 1e3:.1f} ms, "
          f"max expansions {o['expansions'].max()}")


def test_gpu_capacity_and_pool_codes_as_emulated():
    ox, oy = native.obstacle_points("backwards")
    x0, xF = sweep_poses(8), GOAL["backwards"]
    full = emul_plan.plan_raw(x0, xF, ox, oy, 0.6)
    cap = int(np.median(full["N"])) + 1
    small = int(np.median(full["expansions"]))
    for kw in (dict(cap=cap), dict(max_nodes=small), dict(cap=cap, max_nodes=small)):
        o = device.plan_raw(x0, xF, ox, oy, 0.6, **kw)
        e = emul_plan.plan_raw(x0, xF, ox, oy, 0.6, **kw)
        assert np.array_equal(o["status"], e["status"]) and np.array_equal(o["N"], e["N"]), (kw, o["status"], e["status"])
        assert set(o["status"].tolist()) - {0}, kw
        for i in np.nonzero(o["status"] != 0)[0]:
            for k in ("rx", "ry", "ryaw", "xWS", "uWS"):
                assert np.isnan(o[k][i]).all(), (kw, i, k)


def test_gpu_plan_batch_plans_pool_full_poses_on_the_host():
    x0, xF = sweep_poses(16, seed=1), GOAL["backwards"]
    ox, oy = native.obstacle_points("backwards")
    small = int(np.median(emul_plan.plan_raw(x0, xF, ox, oy, 0.6)["expansions"]))
    st = device.plan_raw(x0, xF, ox, oy, 0.6, max_nodes=small)["status"]
    assert (st == device.POOL_FULL).any() and (st == 0).any(), st
    got, host = device.plan_batch(x0, xF, "backwards", max_nodes=small), native.plan_batch(x0, xF, "backwards")
    for i, (g, h) in enumerate(zip(got, host)):
        assert (g is None) == (h is None) and (h is None or g["N"] == h["N"]), i
        if h is not None:
            for k in ("rx", "ry", "ryaw", "xWS", "uWS"):
                d = np.abs(g[k] - h[k]).max()
                assert (d == 0.0) if st[i] == device.POOL_FULL else (d <= 1e-9), (i, k, d)


def test_gpu_no_path_in_a_mixed_batch_as_emulated():
    """Searches that end in NO_PATH -- an empty heap after one expansion, or the expansion budget -- next to searches that find a path,
    in one call: the emulation's status, N and expansion count for every pose, its values within 1e-9, nothing written for the others."""
    from test_plan_device import enclosed_batch
    x0, xF, ox, oy = enclosed_batch()
    x0 = np.concatenate([x0, sweep_poses(27, seed=3)])                  # 32 poses: more than one per warp of the CTA
    for budget in (0, 40):
        o = device.plan_raw(x0, xF, ox, oy, 0.6, max_expansions=budget)
        e = emul_plan.plan_raw(x0, xF, ox, oy, 0.6, max_expansions=budget)
        assert np.array_equal(o["status"], e["status"]) and np.array_equal(o["N"], e["N"]), (budget, o["status"], e["status"])
        assert np.array_equal(o["expansions"], e["expansions"]), budget
        assert (o["status"] == 1).sum() >= 2 and (o["status"] == 0).sum() >= 2, (budget, o["status"])
        for i in range(len(x0)):
            if o["status"][i] != 0:
                for k in ("rx", "ry", "ryaw", "xWS", "uWS"):
                    assert np.isnan(o[k][i]).all(), (budget, i, k)
                continue
            n = int(o["N"][i])
            for k, m in (("rx", n + 1), ("ry", n + 1), ("ryaw", n + 1), ("xWS", 4 * (n + 1)), ("uWS", 2 * n)):
                assert np.abs(o[k][i, :m] - e[k][i, :m]).max() <= 1e-9, (budget, i, k)
                assert np.isnan(o[k][i, m:]).all(), (budget, i, k)


def test_gpu_warm_starts_solve_like_host_ones():
    """Both 512-pose sweeps, planned on the GPU, then solved in one mixed-horizon call and checked: as many converge and pass
    ParkingConstraints as with the host-planned warm starts."""
    from obca_b200 import parking, scenarios
    ego = np.array([3.7, 1.0, 1.0, 1.0]); XYbounds = np.array([-15.0, 15.0, 1.0, 10.0])
    for scenario in ("backwards", "parallel"):
        sc = scenarios.reverse_parking_scenario() if scenario == "backwards" else scenarios.parallel_parking_scenario(4)
        x0 = np.column_stack([sweep_poses(512), np.zeros(512)])
        counts = []
        for plans in (native.plan_batch(x0, sc["xF"], scenario), device.plan_batch(x0, sc["xF"], scenario)):
            idx = [i for i, w in enumerate(plans) if w is not None]
            g = lambda k: [plans[i][k] for i in idx]
            Ns = np.array([plans[i]["N"] for i in idx])
            Ts = plans[idx[0]]["Ts"]
            r = parking.parking_solve_mixed(x0[idx], sc["xF"], Ns, Ts, 2.7, ego, XYbounds, sc["nOb"], sc["vOb"], sc["A"], sc["b"], g("rx"),
                                            g("ry"), g("ryaw"), 0, g("xWS"), g("uWS"), 1)
            feas, _, _ = parking.check_parking_mixed(x0[idx], sc["xF"], Ns, Ts, 2.7, ego, XYbounds, sc["nOb"], sc["vOb"], sc["A"], sc["b"],
                                                     r["xp"], r["up"], r["lp"], r["np"], r["ts"], 0, 1, r["sl"])
            counts.append((len(idx), int((r["exitflag"] == 1).sum()), int(np.asarray(feas).sum())))
        print(scenario, "host (planned, converged, feasible):", counts[0], "gpu:", counts[1])
        assert counts[1][0] == counts[0][0] and counts[1][1] >= counts[0][1] and counts[1][2] >= counts[0][2], (scenario, counts)
