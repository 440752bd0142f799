"""obca_parking_plan_solve_goals on the GPU: plan, solve and check a batch in one call gives, bit for bit, what the composed path gives on
the same inputs -- obca_plan_parking_warmstart_goals, then obca_parking_solve_mixed on the poses that planned, then
obca_check_parking_mixed -- in the caller's pose order, with every entry of a pose that was not solved (and past a solved pose's horizon)
left as the caller had it.  Also: NO_PATH, POOL_FULL and CAPACITY poses in one batch, B = 0 and a batch where nothing plans (no solve),
device memory after the call, and an ordinary mixed solve after it."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import ctypes as C                                   # noqa: E402

from obca_b200 import _lib, parking, scenarios       # noqa: E402
from obca_b200.planner import device, native         # noqa: E402
from test_plan_device import enclosed_batch          # noqa: E402

pytestmark = pytest.mark.gpu
EGO = np.array([3.7, 1.0, 1.0, 1.0]); XYB = np.array([-15.0, 15.0, 1.0, 10.0])


def sweep(B, seed=0):
    rng = np.random.default_rng(seed)
    return np.column_stack([rng.uniform(-9, 9, B), rng.uniform(6.8, 9.3, B), np.zeros(B), np.zeros(B)])


def composed(x0, xF, ox, oy, Ts, sc, Ncap, max_nodes=0, sd=1):
    """The three-call path on the same inputs: planner (stride 512), mixed solve of the poses planned to 2 <= N <= Ncap, mixed check."""
    B = x0.shape[0]
    xF = np.broadcast_to(np.asarray(xF, float).reshape(-1, 4), (B, 4))
    o = device.plan_goals_raw(x0, xF, ox, oy, Ts, sc["L"], 3, cap=512, max_nodes=max_nodes)
    st = o["status"].copy()
    st[(st == 0) & ((o["N"] < 2) | (o["N"] > Ncap))] = 2
    idx = np.flatnonzero(st == 0)
    r = dict(status=st, N=o["N"], expansions=o["expansions"], idx=idx)
    if idx.size == 0:
        return r
    Ns = o["N"][idx]
    rx = [o["rx"][i, :n + 1] for i, n in zip(idx, Ns)]; ry = [o["ry"][i, :n + 1] for i, n in zip(idx, Ns)]
    ryaw = [o["ryaw"][i, :n + 1] for i, n in zip(idx, Ns)]
    xWS = [o["xWS"][i, :4 * (n + 1)].reshape(4, n + 1).T for i, n in zip(idx, Ns)]
    uWS = [o["uWS"][i, :2 * n].reshape(2, n).T for i, n in zip(idx, Ns)]
    s = parking.parking_solve_mixed(x0[idx], xF[idx], Ns, Ts, sc["L"], EGO, XYB, sc["nOb"], sc["vOb"], sc["A"], sc["b"], rx, ry, ryaw, 0,
                                    xWS, uWS, sd)
    feas, _, strict = parking.check_parking_mixed(x0[idx], xF[idx], Ns, Ts, sc["L"], EGO, XYB, sc["nOb"], sc["vOb"], sc["A"], sc["b"],
                                                  s["xp"], s["up"], s["lp"], s["np"], s["ts"], 0, sd, s["sl"])
    r.update({k: v for k, v in s.items() if k != "N"}, feasible=feas, strict=strict)      # N: every pose's, from the planner
    return r


def one_call(x0, xF, ox, oy, Ts, sc, Ncap, max_nodes=0, sd=1):
    return device.plan_solve_goals_raw(x0, xF, ox, oy, Ts, sc["nOb"], sc["vOb"], sc["A"], sc["b"], EGO, XYB, sc["L"], 3, Ncap, 0, sd,
                                       max_nodes)


def assert_same(g, r, Ncap):
    """Every output of the one call equals the composed path's bit for bit; the rest keeps the sentinel fill (NaN, -1)."""
    B = len(g["status"])
    assert np.array_equal(g["status"], r["status"]), (g["status"], r["status"])
    assert np.array_equal(g["N"], r["N"]) and np.array_equal(g["expansions"], r["expansions"])
    solved = np.zeros(B, bool); solved[r["idx"]] = True
    for k, ext in (("xp", 1), ("up", 0), ("ts", 1), ("lp", 1), ("np", 1), ("sl", 1)):
        for q, i in enumerate(r["idx"]):
            n = int(r["N"][i])
            want = r[k][q] if k == "ts" else r[k][q].T
            assert np.array_equal(g[k][i, :n + ext], want), (k, i)
            assert np.isnan(g[k][i, n + ext:]).all(), (k, i)
        assert np.isnan(g[k][~solved]).all(), k
    for k in ("exitflag", "iters", "kkt_err", "feasible", "strict"):
        if r["idx"].size:
            assert np.array_equal(g[k][r["idx"]], np.asarray(r[k])), k
        unset = g[k][~solved]
        assert (np.isnan(unset) if k == "kkt_err" else unset == -1).all(), k


def test_backwards_sweep_one_goal_matches_composed_path():
    sc = scenarios.reverse_parking_scenario()
    ox, oy = native.obstacle_points("backwards")
    x0 = sweep(512, seed=0)
    g = one_call(x0, sc["xF"], ox, oy, 0.6, sc, 319)
    r = composed(x0, sc["xF"], ox, oy, 0.6, sc, 319)
    assert r["idx"].size >= 500, r["status"]
    assert_same(g, r, 319)
    assert g["plan_seconds"] > 0 and g["time"] > 0
    print(f"backwards, 512 poses: {r['idx'].size} solved, {int(g['exitflag'].sum())} converged, {int((g['feasible'] == 1).sum())} pass "
          f"ParkingConstraints; plan {g['plan_seconds'] * 1e3:.0f} ms, solve {g['time'] * 1e3:.0f} ms device time")


def test_free_slot_lot_goal_per_pose_matches_composed_path():
    lot = scenarios.parking_lot_free_slots()
    x0 = sweep(64, seed=1)
    xF = lot["goals"][np.arange(64) % len(lot["goals"])]
    g = one_call(x0, xF, lot["ox"], lot["oy"], lot["Ts"], lot, 319)
    r = composed(x0, xF, lot["ox"], lot["oy"], lot["Ts"], lot, 319)
    assert r["idx"].size >= 60, r["status"]
    assert_same(g, r, 319)
    out = device.plan_solve_goals(x0, xF, lot["ox"], lot["oy"], lot["Ts"], lot["nOb"], lot["vOb"], lot["A"], lot["b"], EGO, XYB, lot["L"])
    for q, i in enumerate(r["idx"]):
        assert np.array_equal(out["xp"][i], r["xp"][q]) and np.array_equal(out["lp"][i], r["lp"][q])
    assert all(out["xp"][i] is None for i in range(64) if i not in set(r["idx"].tolist()))


def test_no_path_pool_full_and_capacity_in_one_batch():
    """Two poses boxed in by a dense patch of points (NO_PATH), a node pool small enough that some searches outgrow it (POOL_FULL) and
    an Ncap below some planned horizons (CAPACITY), next to poses that are solved."""
    x0e, _, ox, oy = enclosed_batch()
    sc = scenarios.reverse_parking_scenario()
    x0 = np.concatenate([np.column_stack([x0e, np.zeros(len(x0e))]), sweep(43, seed=5)])
    for max_nodes in (128, 256, 512, 1024, 2048):
        st = device.plan_goals_raw(x0, sc["xF"], ox, oy, 0.6, max_nodes=max_nodes)
        if (st["status"] == 4).sum() >= 2 and (st["status"] == 0).sum() >= 6:
            break
    Ncap = int(np.median(st["N"][st["status"] == 0]))
    g = one_call(x0, sc["xF"], ox, oy, 0.6, sc, Ncap, max_nodes=max_nodes)
    r = composed(x0, sc["xF"], ox, oy, 0.6, sc, Ncap, max_nodes=max_nodes)
    for code in (0, 1, 2, 4):
        assert (g["status"] == code).sum() >= 1, (code, g["status"])
    assert (g["N"][g["status"] == 2] > Ncap).all()
    assert (g["N"][g["status"] == 1] == -1).all()
    assert_same(g, r, Ncap)
    print(f"max_nodes {max_nodes}, Ncap {Ncap}: status counts {np.bincount(g['status'], minlength=5).tolist()}")
    # host_fallback: the POOL_FULL poses get the host twin's plans, solved and checked; every other pose keeps the one call's outputs
    # (at Ncap = 319, so that the long searches which outgrew the pool are solved, not CAPACITY)
    g = one_call(x0, sc["xF"], ox, oy, 0.6, sc, 319, max_nodes=max_nodes)
    h = device.plan_solve_goals_raw(x0, sc["xF"], ox, oy, 0.6, sc["nOb"], sc["vOb"], sc["A"], sc["b"], EGO, XYB, sc["L"], 3, 319, 0, 1,
                                    max_nodes, host_fallback=True)
    full = g["status"] == 4
    tw = native.plan_cloud_raw(x0[full], sc["xF"], ox, oy, 0.6)
    want = tw["status"].copy(); want[(want == 0) & ((tw["N"] < 2) | (tw["N"] > 319))] = 2
    assert np.array_equal(h["status"][full], want) and np.array_equal(h["N"][full], tw["N"])
    assert (h["status"] != 4).all() and (want == 0).any(), want
    for k in ("xp", "up", "ts", "lp", "np", "sl", "N", "status", "expansions", "exitflag", "iters", "kkt_err", "feasible", "strict"):
        assert np.array_equal(h[k][~full], g[k][~full], equal_nan=k in ("xp", "up", "ts", "lp", "np", "sl", "kkt_err")), k
    for i in np.flatnonzero(full)[want == 0]:
        n = int(h["N"][i])
        assert np.isfinite(h["xp"][i, :n + 1]).all() and np.isnan(h["xp"][i, n + 1:]).all() and h["exitflag"][i] in (0, 1), i
        assert h["feasible"][i] in (0, 1) and h["iters"][i] > 0, i


def _last_times():
    d = C.c_double(0.0); s = C.c_double(0.0)
    _lib.check(_lib.lib().obca_last_times(0, C.byref(d), C.byref(s)))
    return d.value, s.value


def _small_mixed_solve():
    sc = scenarios.reverse_parking_scenario()
    ox, oy = native.obstacle_points("backwards")
    x0 = sweep(16, seed=7)
    r = composed(x0, sc["xF"], ox, oy, 0.6, sc, 319)
    return {k: r[k] for k in ("xp", "up", "ts", "lp", "np", "sl", "exitflag", "iters", "kkt_err")}


def test_empty_batch_and_nothing_planned_run_no_solve():
    _small_mixed_solve()
    before = _last_times()
    sc = scenarios.reverse_parking_scenario()
    x0e, _, ox, oy = enclosed_batch()
    g = one_call(np.zeros((0, 4)), sc["xF"], ox, oy, 0.6, sc, 319)
    assert g["time"] == 0.0 and g["plan_seconds"] == 0.0
    boxed = np.column_stack([x0e[[0, 4]], np.zeros(2)])
    g = one_call(boxed, sc["xF"], ox, oy, 0.6, sc, 319)
    assert g["status"].tolist() == [1, 1] and g["time"] == 0.0
    for k in ("xp", "up", "ts", "lp", "np", "sl", "kkt_err"):
        assert np.isnan(g[k]).all(), k
    for k in ("exitflag", "iters", "feasible", "strict"):
        assert (g[k] == -1).all(), k
    assert _last_times() == before


def test_planner_scratch_is_freed_and_next_mixed_solve_is_unchanged():
    import torch
    ref = _small_mixed_solve()
    sc = scenarios.reverse_parking_scenario()
    ox, oy = native.obstacle_points("backwards")
    x0 = sweep(640, seed=3)                       # more poses than resident planner CTAs: the full planner scratch
    torch.cuda.init()
    one_call(x0, sc["xF"], ox, oy, 0.6, sc, 319)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info(0)
    one_call(x0, sc["xF"], ox, oy, 0.6, sc, 319)
    torch.cuda.synchronize()
    free2, _ = torch.cuda.mem_get_info(0)
    assert abs(free1 - free2) <= 1 << 20, (free1, free2)
    again = _small_mixed_solve()
    for k in ref:
        if isinstance(ref[k], list):
            assert all(np.array_equal(a, b) for a, b in zip(ref[k], again[k])), k
        else:
            assert np.array_equal(ref[k], again[k]), k
