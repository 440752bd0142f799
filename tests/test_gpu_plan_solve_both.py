"""obca_parking_plan_solve_both and obca_quadcopter_plan_solve_both on the GPU: one plan solved and checked with both formulations gives,
bit for bit, what the one-formulation entries give with signed_dist = 0 and 1 on the same inputs -- the shared outputs once, each set
including the entries left as the caller had them.  Also: NO_PATH, POOL_FULL and CAPACITY in one batch, with the host fallback planning
once; B = 0 and a batch where nothing plans (no solve); the times the library reports after the call; device memory after the call and an
ordinary mixed solve after it."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_gpu_plan_solve as pk                        # noqa: E402
import test_gpu_quad_plan_solve as qc                   # noqa: E402
from obca_b200 import _lib, scenarios                   # noqa: E402
from obca_b200.planner import device, native            # noqa: E402
from obca_b200.planner.a_star_3d import quadcopter_environment      # noqa: E402
from test_plan_device import enclosed_batch              # noqa: E402

pytestmark = pytest.mark.gpu
EGO, XYB = pk.EGO, pk.XYB
PK_SHARED = ("N", "status", "expansions")
QC_SHARED = ("N", "Tsb", "status", "expansions")


def park_both(x0, xF, ox, oy, Ts, sc, Ncap, max_nodes=0, host_fallback=False):
    return device.plan_solve_goals_both_raw(x0, xF, ox, oy, Ts, sc["nOb"], sc["vOb"], sc["A"], sc["b"], EGO, XYB, sc["L"], 3, Ncap, 0,
                                            max_nodes, host_fallback=host_fallback)


def park_one(x0, xF, ox, oy, Ts, sc, Ncap, sd, max_nodes=0, host_fallback=False):
    return device.plan_solve_goals_raw(x0, xF, ox, oy, Ts, sc["nOb"], sc["vOb"], sc["A"], sc["b"], EGO, XYB, sc["L"], 3, Ncap, 0, sd,
                                       max_nodes, host_fallback=host_fallback)


def quad_both(x0, xF, sc, Ncap, max_nodes=0, host_fallback=False):
    ox, oy, oz, lo, hi = quadcopter_environment()
    return device.plan_solve_quadcopter_both_raw(x0, xF, ox, oy, oz, lo, hi, 1.0, sc["Ts80"], sc["R"], sc["obs"], 1.0, Ncap, max_nodes,
                                                 host_fallback=host_fallback)


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()


def assert_sets_equal_one_formulation(both, one, shared, rows=None):
    """both (a *_both_raw result) against one[f] (the one-formulation *_raw result with signed_dist = f) for f = 0, 1: the shared outputs
    and every array of each set, bit for bit, sentinels included.  rows: compare the Dist set's sl on these problems only."""
    for f, name in ((0, "dist"), (1, "sd")):
        for k in shared:
            assert same_bits(both[k], one[f][k]), (name, k)
        assert set(both[name]) == set(one[f]) - set(shared) - {"plan_seconds"}, (name, sorted(both[name]))
        for k, v in both[name].items():
            if k == "sl" and name == "dist" and rows is not None:
                assert same_bits(v[rows], one[f][k][rows]), (name, k)
            elif k != "time":
                assert same_bits(v, one[f][k]), (name, k)


def merged(both, name):
    return dict(both[name], **{k: v for k, v in both.items() if k not in ("dist", "sd")})


# ---- parking --------------------------------------------------------------------------------------------------------------------------
def test_parking_backwards_sweep_matches_both_one_formulation_calls():
    sc = scenarios.reverse_parking_scenario()
    ox, oy = native.obstacle_points("backwards")
    x0 = pk.sweep(512, seed=0)
    g = park_both(x0, sc["xF"], ox, oy, 0.6, sc, 319)
    assert pk._last_times()[1] == g["sd"]["time"]      # the library's times report the Signed Distance solve, the last one
    one = [park_one(x0, sc["xF"], ox, oy, 0.6, sc, 319, f) for f in (0, 1)]
    assert_sets_equal_one_formulation(g, one, PK_SHARED)
    # the Dist set is pinned to the one-formulation entry above; the SD set also to the composed path, as tests/test_gpu_plan_solve.py does
    r = pk.composed(x0, sc["xF"], ox, oy, 0.6, sc, 319)
    assert r["idx"].size >= 500, r["status"]
    pk.assert_same(merged(g, "sd"), r, 319)
    assert g["dist"]["time"] > 0 and g["sd"]["time"] > 0
    assert g["plan_seconds"] > 0
    print(f"backwards, 512 poses: plan {g['plan_seconds'] * 1e3:.0f} ms; Dist {int(g['dist']['exitflag'].sum())} converged, "
          f"solve {g['dist']['time'] * 1e3:.0f} ms; SD {int(g['sd']['exitflag'].sum())} converged, solve {g['sd']['time'] * 1e3:.0f} ms")


def test_parking_free_slot_lot_goal_per_pose_matches_both_one_formulation_calls():
    lot = scenarios.parking_lot_free_slots()
    x0 = pk.sweep(64, seed=1)
    xF = lot["goals"][np.arange(64) % len(lot["goals"])]
    g = park_both(x0, xF, lot["ox"], lot["oy"], lot["Ts"], lot, 319)
    one = [park_one(x0, xF, lot["ox"], lot["oy"], lot["Ts"], lot, 319, f) for f in (0, 1)]
    assert_sets_equal_one_formulation(g, one, PK_SHARED)
    r = pk.composed(x0, xF, lot["ox"], lot["oy"], lot["Ts"], lot, 319)
    assert r["idx"].size >= 60, r["status"]
    pk.assert_same(merged(g, "sd"), r, 319)
    out = device.plan_solve_goals_both(x0, xF, lot["ox"], lot["oy"], lot["Ts"], lot["nOb"], lot["vOb"], lot["A"], lot["b"], EGO, XYB,
                                       lot["L"])
    for f, name in ((0, "dist"), (1, "sd")):
        ref = device.plan_solve_goals(x0, xF, lot["ox"], lot["oy"], lot["Ts"], lot["nOb"], lot["vOb"], lot["A"], lot["b"], EGO, XYB,
                                      lot["L"], signed_dist=f)
        for k in ("xp", "up", "ts", "lp", "np", "sl"):
            assert all((a is None and b is None) or same_bits(a, b) for a, b in zip(out[name][k], ref[k])), (name, k)
        for k in ("exitflag", "iters", "kkt_err", "feasible", "strict"):
            assert same_bits(out[name][k], ref[k]), (name, k)
        for k in ("N", "status", "expansions"):
            assert same_bits(out[k], ref[k]), k


def _count_calls(monkeypatch, name):
    calls = []
    fn = getattr(native, name)
    monkeypatch.setattr(native, name, lambda *a, **kw: calls.append(1) or fn(*a, **kw))
    return calls


def test_parking_no_path_pool_full_and_capacity_in_one_batch(monkeypatch):
    x0e, _, ox, oy = enclosed_batch()
    sc = scenarios.reverse_parking_scenario()
    x0 = np.concatenate([np.column_stack([x0e, np.zeros(len(x0e))]), pk.sweep(43, seed=5)])
    for max_nodes in (128, 256, 512, 1024, 2048):
        st = device.plan_goals_raw(x0, sc["xF"], ox, oy, 0.6, max_nodes=max_nodes)
        if (st["status"] == 4).sum() >= 2 and (st["status"] == 0).sum() >= 6:
            break
    Ncap = int(np.median(st["N"][st["status"] == 0]))
    g = park_both(x0, sc["xF"], ox, oy, 0.6, sc, Ncap, max_nodes)
    for code in (0, 1, 2, 4):
        assert (g["status"] == code).sum() >= 1, (code, g["status"])
    one = [park_one(x0, sc["xF"], ox, oy, 0.6, sc, Ncap, f, max_nodes) for f in (0, 1)]
    assert_sets_equal_one_formulation(g, one, PK_SHARED)
    pk.assert_same(merged(g, "sd"), pk.composed(x0, sc["xF"], ox, oy, 0.6, sc, Ncap, max_nodes), Ncap)
    # host_fallback: the POOL_FULL poses are planned once on the host, then solved with both formulations
    one = [park_one(x0, sc["xF"], ox, oy, 0.6, sc, 319, f, max_nodes, host_fallback=True) for f in (0, 1)]
    calls = _count_calls(monkeypatch, "plan_cloud_raw")
    h = park_both(x0, sc["xF"], ox, oy, 0.6, sc, 319, max_nodes, host_fallback=True)
    assert len(calls) == 1
    assert (h["status"] != 4).all(), h["status"]
    # the host-planned poses are solved by obca_parking_solve_mixed, whose sl output a Dist solve does not write: it holds whatever the
    # entry's staging buffer held, so the Dist set's sl is compared on the other poses only
    device_planned = park_one(x0, sc["xF"], ox, oy, 0.6, sc, 319, 1, max_nodes)["status"] != 4
    assert_sets_equal_one_formulation(h, one, PK_SHARED, rows=device_planned)


def test_parking_empty_batch_and_nothing_planned_run_no_solve():
    pk._small_mixed_solve()
    before = pk._last_times()
    sc = scenarios.reverse_parking_scenario()
    x0e, _, ox, oy = enclosed_batch()
    g = park_both(np.zeros((0, 4)), sc["xF"], ox, oy, 0.6, sc, 319)
    assert g["plan_seconds"] == 0.0 and g["dist"]["time"] == 0.0 and g["sd"]["time"] == 0.0
    g = park_both(np.column_stack([x0e[[0, 4]], np.zeros(2)]), sc["xF"], ox, oy, 0.6, sc, 319)
    assert g["status"].tolist() == [1, 1] and g["dist"]["time"] == 0.0 and g["sd"]["time"] == 0.0
    for name in ("dist", "sd"):
        for k in ("xp", "up", "ts", "lp", "np", "sl", "kkt_err"):
            assert np.isnan(g[name][k]).all(), (name, k)
        for k in ("exitflag", "iters", "feasible", "strict"):
            assert (g[name][k] == -1).all(), (name, k)
    assert pk._last_times() == before


def test_parking_device_memory_and_next_mixed_solve_are_unchanged():
    import torch
    ref = pk._small_mixed_solve()
    sc = scenarios.reverse_parking_scenario()
    ox, oy = native.obstacle_points("backwards")
    x0 = pk.sweep(640, seed=3)                       # more poses than resident planner CTAs: the full planner scratch
    torch.cuda.init()
    park_both(x0, sc["xF"], ox, oy, 0.6, sc, 319)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info(0)
    park_both(x0, sc["xF"], ox, oy, 0.6, sc, 319)
    torch.cuda.synchronize()
    free2, _ = torch.cuda.mem_get_info(0)
    assert abs(free1 - free2) <= 1 << 20, (free1, free2)
    again = pk._small_mixed_solve()
    for k in ref:
        if isinstance(ref[k], list):
            assert all(np.array_equal(a, b) for a, b in zip(ref[k], again[k])), k
        else:
            assert np.array_equal(ref[k], again[k]), k


# ---- quadcopter -----------------------------------------------------------------------------------------------------------------------
def _last_profile():
    out = (C.c_ulonglong * 8)()
    _lib.check(_lib.lib().obca_last_profile(0, out))
    return list(out)


def test_quadcopter_config4_pairs_match_both_one_formulation_calls():
    sc = scenarios.quadcopter_batch(64, seed=2)
    one = []
    for f in (0, 1):
        one.append(qc.one_call(sc["x0"], sc["xF"], sc, 511, f))
    counts_sd = _last_profile()[6:]                    # merit and K1 evaluations of the Signed Distance solve
    g = quad_both(sc["x0"], sc["xF"], sc, 511)
    assert _last_profile()[6:] == counts_sd
    assert_sets_equal_one_formulation(g, one, QC_SHARED)
    assert np.isnan(g["dist"]["slack"]).all()
    for f, name in ((0, "dist"), (1, "sd")):
        r = qc.composed(sc["x0"], sc["xF"], sc, 511, f)
        assert r["idx"].size == 64, r["status"]
        qc.assert_same(merged(g, name), r, f)
        assert g[name]["time"] > 0
    out = device.plan_solve_quadcopter_both(sc["x0"], sc["xF"], sc["R"], sc["obs"], sc["Ts80"])
    for f, name in ((0, "dist"), (1, "sd")):
        ref = device.plan_solve_quadcopter(sc["x0"], sc["xF"], sc["R"], sc["obs"], sc["Ts80"], signed_dist=f)
        for k in ("xp", "up", "ts", "lp", "slack"):
            assert all((a is None and b is None) or same_bits(a, b) for a, b in zip(out[name][k], ref[k])), (name, k)
        for k in ("exitflag", "iters", "kkt_err", "feasible", "worst"):
            assert same_bits(out[name][k], ref[k]), (name, k)
        for k in ("N", "Ts", "status", "expansions"):
            assert same_bits(out[k], ref[k]), k
    print(f"config 4, 64 pairs: plan {g['plan_seconds'] * 1e3:.0f} ms; Dist {int((g['dist']['exitflag'] == 1).sum())} converged, solve "
          f"{g['dist']['time'] * 1e3:.0f} ms; SD {int((g['sd']['exitflag'] == 1).sum())} converged, solve {g['sd']['time'] * 1e3:.0f} ms")


def test_quadcopter_no_path_pool_full_and_capacity_in_one_batch(monkeypatch):
    sc = scenarios.quadcopter_batch(30, seed=5)
    xw, xFw = qc._walled(2)
    x0 = np.concatenate([xw, sc["x0"]]); xF = np.concatenate([xFw, sc["xF"]])
    args = native.quadcopter_problem(x0, xF)
    for max_nodes in (1 << 13, 1 << 14, 1 << 15, 1 << 16, 1 << 17):
        st = device.plan_quadcopter_raw(*args, max_nodes=max_nodes)
        if (st["status"] == 4).sum() >= 2 and (st["status"] == 0).sum() >= 6:
            break
    Ncap = int(np.median(st["N"][st["status"] == 0]))
    g = quad_both(x0, xF, sc, Ncap, max_nodes)
    for code in (0, 1, 2, 4):
        assert (g["status"] == code).sum() >= 1, (code, g["status"])
    one = [qc.one_call(x0, xF, sc, Ncap, f, max_nodes) for f in (0, 1)]
    assert_sets_equal_one_formulation(g, one, QC_SHARED)
    for f, name in ((0, "dist"), (1, "sd")):
        qc.assert_same(merged(g, name), qc.composed(x0, xF, sc, Ncap, f, max_nodes), f)
    # host_fallback: the POOL_FULL pairs are planned once on the host, then solved with both formulations
    one = [qc.one_call(x0, xF, sc, 511, f, max_nodes, host_fallback=True) for f in (0, 1)]
    calls = _count_calls(monkeypatch, "astar3d_raw")
    h = quad_both(x0, xF, sc, 511, max_nodes, host_fallback=True)
    assert len(calls) == 1
    assert (h["status"] != 4).all(), h["status"]
    assert_sets_equal_one_formulation(h, one, QC_SHARED)


def test_quadcopter_empty_batch_and_nothing_planned_run_no_solve():
    qc._small_mixed_solve()
    before = _last_profile()
    sc = scenarios.quadcopter_batch(1, seed=2)
    g = quad_both(np.zeros((0, 12)), np.zeros((0, 12)), sc, 511)
    assert g["plan_seconds"] == 0.0 and g["dist"]["time"] == 0.0 and g["sd"]["time"] == 0.0
    x0, xF = qc._walled(2)
    g = quad_both(x0, xF, sc, 511)
    assert g["status"].tolist() == [1, 1] and g["dist"]["time"] == 0.0 and g["sd"]["time"] == 0.0 and g["plan_seconds"] > 0
    assert np.isnan(g["Tsb"]).all()
    for name in ("dist", "sd"):
        for k in ("xp", "up", "ts", "lp", "slack", "kkt_err", "worst"):
            assert np.isnan(g[name][k]).all(), (name, k)
        for k in ("exitflag", "iters", "feasible"):
            assert (g[name][k] == -1).all(), (name, k)
    assert _last_profile() == before


def test_quadcopter_device_memory_and_next_mixed_solve_are_unchanged():
    import torch
    ref = qc._small_mixed_solve()
    sc = scenarios.quadcopter_batch(640, seed=3)      # more pairs than resident planner warps: the full planner scratch
    torch.cuda.init()
    quad_both(sc["x0"], sc["xF"], sc, 511)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info(0)
    quad_both(sc["x0"], sc["xF"], sc, 511)
    torch.cuda.synchronize()
    free2, _ = torch.cuda.mem_get_info(0)
    assert abs(free1 - free2) <= 1 << 20, (free1, free2)
    again = qc._small_mixed_solve()
    for k in ref:
        if isinstance(ref[k], list):
            assert all(np.array_equal(a, b) for a, b in zip(ref[k], again[k])), k
        else:
            assert np.array_equal(ref[k], again[k]), k
