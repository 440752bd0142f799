"""obca_quadcopter_plan_solve on the GPU: plan, build the warm starts, solve and check a batch of quadcopter pairs in one call gives, bit
for bit, what the composed path gives on the same inputs -- obca_plan_quadcopter_warmstart_batch, native.quadcopter_warm_start on every
path, obca_quadcopter_solve_mixed on the pairs that planned, then obca_check_quadcopter_mixed -- in the caller's pair order, with every
entry of a pair that was not solved (and past a solved pair's horizon) left as the caller had it.  Also: NO_PATH, POOL_FULL and CAPACITY
pairs in one batch, with and without the host fallback, B = 0 and a batch where nothing plans (no solve), device memory after the call,
and an ordinary mixed solve after it."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from obca_b200 import _lib, quadcopter, scenarios     # noqa: E402
from obca_b200.planner import device, native          # noqa: E402
from obca_b200.planner.a_star_3d import quadcopter_environment      # noqa: E402

pytestmark = pytest.mark.gpu
ARRAYS = (("xp", 1), ("up", 0), ("ts", 1), ("lp", 1), ("slack", 1))


def composed(x0, xF, sc, Ncap, sd=1, max_nodes=0):
    """The composed path on the same inputs: the GPU planner (stride 1024), the host warm start of every pair planned to 2 <= N <= Ncap,
    the mixed solve of those pairs and the mixed check."""
    s, g, ox, oy, oz, lo, hi, reso = native.quadcopter_problem(x0, xF)
    o = device.plan_quadcopter_raw(s, g, ox, oy, oz, lo, hi, reso, cap=1024, max_nodes=max_nodes)
    st = o["status"].copy()
    st[(st == 0) & ((o["N"] < 2) | (o["N"] > Ncap))] = 2
    idx = np.flatnonzero(st == 0)
    r = dict(status=st, N=o["N"], expansions=o["expansions"], idx=idx)
    if idx.size == 0:
        return r
    ws = [native.quadcopter_warm_start(o["rx"][i, :n + 1].copy(), o["ry"][i, :n + 1].copy(), o["rz"][i, :n + 1].copy(), sc["Ts80"])
          for i, n in zip(idx, o["N"][idx])]
    Ns = o["N"][idx]; Tsb = np.array([w["Ts"] for w in ws])
    q = quadcopter.quadcopter_solve_mixed(x0[idx], xF[idx], Ns, Tsb, sc["R"], sc["obs"], [w["xWS"] for w in ws], 1.0, sd)
    feas, worst = quadcopter.check_quadcopter_mixed(q["xp"], q["up"], q["ts"], x0[idx], xF[idx], Ns, Tsb, q["lp"], sc["obs"], sc["R"])
    r.update({k: v for k, v in q.items() if k not in ("N", "Ts")}, Tsb=Tsb, feasible=feas, worst=worst)
    return r


def one_call(x0, xF, sc, Ncap, sd=1, max_nodes=0, host_fallback=False):
    ox, oy, oz, lo, hi = quadcopter_environment()
    return device.plan_solve_quadcopter_raw(x0, xF, ox, oy, oz, lo, hi, 1.0, sc["Ts80"], sc["R"], sc["obs"], 1.0, sd, Ncap, max_nodes,
                                            host_fallback=host_fallback)


def assert_same(g, r, sd):
    """Every output of the one call equals the composed path's bit for bit; the rest keeps the sentinel fill (NaN, -1)."""
    B = len(g["status"])
    assert np.array_equal(g["status"], r["status"]), (g["status"], r["status"])
    assert np.array_equal(g["N"], r["N"]) and np.array_equal(g["expansions"], r["expansions"])
    solved = np.zeros(B, bool); solved[r["idx"]] = True
    for k, ext in ARRAYS:
        for q, i in enumerate(r["idx"]):
            n = int(r["N"][i])
            if k == "slack" and not sd:
                assert np.isnan(g[k][i]).all(); continue
            want = r[k][q] if k == "ts" else r[k][q].T
            assert np.array_equal(g[k][i, :n + ext], want), (k, i)
            assert np.isnan(g[k][i, n + ext:]).all(), (k, i)
        assert np.isnan(g[k][~solved]).all(), k
    for k in ("Tsb", "exitflag", "iters", "kkt_err", "feasible", "worst"):
        if r["idx"].size:
            assert np.array_equal(g[k][r["idx"]], np.asarray(r[k])), k
        unset = g[k][~solved]
        assert (np.isnan(unset) if k in ("Tsb", "kkt_err", "worst") else unset == -1).all(), k


@pytest.mark.parametrize("sd", [1, 0])
def test_config4_pairs_match_composed_path(sd):
    sc = scenarios.quadcopter_batch(64, seed=2)
    g = one_call(sc["x0"], sc["xF"], sc, 511, sd)
    r = composed(sc["x0"], sc["xF"], sc, 511, sd)
    assert r["idx"].size == 64, r["status"]
    assert_same(g, r, sd)
    assert g["plan_seconds"] > 0 and g["time"] > 0
    out = device.plan_solve_quadcopter(sc["x0"], sc["xF"], sc["R"], sc["obs"], sc["Ts80"], signed_dist=sd)
    for q, i in enumerate(r["idx"]):
        assert np.array_equal(out["xp"][i], r["xp"][q]) and np.array_equal(out["lp"][i], r["lp"][q]) and out["Ts"][i] == r["Tsb"][q]
    print(f"config 4, 64 pairs, signed_dist={sd}: {int((g['exitflag'] == 1).sum())} converged, {int((g['feasible'] == 1).sum())} pass "
          f"constrSatisfaction; plan {g['plan_seconds'] * 1e3:.0f} ms, solve {g['time'] * 1e3:.0f} ms device time")


def _walled(n):
    """n pairs whose start lies inside the first wall (grid x 20..25): every neighbour of the start cell is blocked, so the search ends
    at once with NO_PATH."""
    x0 = np.zeros((n, 12)); x0[:, 0] = 2.2; x0[:, 1] = np.linspace(3.0, 7.0, n); x0[:, 2] = 3.0
    xF = np.zeros((n, 12)); xF[:, 0] = 9.0; xF[:, 1] = 5.0; xF[:, 2] = 2.0
    return x0, xF


def test_no_path_pool_full_and_capacity_in_one_batch():
    """Two pairs starting inside a wall (NO_PATH), a node pool small enough that some searches outgrow it (POOL_FULL) and an Ncap below
    some planned horizons (CAPACITY), next to pairs that are solved."""
    sc = scenarios.quadcopter_batch(30, seed=5)
    xw, xFw = _walled(2)
    x0 = np.concatenate([xw, sc["x0"]]); xF = np.concatenate([xFw, sc["xF"]])
    args = native.quadcopter_problem(x0, xF)
    for max_nodes in (1 << 13, 1 << 14, 1 << 15, 1 << 16, 1 << 17):
        st = device.plan_quadcopter_raw(*args, max_nodes=max_nodes)
        if (st["status"] == 4).sum() >= 2 and (st["status"] == 0).sum() >= 6:
            break
    Ncap = int(np.median(st["N"][st["status"] == 0]))
    g = one_call(x0, xF, sc, Ncap, max_nodes=max_nodes)
    r = composed(x0, xF, sc, Ncap, max_nodes=max_nodes)
    for code in (0, 1, 2, 4):
        assert (g["status"] == code).sum() >= 1, (code, g["status"])
    assert (g["status"][:2] == 1).all() and (g["N"][:2] == -1).all()
    assert (g["N"][g["status"] == 2] > Ncap).all()
    assert_same(g, r, 1)
    print(f"max_nodes {max_nodes}, Ncap {Ncap}: status counts {np.bincount(g['status'], minlength=5).tolist()}")
    # host_fallback: the POOL_FULL pairs get the host library's plans, solved and checked; every other pair keeps the one call's outputs
    # (at Ncap = 511, so that the long searches which outgrew the pool are solved, not CAPACITY)
    g = one_call(x0, xF, sc, 511, max_nodes=max_nodes)
    h = one_call(x0, xF, sc, 511, max_nodes=max_nodes, host_fallback=True)
    full = g["status"] == 4
    tw = native.astar3d_raw(args[0][full], args[1][full], *args[2:], cap=512)
    assert np.array_equal(h["status"][full], tw["status"]) and np.array_equal(h["N"][full], tw["N"])
    assert (h["status"] != 4).all() and (tw["status"] == 0).all(), tw["status"]
    for k in ("xp", "up", "ts", "lp", "slack", "N", "Tsb", "status", "expansions", "exitflag", "iters", "kkt_err", "feasible", "worst"):
        assert np.array_equal(h[k][~full], g[k][~full], equal_nan=True), k
    whole = composed(x0, xF, sc, 511)      # max_nodes = 0: every pair plans on the device, to the host library's paths
    for i in np.flatnonzero(full):
        q = int(np.flatnonzero(whole["idx"] == i)[0]); n = int(h["N"][i])
        assert np.array_equal(h["xp"][i, :n + 1], whole["xp"][q].T) and np.isnan(h["xp"][i, n + 1:]).all(), i
        assert h["Tsb"][i] == whole["Tsb"][q] and h["iters"][i] == whole["iters"][q] and h["feasible"][i] == whole["feasible"][q], i


def _last_profile():
    out = (C.c_ulonglong * 8)()
    _lib.check(_lib.lib().obca_last_profile(0, out))
    return list(out)


def _small_mixed_solve():
    sc = scenarios.quadcopter_mixed_batch(8, seed=7)
    r = quadcopter.quadcopter_solve_mixed(sc["x0"], sc["xF"], sc["Ns"], sc["Ts"], sc["R"], sc["obs"], sc["xWS"], 1.0, 1)
    return {k: r[k] for k in ("xp", "up", "ts", "lp", "slack", "exitflag", "iters", "kkt_err")}


def test_empty_batch_and_nothing_planned_run_no_solve():
    _small_mixed_solve()
    before = _last_profile()
    sc = scenarios.quadcopter_batch(1, seed=2)
    g = one_call(np.zeros((0, 12)), np.zeros((0, 12)), sc, 511)
    assert g["time"] == 0.0 and g["plan_seconds"] == 0.0
    x0, xF = _walled(2)
    g = one_call(x0, xF, sc, 511)
    assert g["status"].tolist() == [1, 1] and g["time"] == 0.0 and g["plan_seconds"] > 0
    for k in ("xp", "up", "ts", "lp", "slack", "Tsb", "kkt_err", "worst"):
        assert np.isnan(g[k]).all(), k
    for k in ("exitflag", "iters", "feasible"):
        assert (g[k] == -1).all(), k
    assert _last_profile() == before


def test_planner_scratch_is_freed_and_next_mixed_solve_is_unchanged():
    import torch
    ref = _small_mixed_solve()
    sc = scenarios.quadcopter_batch(640, seed=3)      # more pairs than resident planner warps: the full planner scratch
    torch.cuda.init()
    one_call(sc["x0"], sc["xF"], sc, 511)
    torch.cuda.synchronize()
    free1, _ = torch.cuda.mem_get_info(0)
    one_call(sc["x0"], sc["xF"], sc, 511)
    torch.cuda.synchronize()
    free2, _ = torch.cuda.mem_get_info(0)
    assert abs(free1 - free2) <= 1 << 20, (free1, free2)
    again = _small_mixed_solve()
    for k in ref:
        if isinstance(ref[k], list):
            assert all(np.array_equal(a, b) for a, b in zip(ref[k], again[k])), k
        else:
            assert np.array_equal(ref[k], again[k]), k
