"""Hybrid A* warm starts with a goal per start pose, on the CPU: the heuristic map split into its goal-independent obstacle map and the
distances from one goal (obca_plan_core.h) equals calc_dist_policy; the relaxation of k_plan_hmap (obca_plan.cuh), emulated on one host
thread, equals the host's Dijkstra bit for bit, edge cases included; the emulated per-goal search equals the host twin
obca_plan_warmstart_cloud_batch in every output; the cloud entry with one shared goal equals obca_plan_warmstart_batch byte for byte; and
the C entry obca_plan_parking_warmstart_goals checks its arguments and refuses to run without a device."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
import emul_plan_goals                                                  # noqa: E402
from obca_b200 import scenarios                                         # noqa: E402
from obca_b200.planner import native                                    # noqa: E402

GOAL = {"backwards": (0.0, 1.3, math.pi / 2), "parallel": (-1.35, 4.0, 0.0)}
RESO = 0.3


def lot_poses(B, seed=0):
    rng = np.random.default_rng(seed)
    return np.column_stack([rng.uniform(-9, 9, B), rng.uniform(6.8, 9.3, B), np.zeros(B)])


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def edge_goals(ox, oy):
    """Goal positions that hit the edge cases of the map: a blocked cell, a goal on row xw and on column yw, goals just outside and far
    outside the grid, and cells on the rim."""
    H, Hs, E, (mnx, mny) = emul_plan_goals.hmaps([(0.0, 0.0)], ox, oy)
    xw, yw = H.shape[1:]
    cell = lambda i, j: ((i + mnx) * RESO, (j + mny) * RESO)      # the position of map cell (i, j), 1-based
    return [cell(xw, yw // 2), cell(xw // 2, yw), cell(xw, yw), cell(0, yw // 2), cell(1, 1), cell(xw - 1, yw - 1), cell(-3, -3),
            cell(xw + 5, 2), (1e3, -1e3)]


@pytest.mark.parametrize("scene", ["backwards", "parallel", "lot", "lot_free"])
def test_split_map_and_relaxation_equal_dijkstra(scene):
    """calc_dist_policy == calc_heur_grid + dist_from_goal == the emulated k_plan_hmap, bit for bit, for the scene's goals, goals
    spread over the grid and the edge cases."""
    if scene in ("backwards", "parallel"):
        ox, oy = native.obstacle_points(scene)
        goals = [GOAL[scene]]
    elif scene == "lot":
        ox, oy = scenarios.parking_lot_points(10)
        goals = [GOAL["backwards"]]
    else:
        lot = scenarios.parking_lot_free_slots()
        ox, oy, goals = lot["ox"], lot["oy"], list(lot["goals"][:, :2])
    rng = np.random.default_rng(1)
    goals = [tuple(g[:2]) for g in goals] + [(rng.uniform(ox.min(), ox.max()), rng.uniform(oy.min(), oy.max())) for _ in range(12)]
    goals += edge_goals(ox, oy)
    ref, split, relax, _ = emul_plan_goals.hmaps(goals, ox, oy)
    for g in range(len(goals)):
        assert same_bits(split[g], ref[g]), (scene, goals[g])
        assert same_bits(relax[g], ref[g]), (scene, goals[g], np.argwhere(relax[g] != ref[g])[:5])
    assert np.isfinite(ref[0]).sum() > 100                                # the scene's own goal reaches most of the free space


def test_relaxation_edge_cases():
    """About 64 goal cells on the 10-car lot: a blocked goal (its neighbours are reached, its own entry is 0), a goal on row xw, goals
    outside the grid (a neighbour of the grid and one far away, all INF), and an enclosed goal (only the goal's entry is finite)."""
    ox, oy = scenarios.parking_lot_points(10)
    # a closed ring of points around (0, 8): its inside is cut off from the rest of the lot
    t = np.linspace(0, 2 * np.pi, 200, endpoint=False)
    ox = np.concatenate([ox, 2.5 * np.cos(t)]); oy = np.concatenate([oy, 8.0 + 2.5 * np.sin(t)])
    ref, _, relax, (mnx, mny) = emul_plan_goals.hmaps([(0.0, 0.0)], ox, oy)
    xw, yw = ref.shape[1:]
    cell = lambda i, j: ((i + mnx) * RESO, (j + mny) * RESO)
    blocked = [(x, 5.8) for x in (-5.2, 2.6, 7.8)]                      # 0.8 m in front of a parked car: blocked, next to free cells
    goals = blocked + [cell(xw, 5), cell(xw, yw), cell(0, 5), cell(-1, -1), (500.0, 500.0), (0.0, 8.0), (6.0, 8.0)]
    rng = np.random.default_rng(2)
    goals += [(rng.uniform(ox.min() - 1, ox.max() + 1), rng.uniform(oy.min() - 1, oy.max() + 1)) for _ in range(64 - len(goals))]
    ref, split, relax, _ = emul_plan_goals.hmaps(goals, ox, oy)
    for g in range(len(goals)):
        assert same_bits(split[g], ref[g]) and same_bits(relax[g], ref[g]), goals[g]
    enclosed = ref[len(blocked) + 5]
    i, j = round(0.0 / RESO) - mnx, round(8.0 / RESO) - mny
    assert enclosed[i - 1, j - 1] == 0.0
    assert np.isfinite(enclosed).sum() < 300 and np.isinf(enclosed).sum() > 2000   # only the inside of the ring
    assert np.isinf(ref[len(blocked) + 4]).all()                        # far outside: nothing reachable
    assert ref[len(blocked)][xw - 1, 4] == 0.0 and ref[len(blocked) + 1][xw - 1, yw - 1] == 0.0   # goals on row xw: written there
    free = ref[len(blocked) + 6]                                         # a goal in the open lane
    for g, (gx, gy) in enumerate(blocked):                               # a blocked goal is still a source
        i, j = round(gx / RESO) - mnx, round(gy / RESO) - mny
        assert np.isinf(free[i - 1, j - 1]) and ref[g][i - 1, j - 1] == 0.0 and np.isfinite(ref[g]).sum() > 100


def test_emulated_goal_search_equals_host_twin():
    """A lot batch with a free slot, or a goal anywhere in the lane, per pose (more than 4 distinct goals): the emulated search and the
    host twin give the same status, N, expansion count, path and warm start, bit for bit."""
    lot = scenarios.parking_lot_free_slots()
    B = 24
    x0 = lot_poses(B, seed=3)
    rng = np.random.default_rng(4)
    xF = np.array([lot["goals"][i % len(lot["goals"])][:3] for i in range(B)])
    lane = rng.integers(0, B, 6)
    xF[lane] = np.column_stack([rng.uniform(-8, 8, 6), rng.uniform(7, 9, 6), rng.choice([0.0, math.pi], 6) + rng.uniform(-0.25, 0.25, 6)])
    assert len({(round(g[0] / RESO), round(g[1] / RESO)) for g in xF}) >= 4
    e = emul_plan_goals.plan_goals_raw(x0, xF, lot["ox"], lot["oy"], 0.6)
    h = native.plan_cloud_raw(x0, xF, lot["ox"], lot["oy"], 0.6, workers=4)
    assert (e["status"] == 0).sum() >= B // 2 and not (e["status"] == 4).any(), e["status"]
    for k in ("status", "N", "expansions"):
        assert np.array_equal(e[k], h[k]), (k, e[k], h[k])
    for k in ("rx", "ry", "ryaw", "xWS", "uWS"):
        assert np.array_equal(e[k], h[k], equal_nan=True), k


def test_cloud_entry_equals_scenario_entry_with_one_goal():
    """obca_plan_warmstart_cloud_batch on a demo cloud with one goal repeated writes obca_plan_warmstart_batch's bytes."""
    for scenario, Ts in (("backwards", 0.6), ("parallel", 0.9)):
        x0 = lot_poses(16, seed=5)
        ox, oy = native.obstacle_points(scenario)
        B, cap = len(x0), 512
        old = dict(rx=np.zeros((B, cap)), ry=np.zeros((B, cap)), ryaw=np.zeros((B, cap)), xWS=np.zeros((B, 4 * cap)), uWS=np.zeros((B, 2 * cap)),
                   N=np.zeros(B, np.int32), status=np.zeros(B, np.int32))
        p = lambda a: a.ctypes.data_as(C.c_void_p)
        xF = np.ascontiguousarray(GOAL[scenario], float)
        x0c = np.ascontiguousarray(x0)
        assert native.lib().obca_plan_warmstart_batch(B, p(x0c), p(xF), native.SCENARIOS[scenario], Ts, 2.7, 3, cap, 4,
                                                      *[p(old[k]) for k in ("rx", "ry", "ryaw", "xWS", "uWS", "N", "status")]) == 0
        new = native.plan_cloud_raw(x0, np.tile(xF, (B, 1)), ox, oy, Ts, workers=4)
        new = {k: np.where(np.isnan(v), 0.0, v) if v.dtype == float else v for k, v in new.items()}
        for k in ("status", "N"):
            ok = old["status"] == 0
            assert np.array_equal(new[k][ok] if k == "N" else new[k], old[k][ok] if k == "N" else old[k]), (scenario, k)
        for i in np.nonzero(old["status"] == 0)[0]:
            n = int(old["N"][i])
            for k, m in (("rx", n + 1), ("ry", n + 1), ("ryaw", n + 1), ("xWS", 4 * (n + 1)), ("uWS", 2 * n)):
                assert old[k][i, :m].tobytes() == new[k][i, :m].tobytes(), (scenario, i, k)


def test_cloud_entry_argument_errors():
    lib = native.lib()
    a = np.zeros(64); i = np.zeros(8, np.int32)
    p = lambda v: v.ctypes.data_as(C.c_void_p)

    def call(B=1, x0=True, xF=True, n_ob=4, Ts=0.6, sampleN=3, cap=16):
        return lib.obca_plan_warmstart_cloud_batch(B, p(a) if x0 else None, p(a) if xF else None, p(a), p(a), n_ob, Ts, 2.7, sampleN, cap, 1,
                                                   p(a), p(a), p(a), p(a), p(a), p(i), p(i), None)
    for kw in (dict(B=-1), dict(x0=False), dict(xF=False), dict(n_ob=0), dict(Ts=0.0), dict(sampleN=0), dict(cap=1)):
        assert call(**kw) == 3, kw


def _goals_call(lib, B=1, x0=True, xF=True, ob=True, n_ob=None, Ts=0.6, sampleN=3, cap=16):
    a = np.zeros(64); i = np.zeros(8, np.int32)
    p = lambda v: v.ctypes.data_as(C.c_void_p)
    return lib.obca_plan_parking_warmstart_goals(B, p(a) if x0 else None, p(a) if xF else None, p(a) if ob else None, p(a),
                                                 4 if n_ob is None else n_ob, Ts, 2.7, sampleN, 0, 0, cap, None, p(a), p(a), p(a), p(a), p(a),
                                                 p(i), p(i), None, None)


def test_goals_cabi_argument_errors_and_no_device():
    import obca_b200
    lib = obca_b200.lib()
    assert "obca_plan_parking_warmstart_goals" in obca_b200._lib.SYMBOLS
    for kw, msg in [(dict(B=-1), b"B < 0"), (dict(x0=False), b"null"), (dict(xF=False), b"null"), (dict(ob=False), b"null"),
                    (dict(n_ob=0), b"n_ob"), (dict(Ts=0.0), b"Ts"), (dict(sampleN=0), b"sampleN"), (dict(cap=1), b"cap")]:
        assert _goals_call(lib, **kw) == -1, kw
        assert msg in lib.obca_last_error(), (kw, lib.obca_last_error())
    if lib.obca_device_count() > 0:
        pytest.skip("CUDA device present")
    assert _goals_call(lib) == -2 and b"no CUDA device" in lib.obca_last_error()
    from obca_b200.planner import device
    lot = scenarios.parking_lot_free_slots()
    with pytest.raises(obca_b200.ObcaError, match="no CUDA device"):
        device.plan_goals_batch(lot_poses(2), lot["goals"][:2], lot["ox"], lot["oy"], 0.6)
    with pytest.raises(obca_b200.ObcaError, match="no CUDA device"):
        device.heuristic_maps(lot["goals"], lot["ox"], lot["oy"])
