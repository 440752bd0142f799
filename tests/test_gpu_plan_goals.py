"""The GPU Hybrid A* planner with a goal per start pose (obca_plan_parking_warmstart_goals): the heuristic maps k_plan_hmap builds equal
the host's Dijkstra bit for bit (in shared memory and, for a large cloud, in global memory); every pose of a mixed batch gets the host
twin's status, and the free-slot poses its N, expansion count and values within 1e-9; with one goal for all it equals obca_plan_parking_warmstart_batch
bit for bit; plan_goals_batch plans POOL_FULL poses on the host; and the car-park flow -- plan, solve with a goal per problem, check --
runs end to end."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
import emul_plan_goals                                                  # noqa: E402
from obca_b200 import parking, scenarios                                # noqa: E402
from obca_b200.planner import device, native                            # noqa: E402
from test_plan_goals import edge_goals, lot_poses                       # noqa: E402

pytestmark = pytest.mark.gpu
KEYS = ("rx", "ry", "ryaw", "xWS", "uWS")


def mixed_goals(lot, B, seed):
    """Free-slot goals for most poses, a goal in the lane for every fourth, heading within 0.25 rad of the lane's direction.  (Not exactly
    along it: from a start pose on the same line, equally long Reeds-Shepp words tie, and the device's sin / cos break such a tie
    differently from the host's.)"""
    rng = np.random.default_rng(seed)
    xF = np.array([lot["goals"][i % len(lot["goals"])][:3] for i in range(B)])
    lane = np.arange(0, B, 4)
    xF[lane] = np.column_stack([rng.uniform(-8, 8, lane.size), rng.uniform(7, 9, lane.size),
                                rng.choice([0.0, math.pi], lane.size) + rng.uniform(-0.25, 0.25, lane.size)])
    return xF


def test_gpu_heuristic_maps_equal_host_dijkstra():
    lot = scenarios.parking_lot_free_slots()
    rng = np.random.default_rng(0)
    big_x = np.concatenate([np.linspace(-30, 30, 601), np.full(601, 30.0)])      # a 200 x 200-cell grid: too big for shared memory
    big_y = np.concatenate([np.full(601, -30.0), np.linspace(-30, 30, 601)])
    for ox, oy, goals in ((lot["ox"], lot["oy"], list(lot["goals"][:, :2])), (*native.obstacle_points("backwards"), [(0.0, 1.3)]),
                          (big_x, big_y, [(0.0, 0.0), (10.0, -5.0)])):
        goals = goals + [(rng.uniform(ox.min(), ox.max()), rng.uniform(oy.min(), oy.max())) for _ in range(40)] + edge_goals(ox, oy)
        ref, _, _, mn = emul_plan_goals.hmaps(goals, ox, oy)
        got, gmn, secs = device.heuristic_maps(goals, ox, oy)
        assert gmn == mn and got.shape == ref.shape
        bad = [g for g in range(len(goals)) if not np.array_equal(got[g].view(np.uint64), ref[g].view(np.uint64))]
        assert not bad, [goals[g] for g in bad[:5]]
        print(f"{ref.shape[1]} x {ref.shape[2]} cells, {len(goals)} maps: k_plan_hmap {secs * 1e3:.2f} ms")


def test_gpu_goal_plans_match_host_twin():
    """Every pose gets the host twin's status.  The poses sent to a free slot also get its N and expansion count, and values within
    1e-9 of its.  The lane goals lie a few metres from start poses on nearly the same line, where the analytic expansion's candidate
    words come close to set_path's 0.01 thresholds; there the device's sin / cos can pick another word than the host's, and such a
    pose may end with another N.  Those are counted and printed, and must stay a small share of the lane goals."""
    lot = scenarios.parking_lot_free_slots()
    B = 256
    x0, xF = lot_poses(B, seed=1), mixed_goals(lot, B, 2)
    o = device.plan_goals_raw(x0, xF, lot["ox"], lot["oy"], 0.6)
    h = native.plan_cloud_raw(x0, xF, lot["ox"], lot["oy"], 0.6)
    assert np.array_equal(o["status"], h["status"]), np.nonzero(o["status"] != h["status"])[0]
    assert (o["status"] == 0).sum() >= B // 2, o["status"]
    lane = np.zeros(B, bool); lane[::4] = True
    differs = (o["N"] != h["N"]) | (o["expansions"] != h["expansions"])
    for i in range(B):
        if o["status"][i] != 0:
            for k in KEYS:
                assert np.isnan(o[k][i]).all(), (i, k)
    worst = 0.0
    for i in np.nonzero(~differs & (o["status"] == 0))[0]:
        n = int(o["N"][i])
        for k, m in (("rx", n + 1), ("ry", n + 1), ("ryaw", n + 1), ("xWS", 4 * (n + 1)), ("uWS", 2 * n)):
            d = float(np.abs(o[k][i, :m] - h[k][i, :m]).max())
            worst = max(worst, d)
            assert d <= 1e-9, (i, k, d)
            assert np.isnan(o[k][i, m:]).all(), (i, k)
    print(f"{B} poses, {len({(round(g[0] / 0.3), round(g[1] / 0.3)) for g in xF})} goal cells: slot goals same decisions, lane goals "
          f"{int(differs[lane].sum())} of {int(lane.sum())} with another N / expansion count (poses {np.nonzero(differs)[0].tolist()}, "
          f"device N {o['N'][differs].tolist()} exp {o['expansions'][differs].tolist()}, host N {h['N'][differs].tolist()} "
          f"exp {h['expansions'][differs].tolist()}), max |device - host| = {worst:.2e}, k_plan {o['seconds'] * 1e3:.1f} ms")
    assert not differs[~lane].any(), np.nonzero(differs & ~lane)[0]
    assert differs[lane].sum() <= lane.sum() // 8, np.nonzero(differs)[0]


@pytest.mark.parametrize("scenario", ["backwards", "parallel"])
def test_gpu_one_goal_equals_batch_entry(scenario):
    goal = {"backwards": (0.0, 1.3, math.pi / 2), "parallel": (-1.35, 4.0, 0.0)}[scenario]
    Ts = 0.6 if scenario == "backwards" else 0.9
    x0 = lot_poses(256, seed=4)
    ox, oy = native.obstacle_points(scenario)
    a = device.plan_raw(x0, goal, ox, oy, Ts)
    b = device.plan_goals_raw(x0, np.tile(goal, (len(x0), 1)), ox, oy, Ts)
    for k in KEYS + ("N", "status", "expansions"):
        assert a[k].tobytes() == b[k].tobytes(), k


def test_gpu_plan_goals_batch_plans_pool_full_poses_on_the_host():
    lot = scenarios.parking_lot_free_slots()
    x0, xF = lot_poses(16, seed=5), mixed_goals(lot, 16, 6)
    small = int(np.median(native.plan_cloud_raw(x0, xF, lot["ox"], lot["oy"], 0.6)["expansions"]))
    st = device.plan_goals_raw(x0, xF, lot["ox"], lot["oy"], 0.6, max_nodes=small)["status"]
    assert (st == device.POOL_FULL).any() and (st == 0).any(), st
    got, host = device.plan_goals_batch(x0, xF, lot["ox"], lot["oy"], 0.6, max_nodes=small), native.plan_cloud_batch(x0, xF, lot["ox"], lot["oy"], 0.6)
    for i, (g, h) in enumerate(zip(got, host)):
        assert (g is None) == (h is None) and (h is None or g["N"] == h["N"]), i
        if h is not None:
            for k in KEYS:
                d = np.abs(g[k] - h[k]).max()
                assert (d == 0.0) if st[i] == device.POOL_FULL else (d <= 1e-9), (i, k, d)


def test_gpu_free_slot_flow_plans_solves_and_checks():
    """examples/sweep_parking_lot.py --free-slots: 64 cars, each sent to one of the row's free slots; one planner call, one mixed-horizon
    solve with xF (B, 4), one check.  Every converged problem passes ParkingConstraints."""
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import sweep_parking_lot
    o = sweep_parking_lot.run(64, seed=0, free_slots=True)
    print(f"free slots: {o['n_planned']} of 64 planned, {o['n_converged']} converged, {o['n_clean']} pass ParkingConstraints, "
          f"goals per slot {o['per_slot']}")
    assert o["n_planned"] >= 48 and o["n_converged"] >= 1
    assert o["n_clean"] == o["n_converged"], o
