"""The 3-D A* of the quadcopter flow as a library: obca_astar3d_batch (libobca_planner.so) against the Python planner
obca_b200/planner/a_star_3d.py -- the same obstacle map, the same paths, N, Ts and warm starts --, its failure codes, the GPU search source
emulated with the kernel's fixed scratch (tests/emul/emul_plan3d.cpp), and the GPU entry's argument checks without a device."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
import emul_plan3d                                                      # noqa: E402
from obca_b200 import scenarios                                         # noqa: E402
from obca_b200.planner import a_star_3d, native                         # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")
OUT = ("rx", "ry", "rz", "N", "status", "expansions")


def _same_map(ox, oy, oz, lo, hi, reso):
    got, mn, w = native.astar3d_obstacle_map(ox, oy, oz, lo, hi, reso)
    ref, rmn, rw = a_star_3d.calc_obstacle_map(np.asarray(ox, float) / reso, np.asarray(oy, float) / reso, np.asarray(oz, float) / reso,
                                               lo, hi, reso)
    assert mn == list(rmn) and w == list(rw)
    assert got.shape == ref.shape and np.array_equal(got, ref), int((got != ref).sum())
    return got


def test_obstacle_map_reference_environment():
    ox, oy, oz, lo, hi = a_star_3d.quadcopter_environment()
    m = _same_map(ox, oy, oz, lo, hi, 1.0)
    assert m.shape == (105, 105, 55) and 0 < m.sum() < m.size


def test_obstacle_map_non_integer_cloud_and_raw_bounds():
    """reso = 0.5: the points are divided by reso, the two bound corners are not (calc_obstacle_map's quirk), so the map spans both."""
    rng = np.random.default_rng(7)
    p = rng.uniform(0.3, 9.7, (60, 3)) * (1.0, 1.0, 0.6)
    m = _same_map(p[:, 0], p[:, 1], p[:, 2], (-1.3, 0.4, 0.0), (10.2, 10.0, 6.0), 0.5)
    assert 0 < m.sum() < m.size


def test_obstacle_map_points_at_the_vehicle_radius():
    """Points exactly VEHICLE_RADIUS / reso from cell centres (3-4-5 and axis offsets): the comparison is `<=`."""
    base = np.array([(5, 5, 5), (12, 7, 4), (8, 14, 9)], float)
    offs = np.array([(1.5, 2.0, 0.0), (2.5, 0.0, 0.0), (0.0, 1.5, 2.0), (-2.0, 0.0, -1.5), (0.0, -2.5, 0.0)])
    for reso in (1.0, 0.5):
        p = (base[:, None, :] + offs[None, :, :]).reshape(-1, 3) * reso
        _same_map(p[:, 0], p[:, 1], p[:, 2], (0.0, 0.0, 0.0), (20.0 * reso, 20.0 * reso, 14.0 * reso), reso)


@pytest.mark.parametrize("fixture", ["quad_astar_pairs", "quad_astar_long_pairs"])
def test_host_library_reproduces_the_planned_fixtures(fixture):
    z = np.load(os.path.join(GOLDEN, fixture + ".npz"))
    plans = native.plan_quadcopter_batch(z["x0"], z["xF"], 0.25, nthreads=4)
    for i, w in enumerate(plans):
        n = int(z["N"][i])
        assert w["N"] == n and w["Ts"] == z["Ts"][i], i
        assert np.array_equal(w["xWS"], z["xWS"][i][:, :n + 1]), i
        assert np.array_equal(w["uWS"], 0.5 * np.ones((4, n))) and w["timeWS"] == 1.0


def test_host_library_default_pair_equals_python_planner():
    sc = scenarios.quadcopter_scenario()
    ref = a_star_3d.plan_quadcopter_warm_start(sc["x0"], sc["xF"], sc["Ts80"])
    got = native.plan_quadcopter_batch([sc["x0"]], [sc["xF"]], sc["Ts80"])[0]
    assert set(got) == set(ref) and got["N"] == ref["N"] and got["Ts"] == ref["Ts"] and got["timeWS"] == ref["timeWS"]
    for k in ("xWS", "uWS"):
        assert np.array_equal(got[k], ref[k]), k
    for a, b in zip(got["path"], ref["path"]):
        assert np.array_equal(a, b)


def small_world(rng, reso=1.0):
    """About 20^3 cells with a few obstacle points (integer or not) and a start and goal cell in it: many tied queue keys."""
    n = int(rng.integers(0, 12))
    p = rng.uniform(0, 20, (n, 3))
    if rng.random() < 0.5:
        p = np.round(p)
    hi = np.array([20.0, 20.0, rng.choice([12.0, 20.0])])
    s = rng.uniform(0, hi) * reso
    g = rng.uniform(0, hi) * reso
    return s, g, p[:, 0] * reso, p[:, 1] * reso, p[:, 2] * reso, (0.0, 0.0, 0.0), tuple(hi * reso)


def _python(s, g, ox, oy, oz, lo, hi, reso):
    return a_star_3d.calc_astar_path(*s, *g, ox, oy, oz, *lo, *hi, reso)


def test_host_library_equals_python_on_random_small_worlds():
    rng = np.random.default_rng(11)
    found = 0
    for t in range(300):
        reso = 1.0 if t % 3 else 0.5
        s, g, ox, oy, oz, lo, hi = small_world(rng, reso)
        ref = _python(s, g, ox, oy, oz, lo, hi, reso)
        got = native.calc_astar_path(*s, *g, ox, oy, oz, *lo, *hi, reso)
        if ref[0] is None:
            assert got[0] is None, t
            continue
        found += 1
        for a, b in zip(got, ref):
            assert np.array_equal(a, b), t
    assert found > 150      # the others are NO_PATH in both (a start or goal boxed in by obstacles or outside the map)


def wall_world():
    pts = np.array([(x, y, z) for x in range(4, 7) for y in range(0, 11) for z in range(0, 11)], float)      # test_planner.py's full wall
    return pts[:, 0], pts[:, 1], pts[:, 2], (0.0, 0.0, 0.0), (10.0, 10.0, 10.0)


def test_no_path_goal_in_obstacle_start_outside_and_start_at_goal():
    ox, oy, oz, lo, hi = wall_world()
    assert _python((1.0, 5.0, 5.0), (9.0, 5.0, 5.0), ox, oy, oz, lo, hi, 1.0) == (None, None, None)
    assert native.calc_astar_path(1.0, 5.0, 5.0, 9.0, 5.0, 5.0, ox, oy, oz, *lo, *hi, 1.0) == (None, None, None)
    # goal cell blocked (next to the wall): never a neighbour
    assert _python((9.0, 2.0, 2.0), (8.0, 5.0, 5.0), ox, oy, oz, lo, hi, 1.0) == (None, None, None)
    assert native.calc_astar_path(9.0, 2.0, 2.0, 8.0, 5.0, 5.0, ox, oy, oz, *lo, *hi, 1.0) == (None, None, None)
    # starts outside the map's interior are never bounds-checked: one step outside the map reaches it, two steps do not
    e = np.zeros(0)
    for s in [(10.0, 5.0, 5.0), (11.0, 5.0, 5.0), (-1.0, 4.0, 4.0), (0.0, 3.0, 3.0), (5.0, 5.0, 10.4)]:
        ref = _python(s, (3.0, 4.0, 6.0), e, e, e, lo, hi, 1.0)
        got = native.calc_astar_path(*s, 3.0, 4.0, 6.0, e, e, e, *lo, *hi, 1.0)
        assert (got[0] is None) == (ref[0] is None), s
        if ref[0] is not None:
            assert all(np.array_equal(a, b) for a, b in zip(got, ref)), s
    assert native.calc_astar_path(11.0, 5.0, 5.0, 3.0, 4.0, 6.0, e, e, e, *lo, *hi, 1.0)[0] is None
    assert native.calc_astar_path(10.0, 5.0, 5.0, 3.0, 4.0, 6.0, e, e, e, *lo, *hi, 1.0)[0] is not None
    # start == goal: a one-point path, even inside an obstacle
    for s in [(2.2, 3.0, 4.0), (5.0, 5.0, 5.0)]:
        ref = _python(s, s, ox, oy, oz, lo, hi, 1.0)
        o = native.astar3d_raw([s], [s], ox, oy, oz, lo, hi, 1.0, cap=4)
        assert o["status"][0] == 0 and o["N"][0] == 0 and o["expansions"][0] == 1
        assert [o["rx"][0, 0], o["ry"][0, 0], o["rz"][0, 0]] == [ref[0][0], ref[1][0], ref[2][0]]
        assert np.isnan(o["rx"][0, 1:]).all()


def test_capacity_and_bad_arguments():
    sc = scenarios.quadcopter_scenario()
    args = native.quadcopter_problem([sc["x0"]], [sc["xF"]])
    full = native.astar3d_raw(*args)
    n = int(full["N"][0])
    o = native.astar3d_raw(*args, cap=n)                                  # n + 1 points do not fit
    assert o["status"][0] == 2 and o["N"][0] == n and o["expansions"][0] == full["expansions"][0]
    for k in ("rx", "ry", "rz"):
        assert np.isnan(o[k]).all(), k
    s, g, ox, oy, oz, lo, hi, reso = args
    for kw in (dict(reso=0.0), dict(reso=np.nan), dict(cap=0), dict(lo=(np.inf, 0, 0)), dict(s=np.full((1, 3), 1e18)),
               dict(hi=(1e4, 1e4, 1e4))):
        a = dict(s=s, g=g, ox=ox, oy=oy, oz=oz, lo=lo, hi=hi, reso=reso, cap=256)
        a.update(kw)
        with pytest.raises(native.PlannerError, match=": 3"):
            native.astar3d_raw(a["s"], a["g"], a["ox"], a["oy"], a["oz"], a["lo"], a["hi"], a["reso"], a["cap"])
    L = native.lib()
    z = np.zeros(64); i = np.full(4, -7, np.int32)
    p = lambda v: v.ctypes.data_as(C.c_void_p)
    assert L.obca_astar3d_batch(-1, p(z), p(z), p(z), p(z), p(z), 1, p(z), p(z), 1.0, 4, 1, p(z), p(z), p(z), p(i), p(i), None) == 3
    assert L.obca_astar3d_batch(1, None, p(z), p(z), p(z), p(z), 1, p(z), p(z), 1.0, 4, 1, p(z), p(z), p(z), p(i), p(i), None) == 3
    assert L.obca_astar3d_batch(1, p(z), p(z), p(z), p(z), p(z), -1, p(z), p(z), 1.0, 4, 1, p(z), p(z), p(z), p(i), p(i), None) == 3
    assert (i == -7).all()


def test_emulated_device_search_pool_full_leaves_outputs():
    sc = scenarios.quadcopter_batch(4, seed=2)
    args = native.quadcopter_problem(sc["x0"], sc["xF"])
    o = emul_plan3d.plan_raw(*args, max_nodes=100, max_queue=64)
    assert (o["status"] == 4).all() and (o["N"] == -1).all() and (o["nodes"] <= 100).all()
    for k in ("rx", "ry", "rz"):
        assert np.isnan(o[k]).all(), k
    o = emul_plan3d.plan_raw(*args, max_nodes=1 << 20, max_queue=40)    # the queue, not the pool, runs out
    assert (o["status"] == 4).all() and (o["queue_max"] <= 40).all() and np.isnan(o["rx"]).all()


def mixed_world():
    """A wall across a 30 x 10 x 10 map: left of it only the x = 1 layer is free.  Pairs that stay right of the wall find paths; a pair
    from the left layer to the right empties the queue (NO_PATH) after ~80 cells; a pair from the right to the left expands the whole right
    side first (~1700 cells)."""
    pts = np.array([(x, y, z) for x in range(4, 7) for y in range(0, 11) for z in range(0, 11)], float)
    starts = np.array([(1, 5, 5), (12, 3, 3), (25, 5, 5), (20, 6, 4), (1, 2, 7), (14, 5, 5), (28, 8, 8)], float)
    goals = np.array([(20, 5, 5), (26, 7, 6), (1, 5, 5), (21, 6, 5), (27, 3, 3), (14, 5, 5), (10, 2, 2)], float)
    return starts, goals, pts[:, 0], pts[:, 1], pts[:, 2], (0.0, 0.0, 0.0), (30.0, 10.0, 10.0), 1.0


def test_emulated_device_search_mixed_batch_equals_host_library():
    args = mixed_world()
    h = native.astar3d_raw(*args, cap=256)
    assert h["status"].tolist() == [1, 0, 1, 0, 1, 0, 0], h["status"]
    e = emul_plan3d.plan_raw(*args, max_nodes=1 << 16, max_queue=1 << 14, cap=256)
    for k in OUT:
        assert np.array_equal(e[k], h[k], equal_nan=True), k
    small = int(np.sort(e["nodes"])[-2]) - 1                            # the two largest searches no longer fit
    e = emul_plan3d.plan_raw(*args, max_nodes=small, max_queue=1 << 14, cap=256)
    full = e["status"] == 4
    assert full.sum() >= 2 and set(e["status"][~full].tolist()) == {0, 1} and (e["nodes"][full] <= small).all()
    for k in OUT:
        assert np.array_equal(e[k][~full], h[k][~full], equal_nan=True), k
    assert np.isnan(e["rx"][full]).all() and (e["N"][full] == -1).all()
    # many config-4 pairs, one scratch reused pair after pair
    sc = scenarios.quadcopter_batch(24, seed=5)
    args = native.quadcopter_problem(sc["x0"], sc["xF"])
    h = native.astar3d_raw(*args)
    e = emul_plan3d.plan_raw(*args)
    for k in OUT:
        assert np.array_equal(e[k], h[k], equal_nan=True), k


def _call(lib, B=1, s=True, ob=True, n_ob=1, reso=1.0, cap=8, max_nodes=0, out=True):
    a = np.zeros(64); i = np.zeros(8, np.int32)
    p = lambda v: v.ctypes.data_as(C.c_void_p)
    return lib.obca_plan_quadcopter_warmstart_batch(B, p(a) if s else None, p(a), p(a) if ob else None, p(a), p(a), n_ob, p(a), p(a), reso,
                                                    max_nodes, cap, None, p(a) if out else None, p(a), p(a), p(i), p(i), None, None)


def test_cabi_argument_errors_and_no_device():
    import obca_b200
    lib = obca_b200.lib()
    assert "obca_plan_quadcopter_warmstart_batch" in obca_b200._lib.SYMBOLS
    for kw, msg in [(dict(B=-1), b"B < 0"), (dict(s=False), b"null"), (dict(ob=False), b"null"), (dict(out=False), b"null"),
                    (dict(n_ob=-1), b"n_ob"), (dict(reso=0.0), b"reso"), (dict(cap=0), b"cap"), (dict(max_nodes=1 << 29), b"max_nodes")]:
        assert _call(lib, **kw) == -1, kw
        assert msg in lib.obca_last_error(), (kw, lib.obca_last_error())
    if lib.obca_device_count() > 0:
        pytest.skip("CUDA device present")
    assert _call(lib) == -2 and b"no CUDA device" in lib.obca_last_error()
    from obca_b200.planner import device
    sc = scenarios.quadcopter_batch(2, seed=2)
    with pytest.raises(obca_b200.ObcaError, match="no CUDA device"):
        device.plan_quadcopter_batch(sc["x0"], sc["xF"])
