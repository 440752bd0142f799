"""The GPU Hybrid A* planner's search source (obca_b200/csrc/obca_plan.cuh), emulated on one host thread (tests/emul/emul_plan.cpp),
against the host planner libobca_planner.so: the same status, horizon, path and warm start, bit for bit; and the C-ABI entry
obca_plan_parking_warmstart_batch's argument checks and its refusal to run without a device."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emul"))
import emul_plan                                                        # noqa: E402
from obca_b200.planner import native                                    # noqa: E402

GOAL = {"backwards": (0.0, 1.3, math.pi / 2), "parallel": (-1.35, 4.0, 0.0)}
TS = {"backwards": 0.6, "parallel": 0.9}                                # native.plan_batch's default at sampleN = 3


def sweep_poses(B, seed=0):
    """The start poses of examples/sweep_parking.py."""
    rng = np.random.default_rng(seed)
    return np.column_stack([rng.uniform(-9, 9, B), rng.uniform(6.8, 9.3, B), np.zeros(B)])


def assert_same_as_host(o, plans, exact=True):
    for i, w in enumerate(plans):
        if w is None:
            assert o["status"][i] == 1, i
            continue
        n = w["N"]
        assert o["status"][i] == 0 and o["N"][i] == n, (i, o["status"][i], o["N"][i], n)
        got = dict(rx=o["rx"][i, :n + 1], ry=o["ry"][i, :n + 1], ryaw=o["ryaw"][i, :n + 1],
                   xWS=o["xWS"][i, :4 * (n + 1)].reshape(4, n + 1).T, uWS=o["uWS"][i, :2 * n].reshape(2, n).T)
        for k, v in got.items():
            if exact:
                assert np.array_equal(v, w[k]), (i, k)
            else:
                assert np.abs(v - w[k]).max() <= 1e-9, (i, k, np.abs(v - w[k]).max())
        assert np.isnan(o["rx"][i, n + 1:]).all() and np.isnan(o["ry"][i, n + 1:]).all() and np.isnan(o["ryaw"][i, n + 1:]).all()
        assert np.isnan(o["xWS"][i, 4 * (n + 1):]).all() and np.isnan(o["uWS"][i, 2 * n:]).all()


@pytest.mark.parametrize("scenario", ["backwards", "parallel"])
def test_emulated_search_equals_host_planner(scenario):
    x0 = sweep_poses(64)
    ox, oy = native.obstacle_points(scenario)
    o = emul_plan.plan_raw(x0, GOAL[scenario], ox, oy, TS[scenario])
    assert_same_as_host(o, native.plan_batch(x0, GOAL[scenario], scenario, workers=4))
    assert (o["expansions"][o["status"] == 0] >= 1).all()


def test_emulated_search_reference_poses():
    """The poses of test_planner_native.test_paths_and_warm_starts_identical."""
    for scenario, x0 in [("backwards", (-6.0, 9.5, 0.0)), ("backwards", (7.0, 8.0, math.pi)), ("backwards", (3.0, 7.5, 0.3)),
                         ("parallel", (-6.0, 9.5, 0.0)), ("parallel", (8.0, 8.0, 0.0))]:
        ox, oy = native.obstacle_points(scenario)
        o = emul_plan.plan_raw([x0], GOAL[scenario], ox, oy, TS[scenario])
        assert_same_as_host(o, [native.plan_warm_start(x0, GOAL[scenario], scenario)])


def test_emulated_budget_capacity_and_pool_codes():
    ox, oy = native.obstacle_points("backwards")
    x0, xF = [(-6.0, 9.5, 0.0)], GOAL["backwards"]
    assert native.calc_hybrid_astar_path(-6.0, 9.5, 0.0, *xF, ox, oy, max_expansions=3)[0] is None
    o = emul_plan.plan_raw(x0, xF, ox, oy, 0.6, max_expansions=3)
    assert o["status"][0] == 1 and o["N"][0] == -1 and o["expansions"][0] == 4 and np.isnan(o["rx"]).all()
    full = emul_plan.plan_raw(x0, xF, ox, oy, 0.6)
    n = int(full["N"][0])
    o = emul_plan.plan_raw(x0, xF, ox, oy, 0.6, cap=n)                  # N + 1 stages do not fit
    assert o["status"][0] == 2 and o["N"][0] == n
    for k in ("rx", "ry", "ryaw", "xWS", "uWS"):
        assert np.isnan(o[k]).all(), k
    small = int(full["expansions"][0])                                  # fewer nodes than the search inserts
    o = emul_plan.plan_raw(x0, xF, ox, oy, 0.6, max_nodes=small)
    assert o["status"][0] == 4 and o["N"][0] == -1
    for k in ("rx", "ry", "ryaw", "xWS", "uWS"):
        assert np.isnan(o[k]).all(), k
    o = emul_plan.plan_raw(x0 * 2, xF, ox, oy, 0.6, max_nodes=small)    # the table is left empty for the next problem
    assert (o["status"] == 4).all()


def enclosed_batch():
    """The backwards cloud plus a dense patch of points around two start poses in the lane: their searches empty the heap after the first
    expansion (every primitive and the analytic path collide).  Three free poses keep searching."""
    ox, oy = native.obstacle_points("backwards")
    gx, gy = np.meshgrid(np.arange(-9.0, -2.0, 0.25), np.arange(6.0, 10.0, 0.25))
    x0 = np.array([(-6.0, 8.0, 0.0), (6.0, 8.0, 0.0), (7.5, 7.0, 0.0), (4.0, 9.0, math.pi), (-6.0, 8.5, 0.3)])
    return x0, GOAL["backwards"], np.concatenate([ox, gx.ravel()]), np.concatenate([oy, gy.ravel()])


def test_emulated_no_path_in_a_mixed_batch():
    """NO_PATH from an empty heap and from the expansion budget, next to poses that are planned, in one batch: the host planner's
    outcome for each pose (sampleN = 1: rx / ry / ryaw are the full path), nothing written for the others."""
    x0, xF, ox, oy = enclosed_batch()
    host = [native.calc_hybrid_astar_path(*p, *xF, ox, oy) for p in x0]
    o = emul_plan.plan_raw(x0, xF, ox, oy, 0.6, sampleN=1)
    assert o["status"].tolist() == [1, 0, 0, 0, 1] and o["expansions"][0] == o["expansions"][4] == 1
    for i, (rx, ry, ryaw) in enumerate(host):
        if rx is None:
            assert o["status"][i] == 1 and o["N"][i] == -1
            for k in ("rx", "ry", "ryaw", "xWS", "uWS"):
                assert np.isnan(o[k][i]).all(), (i, k)
            continue
        n = len(rx)
        assert o["status"][i] == 0 and o["N"][i] == n - 1
        assert np.array_equal(o["rx"][i, :n], rx) and np.array_equal(o["ry"][i, :n], ry) and np.array_equal(o["ryaw"][i, :n], ryaw)
    budget = int(np.sort(o["expansions"])[2]) - 1                      # the budget stops the longer searches of the batch
    b = emul_plan.plan_raw(x0, xF, ox, oy, 0.6, sampleN=1, max_expansions=budget)
    for i in range(len(x0)):
        if o["expansions"][i] > budget + 1:
            assert native.calc_hybrid_astar_path(*x0[i], *xF, ox, oy, max_expansions=budget)[0] is None
            assert b["status"][i] == 1 and b["expansions"][i] == budget + 1 and np.isnan(b["rx"][i]).all()
        else:
            assert b["status"][i] == o["status"][i] and b["expansions"][i] == o["expansions"][i]
            assert np.array_equal(b["rx"][i], o["rx"][i], equal_nan=True)


def _call(lib, B=1, x0=True, xF=True, ob=True, n_ob=None, Ts=0.6, sampleN=3, cap=16):
    a = np.zeros(64); i = np.zeros(8, np.int32)
    p = lambda v: v.ctypes.data_as(C.c_void_p)
    return lib.obca_plan_parking_warmstart_batch(B, p(a) if x0 else None, p(a) if xF else None, p(a) if ob else None, p(a),
                                                 4 if n_ob is None else n_ob, Ts, 2.7, sampleN, 0, 0, cap, None, p(a), p(a), p(a), p(a), p(a),
                                                 p(i), p(i), None, None)


def test_cabi_argument_errors_and_no_device():
    import obca_b200
    lib = obca_b200.lib()
    assert "obca_plan_parking_warmstart_batch" in obca_b200._lib.SYMBOLS
    for kw, msg in [(dict(B=-1), b"B < 0"), (dict(x0=False), b"null"), (dict(xF=False), b"null"), (dict(ob=False), b"null"),
                    (dict(n_ob=0), b"n_ob"), (dict(Ts=0.0), b"Ts"), (dict(sampleN=0), b"sampleN"), (dict(cap=1), b"cap")]:
        assert _call(lib, **kw) == -1, kw
        assert msg in lib.obca_last_error(), (kw, lib.obca_last_error())
    if lib.obca_device_count() > 0:
        pytest.skip("CUDA device present")
    assert _call(lib) == -2 and b"no CUDA device" in lib.obca_last_error()
    from obca_b200.planner import device
    with pytest.raises(obca_b200.ObcaError, match="no CUDA device"):
        device.plan_batch(sweep_poses(2), GOAL["backwards"])
