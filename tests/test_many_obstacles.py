"""Parking problems with up to 16 obstacles and 64 half-spaces, without a GPU: the kernel sources in the development emulation
(tests/emul) against the oracle on the car-park scene (obca_b200.scenarios.parking_lot_scenario), the workspace layout with
the hand-over rows of obstacles 7.., and the shape bounds of the C-ABI."""
import ctypes as C

import numpy as np
import pytest

import emul
import k1_maps
from obca_b200 import scenarios
from oracle import dualmultws_ref, ipm_ref
from oracle.parking_nlp import build_parking_nlp
from oracle.parking_solve import solve_parking


def lot_small(n_cars, N=16, B=1, seed=0):
    """The lot scene at a short horizon (as test_emul_vs_oracle.small_batch): seeded start poses, geometric warm starts."""
    sc = scenarios.parking_lot_scenario(n_cars)
    rng = np.random.default_rng(seed)
    x0 = np.stack([rng.uniform(-10, 10, B), rng.uniform(6.5, 9.5, B), np.zeros(B), np.zeros(B)], 1)
    Ts = 48.0 / N
    rx = np.zeros((B, N + 1)); ry = np.zeros((B, N + 1)); ryaw = np.zeros((B, N + 1))
    xWS = np.zeros((B, N + 1, 4)); uWS = np.zeros((B, N, 2))
    for i in range(B):
        rx[i], ry[i], ryaw[i], xWS[i], uWS[i] = scenarios.warmstart_reverse(x0[i], sc["xF"], N, Ts, sc["L"])
    sc.update(B=B, N=N, x0=x0, rx=rx, ry=ry, ryaw=ryaw, xWS=xWS, uWS=uWS, Ts=Ts, Ts_fix=Ts)
    return sc


def test_lot_scene_shape():
    for n_cars, V in ((5, 21), (6, 25), (10, 41), (15, 61)):
        sc = scenarios.parking_lot_scenario(n_cars)
        assert sc["nOb"] == n_cars + 1 and int(sc["vOb"].sum()) == V and sc["A"].shape == (V, 2)
    # every car lies inside the region of the reference's obstacles 1 and 2 (|x| >= 1.3, y <= 5)
    for x0, x1, y0, y1 in scenarios.parking_lot_cars(15):
        assert (x0 >= 1.3 or x1 <= -1.3) and y1 <= 5.0
    ox, oy = scenarios.parking_lot_points(10)
    assert ox.shape == oy.shape and ox.size > 1000


@pytest.mark.parametrize("n_cars", [6, 10])
@pytest.mark.parametrize("variant,fix", [("sd", 0), ("d", 0), ("sd", 1), ("d", 1)])
def test_iterates_track_generic_dense_ipm_on_lot(n_cars, variant, fix):
    """7 and 11 obstacles (hand-over of obstacles 7.. through the workspace rows): the same iterates as the oracle's dense
    Bunch-Kaufman KKT solve after 1 and 3 iterations, the same solution at convergence (tolerances of
    test_emul_vs_oracle.test_iterates_track_generic_dense_ipm)."""
    sc = lot_small(n_cars)
    lp, npp, _, _ = emul.dualmultws_batch(sc)
    for K, tol in ((1, 1e-6), (3, 1e-6), (400, 1e-7)):
        o = emul.default_opts(); o.max_iter = K
        r = emul.solve_batch(sc, fix, variant, o, lp, npp)
        out, res, _ = solve_parking(sc["x0"][0], sc["xF"], sc["N"], sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"],
                                    sc["vOb"], sc["A"], sc["b"], sc["rx"][0], sc["ry"][0], sc["ryaw"][0], fix,
                                    sc["xWS"][0], sc["uWS"][0], variant, lp[0], npp[0], ipm_ref.IpmOptions(max_iter=K))
        xp, up, ts, _, _, lpo, npo = out
        assert np.abs(xp - r["xp"][0].T).max() < tol and np.abs(up - r["up"][0].T).max() < tol
        assert np.abs(ts - r["ts"][0]).max() < tol
        assert np.abs(lpo - r["lp"][0].T).max() < 10 * tol and np.abs(npo - r["np"][0].T).max() < 10 * tol
        if K == 400:
            assert res.status == 1 and r["status"][0] == 1 and abs(res.iters - r["iters"][0]) <= 3


@pytest.mark.parametrize("variant,fix", [("sd", 0), ("d", 1)])
def test_k1_matches_oracle_on_lot(variant, fix):
    """The stand-alone K1 evaluator on 11 obstacles against the oracle's sympy NLP (tolerances of test_k1_eval)."""
    sc = scenarios.parking_lot_scenario(10)
    N = 14
    rng = np.random.default_rng(7)
    rx, ry, ryaw = rng.normal(size=(3, N + 1))
    x0 = np.array([-6, 9.5, 0.1, 0.2]); xF = sc["xF"]
    nlp = build_parking_nlp(x0, xF, N, 0.7, sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"], sc["b"], rx, ry, ryaw, fix, variant)
    z, yE, yI = k1_maps.random_point(nlp, rng)
    arrays, rowmap = k1_maps.k1_inputs(nlp, z, yE, yI)
    one = dict(N=N, nOb=sc["nOb"], vOb=sc["vOb"], A=sc["A"], b=sc["b"], x0=x0, xF=xF, Ts=0.7, L=sc["L"], ego=sc["ego"],
               XYbounds=sc["XYbounds"], rx=rx, ry=ry, ryaw=ryaw)
    c, gl, fk = emul.eval_batch(one, arrays, fix, variant)
    c_ref, gl_ref, f_ref = k1_maps.oracle_reference(nlp, z, yE, yI, rowmap)
    assert np.abs(c - c_ref).max() < 1e-12 * (1 + np.abs(c_ref).max())
    assert np.abs(gl - gl_ref).max() < 1e-11 * (1 + np.abs(gl_ref).max())
    assert abs(fk.sum() - f_ref) < 1e-11 * (1 + abs(f_ref))


def test_dualws_on_lot_matches_closed_form_distances():
    sc = scenarios.parking_lot_batch(2, 80, seed=0, n_cars=15)
    _, _, d, its = emul.dualmultws_batch(sc)
    assert (its > 0).all() and its.max() <= 30
    g, off = dualmultws_ref.ego_geometry(sc["ego"])
    A = sc["A"]; b = sc["b"].ravel(); vo = np.concatenate([[0], np.cumsum(sc["vOb"])])
    for i in range(2):
        for k in range(0, 81, 8):
            pose = (sc["rx"][i, k], sc["ry"][i, k], sc["ryaw"][i, k])
            for j in range(sc["nOb"]):
                ref = dualmultws_ref.rect_poly_distance(pose, A[vo[j]:vo[j + 1]], b[vo[j]:vo[j + 1]], g, off)
                assert abs(ref - d[i, k, j]) < 2e-5, (i, k, j)


def _layout_total(N, vOb, sd=1):
    vOb = np.ascontiguousarray(vOb, dtype=np.int32)
    return emul.lib().emul_layout_total(N, len(vOb), vOb.ctypes.data_as(C.c_void_p), sd)


@pytest.mark.parametrize("vm,sd", [(2, 1), (4, 1), (4, 0)])
def test_layout_adds_handover_rows_past_six_obstacles(vm, sd):
    """Rows per problem: 34 + 3V + 26 nOb + nOb * nfac (the layout for up to six obstacles, unchanged) + 12 (nOb - 6) above six."""
    # rows per problem of the layout before obstacles past six existed, at N = 80 and N = 127 alike (config 2, the 4-obstacle
    # parallel scene, five obstacles): pinned, so that the formula below is not only checked against itself
    pinned = {((2, 2, 1), 1): 199, ((2, 2, 1), 0): 175, ((2, 2, 1, 1), 1): 252, ((2, 2, 1, 1), 0): 220, ((4,) * 5, 1): 384,
              ((4,) * 5, 0): 344, ((2,) * 5, 1): 314, ((2,) * 5, 0): 274, ((4, 4, 4, 4, 1), 1): 375, ((4, 4, 4, 4, 1), 0): 335}
    for (vOb, s), rows in pinned.items():
        for n, nsp in ((80, 82), (127, 128)):
            assert _layout_total(n, list(vOb), s) == rows * nsp, (vOb, s, n)
    N = 80
    NSP = (N + 2) & ~1
    one = _layout_total(N, [vm], sd) // NSP
    nfac = one - (34 + 3 * vm + 26)
    for nOb in range(1, 17):
        vOb = [vm] * nOb
        V = vm * nOb
        if V > 64:
            continue
        rows = 34 + 3 * V + 26 * nOb + nOb * nfac + 12 * max(nOb - 6, 0)
        assert _layout_total(N, vOb, sd) == rows * NSP, nOb


def _sizes(N, vOb, sd=1):
    import obca_b200
    lib = obca_b200.lib()
    vOb = np.ascontiguousarray(vOb, dtype=np.int32)
    n, m = C.c_longlong(), C.c_longlong()
    rc = lib.obca_parking_eval_sizes(C.c_int(N), C.c_int(len(vOb)), vOb.ctypes.data_as(C.c_void_p), C.c_int(sd), C.byref(n), C.byref(m))
    return rc, n.value, m.value, lib.obca_last_error().decode()


def test_shape_bounds_through_the_c_abi():
    """obca_parking_eval_sizes runs the problem-shape check of every parking entry and needs no device."""
    for sd in (0, 1):
        rc, n, m, _ = _sizes(20, [4] * 16, sd)
        assert rc == 0 and (n, m) == k1_maps.sizes(20, 16, 64, sd)
    rc, _, _, msg = _sizes(20, [4] * 17)
    assert rc == -1 and "nOb <= 16" in msg
    rc, _, _, msg = _sizes(20, [1] * 17)
    assert rc == -1 and "nOb <= 16" in msg
    # sum(vOb) = 65 within 16 obstacles needs an obstacle with 5 half-spaces: refused, naming the per-obstacle bound
    rc, _, _, msg = _sizes(20, [4] * 15 + [5])
    assert rc == -1 and "vOb[j] <= 4" in msg
    rc, _, _, msg = _sizes(20, [2, 5, 1])
    assert rc == -1 and "vOb[j] <= 4" in msg
