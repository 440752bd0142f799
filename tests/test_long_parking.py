"""Parking problems with horizons past 127 steps (up to N = 319), without a GPU: the goldens of the reference's own start pose at
sampleN = 1 (N = 192, tests/golden/make_long_parking_golden.py) are KKT points of the reference NLP that ParkingConstraints
accepts, the kernel sources run through the development emulation (tests/emul) reach them, and the C-ABI refuses a longer
horizon before any device work."""
import ctypes as C
import glob
import os

import numpy as np
import pytest

import emul
from obca_b200 import scenarios
from oracle import checkers, dualmultws_ref, kkt_check

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDENS = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(HERE, "golden", "long_park", "*.npz")))
NMAX = 319


def load(case):
    """A golden and the one-problem scenario dict it was solved on (warm start and DualMultWS result from the file)."""
    g = np.load(os.path.join(HERE, "golden", "long_park", case + ".npz"))
    sc = scenarios.reverse_parking_scenario()
    N = int(g["N"])
    sc.update(B=1, N=N, Ts=float(g["Ts"]), x0=g["x0"][None], rx=g["rx"][None], ry=g["ry"][None], ryaw=g["ryaw"][None],
              xWS=g["xWS"][None], uWS=g["uWS"][None])
    return g, sc


def test_goldens_cover_main_jl_pose_at_sample_n_one():
    assert GOLDENS == ["main_d_n1", "main_sd_n1"]
    for case in GOLDENS:
        g, sc = load(case)
        assert int(g["N"]) == 192 and float(g["Ts"]) == pytest.approx(0.2) and int(g["sampleN"]) == 1
        assert g["xWS"].shape == (193, 4) and g["uWS"].shape == (192, 2) and g["lWS"].shape == (193, 5) and g["nWS"].shape == (193, 12)


def test_fixture_is_what_the_planner_gives():
    """The stored warm start is libobca_planner.so's plan of main.jl's pose at sampleN = 1."""
    from obca_b200.planner import native
    g, sc = load(GOLDENS[0])
    w = native.plan_warm_start(g["x0"][:3], sc["xF"], "backwards", None, sc["L"], 1)
    assert w["N"] == int(g["N"]) and w["Ts"] == float(g["Ts"])
    for k in ("rx", "ry", "ryaw"):
        assert np.array_equal(np.ravel(w[k]), g[k]), k
    assert np.array_equal(np.asarray(w["xWS"])[:193], g["xWS"]) and np.array_equal(np.asarray(w["uWS"])[:192], g["uWS"])


@pytest.mark.parametrize("case", GOLDENS)
def test_golden_is_kkt_point_and_feasible(case):
    g, sc = load(case)
    variant = str(g["variant"])
    assert int(g["status"]) == 1
    r = dict(xp=g["xp"][None], up=g["up"][None], ts=g["ts"][None], lp=g["lp"][None], np=g["np"][None],
             sl=g["sl"][None] if variant == "sd" else None)
    e = kkt_check.reference_kkt_error(sc, 0, r, variant, 0)
    assert e["E0"] < 1e-5 and abs(e["f"] - float(g["f"])) < 1e-9
    assert checkers.ParkingConstraints(sc["x0"][0], sc["xF"], sc["N"], sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"],
                                       sc["A"], sc["b"], g["xp"], g["up"], g["lp"], g["np"], g["ts"], 0, 1 if variant == "sd" else 0) == 1


def test_emulated_dualws_at_long_horizon():
    """DualMultWS of the kernel sources at N = 192: the ego/obstacle distances of the oracle's DualMultWS and the closed form
    (tolerance of test_emul_vs_oracle)."""
    g, sc = load(GOLDENS[0])
    lp, npp, d, its = emul.dualmultws_batch(sc)
    assert (its > 0).all()
    assert np.abs(d[0] - g["dWS"]).max() < 2e-5
    gg, off = dualmultws_ref.ego_geometry(sc["ego"])
    vo = np.concatenate([[0], np.cumsum(sc["vOb"])]); b = sc["b"].ravel()
    for k in range(0, 193, 16):
        pose = (g["rx"][k], g["ry"][k], g["ryaw"][k])
        for j in range(sc["nOb"]):
            ref = dualmultws_ref.rect_poly_distance(pose, sc["A"][vo[j]:vo[j + 1]], b[vo[j]:vo[j + 1]], gg, off)
            assert abs(ref - d[0, k, j]) < 2e-5, (k, j)


@pytest.mark.parametrize("case", GOLDENS)
def test_kernel_sources_reproduce_long_golden(case):
    """The emulated kernel sources from the stored warm start and duals converge to the golden point (tolerances of
    test_golden.test_kernel_sources_reproduce_golden)."""
    g, sc = load(case)
    r = emul.solve_batch(sc, 0, str(g["variant"]), None, g["lWS"][None], g["nWS"][None])
    assert r["status"][0] == 1
    assert np.abs(r["xp"][0].T - g["xp"]).max() < 2e-4 and np.abs(r["up"][0].T - g["up"]).max() < 2e-4
    assert np.abs(r["ts"][0] - g["ts"]).max() < 1e-5


def _args(B, N, Nb=None):
    """Well-formed arguments of obca_parking_solve_batch (Nb None) or obca_parking_solve_mixed for B reverse-parking problems
    laid out for N, outputs filled with 7."""
    sc = scenarios.reverse_parking_scenario()
    NS = N + 1
    k = dict(vOb=np.ascontiguousarray(sc["vOb"], dtype=np.int32), A=np.asfortranarray(sc["A"], dtype=float),
             b=np.ascontiguousarray(sc["b"].ravel()), ego=sc["ego"].copy(), xy=sc["XYbounds"].copy(), x0=np.zeros((B, 4)),
             xF=np.zeros((B, 4)), r=np.zeros((B, NS)), xw=np.zeros((B, 4, NS)), uw=np.zeros((B, 2, N)),
             Nb=None if Nb is None else np.ascontiguousarray(Nb, dtype=np.int32))
    outs = [np.full((B, NS, 4), 7.0), np.full((B, N, 2), 7.0), np.full((B, NS), 7.0), np.full((B, NS, 5), 7.0), np.full((B, NS, 12), 7.0),
            np.full((B, NS, 3), 7.0), np.full(B, 7, np.int32), np.full(B, 7, np.int32), np.full(B, 7.0), np.full(1, 7.0)]
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    head = [C.c_int(B)] + ([] if Nb is None else [p(k["Nb"])]) + [C.c_int(N)]
    args = head + [C.c_int(3), p(k["vOb"]), p(k["A"]), p(k["b"]), p(k["x0"]), p(k["xF"]), C.c_double(0.6), C.c_double(2.7), p(k["ego"]),
                   p(k["xy"]), p(k["r"]), p(k["r"]), p(k["r"]), p(k["xw"]), p(k["uw"]), None, None, C.c_int(0), C.c_int(1), None] + \
        [p(a) for a in outs]
    return args, (k, outs)


def test_horizon_past_the_bound_is_refused_before_any_device_work():
    """N = 320 in every solve entry, and Nmax = 320 in the mixed one with every problem's own horizon short: OBCA_ERR_UNSUPPORTED
    (with or without a device), the message names the bound, and no output is written."""
    import obca_b200
    lib = obca_b200.lib()
    for entry, Nb in (("obca_parking_solve_batch", None), ("obca_parking_solve_batch_dev", None), ("obca_parking_solve_mixed", [20, 40])):
        args, (_, outs) = _args(2, NMAX + 1, Nb)
        assert getattr(lib, entry)(*args) == -4, entry
        msg = lib.obca_last_error().decode()
        assert "319" in msg and "320" in msg, msg
        for a in outs:
            assert (a == 7).all(), entry


def test_longest_horizon_passes_the_shape_checks():
    """N = 319 (and Nmax = 319) is a shape the solve entries take: without a device they stop at OBCA_ERR_NO_DEVICE."""
    import obca_b200
    lib = obca_b200.lib()
    if lib.obca_device_count() > 0:
        pytest.skip("CUDA device present")
    for entry, Nb in (("obca_parking_solve_batch", None), ("obca_parking_solve_batch_dev", None), ("obca_parking_solve_mixed", [20, 319])):
        args, (_, outs) = _args(2, NMAX, Nb)
        assert getattr(lib, entry)(*args) == -2, (entry, lib.obca_last_error())
        assert b"no CUDA device" in lib.obca_last_error()
        for a in outs:
            assert (a == 7).all(), entry
