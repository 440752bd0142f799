"""Parking problems with horizons past 127 steps (up to N = 319) on the GPU (pytest -m gpu): the oracle's goldens of the
reference's own start pose at sampleN = 1 (N = 192), bit-identical schedules at N = 128 .. 319, a mixed batch with Nmax = 319
whose short problems keep the bits of their own layout, the largest obstacle sets at N = 319, the refusal of N = 320, and the
planner -> solve -> checker flow of a sweep at sampleN = 1."""
import contextlib
import ctypes as C
import glob
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDENS = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(HERE, "golden", "long_park", "*.npz")))
ENV_KEYS = ("OBCA_MODE", "OBCA_TAIL_THRESH", "OBCA_CHUNK", "OBCA_GRAPH")


@pytest.fixture(scope="module")
def P():
    import obca_b200
    if obca_b200.lib().obca_device_count() < 1:
        pytest.fail("pytest -m gpu needs a CUDA device (libobca has no CPU fallback)")
    from obca_b200 import parking
    return parking


@contextlib.contextmanager
def env(**kw):
    old = {k: os.environ.get(k) for k in ENV_KEYS}
    try:
        for k in old:
            os.environ.pop(k, None)
        os.environ.update(kw)
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def long_batch(B, N, seed, sc=None):
    """Config-2 start poses (reverse_parking_batch's ranges) with geometric warm starts at horizon N and Ts = 48 / N: the 48 s of
    config 2's N = 80, Ts = 0.6, sampled more finely.  sc: the obstacle set (default: the reverse-parking scene)."""
    from obca_b200 import scenarios
    sc = dict(sc if sc is not None else scenarios.reverse_parking_scenario())
    rng = np.random.default_rng(seed)
    x0 = np.stack([rng.uniform(-10, 10, B), rng.uniform(6.5, 9.5, B), np.zeros(B), np.zeros(B)], 1)
    Ts = 48.0 / N
    w = [scenarios.warmstart_reverse(x0[i], sc["xF"], N, Ts, sc["L"]) for i in range(B)]
    sc.update(B=B, N=N, Ts=Ts, x0=x0, rx=np.stack([a[0] for a in w]), ry=np.stack([a[1] for a in w]), ryaw=np.stack([a[2] for a in w]),
              xWS=np.stack([a[3] for a in w]), uWS=np.stack([a[4] for a in w]))
    return sc


def solve(P, sc, sd=1, lWS=None, nWS=None, opts=None):
    return P.parking_solve_batch(sc["x0"], sc["xF"], sc["N"], sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"],
                                 sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], 0, sc["xWS"], sc["uWS"], sd, lWS, nWS, opts)


def same(r1, r2, keys=("xp", "up", "ts", "lp", "np", "sl", "iters", "exitflag", "kkt_err")):
    for k in keys:
        assert np.array_equal(r1[k], r2[k], equal_nan=True), k


def rounds_of_last_call():
    import obca_b200
    rnd, hand = C.c_int(), C.c_int()
    assert obca_b200.lib().obca_last_schedule(C.c_int(0), C.byref(rnd), C.byref(hand), None) == 0
    return rnd.value


def load_golden(case):
    from obca_b200 import scenarios
    g = np.load(os.path.join(HERE, "golden", "long_park", case + ".npz"))
    sc = scenarios.reverse_parking_scenario()
    sc.update(B=1, N=int(g["N"]), Ts=float(g["Ts"]), x0=g["x0"][None], rx=g["rx"][None], ry=g["ry"][None], ryaw=g["ryaw"][None],
              xWS=g["xWS"][None], uWS=g["uWS"][None])
    return g, sc


@pytest.mark.parametrize("case", GOLDENS)
def test_long_golden_matches_oracle(P, case):
    """main.jl's pose at sampleN = 1 (N = 192): the oracle's solution at the tolerances of
    test_gpu_parking.test_matches_oracle_golden, a KKT point of the reference formulation, accepted by ParkingConstraints."""
    from oracle import checkers, dualmultws_ref, kkt_check
    g, sc = load_golden(case)
    N, variant = sc["N"], str(g["variant"])
    sd = 1 if variant == "sd" else 0
    r = solve(P, sc, sd, g["lWS"][None], g["nWS"][None])
    assert r["exitflag"][0] == 1
    assert np.abs(r["xp"][0] - g["xp"]).max() < 2e-4 and np.abs(r["up"][0] - g["up"]).max() < 2e-4
    assert np.abs(r["ts"][0] - g["ts"]).max() < 1e-5
    vo = np.concatenate([[0], np.cumsum(sc["vOb"])])
    gg, off = dualmultws_ref.ego_geometry(sc["ego"])
    for j in range(sc["nOb"]):
        if sd:
            act = np.flatnonzero(100.0 + 2e4 * g["sl"][j] > 5e-2)
        else:
            dist = np.array([dualmultws_ref.rect_poly_distance((g["xp"][0, k], g["xp"][1, k], g["xp"][2, k]), sc["A"][vo[j]:vo[j + 1]],
                                                               sc["b"].ravel()[vo[j]:vo[j + 1]], gg, off) for k in range(N + 1)])
            act = np.flatnonzero(dist < 0.05 + 2e-4)
        if len(act):
            assert np.abs(r["lp"][0][vo[j]:vo[j + 1]][:, act] - g["lp"][vo[j]:vo[j + 1]][:, act]).max() < 2e-3, j
            assert np.abs(r["np"][0][4 * j:4 * j + 4][:, act] - g["np"][4 * j:4 * j + 4][:, act]).max() < 2e-3, j
    if sd:
        assert np.abs(r["sl"][0] - g["sl"]).max() < 2e-5
    assert kkt_check.reference_kkt_error(sc, 0, r, variant, 0)["E0"] < 1e-4
    args = (sc["x0"][0], sc["xF"], N, sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"], sc["b"],
            r["xp"][0], r["up"][0], r["lp"][0], r["np"][0], r["ts"][0], 0, sd)
    assert checkers.ParkingConstraints(*args) == 1
    # the library's own checker and DualMultWS at N = 192
    feas, _, _ = P.check_parking_batch(sc["x0"], sc["xF"], N, sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"],
                                       sc["b"], r["xp"], r["up"], r["lp"], r["np"], r["ts"], 0, sd, r["sl"])
    assert feas[0] == 1
    _, _, d = P.dualmultws_batch(N, sc["nOb"], sc["vOb"], sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], sc["ego"], want_d=True)
    assert np.abs(d[0] - g["dWS"]).max() < 2e-5


@pytest.mark.parametrize("N", [128, 192, 255, 319])
def test_long_horizon_schedules_bit_identical(P, N):
    """The persistent kernel alone, rounds alone, the automatic schedule and plain launches give the same bits.  B = 640 is more
    than twice the tail kernel's resident CTAs at every one of these horizons (2 per SM at N = 128, 1 above), so rounds run."""
    sc = long_batch(640, N, 21)
    with env(OBCA_MODE="1"):
        r1 = solve(P, sc)
    assert rounds_of_last_call() == 0
    with env(OBCA_MODE="2", OBCA_TAIL_THRESH="0"):
        r2 = solve(P, sc)
    with env():
        r0 = solve(P, sc)
    assert rounds_of_last_call() > 0
    with env(OBCA_GRAPH="0"):
        r3 = solve(P, sc)
    assert r1["exitflag"].mean() > 0.9, r1["exitflag"].mean()
    same(r1, r2); same(r1, r0); same(r1, r3)


def _mixed_raw(sc, Ns, Nmax):
    """obca_parking_solve_mixed through ctypes with NaN-filled outputs, in the C layout: (xp (B,NS,4), up (B,Nmax,2), ts, lp, np, sl,
    exitflag, iters, kkt_err)."""
    import obca_b200
    from obca_b200._lib import f64, ptr
    Ns = np.ascontiguousarray(Ns, dtype=np.int32); B = len(Ns); NS = Nmax + 1
    pad = lambda arrs, rows: np.stack([np.concatenate([np.asarray(a, float), np.zeros((rows - len(a),) + np.shape(a)[1:])]) for a in arrs])
    rx, ry, ryaw = (f64(pad([sc[k][i][:n + 1] for i, n in enumerate(Ns)], NS)) for k in ("rx", "ry", "ryaw"))
    xW = f64(np.transpose(pad([sc["xWS"][i][:n + 1] for i, n in enumerate(Ns)], NS), (0, 2, 1)))
    uW = f64(np.transpose(pad([sc["uWS"][i][:n] for i, n in enumerate(Ns)], Nmax), (0, 2, 1)))
    vOb = np.ascontiguousarray(sc["vOb"], dtype=np.int32); V = int(vOb.sum()); nOb = sc["nOb"]
    r = dict(xp=np.full((B, NS, 4), np.nan), up=np.full((B, Nmax, 2), np.nan), ts=np.full((B, NS), np.nan), lp=np.full((B, NS, V), np.nan),
             np=np.full((B, NS, 4 * nOb), np.nan), sl=np.full((B, NS, nOb), np.nan), exitflag=np.zeros(B, np.int32),
             iters=np.zeros(B, np.int32), kkt_err=np.zeros(B))
    sec = np.zeros(1)
    o = obca_b200.default_opts()
    rc = obca_b200.lib().obca_parking_solve_mixed(
        C.c_int(B), ptr(Ns), C.c_int(Nmax), C.c_int(nOb), ptr(vOb), ptr(np.asfortranarray(sc["A"], dtype=float)),
        ptr(f64(sc["b"].ravel())), ptr(f64(sc["x0"])), ptr(f64(np.broadcast_to(sc["xF"], (B, 4)))), C.c_double(sc["Ts"]),
        C.c_double(sc["L"]), ptr(f64(sc["ego"])), ptr(f64(sc["XYbounds"])), ptr(rx), ptr(ry), ptr(ryaw), ptr(xW), ptr(uW), None, None,
        C.c_int(0), C.c_int(1), C.byref(o), *[ptr(r[k]) for k in ("xp", "up", "ts", "lp", "np", "sl", "exitflag", "iters", "kkt_err")],
        ptr(sec))
    assert rc == 0, obca_b200.lib().obca_last_error()
    return r


def test_mixed_batch_up_to_319(P):
    """Horizons 20 .. 319 in one call laid out for Nmax = 319: every problem gives the bits of its uniform solve at its own N (for
    N <= 127 that is the layout of the 128-stage build), the NaN padding of the outputs is never written, a small OBCA_CHUNK gives
    the same bits, and the mixed checker agrees with the uniform one."""
    from obca_b200 import scenarios
    B, HOR = 112, (20, 64, 127, 128, 200, 255, 319)
    Ns = np.random.default_rng(31).choice(HOR, B)
    assert set(Ns) == set(HOR)
    sc = scenarios.reverse_parking_scenario()
    rng = np.random.default_rng(32)
    x0 = np.stack([rng.uniform(-10, 10, B), rng.uniform(6.5, 9.5, B), np.zeros(B), np.zeros(B)], 1)
    Ts = 0.25
    w = [scenarios.warmstart_reverse(x0[i], sc["xF"], int(Ns[i]), Ts, sc["L"]) for i in range(B)]
    sc.update(B=B, Ts=Ts, x0=x0, rx=[a[0] for a in w], ry=[a[1] for a in w], ryaw=[a[2] for a in w], xWS=[a[3] for a in w],
              uWS=[a[4] for a in w])
    with env():
        rm = _mixed_raw(sc, Ns, 319)
    with env(OBCA_CHUNK="24"):
        rc = _mixed_raw(sc, Ns, 319)
    for k in rm:
        assert np.array_equal(rm[k], rc[k], equal_nan=True), k
    for i, n in enumerate(Ns):
        for key, ext in (("xp", 1), ("ts", 1), ("lp", 1), ("np", 1), ("sl", 1), ("up", 0)):
            assert not np.isnan(rm[key][i, :n + ext]).any() and np.isnan(rm[key][i, n + ext:]).all(), (key, i)
    uni = {}
    for N in HOR:
        idx = np.flatnonzero(Ns == N)
        st = lambda key: np.stack([sc[key][i] for i in idx])
        with env():
            ru = P.parking_solve_batch(x0[idx], sc["xF"], int(N), Ts, sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"],
                                       sc["b"], st("rx"), st("ry"), st("ryaw"), 0, st("xWS"), st("uWS"))
        for q, i in enumerate(idx):
            for key, ext in (("xp", 1), ("ts", 1), ("lp", 1), ("np", 1), ("sl", 1), ("up", 0)):
                m = rm[key][i, :N + ext]
                assert np.array_equal(m.T if m.ndim == 2 else m, ru[key][q]), (N, i, key)
            assert rm["exitflag"][i] == ru["exitflag"][q] and rm["iters"][i] == ru["iters"][q], (N, i)
            assert rm["kkt_err"][i] == ru["kkt_err"][q] or (np.isnan(rm["kkt_err"][i]) and np.isnan(ru["kkt_err"][q])), (N, i)
        uni[N] = (idx, P.check_parking_batch(x0[idx], sc["xF"], int(N), Ts, sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"],
                                             sc["A"], sc["b"], ru["xp"], ru["up"], ru["lp"], ru["np"], ru["ts"], 0, 1, ru["sl"]))
    cut = lambda key, ext: [rm[key][i, :n + ext].T for i, n in enumerate(Ns)]
    feas, e, strict = P.check_parking_mixed(x0, sc["xF"], Ns, Ts, sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"], sc["b"],
                                            cut("xp", 1), cut("up", 0), cut("lp", 1), cut("np", 1), [rm["ts"][i, :n + 1] for i, n in enumerate(Ns)],
                                            0, 1, cut("sl", 1))
    for N, (idx, (f2, e2, s2)) in uni.items():
        assert np.array_equal(feas[idx], f2) and np.array_equal(e[idx], e2) and np.array_equal(strict[idx], s2), N
    conv = rm["exitflag"] == 1
    assert conv.mean() > 0.5, conv.mean()
    assert feas[conv].all()


def _sixteen_by_four(sc):
    """15 parked cars plus the far wall as a 4-half-space box: nOb = 16, sum(vOb) = 64."""
    from obca_b200 import scenarios
    lOb = sc["lOb"][:-1] + [[[-20, 12], [20, 12], [20, 11], [-20, 11], [-20, 12]]]
    A, b = scenarios.obst_hrep(16, [5] * 16, lOb)
    sc = dict(sc)
    sc.update(vOb=np.full(16, 4), A=A, b=b, lOb=lOb)
    return sc


@pytest.mark.parametrize("shape", ["lot15", "16x4"])
def test_largest_shapes_at_319(P, shape):
    """The largest obstacle sets at the longest horizon (about 3.3 MB of workspace per problem): they converge as at N = 127
    (test_gpu_many_obstacles.test_largest_shapes_at_long_horizons), rounds and the persistent kernel give the same bits, and a
    later config-2 call still runs."""
    from obca_b200 import scenarios
    lot = scenarios.parking_lot_scenario(15)
    sc = long_batch(96, 319, 2, lot if shape == "lot15" else _sixteen_by_four(lot))
    with env(OBCA_MODE="1"):
        r1 = solve(P, sc)
    with env(OBCA_MODE="2", OBCA_TAIL_THRESH="0"):
        r2 = solve(P, sc)
    assert r1["exitflag"].mean() > 0.9, r1["exitflag"]
    same(r1, r2)
    r3 = solve(P, scenarios.reverse_parking_batch(8, 80, 0))
    assert r3["exitflag"].sum() >= 7


def test_horizon_past_the_bound_is_refused_on_the_device(P):
    """N = 320 writes no output and leaves the device ready: the next call solves normally."""
    import obca_b200
    from obca_b200 import scenarios
    from obca_b200._lib import f64, ptr
    lib = obca_b200.lib()
    sc = long_batch(4, 320, 3)
    B, N, NS = 4, 320, 321
    outs = [np.full((B, NS, 4), np.nan), np.full((B, N, 2), np.nan), np.full((B, NS), np.nan), np.full((B, NS, 5), np.nan),
            np.full((B, NS, 12), np.nan), np.full((B, NS, 3), np.nan), np.full(B, -7, np.int32), np.full(B, -7, np.int32), np.full(B, np.nan),
            np.full(1, np.nan)]
    o = obca_b200.default_opts()
    rc = lib.obca_parking_solve_batch(C.c_int(B), C.c_int(N), C.c_int(3), ptr(np.ascontiguousarray(sc["vOb"], dtype=np.int32)),
                                      ptr(np.asfortranarray(sc["A"], dtype=float)), ptr(f64(sc["b"].ravel())), ptr(f64(sc["x0"])),
                                      ptr(f64(np.tile(sc["xF"], (B, 1)))), C.c_double(sc["Ts"]), C.c_double(sc["L"]), ptr(f64(sc["ego"])),
                                      ptr(f64(sc["XYbounds"])), ptr(f64(sc["rx"])), ptr(f64(sc["ry"])), ptr(f64(sc["ryaw"])),
                                      ptr(f64(np.transpose(sc["xWS"], (0, 2, 1)))), ptr(f64(np.transpose(sc["uWS"], (0, 2, 1)))), None, None,
                                      C.c_int(0), C.c_int(1), C.byref(o), *[ptr(a) for a in outs])
    assert rc == -4 and b"319" in lib.obca_last_error(), (rc, lib.obca_last_error())
    for a in outs:
        assert (np.isnan(a).all() if a.dtype == np.float64 else (a == -7).all())
    r = solve(P, scenarios.reverse_parking_batch(8, 80, 0))
    assert r["exitflag"].sum() >= 7


@pytest.mark.parametrize("planner", ["host", "gpu"])
def test_planned_sweep_at_sample_n_one(P, planner):
    """48 poses of the backwards sweep planned at sampleN = 1 (Ts = 0.2, horizons past 127), solved in ONE mixed call and checked in
    ONE mixed checker call: at least 90 % converge and every converged problem passes ParkingConstraints."""
    from obca_b200 import scenarios
    from obca_b200.planner import device, native
    sc = scenarios.reverse_parking_scenario()
    rng = np.random.default_rng(0)
    x0 = np.column_stack([rng.uniform(-9, 9, 48), rng.uniform(6.8, 9.3, 48), np.zeros(48), np.zeros(48)])
    plans = native.plan_batch(x0, sc["xF"], "backwards", 0, sampleN=1) if planner == "host" else \
        device.plan_batch(x0, sc["xF"], "backwards", sampleN=1)
    ok = [i for i, w in enumerate(plans) if w is not None]
    assert len(ok) >= 44
    Ts = plans[ok[0]]["Ts"]
    assert Ts == pytest.approx(0.2)
    g = lambda key: [plans[i][key] for i in ok]
    Ns = np.array([plans[i]["N"] for i in ok])
    assert Ns.max() > 127 and Ns.max() <= 319, Ns
    r = P.parking_solve_mixed(x0[ok], sc["xF"], Ns, Ts, sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"], sc["b"],
                              g("rx"), g("ry"), g("ryaw"), 0, g("xWS"), g("uWS"))
    conv = r["exitflag"] == 1
    print("planned", len(ok), "N", Ns.min(), "..", Ns.max(), "converged", int(conv.sum()))
    assert conv.mean() >= 0.9, conv.mean()
    feas, _, _ = P.check_parking_mixed(x0[ok], sc["xF"], Ns, Ts, sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"], sc["b"],
                                       r["xp"], r["up"], r["lp"], r["np"], r["ts"], 0, 1, r["sl"])
    assert np.asarray(feas)[conv].all()
