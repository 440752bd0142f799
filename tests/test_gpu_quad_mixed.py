"""Quadcopter problems with different horizons and sampling times in one solve (obca_quadcopter_solve_mixed) on the GPU: every
problem gives the same bits as the uniform solve of its horizon group (one to four warps per problem in CTAs sized for the
longest horizon), the padding of the outputs is never written, the mixed checker agrees with the uniform one and with the
verbatim constrSatisfaction, and a batch of A*-planned pairs solved in one call equals the per-horizon path."""
import ctypes as C
import os

import numpy as np
import pytest

from obca_b200 import scenarios
from oracle import checkers, kkt_check
from oracle.quadcopter_nlp import build_quadcopter_nlp

pytestmark = pytest.mark.gpu

HORIZONS = (20, 45, 70, 100, 127)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "quad_astar_pairs.npz")


@pytest.fixture(scope="module")
def Q():
    import obca_b200
    if obca_b200.lib().obca_device_count() < 1:
        pytest.fail("pytest -m gpu needs a CUDA device (libobca has no CPU fallback)")
    from obca_b200 import quadcopter
    return quadcopter


def mixed_batch(B=60, seed=5):
    Ns = np.random.default_rng(seed + 100).choice(HORIZONS, B)
    assert len(set(Ns[:10])) > 1 and not (np.diff(Ns) >= 0).all()
    return scenarios.quadcopter_mixed_batch(B, Ns=Ns, seed=seed)


def groups(Ns):
    return {int(N): np.flatnonzero(np.asarray(Ns) == N) for N in np.unique(Ns)}


def solve_groups(Q, sc, sd):
    """The path used before the mixed entry: one uniform solve per horizon (all problems of a horizon share its Ts)."""
    out = {}
    for N, idx in groups(sc["Ns"]).items():
        Ts = float(sc["Ts"][idx[0]])
        assert (sc["Ts"][idx] == Ts).all()
        out[N] = (idx, Q.quadcopter_solve_batch(sc["x0"][idx], sc["xF"][idx], N, Ts, sc["R"], sc["obs"],
                                                np.stack([sc["xWS"][i] for i in idx]), 1.0, sd))
    return out


def assert_same(r, ref, sd):
    keys = ("xp", "up", "ts", "lp") + (("slack",) if sd else ())
    for N, (idx, u) in ref.items():
        for k, i in enumerate(idx):
            for key in keys:
                assert np.array_equal(r[key][i], u[key][k]), (key, i, N)
            assert r["exitflag"][i] == u["exitflag"][k] and r["iters"][i] == u["iters"][k], (i, N)
            assert r["kkt_err"][i] == u["kkt_err"][k] or (np.isnan(r["kkt_err"][i]) and np.isnan(u["kkt_err"][k])), (i, N)


def cert(x0, xF, N, Ts, R, obs, variant, xp, up, ts, lp, sl):
    nlp = build_quadcopter_nlp(x0, xF, N, Ts, R, obs, variant)
    return kkt_check.kkt_certificate(nlp, nlp.lay.pack(xp, up, ts, lp, sl if variant == "sd" else None))


@pytest.mark.parametrize("sd", [1, 0], ids=["sd", "dist"])
def test_mixed_equals_uniform_per_horizon(Q, sd):
    sc = mixed_batch()
    r = Q.quadcopter_solve_mixed(sc["x0"], sc["xF"], sc["Ns"], sc["Ts"], sc["R"], sc["obs"], sc["xWS"], 1.0, sd)
    assert np.array_equal(r["N"], sc["Ns"]) and np.array_equal(r["Ts"], sc["Ts"])
    assert_same(r, solve_groups(Q, sc, sd), sd)
    assert (r["exitflag"] >= 1).mean() > 0.8 and r["time"] > 0


def test_output_padding_is_never_written(Q):
    """Direct C-ABI call with NaN-filled outputs: past each problem's horizon they still hold NaN afterwards."""
    import obca_b200
    from obca_b200._lib import f64, ptr
    sc = mixed_batch(24, seed=8)
    Ns = np.ascontiguousarray(sc["Ns"], dtype=np.int32); B = len(Ns); Nmax = int(Ns.max()); NS = Nmax + 1
    xw = np.full((B, NS, 12), np.nan)                      # input padding NaN too: it must not be read
    for i, w in enumerate(sc["xWS"]):
        xw[i, :w.shape[1]] = w.T
    xp = np.full((B, NS, 12), np.nan); up = np.full((B, Nmax, 4), np.nan); ts = np.full((B, NS), np.nan)
    lp = np.full((B, NS, 30), np.nan); sl = np.full((B, NS, 5), np.nan)
    ef = np.zeros(B, np.int32); it = np.zeros(B, np.int32); err = np.zeros(B); sec = np.zeros(1)
    o = obca_b200.default_opts(); o.max_iter = 3000
    rc = obca_b200.lib().obca_quadcopter_solve_mixed(
        C.c_int(B), ptr(Ns), C.c_int(Nmax), ptr(f64(sc["x0"])), ptr(f64(sc["xF"])), ptr(f64(sc["Ts"])), C.c_double(sc["R"]),
        ptr(f64(sc["obs"])), ptr(xw), C.c_double(1.0), C.c_int(1), C.byref(o), ptr(xp), ptr(up), ptr(ts), ptr(lp), ptr(sl), ptr(ef),
        ptr(it), ptr(err), ptr(sec))
    assert rc == 0, obca_b200.lib().obca_last_error()
    for i, n in enumerate(Ns):
        for a, ext in ((xp, 1), (ts, 1), (lp, 1), (sl, 1), (up, 0)):
            assert not np.isnan(a[i, :n + ext]).any() and np.isnan(a[i, n + ext:]).all(), i
    assert sec[0] > 0 and (ef >= 1).mean() > 0.8


def test_mixed_checker_equals_uniform_checker_and_reference(Q):
    sc = mixed_batch(40, seed=9)
    r = Q.quadcopter_solve_mixed(sc["x0"], sc["xF"], sc["Ns"], sc["Ts"], sc["R"], sc["obs"], sc["xWS"], 1.0, 1)
    feas, worst = Q.check_quadcopter_mixed(r["xp"], r["up"], r["ts"], sc["x0"], sc["xF"], sc["Ns"], sc["Ts"], r["lp"], sc["obs"], sc["R"])
    for N, idx in groups(sc["Ns"]).items():
        st = lambda key: np.stack([r[key][i] for i in idx])
        f2, w2 = Q.check_quadcopter_batch(st("xp"), st("up"), st("ts"), sc["x0"][idx], sc["xF"][idx], float(sc["Ts"][idx[0]]), st("lp"),
                                          sc["obs"], sc["R"])
        assert np.array_equal(feas[idx], f2) and np.array_equal(worst[idx], w2), N
    for i in range(sc["B"]):
        ref = checkers.constrSatisfaction(r["xp"][i], r["up"][i], r["ts"][i], sc["x0"][i], sc["xF"][i], sc["Ts"][i], r["lp"][i], *sc["obs"],
                                          sc["R"])
        assert bool(feas[i]) == ref, i
    assert feas[r["exitflag"] == 1].all()


def test_planned_pairs_in_one_call(Q):
    """The 8 A*-planned config-4 pairs of the fixture (9 distinct horizons among 12 pairs in the full set, 90..127 here) in ONE
    mixed call: the same bits as one call per horizon, every converged trajectory passes constrSatisfaction, and three of them
    are KKT points of the reference NLP."""
    g = np.load(GOLDEN)
    Ns, Ts = g["N"], g["Ts"]
    xWS = [g["xWS"][i][:, :int(n) + 1] for i, n in enumerate(Ns)]
    sc = scenarios.quadcopter_scenario()
    r = Q.quadcopter_solve_mixed(g["x0"], g["xF"], Ns, Ts, sc["R"], sc["obs"], xWS, 1.0, 1)
    for N, idx in groups(Ns).items():
        for T in np.unique(Ts[idx]):
            sub = idx[Ts[idx] == T]
            u = Q.quadcopter_solve_batch(g["x0"][sub], g["xF"][sub], N, float(T), sc["R"], sc["obs"], np.stack([xWS[i] for i in sub]), 1.0, 1)
            for k, i in enumerate(sub):
                for key in ("xp", "up", "ts", "lp", "slack"):
                    assert np.array_equal(r[key][i], u[key][k]), (key, i)
                assert r["exitflag"][i] == u["exitflag"][k] and r["iters"][i] == u["iters"][k] and r["kkt_err"][i] == u["kkt_err"][k]
    conv = np.flatnonzero(r["exitflag"] == 1)
    assert len(conv) >= 6, r["exitflag"]
    for i in conv:
        assert checkers.constrSatisfaction(r["xp"][i], r["up"][i], r["ts"][i], g["x0"][i], g["xF"][i], Ts[i], r["lp"][i], *sc["obs"], sc["R"])
    for i in conv[:3]:
        e = cert(g["x0"][i], g["xF"][i], int(Ns[i]), float(Ts[i]), sc["R"], sc["obs"], "sd", r["xp"][i], r["up"][i], r["ts"][i], r["lp"][i],
                 r["slack"][i])
        assert e["E0"] < 1e-4, (i, e["E0"])
