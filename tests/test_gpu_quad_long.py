"""Quadcopter problems with horizons past 127 stages on the GPU (N + 1 > 128: a CTA of 128 threads, thread t handles the stages
t, t + 128, ...).  The device sweep agrees with the host recursion where two, three and four stages share a thread; in a mixed
batch every problem gives the bits of the uniform solve of its horizon, short and long alike; A*-planned long pairs solve in
one call with the short ones; the mixed checker agrees with the uniform one and with the verbatim constrSatisfaction; and a
horizon past the bound (N + 1 > 512) is refused before any launch."""
import ctypes as C
import os

import numpy as np
import pytest

from obca_b200 import scenarios
from oracle import checkers, kkt_check
from oracle.quadcopter_nlp import build_quadcopter_nlp

pytestmark = pytest.mark.gpu

NMAX = 511                                      # the library's bound: N + 1 <= 512
HORIZONS = (20, 100, 127, 128, 147, 255, 511)   # one to four warps with one stage per thread, then two, three, four stages per thread
HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_LONG = os.path.join(HERE, "golden", "quad_astar_long_pairs.npz")
GOLDEN_SHORT = os.path.join(HERE, "golden", "quad_astar_pairs.npz")


@pytest.fixture(scope="module")
def Q():
    import obca_b200
    if obca_b200.lib().obca_device_count() < 1:
        pytest.fail("pytest -m gpu needs a CUDA device (libobca has no CPU fallback)")
    from obca_b200 import quadcopter
    return quadcopter


def cert(x0, xF, N, Ts, R, obs, variant, xp, up, ts, lp, sl):
    nlp = build_quadcopter_nlp(x0, xF, N, Ts, R, obs, variant)
    return kkt_check.kkt_certificate(nlp, nlp.lay.pack(xp, up, ts, lp, sl if variant == "sd" else None))


@pytest.mark.parametrize("N", [128, 147, 255, 256, 511])
def test_long_horizon_sweep_equals_host_recursion(Q, N):
    """As tests/test_quadcopter.py::test_gpu_tensor_core_sweep_equals_host_recursion, past one stage per thread: the first Newton
    step and the iterate after five iterations agree with the one-thread recursion of the host build (dc = 1e-6), then the full
    solve converges to a KKT point of the reference NLP that both checkers accept."""
    import emul
    import obca_b200
    B = 3
    sc = scenarios.quadcopter_batch(B, N, 2)
    for variant in ("sd", "d"):
        sd = 1 if variant == "sd" else 0
        for it, tol in ((1, 1e-8), (5, 1e-4)):
            oe = emul.default_opts(); oe.max_iter = it; oe.dc = 1e-6
            og = obca_b200.default_opts(); og.max_iter = it; og.dc = 1e-6
            re_ = emul.quad_solve_batch(sc, variant, oe)
            rg = Q.quadcopter_solve_batch(sc["x0"], sc["xF"], N, sc["Ts"], sc["R"], sc["obs"], sc["xWS"], 1.0, sd, og)
            for k in ("xp", "up", "ts", "lp"):
                scale = 1.0 + np.abs(re_[k]).max()
                assert np.abs(rg[k] - re_[k]).max() < tol * scale, (variant, it, k, np.abs(rg[k] - re_[k]).max())
        r = Q.quadcopter_solve_batch(sc["x0"], sc["xF"], N, sc["Ts"], sc["R"], sc["obs"], sc["xWS"], 1.0, sd)
        assert (r["exitflag"] >= 1).all(), (variant, r["exitflag"])
        feas, _ = Q.check_quadcopter_batch(r["xp"], r["up"], r["ts"], sc["x0"], sc["xF"], sc["Ts"], r["lp"], sc["obs"], sc["R"])
        for i in range(B):
            ref = checkers.constrSatisfaction(r["xp"][i], r["up"][i], r["ts"][i], sc["x0"][i], sc["xF"][i], sc["Ts"], r["lp"][i],
                                              *sc["obs"], sc["R"])
            assert bool(feas[i]) == ref, (variant, i)
        assert feas[r["exitflag"] == 1].all()
        i = int(np.argmax(r["exitflag"] == 1))
        e = cert(sc["x0"][i], sc["xF"][i], N, sc["Ts"], sc["R"], sc["obs"], variant, r["xp"][i], r["up"][i], r["ts"][i], r["lp"][i],
                 r["slack"][i])
        assert e["E0"] < 1e-4, (variant, e["E0"])


def long_mixed_batch():
    """Three problems per horizon of HORIZONS, interleaved."""
    Ns = np.random.default_rng(11).permutation(np.repeat(HORIZONS, 3))
    assert len(set(Ns[:7].tolist())) > 2 and not (np.diff(Ns) >= 0).all()
    return scenarios.quadcopter_mixed_batch(len(Ns), Ns=Ns, seed=6)


def solve_mixed_raw(sc, sd):
    """obca_quadcopter_solve_mixed through the C ABI with NaN in the padding of every input and output array; returns the padded
    outputs in the library's layout (B, stages, rows)."""
    import obca_b200
    from obca_b200._lib import f64, ptr
    Ns = np.ascontiguousarray(sc["Ns"], dtype=np.int32); B = len(Ns); Nmax = int(Ns.max()); NS = Nmax + 1
    xw = np.full((B, NS, 12), np.nan)
    for i, w in enumerate(sc["xWS"]):
        xw[i, :w.shape[1]] = w.T
    out = dict(xp=np.full((B, NS, 12), np.nan), up=np.full((B, Nmax, 4), np.nan), ts=np.full((B, NS), np.nan),
               lp=np.full((B, NS, 30), np.nan), slack=np.full((B, NS, 5), np.nan), exitflag=np.zeros(B, np.int32),
               iters=np.zeros(B, np.int32), kkt_err=np.zeros(B), sec=np.zeros(1))
    o = obca_b200.default_opts(); o.max_iter = 3000
    rc = obca_b200.lib().obca_quadcopter_solve_mixed(
        C.c_int(B), ptr(Ns), C.c_int(Nmax), ptr(f64(sc["x0"])), ptr(f64(sc["xF"])), ptr(f64(sc["Ts"])), C.c_double(sc["R"]),
        ptr(f64(sc["obs"])), ptr(xw), C.c_double(1.0), C.c_int(sd), C.byref(o), *(ptr(out[k]) for k in
                                                                                 ("xp", "up", "ts", "lp", "slack", "exitflag", "iters", "kkt_err", "sec")))
    assert rc == 0, obca_b200.lib().obca_last_error()
    return out


@pytest.mark.parametrize("sd", [1, 0], ids=["sd", "dist"])
def test_long_mixed_batch_equals_uniform_per_horizon(Q, sd):
    """Horizons 20..511 interleaved in one call (CTAs of 128 threads for all of them): every problem has the bits of the uniform
    solve of its horizon -- a short problem those of its own round32(N + 1)-thread CTA, a long one those of the uniform entry's
    128-thread CTA -- and the NaN padding of the outputs is never written."""
    sc = long_mixed_batch()
    r = solve_mixed_raw(sc, sd)
    keys = (("xp", 1), ("ts", 1), ("lp", 1), ("up", 0)) + ((("slack", 1),) if sd else ())
    for i, n in enumerate(sc["Ns"]):
        for key, ext in keys:
            assert not np.isnan(r[key][i, :n + ext]).any() and np.isnan(r[key][i, n + ext:]).all(), (key, i, n)
    for N in HORIZONS:
        idx = np.flatnonzero(sc["Ns"] == N)
        Ts = float(sc["Ts"][idx[0]])
        assert (sc["Ts"][idx] == Ts).all()
        u = Q.quadcopter_solve_batch(sc["x0"][idx], sc["xF"][idx], N, Ts, sc["R"], sc["obs"], np.stack([sc["xWS"][i] for i in idx]), 1.0, sd)
        for k, i in enumerate(idx):
            for key, ext in keys:
                got = r[key][i, :N + ext].T if key != "ts" else r[key][i, :N + 1]
                assert np.array_equal(got, u[key][k]), (key, i, N)
            assert r["exitflag"][i] == u["exitflag"][k] and r["iters"][i] == u["iters"][k], (i, N)
            assert r["kkt_err"][i] == u["kkt_err"][k] or (np.isnan(r["kkt_err"][i]) and np.isnan(u["kkt_err"][k])), (i, N)
    assert (r["exitflag"] >= 1).mean() > 0.8, r["exitflag"]


def test_long_mixed_checker_equals_uniform_checker_and_reference(Q):
    """obca_check_quadcopter_mixed at Nmax = 511 against obca_check_quadcopter per horizon and the verbatim constrSatisfaction."""
    sc = long_mixed_batch()
    r = Q.quadcopter_solve_mixed(sc["x0"], sc["xF"], sc["Ns"], sc["Ts"], sc["R"], sc["obs"], sc["xWS"], 1.0, 1)
    feas, worst = Q.check_quadcopter_mixed(r["xp"], r["up"], r["ts"], sc["x0"], sc["xF"], sc["Ns"], sc["Ts"], r["lp"], sc["obs"], sc["R"])
    for N in HORIZONS:
        idx = np.flatnonzero(sc["Ns"] == N)
        st = lambda key: np.stack([r[key][i] for i in idx])
        f2, w2 = Q.check_quadcopter_batch(st("xp"), st("up"), st("ts"), sc["x0"][idx], sc["xF"][idx], float(sc["Ts"][idx[0]]), st("lp"),
                                          sc["obs"], sc["R"])
        assert np.array_equal(feas[idx], f2) and np.array_equal(worst[idx], w2), N
    for i in range(sc["B"]):
        ref = checkers.constrSatisfaction(r["xp"][i], r["up"][i], r["ts"][i], sc["x0"][i], sc["xF"][i], sc["Ts"][i], r["lp"][i], *sc["obs"],
                                          sc["R"])
        assert bool(feas[i]) == ref, i
    assert feas[r["exitflag"] == 1].all()


def test_planned_long_pairs_with_the_short_ones_in_one_call(Q):
    """The A*-planned long pairs (tests/golden/make_quad_astar_long.py) and the short ones of quad_astar_pairs.npz in ONE mixed call:
    the same bits as one call per (N, Ts), every converged trajectory passes constrSatisfaction, and three long ones are KKT
    points of the reference NLP."""
    gl, gs = np.load(GOLDEN_LONG), np.load(GOLDEN_SHORT)
    assert gl["N"].min() > 127
    x0 = np.concatenate([gl["x0"], gs["x0"]]); xF = np.concatenate([gl["xF"], gs["xF"]])
    Ns = np.concatenate([gl["N"], gs["N"]]); Ts = np.concatenate([gl["Ts"], gs["Ts"]])
    xWS = [g["xWS"][i][:, :int(n) + 1] for g in (gl, gs) for i, n in enumerate(g["N"])]
    sc = scenarios.quadcopter_scenario()
    r = Q.quadcopter_solve_mixed(x0, xF, Ns, Ts, sc["R"], sc["obs"], xWS, 1.0, 1)
    for N in np.unique(Ns):
        for T in np.unique(Ts[Ns == N]):
            sub = np.flatnonzero((Ns == N) & (Ts == T))
            u = Q.quadcopter_solve_batch(x0[sub], xF[sub], int(N), float(T), sc["R"], sc["obs"], np.stack([xWS[i] for i in sub]), 1.0, 1)
            for k, i in enumerate(sub):
                for key in ("xp", "up", "ts", "lp", "slack"):
                    assert np.array_equal(r[key][i], u[key][k]), (key, i)
                assert r["exitflag"][i] == u["exitflag"][k] and r["iters"][i] == u["iters"][k] and r["kkt_err"][i] == u["kkt_err"][k]
    conv = np.flatnonzero(r["exitflag"] == 1)
    assert (r["exitflag"][:len(gl["N"])] >= 1).all(), r["exitflag"]
    for i in conv:
        assert checkers.constrSatisfaction(r["xp"][i], r["up"][i], r["ts"][i], x0[i], xF[i], Ts[i], r["lp"][i], *sc["obs"], sc["R"]), i
    for i in conv[:3]:
        e = cert(x0[i], xF[i], int(Ns[i]), float(Ts[i]), sc["R"], sc["obs"], "sd", r["xp"][i], r["up"][i], r["ts"][i], r["lp"][i],
                 r["slack"][i])
        assert e["E0"] < 1e-4, (i, e["E0"])


def test_horizon_past_the_bound_is_refused_before_any_launch(Q):
    """N = 512 in the uniform entry and Nmax = 512 in the mixed one (whatever the problems' own horizons): OBCA_ERR_UNSUPPORTED
    with the bound in the message, and no output written."""
    import obca_b200
    from obca_b200._lib import ptr
    lib = obca_b200.lib()
    sc = scenarios.quadcopter_scenario()
    B, N = 2, NMAX + 1
    NS = N + 1
    x0 = np.zeros((B, 12)); xF = np.zeros((B, 12)); ob = np.ascontiguousarray(sc["obs"], dtype=float); xw = np.zeros((B, NS, 12))
    outs = [np.full((B, NS, 12), 7.0), np.full((B, N, 4), 7.0), np.full((B, NS), 7.0), np.full((B, NS, 30), 7.0), np.full((B, NS, 5), 7.0),
            np.full(B, 7, np.int32), np.full(B, 7, np.int32), np.full(B, 7.0), np.full(1, 7.0)]
    head = [C.c_int(B), C.c_int(N), ptr(x0), ptr(xF), C.c_double(0.04)]
    tail = [C.c_double(sc["R"]), ptr(ob), ptr(xw), C.c_double(1.0), C.c_int(1), None] + [ptr(a) for a in outs]
    assert lib.obca_quadcopter_solve_batch(*head, *tail) == -4
    assert b"511" in lib.obca_last_error(), lib.obca_last_error()
    Nb = np.array([40, 100], np.int32); Tsb = np.array([0.5, 0.2])
    assert lib.obca_quadcopter_solve_mixed(C.c_int(B), ptr(Nb), C.c_int(N), ptr(x0), ptr(xF), ptr(Tsb), *tail) == -4
    assert b"511" in lib.obca_last_error(), lib.obca_last_error()
    for a in outs:
        assert (a == 7).all()
