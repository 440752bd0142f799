"""The PyTorch ops and the device-pointer entries behind them on the GPU: bit for bit what the host-pointer twins return, nothing written
past a problem's horizon, device-resident Nb / Tsb checked before anything is written, ordered after the work queued on the caller's
stream, traceable by torch.compile, and reported by obca_last_* like the twins."""
import ctypes as C

import numpy as np
import pytest
import torch

from obca_b200 import _lib, parking as pk, quadcopter as qc, scenarios
from obca_b200.parking import _pad_stages

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
F64, I32 = torch.float64, torch.int32


@pytest.fixture(scope="module")
def T():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from obca_b200 import torch_ops
    return torch_ops


def _t(a, dtype=F64):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=DEV)


def _h(t):
    return t.cpu().numpy()


def _same_over_horizons(got, ref, Ns, ext, key):
    """got: (B, r, Nmax+ext) tensor; ref: the twin's per-problem list of r x (Ns[i]+ext) arrays."""
    g = _h(got)
    for i, n in enumerate(Ns):
        assert np.array_equal(g[i, ..., :n + ext], ref[i]), (key, i)
        assert not g[i, ..., n + ext:].any(), (key, i)      # zeros past the horizon: never written


# ---- parking --------------------------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def mixed_park():
    sc = scenarios.reverse_parking_mixed_batch(512, (40, 80), seed=3)
    Ns, Nmax = sc["Ns"], int(sc["Ns"].max())
    pad = lambda arrs, cols: _pad_stages([np.asarray(a, float).reshape(-1, cols)[:n + 1] for a, n in zip(arrs, Ns)], Nmax)
    lp, npp = pk.dualmultws_batch(Nmax, sc["nOb"], sc["vOb"], sc["A"], sc["b"], pad(sc["rx"], 1)[..., 0], pad(sc["ry"], 1)[..., 0],
                                  pad(sc["ryaw"], 1)[..., 0], sc["ego"])
    sc.update(lWS=[lp[i, :n + 1] for i, n in enumerate(Ns)], nWS=[npp[i, :n + 1] for i, n in enumerate(Ns)], lWS_pad=lp, nWS_pad=npp)
    tens = dict(x0=_t(sc["x0"]), xF=_t(sc["xF"]), Ns=_t(Ns, I32), rx=_t(pad(sc["rx"], 1)[..., 0]), ry=_t(pad(sc["ry"], 1)[..., 0]),
                ryaw=_t(pad(sc["ryaw"], 1)[..., 0]), xWS=_t(pad(sc["xWS"], 4)),
                uWS=_t(_pad_stages([np.asarray(u, float).reshape(-1, 2)[:n] for u, n in zip(sc["uWS"], Ns)], Nmax)[:, :Nmax]))
    return sc, tens


def _park_args(sc):
    return dict(Ts=sc["Ts"], L=sc["L"], ego_=sc["ego"], XYbounds=sc["XYbounds"], nOb=sc["nOb"], vOb=sc["vOb"], A=sc["A"], b=sc["b"],
                fixTime=0)


@pytest.mark.parametrize("sd", [1, 0], ids=["SignedDist", "Dist"])
@pytest.mark.parametrize("ws", [False, True], ids=["dualws-inside", "caller-lWS-nWS"])
def test_parking_mixed_bit_identical_to_the_host_twin(T, mixed_park, sd, ws):
    sc, t = mixed_park
    Ns = sc["Ns"]
    ref = pk.parking_solve_mixed(sc["x0"], sc["xF"], Ns, sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"],
                                 sc["b"], sc["rx"], sc["ry"], sc["ryaw"], 0, sc["xWS"], sc["uWS"], sd,
                                 sc["lWS"] if ws else None, sc["nWS"] if ws else None)
    got = T.parking_solve_mixed(t["x0"], t["xF"], t["Ns"], **{k: v for k, v in _park_args(sc).items() if k != "fixTime"}, rx=t["rx"],
                                ry=t["ry"], ryaw=t["ryaw"], fixTime=0, xWS=t["xWS"], uWS=t["uWS"], signed_dist=sd,
                                lWS=_t(sc["lWS_pad"]) if ws else None, nWS=_t(sc["nWS_pad"]) if ws else None)
    assert ref["exitflag"].sum() > 0.5 * len(Ns)
    for k in ("exitflag", "iters", "kkt_err"):
        assert np.array_equal(_h(got[k]), ref[k]), k
    for k, ext in (("xp", 1), ("up", 0), ("lp", 1), ("np", 1)) + ((("sl", 1),) if sd else ()):
        _same_over_horizons(got[k], ref[k], Ns, ext, k)
    _same_over_horizons(got["ts"][:, None], [r[None] for r in ref["ts"]], Ns, 1, "ts")
    if not sd:
        assert not got["sl"].any()      # the Distance formulation has no slacks
    assert got["time"].device.type == "cpu" and float(got["time"]) > 0
    # ParkingConstraints on those outputs, against the twin on the twin's outputs
    feas, e, strict = T.check_parking_mixed(t["x0"], t["xF"], t["Ns"], **_park_args(sc), x=got["xp"], u=got["up"], l=got["lp"],
                                            n=got["np"], timeScale=got["ts"], sd=sd, sl=got["sl"] if sd else None)
    rf, re_, rs = pk.check_parking_mixed(sc["x0"], sc["xF"], Ns, **_park_args(sc), x=ref["xp"], u=ref["up"], l=ref["lp"], n=ref["np"],
                                         timeScale=ref["ts"], sd=sd, sl=ref["sl"] if sd else None)
    assert np.array_equal(_h(feas), rf) and np.array_equal(_h(e), re_) and np.array_equal(_h(strict), rs)


def test_parking_uniform_and_checker_bit_identical(T):
    sc = scenarios.reverse_parking_batch(256, 80, seed=5)
    a = dict(x0=sc["x0"], xF=sc["xF"], N=80, **_park_args(sc))
    ref = pk.parking_solve_batch(**{k: v for k, v in a.items() if k != "fixTime"}, rx=sc["rx"], ry=sc["ry"], ryaw=sc["ryaw"], fixTime=0,
                                 xWS=sc["xWS"], uWS=sc["uWS"])
    ta = dict(a, x0=_t(sc["x0"]), xF=_t(sc["xF"]))
    got = T.parking_solve_batch(**{k: v for k, v in ta.items() if k != "fixTime"}, rx=_t(sc["rx"]), ry=_t(sc["ry"]), ryaw=_t(sc["ryaw"]),
                                fixTime=0, xWS=_t(sc["xWS"]), uWS=_t(sc["uWS"]))
    for k in ("xp", "up", "ts", "lp", "np", "sl", "exitflag", "iters", "kkt_err"):
        assert np.array_equal(_h(got[k]), ref[k]), k
    got_c = T.check_parking_batch(**ta, x=got["xp"], u=got["up"], l=got["lp"], n=got["np"], timeScale=got["ts"], sd=1, sl=got["sl"])
    ref_c = pk.check_parking_batch(**a, x=ref["xp"], u=ref["up"], l=ref["lp"], n=ref["np"], timeScale=ref["ts"], sd=1, sl=ref["sl"])
    for g, r in zip(got_c, ref_c):
        assert np.array_equal(_h(g), r)


def test_dualmultws_bit_identical(T):
    sc = scenarios.reverse_parking_batch(256, 80, seed=6)
    ref = pk.dualmultws_batch(80, sc["nOb"], sc["vOb"], sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], sc["ego"], want_d=True)
    got = T.dualmultws_batch(80, sc["nOb"], sc["vOb"], sc["A"], sc["b"], _t(sc["rx"]), _t(sc["ry"]), _t(sc["ryaw"]), sc["ego"], want_d=True)
    for g, r in zip(got, ref):
        assert np.array_equal(_h(g), r)


# ---- quadcopter ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("sd", [1, 0], ids=["SignedDist", "Dist"])
def test_quadcopter_mixed_and_checker_bit_identical(T, sd):
    sc = scenarios.quadcopter_mixed_batch(256, (90, 127), seed=4)
    Ns, Nmax = sc["Ns"], int(sc["Ns"].max())
    ref = qc.quadcopter_solve_mixed(sc["x0"], sc["xF"], Ns, sc["Ts"], sc["R"], sc["obs"], sc["xWS"], signed_dist=sd)
    xw = _pad_stages([np.asarray(w, float).T for w in sc["xWS"]], Nmax).transpose(0, 2, 1)
    got = T.quadcopter_solve_mixed(_t(sc["x0"]), _t(sc["xF"]), _t(Ns, I32), _t(sc["Ts"]), sc["R"], sc["obs"], _t(xw), signed_dist=sd)
    assert (ref["exitflag"] >= 1).any()
    for k in ("exitflag", "iters", "kkt_err"):
        assert np.array_equal(_h(got[k]), ref[k]), k
    for k, ext in (("xp", 1), ("up", 0), ("lp", 1), ("slack", 1)):
        _same_over_horizons(got[k], ref[k], Ns, ext, k)
    _same_over_horizons(got["ts"][:, None], [r[None] for r in ref["ts"]], Ns, 1, "ts")
    feas, worst = T.check_quadcopter_mixed(got["xp"], got["up"], got["ts"], _t(sc["x0"]), _t(sc["xF"]), got["N"], got["Ts"], got["lp"],
                                           sc["obs"], sc["R"])
    rf, rw = qc.check_quadcopter_mixed(ref["xp"], ref["up"], ref["ts"], sc["x0"], sc["xF"], Ns, sc["Ts"], ref["lp"], sc["obs"], sc["R"])
    assert np.array_equal(_h(feas), rf) and np.array_equal(_h(worst), rw)


@pytest.mark.parametrize("sd", [1, 0], ids=["SignedDist", "Dist"])
def test_quadcopter_uniform_and_checker_bit_identical(T, sd):
    sc = scenarios.quadcopter_batch(256, 100, seed=7)
    ref = qc.quadcopter_solve_batch(sc["x0"], sc["xF"], 100, sc["Ts"], sc["R"], sc["obs"], sc["xWS"], signed_dist=sd)
    got = T.quadcopter_solve_batch(_t(sc["x0"]), _t(sc["xF"]), 100, sc["Ts"], sc["R"], sc["obs"], _t(sc["xWS"]), signed_dist=sd)
    for k in ("xp", "up", "ts", "lp", "slack", "exitflag", "iters", "kkt_err"):
        assert np.array_equal(_h(got[k]), ref[k]), k
    if sd:
        assert (ref["exitflag"] >= 1).sum() > 0.8 * 256
    feas, worst = T.check_quadcopter_batch(got["xp"], got["up"], got["ts"], _t(sc["x0"]), _t(sc["xF"]), sc["Ts"], got["lp"], sc["obs"],
                                           sc["R"])
    rf, rw = qc.check_quadcopter_batch(ref["xp"], ref["up"], ref["ts"], sc["x0"], sc["xF"], sc["Ts"], ref["lp"], sc["obs"], sc["R"])
    assert np.array_equal(_h(feas), rf) and np.array_equal(_h(worst), rw)


# ---- raw entries: padding, device-resident argument checks ------------------------------------------------------------------------

def _p(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _raw_park(sc, t, Ns_dev, outs, stream=None):
    vOb, V, A, b = pk._shared(sc["nOb"], sc["vOb"], sc["A"], sc["b"])
    ego, xy = np.asarray(sc["ego"], float).ravel(), np.asarray(sc["XYbounds"], float).ravel()
    c = lambda x: x.transpose(1, 2).contiguous() if x.dim() == 3 else x.contiguous()
    B, Nmax = t["rx"].shape[0], t["rx"].shape[1] - 1
    ins = [c(t[k]) for k in ("x0", "xF", "rx", "ry", "ryaw", "xWS", "uWS")]
    torch.cuda.synchronize()
    return _lib.lib().obca_parking_solve_mixed_dev(
        B, _p(Ns_dev), Nmax, sc["nOb"], _lib.ptr(vOb), _lib.ptr(A), _lib.ptr(b), _p(ins[0]), _p(ins[1]), float(sc["Ts"]), float(sc["L"]),
        _lib.ptr(ego), _lib.ptr(xy), *[_p(x) for x in ins[2:]], None, None, 0, 1, None, *[_p(o) for o in outs], None, stream)


def _nan_park_outs(B, Nmax, V, nOb):
    NS = Nmax + 1
    f = lambda *s: torch.full(s, float("nan"), dtype=F64, device=DEV)
    return [f(B, NS, 4), f(B, Nmax, 2), f(B, NS), f(B, NS, V), f(B, NS, 4 * nOb), f(B, NS, nOb),
            torch.full((B,), -7, dtype=I32, device=DEV), torch.full((B,), -7, dtype=I32, device=DEV), f(B)]


def test_raw_mixed_entries_write_nothing_past_a_horizon(T, mixed_park):
    sc, t = mixed_park
    Ns = sc["Ns"]
    V = int(np.sum(sc["vOb"]))
    outs = _nan_park_outs(len(Ns), int(Ns.max()), V, sc["nOb"])
    assert _raw_park(sc, t, t["Ns"], outs) == 0
    for o, ext in zip(outs[:6], (1, 0, 1, 1, 1, 1)):
        h = _h(o)
        for i, n in enumerate(Ns):
            assert not np.isnan(h[i, :n + ext]).any() and np.isnan(h[i, n + ext:]).all()
    q = scenarios.quadcopter_mixed_batch(64, (90, 127), seed=8)
    Nq, Nm = q["Ns"], int(q["Ns"].max())
    xw = _t(_pad_stages([np.asarray(w, float).T for w in q["xWS"]], Nm))          # (B, Nmax+1, 12): the C-ABI's 12 x (Nmax+1)
    f = lambda *s: torch.full(s, float("nan"), dtype=F64, device=DEV)
    qo = [f(64, Nm + 1, 12), f(64, Nm, 4), f(64, Nm + 1), f(64, Nm + 1, 30), f(64, Nm + 1, 5)]
    ef, it, err = torch.zeros(64, dtype=I32, device=DEV), torch.zeros(64, dtype=I32, device=DEV), f(64)
    ob = np.ascontiguousarray(q["obs"], dtype=float).ravel()
    Nd, Td, x0, xF = _t(Nq, I32), _t(q["Ts"]), _t(q["x0"]), _t(q["xF"])
    torch.cuda.synchronize()
    assert _lib.lib().obca_quadcopter_solve_mixed_dev(64, _p(Nd), Nm, _p(x0), _p(xF), _p(Td), float(q["R"]), _lib.ptr(ob), _p(xw), 1.0, 1, None,
                                                      *[_p(o) for o in qo], _p(ef), _p(it), _p(err), None, None) == 0
    for o, ext in zip(qo, (1, 0, 1, 1, 1)):
        h = _h(o)
        for i, n in enumerate(Nq):
            assert not np.isnan(h[i, :n + ext]).any() and np.isnan(h[i, n + ext:]).all()


def test_bad_device_resident_horizon_or_sampling_time_refused_before_any_write(T, mixed_park):
    sc, t = mixed_park
    Ns = sc["Ns"].copy()
    V = int(np.sum(sc["vOb"]))
    lib = _lib.lib()
    for i, bad in ((37, 1), (300, int(Ns.max()) + 1), (5, -3)):
        Nb = Ns.copy(); Nb[i] = bad; Nb[400] = 0          # the first bad index is named
        outs = _nan_park_outs(len(Ns), int(Ns.max()), V, sc["nOb"])
        assert _raw_park(sc, t, _t(Nb, I32), outs) == -1
        assert lib.obca_last_error().decode() == f"Nb[{i}] = {bad} outside [2, Nmax = {int(Ns.max())}]"
        assert all(torch.isnan(o).all() for o in outs[:6] + outs[8:]) and all((o == -7).all() for o in outs[6:8])
        with pytest.raises(_lib.ObcaError, match=rf"Nb\[{i}\] = {bad} outside"):
            T.parking_solve_mixed(t["x0"], t["xF"], _t(Nb, I32), **{k: v for k, v in _park_args(sc).items() if k != "fixTime"}, rx=t["rx"],
                                  ry=t["ry"], ryaw=t["ryaw"], fixTime=0, xWS=t["xWS"], uWS=t["uWS"])
    q = scenarios.quadcopter_mixed_batch(64, (90, 127), seed=8)
    Nm = int(q["Ns"].max())
    xw = _t(_pad_stages([np.asarray(w, float).T for w in q["xWS"]], Nm).transpose(0, 2, 1))
    for Nq, Ts, msg in ((q["Ns"], np.where(np.arange(64) == 9, np.nan, q["Ts"]), "Tsb[9] = nan is not a finite sampling time > 0"),
                        (q["Ns"], np.where(np.arange(64) == 20, 0.0, q["Ts"]), "Tsb[20] = 0.000000 is not a finite sampling time > 0"),
                        (np.where(np.arange(64) == 50, 1, q["Ns"]), np.where(np.arange(64) == 3, -1.0, q["Ts"]),
                         "Nb[50] = 1 outside [2, Nmax = %d]" % Nm)):      # a bad horizon ranks before any bad sampling time
        with pytest.raises(_lib.ObcaError) as e_host:
            qc.quadcopter_solve_mixed(q["x0"], q["xF"], Nq, Ts, q["R"], q["obs"], q["xWS"])
        with pytest.raises(_lib.ObcaError) as e_dev:
            T.quadcopter_solve_mixed(_t(q["x0"]), _t(q["xF"]), _t(Nq, I32), _t(Ts), q["R"], q["obs"], xw)
        assert msg in str(e_dev.value) and str(e_dev.value) == str(e_host.value)
        z = torch.zeros(64, Nm + 1, dtype=F64, device=DEV)
        with pytest.raises(_lib.ObcaError, match=msg.replace("[", r"\[").replace("]", r"\]")):
            T.check_quadcopter_mixed(xw, xw[:, :4, :Nm], z, _t(q["x0"]), _t(q["xF"]), _t(Nq, I32), _t(Ts),
                                     torch.zeros(64, 30, Nm + 1, dtype=F64, device=DEV), q["obs"], q["R"])


# ---- stream order, torch.compile, reports -------------------------------------------------------------------------------------------

def test_inputs_produced_on_a_side_stream_are_waited_for(T):
    q = scenarios.quadcopter_mixed_batch(128, (90, 127), seed=9)
    Nm = int(q["Ns"].max())
    xw = _pad_stages([np.asarray(w, float).T for w in q["xWS"]], Nm).transpose(0, 2, 1)
    src = {k: torch.as_tensor(np.ascontiguousarray(v)).pin_memory() for k, v in dict(x0=q["x0"], xF=q["xF"], Ts=q["Ts"], xWS=xw).items()}
    ref = T.quadcopter_solve_mixed(_t(q["x0"]), _t(q["xF"]), _t(q["Ns"], I32), _t(q["Ts"]), q["R"], q["obs"], _t(xw))
    dst = {k: torch.full(v.shape, float("nan"), dtype=F64, device=DEV) for k, v in src.items()}
    Nd = torch.zeros(128, dtype=I32, device=DEV)
    Nh = torch.as_tensor(q["Ns"], dtype=I32).pin_memory()
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(1_000_000_000)      # about half a second of device work queued before the inputs land
        for k in dst:
            dst[k].copy_(src[k], non_blocking=True)
        Nd.copy_(Nh, non_blocking=True)
        got = T.quadcopter_solve_mixed(dst["x0"], dst["xF"], Nd, dst["Ts"], q["R"], q["obs"], dst["xWS"])
        feas, worst = T.check_quadcopter_mixed(got["xp"], got["up"], got["ts"], dst["x0"], dst["xF"], Nd, dst["Ts"], got["lp"], q["obs"],
                                               q["R"])
    for k in ("xp", "up", "ts", "lp", "slack", "exitflag", "iters", "kkt_err"):
        assert torch.equal(got[k], ref[k]), k
    rf, rw = T.check_quadcopter_mixed(ref["xp"], ref["up"], ref["ts"], _t(q["x0"]), _t(q["xF"]), _t(q["Ns"], I32), _t(q["Ts"]), ref["lp"],
                                      q["obs"], q["R"])
    assert torch.equal(feas, rf) and torch.equal(worst, rw)


def test_torch_compile_traces_an_op(T):
    sc = scenarios.reverse_parking_batch(64, 80, seed=10)
    vOb, _, A, b = pk._shared(sc["nOb"], sc["vOb"], sc["A"], sc["b"])
    args = (vOb.tolist(), A.ravel(order="F").tolist(), b.tolist(), np.asarray(sc["ego"], float).ravel().tolist())

    def fn(rx, ry, ryaw):
        lp, npp, d = torch.ops.obca.dualmultws(*args, rx, ry, ryaw, [], [])
        return lp * 1.0, npp, d
    rx, ry, ryaw = _t(sc["rx"]), _t(sc["ry"]), _t(sc["ryaw"])
    eager = fn(rx, ry, ryaw)
    compiled = torch.compile(fn, fullgraph=True, backend="aot_eager")(rx, ry, ryaw)
    for g, r in zip(compiled, eager):
        assert torch.equal(g, r)


def test_last_reports_match_the_twin(T):
    lib = _lib.lib()

    def reports():
        dws, slv = C.c_double(), C.c_double()
        prof = (C.c_ulonglong * 8)()
        rounds, handed = C.c_int(), C.c_int()
        assert lib.obca_last_times(0, C.byref(dws), C.byref(slv)) == 0 and lib.obca_last_profile(0, prof) == 0
        assert lib.obca_last_schedule(0, C.byref(rounds), C.byref(handed), None) == 0
        return dws.value, slv.value, list(prof), rounds.value, handed.value

    sc = scenarios.reverse_parking_batch(64, 80, seed=11)      # small enough for the persistent kernel alone: a deterministic schedule
    a = dict(x0=sc["x0"], xF=sc["xF"], N=80, **{k: v for k, v in _park_args(sc).items() if k != "fixTime"})
    ref = pk.parking_solve_batch(**a, rx=sc["rx"], ry=sc["ry"], ryaw=sc["ryaw"], fixTime=0, xWS=sc["xWS"], uWS=sc["uWS"])
    r_twin = reports()
    got = T.parking_solve_batch(**dict(a, x0=_t(sc["x0"]), xF=_t(sc["xF"])), rx=_t(sc["rx"]), ry=_t(sc["ry"]), ryaw=_t(sc["ryaw"]),
                                fixTime=0, xWS=_t(sc["xWS"]), uWS=_t(sc["uWS"]))
    r_tens = reports()
    assert r_tens[2:] == r_twin[2:] and r_tens[4] == 64
    assert r_twin[1] == ref["time"] and r_tens[1] == float(got["time"])      # each reports its own call
    assert r_twin[0] > 0 and r_tens[0] > 0                                     # DualMultWS ran inside both
    q = scenarios.quadcopter_batch(64, 100, seed=12)
    qc.quadcopter_solve_batch(q["x0"], q["xF"], 100, q["Ts"], q["R"], q["obs"], q["xWS"])
    p_twin = reports()[2]
    T.quadcopter_solve_batch(_t(q["x0"]), _t(q["xF"]), 100, q["Ts"], q["R"], q["obs"], _t(q["xWS"]))
    p_tens = reports()[2]
    assert p_tens[6:] == p_twin[6:] and p_twin[7] > 0      # merit and K1 evaluation counts (the others are cycle counters)
