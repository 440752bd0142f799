"""obca_quadcopter_plan_solve without a GPU: the exported symbol and its Python binding's call refused by the library, the argument
refusals that come before any device work (nothing written), and the warm-start arithmetic and index maps of
obca_b200/csrc/obca_qflow.h -- the sampling time, gather and scatter the entry's kernels run -- built for the host and checked against
native.quadcopter_warm_start and numpy repacking of random planner-layout buffers with mixed horizons."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import obca_b200                                    # noqa: E402
from obca_b200 import _lib, scenarios               # noqa: E402
from obca_b200.planner import device, native        # noqa: E402

ENTRY = "obca_quadcopter_plan_solve"


# argument positions of the prototype
X0, XF, OX, OY, OZ, NOB, LO, HI, RESO, MAXN, TS = range(1, 12)
OB, NCAP = 13, 17
OUTS = ["xp", "up", "ts", "lp", "slack", "N", "Tsb", "status", "expansions", "exitflag", "iters", "kkt_err", "feasible", "worst",
        "plan_seconds", "solve_seconds"]


def _call(B=3, Ncap=40, Ts=0.25, reso=1.0, max_nodes=0, x0=None, drop=None):
    """The entry called through ctypes with every output filled with 7; drop: the index of an argument passed as NULL."""
    sc = scenarios.quadcopter_batch(max(B, 1), seed=2)
    Bo = max(B, 1); NS = Ncap + 1
    x0 = np.ascontiguousarray(sc["x0"] if x0 is None else x0, dtype=np.float64)
    xF = np.ascontiguousarray(sc["xF"], dtype=np.float64)
    ob = np.ascontiguousarray(np.asarray(sc["obs"], float).reshape(5, 6))
    ox, oy, oz = np.array([50.0]), np.array([50.0]), np.array([20.0])
    lo, hi = np.zeros(3), np.array([105.0, 105.0, 55.0])
    outs = [np.full((Bo, NS, 12), 7.0), np.full((Bo, Ncap, 4), 7.0), np.full((Bo, NS), 7.0), np.full((Bo, NS, 30), 7.0),
            np.full((Bo, NS, 5), 7.0), np.full(Bo, 7, np.int32), np.full(Bo, 7.0)] + [np.full(Bo, 7, np.int32) for _ in range(4)] + \
        [np.full(Bo, 7.0), np.full(Bo, 7, np.int32), np.full(Bo, 7.0), np.full(1, 7.0), np.full(1, 7.0)]
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    args = [C.c_int(B), p(x0), p(xF), p(ox), p(oy), p(oz), C.c_int(1), p(lo), p(hi), C.c_double(reso), C.c_int(max_nodes),
            C.c_double(Ts), C.c_double(sc["R"]), p(ob), C.c_double(1.0), C.c_int(1), C.byref(_lib.default_opts()), C.c_int(Ncap)] + \
        [p(a) for a in outs]
    if drop is not None:
        args[drop] = None
    lib = obca_b200.lib()
    return getattr(lib, ENTRY)(*args), lib.obca_last_error().decode(), outs


def _untouched(outs):
    return all((a == 7).all() for a in outs)


def test_symbol_and_ctypes_signature_match_the_header():
    lib = obca_b200.lib()
    assert ENTRY in _lib.SYMBOLS
    assert len(getattr(lib, ENTRY).argtypes) == NCAP + 1 + len(OUTS)
    sc = scenarios.quadcopter_batch(2, seed=2)
    with pytest.raises(_lib.ObcaError, match="511"):      # accepted by the binding's types, refused before any device work
        device.plan_solve_quadcopter(sc["x0"], sc["xF"], sc["R"], sc["obs"], sc["Ts80"], Ncap=512)


@pytest.mark.parametrize("drop,name", [(X0, "x0"), (XF, "xF"), (OX, "ox"), (LO, "lo"), (HI, "hi"), (OB, "ob")] +
                         [(NCAP + 1 + i, k) for i, k in enumerate(OUTS) if k in ("xp", "up", "ts", "lp", "N", "Tsb", "status", "exitflag",
                                                                                  "iters", "kkt_err", "feasible")])
def test_null_required_argument_is_refused(drop, name):
    rc, msg, outs = _call(drop=drop)
    assert rc == -1 and msg == "null argument", (name, rc, msg)
    assert _untouched(outs), name


@pytest.mark.parametrize("kw,code,text", [
    (dict(B=-1), -1, "B < 0"),
    (dict(Ncap=1), -1, "Ncap < 2"),
    (dict(Ncap=512), -4, "N = 512 > 511"),
    (dict(Ts=0.0), -1, "Ts must be a finite number > 0"),
    (dict(Ts=float("nan")), -1, "Ts must be a finite number > 0"),
    (dict(Ts=0.02, Ncap=511), -1, "sampling time 0"),          # 0.02 * 80 / 511 * 100 = 0.31 rounds to 0
    (dict(reso=0.0), -1, "reso must be a finite number > 0"),
    (dict(reso=-1.0), -1, "reso must be a finite number > 0"),
    (dict(max_nodes=(1 << 28) + 1), -1, "max_nodes > 2^28"),
])
def test_bad_argument_is_refused_before_any_device_work(kw, code, text):
    rc, msg, outs = _call(**kw)
    assert rc == code and text in msg, (kw, rc, msg)
    assert _untouched(outs), kw


def test_non_finite_start_is_refused():
    sc = scenarios.quadcopter_batch(3, seed=2)
    x0 = sc["x0"].copy(); x0[1, 2] = np.inf
    rc, msg, outs = _call(x0=x0)
    assert rc == -1 and msg == "start / goal coordinates must be finite", msg
    assert _untouched(outs)


def test_valid_call_without_a_device_stops_at_no_device():
    if obca_b200.lib().obca_device_count() > 0:
        pytest.skip("CUDA device present")
    for kw in (dict(), dict(Ts=0.02, Ncap=300), dict(B=0)):      # 0.02 * 80 / 300 * 100 = 0.53 rounds to 1: accepted
        rc, msg, outs = _call(**kw)
        assert rc == -2 and "no CUDA device" in msg, (kw, rc, msg)
        assert _untouched(outs)


# ---- the warm start and index maps of obca_qflow.h, on the host -----------------------------------------------------------------------
HOST_SRC = r'''
#include "obca_qflow.h"
using namespace obca_qflow;
extern "C" double qflow_ts(double Ts, int n) { return warm_start_ts(Ts, n); }
extern "C" void qflow_gather(int Bs, int M, int cap, const int* list, const int* Nb, double Ts, const double* const* in, double* const* out) {
  Gather g{in[0], in[1], in[2], in[3], in[4], Ts, out[0], out[1], out[2], out[3]};
  for (int q = 0; q < Bs; ++q)
    for (int k = 0; k <= M; ++k) gather_stage(g, q, list[q], Nb[q], k, M, cap);
}
extern "C" void qflow_scatter(int Bs, int M, int Ncap, const int* list, const int* Nb, double* const* sd, int* const* si,
                              double* const* dd, int* const* di) {
  Outs s{sd[0], sd[1], sd[2], sd[3], sd[4], sd[5], sd[6], sd[7], si[0], si[1], si[2]};
  Outs d{dd[0], dd[1], dd[2], dd[3], dd[4], dd[5], dd[6], dd[7], di[0], di[1], di[2]};
  for (int q = 0; q < Bs; ++q)
    for (int k = 0; k <= M; ++k) scatter_stage(s, d, q, list[q], Nb[q], k, M, Ncap);
}
'''


@pytest.fixture(scope="module")
def qflow(tmp_path_factory):
    d = tmp_path_factory.mktemp("qflow")
    src = d / "qflow_host.cpp"; so = d / "libqflow_host.so"
    src.write_text(HOST_SRC)
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "obca_b200", "csrc"), "-o", str(so), str(src)])
    lib = C.CDLL(str(so))
    lib.qflow_ts.restype = C.c_double
    lib.qflow_ts.argtypes = [C.c_double, C.c_int]
    return lib


def _ptrs(arrs, ty):
    return (ty * len(arrs))(*[a.ctypes.data_as(ty) for a in arrs])


@pytest.mark.parametrize("Ts", [0.25, 0.2, 0.6, 1 / 3])
def test_sampling_time_equals_the_host_warm_start_bit_for_bit(qflow, Ts):
    for n in range(2, 512):
        want = native.quadcopter_warm_start(np.zeros(n + 1), np.zeros(n + 1), np.zeros(n + 1), Ts)["Ts"]
        got = qflow.qflow_ts(Ts, n)
        assert np.float64(got).tobytes() == np.float64(want).tobytes(), (Ts, n, got, want)


def _gather(qflow, rng, B, Ncap, M_want=None):
    """Random planner outputs (stride Ncap + 1) with mixed horizons; the listed pairs gathered by the host build of gather_stage and by
    what the composed path does: native.quadcopter_warm_start on each path, padded as quadcopter_solve_mixed pads them."""
    from obca_b200.parking import _pad_stages
    cap = Ncap + 1
    N = rng.integers(2, Ncap + 1, B).astype(np.int32)
    if M_want is not None:
        N[:] = np.minimum(N, M_want); N[0] = M_want
    rx, ry, rz = (np.full((B, cap), np.nan) for _ in range(3))
    for p in range(B):
        n = int(N[p])
        rx[p, :n + 1], ry[p, :n + 1], rz[p, :n + 1] = rng.integers(0, 106, (3, n + 1)).astype(float)      # cell * reso
    lst = np.sort(rng.choice(B, max(1, B // 2), replace=False)).astype(np.int32)
    Nb = N[lst]; Bs = len(lst); M = int(Nb.max())
    x0 = rng.standard_normal((B, 12)); xF = rng.standard_normal((B, 12))
    Ts = 0.25
    ws = [native.quadcopter_warm_start(rx[i, :n + 1].copy(), ry[i, :n + 1].copy(), rz[i, :n + 1].copy(), Ts) for i, n in zip(lst, Nb)]
    e_xWS = _pad_stages([w["xWS"].reshape(12, -1)[:, :n + 1].T for w, n in zip(ws, Nb)], M)       # (Bs, M+1, 12)
    out = [np.full((Bs, M + 1, 12), -1.0), np.full((Bs, 12), -1.0), np.full((Bs, 12), -1.0), np.full(Bs, -1.0)]
    inp = [np.ascontiguousarray(a) for a in (rx, ry, rz, x0, xF)]
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    qflow.qflow_gather(Bs, M, cap, p(lst), p(Nb), C.c_double(Ts), _ptrs(inp, C.POINTER(C.c_double)), _ptrs(out, C.POINTER(C.c_double)))
    for got, exp in zip(out, (e_xWS, x0[lst], xF[lst], np.array([w["Ts"] for w in ws]))):
        assert np.array_equal(got, exp)
    return M


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_gather_matches_the_host_warm_start_and_numpy_padding(qflow, seed):
    rng = np.random.default_rng(seed)
    _gather(qflow, rng, int(rng.integers(20, 60)), 150)


@pytest.mark.parametrize("M", [2, 5])
def test_gather_with_fewer_than_twelve_stages(qflow, M):
    """M = 2 and M = 5: fewer stages than x0 / xF have components, which still come over whole."""
    assert _gather(qflow, np.random.default_rng(20 + M), 17, 40, M_want=M) == M


@pytest.mark.parametrize("seed,optional", [(0, True), (1, True), (2, False)])
def test_scatter_matches_numpy_unpadding(qflow, seed, optional):
    """optional False: slack and worst not asked for (null), so nothing is written there."""
    rng = np.random.default_rng(seed)
    B, Ncap = 60, 45
    Bs = 23
    lst = np.sort(rng.choice(B, Bs, replace=False)).astype(np.int32)
    Nb = rng.integers(2, Ncap + 1, Bs).astype(np.int32)
    Nb[0] = 2
    M = int(Nb.max())
    rows = (12, 4, 1, 30, 5); ext = (1, 0, 1, 1, 1)
    src = [rng.standard_normal((Bs, M + e, r)) for r, e in zip(rows, ext)] + [rng.standard_normal(Bs) for _ in range(3)]
    srci = [rng.integers(0, 100, Bs).astype(np.int32) for _ in range(3)]
    dst = [np.full((B, Ncap + e, r), np.nan) for r, e in zip(rows, ext)] + [np.full(B, np.nan) for _ in range(3)]
    dsti = [np.full(B, -7, np.int32) for _ in range(3)]
    exp = [a.copy() for a in dst]; expi = [a.copy() for a in dsti]
    skip = set() if optional else {4, 7}                  # slack, worst
    for q, (pair, n) in enumerate(zip(lst, Nb)):
        for j, (a, s, e) in enumerate(zip(exp, src, ext + (None,) * 3)):
            if j in skip:
                continue
            if e is None:
                a[pair] = s[q]
            else:
                a[pair, :n + e] = s[q, :n + e]
        for a, s in zip(expi, srci):
            a[pair] = s[q]
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    D = C.POINTER(C.c_double); I = C.POINTER(C.c_int)
    dptr = _ptrs(dst, D)
    for j in skip:
        dptr[j] = D()
    qflow.qflow_scatter(Bs, M, Ncap, p(lst), p(Nb), _ptrs(src, D), _ptrs(srci, I), dptr, _ptrs(dsti, I))
    for got, e in zip(dst + dsti, exp + expi):
        assert np.array_equal(got, e, equal_nan=True)
