"""obca_parking_plan_solve_goals without a GPU: the exported symbol and its Python binding's call refused by the library, the argument
refusals that come before any device work (nothing written), and the index maps of obca_b200/csrc/obca_flow.h -- the
listing, gather and scatter the entry's kernels run -- built for the host and checked against numpy repacking of random planner-layout
buffers with mixed horizons."""
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

ENTRY = "obca_parking_plan_solve_goals"


def _scene(B=3, Ncap=40):
    sc = scenarios.reverse_parking_scenario()
    ox, oy = native.obstacle_points("backwards")
    x0 = np.column_stack([np.linspace(-5, 5, B), np.full(B, 8.0), np.zeros(B), np.zeros(B)])
    return sc, ox, oy, x0


def _call(B=3, Ncap=40, vOb=None, drop=None):
    """The entry called through ctypes with outputs filled with 7; drop: the index of an argument passed as NULL."""
    sc, ox, oy, x0 = _scene(max(B, 1), Ncap)
    V = int(sc["vOb"].sum()); nOb = sc["nOb"]; NS = Ncap + 1; Bo = max(B, 1)
    vOb = np.ascontiguousarray(sc["vOb"] if vOb is None else vOb, dtype=np.int32)
    A = np.asfortranarray(sc["A"], dtype=np.float64); b = np.ascontiguousarray(sc["b"], dtype=np.float64).ravel()
    xF = np.ascontiguousarray(np.tile(sc["xF"], (Bo, 1)))
    outs = [np.full((Bo, NS, 4), 7.0), np.full((Bo, Ncap, 2), 7.0), np.full((Bo, NS), 7.0), np.full((Bo, NS, V), 7.0),
            np.full((Bo, NS, 4 * nOb), 7.0), np.full((Bo, NS, nOb), 7.0)] + [np.full(Bo, 7, np.int32) for _ in range(5)] + \
        [np.full(Bo, 7.0), np.full(Bo, 7, np.int32), np.full(Bo, 7, np.int32), np.full(1, 7.0), np.full(1, 7.0)]
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    args = [C.c_int(B), p(x0), p(xF), p(ox), p(oy), C.c_int(ox.size), C.c_double(0.6), C.c_double(2.7), C.c_int(3), C.c_int(0),
            C.c_int(0), C.c_int(nOb), p(vOb), p(A), p(b), p(sc["ego"]), p(sc["XYbounds"]), C.c_int(0), C.c_int(1),
            C.byref(_lib.default_opts()), C.c_int(Ncap)] + [p(a) for a in outs]
    if drop is not None:
        args[drop] = None
    lib = obca_b200.lib()
    return getattr(lib, ENTRY)(*args), lib.obca_last_error().decode(), outs


def test_symbol_and_ctypes_signature_match_the_header():
    assert ENTRY in _lib.SYMBOLS
    sc, ox, oy, x0 = _scene()
    with pytest.raises(_lib.ObcaError, match="319"):      # accepted by the binding's types, refused before any device work
        device.plan_solve_goals_raw(x0, sc["xF"], ox, oy, 0.6, sc["nOb"], sc["vOb"], sc["A"], sc["b"], sc["ego"], sc["XYbounds"], Ncap=320)


@pytest.mark.parametrize("drop,name", [(1, "x0"), (2, "xF"), (3, "ox"), (12, "vOb"), (15, "ego"), (21, "xp"), (27, "N"),
                                       (28, "status"), (30, "exitflag"), (33, "feasible")])
def test_null_required_argument_is_refused(drop, name):
    rc, msg, outs = _call(drop=drop)
    assert rc == -1 and msg == "null argument", (name, rc, msg)
    for a in outs:
        assert (a == 7).all(), name


def test_negative_batch_is_refused():
    rc, msg, outs = _call(B=-1)
    assert rc == -1 and msg == "B < 0"
    for a in outs:
        assert (a == 7).all()


def test_ncap_past_the_solver_bound_is_unsupported():
    rc, msg, outs = _call(Ncap=320)
    assert rc == -4 and "319" in msg and "320" in msg, (rc, msg)
    for a in outs:
        assert (a == 7).all()
    rc, msg, _ = _call(Ncap=1)
    assert rc == -1 and msg == "Ncap < 2", (rc, msg)


def test_bad_vob_gets_the_solvers_shape_message():
    lib = obca_b200.lib()
    bad = np.array([5, 4, 4, 4], np.int32)
    rc, msg, outs = _call(vOb=bad)
    assert rc == -1 and "half-spaces per obstacle" in msg, msg
    for a in outs:
        assert (a == 7).all()
    # the same message as obca_parking_solve_mixed gives for that vOb
    sc = scenarios.reverse_parking_scenario()
    with pytest.raises(_lib.ObcaError) as e:
        from obca_b200 import parking
        parking.parking_solve_mixed(np.zeros((1, 4)), sc["xF"], [4], 0.6, 2.7, sc["ego"], sc["XYbounds"], 4, bad, np.zeros((17, 2)),
                                    np.zeros(17), [np.zeros(5)], [np.zeros(5)], [np.zeros(5)], 0, [np.zeros((5, 4))], [np.zeros((4, 2))])
    assert msg in str(e.value)
    assert lib.obca_last_error().decode() == msg


def test_valid_call_without_a_device_stops_at_no_device():
    if obca_b200.lib().obca_device_count() > 0:
        pytest.skip("CUDA device present")
    rc, msg, outs = _call()
    assert rc == -2 and "no CUDA device" in msg
    for a in outs:
        assert (a == 7).all()


# ---- the index maps of obca_flow.h, on the host --------------------------------------------------------------------------------------
HOST_SRC = r'''
#include "obca_flow.h"
using namespace obca_flow;
extern "C" int flow_list(int B, int Ncap, int* status, const int* N, int* list, int* Nb, int* nmax) {
  int q = 0; *nmax = 0;
  for (int p = 0; p < B; ++p) {
    if (listed(status[p], N[p], Ncap)) { list[q] = p; Nb[q++] = N[p]; if (N[p] > *nmax) *nmax = N[p]; }
    else if (status[p] == 0) status[p] = 2;
  }
  return q;
}
extern "C" void flow_gather(int Bs, int M, int cap, const int* list, const int* Nb, const double* const* in, double* const* out) {
  Gather g{in[0], in[1], in[2], in[3], in[4], in[5], in[6], out[0], out[1], out[2], out[3], out[4], out[5], out[6]};
  for (int q = 0; q < Bs; ++q)
    for (int k = 0; k <= M; ++k) gather_stage(g, q, list[q], Nb[q], k, M, cap);
}
extern "C" void flow_scatter(int Bs, int M, int Ncap, int V, int nOb, const int* list, const int* Nb, double* const* sd, int* const* si,
                             double* const* dd, int* const* di) {
  Outs s{sd[0], sd[1], sd[2], sd[3], sd[4], sd[5], sd[6], si[0], si[1], si[2], si[3]};
  Outs d{dd[0], dd[1], dd[2], dd[3], dd[4], dd[5], dd[6], di[0], di[1], di[2], di[3]};
  for (int q = 0; q < Bs; ++q)
    for (int k = 0; k <= M; ++k) scatter_stage(s, d, V, nOb, q, list[q], Nb[q], k, M, Ncap);
}
'''


@pytest.fixture(scope="module")
def flow(tmp_path_factory):
    d = tmp_path_factory.mktemp("flow")
    src = d / "flow_host.cpp"; so = d / "libflow_host.so"
    src.write_text(HOST_SRC)
    subprocess.check_call([os.environ.get("CXX", "g++"), "-O1", "-std=c++17", "-shared", "-fPIC", "-I",
                           os.path.join(ROOT, "obca_b200", "csrc"), "-o", str(so), str(src)])
    return C.CDLL(str(so))


def _ptrs(arrs, ty):
    return (ty * len(arrs))(*[a.ctypes.data_as(ty) for a in arrs])


def _planner_batch(rng, B, cap):
    """Random planner outputs (stride cap) with mixed statuses and horizons; entries past a pose's horizon hold NaN."""
    status = rng.choice([0, 0, 0, 0, 1, 2, 4], B).astype(np.int32)
    N = rng.integers(0, cap + 8, B).astype(np.int32)
    N[rng.random(B) < 0.1] = 1                      # a plan too short for the solver
    rx, ry, ryaw = (np.full((B, cap), np.nan) for _ in range(3))
    xWS = np.full((B, 4 * cap), np.nan); uWS = np.full((B, 2 * cap), np.nan)
    for p in range(B):
        n = int(N[p])
        if status[p] == 0 and n + 1 <= cap:
            rx[p, :n + 1], ry[p, :n + 1], ryaw[p, :n + 1] = rng.standard_normal((3, n + 1))
            xWS[p, :4 * (n + 1)] = rng.standard_normal(4 * (n + 1)); uWS[p, :2 * n] = rng.standard_normal(2 * n)
    return status, N, rx, ry, ryaw, xWS, uWS


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_list_and_gather_match_numpy_repacking(flow, seed):
    rng = np.random.default_rng(seed)
    _list_and_gather(flow, rng, int(rng.integers(20, 60)))


@pytest.mark.parametrize("Ncap", [2, 3])
def test_list_and_gather_with_fewer_than_four_stages(flow, Ncap):
    """M = 2 (Ncap = 2, or a batch whose longest plan is N = 2) and M = 3: x0 and xF still come over whole."""
    assert _list_and_gather(flow, np.random.default_rng(10 + Ncap), Ncap) == Ncap


def _list_and_gather(flow, rng, Ncap):
    B = 97
    cap = Ncap + 1
    status, N, rx, ry, ryaw, xWS, uWS = _planner_batch(rng, B, cap)
    N[status == 2] = Ncap + 1 + rng.integers(0, 5, int((status == 2).sum()))      # the planner's own CAPACITY: past the stride
    x0 = rng.standard_normal((B, 4)); xF = rng.standard_normal((B, 4))
    want = [p for p in range(B) if status[p] == 0 and 2 <= N[p] <= Ncap]
    st = status.copy(); lst = np.zeros(B, np.int32); Nb = np.zeros(B, np.int32); nmax = C.c_int(0)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    Bs = flow.flow_list(B, Ncap, p(st), p(N), p(lst), p(Nb), C.byref(nmax))
    assert Bs == len(want) and lst[:Bs].tolist() == want and Nb[:Bs].tolist() == N[want].tolist()
    M = nmax.value
    assert M == int(N[want].max())
    bad = (status == 0) & ((N < 2) | (N > Ncap))
    assert (st[bad] == 2).all() and (st[~bad] == status[~bad]).all()
    # numpy: what examples/sweep_parking_lot.py cuts from the planner's arrays, padded with parking._pad_stages
    from obca_b200.parking import _pad_stages
    Ns = N[want]
    e_rx = _pad_stages([rx[i, :n + 1] for i, n in zip(want, Ns)], M)
    e_ry = _pad_stages([ry[i, :n + 1] for i, n in zip(want, Ns)], M)
    e_ryaw = _pad_stages([ryaw[i, :n + 1] for i, n in zip(want, Ns)], M)
    e_xW = np.transpose(_pad_stages([xWS[i, :4 * (n + 1)].reshape(4, n + 1).T for i, n in zip(want, Ns)], M), (0, 2, 1))
    e_uW = np.transpose(_pad_stages([uWS[i, :2 * n].reshape(2, n).T for i, n in zip(want, Ns)], M)[:, :M], (0, 2, 1))
    out = [np.full((Bs, M + 1), -1.0) for _ in range(3)] + [np.full((Bs, 4, M + 1), -1.0), np.full((Bs, 2, M), -1.0),
                                                           np.full((Bs, 4), -1.0), np.full((Bs, 4), -1.0)]
    inp = [np.ascontiguousarray(a) for a in (rx, ry, ryaw, xWS, uWS, x0, xF)]
    flow.flow_gather(Bs, M, cap, p(lst), p(Nb), _ptrs(inp, C.POINTER(C.c_double)), _ptrs(out, C.POINTER(C.c_double)))
    for got, exp in zip(out, (e_rx, e_ry, e_ryaw, e_xW, e_uW, x0[want], xF[want])):
        assert np.array_equal(got, exp)
    return M


@pytest.mark.parametrize("seed", [0, 1])
def test_scatter_matches_numpy_unpadding(flow, seed):
    rng = np.random.default_rng(seed)
    B, Ncap, V, nOb = 60, 45, 7, 3
    Bs = 23
    lst = np.sort(rng.choice(B, Bs, replace=False)).astype(np.int32)
    Nb = rng.integers(2, Ncap + 1, Bs).astype(np.int32)
    M = int(Nb.max())
    rows = (4, 2, 1, V, 4 * nOb, nOb); ext = (1, 0, 1, 1, 1, 1)
    src = [rng.standard_normal((Bs, M + e, r)) for r, e in zip(rows, ext)] + [rng.standard_normal(Bs)]
    srci = [rng.integers(0, 100, Bs).astype(np.int32) for _ in range(4)]
    dst = [np.full((B, Ncap + e, r), np.nan) for r, e in zip(rows, ext)] + [np.full(B, np.nan)]
    dsti = [np.full(B, -7, np.int32) for _ in range(4)]
    exp = [a.copy() for a in dst]; expi = [a.copy() for a in dsti]
    for q, (pose, n) in enumerate(zip(lst, Nb)):
        for a, s, e in zip(exp, src, ext + (None,)):
            if e is None:
                a[pose] = s[q]
            else:
                a[pose, :n + e] = s[q, :n + e]
        for a, s in zip(expi, srci):
            a[pose] = s[q]
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    D = C.POINTER(C.c_double); I = C.POINTER(C.c_int)
    flow.flow_scatter(Bs, M, Ncap, V, nOb, p(lst), p(Nb), _ptrs(src, D), _ptrs(srci, I), _ptrs(dst, D), _ptrs(dsti, I))
    for got, e in zip(dst + dsti, exp + expi):
        assert np.array_equal(got, e, equal_nan=True)
