"""obca_parking_plan_solve_both and obca_quadcopter_plan_solve_both without a GPU: the exported symbols and their Python bindings' calls
refused by the library, the layout of the two output-set structs against their ctypes Structures (compiled from the
header), and the argument refusals that come before any device work -- those of the one-formulation entries plus a null set or a null
required field of either set, named in the message -- with nothing written to either set or to the shared outputs."""
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

PARK, QUAD = "obca_parking_plan_solve_both", "obca_quadcopter_plan_solve_both"
PK_REQUIRED = ("xp", "up", "ts", "lp", "np", "exitflag", "iters", "kkt_err", "feasible")
QC_REQUIRED = ("xp", "up", "ts", "lp", "exitflag", "iters", "kkt_err", "feasible")


def _untouched(arrs):
    return all((a == 7).all() for a in arrs)


# ---- parking --------------------------------------------------------------------------------------------------------------------------
# argument positions of the prototype
PK_X0, PK_XF, PK_OX, PK_VOB, PK_EGO, PK_NCAP, PK_N, PK_STATUS, PK_DIST, PK_SD = 1, 2, 3, 12, 15, 19, 20, 21, 24, 25


def _park_set(B, Ncap, V, nOb):
    NS = Ncap + 1
    d = dict(xp=np.full((B, NS, 4), 7.0), up=np.full((B, Ncap, 2), 7.0), ts=np.full((B, NS), 7.0), lp=np.full((B, NS, V), 7.0),
             np=np.full((B, NS, 4 * nOb), 7.0), sl=np.full((B, NS, nOb), 7.0), exitflag=np.full(B, 7, np.int32),
             iters=np.full(B, 7, np.int32), kkt_err=np.full(B, 7.0), feasible=np.full(B, 7, np.int32), strict=np.full(B, 7, np.int32),
             solve_seconds=np.full(1, 7.0))
    return d


def _park_call(B=3, Ncap=40, vOb=None, drop=None, field=None):
    """The entry called through ctypes with every output of both sets and the shared ones filled with 7.  drop: the index of an argument
    passed as NULL; field: (set, name) of a set's field passed as NULL."""
    sc = scenarios.reverse_parking_scenario()
    ox, oy = native.obstacle_points("backwards")
    Bo = max(B, 1)
    x0 = np.column_stack([np.linspace(-5, 5, Bo), np.full(Bo, 8.0), np.zeros(Bo), np.zeros(Bo)])
    V = int(sc["vOb"].sum()); nOb = sc["nOb"]
    vOb = np.ascontiguousarray(sc["vOb"] if vOb is None else vOb, dtype=np.int32)
    A = np.asfortranarray(sc["A"], dtype=np.float64); b = np.ascontiguousarray(sc["b"], dtype=np.float64).ravel()
    xF = np.ascontiguousarray(np.tile(sc["xF"], (Bo, 1)))
    shared = [np.full(Bo, 7, np.int32) for _ in range(3)] + [np.full(1, 7.0)]
    sets = {f: _park_set(Bo, Ncap, V, nOb) for f in ("dist", "sd")}
    structs = {f: _lib.ParkingFlowOut(*[None if field == (f, k) else a.ctypes.data for k, a in sets[f].items()]) for f in sets}
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    args = [C.c_int(B), p(x0), p(xF), p(ox), p(oy), C.c_int(ox.size), C.c_double(0.6), C.c_double(2.7), C.c_int(3), C.c_int(0),
            C.c_int(0), C.c_int(nOb), p(vOb), p(A), p(b), p(sc["ego"]), p(sc["XYbounds"]), C.c_int(0), C.byref(_lib.default_opts()),
            C.c_int(Ncap)] + [p(a) for a in shared] + [C.byref(structs["dist"]), C.byref(structs["sd"])]
    lib = obca_b200.lib()
    assert len(args) == len(getattr(lib, PARK).argtypes)
    if drop is not None:
        args[drop] = None
    rc = getattr(lib, PARK)(*args)
    return rc, lib.obca_last_error().decode(), shared + list(sets["dist"].values()) + list(sets["sd"].values())


def test_parking_symbol_and_ctypes_signature_match_the_header():
    assert PARK in _lib.SYMBOLS
    sc = scenarios.reverse_parking_scenario()
    ox, oy = native.obstacle_points("backwards")
    x0 = np.zeros((2, 4)); x0[:, 1] = 8.0
    with pytest.raises(_lib.ObcaError, match="319"):      # accepted by the binding's types, refused before any device work
        device.plan_solve_goals_both_raw(x0, sc["xF"], ox, oy, 0.6, sc["nOb"], sc["vOb"], sc["A"], sc["b"], sc["ego"], sc["XYbounds"],
                                         Ncap=320)


@pytest.mark.parametrize("drop,name", [(PK_X0, "x0"), (PK_XF, "xF"), (PK_OX, "ox"), (PK_VOB, "vOb"), (PK_EGO, "ego"), (PK_N, "N"),
                                       (PK_STATUS, "status")])
def test_parking_null_required_argument_is_refused(drop, name):
    rc, msg, outs = _park_call(drop=drop)
    assert rc == -1 and msg == "null argument", (name, rc, msg)
    assert _untouched(outs), name


@pytest.mark.parametrize("drop,name", [(PK_DIST, "dist"), (PK_SD, "sd")])
def test_parking_null_set_is_refused(drop, name):
    rc, msg, outs = _park_call(drop=drop)
    assert rc == -1 and msg == "null argument: " + name, (rc, msg)
    assert _untouched(outs)


@pytest.mark.parametrize("field", [(f, k) for f in ("dist", "sd") for k in PK_REQUIRED])
def test_parking_null_required_field_is_refused_and_named(field):
    rc, msg, outs = _park_call(field=field)
    assert rc == -1 and msg == f"null argument: {field[0]}.{field[1]}", (field, rc, msg)
    assert _untouched(outs)


@pytest.mark.parametrize("kw,code,text", [
    (dict(B=-1), -1, "B < 0"),
    (dict(Ncap=1), -1, "Ncap < 2"),
    (dict(Ncap=320), -4, "N = 320 > 319"),
    (dict(vOb=np.array([5, 4, 4, 4], np.int32)), -1, "half-spaces per obstacle"),
])
def test_parking_bad_argument_is_refused_before_any_device_work(kw, code, text):
    rc, msg, outs = _park_call(**kw)
    assert rc == code and text in msg, (kw, rc, msg)
    assert _untouched(outs), kw


@pytest.mark.parametrize("field", [(f, k) for f in ("dist", "sd") for k in ("sl", "strict", "solve_seconds")])
def test_parking_valid_call_without_a_device_stops_at_no_device(field):
    """Every optional field may be null; a valid call then needs the device, with nothing written before."""
    if obca_b200.lib().obca_device_count() > 0:
        pytest.skip("CUDA device present")
    for kw in (dict(), dict(field=field), dict(B=0)):
        rc, msg, outs = _park_call(**kw)
        assert rc == -2 and "no CUDA device" in msg, (kw, rc, msg)
        assert _untouched(outs), kw


# ---- quadcopter -----------------------------------------------------------------------------------------------------------------------
QC_X0, QC_XF, QC_OX, QC_LO, QC_HI, QC_OB, QC_NCAP, QC_N, QC_TSB, QC_STATUS, QC_DIST, QC_SD = 1, 2, 3, 7, 8, 13, 16, 17, 18, 19, 22, 23


def _quad_set(B, Ncap):
    NS = Ncap + 1
    return dict(xp=np.full((B, NS, 12), 7.0), up=np.full((B, Ncap, 4), 7.0), ts=np.full((B, NS), 7.0), lp=np.full((B, NS, 30), 7.0),
                slack=np.full((B, NS, 5), 7.0), exitflag=np.full(B, 7, np.int32), iters=np.full(B, 7, np.int32), kkt_err=np.full(B, 7.0),
                feasible=np.full(B, 7, np.int32), worst=np.full(B, 7.0), solve_seconds=np.full(1, 7.0))


def _quad_call(B=3, Ncap=40, Ts=0.25, reso=1.0, max_nodes=0, x0=None, drop=None, field=None):
    """As _park_call, for the quadcopter entry."""
    sc = scenarios.quadcopter_batch(max(B, 1), seed=2)
    Bo = max(B, 1)
    x0 = np.ascontiguousarray(sc["x0"] if x0 is None else x0, dtype=np.float64)
    xF = np.ascontiguousarray(sc["xF"], dtype=np.float64)
    ob = np.ascontiguousarray(np.asarray(sc["obs"], float).reshape(5, 6))
    ox, oy, oz = np.array([50.0]), np.array([50.0]), np.array([20.0])
    lo, hi = np.zeros(3), np.array([105.0, 105.0, 55.0])
    shared = [np.full(Bo, 7, np.int32), np.full(Bo, 7.0), np.full(Bo, 7, np.int32), np.full(Bo, 7, np.int32), np.full(1, 7.0)]
    sets = {f: _quad_set(Bo, Ncap) for f in ("dist", "sd")}
    structs = {f: _lib.QuadcopterFlowOut(*[None if field == (f, k) else a.ctypes.data for k, a in sets[f].items()]) for f in sets}
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    args = [C.c_int(B), p(x0), p(xF), p(ox), p(oy), p(oz), C.c_int(1), p(lo), p(hi), C.c_double(reso), C.c_int(max_nodes),
            C.c_double(Ts), C.c_double(sc["R"]), p(ob), C.c_double(1.0), C.byref(_lib.default_opts()), C.c_int(Ncap)] + \
        [p(a) for a in shared] + [C.byref(structs["dist"]), C.byref(structs["sd"])]
    lib = obca_b200.lib()
    assert len(args) == len(getattr(lib, QUAD).argtypes)
    if drop is not None:
        args[drop] = None
    rc = getattr(lib, QUAD)(*args)
    return rc, lib.obca_last_error().decode(), shared + list(sets["dist"].values()) + list(sets["sd"].values())


def test_quadcopter_symbol_and_ctypes_signature_match_the_header():
    assert QUAD in _lib.SYMBOLS
    sc = scenarios.quadcopter_batch(2, seed=2)
    with pytest.raises(_lib.ObcaError, match="511"):      # accepted by the binding's types, refused before any device work
        device.plan_solve_quadcopter_both(sc["x0"], sc["xF"], sc["R"], sc["obs"], sc["Ts80"], Ncap=512)


@pytest.mark.parametrize("drop,name", [(QC_X0, "x0"), (QC_XF, "xF"), (QC_OX, "ox"), (QC_LO, "lo"), (QC_HI, "hi"), (QC_OB, "ob"),
                                       (QC_N, "N"), (QC_TSB, "Tsb"), (QC_STATUS, "status")])
def test_quadcopter_null_required_argument_is_refused(drop, name):
    rc, msg, outs = _quad_call(drop=drop)
    assert rc == -1 and msg == "null argument", (name, rc, msg)
    assert _untouched(outs), name


@pytest.mark.parametrize("drop,name", [(QC_DIST, "dist"), (QC_SD, "sd")])
def test_quadcopter_null_set_is_refused(drop, name):
    rc, msg, outs = _quad_call(drop=drop)
    assert rc == -1 and msg == "null argument: " + name, (rc, msg)
    assert _untouched(outs)


@pytest.mark.parametrize("field", [(f, k) for f in ("dist", "sd") for k in QC_REQUIRED])
def test_quadcopter_null_required_field_is_refused_and_named(field):
    rc, msg, outs = _quad_call(field=field)
    assert rc == -1 and msg == f"null argument: {field[0]}.{field[1]}", (field, rc, msg)
    assert _untouched(outs)


@pytest.mark.parametrize("kw,code,text", [
    (dict(B=-1), -1, "B < 0"),
    (dict(Ncap=1), -1, "Ncap < 2"),
    (dict(Ncap=512), -4, "N = 512 > 511"),
    (dict(Ts=0.0), -1, "Ts must be a finite number > 0"),
    (dict(Ts=float("nan")), -1, "Ts must be a finite number > 0"),
    (dict(Ts=0.02, Ncap=511), -1, "sampling time 0"),
    (dict(reso=0.0), -1, "reso must be a finite number > 0"),
    (dict(max_nodes=(1 << 28) + 1), -1, "max_nodes > 2^28"),
    (dict(x0=np.where(np.arange(36).reshape(3, 12) == 14, np.inf, scenarios.quadcopter_batch(3, seed=2)["x0"])), -1,
     "start / goal coordinates must be finite"),
])
def test_quadcopter_bad_argument_is_refused_before_any_device_work(kw, code, text):
    rc, msg, outs = _quad_call(**kw)
    assert rc == code and text in msg, (kw, rc, msg)
    assert _untouched(outs)


@pytest.mark.parametrize("field", [(f, k) for f in ("dist", "sd") for k in ("slack", "worst", "solve_seconds")])
def test_quadcopter_valid_call_without_a_device_stops_at_no_device(field):
    if obca_b200.lib().obca_device_count() > 0:
        pytest.skip("CUDA device present")
    for kw in (dict(), dict(field=field), dict(B=0)):
        rc, msg, outs = _quad_call(**kw)
        assert rc == -2 and "no CUDA device" in msg, (kw, rc, msg)
        assert _untouched(outs), kw


# ---- the output-set structs: include/obca.h against the ctypes Structures -------------------------------------------------------------
LAYOUT_SRC = r'''
#include <cstddef>
#include <cstdio>
#include "obca.h"
#define F(S, f) printf(" %s=%zu", #f, offsetof(S, f))
int main() {
  printf("parking %zu", sizeof(obca_parking_flow_out));
  F(obca_parking_flow_out, xp); F(obca_parking_flow_out, up); F(obca_parking_flow_out, ts); F(obca_parking_flow_out, lp);
  F(obca_parking_flow_out, np); F(obca_parking_flow_out, sl); F(obca_parking_flow_out, exitflag); F(obca_parking_flow_out, iters);
  F(obca_parking_flow_out, kkt_err); F(obca_parking_flow_out, feasible); F(obca_parking_flow_out, strict);
  F(obca_parking_flow_out, solve_seconds);
  printf("\nquadcopter %zu", sizeof(obca_quadcopter_flow_out));
  F(obca_quadcopter_flow_out, xp); F(obca_quadcopter_flow_out, up); F(obca_quadcopter_flow_out, ts); F(obca_quadcopter_flow_out, lp);
  F(obca_quadcopter_flow_out, slack); F(obca_quadcopter_flow_out, exitflag); F(obca_quadcopter_flow_out, iters);
  F(obca_quadcopter_flow_out, kkt_err); F(obca_quadcopter_flow_out, feasible); F(obca_quadcopter_flow_out, worst);
  F(obca_quadcopter_flow_out, solve_seconds);
  printf("\n");
  return 0;
}
'''


def test_struct_layout_matches_ctypes(tmp_path):
    src = tmp_path / "layout.cpp"; exe = tmp_path / "layout"
    src.write_text(LAYOUT_SRC)
    subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    lines = subprocess.check_output([str(exe)], text=True).split("\n")
    for line, S in zip(lines, (_lib.ParkingFlowOut, _lib.QuadcopterFlowOut)):
        _, size, *fields = line.split()
        got = dict(f.split("=") for f in fields)
        assert int(size) == C.sizeof(S), (line, C.sizeof(S))
        assert list(got) == [f for f, _ in S._fields_], (list(got), S._fields_)
        for f, _ in S._fields_:
            assert int(got[f]) == getattr(S, f).offset, (S.__name__, f)
