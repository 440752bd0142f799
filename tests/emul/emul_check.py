"""ctypes loader for the DEVELOPMENT host run of the constraint checkers with the kernels' reduction (tests/emul/emul_check.cpp).
Test tool only."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from emul import _p

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libobca_emul_check.so")
SRC = os.path.join(HERE, "emul_check.cpp")


def build(force=False):
    csrc = os.path.join(HERE, "../../obca_b200/csrc")
    srcs = [SRC] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))]
    if force or not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-std=c++17", "-o", SO, SRC])
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.emul_check_parking.restype = C.c_int
        _lib.emul_check_parking.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 5 + [C.c_double, C.c_double] + [C.c_void_p] * 8 + \
            [C.c_int, C.c_int, C.c_uint64] + [C.c_void_p] * 3
        _lib.emul_check_quadcopter.restype = C.c_int
        _lib.emul_check_quadcopter.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_double, C.c_void_p, C.c_void_p, C.c_double,
                                                                             C.c_uint64, C.c_void_p, C.c_void_p]
    return _lib


def _cm(a):
    """A Julia-shaped r x c array as the C-ABI's column-major block."""
    return np.ascontiguousarray(np.asarray(a, float).T)


def check_parking(p, seed=0):
    """p: dict of one parking problem in the oracle's arguments (x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, x 4x(N+1), u 2xN,
    l Vx(N+1), n 4nOb x(N+1), timeScale (N+1), fixTime, sd, sl nOb x(N+1) or None).  Returns (feasible, e (7,), strict)."""
    vOb = np.ascontiguousarray(p["vOb"], np.int32)
    A = np.asfortranarray(np.asarray(p["A"], float).reshape(-1, 2))
    arrs = [np.ascontiguousarray(np.asarray(p[k], float).ravel()) for k in ("b", "x0", "xF", "ego", "XYbounds", "timeScale")]
    x, u, l, n = (_cm(p[k]) for k in ("x", "u", "l", "n"))
    sl = _cm(p["sl"]) if p.get("sl") is not None else None
    feas = np.zeros(1, np.int32); e = np.zeros(7, np.int32); strict = np.zeros(1, np.int32)
    rc = lib().emul_check_parking(int(p["N"]), int(p["nOb"]), _p(vOb), _p(A), _p(arrs[0]), _p(arrs[1]), _p(arrs[2]), float(p["Ts"]),
                                  float(p["L"]), _p(arrs[3]), _p(arrs[4]), _p(x), _p(u), _p(l), _p(n), _p(arrs[5]), _p(sl),
                                  int(p["fixTime"]), int(p["sd"]), int(seed), _p(feas), _p(e), _p(strict))
    assert rc == 0, rc
    return int(feas[0]), e, int(strict[0])


def check_quadcopter(q, seed=0):
    """q: dict of one quadcopter problem (x 12x(N+1), u 4xN, timeScale (N+1), x0, xF, Ts, lam 30x(N+1), obs (5, 6), R).
    Returns (feasible, worst)."""
    x, u, lam = (_cm(q[k]) for k in ("x", "u", "lam"))
    ts, x0, xF, ob = (np.ascontiguousarray(np.asarray(q[k], float).ravel()) for k in ("timeScale", "x0", "xF", "obs"))
    feas = np.zeros(1, np.int32); worst = np.zeros(1)
    rc = lib().emul_check_quadcopter(x.shape[0] - 1, _p(x), _p(u), _p(ts), _p(x0), _p(xF), float(q["Ts"]), _p(lam), _p(ob), float(q["R"]),
                                     int(seed), _p(feas), _p(worst))
    assert rc == 0, rc
    return int(feas[0]), float(worst[0])
