"""ctypes loader for the DEVELOPMENT emulation of a quadcopter batch with a horizon and a sampling time per problem
(tests/emul/emul_quad_mixed.cpp).  Test tool only."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from emul import _p

HERE = os.path.dirname(os.path.abspath(__file__))
SO = os.path.join(HERE, "libobca_emul_quad_mixed.so")
SRC = os.path.join(HERE, "emul_quad_mixed.cpp")


def build(force=False):
    csrc = os.path.join(HERE, "../../obca_b200/csrc")
    srcs = [SRC] + [os.path.join(csrc, f) for f in os.listdir(csrc) if f.endswith((".cuh", ".h"))]
    if force or not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-fopenmp", "-shared", "-fPIC", "-std=c++17", "-o", SO, SRC])
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
    return _lib


def quad_solve_mixed(sc, Nmax, variant="sd", opts=None):
    """Quadcopter problems with horizons sc["Ns"][i] and sampling times sc["Ts"][i] in ONE emulated batch laid out for Nmax
    (obca_quadcopter_solve_mixed's layout).  sc: as from scenarios.quadcopter_mixed_batch (xWS[i] 12 x (Ns[i]+1)).  The padding
    of the inputs and of the outputs is NaN.  Returns the padded outputs in the Julia orientation: xp (B, 12, Nmax+1),
    up (B, 4, Nmax), ts (B, Nmax+1), lp (B, 30, Nmax+1), slack (B, 5, Nmax+1)."""
    Ns = np.ascontiguousarray(sc["Ns"], dtype=np.int32)
    B, NS = len(Ns), Nmax + 1
    Tsb = np.ascontiguousarray(np.broadcast_to(np.asarray(sc["Ts"], float), (B,)))
    x0 = np.ascontiguousarray(sc["x0"], dtype=float); xF = np.ascontiguousarray(sc["xF"], dtype=float)
    obs = np.ascontiguousarray(sc["obs"], dtype=float)
    xWS = np.full((B, NS, 12), np.nan)
    for i, w in enumerate(sc["xWS"]):
        xWS[i, :w.shape[1]] = np.asarray(w, float).T
    sd = 1 if variant == "sd" else 0
    xp = np.full((B, NS, 12), np.nan); up = np.full((B, Nmax, 4), np.nan); ts = np.full((B, NS), np.nan)
    lp = np.full((B, NS, 30), np.nan); sl = np.full((B, NS, 5), np.nan)
    status = np.zeros(B, np.int32); iters = np.zeros(B, np.int32); err = np.zeros(B)
    f = lib().emul_quadcopter_solve_mixed
    f.restype = C.c_int
    f.argtypes = [C.c_int, C.c_void_p, C.c_int] + [C.c_void_p] * 3 + [C.c_double, C.c_void_p, C.c_void_p, C.c_double, C.c_int] + \
                 [C.c_void_p] * 9
    rc = f(B, _p(Ns), Nmax, _p(x0), _p(xF), _p(Tsb), float(sc["R"]), _p(obs), _p(xWS), float(sc.get("timeWS", 1.0)), sd,
           C.cast(C.byref(opts), C.c_void_p) if opts is not None else None, _p(xp), _p(up), _p(ts), _p(lp), _p(sl), _p(status),
           _p(iters), _p(err))
    assert rc == 0, rc
    T = lambda a: np.transpose(a, (0, 2, 1))
    return dict(xp=T(xp), up=T(up), ts=ts, lp=T(lp), slack=T(sl), status=status, iters=iters, err=err, Ns=Ns)
