"""ctypes loader for the DEVELOPMENT emulation of the GPU Hybrid A* planner (tests/emul/emul_plan.cpp).  Test tool only."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SO = os.path.join(HERE, "libobca_emul_plan.so")
SRC = os.path.join(HERE, "emul_plan.cpp")


def build(force=False):
    srcs = [SRC, os.path.join(ROOT, "obca_b200", "csrc", "obca_plan.cuh"), os.path.join(ROOT, "obca_b200", "planner", "csrc", "obca_plan_core.h"),
            os.path.join(ROOT, "include", "obca_planner.h")]
    if force or not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", SO, SRC])
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        f = _lib.emul_plan_batch
        f.restype = C.c_int
        f.argtypes = [C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_double, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 8
    return _lib


def plan_raw(x0s, xF, ox, oy, Ts, L=2.7, sampleN=3, cap=512, max_expansions=0, max_nodes=32768):
    """obca_plan_parking_warmstart_batch's raw outputs, emulated; output buffers start as NaN (N as -1)."""
    x0s = np.ascontiguousarray(np.asarray(x0s, float)[:, :3]); B = x0s.shape[0]
    xF = np.ascontiguousarray(np.asarray(xF, float)[:3]); ox = np.ascontiguousarray(ox, float); oy = np.ascontiguousarray(oy, float)
    o = dict(rx=np.full((B, cap), np.nan), ry=np.full((B, cap), np.nan), ryaw=np.full((B, cap), np.nan), xWS=np.full((B, 4 * cap), np.nan),
             uWS=np.full((B, 2 * cap), np.nan), N=np.full(B, -1, np.int32), status=np.full(B, -1, np.int32), expansions=np.zeros(B, np.int32))
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib().emul_plan_batch(B, p(x0s), p(xF), p(ox), p(oy), int(ox.size), float(Ts), float(L), int(sampleN), int(max_expansions),
                               int(max_nodes), int(cap), *[p(o[k]) for k in ("rx", "ry", "ryaw", "xWS", "uWS", "N", "status", "expansions")])
    assert rc == 0, rc
    return o
