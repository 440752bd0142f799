"""ctypes loader for the DEVELOPMENT emulation of the GPU 3-D A* planner (tests/emul/emul_plan3d.cpp).  Test tool only."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SO = os.path.join(HERE, "libobca_emul_plan3d.so")
SRC = os.path.join(HERE, "emul_plan3d.cpp")


def build(force=False):
    srcs = [SRC, os.path.join(ROOT, "obca_b200", "planner", "csrc", "obca_astar3d_core.h"), os.path.join(ROOT, "include", "obca_planner.h")]
    if force or not os.path.exists(SO) or any(os.path.getmtime(s) > os.path.getmtime(SO) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-shared", "-fPIC", "-o", SO, SRC])
    return SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        f = _lib.emul_plan3d_batch
        f.restype = C.c_int
        f.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 8
    return _lib


def plan_raw(starts, goals, ox, oy, oz, lo, hi, reso, max_nodes=1 << 18, max_queue=1 << 16, cap=1024):
    """The GPU entry's raw outputs, emulated, plus the nodes and the longest queue of every search; output buffers start as NaN
    (N, nodes and queue_max as -1)."""
    f = lambda a: np.ascontiguousarray(np.asarray(a, float))
    s = f(np.asarray(starts, float).reshape(-1, 3)); g = f(np.asarray(goals, float).reshape(-1, 3)); B = s.shape[0]
    ox, oy, oz, lo, hi = f(ox), f(oy), f(oz), f(lo), f(hi)
    o = dict(rx=np.full((B, cap), np.nan), ry=np.full((B, cap), np.nan), rz=np.full((B, cap), np.nan), N=np.full(B, -1, np.int32),
             status=np.full(B, -1, np.int32), expansions=np.full(B, -1, np.int32), nodes=np.full(B, -1, np.int32),
             queue_max=np.full(B, -1, np.int32))
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib().emul_plan3d_batch(B, p(s), p(g), p(ox), p(oy), p(oz), int(ox.size), p(lo), p(hi), float(reso), int(max_nodes), int(max_queue),
                                 int(cap), *[p(o[k]) for k in ("rx", "ry", "rz", "N", "status", "expansions", "nodes", "queue_max")])
    assert rc == 0, rc
    return o
