"""ctypes loader for the DEVELOPMENT emulation of the GPU Hybrid A* planner with a goal per start pose and of its heuristic maps
(tests/emul/emul_plan_goals.cpp).  Test tool only."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SO = os.path.join(HERE, "libobca_emul_plan_goals.so")
SRC = os.path.join(HERE, "emul_plan_goals.cpp")


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
        g = _lib.emul_plan_goals
        g.restype = C.c_int
        g.argtypes = [C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_double, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 8
        h = _lib.emul_plan_hmaps
        h.restype = C.c_int
        h.argtypes = [C.c_int] + [C.c_void_p] * 3 + [C.c_int] + [C.c_void_p] * 3 + [C.c_longlong]
    return _lib


def plan_goals_raw(x0s, xFs, ox, oy, Ts, L=2.7, sampleN=3, cap=512, max_expansions=0, max_nodes=32768):
    """obca_plan_parking_warmstart_goals's raw outputs (a goal per pose, xFs (B, >= 3)), emulated; output buffers start as NaN (N as -1)."""
    x0s = np.ascontiguousarray(np.asarray(x0s, float)[:, :3]); B = x0s.shape[0]
    xFs = np.ascontiguousarray(np.asarray(xFs, float).reshape(B, -1)[:, :3]); ox = np.ascontiguousarray(ox, float); oy = np.ascontiguousarray(oy, float)
    o = dict(rx=np.full((B, cap), np.nan), ry=np.full((B, cap), np.nan), ryaw=np.full((B, cap), np.nan), xWS=np.full((B, 4 * cap), np.nan),
             uWS=np.full((B, 2 * cap), np.nan), N=np.full(B, -1, np.int32), status=np.full(B, -1, np.int32), expansions=np.zeros(B, np.int32))
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = lib().emul_plan_goals(B, p(x0s), p(xFs), p(ox), p(oy), int(ox.size), float(Ts), float(L), int(sampleN), int(max_expansions),
                               int(max_nodes), int(cap), *[p(o[k]) for k in ("rx", "ry", "ryaw", "xWS", "uWS", "N", "status", "expansions")])
    assert rc == 0, rc
    return o


def hmaps(goals, ox, oy):
    """The heuristic maps of the goals (G, >= 2) among the cloud three ways, each (G, xw, yw): calc_dist_policy, its two parts
    (calc_heur_grid + dist_from_goal), and the relaxation of k_plan_hmap; plus (minx, miny)."""
    g = np.ascontiguousarray(np.asarray(goals, float).reshape(-1, np.shape(goals)[-1])[:, :2]); G = g.shape[0]
    ox = np.ascontiguousarray(ox, float); oy = np.ascontiguousarray(oy, float)
    mn = np.zeros(2, np.int64); w = np.zeros(2, np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    assert lib().emul_plan_hmaps(G, p(g), p(ox), p(oy), int(ox.size), p(mn), p(w), None, 0) == 2
    m = np.zeros(3 * G * int(w[0]) * int(w[1]))
    assert lib().emul_plan_hmaps(G, p(g), p(ox), p(oy), int(ox.size), p(mn), p(w), p(m), m.size) == 0
    m = m.reshape(3, G, int(w[0]), int(w[1]))
    return m[0], m[1], m[2], (int(mn[0]), int(mn[1]))
