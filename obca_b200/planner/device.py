"""The GPU warm-start producers of libobca.so (include/obca.h), with the search decisions of the host planners (obca_b200.planner.native):
  - obca_plan_parking_warmstart_batch, Hybrid A*: B start poses towards one goal in one call (plan_raw, plan_batch);
  - obca_plan_quadcopter_warmstart_batch, the 3-D A* of the quadcopter flow: B start / goal pairs in one call (plan_quadcopter_raw,
    plan_quadcopter_batch).
Without a CUDA device the calls raise.  A search that outgrows the device's scratch comes back as POOL_FULL in `status` (the *_raw
functions); the *_batch functions plan those problems with the host planner, which makes the same decisions."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .. import _lib
from . import native

POOL_FULL = 4


def plan_raw(x0s, xF, ox, oy, Ts, L=2.7, sampleN=3, cap=512, max_nodes=0, max_expansions=0, opts=None):
    """The entry's outputs as arrays (rx, ry, ryaw (B, cap), xWS (B, 4 cap), uWS (B, 2 cap), N, status, expansions, seconds).  The
    output buffers start as NaN (N as -1): entries the planner does not write stay so."""
    x0s = np.ascontiguousarray(np.asarray(x0s, float)[:, :3]); B = x0s.shape[0]
    xF = np.ascontiguousarray(np.asarray(xF, float)[:3]); ox = np.ascontiguousarray(ox, float); oy = np.ascontiguousarray(oy, float)
    o = dict(rx=np.full((B, cap), np.nan), ry=np.full((B, cap), np.nan), ryaw=np.full((B, cap), np.nan), xWS=np.full((B, 4 * cap), np.nan),
             uWS=np.full((B, 2 * cap), np.nan), N=np.full(B, -1, np.int32), status=np.full(B, -1, np.int32), expansions=np.zeros(B, np.int32))
    secs = C.c_double(0.0)
    opts = opts if opts is not None else _lib.default_opts()
    p = _lib.ptr
    L_ = _lib.lib()
    f = L_.obca_plan_parking_warmstart_batch
    f.restype = C.c_int
    f.argtypes = [C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_double, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 10
    rc = f(B, p(x0s), p(xF), p(ox), p(oy), int(ox.size), float(Ts), float(L), int(sampleN), int(max_expansions), int(max_nodes), int(cap),
           C.cast(C.byref(opts), C.c_void_p), *[p(o[k]) for k in ("rx", "ry", "ryaw", "xWS", "uWS", "N", "status", "expansions")],
           C.cast(C.byref(secs), C.c_void_p))
    _lib.check(rc)
    o["seconds"] = secs.value
    return o


def plan_quadcopter_raw(starts, goals, ox, oy, oz, lo, hi, reso, cap=1024, max_nodes=0, opts=None):
    """obca_plan_quadcopter_warmstart_batch's outputs as arrays (rx, ry, rz (B, cap), N, status, expansions, seconds): the outputs of
    native.astar3d_raw, planned on the GPU.  The output buffers start as NaN (N and expansions as -1): entries the planner does not write
    stay so."""
    f = lambda a: np.ascontiguousarray(np.asarray(a, float))
    s = f(np.asarray(starts, float).reshape(-1, 3)); g = f(np.asarray(goals, float).reshape(-1, 3)); B = s.shape[0]
    ox, oy, oz, lo, hi = f(ox), f(oy), f(oz), f(lo), f(hi)
    o = dict(rx=np.full((B, cap), np.nan), ry=np.full((B, cap), np.nan), rz=np.full((B, cap), np.nan), N=np.full(B, -1, np.int32),
             status=np.full(B, -1, np.int32), expansions=np.full(B, -1, np.int32))
    secs = C.c_double(0.0)
    opts = opts if opts is not None else _lib.default_opts()
    p = _lib.ptr
    fn = _lib.lib().obca_plan_quadcopter_warmstart_batch
    fn.restype = C.c_int
    fn.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_int] + [C.c_void_p] * 8
    rc = fn(B, p(s), p(g), p(ox), p(oy), p(oz), int(ox.size), p(lo), p(hi), float(reso), int(max_nodes), int(cap), C.cast(C.byref(opts), C.c_void_p),
            *[p(o[k]) for k in ("rx", "ry", "rz", "N", "status", "expansions")], C.cast(C.byref(secs), C.c_void_p))
    _lib.check(rc)
    o["seconds"] = secs.value
    return o


def plan_quadcopter_batch(x0s, xFs, Ts=0.25, cap=1024, max_nodes=0, opts=None):
    """native.plan_quadcopter_batch on the GPU: for every pair the dictionary of a_star_3d.plan_quadcopter_warm_start (None where no path
    was found).  Pairs whose search outgrew the device's scratch (POOL_FULL, see include/obca.h) are planned by the host library, which
    makes the same decisions; raises if a path did not fit `cap`, as native.plan_quadcopter_batch does."""
    s, g, ox, oy, oz, lo, hi, reso = native.quadcopter_problem(x0s, xFs)
    o = plan_quadcopter_raw(s, g, ox, oy, oz, lo, hi, reso, cap, max_nodes, opts)
    st = o["status"].copy()
    full = np.nonzero(st == POOL_FULL)[0]
    if full.size:
        h = native.astar3d_raw(s[full], g[full], ox, oy, oz, lo, hi, reso, cap)
        for k in ("rx", "ry", "rz", "N", "status"):
            o[k][full] = h[k]
        st[full] = h["status"]
    if (st > 1).any():
        raise native.PlannerError(f"obca_plan_quadcopter_warmstart_batch: status {st[st > 1][:5]} at pairs {np.nonzero(st > 1)[0][:5]}")
    out = []
    for i in range(len(st)):
        if st[i]:
            out.append(None); continue
        n = int(o["N"][i]) + 1
        out.append(native.quadcopter_warm_start(o["rx"][i, :n].copy(), o["ry"][i, :n].copy(), o["rz"][i, :n].copy(), Ts))
    return out


def plan_batch(x0s, xF, scenario="backwards", Ts=None, L=2.7, sampleN=3, cap=512, max_nodes=0, opts=None):
    """native.plan_batch on the GPU: the same list of dictionaries (None where no path was found).  Poses whose search outgrew the
    device's scratch (POOL_FULL, see include/obca.h) are planned by the host planner (native.plan_warm_start); raises if a pose did not
    fit `cap`, as native.plan_batch does."""
    ox, oy = native.obstacle_points(scenario)
    Ts = Ts or (0.6 if scenario == "backwards" else 0.9) / 3 * sampleN
    o = plan_raw(x0s, xF, ox, oy, Ts, L, sampleN, cap, max_nodes, 0, opts)
    st = o["status"]
    bad = (st > 1) & (st != POOL_FULL)
    if bad.any():
        raise native.PlannerError(f"obca_plan_parking_warmstart_batch: status {st[bad][:5]} at poses {np.nonzero(bad)[0][:5]}")
    x0s = np.asarray(x0s, float)
    out = []
    for i in range(len(st)):
        if st[i] == POOL_FULL:
            out.append(native.plan_warm_start(x0s[i, :3], xF, scenario, Ts, L, sampleN, cap)); continue
        if st[i]:
            out.append(None); continue
        n = int(o["N"][i])
        out.append(dict(rx=o["rx"][i, :n + 1].copy(), ry=o["ry"][i, :n + 1].copy(), ryaw=o["ryaw"][i, :n + 1].copy(),
                        xWS=o["xWS"][i, :4 * (n + 1)].reshape(4, n + 1).T.copy(), uWS=o["uWS"][i, :2 * n].reshape(2, n).T.copy(), N=n, Ts=Ts))
    return out
