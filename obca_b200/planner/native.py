"""ctypes binding of the native warm-start producer libobca_planner.so (include/obca_planner.h; built in-tree by
__graft_entry__.build() from obca_b200/planner/csrc/obca_planner.cpp).  Same results as the Python modules of this package -- which
stay the documented, line-by-line restatement of the reference -- at about 1/100 of the time."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .._lib import declare, prototypes

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(HERE, "libobca_planner.so")
HEADER = os.path.join(os.path.dirname(os.path.dirname(HERE)), "include", "obca_planner.h")
_lib = None


class PlannerError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise PlannerError(f"{SO_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'`")
        _lib = declare(C.CDLL(SO_PATH), prototypes(HEADER, PlannerError))
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


SCENARIOS = {"backwards": 0, "parallel": 1}


def obstacle_points(scenario: str):
    n = C.c_int(0)
    ox = np.zeros(1024); oy = np.zeros(1024)
    rc = lib().obca_scenario_obstacle_points(SCENARIOS[scenario], 1024, _p(ox), _p(oy), C.byref(n))
    if rc:
        raise PlannerError(f"obca_scenario_obstacle_points: {rc}")
    return ox[:n.value].copy(), oy[:n.value].copy()


def calc_hybrid_astar_path(sx, sy, syaw, gx, gy, gyaw, ox, oy, xyreso=0.0, yawreso=0.0, max_expansions=200000, cap=8192):
    """(rx, ry, ryaw) sampled every 0.1 m, or (None, None, None) when no path is found (hybrid_a_star.jl:104-190)."""
    ox = np.ascontiguousarray(ox, float); oy = np.ascontiguousarray(oy, float)
    rx = np.zeros(cap); ry = np.zeros(cap); ryaw = np.zeros(cap); n = C.c_int(0)
    rc = lib().obca_hybrid_astar(float(sx), float(sy), float(syaw), float(gx), float(gy), float(gyaw), _p(ox), _p(oy), int(ox.size), float(xyreso),
                                 float(yawreso), int(max_expansions), cap, _p(rx), _p(ry), _p(ryaw), C.byref(n))
    if rc == 1:
        return None, None, None
    if rc:
        raise PlannerError(f"obca_hybrid_astar: {rc}")
    return rx[:n.value].copy(), ry[:n.value].copy(), ryaw[:n.value].copy()


def plan_warm_start(x0, xF, scenario="backwards", Ts=None, L=2.7, sampleN=3, cap=1024):
    """main.jl:215-248 in one native call; same dictionary as obca_b200.planner.warmstart.plan_warm_start (without the full path)."""
    x0 = np.ascontiguousarray(np.asarray(x0, float)[:3]); xF = np.ascontiguousarray(np.asarray(xF, float)[:3])
    rx = np.zeros(cap); ry = np.zeros(cap); ryaw = np.zeros(cap); xWS = np.zeros(4 * cap); uWS = np.zeros(2 * cap); N = C.c_int(0)
    rc = lib().obca_plan_warmstart(_p(x0), _p(xF), SCENARIOS[scenario], float(Ts or 0.0), float(L), int(sampleN), cap, _p(rx), _p(ry), _p(ryaw),
                                   _p(xWS), _p(uWS), C.byref(N))
    if rc == 1:
        return None
    if rc:
        raise PlannerError(f"obca_plan_warmstart: {rc}")
    n = N.value
    Ts = Ts or (0.6 if scenario == "backwards" else 0.9) / 3 * sampleN
    return dict(rx=rx[:n + 1].copy(), ry=ry[:n + 1].copy(), ryaw=ryaw[:n + 1].copy(), xWS=xWS[:4 * (n + 1)].reshape(4, n + 1).T.copy(),
                uWS=uWS[:2 * n].reshape(2, n).T.copy(), N=n, Ts=Ts)


def plan_batch(x0s, xF, scenario="backwards", workers=0, Ts=None, L=2.7, sampleN=3, cap=512):
    """Hybrid A* warm starts for many start poses on a pool of host threads (the randomised sweeps of main.jl:165-168); same list of
    dictionaries as obca_b200.planner.warmstart.plan_batch (None where no path was found)."""
    x0s = np.ascontiguousarray(np.asarray(x0s, float)[:, :3]); B = x0s.shape[0]
    xF = np.ascontiguousarray(np.asarray(xF, float)[:3])
    rx = np.zeros((B, cap)); ry = np.zeros((B, cap)); ryaw = np.zeros((B, cap)); xWS = np.zeros((B, 4 * cap)); uWS = np.zeros((B, 2 * cap))
    N = np.zeros(B, np.int32); st = np.zeros(B, np.int32)
    rc = lib().obca_plan_warmstart_batch(B, _p(x0s), _p(xF), SCENARIOS[scenario], float(Ts or 0.0), float(L), int(sampleN), cap, int(workers),
                                         _p(rx), _p(ry), _p(ryaw), _p(xWS), _p(uWS), _p(N), _p(st))
    if rc or (st > 1).any():
        raise PlannerError(f"obca_plan_warmstart_batch: {rc}, status {st[st > 1][:5]}")
    Ts = Ts or (0.6 if scenario == "backwards" else 0.9) / 3 * sampleN
    out = []
    for i in range(B):
        if st[i]:
            out.append(None); continue
        n = int(N[i])
        out.append(dict(rx=rx[i, :n + 1].copy(), ry=ry[i, :n + 1].copy(), ryaw=ryaw[i, :n + 1].copy(), xWS=xWS[i, :4 * (n + 1)].reshape(4, n + 1).T.copy(),
                        uWS=uWS[i, :2 * n].reshape(2, n).T.copy(), N=n, Ts=Ts))
    return out


def plan_cloud_raw(x0s, xFs, ox, oy, Ts, L=2.7, sampleN=3, cap=512, workers=0):
    """obca_plan_warmstart_cloud_batch's outputs as arrays: rx, ry, ryaw (B, cap), xWS (B, 4 cap), uWS (B, 2 cap), N, status, expansions --
    the layout of device.plan_goals_raw.  x0s (B, >= 3) start poses, xFs (B, >= 3) or (>= 3,) goals, (ox, oy) any point cloud.  The output
    buffers start as NaN (N as -1)."""
    x0s = np.ascontiguousarray(np.asarray(x0s, float)[:, :3]); B = x0s.shape[0]
    xFs = np.asarray(xFs, float)
    xFs = np.ascontiguousarray(np.broadcast_to(xFs[:3], (B, 3)) if xFs.ndim == 1 else xFs.reshape(B, -1)[:, :3])
    ox = np.ascontiguousarray(ox, float); oy = np.ascontiguousarray(oy, float)
    o = dict(rx=np.full((B, cap), np.nan), ry=np.full((B, cap), np.nan), ryaw=np.full((B, cap), np.nan), xWS=np.full((B, 4 * cap), np.nan),
             uWS=np.full((B, 2 * cap), np.nan), N=np.full(B, -1, np.int32), status=np.full(B, -1, np.int32), expansions=np.zeros(B, np.int32))
    rc = lib().obca_plan_warmstart_cloud_batch(B, _p(x0s), _p(xFs), _p(ox), _p(oy), int(ox.size), float(Ts), float(L), int(sampleN), int(cap),
                                               int(workers), *[_p(o[k]) for k in ("rx", "ry", "ryaw", "xWS", "uWS", "N", "status", "expansions")])
    if rc:
        raise PlannerError(f"obca_plan_warmstart_cloud_batch: {rc}")
    return o


def warm_starts(o, Ts):
    """The list of dictionaries of plan_batch from raw planner outputs (plan_cloud_raw, device.plan_goals_raw): None where the status is
    not OK."""
    out = []
    for i in range(len(o["status"])):
        if o["status"][i]:
            out.append(None); continue
        n = int(o["N"][i])
        out.append(dict(rx=o["rx"][i, :n + 1].copy(), ry=o["ry"][i, :n + 1].copy(), ryaw=o["ryaw"][i, :n + 1].copy(),
                        xWS=o["xWS"][i, :4 * (n + 1)].reshape(4, n + 1).T.copy(), uWS=o["uWS"][i, :2 * n].reshape(2, n).T.copy(), N=n, Ts=Ts))
    return out


def plan_cloud_batch(x0s, xFs, ox, oy, Ts, L=2.7, sampleN=3, cap=512, workers=0):
    """Hybrid A* warm starts for many start poses, each with its own goal, among any point cloud, on a pool of host threads: the list
    of dictionaries of plan_batch (None where no path was found).  Ts: the warm start's sampling time (> 0)."""
    o = plan_cloud_raw(x0s, xFs, ox, oy, Ts, L, sampleN, cap, workers)
    st = o["status"]
    if (st > 1).any():
        raise PlannerError(f"obca_plan_warmstart_cloud_batch: status {st[st > 1][:5]} at poses {np.nonzero(st > 1)[0][:5]}")
    return warm_starts(o, Ts)


def reeds_shepp_length(sx, sy, syaw, gx, gy, gyaw, maxc):
    return lib().obca_reeds_shepp_length(float(sx), float(sy), float(syaw), float(gx), float(gy), float(gyaw), float(maxc))


# ---- the 3-D A* of the quadcopter flow (obca_astar3d_batch; same decisions as obca_b200.planner.a_star_3d.calc_astar_path) ----

def _f64(a):
    return np.ascontiguousarray(np.asarray(a, float))


def astar3d_obstacle_map(ox, oy, oz, lo, hi, reso):
    """(blocked (w0, w1, w2) bool, mn, w): the map the 3-D A* entries build; equals a_star_3d.calc_obstacle_map(ox / reso, ..., lo, hi, reso)."""
    ox, oy, oz, lo, hi = _f64(ox), _f64(oy), _f64(oz), _f64(lo), _f64(hi)
    mn = np.zeros(3, np.int64); w = np.zeros(3, np.int32)
    rc = lib().obca_astar3d_obstacle_map(_p(ox), _p(oy), _p(oz), int(ox.size), _p(lo), _p(hi), float(reso), _p(mn), _p(w), None, 0)
    if rc not in (0, 2):
        raise PlannerError(f"obca_astar3d_obstacle_map: {rc}")
    blocked = np.zeros(int(np.prod(w.astype(np.int64))), np.uint8)
    rc = lib().obca_astar3d_obstacle_map(_p(ox), _p(oy), _p(oz), int(ox.size), _p(lo), _p(hi), float(reso), _p(mn), _p(w), _p(blocked), blocked.size)
    if rc:
        raise PlannerError(f"obca_astar3d_obstacle_map: {rc}")
    return blocked.reshape(tuple(w.tolist())).astype(bool), mn.tolist(), w.tolist()


def astar3d_raw(starts, goals, ox, oy, oz, lo, hi, reso, cap=1024, nthreads=0):
    """obca_astar3d_batch's outputs as arrays: rx, ry, rz (B, cap), N, status, expansions.  The output buffers start as NaN (N as -1)."""
    s = _f64(np.asarray(starts, float).reshape(-1, 3)); g = _f64(np.asarray(goals, float).reshape(-1, 3)); B = s.shape[0]
    ox, oy, oz, lo, hi = _f64(ox), _f64(oy), _f64(oz), _f64(lo), _f64(hi)
    o = dict(rx=np.full((B, cap), np.nan), ry=np.full((B, cap), np.nan), rz=np.full((B, cap), np.nan), N=np.full(B, -1, np.int32),
             status=np.full(B, -1, np.int32), expansions=np.full(B, -1, np.int32))
    rc = lib().obca_astar3d_batch(B, _p(s), _p(g), _p(ox), _p(oy), _p(oz), int(ox.size), _p(lo), _p(hi), float(reso), int(cap), int(nthreads),
                                  *[_p(o[k]) for k in ("rx", "ry", "rz", "N", "status", "expansions")])
    if rc:
        raise PlannerError(f"obca_astar3d_batch: {rc}")
    return o


def calc_astar_path(sx, sy, sz, gx, gy, gz, ox, oy, oz, xmin, ymin, zmin, xmax, ymax, zmax, reso, cap=4096):
    """a_star_3d.calc_astar_path in one native call: (rx, ry, rz), or (None, None, None) when there is no path."""
    o = astar3d_raw([(sx, sy, sz)], [(gx, gy, gz)], ox, oy, oz, (xmin, ymin, zmin), (xmax, ymax, zmax), reso, cap, 1)
    st = int(o["status"][0])
    if st == 1:
        return None, None, None
    if st:
        raise PlannerError(f"obca_astar3d_batch: status {st}")
    n = int(o["N"][0]) + 1
    return o["rx"][0, :n].copy(), o["ry"][0, :n].copy(), o["rz"][0, :n].copy()


def quadcopter_warm_start(rx, ry, rz, Ts):
    """The dictionary of a_star_3d.plan_quadcopter_warm_start for the path (rx, ry, rz) on the 10x grid (mainQuadcopter.jl:130-137)."""
    from .grid_policy import jround
    N = rx.size - 1
    Ts_as = jround(Ts * 80 / N * 100) / 100
    xWS = np.zeros((12, N + 1))
    xWS[0], xWS[1], xWS[2] = rx / 10.0, ry / 10.0, rz / 10.0
    return dict(N=N, Ts=Ts_as, xWS=xWS, uWS=0.5 * np.ones((4, N)), timeWS=1.0, path=(rx, ry, rz))


def quadcopter_problem(x0s, xFs):
    """The inputs of plan_quadcopter_warm_start for a batch: starts and goals on the 10x grid (B, 3), the environment's points and
    bounds, reso = 1."""
    from .a_star_3d import quadcopter_environment
    x0s = np.asarray(x0s, float).reshape(len(x0s), -1)[:, :3]; xFs = np.asarray(xFs, float).reshape(len(xFs), -1)[:, :3]
    ox, oy, oz, lo, hi = quadcopter_environment()
    return x0s * 10.0, xFs * 10.0, ox, oy, oz, lo, hi, 1.0


def plan_quadcopter_batch(x0s, xFs, Ts=0.25, nthreads=0, cap=1024):
    """a_star_3d.plan_quadcopter_warm_start for every pair (x0s[i], xFs[i]) on a pool of host threads: the same list of dictionaries
    (None where no path was found)."""
    s, g, ox, oy, oz, lo, hi, reso = quadcopter_problem(x0s, xFs)
    o = astar3d_raw(s, g, ox, oy, oz, lo, hi, reso, cap, nthreads)
    st = o["status"]
    if (st > 1).any():
        raise PlannerError(f"obca_astar3d_batch: status {st[st > 1][:5]} at pairs {np.nonzero(st > 1)[0][:5]}")
    out = []
    for i in range(len(st)):
        if st[i]:
            out.append(None); continue
        n = int(o["N"][i]) + 1
        out.append(quadcopter_warm_start(o["rx"][i, :n].copy(), o["ry"][i, :n].copy(), o["rz"][i, :n].copy(), Ts))
    return out
