"""The GPU warm-start producers of libobca.so (include/obca.h), with the search decisions of the host planners (obca_b200.planner.native):
  - obca_plan_parking_warmstart_batch, Hybrid A*: B start poses towards one goal in one call (plan_raw, plan_batch);
  - obca_plan_parking_warmstart_goals, the same with a goal per pose among any point cloud (plan_goals_raw, plan_goals_batch);
  - obca_plan_quadcopter_warmstart_batch, the 3-D A* of the quadcopter flow: B start / goal pairs in one call (plan_quadcopter_raw,
    plan_quadcopter_batch);
  - obca_parking_plan_solve_goals and obca_quadcopter_plan_solve, which plan, solve and check a batch in one call without leaving the
    device (plan_solve_goals, plan_solve_quadcopter and their *_raw twins);
  - obca_parking_plan_solve_both and obca_quadcopter_plan_solve_both, the same with one plan solved and checked with both formulations
    (plan_solve_goals_both, plan_solve_quadcopter_both and their *_raw twins).
Without a CUDA device the calls raise.  A search that outgrows the device's scratch comes back as POOL_FULL in `status` (the *_raw
functions); the *_batch functions plan those problems with the host planner, which makes the same decisions."""
from __future__ import annotations

import ctypes as C

import numpy as np

from .. import _lib
from . import native

POOL_FULL = 4


def _plan_call(entry, x0s, xF, ox, oy, Ts, L, sampleN, cap, max_nodes, max_expansions, opts):
    x0s = np.ascontiguousarray(np.asarray(x0s, float)[:, :3]); B = x0s.shape[0]
    ox = np.ascontiguousarray(ox, float); oy = np.ascontiguousarray(oy, float)
    o = dict(rx=np.full((B, cap), np.nan), ry=np.full((B, cap), np.nan), ryaw=np.full((B, cap), np.nan), xWS=np.full((B, 4 * cap), np.nan),
             uWS=np.full((B, 2 * cap), np.nan), N=np.full(B, -1, np.int32), status=np.full(B, -1, np.int32), expansions=np.zeros(B, np.int32))
    secs = C.c_double(0.0)
    p = _lib.ptr
    rc = getattr(_lib.lib(), entry)(B, p(x0s), p(xF), p(ox), p(oy), int(ox.size), float(Ts), float(L), int(sampleN), int(max_expansions),
                                    int(max_nodes), int(cap), _lib.opts_arg(opts),
                                    *[p(o[k]) for k in ("rx", "ry", "ryaw", "xWS", "uWS", "N", "status", "expansions")], C.byref(secs))
    _lib.check(rc)
    o["seconds"] = secs.value
    return o


def plan_raw(x0s, xF, ox, oy, Ts, L=2.7, sampleN=3, cap=512, max_nodes=0, max_expansions=0, opts=None):
    """The entry's outputs as arrays (rx, ry, ryaw (B, cap), xWS (B, 4 cap), uWS (B, 2 cap), N, status, expansions, seconds).  The
    output buffers start as NaN (N as -1): entries the planner does not write stay so."""
    xF = np.ascontiguousarray(np.asarray(xF, float)[:3])
    return _plan_call("obca_plan_parking_warmstart_batch", x0s, xF, ox, oy, Ts, L, sampleN, cap, max_nodes, max_expansions, opts)


def plan_goals_raw(x0s, xFs, ox, oy, Ts, L=2.7, sampleN=3, cap=512, max_nodes=0, max_expansions=0, opts=None, host_fallback=False):
    """obca_plan_parking_warmstart_goals's outputs as arrays, as plan_raw: start poses x0s (B, >= 3), goals xFs (B, >= 3) or one goal
    (>= 3,) for all.  host_fallback: poses whose search outgrew the device's scratch (POOL_FULL) are planned by the host twin
    (native.plan_cloud_raw, the same decisions) and their entries replaced by its outputs."""
    B = np.shape(x0s)[0]
    xFs = np.asarray(xFs, float)
    xFs = np.ascontiguousarray(np.broadcast_to(xFs[:3], (B, 3)) if xFs.ndim == 1 else xFs.reshape(B, -1)[:, :3])
    o = _plan_call("obca_plan_parking_warmstart_goals", x0s, xFs, ox, oy, Ts, L, sampleN, cap, max_nodes, max_expansions, opts)
    full = np.nonzero(o["status"] == POOL_FULL)[0]
    if host_fallback and full.size:
        h = native.plan_cloud_raw(np.asarray(x0s, float)[full], xFs[full], ox, oy, Ts, L, sampleN, cap)
        for k in ("rx", "ry", "ryaw", "xWS", "uWS", "N", "status", "expansions"):
            o[k][full] = h[k]
    return o


def plan_goals_batch(x0s, xFs, ox, oy, Ts, L=2.7, sampleN=3, cap=512, max_nodes=0, opts=None):
    """native.plan_cloud_batch on the GPU: for every start pose x0s[i] and its goal xFs[i] ((B, >= 3), or one goal for all) among the
    cloud (ox, oy), the dictionary of plan_batch (None where no path was found).  Poses whose search outgrew the device's scratch
    (POOL_FULL) are planned by the host twin, which makes the same decisions; raises if a pose did not fit `cap`."""
    o = plan_goals_raw(x0s, xFs, ox, oy, Ts, L, sampleN, cap, max_nodes, 0, opts, host_fallback=True)
    st = o["status"]
    if (st > 1).any():
        raise native.PlannerError(f"obca_plan_parking_warmstart_goals: status {st[st > 1][:5]} at poses {np.nonzero(st > 1)[0][:5]}")
    return native.warm_starts(o, Ts)


def heuristic_maps(goals, ox, oy, opts=None):
    """The heuristic maps k_plan_hmap builds for the goals (G, >= 2) among the cloud, read back (obca_plan_parking_heuristic_maps):
    (maps (G, xw, yw), (minx, miny), device seconds of the kernel)."""
    g = np.ascontiguousarray(np.asarray(goals, float).reshape(len(goals), -1)[:, :2]); G = g.shape[0]
    ox = np.ascontiguousarray(ox, float); oy = np.ascontiguousarray(oy, float)
    mn = np.zeros(2, np.int64); w = np.zeros(2, np.int32); secs = C.c_double(0.0)
    p = _lib.ptr
    f = _lib.lib().obca_plan_parking_heuristic_maps
    f(G, p(g), p(ox), p(oy), int(ox.size), _lib.opts_arg(opts), p(mn), p(w), None, 0, None)      # reads the size
    m = np.zeros(G * int(w[0]) * int(w[1]))
    rc = f(G, p(g), p(ox), p(oy), int(ox.size), _lib.opts_arg(opts), p(mn), p(w), p(m), m.size, C.byref(secs))
    _lib.check(rc)
    return m.reshape(G, int(w[0]), int(w[1])), (int(mn[0]), int(mn[1])), secs.value


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
    p = _lib.ptr
    rc = _lib.lib().obca_plan_quadcopter_warmstart_batch(B, p(s), p(g), p(ox), p(oy), p(oz), int(ox.size), p(lo), p(hi), float(reso),
                                                         int(max_nodes), int(cap), _lib.opts_arg(opts),
                                                         *[p(o[k]) for k in ("rx", "ry", "rz", "N", "status", "expansions")], C.byref(secs))
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


_PK_SET = ("xp", "up", "ts", "lp", "np", "sl", "exitflag", "iters", "kkt_err", "feasible", "strict")
_QC_SET = ("xp", "up", "ts", "lp", "slack", "exitflag", "iters", "kkt_err", "feasible", "worst")


def _parking_flow_inputs(x0s, xFs, ox, oy, nOb, vOb, A, b):
    """The flow entries' parking inputs as contiguous arrays: x0s (B, 4), xFs (B, 4), ox, oy and the obstacles (vOb, V, A, b)."""
    from .._lib import f64
    from ..parking import _shared
    x0s = f64(np.asarray(x0s, float).reshape(-1, 4)); B = x0s.shape[0]
    xFs = f64(np.broadcast_to(np.asarray(xFs, float).reshape(-1, 4), (B, 4)))
    vOb, V, A, b = _shared(nOb, vOb, A, b)
    return x0s, xFs, f64(ox), f64(oy), vOb, V, A, b


def _parking_set(B, Ncap, V, nOb):
    """One formulation's output arrays of the parking flow for B poses, NaN-filled (the integers -1)."""
    NS = Ncap + 1
    nan = lambda *s: np.full(s, np.nan)
    i32 = lambda: np.full(B, -1, np.int32)
    return dict(xp=nan(B, NS, 4), up=nan(B, Ncap, 2), ts=nan(B, NS), lp=nan(B, NS, V), np=nan(B, NS, 4 * nOb), sl=nan(B, NS, nOb),
                exitflag=i32(), iters=i32(), kkt_err=nan(B), feasible=i32(), strict=i32())


def plan_solve_goals_raw(x0s, xFs, ox, oy, Ts, nOb, vOb, A, b, ego, XYbounds, L=2.7, sampleN=3, Ncap=319, fixTime=0, signed_dist=1,
                         max_nodes=0, max_expansions=0, opts=None, host_fallback=False):
    """obca_parking_plan_solve_goals's outputs as arrays: plan every start pose x0s (B, 4: x, y, yaw, v) towards its goal xFs ((B, 4), or
    (4,) for all), solve the poses that planned and check the results, in one call.  Per-pose arrays in the entry's layout for Ncap,
    row-major views of the column-major blocks: xp (B, Ncap+1, 4), up (B, Ncap, 2), ts (B, Ncap+1), lp (B, Ncap+1, V),
    np (B, Ncap+1, 4nOb), sl (B, Ncap+1, nOb); one value per pose: N, status, expansions, exitflag, iters, kkt_err, feasible, strict; and
    plan_seconds, time (the solve's device seconds).  The buffers start as NaN (the integers as -1): entries the call does not write stay
    so.  host_fallback: the poses whose search outgrew the device's scratch (POOL_FULL) are planned by the host twin (native.plan_cloud_raw,
    the same decisions), and those that plan to 2 <= N <= Ncap are solved and checked by parking_solve_mixed / check_parking_mixed in one
    more call each (their solve time is not in `time`), as plan_goals_raw(host_fallback=True) does for the planner alone."""
    from .._lib import f64
    x0s, xFs, ox, oy, vOb, V, A, b = _parking_flow_inputs(x0s, xFs, ox, oy, nOb, vOb, A, b)
    B = x0s.shape[0]
    i32 = lambda: np.full(B, -1, np.int32)
    o = dict(_parking_set(B, Ncap, V, nOb), N=i32(), status=i32(), expansions=i32())
    secs = np.zeros(2)
    p = _lib.ptr
    rc = _lib.lib().obca_parking_plan_solve_goals(
        B, p(x0s), p(xFs), p(ox), p(oy), int(ox.size), float(Ts), float(L), int(sampleN), int(max_expansions), int(max_nodes), int(nOb),
        p(vOb), p(A), p(b), p(f64(np.asarray(ego).ravel())), p(f64(np.asarray(XYbounds).ravel())), int(fixTime), int(signed_dist),
        _lib.opts_arg(opts), int(Ncap),
        *[p(o[k]) for k in ("xp", "up", "ts", "lp", "np", "sl", "N", "status", "expansions", "exitflag", "iters", "kkt_err", "feasible",
                            "strict")], p(secs[:1]), p(secs[1:]))
    _lib.check(rc)
    o["plan_seconds"], o["time"] = float(secs[0]), float(secs[1])
    full = np.flatnonzero(o["status"] == POOL_FULL)
    if host_fallback and full.size:
        h, ok = _plan_on_host(o, full, x0s, xFs, ox, oy, Ts, L, sampleN, Ncap)
        _solve_on_host_plans(o, full, h, ok, x0s, xFs, Ts, nOb, vOb, A, b, ego, XYbounds, L, fixTime, signed_dist, opts)
    return o


def plan_solve_goals_both_raw(x0s, xFs, ox, oy, Ts, nOb, vOb, A, b, ego, XYbounds, L=2.7, sampleN=3, Ncap=319, fixTime=0, max_nodes=0,
                              max_expansions=0, opts=None, host_fallback=False):
    """obca_parking_plan_solve_both's outputs as arrays: plan_solve_goals_raw's arguments without signed_dist; every pose is planned once,
    then solved and checked with the Distance and then the Signed Distance formulation.  Returns the shared N, status, expansions and
    plan_seconds, and under "dist" and "sd" the per-formulation keys of plan_solve_goals_raw (xp, up, ts, lp, np, sl, exitflag, iters,
    kkt_err, feasible, strict, time), each what plan_solve_goals_raw with signed_dist = 0 / 1 returns for the same inputs.
    host_fallback: the POOL_FULL poses are planned once by the host twin, then solved and checked with both formulations."""
    from .._lib import f64
    x0s, xFs, ox, oy, vOb, V, A, b = _parking_flow_inputs(x0s, xFs, ox, oy, nOb, vOb, A, b)
    B = x0s.shape[0]
    i32 = lambda: np.full(B, -1, np.int32)
    o = dict(N=i32(), status=i32(), expansions=i32(), dist=_parking_set(B, Ncap, V, nOb), sd=_parking_set(B, Ncap, V, nOb))
    secs = np.zeros(3)
    sets = [_lib.ParkingFlowOut(*[o[f][k].ctypes.data for k in _PK_SET], secs[j + 1:j + 2].ctypes.data) for j, f in enumerate(("dist", "sd"))]
    p = _lib.ptr
    rc = _lib.lib().obca_parking_plan_solve_both(
        B, p(x0s), p(xFs), p(ox), p(oy), int(ox.size), float(Ts), float(L), int(sampleN), int(max_expansions), int(max_nodes), int(nOb),
        p(vOb), p(A), p(b), p(f64(np.asarray(ego).ravel())), p(f64(np.asarray(XYbounds).ravel())), int(fixTime), _lib.opts_arg(opts),
        int(Ncap), p(o["N"]), p(o["status"]), p(o["expansions"]), p(secs[:1]), *[C.byref(s) for s in sets])
    _lib.check(rc)
    o["plan_seconds"] = float(secs[0])
    o["dist"]["time"], o["sd"]["time"] = float(secs[1]), float(secs[2])
    full = np.flatnonzero(o["status"] == POOL_FULL)
    if host_fallback and full.size:
        h, ok = _plan_on_host(o, full, x0s, xFs, ox, oy, Ts, L, sampleN, Ncap)
        for sd, f in ((0, "dist"), (1, "sd")):
            _solve_on_host_plans(o[f], full, h, ok, x0s, xFs, Ts, nOb, vOb, A, b, ego, XYbounds, L, fixTime, sd, opts)
    return o


def _plan_on_host(o, full, x0s, xFs, ox, oy, Ts, L, sampleN, Ncap):
    """Plan the poses `full` with the host twin; their status, N and expansions in o get its outputs (OBCA_PLAN_CAPACITY for a horizon
    outside [2, Ncap]).  Returns the host twin's outputs and the positions in `full` of the poses to solve."""
    h = native.plan_cloud_raw(x0s[full], xFs[full], ox, oy, Ts, L, sampleN)
    st = h["status"].copy()
    st[(st == 0) & ((h["N"] < 2) | (h["N"] > Ncap))] = 2
    o["status"][full] = st; o["N"][full] = h["N"]; o["expansions"][full] = h["expansions"]
    return h, np.flatnonzero(st == 0)


def _solve_on_host_plans(o, full, h, ok, x0s, xFs, Ts, nOb, vOb, A, b, ego, XYbounds, L, fixTime, signed_dist, opts):
    """Solve and check the poses full[ok] on the host twin's plans h (_plan_on_host) with one formulation; their entries of o (one
    formulation's arrays in the layout of plan_solve_goals_raw) get the results."""
    from .. import parking
    if ok.size == 0:
        return
    Ns = h["N"][ok]
    rx = [h["rx"][i, :n + 1] for i, n in zip(ok, Ns)]; ry = [h["ry"][i, :n + 1] for i, n in zip(ok, Ns)]
    ryaw = [h["ryaw"][i, :n + 1] for i, n in zip(ok, Ns)]
    xWS = [h["xWS"][i, :4 * (n + 1)].reshape(4, n + 1).T for i, n in zip(ok, Ns)]
    uWS = [h["uWS"][i, :2 * n].reshape(2, n).T for i, n in zip(ok, Ns)]
    x0, xF = x0s[full[ok]], xFs[full[ok]]
    r = parking.parking_solve_mixed(x0, xF, Ns, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS, signed_dist, opts=opts)
    feas, _, strict = parking.check_parking_mixed(x0, xF, Ns, Ts, L, ego, XYbounds, nOb, vOb, A, b, r["xp"], r["up"], r["lp"], r["np"], r["ts"],
                                                  fixTime, signed_dist, r["sl"], opts=opts)
    for q, (i, n) in enumerate(zip(full[ok], Ns)):
        for k, ext in (("xp", 1), ("up", 0), ("lp", 1), ("np", 1), ("sl", 1)):
            o[k][i, :n + ext] = r[k][q].T
        o["ts"][i, :n + 1] = r["ts"][q]
    for k, v in (("exitflag", r["exitflag"]), ("iters", r["iters"]), ("kkt_err", r["kkt_err"]), ("feasible", feas), ("strict", strict)):
        o[k][full[ok]] = v


def _parking_lists(o, ok, N):
    """One formulation's arrays of plan_solve_goals_raw as per-pose lists in the Julia shapes (None where ok[i] is False)."""
    cut = lambda a, ext: [a[i, :n + ext].T.copy() if ok[i] else None for i, n in enumerate(N)]
    out = dict(xp=cut(o["xp"], 1), up=cut(o["up"], 0), ts=[o["ts"][i, :n + 1].copy() if ok[i] else None for i, n in enumerate(N)],
               lp=cut(o["lp"], 1), np=cut(o["np"], 1), sl=cut(o["sl"], 1))
    for k in ("exitflag", "iters", "feasible", "strict"):
        out[k] = np.where(ok, o[k], 0).astype(np.int32)
    out.update(kkt_err=np.where(ok, o["kkt_err"], np.nan), time=o["time"])
    return out


def plan_solve_goals(x0s, xFs, ox, oy, Ts, nOb, vOb, A, b, ego, XYbounds, L=2.7, sampleN=3, Ncap=319, fixTime=0, signed_dist=1,
                     max_nodes=0, max_expansions=0, opts=None, host_fallback=False):
    """main.jl:215-269 for a batch in one call (obca_parking_plan_solve_goals): plan, solve and check every start pose x0s (B, 4) towards
    its goal xFs ((B, 4), or (4,) for all).  Returns the keys of parking.parking_solve_mixed in the caller's pose order -- per-pose lists
    in the Julia shapes (xp[i] 4 x (N[i]+1), up[i] 2 x N[i], ts[i], lp[i], np[i], sl[i]), None where the pose was not solved, and the
    arrays exitflag, iters, kkt_err, N, time -- plus status (OBCA_PLAN_* of include/obca.h: 0 solved, 1 no path, 2 horizon over Ncap,
    4 POOL_FULL: the search outgrew the device's scratch), expansions, feasible (ParkingConstraints' value), strict and plan_seconds.
    host_fallback: plan, solve and check the POOL_FULL poses on the host twin's plans (see plan_solve_goals_raw)."""
    o = plan_solve_goals_raw(x0s, xFs, ox, oy, Ts, nOb, vOb, A, b, ego, XYbounds, L, sampleN, Ncap, fixTime, signed_dist, max_nodes,
                             max_expansions, opts, host_fallback)
    out = _parking_lists(o, o["status"] == 0, o["N"])
    out.update(N=o["N"].copy(), status=o["status"].copy(), expansions=o["expansions"].copy(), plan_seconds=o["plan_seconds"])
    return out


def plan_solve_goals_both(x0s, xFs, ox, oy, Ts, nOb, vOb, A, b, ego, XYbounds, L=2.7, sampleN=3, Ncap=319, fixTime=0, max_nodes=0,
                          max_expansions=0, opts=None, host_fallback=False):
    """main.jl:215-269 as the reference runs it, for a batch in one call (obca_parking_plan_solve_both): every pose planned once, then
    solved and checked with ParkingDist and ParkingSignedDist.  Returns the shared N, status, expansions and plan_seconds, and under
    "dist" and "sd" the per-formulation keys of plan_solve_goals (per-pose lists in the Julia shapes, None where the pose was not solved,
    and exitflag, iters, kkt_err, feasible, strict, time)."""
    o = plan_solve_goals_both_raw(x0s, xFs, ox, oy, Ts, nOb, vOb, A, b, ego, XYbounds, L, sampleN, Ncap, fixTime, max_nodes, max_expansions,
                                  opts, host_fallback)
    ok = o["status"] == 0
    return dict(N=o["N"].copy(), status=o["status"].copy(), expansions=o["expansions"].copy(), plan_seconds=o["plan_seconds"],
                dist=_parking_lists(o["dist"], ok, o["N"]), sd=_parking_lists(o["sd"], ok, o["N"]))


def plan_solve_batch(x0s, xF, nOb, vOb, A, b, ego, XYbounds, scenario="backwards", Ts=None, L=2.7, sampleN=3, Ncap=319, **kw):
    """plan_solve_goals with one goal xF (4,) for every pose among the demo cloud of `scenario`, as plan_batch relates to
    plan_goals_batch: the sweeps of main.jl:165-168 planned, solved and checked in one call."""
    ox, oy = native.obstacle_points(scenario)
    Ts = Ts or (0.6 if scenario == "backwards" else 0.9) / 3 * sampleN
    return plan_solve_goals(x0s, np.asarray(xF, float)[:4], ox, oy, Ts, nOb, vOb, A, b, ego, XYbounds, L, sampleN, Ncap, **kw)


def _quadcopter_flow_inputs(x0s, xFs, ox, oy, oz, lo, hi, obs):
    """The flow entries' quadcopter inputs as contiguous arrays: x0s, xFs (B, 12), the cloud and bounds, and ob (5, 6)."""
    from .._lib import f64
    x0s = f64(np.asarray(x0s, float).reshape(-1, 12)); B = x0s.shape[0]
    xFs = f64(np.broadcast_to(np.asarray(xFs, float).reshape(-1, 12), (B, 12)))
    ox, oy, oz, lo, hi = (f64(np.asarray(a, float).ravel()) for a in (ox, oy, oz, lo, hi))
    return x0s, xFs, ox, oy, oz, lo, hi, f64(np.asarray(obs, float).reshape(5, 6))


def _quadcopter_set(B, Ncap):
    """One formulation's output arrays of the quadcopter flow for B pairs, NaN-filled (the integers -1)."""
    NS = Ncap + 1
    nan = lambda *s: np.full(s, np.nan)
    i32 = lambda: np.full(B, -1, np.int32)
    return dict(xp=nan(B, NS, 12), up=nan(B, Ncap, 4), ts=nan(B, NS), lp=nan(B, NS, 30), slack=nan(B, NS, 5), exitflag=i32(), iters=i32(),
                kkt_err=nan(B), feasible=i32(), worst=nan(B))


def plan_solve_quadcopter_raw(x0s, xFs, ox, oy, oz, lo, hi, reso, Ts, R, obs, timeWS=1.0, signed_dist=1, Ncap=511, max_nodes=0,
                              opts=None, host_fallback=False):
    """obca_quadcopter_plan_solve's outputs as arrays: plan every pair x0s[i] -> xFs[i] ((B, 12) in the solve's units; the planner takes
    10 x rows 0-2) among the cloud (ox, oy, oz, lo, hi, reso in the planner's units), build the warm starts, solve the pairs that
    planned and check the results, in one call.  Per-pair arrays in the entry's layout for Ncap, row-major views of the column-major
    blocks: xp (B, Ncap+1, 12), up (B, Ncap, 4), ts (B, Ncap+1), lp (B, Ncap+1, 30), slack (B, Ncap+1, 5); one value per pair: N, Tsb,
    status, expansions, exitflag, iters, kkt_err, feasible, worst; and plan_seconds, time (the solve's device seconds).  The buffers start
    as NaN (the integers as -1): entries the call does not write stay so.  opts None: defaults with max_iter = 3000, as
    quadcopter.quadcopter_solve_mixed.  host_fallback: the pairs whose search outgrew the device's scratch (POOL_FULL) are planned by the
    host library (native.astar3d_raw, the same decisions), and those that plan to 2 <= N <= Ncap get their warm starts from
    native.quadcopter_warm_start and are solved and checked by quadcopter_solve_mixed / check_quadcopter_mixed in one more call each
    (their solve time is not in `time`)."""
    x0s, xFs, ox, oy, oz, lo, hi, ob = _quadcopter_flow_inputs(x0s, xFs, ox, oy, oz, lo, hi, obs)
    B = x0s.shape[0]
    i32 = lambda: np.full(B, -1, np.int32)
    o = dict(_quadcopter_set(B, Ncap), N=i32(), Tsb=np.full(B, np.nan), status=i32(), expansions=i32())
    secs = np.zeros(2)
    p = _lib.ptr
    rc = _lib.lib().obca_quadcopter_plan_solve(
        B, p(x0s), p(xFs), p(ox), p(oy), p(oz), int(ox.size), p(lo), p(hi), float(reso), int(max_nodes), float(Ts), float(R), p(ob),
        float(timeWS), int(signed_dist), _lib.opts_arg(opts), int(Ncap),
        *[p(o[k]) for k in ("xp", "up", "ts", "lp", "slack", "N", "Tsb", "status", "expansions", "exitflag", "iters", "kkt_err",
                            "feasible", "worst")], p(secs[:1]), p(secs[1:]))
    _lib.check(rc)
    o["plan_seconds"], o["time"] = float(secs[0]), float(secs[1])
    full = np.flatnonzero(o["status"] == POOL_FULL)
    if host_fallback and full.size:
        ws = _plan_quadcopter_on_host(o, full, x0s, xFs, ox, oy, oz, lo, hi, reso, Ts, Ncap)
        _solve_quadcopter_on_host_plans(o, full, ws, x0s, xFs, R, obs, timeWS, signed_dist, opts)
    return o


def plan_solve_quadcopter_both_raw(x0s, xFs, ox, oy, oz, lo, hi, reso, Ts, R, obs, timeWS=1.0, Ncap=511, max_nodes=0, opts=None,
                                   host_fallback=False):
    """obca_quadcopter_plan_solve_both's outputs as arrays: plan_solve_quadcopter_raw's arguments without signed_dist; every pair is
    planned and warm-started once, then solved and checked with the Distance and then the Signed Distance formulation.  Returns the
    shared N, Tsb, status, expansions and plan_seconds, and under "dist" and "sd" the per-formulation keys of plan_solve_quadcopter_raw
    (xp, up, ts, lp, slack, exitflag, iters, kkt_err, feasible, worst, time), each what plan_solve_quadcopter_raw with signed_dist = 0 / 1
    returns for the same inputs (the Dist set's slack is never written).  host_fallback: the POOL_FULL pairs are planned once by the host
    library, then solved and checked with both formulations."""
    x0s, xFs, ox, oy, oz, lo, hi, ob = _quadcopter_flow_inputs(x0s, xFs, ox, oy, oz, lo, hi, obs)
    B = x0s.shape[0]
    i32 = lambda: np.full(B, -1, np.int32)
    o = dict(N=i32(), Tsb=np.full(B, np.nan), status=i32(), expansions=i32(), dist=_quadcopter_set(B, Ncap), sd=_quadcopter_set(B, Ncap))
    secs = np.zeros(3)
    sets = [_lib.QuadcopterFlowOut(*[o[f][k].ctypes.data for k in _QC_SET], secs[j + 1:j + 2].ctypes.data)
            for j, f in enumerate(("dist", "sd"))]
    p = _lib.ptr
    rc = _lib.lib().obca_quadcopter_plan_solve_both(
        B, p(x0s), p(xFs), p(ox), p(oy), p(oz), int(ox.size), p(lo), p(hi), float(reso), int(max_nodes), float(Ts), float(R), p(ob),
        float(timeWS), _lib.opts_arg(opts), int(Ncap), p(o["N"]), p(o["Tsb"]), p(o["status"]), p(o["expansions"]), p(secs[:1]),
        *[C.byref(s) for s in sets])
    _lib.check(rc)
    o["plan_seconds"] = float(secs[0])
    o["dist"]["time"], o["sd"]["time"] = float(secs[1]), float(secs[2])
    full = np.flatnonzero(o["status"] == POOL_FULL)
    if host_fallback and full.size:
        ws = _plan_quadcopter_on_host(o, full, x0s, xFs, ox, oy, oz, lo, hi, reso, Ts, Ncap)
        for sd, f in ((0, "dist"), (1, "sd")):
            _solve_quadcopter_on_host_plans(o[f], full, ws, x0s, xFs, R, obs, timeWS, sd, opts)
    return o


def _plan_quadcopter_on_host(o, full, x0s, xFs, ox, oy, oz, lo, hi, reso, Ts, Ncap):
    """Plan the pairs `full` with the host library and build the warm starts of the ones it plans to 2 <= N <= Ncap; their status, N,
    expansions and Tsb in o get its outputs (OBCA_PLAN_CAPACITY for a horizon outside [2, Ncap]).  Returns the positions in `full` of the
    pairs to solve, their horizons and their warm starts (native.quadcopter_warm_start)."""
    h = native.astar3d_raw(x0s[full, :3] * 10.0, xFs[full, :3] * 10.0, ox, oy, oz, lo, hi, reso, Ncap + 1)
    st = h["status"].copy()
    st[(st == 0) & (h["N"] < 2)] = 2
    o["status"][full] = st; o["N"][full] = h["N"]; o["expansions"][full] = h["expansions"]
    ok = np.flatnonzero(st == 0)
    Ns = h["N"][ok]
    ws = [native.quadcopter_warm_start(h["rx"][i, :n + 1].copy(), h["ry"][i, :n + 1].copy(), h["rz"][i, :n + 1].copy(), Ts)
          for i, n in zip(ok, Ns)]
    o["Tsb"][full[ok]] = [w["Ts"] for w in ws]
    return ok, Ns, ws


def _solve_quadcopter_on_host_plans(o, full, plans, x0s, xFs, R, obs, timeWS, signed_dist, opts):
    """Solve and check the pairs of `plans` (_plan_quadcopter_on_host) with one formulation; their entries of o (one formulation's arrays
    in the layout of plan_solve_quadcopter_raw) get the results."""
    from .. import quadcopter
    ok, Ns, ws = plans
    if ok.size == 0:
        return
    Tsb = np.array([w["Ts"] for w in ws])
    x0, xF = x0s[full[ok]], xFs[full[ok]]
    r = quadcopter.quadcopter_solve_mixed(x0, xF, Ns, Tsb, R, obs, [w["xWS"] for w in ws], timeWS, signed_dist, opts=opts)
    feas, worst = quadcopter.check_quadcopter_mixed(r["xp"], r["up"], r["ts"], x0, xF, Ns, Tsb, r["lp"], obs, R, opts=opts)
    for q, (i, n) in enumerate(zip(full[ok], Ns)):
        for k, ext in (("xp", 1), ("up", 0), ("lp", 1)) + ((("slack", 1),) if signed_dist else ()):
            o[k][i, :n + ext] = r[k][q].T
        o["ts"][i, :n + 1] = r["ts"][q]
    for k, v in (("exitflag", r["exitflag"]), ("iters", r["iters"]), ("kkt_err", r["kkt_err"]), ("feasible", feas), ("worst", worst)):
        o[k][full[ok]] = v


def _quadcopter_lists(o, ok, N, signed_dist):
    """One formulation's arrays of plan_solve_quadcopter_raw as per-pair lists in the Julia shapes (None where ok[i] is False)."""
    cut = lambda a, ext: [a[i, :n + ext].T.copy() if ok[i] else None for i, n in enumerate(N)]
    out = dict(xp=cut(o["xp"], 1), up=cut(o["up"], 0), ts=[o["ts"][i, :n + 1].copy() if ok[i] else None for i, n in enumerate(N)],
               lp=cut(o["lp"], 1), slack=cut(o["slack"], 1) if signed_dist else [None] * len(ok))
    for k in ("exitflag", "iters", "feasible"):
        out[k] = np.where(ok, o[k], 0).astype(np.int32)
    out.update(kkt_err=np.where(ok, o["kkt_err"], np.nan), worst=np.where(ok, o["worst"], np.nan), time=o["time"])
    return out


def plan_solve_quadcopter(x0s, xFs, R, obs, Ts=0.25, signed_dist=1, Ncap=511, max_nodes=0, opts=None, host_fallback=False):
    """mainQuadcopter.jl:114-154 for a batch in one call (obca_quadcopter_plan_solve): plan every start / goal pair (x0s, xFs (B, 12))
    among the environment of a_star_3d.quadcopter_environment() (reso = 1), build the warm starts, solve and check.  Returns the keys of
    quadcopter.quadcopter_solve_mixed in the caller's pair order -- per-pair lists in the Julia shapes (xp[i] 12 x (N[i]+1), up[i]
    4 x N[i], ts[i], lp[i] 30 x (N[i]+1), slack[i] 5 x (N[i]+1), the last for signed_dist = 1 only), None where the pair was not solved,
    and the arrays exitflag, iters, kkt_err, N, Ts (the pairs' sampling times), time -- plus status (OBCA_PLAN_* of include/obca.h:
    0 solved, 1 no path, 2 horizon outside [2, Ncap], 4 POOL_FULL: the search outgrew the device's scratch), expansions, feasible
    (constrSatisfaction's value), worst and plan_seconds.  host_fallback: plan, solve and check the POOL_FULL pairs on the host library's
    plans (see plan_solve_quadcopter_raw)."""
    from .a_star_3d import quadcopter_environment
    ox, oy, oz, lo, hi = quadcopter_environment()
    o = plan_solve_quadcopter_raw(x0s, xFs, ox, oy, oz, lo, hi, 1.0, Ts, R, obs, 1.0, signed_dist, Ncap, max_nodes, opts, host_fallback)
    ok = o["status"] == 0
    out = _quadcopter_lists(o, ok, o["N"], signed_dist)
    out.update(N=o["N"].copy(), Ts=np.where(ok, o["Tsb"], np.nan), status=o["status"].copy(), expansions=o["expansions"].copy(),
               plan_seconds=o["plan_seconds"])
    return out


def plan_solve_quadcopter_both(x0s, xFs, R, obs, Ts=0.25, Ncap=511, max_nodes=0, opts=None, host_fallback=False):
    """mainQuadcopter.jl:114-154 as the reference runs it, for a batch in one call (obca_quadcopter_plan_solve_both): every pair planned
    and warm-started once, then solved and checked with QuadcopterDist and QuadcopterSignedDist.  Returns the shared N, Ts, status,
    expansions and plan_seconds, and under "dist" and "sd" the per-formulation keys of plan_solve_quadcopter (per-pair lists in the Julia
    shapes, None where the pair was not solved -- slack for "sd" only --, and exitflag, iters, kkt_err, feasible, worst, time)."""
    from .a_star_3d import quadcopter_environment
    ox, oy, oz, lo, hi = quadcopter_environment()
    o = plan_solve_quadcopter_both_raw(x0s, xFs, ox, oy, oz, lo, hi, 1.0, Ts, R, obs, 1.0, Ncap, max_nodes, opts, host_fallback)
    ok = o["status"] == 0
    return dict(N=o["N"].copy(), Ts=np.where(ok, o["Tsb"], np.nan), status=o["status"].copy(), expansions=o["expansions"].copy(),
                plan_seconds=o["plan_seconds"], dist=_quadcopter_lists(o["dist"], ok, o["N"], 0),
                sd=_quadcopter_lists(o["sd"], ok, o["N"], 1))
