"""Host-side mirror of the reference's parking NLP drivers, same names / argument order / return tuples:

    ParkingSignedDist   AutonomousParking/ParkingSignedDist.jl:29   -> (xp, up, timeScalep, exitflag, time, lp, np) :313
    ParkingDist         AutonomousParking/ParkingDist.jl:29         -> same 7-tuple :313
    DualMultWS          AutonomousParking/DualMultWS.jl:29          -> (lp, np) :86
    ParkingConstraints  AutonomousParking/ParkingConstraints.jl:29  -> 0/1 :143-147

Julia is not installed in this image, so the host side above the C-ABI is Python (ctypes) instead of the Julia
shims in julia/ (INTEGRATION.md); numpy arrays carry the same shapes the Julia caller uses (x0, xF 1x4 rows,
vOb = half-space counts, xWS (N+1)x4, uWS >= N rows).  All computation happens in libobca.so on the GPU.
Failure is reported the reference's way: exitflag 0, never an exception for a non-converged solve.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from ._lib import opts_arg, check, f64, lib, ptr

ego = None   # DualMultWS reads a global `ego` in the reference (DualMultWS.jl:39); set obca_b200.parking.ego


def _shared(nOb, vOb, A, b):
    vOb = np.ascontiguousarray(np.asarray(vOb).ravel(), dtype=np.int32)
    assert len(vOb) == nOb
    V = int(vOb.sum())
    A = np.asfortranarray(np.asarray(A, dtype=np.float64).reshape(V, 2))
    b = f64(np.asarray(b).ravel())
    return vOb, V, A, b


def parking_solve_batch(x0, xF, N, Ts, L, ego_, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS,
                        signed_dist=1, lWS=None, nWS=None, opts=None):
    """Batched driver.  x0 (B,4); xF (4,) or (B,4); rx, ry, ryaw (B,N+1); xWS (B,N+1,4); uWS (B,>=N,2);
    optional lWS (B,N+1,V), nWS (B,N+1,4nOb).  Returns dict with Julia-shaped stacks:
    xp (B,4,N+1), up (B,2,N), ts (B,N+1), lp (B,V,N+1), np (B,4nOb,N+1), sl (B,nOb,N+1), exitflag, iters, kkt_err, time."""
    x0 = f64(np.atleast_2d(x0)); B = x0.shape[0]
    NS = N + 1
    vOb, V, A, b = _shared(nOb, vOb, A, b)
    xF = f64(np.broadcast_to(np.asarray(xF, dtype=np.float64).reshape(-1, 4), (B, 4)))
    rx = f64(np.asarray(rx).reshape(B, NS)); ry = f64(np.asarray(ry).reshape(B, NS)); ryaw = f64(np.asarray(ryaw).reshape(B, NS))
    xWS = f64(np.transpose(np.asarray(xWS, dtype=np.float64).reshape(B, -1, 4)[:, :NS, :], (0, 2, 1)))   # column-major (N+1)x4
    uWS = f64(np.transpose(np.asarray(uWS, dtype=np.float64).reshape(B, -1, 2)[:, :N, :], (0, 2, 1)))    # uWS[1:N,:] (:217)
    lW = nW = None
    if lWS is not None:
        lW = f64(np.transpose(np.asarray(lWS, dtype=np.float64).reshape(B, NS, V), (0, 2, 1)))
        nW = f64(np.transpose(np.asarray(nWS, dtype=np.float64).reshape(B, NS, 4 * nOb), (0, 2, 1)))
    xp = np.zeros((B, NS, 4)); up = np.zeros((B, N, 2)); ts = np.zeros((B, NS))
    lp = np.zeros((B, NS, V)); npp = np.zeros((B, NS, 4 * nOb)); sl = np.zeros((B, NS, nOb))
    ef = np.zeros(B, np.int32); it = np.zeros(B, np.int32); err = np.zeros(B); sec = np.zeros(1)
    check(lib().obca_parking_solve_batch(
        B, N, nOb, ptr(vOb), ptr(A), ptr(b), ptr(x0), ptr(xF), float(Ts), float(L), ptr(f64(np.asarray(ego_).ravel())),
        ptr(f64(np.asarray(XYbounds).ravel())), ptr(rx), ptr(ry), ptr(ryaw), ptr(xWS), ptr(uWS), ptr(lW), ptr(nW), int(fixTime),
        int(signed_dist), opts_arg(opts), ptr(xp), ptr(up), ptr(ts), ptr(lp), ptr(npp), ptr(sl), ptr(ef), ptr(it), ptr(err), ptr(sec)))
    T = lambda a: np.transpose(a, (0, 2, 1))
    return dict(xp=T(xp), up=T(up), ts=ts, lp=T(lp), np=T(npp), sl=T(sl), exitflag=ef, iters=it, kkt_err=err,
                time=float(sec[0]))


def _pad_stages(arrs, Nmax):
    """Per-problem arrays with their stages along axis 0 (lengths may differ) -> (B, Nmax+1, ...) zero-padded."""
    first = np.asarray(arrs[0], dtype=np.float64)
    out = np.zeros((len(arrs), Nmax + 1) + first.shape[1:])
    for i, a in enumerate(arrs):
        a = np.asarray(a, dtype=np.float64)
        out[i, :a.shape[0]] = a
    return out


def parking_solve_mixed(x0, xF, Ns, Ts, L, ego_, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS,
                        signed_dist=1, lWS=None, nWS=None, opts=None):
    """One batched solve of problems with different horizons Ns[i] (obca_parking_solve_mixed).  x0 (B,4); xF (4,) or
    (B,4); per-problem lists: rx[i], ry[i], ryaw[i] of length Ns[i]+1, xWS[i] (Ns[i]+1,4), uWS[i] with >= Ns[i] rows,
    optional lWS[i] (Ns[i]+1,V), nWS[i] (Ns[i]+1,4nOb).  Problem i gives exactly what parking_solve_batch gives it at
    N = Ns[i].  Returns dict of per-problem lists in the Julia shapes (xp[i] 4x(Ns[i]+1), up[i] 2xNs[i], ts[i] Ns[i]+1,
    lp[i] Vx(Ns[i]+1), np[i] 4nOb x(Ns[i]+1), sl[i] nOb x(Ns[i]+1)), the arrays exitflag, iters, kkt_err, N, and time."""
    Ns = np.ascontiguousarray(np.asarray(Ns).ravel(), dtype=np.int32)
    x0 = f64(np.atleast_2d(x0)); B = x0.shape[0]
    assert len(Ns) == B
    Nmax = int(Ns.max()); NS = Nmax + 1
    vOb, V, A, b = _shared(nOb, vOb, A, b)
    xF = f64(np.broadcast_to(np.asarray(xF, dtype=np.float64).reshape(-1, 4), (B, 4)))
    rx = f64(_pad_stages([np.ravel(r)[:n + 1] for r, n in zip(rx, Ns)], Nmax))
    ry = f64(_pad_stages([np.ravel(r)[:n + 1] for r, n in zip(ry, Ns)], Nmax))
    ryaw = f64(_pad_stages([np.ravel(r)[:n + 1] for r, n in zip(ryaw, Ns)], Nmax))
    T = lambda a: f64(np.transpose(a, (0, 2, 1)))
    xW = T(_pad_stages([np.asarray(w, float).reshape(-1, 4)[:n + 1] for w, n in zip(xWS, Ns)], Nmax))
    uW = T(_pad_stages([np.asarray(w, float).reshape(-1, 2)[:n] for w, n in zip(uWS, Ns)], Nmax)[:, :Nmax])
    lW = nW = None
    if lWS is not None:
        lW = T(_pad_stages([np.asarray(w, float).reshape(-1, V)[:n + 1] for w, n in zip(lWS, Ns)], Nmax))
        nW = T(_pad_stages([np.asarray(w, float).reshape(-1, 4 * nOb)[:n + 1] for w, n in zip(nWS, Ns)], Nmax))
    xp = np.zeros((B, NS, 4)); up = np.zeros((B, Nmax, 2)); ts = np.zeros((B, NS))
    lp = np.zeros((B, NS, V)); npp = np.zeros((B, NS, 4 * nOb)); sl = np.zeros((B, NS, nOb))
    ef = np.zeros(B, np.int32); it = np.zeros(B, np.int32); err = np.zeros(B); sec = np.zeros(1)
    check(lib().obca_parking_solve_mixed(
        B, ptr(Ns), Nmax, nOb, ptr(vOb), ptr(A), ptr(b), ptr(x0), ptr(xF), float(Ts), float(L), ptr(f64(np.asarray(ego_).ravel())),
        ptr(f64(np.asarray(XYbounds).ravel())), ptr(rx), ptr(ry), ptr(ryaw), ptr(xW), ptr(uW), ptr(lW), ptr(nW), int(fixTime),
        int(signed_dist), opts_arg(opts), ptr(xp), ptr(up), ptr(ts), ptr(lp), ptr(npp), ptr(sl), ptr(ef), ptr(it), ptr(err), ptr(sec)))
    cut = lambda a, ext: [a[i, :n + ext].T.copy() for i, n in enumerate(Ns)]
    return dict(xp=cut(xp, 1), up=cut(up, 0), ts=[ts[i, :n + 1].copy() for i, n in enumerate(Ns)], lp=cut(lp, 1),
                np=cut(npp, 1), sl=cut(sl, 1), exitflag=ef, iters=it, kkt_err=err, N=Ns.copy(), time=float(sec[0]))


def _single(signed_dist, x0, xF, N, Ts, L, ego_, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS):
    r = parking_solve_batch(np.asarray(x0, float).reshape(1, 4), np.asarray(xF, float).reshape(1, 4), N, Ts, L, ego_,
                            XYbounds, nOb, vOb, A, b, np.asarray(rx, float).reshape(1, -1),
                            np.asarray(ry, float).reshape(1, -1), np.asarray(ryaw, float).reshape(1, -1), fixTime,
                            np.asarray(xWS, float)[None], np.asarray(uWS, float)[None], signed_dist)
    tsp = np.ones((1, N + 1)) if fixTime else r["ts"][0].copy()        # ParkingSignedDist.jl:304-308
    return r["xp"][0], r["up"][0], tsp, int(r["exitflag"][0]), r["time"], r["lp"][0], r["np"][0]


def ParkingSignedDist(x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS):
    return _single(1, x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS)


def ParkingDist(x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS):
    return _single(0, x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS)


def dualmultws_batch(N, nOb, vOb, A, b, rx, ry, ryaw, ego_, opts=None, want_d=False):
    rx = f64(np.atleast_2d(rx)); B = rx.shape[0]; NS = N + 1
    ry = f64(np.atleast_2d(ry)); ryaw = f64(np.atleast_2d(ryaw))
    vOb, V, A, b = _shared(nOb, vOb, A, b)
    lp = np.zeros((B, V, NS)); npp = np.zeros((B, 4 * nOb, NS)); d = np.zeros((B, nOb, NS))
    check(lib().obca_dualmultws_batch(B, N, nOb, ptr(vOb), ptr(A), ptr(b), ptr(f64(np.asarray(ego_).ravel())), ptr(rx), ptr(ry),
                                      ptr(ryaw), opts_arg(opts), ptr(lp), ptr(npp), ptr(d)))
    T = lambda a: np.transpose(a, (0, 2, 1)).copy()
    return (T(lp), T(npp), T(d)) if want_d else (T(lp), T(npp))


def DualMultWS(N, nOb, vOb, A, b, rx, ry, ryaw):
    """DualMultWS.jl:29 -- returns lp (N+1)xsum(vOb), np (N+1)x4nOb.  Uses the module-level `ego` like the reference."""
    if ego is None:
        raise NameError("ego not defined (DualMultWS.jl:39 reads the global `ego`): set obca_b200.parking.ego")
    lp, npp = dualmultws_batch(N, nOb, vOb, A, b, np.asarray(rx, float).reshape(1, -1),
                               np.asarray(ry, float).reshape(1, -1), np.asarray(ryaw, float).reshape(1, -1), ego)
    return lp[0], npp[0]


def check_parking_batch(x0, xF, N, Ts, L, ego_, XYbounds, nOb, vOb, A, b, x, u, l, n, timeScale, fixTime, sd,
                        sl=None, opts=None):
    """x (B,4,N+1), u (B,2,N), l (B,V,N+1), n (B,4nOb,N+1), timeScale (B,N+1) -- Julia shapes, stacked."""
    x = np.asarray(x, float); B = x.shape[0]; NS = N + 1
    vOb, V, A, b = _shared(nOb, vOb, A, b)
    T = lambda a: f64(np.transpose(np.asarray(a, float), (0, 2, 1)))
    xx, uu, ll, nn = T(x), T(u), T(l), T(n)
    tt = f64(np.asarray(timeScale, float).reshape(B, NS))
    ss = T(sl) if sl is not None else None
    x0 = f64(np.broadcast_to(np.asarray(x0, float).reshape(-1, 4), (B, 4)))
    xF = f64(np.broadcast_to(np.asarray(xF, float).reshape(-1, 4), (B, 4)))
    feas = np.zeros(B, np.int32); e = np.zeros((B, 7), np.int32); strict = np.zeros(B, np.int32)
    check(lib().obca_check_parking(B, N, nOb, ptr(vOb), ptr(A), ptr(b), ptr(x0), ptr(xF), float(Ts), float(L),
                                   ptr(f64(np.asarray(ego_).ravel())), ptr(f64(np.asarray(XYbounds).ravel())), ptr(xx), ptr(uu),
                                   ptr(ll), ptr(nn), ptr(tt), ptr(ss), int(fixTime), int(sd), opts_arg(opts), ptr(feas), ptr(e),
                                   ptr(strict)))
    return feas, e, strict


def check_parking_mixed(x0, xF, Ns, Ts, L, ego_, XYbounds, nOb, vOb, A, b, x, u, l, n, timeScale, fixTime, sd, sl=None,
                        opts=None):
    """check_parking_batch over problems with different horizons Ns[i] (obca_check_parking_mixed): per-problem lists
    x[i] 4x(Ns[i]+1), u[i] 2xNs[i], l[i] Vx(Ns[i]+1), n[i] 4nOb x(Ns[i]+1), timeScale[i] Ns[i]+1, sl[i] nOb x(Ns[i]+1)."""
    Ns = np.ascontiguousarray(np.asarray(Ns).ravel(), dtype=np.int32)
    B = len(Ns); Nmax = int(Ns.max())
    vOb, V, A, b = _shared(nOb, vOb, A, b)
    P = lambda arrs, ext: f64(_pad_stages([np.asarray(a, float).T[:k + ext] for a, k in zip(arrs, Ns)], Nmax))
    xx, ll, nn = P(x, 1), P(l, 1), P(n, 1)
    uu = f64(P(u, 0)[:, :Nmax])          # (a slice: contiguous again before its pointer is taken)
    tt = f64(_pad_stages([np.ravel(t)[:k + 1] for t, k in zip(timeScale, Ns)], Nmax))
    ss = P(sl, 1) if sl is not None else None
    x0 = f64(np.broadcast_to(np.asarray(x0, float).reshape(-1, 4), (B, 4)))
    xF = f64(np.broadcast_to(np.asarray(xF, float).reshape(-1, 4), (B, 4)))
    feas = np.zeros(B, np.int32); e = np.zeros((B, 7), np.int32); strict = np.zeros(B, np.int32)
    check(lib().obca_check_parking_mixed(B, ptr(Ns), Nmax, nOb, ptr(vOb), ptr(A), ptr(b), ptr(x0), ptr(xF), float(Ts), float(L),
                                         ptr(f64(np.asarray(ego_).ravel())), ptr(f64(np.asarray(XYbounds).ravel())), ptr(xx),
                                         ptr(uu), ptr(ll), ptr(nn), ptr(tt), ptr(ss), int(fixTime), int(sd), opts_arg(opts), ptr(feas),
                                         ptr(e), ptr(strict)))
    return feas, e, strict


def ParkingConstraints(x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, x, u, l, n, timeScale, fixTime, sd):
    feas, _, _ = check_parking_batch(x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, np.asarray(x, float)[None],
                                     np.asarray(u, float)[None], np.asarray(l, float)[None],
                                     np.asarray(n, float)[None], np.asarray(timeScale, float).reshape(1, -1), fixTime, sd)
    return int(feas[0])


def eval_batch(x0, xF, N, Ts, L, ego_, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, signed_dist, xp, up, ts, lp, np_, sl=None,
               y=None, reps=1, opts=None):
    """K1 stand-alone (obca_parking_eval_batch_dev): fused evaluation of the reference NLP at B points.
    xp (B,4,N+1), up (B,2,N), ts (B,N+1), lp (B,V,N+1), np_ (B,4nOb,N+1), sl (B,nOb,N+1) -- Julia shapes, stacked;
    y (B,m) row multipliers in the K1 row order (include/obca.h) or None.  Device buffers are torch tensors
    (plumbing only).  Returns c (B,m), gradL (B,n), f (B,), kernel_ms."""
    import torch
    xp = np.asarray(xp, float); B = xp.shape[0]; NS = N + 1
    vOb, V, A, b = _shared(nOb, vOb, A, b)
    nn = C.c_longlong(); mm = C.c_longlong()
    check(lib().obca_parking_eval_sizes(N, nOb, ptr(vOb), int(signed_dist), C.byref(nn), C.byref(mm)))
    n, m = nn.value, mm.value
    o = opts if opts is not None else _lib.default_opts()
    dev = torch.device("cuda", o.device)
    T = lambda a: np.ascontiguousarray(np.transpose(np.asarray(a, float), (0, 2, 1)))
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).to(dev)
    bx0 = d(np.broadcast_to(np.asarray(x0, float).reshape(-1, 4), (B, 4))); bxF = d(np.broadcast_to(np.asarray(xF, float).reshape(-1, 4), (B, 4)))
    brx, bry, bryaw = d(np.asarray(rx).reshape(B, NS)), d(np.asarray(ry).reshape(B, NS)), d(np.asarray(ryaw).reshape(B, NS))
    dxp, dup, dlp, dnp = d(T(xp)), d(T(up)), d(T(lp)), d(T(np_))
    dts = d(np.asarray(ts, float).reshape(B, NS)) if ts is not None else None
    dsl = d(T(sl)) if sl is not None else None
    dy = d(np.asarray(y, float).reshape(B, m)) if y is not None else None
    c = torch.zeros((B, m), dtype=torch.float64, device=dev); g = torch.zeros((B, n), dtype=torch.float64, device=dev)
    fk = torch.zeros((B, NS), dtype=torch.float64, device=dev)
    ms = np.zeros(1)
    P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    torch.cuda.synchronize(dev)      # the library launches on its own stream: torch's copies / fills must have landed first
    check(lib().obca_parking_eval_batch_dev(
        B, N, nOb, ptr(vOb), ptr(A), ptr(b), P(bx0), P(bxF), float(Ts), float(L), ptr(f64(np.asarray(ego_).ravel())),
        ptr(f64(np.asarray(XYbounds).ravel())), P(brx), P(bry), P(bryaw), P(dxp), P(dup), P(dts), P(dlp), P(dnp), P(dsl), P(dy),
        int(fixTime), int(signed_dist), C.byref(o), P(c), P(g), P(fk), int(reps), ptr(ms)))
    return c.cpu().numpy(), g.cpu().numpy(), fk.sum(1).cpu().numpy(), float(ms[0])


def parking_solve_planned(x0s, xF, plans, Ts, L, ego_, XYbounds, nOb, vOb, A, b, fixTime=0, signed_dist=1, opts=None,
                          solve=None):
    """Solve problems whose warm starts came from the Hybrid A* producer (obca_b200.planner.warmstart.plan_batch): their horizons
    differ; this path groups the problems by N, every group goes through parking_solve_batch (parking_solve_mixed does the
    same in one call, with the same bits per problem), and the results come back in the caller's order (lists of per-problem arrays in the Julia shapes
    4 x (N_i+1), 2 x N_i, ...; None where the planner found no path).  `solve`: injection point for tests."""
    from .planner.warmstart import group_by_horizon
    solve = solve or parking_solve_batch
    x0s = np.asarray(x0s, float).reshape(-1, 4)
    out = dict(xp=[None] * len(plans), up=[None] * len(plans), ts=[None] * len(plans), lp=[None] * len(plans), np=[None] * len(plans),
               exitflag=np.zeros(len(plans), np.int32), iters=np.zeros(len(plans), np.int32), N=np.zeros(len(plans), np.int32), time=0.0)
    for N, idx in group_by_horizon(plans).items():
        g = [plans[i] for i in idx]
        r = solve(x0s[idx], xF, N, Ts, L, ego_, XYbounds, nOb, vOb, A, b, np.stack([w["rx"] for w in g]), np.stack([w["ry"] for w in g]),
                  np.stack([w["ryaw"] for w in g]), fixTime, np.stack([w["xWS"] for w in g]), np.stack([w["uWS"][:N] for w in g]),
                  signed_dist, None, None, opts)
        for k, i in enumerate(idx):
            for key in ("xp", "up", "ts", "lp", "np"):
                out[key][i] = r[key][k]
            out["exitflag"][i] = r["exitflag"][k]; out["iters"][i] = r["iters"][k]; out["N"][i] = N
        out["time"] += float(r["time"])
    return out
