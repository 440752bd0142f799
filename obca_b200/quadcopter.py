"""Host-side mirror of the reference's quadcopter NLP drivers, same names / argument order / return tuples:

    QuadcopterSignedDist  QuadcopterNavigation/QuadcopterSignedDist.jl:25 -> (xp, up, timeScalep, exitflag, time, lp, status) :298
    QuadcopterDist        QuadcopterNavigation/QuadcopterDist.jl:25       -> same 7-tuple :280
    constrSatisfaction    QuadcopterNavigation/constrSatisfaction.jl:25   -> Bool

All computation happens in libobca.so on the GPU (obca_quadcopter_solve_batch / obca_check_quadcopter, and their _mixed
twins for a batch whose problems have their own horizon and sampling time)."""
from __future__ import annotations

import numpy as np

from ._lib import opts_arg, check, f64, lib, ptr
from .parking import _pad_stages


def quadcopter_solve_batch(x0, xF, N, Ts, R, obs, xWS, timeWS=1.0, signed_dist=1, opts=None):
    """x0, xF (B,12); obs (5,6) = ob1..ob5; xWS (B,12,N+1).  Returns dict with Julia-shaped stacks:
    xp (B,12,N+1), up (B,4,N), ts (B,N+1), lp (B,30,N+1), slack (B,5,N+1), exitflag, iters, kkt_err, time.  opts None: the library's
    defaults with max_iter = 3000 (the reference leaves Ipopt's default max_iter)."""
    x0 = f64(np.atleast_2d(x0)); B = x0.shape[0]; NS = N + 1
    xF = f64(np.broadcast_to(np.asarray(xF, float).reshape(-1, 12), (B, 12)))
    ob = f64(np.asarray(obs, float).reshape(5, 6))                       # rows = obstacles == 6 x 5 column-major
    xw = f64(np.transpose(np.asarray(xWS, float).reshape(B, 12, -1)[:, :, :NS], (0, 2, 1)))
    xp = np.zeros((B, NS, 12)); up = np.zeros((B, N, 4)); ts = np.zeros((B, NS)); lp = np.zeros((B, NS, 30)); sl = np.zeros((B, NS, 5))
    ef = np.zeros(B, np.int32); it = np.zeros(B, np.int32); err = np.zeros(B); sec = np.zeros(1)
    check(lib().obca_quadcopter_solve_batch(B, N, ptr(x0), ptr(xF), float(Ts), float(R), ptr(ob), ptr(xw), float(timeWS), int(signed_dist),
                                            opts_arg(opts), ptr(xp), ptr(up), ptr(ts), ptr(lp), ptr(sl), ptr(ef), ptr(it), ptr(err),
                                            ptr(sec)))
    T = lambda a: np.transpose(a, (0, 2, 1))
    return dict(xp=T(xp), up=T(up), ts=ts, lp=T(lp), slack=T(sl), exitflag=ef, iters=it, kkt_err=err, time=float(sec[0]))


def _per_problem(Ns, Ts):
    Ns = np.ascontiguousarray(np.asarray(Ns).ravel(), dtype=np.int32)
    Tsb = f64(np.broadcast_to(np.asarray(Ts, float).ravel() if np.ndim(Ts) else float(Ts), (len(Ns),)))
    return Ns, Tsb, int(Ns.max())


def quadcopter_solve_mixed(x0, xF, Ns, Ts, R, obs, xWS, timeWS=1.0, signed_dist=1, opts=None):
    """One batched solve of problems with different horizons Ns[i] and sampling times (obca_quadcopter_solve_mixed).
    x0, xF (B,12); Ts scalar or (B,); obs (5,6); xWS per-problem list, xWS[i] 12x(Ns[i]+1).  Problem i gives exactly what
    quadcopter_solve_batch gives it at N = Ns[i], Ts = Ts[i].  Returns dict of per-problem lists in the Julia shapes
    (xp[i] 12x(Ns[i]+1), up[i] 4xNs[i], ts[i] Ns[i]+1, lp[i] 30x(Ns[i]+1), slack[i] 5x(Ns[i]+1)), the arrays exitflag,
    iters, kkt_err, N, Ts, and time."""
    x0 = f64(np.atleast_2d(x0)); B = x0.shape[0]
    Ns, Tsb, Nmax = _per_problem(Ns, Ts)
    assert len(Ns) == B
    NS = Nmax + 1
    xF = f64(np.broadcast_to(np.asarray(xF, float).reshape(-1, 12), (B, 12)))
    ob = f64(np.asarray(obs, float).reshape(5, 6))
    xw = f64(_pad_stages([np.asarray(w, float).reshape(12, -1)[:, :n + 1].T for w, n in zip(xWS, Ns)], Nmax))
    xp = np.zeros((B, NS, 12)); up = np.zeros((B, Nmax, 4)); ts = np.zeros((B, NS)); lp = np.zeros((B, NS, 30)); sl = np.zeros((B, NS, 5))
    ef = np.zeros(B, np.int32); it = np.zeros(B, np.int32); err = np.zeros(B); sec = np.zeros(1)
    check(lib().obca_quadcopter_solve_mixed(B, ptr(Ns), Nmax, ptr(x0), ptr(xF), ptr(Tsb), float(R), ptr(ob), ptr(xw), float(timeWS),
                                            int(signed_dist), opts_arg(opts), ptr(xp), ptr(up), ptr(ts), ptr(lp), ptr(sl), ptr(ef), ptr(it),
                                            ptr(err), ptr(sec)))
    cut = lambda a, ext: [a[i, :n + ext].T.copy() for i, n in enumerate(Ns)]
    return dict(xp=cut(xp, 1), up=cut(up, 0), ts=[ts[i, :n + 1].copy() for i, n in enumerate(Ns)], lp=cut(lp, 1), slack=cut(sl, 1),
                exitflag=ef, iters=it, kkt_err=err, N=Ns.copy(), Ts=Tsb.copy(), time=float(sec[0]))


def _single(sd, x0, xF, N, Ts, R, ob1, ob2, ob3, ob4, ob5, xWS, uWS, timeWS):
    obs = np.stack([np.asarray(o, float).ravel() for o in (ob1, ob2, ob3, ob4, ob5)])
    r = quadcopter_solve_batch(np.asarray(x0, float).reshape(1, 12), np.asarray(xF, float).reshape(1, 12), N, Ts, R, obs,
                               np.asarray(xWS, float)[None], timeWS, sd)
    ef = int(r["exitflag"][0])
    return r["xp"][0], r["up"][0], r["ts"][0], ef, r["time"], r["lp"][0], ("Optimal" if ef >= 1 else "Error")


def QuadcopterSignedDist(x0, xF, N, Ts, R, ob1, ob2, ob3, ob4, ob5, xWS, uWS, timeWS):
    return _single(1, x0, xF, N, Ts, R, ob1, ob2, ob3, ob4, ob5, xWS, uWS, timeWS)


def QuadcopterDist(x0, xF, N, Ts, R, ob1, ob2, ob3, ob4, ob5, xWS, uWS, timeWS):
    return _single(0, x0, xF, N, Ts, R, ob1, ob2, ob3, ob4, ob5, xWS, uWS, timeWS)


def check_quadcopter_batch(x, u, timeScale, x0, xF, Ts, lam, obs, R, opts=None):
    """x (B,12,N+1), u (B,4,N), timeScale (B,N+1), lam (B,30,N+1)."""
    x = np.asarray(x, float); B = x.shape[0]; N = x.shape[2] - 1
    T = lambda a: f64(np.transpose(np.asarray(a, float), (0, 2, 1)))
    x0 = f64(np.broadcast_to(np.asarray(x0, float).reshape(-1, 12), (B, 12))); xF = f64(np.broadcast_to(np.asarray(xF, float).reshape(-1, 12), (B, 12)))
    xx, uu, ll = T(x), T(u), T(lam)
    tt = f64(np.asarray(timeScale, float).reshape(B, N + 1))
    ob = f64(np.asarray(obs, float).reshape(5, 6))
    feas = np.zeros(B, np.int32); worst = np.zeros(B)
    check(lib().obca_check_quadcopter(B, N, ptr(xx), ptr(uu), ptr(tt), ptr(x0), ptr(xF), float(Ts), ptr(ll), ptr(ob), float(R),
                                      opts_arg(opts), ptr(feas), ptr(worst)))
    return feas, worst


def check_quadcopter_mixed(x, u, timeScale, x0, xF, Ns, Ts, lam, obs, R, opts=None):
    """check_quadcopter_batch over problems with different horizons Ns[i] and sampling times Ts (scalar or (B,))
    (obca_check_quadcopter_mixed): per-problem lists x[i] 12x(Ns[i]+1), u[i] 4xNs[i], timeScale[i] Ns[i]+1,
    lam[i] 30x(Ns[i]+1)."""
    Ns, Tsb, Nmax = _per_problem(Ns, Ts)
    B = len(Ns)
    P = lambda arrs, ext: f64(_pad_stages([np.asarray(a, float).T[:k + ext] for a, k in zip(arrs, Ns)], Nmax))
    xx, ll = P(x, 1), P(lam, 1)
    uu = f64(P(u, 0)[:, :Nmax])
    tt = f64(_pad_stages([np.ravel(t)[:k + 1] for t, k in zip(timeScale, Ns)], Nmax))
    x0 = f64(np.broadcast_to(np.asarray(x0, float).reshape(-1, 12), (B, 12))); xF = f64(np.broadcast_to(np.asarray(xF, float).reshape(-1, 12), (B, 12)))
    ob = f64(np.asarray(obs, float).reshape(5, 6))
    feas = np.zeros(B, np.int32); worst = np.zeros(B)
    check(lib().obca_check_quadcopter_mixed(B, ptr(Ns), Nmax, ptr(xx), ptr(uu), ptr(tt), ptr(x0), ptr(xF), ptr(Tsb), ptr(ll), ptr(ob),
                                            float(R), opts_arg(opts), ptr(feas), ptr(worst)))
    return feas, worst


def constrSatisfaction(x, u, timeScale, x0, xF, Ts, lam, ob1, ob2, ob3, ob4, ob5, R):
    obs = np.stack([np.asarray(o, float).ravel() for o in (ob1, ob2, ob3, ob4, ob5)])
    feas, _ = check_quadcopter_batch(np.asarray(x, float)[None], np.asarray(u, float)[None], np.asarray(timeScale, float).reshape(1, -1),
                                     x0, xF, Ts, np.asarray(lam, float)[None], obs, R)
    return bool(feas[0])
