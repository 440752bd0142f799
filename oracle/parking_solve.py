"""ORACLE (test infrastructure only).  Glue: reference parking NLP (parking_nlp.py) + IPOPT stand-in (ipm_ref.py).

solve_parking(...) takes the 17 arguments of ParkingSignedDist.jl:29 / ParkingDist.jl:29 and returns the
reference's 7-tuple plus the full solver result.
"""
from __future__ import annotations

import time

import numpy as np

from . import ipm_ref
from .dualmultws_ref import dualmultws, dualmultws_ipm
from .parking_nlp import build_parking_nlp, initial_point


def solver_view(nlp):
    """Bounds on the pinned end states are redundant (x[:,1]==x0, x[:,N+1]==xF, ParkingSignedDist.jl:122-131);
    the solver drops them so that no barrier term sits on a fixed variable (same KKT points)."""
    lay = nlp.lay
    for k in (0, lay.N):
        for i in range(4):
            nlp.zL[lay.x(i, k)] = -np.inf; nlp.zU[lay.x(i, k)] = np.inf
    return nlp


def dc_mask(nlp):
    """always-on dual regularisation rows: norm rows (sd) and the terminal dynamics rows (DESIGN.md)."""
    m = np.zeros(nlp.mE, bool)
    N = nlp.lay.N
    for fam in nlp.eq:
        if fam.name.startswith("norm"):
            m[fam.row0:fam.row0 + fam.n] = True
        if fam.name.startswith("dyn"):
            m[fam.row0 + N - 1] = True
    return m


def stage_order(nlp):
    """Stage-interleaved symmetric ordering of the KKT unknowns (variables of stage k, then the equality rows whose
    last variable lives in stage k): keeps the LDL' factor banded.  Used by ipm_ref's sparse path."""
    lay = nlp.lay
    vs = np.zeros(nlp.n, int)
    NS = lay.NS
    vs[lay.oX:lay.oX + 4 * NS] = np.repeat(np.arange(NS), 4)
    if not lay.fixTime:
        vs[lay.oT:lay.oT + NS] = np.arange(NS)
    vs[lay.oU:lay.oU + 2 * lay.N] = np.repeat(np.arange(lay.N), 2)
    vs[lay.oL:lay.oN] = np.repeat(np.arange(NS), lay.V)
    vs[lay.oN:lay.oS] = np.repeat(np.arange(NS), 4 * lay.nOb)
    if lay.variant == "sd":
        vs[lay.oS:] = np.repeat(np.arange(NS), lay.nOb)
    rs = np.zeros(nlp.mE, int)
    for fam in nlp.eq:
        rs[fam.row0:fam.row0 + fam.n] = vs[fam.idx].max(axis=1)
    key = np.concatenate([2 * vs, 2 * rs + 1])
    return np.argsort(key, kind="stable")


def solve_parking(x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS,
                  variant="sd", lWS=None, nWS=None, opts=None, verbose=False, one_time_scale=False):
    """one_time_scale: measure the dual infeasibility of the time scales as that of the one variable t the CUDA solver carries
    (ipm_ref.IpmOptions.dual_sum_groups): the same Newton steps, and the barrier updates and the stopping test of the kernels."""
    nlp = solver_view(build_parking_nlp(x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw,
                                        fixTime, variant))
    if lWS is None:
        lWS, nWS, _, _ = dualmultws_ipm(N, nOb, vOb, A, b, rx, ry, ryaw, ego)   # ParkingSignedDist.jl:219
    z0 = initial_point(nlp.lay, xWS, uWS, lWS, nWS)
    o = opts or ipm_ref.IpmOptions()
    o.dc_rows = dc_mask(nlp)
    if o.linsolve == "sparse":
        o.order = stage_order(nlp)
    if one_time_scale and not fixTime:
        o.dual_sum_groups = [nlp.lay.ts(np.arange(N + 1))]
    o.verbose = verbose
    t0 = time.time()
    res = ipm_ref.solve(nlp, z0, o)
    dt = time.time() - t0
    xp, up, ts, lp, np_, sl = nlp.lay.unpack(res.z)
    exitflag = 1 if res.status == 1 else 0
    return (xp, up, ts, exitflag, dt, lp, np_), res, nlp
