"""ORACLE (test infrastructure only -- never imported by the product path).

Verbatim numpy restatement of AutonomousParking/ParkingConstraints.jl:29-149, INCLUDING its quirks
(SURVEY.md A.4-Q3): c3[1,i] overwritten (only the v-row survives, :76-79), c6[.,i] overwritten per obstacle (only
the last obstacle is audited, :117-128), c5 scaled by timeScale[1] only (:92), sd=1 ignores sl and uses abs(pp)-1.
Shapes as in Julia: x 4x(N+1), u 2xN, l Vx(N+1), n 4nOb x(N+1), timeScale (N+1).
"""
from __future__ import annotations

import numpy as np


def ParkingConstraints(x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, x, u, l, n, timeScale, fixTime, sd,
                       return_e=False):
    x0 = np.asarray(x0, float).ravel(); xF = np.asarray(xF, float).ravel()
    x = np.asarray(x, float); u = np.asarray(u, float); l = np.asarray(l, float); n = np.asarray(n, float)
    timeScale = np.asarray(timeScale, float).ravel()
    vOb = [int(v) for v in np.asarray(vOb).ravel()]
    A = np.asarray(A, float).reshape(-1, 2); b = np.asarray(b, float).ravel()
    ego = np.asarray(ego, float).ravel()
    dmin = 0.05                                                      # :33
    c0 = np.zeros(5); c1 = np.zeros(4); c2 = np.zeros(4); c3 = np.zeros((4, N)); c6 = np.zeros((4, N + 1))
    c0[0] = np.max(np.abs(u[0, :])) - 0.6                            # :45
    c0[1] = np.max(np.abs(u[1, :])) - 0.4
    c0[2] = np.max(np.abs(timeScale - 1)) - 0.2
    c0[3] = -np.min(l)
    c0[4] = -np.min(n)
    c1[:] = np.abs(x[:, 0] - x0)                                     # :52-55
    c2[:] = np.abs(x[:, N] - xF)                                     # :58-61
    for i in range(N):
        if fixTime == 1:
            c3[0, i] = x[0, i + 1] - (x[0, i] + Ts * (x[3, i] + Ts / 2 * u[1, i]) * np.cos(x[2, i] + Ts / 2 * x[3, i] * np.tan(u[0, i]) / L))
            c3[1, i] = x[1, i + 1] - (x[1, i] + Ts * (x[3, i] + Ts / 2 * u[1, i]) * np.sin(x[2, i] + Ts / 2 * x[3, i] * np.tan(u[0, i]) / L))
            c3[2, i] = x[2, i + 1] - (x[2, i] + Ts * (x[3, i] + Ts / 2 * u[1, i]) * np.tan(u[0, i]) / L)
            c3[3, i] = x[3, i + 1] - (x[3, i] + Ts * u[1, i])
        else:
            # :76-79 -- four assignments to c3[1,i]; the last one wins
            c3[0, i] = x[3, i + 1] - (x[3, i] + timeScale[i] * Ts * u[1, i])
    if fixTime == 1:
        c5 = np.max(np.abs(np.diff(np.concatenate([[0.0], u[0, :]]))) / Ts) - 0.6      # :88
        c4 = 0.0
    else:
        c4 = np.max(np.abs(np.diff(timeScale)))                                        # :91
        c5 = np.max(np.abs(np.diff(np.concatenate([[0.0], u[0, :]]))) / (timeScale[0] * Ts)) - 0.6   # :92
    W_ev = ego[1] + ego[3]; L_ev = ego[0] + ego[2]
    g = np.array([L_ev / 2, W_ev / 2, L_ev / 2, W_ev / 2])
    offset = (ego[0] + ego[2]) / 2 - ego[2]
    off = np.concatenate([[0], np.cumsum(vOb)]).astype(int)
    for i in range(N + 1):
        for j in range(nOb):
            Aj = A[off[j]:off[j + 1]]; lj = l[off[j]:off[j + 1], i]; nj = n[4 * j:4 * j + 4, i]; bj = b[off[j]:off[j + 1]]
            p1 = Aj[:, 0] @ lj; p2 = Aj[:, 1] @ lj
            if sd == 1:
                c6[0, i] = abs(p1 ** 2 + p2 ** 2) - 1                # :117
            else:
                c6[0, i] = p1 ** 2 + p2 ** 2 - 1                     # :119
            c6[1, i] = abs((nj[0] - nj[2]) + np.cos(x[2, i]) * p1 + np.sin(x[2, i]) * p2)     # :123
            c6[2, i] = abs((nj[1] - nj[3]) - np.sin(x[2, i]) * p1 + np.cos(x[2, i]) * p2)     # :124
            c6[3, i] = -(-g @ nj + (x[0, i] + np.cos(x[2, i]) * offset) * p1
                         + (x[1, i] + np.sin(x[2, i]) * offset) * p2 - bj @ lj) + dmin         # :127-128
    e = np.zeros(7, int)
    e[0] = np.max(c0) <= 5e-5; e[1] = np.max(c1) <= 5e-5; e[2] = np.max(c2) <= 5e-5
    e[3] = np.max(np.abs(c3)) <= 5e-5; e[4] = c4 <= 5e-5; e[5] = c5 <= 5e-5; e[6] = np.max(c6) <= 5e-5
    ok = 1 if e.sum() == 7 else 0
    return (ok, e) if return_e else ok


def _nanmax(*v):
    """max that propagates NaN, like Julia's maximum (the built-in max(0.0, nan) is 0.0)."""
    return float(np.max(np.array(v, float)))


def strict_check(x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, x, u, l, n, timeScale, fixTime, sd, sl=None,
                 tol=5e-5):
    """Quirk-free audit: every dynamics row, every obstacle, box bounds, |pp-1| (sd) and slack-aware distance.  Returns (ok, worst);
    a NaN in any value it reads makes worst NaN and ok 0."""
    x0 = np.asarray(x0, float).ravel(); xF = np.asarray(xF, float).ravel()
    x = np.asarray(x, float); u = np.asarray(u, float); l = np.asarray(l, float); n = np.asarray(n, float)
    ts = np.asarray(timeScale, float).ravel()
    vOb = [int(v) for v in np.asarray(vOb).ravel()]
    A = np.asarray(A, float).reshape(-1, 2); b = np.asarray(b, float).ravel()
    ego = np.asarray(ego, float).ravel(); XYb = np.asarray(XYbounds, float).ravel()
    worst = 0.0
    h = np.full(N, Ts) if fixTime else ts[:N] * Ts
    vm = x[3, :N] + h / 2 * u[1]; th = x[2, :N] + h / 2 * x[3, :N] * np.tan(u[0]) / L
    f = np.stack([x[0, :N] + h * vm * np.cos(th), x[1, :N] + h * vm * np.sin(th), x[2, :N] + h * vm * np.tan(u[0]) / L,
                  x[3, :N] + h * u[1]])
    worst = _nanmax(worst, np.abs(x[:, 1:] - f).max(), np.abs(x[:, 0] - x0).max(), np.abs(x[:, N] - xF).max())
    worst = _nanmax(worst, np.abs(u[0]).max() - 0.6, np.abs(u[1]).max() - 0.4, -l.min(), -n.min())
    if not fixTime:
        worst = _nanmax(worst, np.abs(ts - 1).max() - 0.2, np.abs(np.diff(ts)).max())
    worst = _nanmax(worst, (np.abs(np.diff(np.concatenate([[0.0], u[0]]))) / h).max() - 0.6)
    xi = x[:, 1:N]
    worst = _nanmax(worst, (XYb[0] - xi[0]).max(), (xi[0] - XYb[1]).max(), (XYb[2] - xi[1]).max(), (xi[1] - XYb[3]).max(),
                (-1 - xi[3]).max(), (xi[3] - 2).max())
    g = np.array([(ego[0] + ego[2]) / 2, (ego[1] + ego[3]) / 2, (ego[0] + ego[2]) / 2, (ego[1] + ego[3]) / 2])
    offset = (ego[0] + ego[2]) / 2 - ego[2]
    off = np.concatenate([[0], np.cumsum(vOb)]).astype(int)
    c, s = np.cos(x[2]), np.sin(x[2])
    for j in range(nOb):
        Aj = A[off[j]:off[j + 1]]; lj = l[off[j]:off[j + 1]]; nj = n[4 * j:4 * j + 4]; bj = b[off[j]:off[j + 1]]
        p1 = Aj[:, 0] @ lj; p2 = Aj[:, 1] @ lj; pp = p1 ** 2 + p2 ** 2
        worst = _nanmax(worst, (np.abs(pp - 1) if sd else pp - 1).max())
        worst = _nanmax(worst, np.abs(nj[0] - nj[2] + c * p1 + s * p2).max(), np.abs(nj[1] - nj[3] - s * p1 + c * p2).max())
        dist = -g @ nj + (x[0] + c * offset) * p1 + (x[1] + s * offset) * p2 - bj @ lj
        if sd and sl is not None:
            dist = dist + np.asarray(sl, float)[j]
        worst = _nanmax(worst, (0.05 - dist).max())
    return (1 if worst <= tol else 0), worst


def constrSatisfaction(x, u, timeScale, x0, xF, Ts, lam, ob1, ob2, ob3, ob4, ob5, R):
    """Verbatim numpy restatement of QuadcopterNavigation/constrSatisfaction.jl:25-204 (tolerance 1e-3; rows for
    i = 1..N only; Dist-variant box on x10; one-sided norm row; quirk Q5 in the body-rate rows)."""
    mass, g = 0.5, 9.81
    k_F, k_M = 0.0611, 0.0015
    I = np.array([3.9, 4.4, 4.9]) * 1e-3
    L = 0.225
    x = np.asarray(x, float); u = np.asarray(u, float); ts = np.asarray(timeScale, float).ravel(); lam = np.asarray(lam, float)
    x0 = np.asarray(x0, float).ravel(); xF = np.asarray(xF, float).ravel()
    ls = [lam[6 * o:6 * o + 6] for o in range(5)]
    bs = [np.asarray(b, float).ravel() for b in (ob1, ob2, ob3, ob4, ob5)]
    N = x.shape[1] - 1
    if np.abs(x[:, 0] - x0).max() > 1e-3: return False              # :56-61
    if np.abs(x[:, -1] - xF).max() > 1e-3: return False             # :63-68
    A = np.vstack([np.eye(3), -np.eye(3)])
    xl = x.ravel(order="F")                                          # linear (column-major) indexing
    lo = np.array([0, 0, 0, -3, -0.2, -0.2, -1, -1, -1, -1.5, -1, -1.0]); hi = np.array([10, 10, 5, 3, 0.2, 0.2, 1, 1, 1, 3, 1, 1.0])
    for i in range(N):
        if (1.2 - u[:, i]).max() > 0 or (u[:, i] - 7.8).max() > 0: return False
        if (lo - x[:, i]).max() > 0 or (x[:, i] - hi).max() > 0: return False
        h = ts[i] * Ts
        F = k_F * (u[:, i] ** 2).sum()
        xi = x[:, i]
        s = np.zeros(13)
        s[0] = x[0, i + 1] - (xi[0] + h * xi[6]); s[1] = x[1, i + 1] - (xi[1] + h * xi[7]); s[2] = x[2, i + 1] - (xi[2] + h * xi[8])
        s[3] = x[3, i + 1] - (xi[3] + h * (np.cos(xi[4]) * xi[9] + np.sin(xi[4]) * xi[11]))
        s[4] = x[4, i + 1] - (xi[4] + h * (np.sin(xi[4]) * np.tan(xi[3]) * xi[9] + xi[10] - np.cos(xi[4]) * np.tan(xi[3]) * xi[11]))
        s[5] = x[5, i + 1] - (xi[5] + h * (-np.sin(xi[4]) / np.cos(xi[3]) * xi[9] + np.cos(xi[4]) / np.cos(xi[3]) * xi[11]))
        s[6] = x[6, i + 1] - (xi[6] + h / mass * (F * (np.sin(xi[3]) * np.cos(xi[4]) * np.sin(xi[5]) + np.sin(xi[4]) * np.cos(xi[5]))))
        s[7] = x[7, i + 1] - (xi[7] + h / mass * (F * (-np.sin(xi[3]) * np.cos(xi[4]) * np.cos(xi[5]) + np.sin(xi[4]) * np.sin(xi[5]))))
        s[8] = x[8, i + 1] - (xi[8] + h / mass * (F * (np.cos(xi[3]) * np.cos(xi[4])) - mass * g))
        s[9] = x[9, i + 1] - (xi[9] + h / I[0] * (L * k_F * (u[1, i] ** 2 - u[3, i] ** 2) - (I[2] - I[1]) * xl[10] * xl[11]))
        s[10] = x[10, i + 1] - (xi[10] + h / I[1] * (L * k_F * (u[2, i] ** 2 - u[0, i] ** 2) - (I[0] - I[2]) * xl[9] * xl[11]))
        s[11] = x[11, i + 1] - (xi[11] + h / I[2] * (k_M * (u[0, i] ** 2 - u[1, i] ** 2 + u[2, i] ** 2 - u[3, i] ** 2) - (I[1] - I[0]) * xl[9] * xl[10]))
        s[12] = ts[i] - ts[i + 1]
        if np.abs(s).max() > 1e-3: return False
        if lam.min() < -1e-3: return False
        t1 = np.array([(l[0, i] - l[3, i]) ** 2 + (l[1, i] - l[4, i]) ** 2 + (l[2, i] - l[5, i]) ** 2 - 1 for l in ls])
        if t1.max() > 1e-3: return False
        t2 = np.array([-(b @ l[:, i]) + xi[0] * (A[:, 0] @ l[:, i]) + xi[1] * (A[:, 1] @ l[:, i]) + xi[2] * (A[:, 2] @ l[:, i]) - R
                       for l, b in zip(ls, bs)])
        if t2.min() < -1e-3: return False
    return True


def quad_dynamics_rows(x, u, ts, Ts, i):
    """The 13 dynamics rows of constrSatisfaction.jl:135-154 at stage i (0-based), quirk Q5 included: x[9..11] of stage 0 in the
    body-rate rows.  x 12x(N+1), u 4xN, ts (N+1)."""
    mass, g = 0.5, 9.81
    k_F, k_M = 0.0611, 0.0015
    I = np.array([3.9, 4.4, 4.9]) * 1e-3
    L = 0.225
    xl = x.ravel(order="F")
    h = ts[i] * Ts
    F = k_F * (u[:, i] ** 2).sum()
    xi = x[:, i]
    s = np.zeros(13)
    s[0] = x[0, i + 1] - (xi[0] + h * xi[6]); s[1] = x[1, i + 1] - (xi[1] + h * xi[7]); s[2] = x[2, i + 1] - (xi[2] + h * xi[8])
    s[3] = x[3, i + 1] - (xi[3] + h * (np.cos(xi[4]) * xi[9] + np.sin(xi[4]) * xi[11]))
    s[4] = x[4, i + 1] - (xi[4] + h * (np.sin(xi[4]) * np.tan(xi[3]) * xi[9] + xi[10] - np.cos(xi[4]) * np.tan(xi[3]) * xi[11]))
    s[5] = x[5, i + 1] - (xi[5] + h * (-np.sin(xi[4]) / np.cos(xi[3]) * xi[9] + np.cos(xi[4]) / np.cos(xi[3]) * xi[11]))
    s[6] = x[6, i + 1] - (xi[6] + h / mass * (F * (np.sin(xi[3]) * np.cos(xi[4]) * np.sin(xi[5]) + np.sin(xi[4]) * np.cos(xi[5]))))
    s[7] = x[7, i + 1] - (xi[7] + h / mass * (F * (-np.sin(xi[3]) * np.cos(xi[4]) * np.cos(xi[5]) + np.sin(xi[4]) * np.sin(xi[5]))))
    s[8] = x[8, i + 1] - (xi[8] + h / mass * (F * (np.cos(xi[3]) * np.cos(xi[4])) - mass * g))
    s[9] = x[9, i + 1] - (xi[9] + h / I[0] * (L * k_F * (u[1, i] ** 2 - u[3, i] ** 2) - (I[2] - I[1]) * xl[10] * xl[11]))
    s[10] = x[10, i + 1] - (xi[10] + h / I[1] * (L * k_F * (u[2, i] ** 2 - u[0, i] ** 2) - (I[0] - I[2]) * xl[9] * xl[11]))
    s[11] = x[11, i + 1] - (xi[11] + h / I[2] * (k_M * (u[0, i] ** 2 - u[1, i] ** 2 + u[2, i] ** 2 - u[3, i] ** 2) - (I[1] - I[0]) * xl[9] * xl[10]))
    s[12] = ts[i] - ts[i + 1]
    return s


def constr_worst(x, u, timeScale, x0, xF, Ts, lam, ob1, ob2, ob3, ob4, ob5, R):
    """The `worst` of the quadcopter checker, group by group from constrSatisfaction.jl:25-204 like constrSatisfaction above:
    the largest contribution of its groups, where a group is what one test of the reference reads (start, end; per stage i = 1..N
    the u lower / upper and x lower / upper boxes, which contribute 1.0 when violated, the 13 dynamics rows, the 5 norm rows, the
    negated 5 distance rows; the negated lambda matrix, once).  A group whose value is NaN never fails in the reference and
    contributes nothing here.  constr_worst(...) <= 1e-3 is constrSatisfaction(...)."""
    x = np.asarray(x, float); u = np.asarray(u, float); ts = np.asarray(timeScale, float).ravel(); lam = np.asarray(lam, float)
    x0 = np.asarray(x0, float).ravel(); xF = np.asarray(xF, float).ravel()
    ls = [lam[6 * o:6 * o + 6] for o in range(5)]
    bs = [np.asarray(b, float).ravel() for b in (ob1, ob2, ob3, ob4, ob5)]
    N = x.shape[1] - 1
    A = np.vstack([np.eye(3), -np.eye(3)])
    lo = np.array([0, 0, 0, -3, -0.2, -0.2, -1, -1, -1, -1.5, -1, -1.0]); hi = np.array([10, 10, 5, 3, 0.2, 0.2, 1, 1, 1, 3, 1, 1.0])
    worst = [0.0]
    add = lambda v: worst.append(float(v)) if not np.isnan(v) else None
    add(np.abs(x[:, 0] - x0).max())                                  # :56-61
    add(np.abs(x[:, -1] - xF).max())                                 # :63-68
    add(-lam.min())                                                  # :162, the whole matrix at every i
    for i in range(N):
        for grp in (1.2 - u[:, i], u[:, i] - 7.8, lo - x[:, i], x[:, i] - hi):      # :83, :95, :108, :120
            if grp.max() > 0:
                add(1.0)
        xi = x[:, i]
        s = quad_dynamics_rows(x, u, ts, Ts, i)
        add(np.abs(s).max())                                         # :156
        add(np.array([(l[0, i] - l[3, i]) ** 2 + (l[1, i] - l[4, i]) ** 2 + (l[2, i] - l[5, i]) ** 2 - 1 for l in ls]).max())   # :178
        add(-np.array([-(b @ l[:, i]) + xi[0] * (A[:, 0] @ l[:, i]) + xi[1] * (A[:, 1] @ l[:, i]) + xi[2] * (A[:, 2] @ l[:, i]) - R
                       for l, b in zip(ls, bs)]).min())              # :195
    return max(worst)
