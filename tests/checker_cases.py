"""Test inputs for the constraint checkers (ParkingConstraints / the strict audit, constrSatisfaction): feasible bases and one-change
cases around them -- values just inside and just outside each group's threshold, the reference's quirks, and NaN / +-Inf entries --
at the stage positions where each lane, warp and pass of the kernels' 128-thread reduction holds the deciding value.  Shared by
tests/test_checkers_emul.py (the checker sources on the host) and tests/test_gpu_checkers.py (the kernels); both compare with the
oracle (oracle/checkers.py)."""
from __future__ import annotations

import os

import numpy as np

from oracle import checkers

HERE = os.path.dirname(os.path.abspath(__file__))
TOL_P, TOL_Q = 5e-5, 1e-3
REL = 1e-6                       # just inside / outside: (1 -+ REL) times the threshold, far above the FMA contraction's rounding
NONFINITE = (np.nan, np.inf, -np.inf)
PARK_KEYS = ("x0", "xF", "x", "u", "l", "n", "timeScale", "sl")
QUAD_KEYS = ("x0", "xF", "x", "u", "timeScale", "lam")


def positions(N):
    """Stage positions that put the deciding value on lane 0, 1, 31 and 32 of the first pass, the last lane of a pass, the first
    and second lane of the next passes, and the horizon's last control and state."""
    return sorted({k for k in (0, 1, 31, 32, 127, 128, 129, 255, 256, N - 1, N) if 0 <= k <= N})


def _copy(p, keys):
    q = dict(p)
    for k in keys:
        if q.get(k) is not None:
            q[k] = np.array(q[k], float)
    return q


# ---- parking ---------------------------------------------------------------------------------------------------------------------

_DIRS = ((1.0, 0.0), (0.0, 1.0), (-1.0, 0.0), (0.0, -1.0))


def park_base(N, vOb, fixTime, sd, with_sl, yaw=0.0, XYbounds=(-15.0, 15.0, 1.0, 10.0)):
    """A car at rest at (0, 5) with the given yaw, among len(vOb) obstacles whose half-spaces are axis-aligned: feasible by
    construction for the reference and the strict audit.  Obstacle j's multiplier sits on one unit row r*_j (row 0 for the last
    obstacle), so |A' l| = 1, n balances it, and its distance row is 9 + (nOb - 1 - j) (the last obstacle is the closest)."""
    nOb = len(vOb)
    cy, sy = np.cos(yaw), np.sin(yaw)
    V = int(sum(vOb))
    ego = np.array([3.7, 1.0, 1.0, 1.0])
    g = np.array([2.35, 1.0, 2.35, 1.0]); off = 1.35
    X, Y = 0.0, 5.0
    A = np.zeros((V, 2)); b = np.zeros(V)
    l = np.zeros((V, N + 1)); n = np.zeros((4 * nOb, N + 1))
    rstar = []
    r0 = 0
    for j, v in enumerate(vOb):
        rs = 0 if j == nOb - 1 else j % v
        rstar.append(r0 + rs)
        for r in range(v):
            d1, d2 = _DIRS[r % 4]
            A[r0 + r] = (d1, d2)
            q1, q2 = cy * d1 + sy * d2, sy * d1 - cy * d2          # n0 - n2 = -q1, n1 - n3 = q2 (:123-124)
            gn = g[0] * abs(q1) + g[1] * abs(q2)
            b[r0 + r] = (X + cy * off) * d1 + (Y + sy * off) * d2 - gn - (9.0 + nOb - 1 - j)
        d1, d2 = A[r0 + rs]
        q1, q2 = cy * d1 + sy * d2, sy * d1 - cy * d2
        l[r0 + rs] = 1.0
        n[4 * j:4 * j + 4] = np.array([max(-q1, 0.0), max(q2, 0.0), max(q1, 0.0), max(-q2, 0.0)])[:, None]
        r0 += v
    x = np.zeros((4, N + 1)); x[0] = X; x[1] = Y; x[2] = yaw
    return dict(N=N, Ts=0.6, L=2.7, ego=ego, XYbounds=np.array(XYbounds, float), nOb=nOb, vOb=np.array(vOb), A=A, b=b,
                fixTime=fixTime, sd=sd, x0=x[:, 0].copy(), xF=x[:, N].copy(), x=x, u=np.zeros((2, N)), l=l, n=n,
                timeScale=np.ones(N + 1), sl=np.zeros((nOb, N + 1)) if with_sl else None, rstar=rstar)


def park_oracle(p):
    """(feasible, e (7,), strict) of the oracle for one problem."""
    args = (p["x0"], p["xF"], p["N"], p["Ts"], p["L"], p["ego"], p["XYbounds"], p["nOb"], p["vOb"], p["A"], p["b"], p["x"], p["u"],
            p["l"], p["n"], p["timeScale"], p["fixTime"], p["sd"])
    with np.errstate(all="ignore"):
        ok, e = checkers.ParkingConstraints(*args, return_e=True)
        st, _ = checkers.strict_check(*args, sl=p["sl"] if p["sd"] else None)
    return int(ok), np.asarray(e, np.int32), int(st)


def _dist(p, j, k):
    """The distance row of obstacle j at stage k (the oracle's formula, no slack)."""
    vo = np.concatenate([[0], np.cumsum(p["vOb"])]).astype(int)
    ego = p["ego"]; g = np.array([(ego[0] + ego[2]) / 2, (ego[1] + ego[3]) / 2] * 2); off = (ego[0] + ego[2]) / 2 - ego[2]
    lj = p["l"][vo[j]:vo[j + 1], k]; Aj = p["A"][vo[j]:vo[j + 1]]
    p1, p2 = Aj[:, 0] @ lj, Aj[:, 1] @ lj
    c, s = np.cos(p["x"][2, k]), np.sin(p["x"][2, k])
    return -g @ p["n"][4 * j:4 * j + 4, k] + (p["x"][0, k] + c * off) * p1 + (p["x"][1, k] + s * off) * p2 - p["b"][vo[j]:vo[j + 1]] @ lj


def park_threshold_cases(p):
    """Each of the seven groups of ParkingConstraints just inside and just outside its threshold (synthetic bases)."""
    N, nOb, Ts = p["N"], p["nOb"], p["Ts"]
    last = nOb - 1; r = p["rstar"][last]
    out = []

    def add(name, **ch):
        q = _copy(p, PARK_KEYS)
        for key, f in ch.items():
            f(q[key])
        out.append((name, q))

    for side, s in (("in", 1 - REL), ("out", 1 + REL)):
        t = TOL_P * s
        for i in range(4):
            add(f"c1 x0[{i}] {side}", x0=lambda a, i=i: a.__setitem__(i, a[i] + t))
            add(f"c2 xF[{i}] {side}", xF=lambda a, i=i: a.__setitem__(i, a[i] - t))
        for k in positions(N):
            if k < N:
                add(f"c0 u1 k={k} {side}", u=lambda a, k=k: a.__setitem__((0, k), -(0.6 + t)))
                add(f"c0 u2 k={k} {side}", u=lambda a, k=k: a.__setitem__((1, k), 0.4 + t))
                add(f"c5 du1 k={k} {side}", u=lambda a, k=k: a.__setitem__((0, k), (0.6 + t) * Ts))
            add(f"c0 ts k={k} {side}", timeScale=lambda a, k=k: a.__setitem__(k, 1.2 + t))
            add(f"c4 ts k={k} {side}", timeScale=lambda a, k=k: a.__setitem__(k, 1.0 + t))
            add(f"c0 l k={k} {side}", l=lambda a, k=k: a.__setitem__((r + 1 if p["vOb"][last] > 1 else r, k), -t))
            add(f"c0 n k={k} {side}", n=lambda a, k=k: a.__setitem__((4 * last + 1, k), -t))
            if k >= 1:
                for row in range(4):
                    add(f"c3 x[{row}] k={k} {side}", x=lambda a, k=k, row=row: a.__setitem__((row, k), a[row, k] + t))
            add(f"c6 pp k={k} {side}", l=lambda a, k=k: a.__setitem__((r, k), np.sqrt(1.0 + t)))
            add(f"c6 n02 k={k} {side}", n=lambda a, k=k: a.__setitem__((4 * last + 0, k), a[4 * last + 0, k] + t))
            add(f"c6 n13 k={k} {side}", n=lambda a, k=k: a.__setitem__((4 * last + 1, k), a[4 * last + 1, k] + t))
            dk = _dist(p, last, k)
            add(f"c6 dist k={k} {side}", x=lambda a, k=k, dk=dk: a.__setitem__((0, k), a[0, k] - (dk - 0.05 + t)))
    return out


def park_quirk_cases(p):
    """The reference's quirks: each case passes the reference and fails the strict audit, or the other way round, in some of the
    variants (fixTime, sd, sl)."""
    N, nOb, Ts = p["N"], p["nOb"], p["Ts"]
    last = nOb - 1; r = p["rstar"][last]
    out = []
    for k in positions(N):
        if 1 <= k <= N - 1:
            q = _copy(p, PARK_KEYS); q["x"][0, k] += 1e-3; out.append((f"dynamics row x k={k}", q))
        if nOb >= 2:
            q = _copy(p, PARK_KEYS); q["n"][0, k] += 1e-3; out.append((f"first obstacle c6 k={k}", q))
        q = _copy(p, PARK_KEYS)
        q["l"][r, k] *= 0.9; q["n"][4 * last:4 * last + 4, k] *= 0.9
        out.append((f"|pp-1| k={k}", q))
        if 1 <= k <= N - 1:
            q = _copy(p, PARK_KEYS)
            q["timeScale"][:] = 1.0 + 4e-5 * np.arange(N + 1)
            q["u"][0, k] = (0.6 + TOL_P) * Ts * (q["timeScale"][0] + q["timeScale"][k]) / 2
            out.append((f"c5 ts[0] vs ts[k] k={k}", q))
        q = _copy(p, PARK_KEYS); q["timeScale"][k] = 1.2 + 1e-3; out.append((f"|ts-1| k={k}", q))
    q = _copy(p, PARK_KEYS); q["timeScale"][:] = 0.0; out.append(("timeScale zeros", q))
    # the slack: the last obstacle 1e-3 inside the margin, its slack 2e-3 (the whole trajectory moves, so the dynamics hold)
    q = _copy(p, PARK_KEYS)
    sh = _dist(p, last, 0) - 0.05 + 1e-3
    q["x"][0] -= sh; q["x0"][0] -= sh; q["xF"][0] -= sh
    if q["sl"] is not None:
        q["sl"][last] = 2e-3
    out.append(("slack", q))
    return out


def park_box_cases(N, vOb, fixTime, sd, with_sl):
    """The strict audit's X / Y box (the reference never checks it), each bound just inside and just outside its threshold at each
    stage position k, with every other group feasible: the car drives with constant deceleration along x (yaw 0) or y (yaw pi/2),
    integrated with the reference's dynamics so that every dynamics row holds, and its position peaks at stage k alone (its
    neighbours lie at least 2.5e-6 inside).  The strict audit checks the box at stages 1..N-1 only: at k = 0 and k = N it passes.
    Returns [(scene, cases)], one scene per axis (the box is tight around the car: the batch shares XYbounds)."""
    out = []
    for axis, yaw in ((0, 0.0), (1, np.pi / 2)):
        base = park_base(N, vOb, fixTime, sd, with_sl, yaw=yaw, XYbounds=(-1.0, 1.0, 4.0, 6.0))
        Ts, L = base["Ts"], base["L"]
        cases = []
        for k in positions(N):
            M = max(k, N - k, 1)
            acc = min(0.4, 0.5 / (Ts * Ts * M * M))
            for bound, sign in ((base["XYbounds"][2 * axis + 1], 1.0), (base["XYbounds"][2 * axis], -1.0)):
                for side, s in (("in", 1 - REL), ("out", 1 + REL)):
                    q = _copy(base, PARK_KEYS)
                    x, u = q["x"], q["u"]
                    u[1] = -sign * acc
                    x[3, 0] = sign * acc * Ts * k
                    for j in range(N):                        # ParkingConstraints.jl:66-69 with h = Ts (timeScale = 1)
                        h = Ts
                        vm = x[3, j] + h / 2 * u[1, j]; th = x[2, j] + h / 2 * x[3, j] * np.tan(u[0, j]) / L
                        x[:, j + 1] = (x[0, j] + h * vm * np.cos(th), x[1, j] + h * vm * np.sin(th), x[2, j] + h * vm * np.tan(u[0, j]) / L,
                                       x[3, j] + h * u[1, j])
                    x[axis] += bound + sign * TOL_P * s - x[axis, k]
                    q["x0"] = x[:, 0].copy(); q["xF"] = x[:, N].copy()
                    cases.append((f"box {'xy'[axis]} {'upper' if sign > 0 else 'lower'} {side} k={k}", q))
        out.append((base, cases))
    return out


def park_nonfinite_cases(p, every=1):
    """NaN, +Inf and -Inf in each row of x, u, l (the last obstacle and the first), n (the last obstacle's rows and the first's),
    timeScale and sl at the stage positions, and in x0 and xF.  every > 1 takes one value per (row, position), in turn."""
    N, nOb = p["N"], p["nOb"]
    last = nOb - 1
    rows = [("x", i) for i in range(4)] + [("u", 0), ("u", 1), ("l", p["rstar"][last]), ("l", p["rstar"][0] if nOb > 1 else 0)]
    rows += [("n", 4 * last + i) for i in range(4)] + ([("n", 0)] if nOb > 1 else []) + [("timeScale", None)]
    if p.get("sl") is not None:
        rows += [("sl", last), ("sl", 0)]
    out = []
    c = 0
    for k in positions(N):
        for key, row in rows:
            if key == "u" and k == N:
                continue
            for v in NONFINITE:
                c += 1
                if c % every:
                    continue
                q = _copy(p, PARK_KEYS)
                if row is None:
                    q[key][k] = v
                else:
                    q[key][row, k] = v
                out.append((f"{v} in {key}[{row}] k={k}", q))
    for key in ("x0", "xF"):
        for i in range(4):
            for v in NONFINITE:
                q = _copy(p, PARK_KEYS); q[key][i] = v; out.append((f"{v} in {key}[{i}]", q))
    q = _copy(p, PARK_KEYS); q["x"][:] = np.nan; out.append(("all-NaN x", q))
    return out


def park_cases(p, every=1):
    return park_threshold_cases(p) + park_quirk_cases(p) + park_nonfinite_cases(p, every)


def park_golden_bases():
    """The converged parking goldens with their scenes, as bases: (name, problem)."""
    import glob
    from obca_b200 import scenarios
    out = []
    for path in sorted(glob.glob(os.path.join(HERE, "golden", "*.npz"))):
        name = os.path.basename(path)[:-4]
        if name.startswith(("_", "quad_")):
            continue
        g = np.load(path)
        kind = str(g["scenario"]) if "scenario" in g else "reverse"
        sc = (scenarios.parallel_parking_batch(8, 80, int(g["seed"]), int(kind[-1])) if kind.startswith("parallel")
              else scenarios.reverse_parking_batch(8, 80, int(g["seed"])))
        out.append((name, _golden_problem(g, sc, sc["x0"][int(g["index"])], int(g["fixTime"]))))
    for path in sorted(glob.glob(os.path.join(HERE, "golden", "lot", "*.npz"))):
        g = np.load(path)
        sc = scenarios.parking_lot_batch(8, 80, int(g["seed"]), int(str(g["scenario"])[3:]))
        out.append(("lot/" + os.path.basename(path)[:-4], _golden_problem(g, sc, sc["x0"][int(g["index"])], int(g["fixTime"]))))
    for path in sorted(glob.glob(os.path.join(HERE, "golden", "long_park", "*.npz"))):
        g = np.load(path)
        sc = scenarios.reverse_parking_scenario()
        sc.update(N=int(g["N"]), Ts=float(g["Ts"]))
        out.append(("long_park/" + os.path.basename(path)[:-4], _golden_problem(g, sc, g["x0"], 0)))
    return out


def _golden_problem(g, sc, x0, fix):
    sd = 1 if str(g["variant"]) == "sd" else 0
    return dict(N=int(g["xp"].shape[1]) - 1, Ts=sc["Ts_fix"] if fix else sc["Ts"], L=sc["L"], ego=np.asarray(sc["ego"], float),
                XYbounds=np.asarray(sc["XYbounds"], float), nOb=int(sc["nOb"]), vOb=np.asarray(sc["vOb"]),
                A=np.asarray(sc["A"], float).reshape(-1, 2), b=np.asarray(sc["b"], float).ravel(), fixTime=fix, sd=sd,
                x0=np.asarray(x0, float).ravel(), xF=np.asarray(sc["xF"], float).ravel(), x=g["xp"], u=g["up"], l=g["lp"], n=g["np"],
                timeScale=g["ts"], sl=g["sl"] if sd else None)


def park_golden_cases(p):
    """Clear violations and non-finite entries on a converged golden (realistic magnitudes)."""
    N = p["N"]
    out = [("golden", _copy(p, PARK_KEYS))]
    for k in positions(N):
        for key, row, d in (("x", 3, 1e-3), ("x", 0, 1e-3), ("l", 0, -1e-3), ("n", 0, -1e-3)):
            q = _copy(p, PARK_KEYS); q[key][row, k] += d; out.append((f"{key}[{row}] + {d} k={k}", q))
        for key, row in (("x", 2), ("u", 1), ("l", int(sum(p["vOb"])) - 1), ("n", 4 * p["nOb"] - 1), ("timeScale", None)):
            if key == "u" and k == N:
                continue
            for v in NONFINITE:
                q = _copy(p, PARK_KEYS)
                if row is None:
                    q[key][k] = v
                else:
                    q[key][row, k] = v
                out.append((f"{v} in {key}[{row}] k={k}", q))
    return out


# ---- quadcopter ------------------------------------------------------------------------------------------------------------------

QLO = np.array([0, 0, 0, -3, -0.2, -0.2, -1, -1, -1, -1.5, -1, -1.0])
QHI = np.array([10, 10, 5, 3, 0.2, 0.2, 1, 1, 1, 3, 1, 1.0])


def quad_base(N, Ts=0.2, ts=1.0, ground=False):
    """A quadcopter hovering at (5, 5, 2): feasible by construction (dynamics residuals of a few ulps).  Five boxes on its +x side,
    obstacle o's multiplier 1 on its -x face (norm row 0, distance row 1 + o); or, with ground, five boxes below z = -1 - o with
    the multiplier on their top face, so that the distance rows hold wherever the drone is in the x / y / z box."""
    R = 0.5
    uh = np.sqrt(0.5 * 9.81 / (4 * 0.0611))
    x = np.zeros((12, N + 1)); x[0] = 5.0; x[1] = 5.0; x[2] = 2.0
    obs = np.zeros((5, 6)); lam = np.zeros((30, N + 1))
    for o in range(5):
        if ground:
            lo = np.array([0.0, 0.0, -10.0]); hi = np.array([10.0, 10.0, -1.0 - o])
            lam[6 * o + 2] = 1.0
        else:
            lo = np.array([5.0 + R + 1.0 + o, 0.0, 0.0]); hi = lo + np.array([1.0, 10.0, 5.0])
            lam[6 * o + 3] = 1.0
        obs[o] = np.concatenate([hi, -lo])
    return dict(N=N, Ts=Ts, R=R, obs=obs, x=x, u=np.full((4, N), uh), timeScale=np.full(N + 1, ts), x0=x[:, 0].copy(),
                xF=x[:, N].copy(), lam=lam)


def _quad_roll(q, k0):
    """x[:, k0+1:] integrated from x[:, k0] with the reference's dynamics (constrSatisfaction.jl:135-153), so every dynamics row
    holds; x0 and xF follow the trajectory."""
    x = q["x"]
    for j in range(k0, q["N"]):
        x[:, j + 1] = 0.0
        x[:, j + 1] = -checkers.quad_dynamics_rows(x, q["u"], q["timeScale"], q["Ts"], j)[:12]
    q["x0"] = x[:, 0].copy(); q["xF"] = x[:, -1].copy()


def quad_box_cases(N, Ts=0.2):
    """Each box group of constrSatisfaction (:83, :95, :108, :120) just inside and just outside each of its bounds, with every
    other group feasible: the drone hovers among the ground boxes with timeScale 1e-5, one state entry starts at the bound and the
    trajectory is integrated with the reference's dynamics (that entry stays at its value, the others drift by less than 1e-2);
    one rotor's input sits at its bound at stage k alone.  Also the Dist-variant bound of x10 under SD ([-1.5, 3], not [-1, 1]).
    Returns (scene, cases)."""
    base = quad_base(N, Ts, ts=1e-5, ground=True)
    m = lambda v: REL * max(1.0, abs(v))
    out = []

    def add(name, f, k0):
        q = _copy(base, QUAD_KEYS)
        f(q)
        _quad_roll(q, k0)
        out.append((name, q))

    for i in range(12):
        for side, vlo, vhi in (("in", QLO[i] + m(QLO[i]), QHI[i] - m(QHI[i])), ("out", QLO[i] - m(QLO[i]), QHI[i] + m(QHI[i]))):
            add(f"x[{i}] lower {side}", lambda q, i=i, v=vlo: q["x"].__setitem__((i, 0), v), 0)
            add(f"x[{i}] upper {side}", lambda q, i=i, v=vhi: q["x"].__setitem__((i, 0), v), 0)
    add("x10 Dist box under SD", lambda q: q["x"].__setitem__((9, 0), 2.0), 0)
    for k in positions(N):
        if k < N:
            for j in range(4):
                for side, vlo, vhi in (("in", 1.2 + m(1.2), 7.8 - m(7.8)), ("out", 1.2 - m(1.2), 7.8 + m(7.8))):
                    add(f"u[{j}] lower {side} k={k}", lambda q, j=j, k=k, v=vlo: q["u"].__setitem__((j, k), v), k)
                    add(f"u[{j}] upper {side} k={k}", lambda q, j=j, k=k, v=vhi: q["u"].__setitem__((j, k), v), k)
    return base, out


def quad_oracle(q):
    """(feasible, worst) of the oracle; asserts that constr_worst <= 1e-3 is constrSatisfaction."""
    args = (q["x"], q["u"], q["timeScale"], q["x0"], q["xF"], q["Ts"], q["lam"], *q["obs"], q["R"])
    with np.errstate(all="ignore"):
        ok = bool(checkers.constrSatisfaction(*args))
        w = checkers.constr_worst(*args)
    assert (w <= TOL_Q) == ok, (w, ok)
    return int(ok), w


def quad_cases(p, every=1):
    N = p["N"]
    out = []

    def add(name, f):
        q = _copy(p, QUAD_KEYS)
        f(q)
        out.append((name, q))

    for k in positions(N):
        if k < N:
            for side, s in (("in", 1 - REL), ("out", 1 + REL)):
                t = TOL_Q * s
                for i in range(12):
                    add(f"dyn[{i}] {side} k={k}", lambda q, i=i, k=k, t=t: q["x"].__setitem__((i, k + 1), q["x"][i, k + 1] + t))
                add(f"dyn[ts] {side} k={k}", lambda q, k=k, t=t: q["timeScale"].__setitem__(k + 1, 1.0 + t))
                for o in range(5):
                    add(f"norm[{o}] {side} k={k}", lambda q, o=o, k=k, t=t: q["lam"].__setitem__((6 * o + 3, k), np.sqrt(1.0 + t)))
                    dist = 1.0 + o                                     # lo_x - x - R with the multiplier 1
                    add(f"dist[{o}] {side} k={k}",
                        lambda q, o=o, k=k, t=t, dist=dist: q["lam"].__setitem__((6 * o + 3, k), (p["R"] - t) / (dist + p["R"])))
        for side, s in (("in", 1 - REL), ("out", 1 + REL)):
            add(f"lambda {side} k={k}", lambda q, k=k, s=s: q["lam"].__setitem__((6 * (k % 5) + 1, k), -TOL_Q * s))
        k2 = (k + 1) % (N + 1)
        add(f"lambda group off by NaN at k={k2}, -0.5 at k={k}",
            lambda q, k=k, k2=k2: (q["lam"].__setitem__((1, k), -0.5), q["lam"].__setitem__((29, k2), np.nan)))
        if k < N:
            add(f"dyn violation + NaN lambda k={k}",
                lambda q, k=k: (q["x"].__setitem__((6, k + 1), 0.5), q["lam"].__setitem__((29, k), np.nan),
                                q["lam"].__setitem__((29, k + 1), np.nan)))
            add(f"u box violation + NaN x k={k}",
                lambda q, k=k: (q["u"].__setitem__((0, k), 8.0), q["x"].__setitem__((4, k), np.nan)))
            add(f"norm violation + NaN ts k={k}",
                lambda q, k=k: (q["lam"].__setitem__((3, k), 1.5), q["timeScale"].__setitem__(k, np.nan)))
    # Q5: the body-rate rows of every stage read x[9..11] of stage 0
    add("Q5", lambda q: (q["x"].__setitem__((10, 0), 0.5), q["x"].__setitem__((11, 0), 0.5), q["x0"].__setitem__(slice(None), q["x"][:, 0])))
    add("Q5 inside", lambda q: (q["x"].__setitem__((10, 0), 0.01), q["x"].__setitem__((11, 0), 0.01),
                                q["x0"].__setitem__(slice(None), q["x"][:, 0])))
    c = 0
    rows = [("x", i) for i in range(12)] + [("u", j) for j in range(4)] + [("lam", r) for r in (0, 3, 29)] + [("timeScale", None)]
    for k in positions(N):
        for key, row in rows:
            if key == "u" and k == N:
                continue
            for v in NONFINITE:
                c += 1
                if c % every:
                    continue
                add(f"{v} in {key}[{row}] k={k}",
                    lambda q, key=key, row=row, k=k, v=v: q[key].__setitem__(k if row is None else (row, k), v))
    for key in ("x0", "xF"):
        for i in (0, 9):
            for v in NONFINITE:
                add(f"{v} in {key}[{i}]", lambda q, key=key, i=i, v=v: q[key].__setitem__(i, v))
    return out


def same_worst(a, b):
    """worst of the kernels against constr_worst: 1e-12 (1 + |worst|), or the same infinity."""
    return a == b or abs(a - b) <= 1e-12 * (1 + abs(b))


def thin(cases, n):
    """At most about n of the cases, evenly spread (the oracle's loops are slow at long horizons with many obstacles)."""
    return cases[::max(1, len(cases) // n)]


def quad_golden_bases():
    import glob
    from obca_b200 import scenarios
    out = []
    for path in sorted(glob.glob(os.path.join(HERE, "golden", "quad_[ds]*_p[0-9].npz"))):
        g = np.load(path)
        N, i = int(g["N"]), int(g["index"])
        sc = scenarios.quadcopter_batch(4, N, int(g["seed"]))
        out.append((os.path.basename(path)[:-4],
                    dict(N=N, Ts=float(sc["Ts"]), R=float(sc["R"]), obs=np.asarray(sc["obs"], float), x=g["xp"], u=g["up"],
                         timeScale=g["ts"], x0=np.asarray(sc["x0"][i], float), xF=np.asarray(sc["xF"][i], float), lam=g["lp"])))
    return out


def quad_golden_cases(p):
    N = p["N"]
    out = [("golden", _copy(p, QUAD_KEYS))]
    for k in positions(N):
        for key, row, d in (("x", 0, 2e-3), ("x", 9, 2e-3), ("lam", 5, -2e-3)):
            q = _copy(p, QUAD_KEYS); q[key][row, k] += d; out.append((f"{key}[{row}] + {d} k={k}", q))
        for key, row in (("x", 3), ("u", 2), ("lam", 17), ("timeScale", None)):
            if key == "u" and k == N:
                continue
            for v in NONFINITE:
                q = _copy(p, QUAD_KEYS)
                q[key][k if row is None else (row, k)] = v
                out.append((f"{v} in {key}[{row}] k={k}", q))
    return out
