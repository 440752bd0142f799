"""Host-side input producers for the OBCA hot path (NOT on the GPU path).

* ``obst_hrep``           -- twin of AutonomousParking/obstHrep.jl:31-102 (vertices -> stacked H-rep).
* ``reverse_parking_*``   -- scenario constants of AutonomousParking/main.jl:36-213 ("backwards").
* ``warmstart_reverse``   -- deterministic geometric warm start (straight / left arc / reverse right arc /
  reverse straight): the cheap synthetic stand-in for the Hybrid A* + veloSmooth pipeline of main.jl:217-248 that
  the benchmark batches use (the pipeline itself is obca_b200/planner/, SURVEY.md section 8f-1).  Produces the same
  artefacts main.jl hands to ParkingSignedDist: rx, ry, ryaw (N+1), xWS (N+1)x4, uWS Nx2.
* ``reverse_parking_batch`` -- BASELINE config 2: randomised start poses, numpy default_rng(seed).
* ``reverse_parking_mixed_batch`` -- the same with a seeded horizon per problem (input of parking_solve_mixed).
* ``parking_lot_*``       -- the reverse-parking slot in a row of parked cars (n_cars + 1 obstacles): scene, batch, point cloud;
                            parking_lot_free_slots: the same row with some cars left out, a goal per free slot.
* ``quadcopter_mixed_batch`` -- BASELINE config 4 with a seeded horizon and its sampling time per problem (input of
  quadcopter_solve_mixed).
"""
from __future__ import annotations

import math

import numpy as np


def obst_hrep(nOb, vOb, lOb):
    """obstHrep.jl:31-102.  vOb = vertex counts (incl. repeated/last vertex), lOb = list of vertex lists."""
    vOb = [int(v) for v in np.asarray(vOb).ravel()]
    if nOb != len(lOb):
        print("ERROR in number of obstacles")           # obstHrep.jl:34-36 (prints, does not throw)
    rows = sum(vOb) - nOb
    A_all = np.zeros((rows, 2)); b_all = np.zeros((rows, 1))
    r = 0
    for i in range(nOb):
        for j in range(vOb[i] - 1):
            v1 = np.asarray(lOb[i][j], float).ravel(); v2 = np.asarray(lOb[i][j + 1], float).ravel()
            if v1[0] == v2[0]:                           # vertical edge, :57-64
                if v2[1] < v1[1]:
                    A_tmp, b_tmp = [1.0, 0.0], v1[0]
                else:
                    A_tmp, b_tmp = [-1.0, 0.0], -v1[0]
            elif v1[1] == v2[1]:                         # horizontal edge, :65-72
                if v1[0] < v2[0]:
                    A_tmp, b_tmp = [0.0, 1.0], v1[1]
                else:
                    A_tmp, b_tmp = [0.0, -1.0], -v1[1]
            else:                                        # general edge (not normalised), :73-85
                ab = np.linalg.solve(np.array([[v1[0], 1.0], [v2[0], 1.0]]), np.array([v1[1], v2[1]]))
                a_, b_ = ab
                if v1[0] < v2[0]:
                    A_tmp, b_tmp = [-a_, 1.0], b_
                else:
                    A_tmp, b_tmp = [a_, -1.0], -b_
            A_all[r] = A_tmp; b_all[r, 0] = b_tmp
            r += 1
    return A_all, b_all


# ----------------------------------------------------------------------------------------------
# scenario constants (main.jl)
# ----------------------------------------------------------------------------------------------
EGO = np.array([3.7, 1.0, 1.0, 1.0])          # main.jl:73
WHEELBASE = 2.7                               # main.jl:63
XYBOUNDS = np.array([-15.0, 15.0, 1.0, 10.0])  # main.jl:210


def reverse_parking_scenario():
    """main.jl:99-108 ("backwards"): obstacles, H-rep, goal, Ts (variable time)."""
    nOb = 3
    vOb = [3, 3, 2]
    lOb = [[[-20, 5], [-1.3, 5], [-1.3, -5]],
           [[1.3, -5], [1.3, 5], [20, 5]],
           [[20, 11], [-20, 11]]]
    A, b = obst_hrep(nOb, vOb, lOb)
    return dict(nOb=nOb, vOb=np.array(vOb) - 1, A=A, b=b, xF=np.array([0.0, 1.3, math.pi / 2, 0.0]),
                Ts=0.6, Ts_fix=0.55, L=WHEELBASE, ego=EGO.copy(), XYbounds=XYBOUNDS.copy(), lOb=lOb)


def parallel_parking_scenario(n_obstacles=3):
    """main.jl:154-162 ("parallel").  The reference lists 4 obstacles; BASELINE config 3 keeps the first 3."""
    lOb = [[[-20, 5], [-3.0, 5], [-3.0, 0]],
           [[3.0, 0], [3.0, 5], [20, 5]],
           [[-3, 2.5], [3, 2.5]],
           [[20, 11], [-20, 11]]][:n_obstacles]
    vOb = [3, 3, 2, 2][:n_obstacles]
    A, b = obst_hrep(n_obstacles, vOb, lOb)
    return dict(nOb=n_obstacles, vOb=np.array(vOb) - 1, A=A, b=b,
                xF=np.array([-WHEELBASE / 2, 4.0, 0.0, 0.0]), Ts=0.9, Ts_fix=0.95, L=WHEELBASE,
                ego=EGO.copy(), XYbounds=XYBOUNDS.copy(), lOb=lOb)


# ----------------------------------------------------------------------------------------------
# geometric warm start
# ----------------------------------------------------------------------------------------------
def _integrate_path(x, y, yaw, segs, L):
    """segs: list of (signed_length, curvature).  Returns a function s -> (x,y,yaw,delta,dir) over total |length|."""
    knots = []
    s_acc = 0.0
    for (ln, kap) in segs:
        knots.append((s_acc, abs(ln), math.copysign(1.0, ln) if ln != 0 else 1.0, kap, x, y, yaw))
        d = ln
        if abs(kap) < 1e-12:
            x, y = x + d * math.cos(yaw), y + d * math.sin(yaw)
        else:
            x += (math.sin(yaw + kap * d) - math.sin(yaw)) / kap
            y -= (math.cos(yaw + kap * d) - math.cos(yaw)) / kap
            yaw += kap * d
        s_acc += abs(ln)
    return knots, s_acc, (x, y, yaw)


def _eval_knot(knot, ds, L):
    _, _, sgn, kap, x, y, yaw = knot
    d = sgn * ds
    if abs(kap) < 1e-12:
        return x + d * math.cos(yaw), y + d * math.sin(yaw), yaw, 0.0
    xn = x + (math.sin(yaw + kap * d) - math.sin(yaw)) / kap
    yn = y - (math.cos(yaw + kap * d) - math.cos(yaw)) / kap
    return xn, yn, yaw + kap * d, math.atan(L * kap)


def warmstart_from_segments(x0, segs, N, Ts, L):
    """Rest-to-rest smoothstep speed profile on every segment; segment durations ~ (length + 1 m)."""
    knots, total, _ = _integrate_path(x0[0], x0[1], x0[2], segs, L)
    T = N * Ts
    w = np.array([k[1] + 1.0 for k in knots]); dur = T * w / w.sum()
    t_edges = np.concatenate([[0.0], np.cumsum(dur)])
    tt = np.arange(N + 1) * Ts
    xWS = np.zeros((N + 1, 4)); uWS = np.zeros((N, 2))
    for i, t in enumerate(tt):
        q = min(np.searchsorted(t_edges, t, side="right") - 1, len(knots) - 1)
        tau = min(max((t - t_edges[q]) / dur[q], 0.0), 1.0)
        ln, sgn = knots[q][1], knots[q][2]
        ds = ln * (3 * tau ** 2 - 2 * tau ** 3)
        v = sgn * ln / dur[q] * 6 * tau * (1 - tau)
        acc = sgn * ln / dur[q] ** 2 * 6 * (1 - 2 * tau)
        x, y, yaw, de = _eval_knot(knots[q], ds, L)
        xWS[i] = [x, y, yaw, v]
        if i < N:
            uWS[i] = [de, acc]
    return xWS, uWS


def warmstart_reverse(x0, xF, N, Ts, L, y_e=3.8, R0=4.5):
    """Warm start for the reverse-parking slot of main.jl:99-108 (goal pose heading +y, slot below y=5)."""
    X0, Y0 = float(x0[0]), float(x0[1])
    segs = []
    if Y0 - y_e >= R0:                      # single reverse arc
        R = Y0 - y_e
        x_s = xF[0] + R
        segs.append((x_s - X0, 0.0))
        segs.append((-R * (math.pi / 2), -1.0 / R))
    else:                                   # forward-left arc to heading alpha, then reverse-right arc to pi/2
        R = R0
        ca = (Y0 + R - y_e) / (2 * R)
        alpha = math.acos(min(1.0, ca))
        x_s = xF[0] + R - 2 * R * math.sin(alpha)
        segs.append((x_s - X0, 0.0))
        segs.append((R * alpha, 1.0 / R))
        segs.append((-R * (math.pi / 2 - alpha), -1.0 / R))
    segs.append((-(y_e - xF[1]), 0.0))
    segs = [sg for sg in segs if abs(sg[0]) > 1e-9]
    xWS, uWS = warmstart_from_segments([X0, Y0, float(x0[2])], segs, N, Ts, L)
    xWS[0] = x0; xWS[-1] = xF               # exact end poses (main.jl path starts/ends on x0/xF)
    return xWS[:, 0].copy(), xWS[:, 1].copy(), xWS[:, 2].copy(), xWS, uWS


def reverse_parking_batch(B, N=80, seed=0):
    """BASELINE.json config 2: X0~U(-10,10), Y0~U(6.5,9.5), psi0=v0=0 (ranges of main.jl:165-168)."""
    sc = reverse_parking_scenario()
    rng = np.random.default_rng(seed)
    X0 = rng.uniform(-10, 10, B); Y0 = rng.uniform(6.5, 9.5, B)
    x0 = np.stack([X0, Y0, np.zeros(B), np.zeros(B)], 1)
    rx = np.zeros((B, N + 1)); ry = np.zeros((B, N + 1)); ryaw = np.zeros((B, N + 1))
    xWS = np.zeros((B, N + 1, 4)); uWS = np.zeros((B, N, 2))
    for i in range(B):
        rx[i], ry[i], ryaw[i], xWS[i], uWS[i] = warmstart_reverse(x0[i], sc["xF"], N, sc["Ts"], sc["L"])
    sc.update(B=B, N=N, x0=x0, rx=rx, ry=ry, ryaw=ryaw, xWS=xWS, uWS=uWS)
    return sc


# ----------------------------------------------------------------------------------------------
# a row of a car park: the reverse-parking slot between parked cars
# ----------------------------------------------------------------------------------------------
LOT_SLOT = 2.6                  # slot width: the target slot is [-1.3, 1.3]
LOT_CAR = (1.9, 4.6)            # parked car: width, length
LOT_KERB = 5.0                  # the cars' fronts are on y = 5 (the kerb line of main.jl:99-101)


def parking_lot_cars(n_cars):
    """The parked cars as clockwise rectangles [x_lo, x_hi, y_lo, y_hi], centred in the slots that alternate right and
    left of the target slot (x = 2.6, -2.6, 5.2, -5.2, ...)."""
    w, l = LOT_CAR
    cars = []
    for i in range(n_cars):
        c = LOT_SLOT * (i // 2 + 1) * (1 if i % 2 == 0 else -1)
        cars.append((c - w / 2, c + w / 2, LOT_KERB - l, LOT_KERB))
    return cars


def parking_lot_scenario(n_cars=10):
    """The "backwards" scene of main.jl:99-108 in a row of a car park: obstacles 1 and 2 (the half-planes beside the slot) are
    replaced by n_cars parked cars (4 half-spaces each), the far wall (obstacle 3, y >= 11) stays; goal, Ts, XYbounds as in
    reverse_parking_scenario.  nOb = n_cars + 1, sum(vOb) = 4 n_cars + 1.  Every car lies inside the region of the reference's
    obstacles 1 and 2, so the start poses and warm starts of reverse_parking_batch stay collision-free."""
    return _lot_scene(parking_lot_cars(n_cars))


def _lot_scene(cars):
    lOb = [[[x0, y1], [x1, y1], [x1, y0], [x0, y0], [x0, y1]] for x0, x1, y0, y1 in cars]
    lOb.append([[20, 11], [-20, 11]])
    vOb = [5] * len(cars) + [2]
    nOb = len(cars) + 1
    A, b = obst_hrep(nOb, vOb, lOb)
    sc = reverse_parking_scenario()
    sc.update(nOb=nOb, vOb=np.array(vOb) - 1, A=A, b=b, lOb=lOb)
    return sc


def parking_lot_batch(B, N=80, seed=0, n_cars=10):
    """reverse_parking_batch (start poses, warm starts) with the obstacles of parking_lot_scenario(n_cars)."""
    sc = reverse_parking_batch(B, N, seed)
    lot = parking_lot_scenario(n_cars)
    for k in ("nOb", "vOb", "A", "b", "lOb"):
        sc[k] = lot[k]
    return sc


def parking_lot_points(n_cars=10):
    """The point cloud Hybrid A* plans against in the lot: every car outline sampled at 0.1 m, and the far wall y = 11 at
    1 m spacing, as main.jl:111-142 samples the reference's obstacles."""
    return _lot_points(parking_lot_cars(n_cars))


def _lot_points(cars):
    ox, oy = [], []

    def line(a, b, n):
        for t in np.linspace(0.0, 1.0, n + 1):
            ox.append(a[0] + t * (b[0] - a[0])); oy.append(a[1] + t * (b[1] - a[1]))
    for x0, x1, y0, y1 in cars:
        nx, ny = int(round((x1 - x0) / 0.1)), int(round((y1 - y0) / 0.1))
        line((x0, y1), (x1, y1), nx); line((x1, y0), (x0, y0), nx)
        line((x0, y0), (x0, y1), ny); line((x1, y1), (x1, y0), ny)
    for i in range(-12, 13):
        ox.append(float(i)); oy.append(11.0)
    return np.array(ox), np.array(oy)


def parking_lot_free_slots(n_cars=10, free=(0, 3, 5)):
    """The row of parking_lot_scenario(n_cars) with the parked cars of index `free` left out: several free slots.  The scene
    (nOb, vOb, A, b, lOb) and the point cloud (ox, oy) hold only the cars that remain.  slots: the x of every free slot, the
    target slot x = 0 first, then the slots of the cars left out in the order of `free`; goals (n_slots, 4): the goal pose
    [x_slot, 1.3, pi/2, 0] of each, the reverse-parking goal moved to that slot."""
    cars = parking_lot_cars(n_cars)
    kept = [c for i, c in enumerate(cars) if i not in set(free)]
    sc = _lot_scene(kept)
    sc["ox"], sc["oy"] = _lot_points(kept)
    sc["slots"] = np.array([0.0] + [(cars[i][0] + cars[i][1]) / 2 for i in free])
    sc["goals"] = np.array([[x, 1.3, np.pi / 2, 0.0] for x in sc["slots"]])
    return sc


def reverse_parking_mixed_batch(B, N_range=(40, 80), seed=0, Ns=None):
    """Reverse parking with a horizon per problem (what a planned sweep looks like): start poses as in
    reverse_parking_batch, N_i ~ uniform over N_range (inclusive) from the same seeded generator unless Ns is given, and
    every warm start built at its problem's own N_i.  rx, ry, ryaw, xWS, uWS are per-problem lists; Ns the horizons."""
    sc = reverse_parking_scenario()
    rng = np.random.default_rng(seed)
    X0 = rng.uniform(-10, 10, B); Y0 = rng.uniform(6.5, 9.5, B)
    Ns = np.asarray(Ns if Ns is not None else rng.integers(N_range[0], N_range[1] + 1, B), dtype=np.int32)
    x0 = np.stack([X0, Y0, np.zeros(B), np.zeros(B)], 1)
    rx, ry, ryaw, xWS, uWS = [], [], [], [], []
    for i in range(B):
        r = warmstart_reverse(x0[i], sc["xF"], int(Ns[i]), sc["Ts"], sc["L"])
        rx.append(r[0]); ry.append(r[1]); ryaw.append(r[2]); xWS.append(r[3]); uWS.append(r[4])
    sc.update(B=B, Ns=Ns, x0=x0, rx=rx, ry=ry, ryaw=ryaw, xWS=xWS, uWS=uWS)
    return sc


# ----------------------------------------------------------------------------------------------
# quadcopter (QuadcopterNavigation/mainQuadcopter.jl)
# ----------------------------------------------------------------------------------------------
def quadcopter_scenario():
    """mainQuadcopter.jl:36-55: ball ego R = 0.25, five boxes b = [x_up, y_up, z_up, -x_lo, -y_lo, -z_lo]
    (A = [I; -I], QuadcopterSignedDist.jl:162-163): a wall with a gap below z = 0.6 and a wall with a window."""
    obs = np.array([[2.5, 12, 7, -2, 2, -0.6],      # ob12
                    [7.5, 12, 7, -7, -5, 2],        # ob22
                    [7.5, 4, 7, -7, 2, 2],          # ob32
                    [7.5, 5, 2, -7, -4, 2],         # ob42
                    [7.5, 5, 7, -7, -4, -3]])       # ob52
    return dict(R=0.25, obs=obs, Ts80=0.25, x0=np.array([1, 1, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0.0]),
                xF=np.array([9, 3, 2, 0, 0, 0, 0, 0, 0, 0, 0, 0.0]))


def warmstart_quadcopter(x0, xF, N):
    """Position warm start standing in for the 3-D A* of mainQuadcopter.jl:122-135 (out of scope): a polyline
    start -> under wall 1 -> through the window of wall 2 -> goal, sampled at N+1 equal arc-length points; all other
    states 0 like xWS_as (:134)."""
    p0 = np.asarray(x0[:3], float); p5 = np.asarray(xF[:3], float)
    way = np.array([p0, [1.6, p0[1], 0.17], [2.9, p0[1], 0.17], [6.6, 4.5, 2.5], [7.9, 4.5, 2.5], p5])
    seg = np.linalg.norm(np.diff(way, axis=0), axis=1)
    s = np.concatenate([[0], np.cumsum(seg)])
    q = np.linspace(0, s[-1], N + 1)
    xWS = np.zeros((12, N + 1))
    for d in range(3):
        xWS[d] = np.interp(q, s, way[:, d])
    return xWS


def quadcopter_batch(B, N=100, seed=2):
    """BASELINE config 4: x0 = [1, Y, Z, 0..], xF = [9, Y', Z', 0..], Y ~ U(0.5, 9.5), Z ~ U(0.5, 4.5)
    (mainQuadcopter.jl:48-51), Ts * N = 20 (:131)."""
    sc = quadcopter_scenario()
    rng = np.random.default_rng(seed)
    x0 = np.zeros((B, 12)); xF = np.zeros((B, 12))
    x0[:, 0] = 1; xF[:, 0] = 9
    x0[:, 1] = rng.uniform(0.5, 9.5, B); x0[:, 2] = rng.uniform(0.5, 4.5, B)
    xF[:, 1] = rng.uniform(0.5, 9.5, B); xF[:, 2] = rng.uniform(0.5, 4.5, B)
    Ts = round((sc["Ts80"] * 80 / N) * 100) / 100
    xWS = np.stack([warmstart_quadcopter(x0[i], xF[i], N) for i in range(B)])
    sc.update(B=B, N=N, Ts=Ts, x0=x0, xF=xF, xWS=xWS, timeWS=1.0)
    return sc


def quadcopter_mixed_batch(B, N_range=(90, 127), seed=2, Ns=None):
    """Config 4 with a horizon and a sampling time per problem (what a batch of 3-D A* warm starts looks like,
    mainQuadcopter.jl:122-137): x0 / xF drawn exactly as in quadcopter_batch, then N_i ~ uniform over N_range (inclusive)
    from the same generator unless Ns is given, Ts_i = round(Ts80 * 80 / N_i, 2) (:131) and the warm start at N_i.
    The default range is the one the 3-D A* gives for config-4 start / goal pairs.  Ns, Ts are arrays; xWS[i] is
    12 x (N_i+1)."""
    sc = quadcopter_scenario()
    rng = np.random.default_rng(seed)
    x0 = np.zeros((B, 12)); xF = np.zeros((B, 12))
    x0[:, 0] = 1; xF[:, 0] = 9
    x0[:, 1] = rng.uniform(0.5, 9.5, B); x0[:, 2] = rng.uniform(0.5, 4.5, B)
    xF[:, 1] = rng.uniform(0.5, 9.5, B); xF[:, 2] = rng.uniform(0.5, 4.5, B)
    Ns = np.asarray(Ns if Ns is not None else rng.integers(N_range[0], N_range[1] + 1, B), dtype=np.int32)
    Ts = np.array([round((sc["Ts80"] * 80 / int(n)) * 100) / 100 for n in Ns])      # as quadcopter_batch
    xWS = [warmstart_quadcopter(x0[i], xF[i], int(Ns[i])) for i in range(B)]
    sc.update(B=B, Ns=Ns, Ts=Ts, x0=x0, xF=xF, xWS=xWS, timeWS=1.0)
    return sc


# ----------------------------------------------------------------------------------------------
# parallel parking (BASELINE config 3)
# ----------------------------------------------------------------------------------------------
def warmstart_parallel(x0, xF, N, Ts, L, R=4.5):
    """Warm start for the parallel-parking slot of main.jl:154-162 (goal heading 0, slot between x=-3 and x=3 below
    y=5): straight along the lane to the start of a reverse S-curve (right-steer arc, then left-steer arc), standing in
    for Hybrid A* (out of scope)."""
    X0, Y0 = float(x0[0]), float(x0[1])
    dy = Y0 - float(xF[1])
    th = math.acos(max(-1.0, min(1.0, 1.0 - dy / (2 * R))))
    x_s = float(xF[0]) + 2 * R * math.sin(th)
    segs = [(x_s - X0, 0.0), (-R * th, -1.0 / R), (-R * th, 1.0 / R)]
    segs = [sg for sg in segs if abs(sg[0]) > 1e-9]
    xWS, uWS = warmstart_from_segments([X0, Y0, float(x0[2])], segs, N, Ts, L)
    xWS[0] = x0; xWS[-1] = xF
    return xWS[:, 0].copy(), xWS[:, 1].copy(), xWS[:, 2].copy(), xWS, uWS


def parallel_parking_batch(B, N=80, seed=1, n_obstacles=3):
    """BASELINE.json config 3: parallel parking, N=80, seed 1; n_obstacles=3 (obstacles 1-3 of main.jl:154-157, the
    wall at y=11 dropped -- XYbounds y<=10 makes it inactive) or 4 (the reference's own list)."""
    sc = parallel_parking_scenario(n_obstacles)
    rng = np.random.default_rng(seed)
    X0 = rng.uniform(-10, 10, B); Y0 = rng.uniform(6.5, 9.5, B)
    x0 = np.stack([X0, Y0, np.zeros(B), np.zeros(B)], 1)
    rx = np.zeros((B, N + 1)); ry = np.zeros((B, N + 1)); ryaw = np.zeros((B, N + 1))
    xWS = np.zeros((B, N + 1, 4)); uWS = np.zeros((B, N, 2))
    for i in range(B):
        rx[i], ry[i], ryaw[i], xWS[i], uWS[i] = warmstart_parallel(x0[i], sc["xF"], N, sc["Ts"], sc["L"])
    sc.update(B=B, N=N, x0=x0, rx=rx, ry=ry, ryaw=ryaw, xWS=xWS, uWS=uWS)
    return sc
