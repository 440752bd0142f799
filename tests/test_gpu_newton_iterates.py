"""The parking solver's Newton iterates on the GPU against the oracle's interior-point method (oracle/ipm_ref.py, sparse
path), iteration by iteration (pytest -m gpu).

The other GPU tests look at converged points, or compare the schedules with each other.  An interior-point method with a
wrong Hessian term, a wrong Jacobian entry in the condensation onto the stage model, or a KKT sweep that drops part of a
gain still reaches the same KKT point, because it stops on the constraint values and gradL alone: it only takes other
steps.  Here the library runs K iterations (max_iter = K, retry = 0) and every problem of the batch is compared with its
own oracle run from the same warm start and the same DualMultWS multipliers after each pinned K, in both schedules (the
tail kernel alone, and the rounds k_pk_eval / k_pk_sweep / k_pk_step alone).

The shapes make every path that only the device build runs take part at least once: the cp.async ring of k_pk_sweep with
fewer stages than SWEEP_DEPTH = 8 (N = 4, 7), the bulk copy of the stage slots out of k_pk_eval, the step rows of
k_pk_step in shared memory (config 2 at N = 80: 40 rows of 82 doubles) and in workspace rows (by step_rows_in_smem, where 5
CTAs no longer fit on an SM with them: the lot, 226 rows, and config 2 at N = 319, 40 rows of 320 doubles), the
hand-over rows of obstacles 7 to 16 (the lot), horizons past 127 up to 319, and per-problem horizons in one padded batch.

The oracle measures the dual infeasibility of the time scales as that of the one variable t the kernels carry for them
(solve_parking(..., one_time_scale=True)).  The reference formulation ties the N + 1 time scales with chain rows; the
kernels eliminate the chain (DESIGN.md section 3).  Both take the same Newton steps, but the optimality error of the
tied formulation has one entry per stage, |dL/dts[k]| with the chain multipliers, where that of the eliminated one has
|sum_k dL/dts[k]|.  The barrier update compares that error with kappa_eps * mu, so the two formulations update mu at
different iterations: on the lot at N = 80, problem 0, the oracle's error at iteration 5 is 0.77 (mu drops to 0.02) and
the kernels' is 2.84 (mu stays 0.1), and the iterates split by 1e-2 there.  Measured the kernels' way, the oracle takes
the same discrete decisions as the kernel sources (tests/emul) through K = 6 on the shapes pinned that far.

K: 1, 2, 3, and further up to 6 where the emulation of the kernel sources was measured against the oracle on these inputs
(iterates within 1e-10, the same inertia-correction factorization counts).

Tolerances: 1e-7 (primal xp, up, ts) and 1e-6 (the multipliers lp, np of the distance reformulation), scaled by
1 + max|oracle|.  The emulation meets the oracle at these pins to within 3e-9 on a CPU, and a device build of the same
sources differs from it only by FMA contraction and the order of a few sums."""
import multiprocessing
import os
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

B = 8
PRIMAL_TOL, DUAL_TOL = 1e-7, 1e-6
ENV_KEYS = ("OBCA_MODE", "OBCA_TAIL_THRESH", "OBCA_CHUNK")
SCHEDULES = {"tail": {"OBCA_MODE": "1"}, "rounds": {"OBCA_MODE": "2", "OBCA_TAIL_THRESH": "0"}}


def sixteen_by_four(sc):
    """The lot with the far wall as a 4-half-space box: nOb = 16, sum(vOb) = 64 (test_gpu_long_parking.test_largest_shapes_at_319)."""
    from obca_b200 import scenarios
    lOb = sc["lOb"][:-1] + [[[-20, 12], [20, 12], [20, 11], [-20, 11], [-20, 12]]]
    A, b = scenarios.obst_hrep(16, [5] * 16, lOb)
    sc = dict(sc)
    sc.update(nOb=16, vOb=np.full(16, 4), A=A, b=b, lOb=lOb)
    return sc


def scene(kind, N):
    from obca_b200 import scenarios
    if kind == "cfg2":
        return scenarios.reverse_parking_batch(B, N, 0)
    if kind == "par4":
        return scenarios.parallel_parking_batch(B, N, 1, 4)
    if kind == "lot":
        return scenarios.parking_lot_batch(B, N, 0, 15)
    return sixteen_by_four(scenarios.parking_lot_batch(B, N, 0, 15))


# (scene, N, variant + fixTime): pinned K
PINS = {
    ("cfg2", 80, "sd0"): (1, 2, 3, 4, 5, 6), ("cfg2", 80, "d0"): (1, 2, 3, 4, 5, 6),
    ("cfg2", 80, "sd1"): (1, 2, 3), ("cfg2", 80, "d1"): (1, 2, 3),
    ("cfg2", 4, "sd0"): (1, 2, 3), ("cfg2", 7, "sd0"): (1, 2, 3),
    ("par4", 128, "sd0"): (1, 2, 3), ("par4", 128, "d1"): (1, 2, 3),
    ("lot", 80, "sd0"): (1, 2, 3, 4, 5, 6), ("lot", 80, "d0"): (1, 2, 3),
    ("lot", 200, "sd0"): (1, 2, 3, 4, 5, 6), ("lot", 200, "d0"): (1, 2, 3),
    ("cfg2", 319, "sd0"): (1, 2, 3, 4, 5, 6), ("cfg2", 319, "d1"): (1, 2, 3),
    ("x16", 319, "sd0"): (1, 2, 3),
}
MIXED_NS = (4, 40, 128, 200, 319)
MIXED_K = (1, 2, 3)


@pytest.fixture(scope="module")
def P():
    import obca_b200
    if obca_b200.lib().obca_device_count() < 1:
        pytest.fail("pytest -m gpu needs a CUDA device (libobca has no CPU fallback)")
    from obca_b200 import parking
    return parking


@pytest.fixture(params=sorted(SCHEDULES))
def schedule(request):
    """Runs the test under one schedule: OBCA_MODE=1 (tail kernel) or OBCA_MODE=2, OBCA_TAIL_THRESH=0 (rounds only)."""
    old = {k: os.environ.get(k) for k in ENV_KEYS}
    try:
        for k in old:
            os.environ.pop(k, None)
        os.environ.update(SCHEDULES[request.param])
        yield request.param
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _oracle_one(args):
    """One oracle run (a process-pool task): the unpacked iterate after every K in Ks, and the log."""
    from oracle import ipm_ref
    from oracle.parking_solve import solve_parking
    x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fix, xWS, uWS, variant, lWS, nWS, Ks, max_iter = args
    o = ipm_ref.IpmOptions(max_iter=max_iter, linsolve="sparse", snapshots=tuple(Ks))
    _, res, nlp = solve_parking(x0, xF, N, Ts, L, ego, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fix, xWS, uWS, variant, lWS, nWS, o,
                                one_time_scale=True)
    return {K: nlp.lay.unpack(res.snaps.get(K, res.z)) for K in Ks}, [e["dw"] for e in res.log]


def oracle_runs(problems):
    """problems: argument tuples of _oracle_one.  Independent runs go to separate processes (spawned: no CUDA state inherited)."""
    n = min(len(problems), os.cpu_count() or 1, 8)
    if n <= 1:
        return [_oracle_one(p) for p in problems]
    with ProcessPoolExecutor(n, mp_context=multiprocessing.get_context("spawn")) as ex:
        return list(ex.map(_oracle_one, problems))


_CACHE = {}


def pinned_case(P, kind, N, vf):
    """The scene, the DualMultWS multipliers (from the library) and the oracle's runs of one pinned case, once per module."""
    key = (kind, N, vf)
    if key not in _CACHE:
        sc = scene(kind, N)
        fix = int(vf[-1])
        Ts = sc["Ts_fix"] if fix else sc["Ts"]
        lWS, nWS = P.dualmultws_batch(N, sc["nOb"], sc["vOb"], sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], sc["ego"])
        Ks = PINS[key]
        runs = oracle_runs([(sc["x0"][i], sc["xF"], N, Ts, sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"], sc["b"],
                             sc["rx"][i], sc["ry"][i], sc["ryaw"][i], fix, sc["xWS"][i], sc["uWS"][i], vf[:-1], lWS[i], nWS[i], Ks, max(Ks))
                            for i in range(B)])
        _CACHE[key] = (sc, Ts, lWS, nWS, runs)
    return _CACHE[key]


def opts(K):
    import obca_b200
    o = obca_b200.default_opts(retry=0)
    o.max_iter = K
    return o


def compare(got, ref, what):
    """got: library outputs of one problem in the Julia shapes (xp 4 x NS, ...); ref: the oracle's unpacked iterate."""
    xp, up, ts, lp, np_, _ = ref
    sp = 1 + max(np.abs(xp).max(), np.abs(up).max(), np.abs(ts).max())
    sd = 1 + max(np.abs(lp).max(), np.abs(np_).max())
    ep = max(np.abs(got["xp"] - xp).max(), np.abs(got["up"] - up).max(), np.abs(got["ts"] - ts).max()) / sp
    ed = max(np.abs(got["lp"] - lp).max(), np.abs(got["np"] - np_).max()) / sd
    assert ep < PRIMAL_TOL and ed < DUAL_TOL, f"{what}: primal {ep:.2e} (tol {PRIMAL_TOL}), dual {ed:.2e} (tol {DUAL_TOL})"


@pytest.mark.parametrize("kind,N,vf", sorted(PINS))
def test_iterates_match_oracle(P, schedule, kind, N, vf):
    sc, Ts, lWS, nWS, runs = pinned_case(P, kind, N, vf)
    fix = int(vf[-1])
    for K in PINS[(kind, N, vf)]:
        r = P.parking_solve_batch(sc["x0"], sc["xF"], N, Ts, sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"], sc["b"],
                                  sc["rx"], sc["ry"], sc["ryaw"], fix, sc["xWS"], sc["uWS"], 1 if vf[:-1] == "sd" else 0, lWS, nWS, opts(K))
        for i in range(B):
            got = {k: r[k][i] for k in ("xp", "up", "ts", "lp", "np")}
            compare(got, runs[i][0][K], f"{kind} N={N} {vf} {schedule} problem {i} after K={K}")


def test_mixed_batch_iterates_match_oracle(P, schedule):
    """Horizons 4, 40, 128, 200 and 319 in one padded batch (obca_parking_solve_mixed): every problem follows its own
    oracle run."""
    from obca_b200 import scenarios
    sc = scenarios.reverse_parking_mixed_batch(len(MIXED_NS), seed=3, Ns=MIXED_NS)
    if "mixed" not in _CACHE:
        lw = [P.dualmultws_batch(int(n), sc["nOb"], sc["vOb"], sc["A"], sc["b"], sc["rx"][i][None], sc["ry"][i][None],
                                 sc["ryaw"][i][None], sc["ego"]) for i, n in enumerate(MIXED_NS)]
        lWS = [a[0][0] for a in lw]; nWS = [a[1][0] for a in lw]
        runs = oracle_runs([(sc["x0"][i], sc["xF"], int(n), sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"],
                             sc["b"], sc["rx"][i], sc["ry"][i], sc["ryaw"][i], 0, sc["xWS"][i], sc["uWS"][i], "sd", lWS[i], nWS[i],
                             MIXED_K, max(MIXED_K)) for i, n in enumerate(MIXED_NS)])
        _CACHE["mixed"] = (lWS, nWS, runs)
    lWS, nWS, runs = _CACHE["mixed"]
    for K in MIXED_K:
        r = P.parking_solve_mixed(sc["x0"], sc["xF"], sc["Ns"], sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"],
                                  sc["b"], sc["rx"], sc["ry"], sc["ryaw"], 0, sc["xWS"], sc["uWS"], 1, lWS, nWS, opts(K))
        for i, n in enumerate(MIXED_NS):
            got = {k: r[k][i] for k in ("xp", "up", "ts", "lp", "np")}
            compare(got, runs[i][0][K], f"mixed problem {i} (N={n}) {schedule} after K={K}")


# one pinned case per formulation and per half-space bound of the kernel instances (VM = 2: at most 2 half-spaces per obstacle,
# config 2 and the parallel scene; VM = 4: the lot) whose oracle run corrects the inertia inside the pinned window.  Config 2
# at N = 80 in Dist with free time corrects none by K = 6; with fixed time, start pose 0 of reverse_parking_batch(8, 80, 0)
# (x0 = (2.74, 8.13)) does at iteration 3 (dw = 1)
INERTIA = {("sd", 2): ("par4", 128, "sd0"), ("sd", 4): ("lot", 80, "sd0"), ("d", 2): ("cfg2", 80, "d1"), ("d", 4): ("lot", 200, "d0")}


@pytest.mark.parametrize("variant,vm", sorted(INERTIA))
def test_pinned_window_runs_inertia_correction(P, variant, vm):
    kind, N, vf = INERTIA[(variant, vm)]
    sc, _, _, _, runs = pinned_case(P, kind, N, vf)
    assert vf[:-1] == variant and (2 if int(np.max(sc["vOb"])) <= 2 else 4) == vm
    K = max(PINS[(kind, N, vf)])
    hits = [(i, it) for i, run in enumerate(runs) for it, dw in enumerate(run[1][:K]) if dw > 0]
    assert hits, f"{kind} N={N} {vf}: no inertia correction in the first {K} iterations"


def test_pinned_window_grows_dw_by_kw_plus(P):
    """A correction after an earlier one starts at kw_minus * dw_last and grows by kw_plus: on the lot at N = 80 (SD), problem 0,
    iteration 4 tries 0.333 / 3 and takes 0.889 = 0.111 * 8, inside the pinned window."""
    import obca_b200
    o = obca_b200.default_opts()
    _, _, _, _, runs = pinned_case(P, "lot", 80, "sd0")
    K = max(PINS[("lot", 80, "sd0")])
    grown = []
    for i, run in enumerate(runs):
        last = 0.0
        for it, dw in enumerate(run[1][:K]):
            if dw > 0 and last > 0 and dw > 1.5 * max(o.dw_min, o.kw_minus * last):
                grown.append((i, it + 1))
            last = dw if dw > 0 else last
    assert (0, 4) in grown, grown


def _oracle_converged(args):
    from oracle import ipm_ref
    from oracle.parking_solve import solve_parking
    out, res, _ = solve_parking(*args, ipm_ref.IpmOptions(linsolve="sparse"), one_time_scale=True)
    return out, res.status, res.iters


@pytest.mark.parametrize("N", [80, 319])
def test_converged_point_and_iteration_count_match_oracle(P, N):
    """At the default max_iter: the problems of config 2 that the oracle solves converge where it does (the tolerances of
    test_gpu_parking.test_matches_oracle_golden) within 3 iterations of it.  Measured the kernels' way the oracle also takes the
    kernels' iteration count (the pose of reverse_parking_batch(1, N, 0): 85 at N = 80, 56 at N = 319; measured the reference
    formulation's way, 89 and 89).  Problems that run out of iterations must do so on both sides."""
    sc = scene("cfg2", N)
    lWS, nWS = P.dualmultws_batch(N, sc["nOb"], sc["vOb"], sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], sc["ego"])
    r = P.parking_solve_batch(sc["x0"], sc["xF"], N, sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"], sc["b"],
                              sc["rx"], sc["ry"], sc["ryaw"], 0, sc["xWS"], sc["uWS"], 1, lWS, nWS, opts(200))
    problems = [(sc["x0"][i], sc["xF"], N, sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"], sc["b"], sc["rx"][i],
                 sc["ry"][i], sc["ryaw"][i], 0, sc["xWS"][i], sc["uWS"][i], "sd", lWS[i], nWS[i]) for i in range(B)]
    n = min(B, os.cpu_count() or 1)
    with ProcessPoolExecutor(n, mp_context=multiprocessing.get_context("spawn")) as ex:
        ref = list(ex.map(_oracle_converged, problems))
    assert sum(status for _, status, _ in ref) >= B // 2
    for i, ((xp, up, ts, _, _, lp, np_), status, iters) in enumerate(ref):
        assert r["exitflag"][i] == (status == 1), (i, status, r["exitflag"][i])     # the same problems run out of iterations
        if status != 1:
            continue
        assert abs(int(r["iters"][i]) - iters) <= 3, (i, int(r["iters"][i]), iters)
        assert np.abs(r["xp"][i] - xp).max() < 2e-4 and np.abs(r["up"][i] - up).max() < 2e-4, i
        assert np.abs(r["ts"][i] - ts).max() < 1e-5, i
        assert np.abs(r["lp"][i] - lp).max() < 5e-3 and np.abs(r["np"][i] - np_).max() < 5e-3, i
