"""CPU tests of the KERNEL SOURCES (obca_b200/csrc/*.cuh compiled by g++ into the development emulation of one CTA,
tests/emul/) against the oracle.  These run without a GPU; the same comparisons run through the C-ABI on the GPU in
tests/test_gpu_parking.py."""
import numpy as np
import pytest

import emul
from obca_b200 import scenarios
from oracle import checkers, dualmultws_ref, ipm_ref, kkt_check
from oracle.parking_solve import solve_parking

T = lambda a: np.transpose(a, (0, 2, 1))


def small_batch(N=16, B=2, seed=0):
    sc = scenarios.reverse_parking_scenario()
    rng = np.random.default_rng(seed)
    x0 = np.stack([rng.uniform(-10, 10, B), rng.uniform(6.5, 9.5, B), np.zeros(B), np.zeros(B)], 1)
    Ts = 48.0 / N
    rx = np.zeros((B, N + 1)); ry = np.zeros((B, N + 1)); ryaw = np.zeros((B, N + 1))
    xWS = np.zeros((B, N + 1, 4)); uWS = np.zeros((B, N, 2))
    for i in range(B):
        rx[i], ry[i], ryaw[i], xWS[i], uWS[i] = scenarios.warmstart_reverse(x0[i], sc["xF"], N, Ts, sc["L"])
    sc.update(B=B, N=N, x0=x0, rx=rx, ry=ry, ryaw=ryaw, xWS=xWS, uWS=uWS, Ts=Ts, Ts_fix=Ts)
    return sc


def test_dualws_kernel_math_vs_oracle(cfg2):
    lp, npp, d, its = emul.dualmultws_batch(cfg2)
    assert (its > 0).all() and its.max() <= 30
    g, off = dualmultws_ref.ego_geometry(cfg2["ego"])
    A = cfg2["A"]; b = cfg2["b"].ravel(); vo = np.concatenate([[0], np.cumsum(cfg2["vOb"])])
    for i in range(2):
        for k in range(0, 81, 8):
            pose = (cfg2["rx"][i, k], cfg2["ry"][i, k], cfg2["ryaw"][i, k])
            for j in range(3):
                Aj, bj = A[vo[j]:vo[j + 1]], b[vo[j]:vo[j + 1]]
                assert abs(dualmultws_ref.rect_poly_distance(pose, Aj, bj, g, off) - d[i, k, j]) < 2e-5
                lam, mu, dd = dualmultws_ref.solve_one(Aj, bj, pose, g, off)      # SLSQP restatement of DualMultWS.jl
                assert abs(dd - d[i, k, j]) < 2e-5
                assert np.abs(lam - lp[i, k, vo[j]:vo[j + 1]]).max() < 2e-3 and np.abs(mu - npp[i, k, 4 * j:4 * j + 4]).max() < 2e-3


def _oracle_factorizations(log):
    """Factorizations the oracle's inertia correction needed in the logged iterations (Algorithm IC of ipm_ref.solve with
    the default dw_first, kw_minus, kw_plus, kw_plus_first), to set against the emulation's count."""
    n, last = 0, 0.0
    for e in log:
        if e["dw"] > 0:
            start, grow = (1e-4, 100.0) if last == 0.0 else (max(1e-12, last / 3.0), 8.0)
            n += 1 + int(round(np.log(e["dw"] / start) / np.log(grow)))
            last = e["dw"]
        n += 1
    return n


# the shapes of tests/test_gpu_newton_iterates.py (scene, N): its problem 0 against the sparse oracle for K <= 3
GPU_SHAPES = [("sd", 0, s) for s in (("cfg2", 4), ("cfg2", 7), ("par4", 128), ("lot", 80), ("lot", 200), ("cfg2", 319), ("x16", 319))] + \
             [("d", 1, ("cfg2", 80)), ("d", 0, ("lot", 200)), ("d", 1, ("par4", 128))]


@pytest.mark.parametrize("variant,fix,shape", [pytest.param(v, f, None, id=f"{v}-{f}") for v, f in (("sd", 0), ("d", 0), ("sd", 1), ("d", 1))] +
                         [pytest.param(v, f, s, id=f"{v}-{f}-{s[0]}{s[1]}") for v, f, s in GPU_SHAPES])
def test_iterates_track_generic_dense_ipm(variant, fix, shape):
    """K1+K3+K4 (fused eval, condensation, Riccati KKT solve, line search) against the oracle's generic dense
    Bunch-Kaufman KKT solve: same iterates for the first iterations, same solution at convergence.  With a shape: the
    first three iterates at the shapes the GPU pins (the sparse oracle, the same inertia corrections)."""
    if shape is not None:
        from test_gpu_newton_iterates import scene
        sc = scene(*shape)
        sc.update({k: sc[k][:1] for k in ("x0", "rx", "ry", "ryaw", "xWS", "uWS")}, B=1)     # problem 0 alone
        lp, npp, _, _ = emul.dualmultws_batch(sc)
        Ts = sc["Ts_fix"] if fix else sc["Ts"]
        _, res, nlp = solve_parking(sc["x0"][0], sc["xF"], sc["N"], Ts, sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"],
                                    sc["b"], sc["rx"][0], sc["ry"][0], sc["ryaw"][0], fix, sc["xWS"][0], sc["uWS"][0], variant, lp[0], npp[0],
                                    ipm_ref.IpmOptions(max_iter=3, linsolve="sparse", snapshots=(1, 2, 3)), one_time_scale=True)
        for K in (1, 2, 3):
            o = emul.default_opts(); o.max_iter = K
            r = emul.solve_batch(sc, fix, variant, o, lp, npp)
            xp, up, ts, lpo, npo, _ = nlp.lay.unpack(res.snaps[K])
            sp = 1 + max(np.abs(xp).max(), np.abs(up).max(), np.abs(ts).max())
            sd = 1 + max(np.abs(lpo).max(), np.abs(npo).max())
            assert max(np.abs(xp - r["xp"][0].T).max(), np.abs(up - r["up"][0].T).max(), np.abs(ts - r["ts"][0]).max()) < 1e-7 * sp, K
            assert max(np.abs(lpo - r["lp"][0].T).max(), np.abs(npo - r["np"][0].T).max()) < 1e-6 * sd, K
            assert r["nfact"][0] == _oracle_factorizations(res.log[:K]), K
        return
    sc = small_batch()
    lp, npp, _, _ = emul.dualmultws_batch(sc)
    i = 0
    for K, tol in ((1, 1e-6), (3, 1e-6), (400, 1e-7)):
        o = emul.default_opts(); o.max_iter = K
        r = emul.solve_batch(sc, fix, variant, o, lp, npp)
        out, res, nlp = solve_parking(sc["x0"][i], sc["xF"], sc["N"], sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], 3,
                                      sc["vOb"], sc["A"], sc["b"], sc["rx"][i], sc["ry"][i], sc["ryaw"][i], fix,
                                      sc["xWS"][i], sc["uWS"][i], variant, lp[i], npp[i], ipm_ref.IpmOptions(max_iter=K))
        xp, up, ts, ef, _, lpo, npo = out
        assert np.abs(xp - r["xp"][i].T).max() < tol and np.abs(up - r["up"][i].T).max() < tol
        assert np.abs(ts - r["ts"][i]).max() < tol
        assert np.abs(lpo - r["lp"][i].T).max() < 10 * tol and np.abs(npo - r["np"][i].T).max() < 10 * tol
        if K == 400:
            assert res.status == 1 and r["status"][i] == 1 and abs(res.iters - r["iters"][i]) <= 3


def test_config2_solutions_are_kkt_points_of_reference_nlp(cfg2):
    lp, npp, _, _ = emul.dualmultws_batch(cfg2)
    r = emul.solve_batch(cfg2, 0, "sd", None, lp, npp)
    assert (r["status"] == 1).all()
    rr = dict(xp=T(r["xp"]), up=T(r["up"]), ts=r["ts"], lp=T(r["lp"]), np=T(r["np"]), sl=T(r["sl"]))
    for i in (0, 3):
        e = kkt_check.reference_kkt_error(cfg2, i, rr)
        assert e["E0"] < 1e-5 and abs(e["E0"] - r["err"][i]) < 5e-6
        ok, e7 = checkers.ParkingConstraints(cfg2["x0"][i], cfg2["xF"], 80, cfg2["Ts"], cfg2["L"], cfg2["ego"],
                                             cfg2["XYbounds"], 3, cfg2["vOb"], cfg2["A"], cfg2["b"], rr["xp"][i], rr["up"][i],
                                             rr["lp"][i], rr["np"][i], rr["ts"][i], 0, 1, return_e=True)
        assert ok == 1, e7
        ok2, worst = checkers.strict_check(cfg2["x0"][i], cfg2["xF"], 80, cfg2["Ts"], cfg2["L"], cfg2["ego"], cfg2["XYbounds"], 3,
                                           cfg2["vOb"], cfg2["A"], cfg2["b"], rr["xp"][i], rr["up"][i], rr["lp"][i], rr["np"][i],
                                           rr["ts"][i], 0, 1, rr["sl"][i])
        assert ok2 == 1, worst


def test_warp_kkt_lane_code_matches_serial_riccati(tmp_path):
    """K3: the lane functions of the warp-cooperative sweep (kl_step1/2/3, run for 32 emulated lanes) and the plain
    serial Riccati recursion (riccati_step) give the same Newton steps."""
    import os, subprocess, sys
    script = tmp_path / "run.py"
    script.write_text(
        "import sys, numpy as np\n"
        f"sys.path.insert(0, {repr(os.path.join(os.path.dirname(__file__), 'emul'))}); sys.path.insert(0, {repr(os.path.dirname(os.path.dirname(__file__)))})\n"
        "import emul\nfrom obca_b200 import scenarios\n"
        "sc = scenarios.reverse_parking_batch(4, 80, 0)\n"
        "lp, npp, _, _ = emul.dualmultws_batch(sc)\n"
        "o = emul.default_opts(); o.max_iter = 3\n"
        "r = emul.solve_batch(sc, 0, 'sd', o, lp, npp)\n"
        "np.savez(sys.argv[1], xp=r['xp'], up=r['up'], lp=r['lp'], np=r['np'], ts=r['ts'])\n")
    outs = []
    for mode in ("warp", "serial"):
        env = dict(os.environ)
        if mode == "serial":
            env["OBCA_EMUL_SERIAL_KKT"] = "1"
        f = str(tmp_path / f"{mode}.npz")
        subprocess.check_call([sys.executable, str(script), f], env=env)
        outs.append(np.load(f))
    for key in ("xp", "up", "lp", "np", "ts"):
        assert np.abs(outs[0][key] - outs[1][key]).max() < 1e-7, key   # round-off x 1/dc (terminal penalty 1e9)


def test_maximum_shape_on_the_host_build():
    """Largest shape the kernels are built for: N + 1 = 128 stages, 5 obstacles, up to 4 half-spaces per obstacle (the VM = 4
    instantiation with ragged counts 2, 2, 1, 4, 4): converges, KKT point of the reference NLP, passes the verbatim checker."""
    N = 127
    sc = scenarios.reverse_parking_batch(2, N, seed=4)

    def box(xl, xu, yl, yu):                      # {x : A x <= b}
        return np.array([[1.0, 0], [-1, 0], [0, 1], [0, -1]]), np.array([[xu], [-xl], [yu], [-yl]])
    A1, b1 = box(11, 13, 6, 8); A2, b2 = box(-13, -11, 6, 8)
    sc["A"] = np.vstack([sc["A"], A1, A2]); sc["b"] = np.vstack([np.asarray(sc["b"]).reshape(-1, 1), b1, b2])
    sc["vOb"] = np.array(list(sc["vOb"]) + [4, 4]); sc["nOb"] = 5
    lp, npp, _, _ = emul.dualmultws_batch(sc)
    r = emul.solve_batch(sc, 0, "sd", None, lp, npp)
    assert (r["status"] == 1).all() and r["lp"].shape == (2, N + 1, 13) and r["np"].shape == (2, N + 1, 20)
    rr = dict(xp=T(r["xp"]), up=T(r["up"]), ts=r["ts"], lp=T(r["lp"]), np=T(r["np"]), sl=T(r["sl"]))
    e = kkt_check.reference_kkt_error(sc, 0, rr)
    assert e["E0"] < 1e-5
    assert checkers.ParkingConstraints(sc["x0"][0], sc["xF"], N, sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], 5, sc["vOb"], sc["A"], sc["b"],
                                       rr["xp"][0], rr["up"][0], rr["lp"][0], rr["np"][0], rr["ts"][0], 0, 1)
