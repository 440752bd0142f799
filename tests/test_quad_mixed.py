"""Quadcopter problems with different horizons and sampling times in one batch (obca_quadcopter_solve_mixed), CPU side: the
kernel sources run through the development emulation in the padded layout of the mixed entry, the C-ABI validates the
per-problem horizons and sampling times, and the A*-planned fixture of the GPU tests is what the planner produces."""
import ctypes as C
import os

import numpy as np
import pytest

import emul
import emul_quad_mixed
from obca_b200 import scenarios

NS_MIX = [20, 12, 33, 33, 12, 20, 20]      # interleaved, not sorted; the last problem gets a sampling time of its own
NMAX = 40                                  # layout larger than every horizon of the batch
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "quad_astar_pairs.npz")


def _mixed_scenario():
    sc = scenarios.quadcopter_mixed_batch(len(NS_MIX), Ns=NS_MIX, seed=2)
    assert sc["Ts"][0] == sc["Ts"][5] == 1.0 and sc["Ts"][1] == 1.67 and sc["Ts"][2] == 0.61      # round(0.25 * 80 / N, 2)
    sc["Ts"] = sc["Ts"].copy()
    sc["Ts"][6] = 0.9                      # same N as problems 0 and 5, another Ts
    return sc


@pytest.mark.parametrize("variant", ["sd", "d"])
def test_emulated_quad_mixed_batch_equals_uniform_per_group(variant):
    """Every problem of a mixed batch (N in {12, 20, 33} interleaved, Ts per problem, arrays laid out for Nmax = 40, the batch's
    shared Ts NaN) gives the same bits as the uniform solve of its (N, Ts) group; the NaN padding of the inputs is never read
    and that of the outputs never written."""
    sc = _mixed_scenario()
    o = emul.default_opts(); o.max_iter = 300
    r = emul_quad_mixed.quad_solve_mixed(sc, NMAX, variant, o)
    keys = (("xp", 1), ("ts", 1), ("lp", 1), ("up", 0)) + ((("slack", 1),) if variant == "sd" else ())
    groups = {}
    for i, (N, Ts) in enumerate(zip(NS_MIX, sc["Ts"])):
        groups.setdefault((N, float(Ts)), []).append(i)
    assert len(groups) == 4
    for (N, Ts), idx in groups.items():
        g = dict(B=len(idx), N=N, Ts=Ts, R=sc["R"], obs=sc["obs"], x0=sc["x0"][idx], xF=sc["xF"][idx],
                 xWS=np.stack([sc["xWS"][i] for i in idx]), timeWS=1.0)
        u = emul.quad_solve_batch(g, variant, o)
        for k, i in enumerate(idx):
            for key, ext in keys:
                a = r[key][i]
                cut, pad = (a[:N + ext], a[N + ext:]) if a.ndim == 1 else (a[:, :N + ext], a[:, N + ext:])
                assert np.array_equal(cut, u[key][k]), (key, i, N)
                assert np.isnan(pad).all(), (key, i, N)
            assert r["iters"][i] == u["iters"][k] and r["status"][i] == u["status"][k] and r["err"][i] == u["err"][k], (i, N)
    assert (r["status"] == 1).sum() >= 4


def _mixed_args(B, Nb, Nmax, Tsb):
    """Well-formed argument list of obca_quadcopter_solve_mixed for B config-4 problems laid out for Nmax."""
    sc = scenarios.quadcopter_scenario()
    NS = Nmax + 1
    keep = dict(x0=np.zeros((B, 12)), xF=np.zeros((B, 12)), ob=np.ascontiguousarray(sc["obs"], dtype=float),
                xw=np.zeros((B, NS, 12)), xp=np.zeros((B, NS, 12)), up=np.zeros((B, Nmax, 4)), ts=np.zeros((B, NS)),
                lp=np.zeros((B, NS, 30)), sl=np.zeros((B, NS, 5)), ef=np.zeros(B, np.int32), it=np.zeros(B, np.int32),
                err=np.zeros(B), sec=np.zeros(1), Nb=None if Nb is None else np.ascontiguousarray(Nb, dtype=np.int32),
                Tsb=None if Tsb is None else np.ascontiguousarray(Tsb, dtype=float))
    p = lambda a: None if a is None else a.ctypes.data_as(C.c_void_p)
    k = keep
    args = [C.c_int(B), p(k["Nb"]), C.c_int(Nmax), p(k["x0"]), p(k["xF"]), p(k["Tsb"]), C.c_double(0.25), p(k["ob"]), p(k["xw"]),
            C.c_double(1.0), C.c_int(1), None, p(k["xp"]), p(k["up"]), p(k["ts"]), p(k["lp"]), p(k["sl"]), p(k["ef"]), p(k["it"]),
            p(k["err"]), p(k["sec"])]
    return args, keep


def _check_args(args, keep):
    """obca_check_quadcopter_mixed's argument list over the same arrays (x = xp, u = up, timeScale = ts, lambda = lp)."""
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    return [args[0], args[1], args[2], args[12], args[13], args[14], args[3], args[4], args[5], args[15], args[7], args[6], None,
            p(keep["ef"]), p(keep["err"])]


def test_mixed_entries_reject_bad_horizons_and_sampling_times():
    import obca_b200
    lib = obca_b200.lib()
    ok_ts = [0.2, 0.2, 0.2]
    for Nb, Nmax, Tsb, what in ((None, 40, ok_ts, b"Nb"), ([12, 1, 30], 40, ok_ts, b"Nb[1]"), ([12, 41, 30], 40, ok_ts, b"Nb[1]"),
                                ([12, 20, 30], 20, ok_ts, b"Nb[2]"), ([12, 20, 30], 40, None, b"Tsb"),
                                ([12, 20, 30], 40, [0.2, np.nan, 0.2], b"Tsb[1]"), ([12, 20, 30], 40, [0.2, 0.2, np.inf], b"Tsb[2]"),
                                ([12, 20, 30], 40, [0.0, 0.2, 0.2], b"Tsb[0]"), ([12, 20, 30], 40, [0.2, -0.1, 0.2], b"Tsb[1]")):
        args, keep = _mixed_args(3, Nb, Nmax, Tsb)
        assert lib.obca_quadcopter_solve_mixed(*args) == -1, (Nb, Nmax, Tsb)
        assert what in lib.obca_last_error(), lib.obca_last_error()
        assert not keep["xp"].any() and not keep["ef"].any() and not keep["err"].any()
        assert lib.obca_check_quadcopter_mixed(*_check_args(args, keep)) == -1, (Nb, Nmax, Tsb)
        assert what in lib.obca_last_error(), lib.obca_last_error()
        assert not keep["ef"].any() and not keep["err"].any()


def test_mixed_entry_long_horizon_and_no_device_like_the_uniform_entry():
    """Nmax + 1 > 128 is answered like the uniform entry at N = Nmax; without a device a well-formed call is refused."""
    import obca_b200
    lib = obca_b200.lib()
    args, _ = _mixed_args(2, [130, 40], 130, [0.15, 0.5])
    uni = args[:1] + args[2:5] + [C.c_double(0.15)] + args[6:]
    assert lib.obca_quadcopter_solve_mixed(*args) == lib.obca_quadcopter_solve_batch(*uni)
    if lib.obca_device_count() > 0:
        pytest.skip("CUDA device present")
    args, keep = _mixed_args(3, [12, 40, 30], 40, [1.67, 0.5, 0.67])
    assert lib.obca_quadcopter_solve_mixed(*args) == -2 and b"no CUDA device" in lib.obca_last_error()
    assert lib.obca_check_quadcopter_mixed(*_check_args(args, keep)) == -2


def test_planned_fixture_is_what_the_planner_gives():
    """tests/golden/quad_astar_pairs.npz (tests/golden/make_quad_astar.py): the pairs are those of quadcopter_batch(12, seed=2),
    and two of them re-planned by the 3-D A* give exactly the stored N, Ts and warm start."""
    from obca_b200.planner.a_star_3d import plan_quadcopter_warm_start
    g = np.load(GOLDEN)
    sc = scenarios.quadcopter_batch(12, seed=2)
    assert np.array_equal(g["x0"], sc["x0"][:8]) and np.array_equal(g["xF"], sc["xF"][:8])
    assert len(set(g["N"].tolist())) >= 5 and g["N"].max() <= 127
    for i in (0, 3):
        p = plan_quadcopter_warm_start(g["x0"][i], g["xF"][i], sc["Ts80"])
        N = int(g["N"][i])
        assert p["N"] == N and p["Ts"] == g["Ts"][i]
        assert np.array_equal(p["xWS"], g["xWS"][i][:, :N + 1]) and np.isnan(g["xWS"][i][:, N + 1:]).all()
