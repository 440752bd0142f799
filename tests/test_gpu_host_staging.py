"""Host-pointer entries of libobca.so on the GPU, on the paths the Python wrappers never take: every optional output passed as NULL
gives the same required outputs, bit for bit, as the call that passes it; the host-pointer parking solve equals the device-pointer
one; and a small batch gives the same bits before and after a larger one has grown the staging buffer it reuses."""
import ctypes as C
import os
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "obca.h")


@pytest.fixture(scope="module")
def lib():
    import obca_b200
    if obca_b200.lib().obca_device_count() < 1:
        pytest.fail("pytest -m gpu needs a CUDA device (libobca has no CPU fallback)")
    return obca_b200.lib()


def arg_index(fn, param):
    """Position of the parameter `param` of the C function `fn` in include/obca.h."""
    proto = re.search(r"\b" + fn + r"\(([^)]*)\)", open(HEADER).read()).group(1)
    names = [re.findall(r"\w+", a)[-1] for a in proto.split(",")]
    return names.index(param)


class _Lib:
    """libobca.so with its function fn called with NULL for some of its parameters."""

    def __init__(self, real, fn, params):
        self._real, self._fn, self._pos = real, fn, {arg_index(fn, p) for p in params}

    def __getattr__(self, name):
        f = getattr(self._real, name)
        if name != self._fn:
            return f
        return lambda *args: f(*[None if i in self._pos else a for i, a in enumerate(args)])


def with_null(monkeypatch, lib, fn, params, call):
    """call() with the C function fn receiving NULL for params (the wrappers pass every pointer)."""
    from obca_b200 import _lib, parking, quadcopter
    proxy = _Lib(lib, fn, params)
    with monkeypatch.context() as m:
        for mod in (_lib, parking, quadcopter):
            m.setattr(mod, "lib", lambda: proxy)
        return call()


def assert_equal(a, b, keys):
    for k in keys:
        if isinstance(a[k], list):
            assert all(np.array_equal(x, y, equal_nan=True) for x, y in zip(a[k], b[k])), k
        else:
            assert np.array_equal(a[k], b[k], equal_nan=True), k


PARK_OUT = ("xp", "up", "ts", "lp", "np", "exitflag", "iters", "kkt_err")
QUAD_OUT = ("xp", "up", "ts", "lp", "exitflag", "iters", "kkt_err")


def park_batch(B, seed):
    from obca_b200 import scenarios
    return scenarios.reverse_parking_batch(B, 60, seed=seed)


def park_solve(sc):
    from obca_b200 import parking
    return parking.parking_solve_batch(sc["x0"], sc["xF"], 60, sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"],
                                       sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], 0, sc["xWS"], sc["uWS"])


def park_check(sc, r):
    from obca_b200 import parking
    return parking.check_parking_batch(sc["x0"], sc["xF"], 60, sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"],
                                       sc["A"], sc["b"], r["xp"], r["up"], r["lp"], r["np"], r["ts"], 0, 1, r["sl"])


def park_mixed():
    from obca_b200 import scenarios
    Ns = np.random.default_rng(7).choice((30, 45, 60), 12)
    return scenarios.reverse_parking_mixed_batch(12, Ns=Ns, seed=7)


def park_solve_mixed(sc):
    from obca_b200 import parking
    return parking.parking_solve_mixed(sc["x0"], sc["xF"], sc["Ns"], sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"],
                                       sc["vOb"], sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], 0, sc["xWS"], sc["uWS"])


def park_check_mixed(sc, r):
    from obca_b200 import parking
    return parking.check_parking_mixed(sc["x0"], sc["xF"], sc["Ns"], sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"],
                                       sc["vOb"], sc["A"], sc["b"], r["xp"], r["up"], r["lp"], r["np"], r["ts"], 0, 1, r["sl"])


def quad_batch(B, seed):
    from obca_b200 import scenarios
    return scenarios.quadcopter_batch(B, 60, seed=seed)


def quad_solve(sc):
    from obca_b200 import quadcopter
    return quadcopter.quadcopter_solve_batch(sc["x0"], sc["xF"], 60, sc["Ts"], sc["R"], sc["obs"], sc["xWS"], 1.0, 1)


def quad_check(sc, r):
    from obca_b200 import quadcopter
    return quadcopter.check_quadcopter_batch(r["xp"], r["up"], r["ts"], sc["x0"], sc["xF"], sc["Ts"], r["lp"], sc["obs"], sc["R"])


def quad_mixed():
    from obca_b200 import scenarios
    Ns = np.random.default_rng(8).choice((40, 70, 100), 8)
    return scenarios.quadcopter_mixed_batch(8, Ns=Ns, seed=8)


def quad_solve_mixed(sc):
    from obca_b200 import quadcopter
    return quadcopter.quadcopter_solve_mixed(sc["x0"], sc["xF"], sc["Ns"], sc["Ts"], sc["R"], sc["obs"], sc["xWS"], 1.0, 1)


def quad_check_mixed(sc, r):
    from obca_b200 import quadcopter
    return quadcopter.check_quadcopter_mixed(r["xp"], r["up"], r["ts"], sc["x0"], sc["xF"], sc["Ns"], sc["Ts"], r["lp"], sc["obs"],
                                             sc["R"])


def test_parking_solves_without_slacks(lib, monkeypatch):
    for fn, sc, solve in (("obca_parking_solve_batch", park_batch(8, 0), park_solve),
                          ("obca_parking_solve_mixed", park_mixed(), park_solve_mixed)):
        full = solve(sc)
        assert full["exitflag"].sum() > 0
        assert_equal(with_null(monkeypatch, lib, fn, ["sl"], lambda: solve(sc)), full, PARK_OUT)


def test_parking_checkers_without_counts_or_strict_audit(lib, monkeypatch):
    for fn, sc, solve, chk in (("obca_check_parking", park_batch(8, 1), park_solve, park_check),
                               ("obca_check_parking_mixed", park_mixed(), park_solve_mixed, park_check_mixed)):
        r = solve(sc)
        feas = chk(sc, r)[0]
        assert feas.any()
        for params in (["e"], ["strict"], ["e", "strict"]):
            assert np.array_equal(with_null(monkeypatch, lib, fn, params, lambda: chk(sc, r))[0], feas), (fn, params)


def test_quadcopter_solves_without_slacks(lib, monkeypatch):
    for fn, sc, solve in (("obca_quadcopter_solve_batch", quad_batch(6, 2), quad_solve),
                          ("obca_quadcopter_solve_mixed", quad_mixed(), quad_solve_mixed)):
        full = solve(sc)
        assert full["exitflag"].sum() > 0
        assert_equal(with_null(monkeypatch, lib, fn, ["slack"], lambda: solve(sc)), full, QUAD_OUT)


def test_quadcopter_checkers_without_worst(lib, monkeypatch):
    for fn, sc, solve, chk in (("obca_check_quadcopter", quad_batch(6, 3), quad_solve, quad_check),
                               ("obca_check_quadcopter_mixed", quad_mixed(), quad_solve_mixed, quad_check_mixed)):
        r = solve(sc)
        feas = chk(sc, r)[0]
        assert feas.any()
        assert np.array_equal(with_null(monkeypatch, lib, fn, ["worst"], lambda: chk(sc, r))[0], feas), fn


def test_dualmultws_without_distances(lib, monkeypatch):
    from obca_b200 import parking
    sc = park_batch(8, 4)
    call = lambda: parking.dualmultws_batch(60, sc["nOb"], sc["vOb"], sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], sc["ego"],
                                            want_d=True)
    full = call()
    got = with_null(monkeypatch, lib, "obca_dualmultws_batch", ["d"], call)
    assert np.array_equal(got[0], full[0]) and np.array_equal(got[1], full[1])


def test_planners_without_expansion_counts(lib, monkeypatch):
    from obca_b200 import scenarios
    from obca_b200.planner import device, native
    rng = np.random.default_rng(0)
    x0 = np.column_stack([rng.uniform(-9, 9, 16), rng.uniform(6.8, 9.3, 16), np.zeros(16)])
    ox, oy = native.obstacle_points("backwards")
    goal = scenarios.reverse_parking_scenario()["xF"]
    call = lambda: device.plan_raw(x0, goal, ox, oy, 0.6)
    full = call()
    assert (full["status"] == 0).any()
    got = with_null(monkeypatch, lib, "obca_plan_parking_warmstart_batch", ["expansions"], call)
    assert_equal(got, full, ("rx", "ry", "ryaw", "xWS", "uWS", "N", "status"))
    sc = scenarios.quadcopter_batch(8, seed=2)
    args = native.quadcopter_problem(sc["x0"], sc["xF"])
    call = lambda: device.plan_quadcopter_raw(*args)
    full = call()
    assert (full["status"] == 0).any()
    got = with_null(monkeypatch, lib, "obca_plan_quadcopter_warmstart_batch", ["expansions"], call)
    assert_equal(got, full, ("rx", "ry", "rz", "N", "status"))
    assert (got["expansions"] == -1).all()      # never copied in or out


def test_host_pointer_solve_equals_device_pointer_solve(lib):
    import torch
    from obca_b200 import _lib, parking
    sc = park_batch(16, 5)
    host = park_solve(sc)
    B, N = 16, 60
    NS = N + 1
    vOb, V, A, b = parking._shared(sc["nOb"], sc["vOb"], sc["A"], sc["b"])
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64)).cuda()
    T = lambda a: np.transpose(np.asarray(a, float), (0, 2, 1))
    ins = [dev(sc["x0"]), dev(np.broadcast_to(np.asarray(sc["xF"], float).reshape(-1, 4), (B, 4))),
           dev(np.reshape(sc["rx"], (B, NS))), dev(np.reshape(sc["ry"], (B, NS))), dev(np.reshape(sc["ryaw"], (B, NS))),
           dev(T(np.reshape(sc["xWS"], (B, -1, 4))[:, :NS])), dev(T(np.reshape(sc["uWS"], (B, -1, 2))[:, :N]))]
    z = lambda *s: torch.zeros(s, dtype=torch.float64, device="cuda")
    xp, up, ts, lp, npp, sl, err = z(B, NS, 4), z(B, N, 2), z(B, NS), z(B, NS, V), z(B, NS, 4 * sc["nOb"]), z(B, NS, sc["nOb"]), z(B)
    ef, it = (torch.zeros(B, dtype=torch.int32, device="cuda") for _ in range(2))
    p = lambda t: C.c_void_p(t.data_ptr())
    sec = np.zeros(1)
    o = _lib.default_opts()
    torch.cuda.synchronize()
    _lib.check(lib.obca_parking_solve_batch_dev(
        C.c_int(B), C.c_int(N), C.c_int(sc["nOb"]), _lib.ptr(vOb), _lib.ptr(A), _lib.ptr(b), p(ins[0]), p(ins[1]), C.c_double(sc["Ts"]),
        C.c_double(sc["L"]), _lib.ptr(_lib.f64(np.ravel(sc["ego"]))), _lib.ptr(_lib.f64(np.ravel(sc["XYbounds"]))), p(ins[2]), p(ins[3]),
        p(ins[4]), p(ins[5]), p(ins[6]), None, None, C.c_int(0), C.c_int(1), C.byref(o), p(xp), p(up), p(ts), p(lp), p(npp), p(sl),
        p(ef), p(it), p(err), _lib.ptr(sec)))
    got = dict(xp=T(xp.cpu()), up=T(up.cpu()), ts=ts.cpu().numpy(), lp=T(lp.cpu()), np=T(npp.cpu()), sl=T(sl.cpu()),
               exitflag=ef.cpu().numpy(), iters=it.cpu().numpy(), kkt_err=err.cpu().numpy())
    assert host["exitflag"].sum() > 0
    assert_equal(got, host, PARK_OUT + ("sl",))


def test_small_batch_after_a_larger_one(lib):
    """The staging buffer of a device only grows and is reused: a small batch gives the same bits before and after a larger one."""
    small, large = park_batch(4, 6), park_batch(96, 7)
    r1 = park_solve(small)
    c1 = park_check(small, r1)
    rl = park_solve(large)
    park_check(large, rl)
    r2 = park_solve(small)
    c2 = park_check(small, r1)
    assert_equal(r2, r1, PARK_OUT + ("sl",))
    assert all(np.array_equal(a, b) for a, b in zip(c1, c2))
    qs, ql = quad_batch(4, 8), quad_batch(64, 9)
    q1 = quad_solve(qs)
    k1 = quad_check(qs, q1)
    quad_check(ql, quad_solve(ql))
    q2 = quad_solve(qs)
    k2 = quad_check(qs, q1)
    assert_equal(q2, q1, QUAD_OUT + ("slack",))
    assert all(np.array_equal(a, b) for a, b in zip(k1, k2))
