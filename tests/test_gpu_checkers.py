"""The constraint-checker kernels (k_check: ParkingConstraints + the strict audit; k_quad_check: constrSatisfaction) against the
oracle (oracle/checkers.py) on the catalogue of tests/checker_cases.py, batched: every problem of a batch is a feasible base plus one
change -- a group just inside or just outside its threshold, a quirk of the reference, or a NaN / +-Inf entry -- at stage positions
on every lane, warp and pass of the 128-thread reduction.  The uniform, mixed-horizon (NaN in all padding) and tensor entries; and
the in-solver verdict of the parking retry path against the oracle."""

import numpy as np
import pytest

import checker_cases as cc

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def lib():
    import obca_b200
    if obca_b200.lib().obca_device_count() < 1:
        pytest.fail("pytest -m gpu needs a CUDA device (libobca has no CPU fallback)")
    return obca_b200


def _stack(cases, key):
    return np.stack([q[key] for _, q in cases])


def _park_kernel(cases, p):
    from obca_b200 import parking
    sl = _stack(cases, "sl") if p.get("sl") is not None else None
    args = (_stack(cases, "x0"), _stack(cases, "xF"), p["N"], p["Ts"], p["L"], p["ego"], p["XYbounds"], p["nOb"], p["vOb"], p["A"],
            p["b"], _stack(cases, "x"), _stack(cases, "u"), _stack(cases, "l"), _stack(cases, "n"), _stack(cases, "timeScale"),
            p["fixTime"], p["sd"])
    return parking.check_parking_batch(*args, sl)


def _park_compare(cases, got):
    feas, e, strict = got
    bad = []
    for i, (name, q) in enumerate(cases):
        want = cc.park_oracle(q)
        if (feas[i], strict[i]) != (want[0], want[2]) or not np.array_equal(e[i], want[1]):
            bad.append((name, int(feas[i]), e[i].tolist(), int(strict[i]), want))
    assert not bad, (len(bad), bad[:8])


# every variant (fixTime, sd, sl passed) at N = 80; the horizons and obstacle shapes of the kernels' edges, a variant each in turn
_VARIANTS = [(f, sd, sl) for f in (0, 1) for sd in (0, 1) for sl in ((0, 1) if sd else (0,))]
_SHAPES = [(2, [4, 4, 4]), (4, [2, 2, 1, 1]), (127, [3, 4, 4]), (128, [2, 2, 1, 1]), (129, [4] * 16), (255, [4, 4, 4]),
           (256, [2, 2, 1, 1]), (319, [4] * 16)]
PARK = [(80, [2, 2, 1, 1], *v, None) for v in _VARIANTS]
PARK += [(N, vOb, *_VARIANTS[i % len(_VARIANTS)], 120 if len(vOb) == 16 else 400) for i, (N, vOb) in enumerate(_SHAPES)]


@pytest.mark.parametrize("N,vOb,fix,sd,sl,most", PARK)
def test_parking_checker_matches_oracle(lib, N, vOb, fix, sd, sl, most):
    p = cc.park_base(N, vOb, fix, sd, sl)
    cases = [("base", p)] + cc.park_cases(p)
    cases = cases[:1] + (cc.thin(cases[1:], most) if most else cases[1:])
    assert cc.park_oracle(p) == (1, pytest.approx(np.ones(7)), 1)
    _park_compare(cases, _park_kernel(cases, p))


@pytest.mark.parametrize("N,vOb,fix,sd,sl", [(2, [4, 4, 4], 0, 1, 1), (4, [2, 2, 1, 1], 1, 1, 0), (80, [3, 4, 4], 1, 0, 0),
                                         (129, [2, 2, 1, 1], 0, 0, 0), (256, [4, 4, 4], 0, 1, 0), (319, [4] * 16, 1, 1, 1)])
def test_parking_strict_box_matches_oracle(lib, N, vOb, fix, sd, sl):
    """The strict audit's X / Y box alone decides (tests/checker_cases.park_box_cases): the reference passes every case, the
    strict audit flips between just inside and just outside, at each stage position."""
    for base, cases in cc.park_box_cases(N, vOb, fix, sd, sl):
        cases = [("base", base)] + cases
        for name, q in cases[1:]:
            want = cc.park_oracle(q)
            k = int(name.split("k=")[1])
            assert want[0] == 1 and want[2] == (0 if " out " in name and 1 <= k <= N - 1 else 1), (name, want)
        _park_compare(cases, _park_kernel(cases, base))


@pytest.mark.parametrize("name,p", cc.park_golden_bases(), ids=lambda v: v if isinstance(v, str) else "")
def test_parking_checker_matches_oracle_on_goldens(lib, name, p):
    assert cc.park_oracle(p)[0] == 1
    cases = cc.park_golden_cases(p)
    _park_compare(cases, _park_kernel(cc.thin(cases, 100 if p["nOb"] > 4 or p["N"] > 80 else 400), p))


def _pad(a, NS, axis=-1):
    """a padded with NaN to NS entries along its stage axis."""
    w = [(0, 0)] * a.ndim
    w[axis] = (0, NS - a.shape[axis])
    return np.pad(a, w, constant_values=np.nan)


def test_parking_mixed_and_tensor_entries_with_nan_padding(lib):
    """obca_check_parking_mixed_dev with three horizons in one batch and NaN in every padding entry: the verdicts of the oracle on
    the truncated arrays (a read of the padding would show as a NaN).  The tensor entry of the uniform check gives the bits of its
    host twin on a batch of NaN cases."""
    import torch
    from obca_b200 import torch_ops
    vOb = [2, 2, 1, 1]
    allc, Ns = [], []
    for N in (80, 129, 255):
        p = cc.park_base(N, vOb, 0, 1, 1)
        cs = cc.thin([("base", p)] + cc.park_cases(p), 120)
        allc += cs; Ns += [N] * len(cs)
    Nmax = max(Ns); NS = Nmax + 1
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    st = lambda key, ns: np.stack([_pad(q[key], ns) for _, q in allc])
    x, u, l, n, ts, sl = st("x", NS), st("u", Nmax), st("l", NS), st("n", NS), st("timeScale", NS), st("sl", NS)
    p = cc.park_base(Nmax, vOb, 0, 1, 1)
    f, e, s = torch_ops.check_parking_mixed(d(_stack(allc, "x0")), d(_stack(allc, "xF")), d(np.array(Ns, np.int32)), p["Ts"], p["L"],
                                            p["ego"], p["XYbounds"], p["nOb"], vOb, p["A"], p["b"], d(x), d(u), d(l), d(n), d(ts), 0, 1,
                                            sl=d(sl))
    torch.cuda.synchronize()
    _park_compare(allc, (f.cpu().numpy(), e.cpu().numpy(), s.cpu().numpy()))
    # the tensor entry against the host-pointer entry on NaN cases of one horizon
    p = cc.park_base(129, vOb, 1, 1, 1)
    cs = [c for c in cc.park_nonfinite_cases(p, every=2)]
    host = _park_kernel(cs, p)
    dev = torch_ops.check_parking_batch(d(_stack(cs, "x0")), d(_stack(cs, "xF")), 129, p["Ts"], p["L"], p["ego"], p["XYbounds"], p["nOb"],
                                        vOb, p["A"], p["b"], d(_stack(cs, "x")), d(_stack(cs, "u")), d(_stack(cs, "l")),
                                        d(_stack(cs, "n")), d(_stack(cs, "timeScale")), 1, 1, sl=d(_stack(cs, "sl")))
    torch.cuda.synchronize()
    for h, t in zip(host, dev):
        assert np.array_equal(h, t.cpu().numpy())
    _park_compare(cs, host)


# ---- quadcopter ------------------------------------------------------------------------------------------------------------------

def _quad_kernel(cases, p):
    from obca_b200 import quadcopter
    return quadcopter.check_quadcopter_batch(_stack(cases, "x"), _stack(cases, "u"), _stack(cases, "timeScale"), _stack(cases, "x0"),
                                             _stack(cases, "xF"), p["Ts"], _stack(cases, "lam"), p["obs"], p["R"])


def _quad_compare(cases, got):
    feas, worst = got
    bad = []
    for i, (name, q) in enumerate(cases):
        ok, w = cc.quad_oracle(q)
        if feas[i] != ok or not cc.same_worst(float(worst[i]), w):
            bad.append((name, int(feas[i]), float(worst[i]), ok, w))
    assert not bad, (len(bad), bad[:8])


@pytest.mark.parametrize("N,most", [(2, None), (40, None), (127, 400), (128, 400), (129, 400), (511, 120)])
def test_quadcopter_checker_matches_oracle(lib, N, most):
    p = cc.quad_base(N)
    cases = [("base", p)] + cc.quad_cases(p)
    cases = cases[:1] + (cc.thin(cases[1:], most) if most else cases[1:])
    assert cc.quad_oracle(p)[0] == 1
    _quad_compare(cases, _quad_kernel(cases, p))


@pytest.mark.parametrize("N", [2, 40, 128, 129, 511])
def test_quadcopter_box_matches_oracle(lib, N):
    """Each box group alone decides (tests/checker_cases.quad_box_cases): worst is 1.0 just outside a bound, below 1e-6 just
    inside."""
    base, cases = cc.quad_box_cases(N)
    cases = [("base", base)] + cases
    for name, q in cases[1:]:
        ok, w = cc.quad_oracle(q)
        assert (ok, w == 1.0) == ((0, True) if " out" in name else (1, False)) and (ok == 0 or w < 1e-6), (name, ok, w)
    _quad_compare(cases, _quad_kernel(cases, base))


@pytest.mark.parametrize("name,p", cc.quad_golden_bases(), ids=lambda v: v if isinstance(v, str) else "")
def test_quadcopter_checker_matches_oracle_on_goldens(lib, name, p):
    assert cc.quad_oracle(p)[0] == 1
    cases = cc.quad_golden_cases(p)
    _quad_compare(cases, _quad_kernel(cases, p))


def test_quadcopter_mixed_and_tensor_entries_with_nan_padding(lib):
    """obca_check_quadcopter_mixed_dev with three horizons and sampling times in one batch, NaN in every padding entry: the oracle's
    verdicts on the truncated arrays, and worst bit-identical to the uniform entry of each horizon."""
    import torch
    from obca_b200 import torch_ops
    allc, Ns, Tss, uni = [], [], [], []
    for N, Ts in ((40, 0.2), (128, 0.15), (129, 0.25)):
        p = cc.quad_base(N, Ts)
        cs = cc.thin([("base", p)] + cc.quad_cases(p), 150)
        allc += cs; Ns += [N] * len(cs); Tss += [Ts] * len(cs)
        uni.append(_quad_kernel(cs, p))
    Nmax = max(Ns); NS = Nmax + 1
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    st = lambda key, ns: np.stack([_pad(q[key], ns) for _, q in allc])
    f, w = torch_ops.check_quadcopter_mixed(d(st("x", NS)), d(st("u", Nmax)), d(st("timeScale", NS)), d(_stack(allc, "x0")),
                                            d(_stack(allc, "xF")), d(np.array(Ns, np.int32)), d(np.array(Tss)), d(st("lam", NS)),
                                            allc[0][1]["obs"], allc[0][1]["R"])
    torch.cuda.synchronize()
    f, w = f.cpu().numpy(), w.cpu().numpy()
    _quad_compare(allc, (f, w))
    uf, uw = np.concatenate([u[0] for u in uni]), np.concatenate([u[1] for u in uni])
    assert np.array_equal(f, uf) and np.array_equal(w.view(np.int64), uw.view(np.int64))
    # the tensor entry of the uniform check against its host twin on NaN cases
    p = cc.quad_base(128)
    cs = [c for c in cc.quad_cases(p, every=2) if "nan" in c[0] or "inf" in c[0]]
    host = _quad_kernel(cs, p)
    dev = torch_ops.check_quadcopter_batch(d(_stack(cs, "x")), d(_stack(cs, "u")), d(_stack(cs, "timeScale")), d(_stack(cs, "x0")),
                                           d(_stack(cs, "xF")), p["Ts"], d(_stack(cs, "lam")), p["obs"], p["R"])
    torch.cuda.synchronize()
    assert np.array_equal(host[0], dev[0].cpu().numpy()) and np.array_equal(host[1].view(np.int64), dev[1].cpu().numpy().view(np.int64))


# ---- the retry decision inside the parking solver --------------------------------------------------------------------------------

def _opts(**kw):
    import obca_b200
    o = obca_b200.default_opts()
    for k, v in kw.items():
        setattr(o, k, v)
    return o


def _solve(sc, sd, opts):
    from obca_b200 import parking
    return parking.parking_solve_batch(sc["x0"], sc["xF"], sc["N"], sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"],
                                       sc["A"], sc["b"], sc["rx"], sc["ry"], sc["ryaw"], 0, sc["xWS"], sc["uWS"], sd, None, None, opts)


def _oracle_verdict(sc, r, i, sd):
    from oracle import checkers
    return checkers.ParkingConstraints(sc["x0"][i], sc["xF"], sc["N"], sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"],
                                       sc["A"], sc["b"], r["xp"][i], r["up"][i], r["lp"][i], r["np"][i], r["ts"][i], 0, sd)


def test_retry_decision_signed_dist_matches_oracle(lib):
    """ParkingSignedDist.jl:278-283: after a second failure the exitflag is ParkingConstraints (sd = 1) on the returned point --
    the oracle's verdict, for every problem the checker decided (config 2, iteration limits that force failures)."""
    from obca_b200 import scenarios
    sc = scenarios.reverse_parking_batch(160, 80, seed=11)
    decided = 0
    for K in (20, 45):
        r0 = _solve(sc, 1, _opts(max_iter=K, retry=0))
        r1 = _solve(sc, 1, _opts(max_iter=K, retry=1))
        both = (r0["exitflag"] != 1) & (r1["iters"] - r0["iters"] == K) & (r1["kkt_err"] > 1e-5)
        for i in np.flatnonzero(both):
            assert r1["exitflag"][i] == _oracle_verdict(sc, r1, i, 1), i
        decided += int(both.sum())
    assert decided > 0


def test_retry_decision_dist_and_q4_match_oracle(lib):
    """ParkingDist.jl:245-289: the accept / re-solve choice after the first failure is ParkingConstraints (sd = 0) on the first
    attempt's point, and after a second failure the exitflag is its verdict (q4 = 0) or the inverse (q4 = 1) -- both the oracle's.
    Two iteration limits, so that both choices occur."""
    from obca_b200 import scenarios
    sc = scenarios.reverse_parking_batch(160, 80, seed=12)
    n_acc = n_res = n_both = 0
    for K in (30, 45):
        r0 = _solve(sc, 0, _opts(max_iter=K, retry=0))
        ra = _solve(sc, 0, _opts(max_iter=K, retry=1, q4=0))
        rb = _solve(sc, 0, _opts(max_iter=K, retry=1, q4=1))
        for i in np.flatnonzero(r0["exitflag"] != 1):
            fa, fb = int(ra["exitflag"][i]), int(rb["exitflag"][i])
            if _oracle_verdict(sc, r0, i, 0) == 1:                                     # :259-262: accepted, no second solve
                assert (fa, fb) == (1, 1) and ra["iters"][i] == r0["iters"][i] and np.array_equal(ra["xp"][i], r0["xp"][i]), i
                n_acc += 1
                continue
            n_res += 1                                                                 # :263: solved again from the last iterate
            assert ra["iters"][i] >= r0["iters"][i] and ra["iters"][i] - r0["iters"][i] <= K, i
            # the second attempt either converged (exitflag 1 whatever q4) or failed, and then the checker decided on its point
            # (:278-282); a second attempt that stopped at its first check (no iteration) falls in one of the two as well
            if (fa, fb) != (1, 1):
                v = _oracle_verdict(sc, ra, i, 0)
                assert (fa, fb) == (v, 1 - v), (i, fa, fb, v)
                n_both += 1
    assert n_acc > 0 and n_res > 0 and n_both > 0, (n_acc, n_res, n_both)
