"""The constraint checkers' sources (obca_check.cuh, quad_check_stage in obca_quad.cuh) on the host with the kernels' reduction
(tests/emul/emul_check.cpp), against the oracle (oracle/checkers.py) on the catalogue of tests/checker_cases.py: every flag of
ParkingConstraints, the strict audit, constrSatisfaction and its worst violation, at the thresholds, the quirks and NaN / +-Inf
entries.  Each case runs again with the merges in seeded random orders: the verdicts must not depend on the order.  Also pins the
oracle's own non-finite semantics on small hand-written cases."""
import numpy as np
import pytest

import checker_cases as cc
import emul_check
from oracle import checkers

SEEDS = (1, 2, 3)

# (N, vOb, fixTime, sd, sl passed, at most this many cases): every variant at N = 80, the shapes' edges in turn
PARK = [(80, [3, 4, 4], f, sd, sl, None) for f in (0, 1) for sd in (0, 1) for sl in ((0, 1) if sd else (0,))]
PARK += [(2, [4, 4, 4], 0, 1, 1, None), (4, [2, 2, 1, 1], 1, 0, 0, None), (129, [2, 2, 1, 1], 0, 1, 1, 400),
         (256, [4, 4, 4], 1, 1, 0, 250), (319, [4] * 16, 0, 0, 0, 60)]


def _park_equal(p, cases):
    bad = []
    for name, q in cases:
        want = cc.park_oracle(q)
        got = emul_check.check_parking(q)
        if got[0] != want[0] or not np.array_equal(got[1], want[1]) or got[2] != want[2]:
            bad.append((name, got, want))
        for s in SEEDS:
            again = emul_check.check_parking(q, seed=s)
            assert again[0] == got[0] and np.array_equal(again[1], got[1]) and again[2] == got[2], (name, s)
    assert not bad, bad[:10]


@pytest.mark.parametrize("N,vOb,fix,sd,sl,most", PARK)
def test_parking_checker_sources_match_oracle(N, vOb, fix, sd, sl, most):
    p = cc.park_base(N, vOb, fix, sd, sl)
    assert cc.park_oracle(p) == (1, pytest.approx(np.ones(7)), 1)
    cases = cc.park_cases(p)
    _park_equal(p, cc.thin(cases, most) if most else cases)


@pytest.mark.parametrize("N,vOb,fix,sd,sl", [(2, [4, 4, 4], 0, 1, 1), (80, [3, 4, 4], 1, 0, 0), (129, [2, 2, 1, 1], 0, 0, 0),
                                         (319, [4] * 16, 1, 1, 1)])
def test_parking_strict_box_sources_match_oracle(N, vOb, fix, sd, sl):
    """The strict audit's X / Y box alone decides: the reference passes every case, the strict audit flips between in and out."""
    for base, cases in cc.park_box_cases(N, vOb, fix, sd, sl):
        assert cc.park_oracle(base) == (1, pytest.approx(np.ones(7)), 1)
        for name, q in cases:
            want = cc.park_oracle(q)
            k = int(name.split("k=")[1])
            assert want[0] == 1 and want[2] == (0 if " out " in name and 1 <= k <= N - 1 else 1), (name, want)
        _park_equal(base, cases)


@pytest.mark.parametrize("name,p", cc.park_golden_bases(), ids=lambda v: v if isinstance(v, str) else "")
def test_parking_checker_sources_match_oracle_on_goldens(name, p):
    assert cc.park_oracle(p)[0] == 1
    _park_equal(p, cc.thin(cc.park_golden_cases(p), 80 if p["N"] > 80 else 400))


def _quad_equal(cases):
    bad = []
    for name, q in cases:
        want = cc.quad_oracle(q)
        got = emul_check.check_quadcopter(q)
        if got[0] != want[0] or not cc.same_worst(got[1], want[1]):
            bad.append((name, got, want))
        for s in SEEDS:
            assert emul_check.check_quadcopter(q, seed=s) == got, (name, s)
    assert not bad, bad[:10]


@pytest.mark.parametrize("N,most", [(2, None), (40, None), (128, 250), (511, 60)])
def test_quadcopter_checker_sources_match_oracle(N, most):
    p = cc.quad_base(N)
    assert cc.quad_oracle(p)[0] == 1
    cases = cc.quad_cases(p)
    _quad_equal(cc.thin(cases, most) if most else cases)


@pytest.mark.parametrize("N", [2, 129, 511])
def test_quadcopter_box_sources_match_oracle(N):
    """Each box group alone decides: worst is 1.0 just outside a bound and below 1e-6 just inside."""
    base, cases = cc.quad_box_cases(N)
    assert cc.quad_oracle(base)[0] == 1
    for name, q in cases:
        ok, w = cc.quad_oracle(q)
        assert (ok, w == 1.0) == ((0, True) if " out" in name else (1, False)) and (ok == 0 or w < 1e-6), (name, ok, w)
    _quad_equal(cases)


@pytest.mark.parametrize("name,p", cc.quad_golden_bases(), ids=lambda v: v if isinstance(v, str) else "")
def test_quadcopter_checker_sources_match_oracle_on_goldens(name, p):
    assert cc.quad_oracle(p)[0] == 1
    _quad_equal(cc.quad_golden_cases(p))


def test_parking_nan_is_rejected():
    """A NaN in one entry of a feasible trajectory: ParkingConstraints' maximum() propagates it, so the group fails."""
    p = cc.park_base(80, [3, 4, 4], 0, 1, 1)
    for key, idx in (("x", (2, 40)), ("u", (1, 0)), ("l", (0, 80)), ("timeScale", 7)):
        q = cc._copy(p, cc.PARK_KEYS); q[key][idx] = np.nan
        ok, e, st = emul_check.check_parking(q)
        assert (ok, st) == (0, 0) and e.sum() < 7
        assert cc.park_oracle(q)[0] == 0


def test_parking_fixed_time_reads_timescale():
    """ParkingConstraints.jl:47 checks |timeScale - 1| whatever fixTime is; the strict audit exempts fixed time."""
    p = cc.park_base(80, [3, 4, 4], 1, 0, 0)
    p["timeScale"] = np.zeros(81)
    ok, e, st = emul_check.check_parking(p)
    assert ok == 0 and list(e) == [0, 1, 1, 1, 1, 1, 1] and st == 1
    assert cc.park_oracle(p) == (0, pytest.approx(e), 1)


def test_quadcopter_nan_does_not_hide_a_violation():
    """A NaN group of constrSatisfaction never fails, but the other groups of its stage still do."""
    p = cc.quad_base(10)
    p["x"][6, 5] += 0.5
    p["lam"][29, 4] = p["lam"][29, 5] = np.nan
    ok, w = emul_check.check_quadcopter(p)
    assert ok == 0 and w > 0.1
    assert cc.quad_oracle(p) == (0, pytest.approx(w, rel=1e-12))


# ---- the oracle's own semantics --------------------------------------------------------------------------------------------------

def _args(p):
    return (p["x0"], p["xF"], p["N"], p["Ts"], p["L"], p["ego"], p["XYbounds"], p["nOb"], p["vOb"], p["A"], p["b"], p["x"], p["u"],
            p["l"], p["n"], p["timeScale"], p["fixTime"], p["sd"])


@pytest.mark.parametrize("key,idx,v", [("x", (2, 3), np.nan), ("u", (0, 3), np.nan), ("n", (1, 0), np.nan), ("l", (0, 2), np.nan),
                                       ("x", (0, 4), np.inf), ("u", (1, 3), -np.inf), ("sl", (2, 4), np.nan)])
def test_oracle_strict_check_propagates_non_finite(key, idx, v):
    p = cc.park_base(4, [3, 4, 4], 0, 1, 1)
    assert checkers.strict_check(*_args(p), sl=p["sl"]) == (1, 0.0)
    p[key][idx] = v
    with np.errstate(all="ignore"):
        ok, w = checkers.strict_check(*_args(p), sl=p["sl"])
    assert ok == 0 and (np.isnan(w) or w == np.inf)


def test_oracle_strict_check_nan_gives_nan():
    p = cc.park_base(4, [3, 4, 4], 0, 1, 1)
    p["x"][2, 2] = np.nan
    with np.errstate(all="ignore"):
        ok, w = checkers.strict_check(*_args(p), sl=p["sl"])
    assert ok == 0 and np.isnan(w)


def _qargs(q):
    return (q["x"], q["u"], q["timeScale"], q["x0"], q["xF"], q["Ts"], q["lam"], *q["obs"], q["R"])


def _neg(q):
    """-0.5 on two multipliers of obstacle 0 at stage 1 whose difference enters its rows: only the lambda group sees them."""
    q["lam"][1, 1] = q["lam"][4, 1] = -0.5


@pytest.mark.parametrize("change,ok,worst", [
    (lambda q: None, True, None),
    (lambda q: q["lam"].__setitem__((29, 1), np.nan), True, None),                                    # lambda group off, rows of o=4 NaN
    (lambda q: (_neg(q), q["lam"].__setitem__((29, 2), np.nan)), True, None),                         # the -0.5 is not seen
    (lambda q: _neg(q), False, 0.5),
    (lambda q: (q["x"].__setitem__((6, 2), 0.5), q["lam"].__setitem__((29, 1), np.nan)), False, 0.5),      # NaN does not mask
    (lambda q: q["u"].__setitem__((0, 1), np.inf), False, 1.0),                                        # box: 1.0; dynamics: inf * 0
    (lambda q: (q["u"].__setitem__((0, 1), 8.0), q["u"].__setitem__((1, 1), np.nan)), True, None),    # the upper group's max is NaN
    (lambda q: q["x0"].__setitem__(0, np.nan), True, None),                                            # norm(NaN) > tol is false
    (lambda q: q["lam"].__setitem__((3, 1), np.inf), False, np.inf),                                   # norm row inf; distance rows NaN
])
def test_oracle_constr_worst(change, ok, worst):
    q = cc.quad_base(3)
    change(q)
    with np.errstate(all="ignore"):
        assert checkers.constrSatisfaction(*_qargs(q)) == ok
        w = checkers.constr_worst(*_qargs(q))
    assert (w <= 1e-3) == ok
    if worst is not None:
        assert w == worst or abs(w - worst) < 1e-9
