"""The rare branches of the interior-point driver (IpmDriver, obca_solver.cuh), CPU side: the kernel sources run through the
development emulation with option settings that drive the iteration limit, the barrier kick that stands in for Ipopt's
restoration phase, the line-search failure once no kick is left, and the inertia-correction failure once delta_w passes its
cap.  Each setting is checked to reach its branch, for the parking model (BASELINE config 2 problems) and for the quadcopter
model (signed distance, N = 40)."""
import pytest

import emul
from obca_b200 import scenarios


@pytest.fixture(scope="module", params=["parking", "quadcopter"])
def solve(request):
    """solve(**opts) -> the emulation's results for a fixed batch of the model, with the given options changed."""
    if request.param == "parking":
        sc = scenarios.reverse_parking_batch(8, 80, 0)
        lp, npp, _, _ = emul.dualmultws_batch(sc)
        base = {}
        run = lambda o: emul.solve_batch(sc, 0, "sd", o, lp, npp)
    else:
        sc = scenarios.quadcopter_batch(4, N=40, seed=2)
        base = {"max_iter": 300}
        run = lambda o: emul.quad_solve_batch(sc, "sd", o)

    def f(**kw):
        o = emul.default_opts()
        for k, v in {**base, **kw}.items():
            setattr(o, k, v)
        return run(o)
    return f


def test_iteration_limit_gives_status_0(solve):
    r = solve(max_iter=4)
    assert (r["status"] == 0).all() and (r["iters"] == 4).all()


def test_line_search_failure_without_kicks_gives_status_minus_1(solve):
    """One trial step per line search and no barrier kick: a rejected trial step ends the attempt."""
    r = solve(max_backtrack=1, max_kick=0)
    assert (r["status"] == -1).any() and set(r["status"].tolist()) <= {1, -1}


def test_barrier_kick_recovers_from_a_failed_line_search(solve):
    """Same single-trial line search with the default kicks: a problem whose line search fails without a kick (previous test)
    converges after raising the barrier parameter, and the kick costs it iterations."""
    none = solve(max_backtrack=1, max_kick=0)
    kick = solve(max_backtrack=1)
    rescued = (none["status"] == -1) & (kick["status"] == 1)
    assert rescued.any()
    assert (kick["iters"][rescued] > none["iters"][rescued]).all()


def test_delta_w_cap_gives_status_minus_2(solve):
    """delta_w capped below its first trial value: the first inertia correction ends the attempt, so every problem whose default
    solve corrects the inertia at least once (more factorisations than iterations + 1) ends with status -2, before the
    iteration count of its default solve."""
    ref = solve()
    corrected = ref["nfact"] > ref["iters"] + 1
    assert corrected.any()
    r = solve(dw_max=0.1 * emul.default_opts().dw_first)
    assert (r["status"][corrected] == -2).all()
    assert (r["iters"][corrected] < ref["iters"][corrected]).all()
