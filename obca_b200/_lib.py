"""ctypes binding of libobca.so (include/obca.h).  The library is the product; there is no Python/CPU fallback:
if the shared object is missing or no CUDA device is visible, calls raise."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("OBCA_SO", os.path.join(HERE, "libobca.so"))   # OBCA_SO: development override

SYMBOLS = ["obca_version", "obca_device_count", "obca_last_error", "obca_default_opts", "obca_parking_solve_batch",
           "obca_parking_solve_batch_dev", "obca_dualmultws_batch", "obca_check_parking",
           "obca_parking_eval_batch_dev", "obca_parking_eval_sizes", "obca_last_profile", "obca_last_schedule",
           "obca_last_times", "obca_parking_solve_mixed", "obca_check_parking_mixed",
           "obca_quadcopter_solve_batch", "obca_check_quadcopter", "obca_quadcopter_solve_mixed",
           "obca_check_quadcopter_mixed", "obca_plan_parking_warmstart_batch", "obca_plan_quadcopter_warmstart_batch",
           "obca_plan_parking_warmstart_goals", "obca_plan_parking_heuristic_maps", "obca_parking_plan_solve_goals",
           "obca_quadcopter_plan_solve", "obca_parking_plan_solve_both", "obca_quadcopter_plan_solve_both"]


class ObcaOpts(C.Structure):
    _fields_ = [("tol", C.c_double), ("max_iter", C.c_int), ("mu_init", C.c_double), ("mu_min", C.c_double),
                ("kappa_eps", C.c_double), ("kappa_mu", C.c_double), ("theta_mu", C.c_double), ("tau_min", C.c_double),
                ("kappa1", C.c_double), ("kappa2", C.c_double), ("kappa_sigma", C.c_double), ("s_max", C.c_double),
                ("dual_inf_tol", C.c_double), ("constr_viol_tol", C.c_double), ("compl_inf_tol", C.c_double),
                ("dw_min", C.c_double), ("dw_first", C.c_double), ("dw_max", C.c_double), ("kw_minus", C.c_double),
                ("kw_plus", C.c_double), ("kw_plus_first", C.c_double),
                ("gamma_theta", C.c_double), ("gamma_phi", C.c_double), ("delta", C.c_double), ("s_theta", C.c_double),
                ("s_phi", C.c_double), ("eta_phi", C.c_double), ("gamma_alpha", C.c_double),
                ("max_backtrack", C.c_int), ("dc", C.c_double), ("max_kick", C.c_int), ("quad_dual_ws", C.c_int), ("device", C.c_int), ("retry", C.c_int), ("q4", C.c_int)]


class ParkingFlowOut(C.Structure):
    """obca_parking_flow_out: one formulation's output arrays (host pointers) of obca_parking_plan_solve_both."""
    _fields_ = [(k, C.c_void_p) for k in ("xp", "up", "ts", "lp", "np", "sl", "exitflag", "iters", "kkt_err", "feasible", "strict",
                                          "solve_seconds")]


class QuadcopterFlowOut(C.Structure):
    """obca_quadcopter_flow_out: one formulation's output arrays of obca_quadcopter_plan_solve_both."""
    _fields_ = [(k, C.c_void_p) for k in ("xp", "up", "ts", "lp", "slack", "exitflag", "iters", "kkt_err", "feasible", "worst",
                                          "solve_seconds")]


class ObcaError(RuntimeError):
    pass


_lib = None


def lib():
    """Load libobca.so (built in-tree by __graft_entry__.build()).  Raises if it is not there."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise ObcaError(f"{SO_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                            "(the OBCA hot path has no CPU fallback)")
        _lib = C.CDLL(SO_PATH)
        _lib.obca_last_error.restype = C.c_char_p
        for s in SYMBOLS:
            getattr(_lib, s)
    return _lib


def default_opts(device=0, retry=1) -> ObcaOpts:
    o = ObcaOpts()
    lib().obca_default_opts(C.byref(o))
    o.device = device
    o.retry = retry
    return o


def check(rc):
    if rc != 0:
        raise ObcaError(f"libobca error {rc}: {lib().obca_last_error().decode()}")


def ptr(a):
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    return a.ctypes.data_as(C.c_void_p)


def f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)
