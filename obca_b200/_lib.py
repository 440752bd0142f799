"""ctypes binding of libobca.so (include/obca.h).  The library is the product; there is no Python/CPU fallback:
if the shared object is missing or no CUDA device is visible, calls raise."""
from __future__ import annotations

import ctypes as C
import os
import re

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("OBCA_SO", os.path.join(HERE, "libobca.so"))   # OBCA_SO: development override
HEADER = os.path.join(os.path.dirname(HERE), "include", "obca.h")


class ObcaError(RuntimeError):
    pass


_ARG = {"int": C.c_int, "double": C.c_double, "long long": C.c_longlong}
_RET = {"int": C.c_int, "double": C.c_double, "void": None, "const char *": C.c_char_p}


def prototypes(header, error):
    """{name: (restype, argtypes)} of every function `ret name(args);` the C header declares, in header order.  Every pointer
    argument is c_void_p; int, double and long long arguments and int, double, void and const char* returns are typed as in C.
    Any other type raises `error` naming the function: the binding never guesses a type."""
    if not os.path.exists(header):
        raise error(f"{header} not found: it declares the library's C-ABI")
    with open(header) as f:
        src = re.sub(r"/\*.*?\*/|//[^\n]*", " ", f.read(), flags=re.S)
    src = re.sub(r"^[ \t]*#.*$", " ", src, flags=re.M)
    src = " ".join(src.replace("*", " * ").split())      # one space between words and around every '*'
    out = {}
    for ret, name, args in re.findall(r"([\w *]+?) ?\b(\w+) ?\(([^()]*)\) ?;", src):
        if ret.strip() not in _RET:
            raise error(f"{header}: {name}: no ctypes type for the return type '{ret.strip()}'")
        types = []
        for a in ([] if args.strip() == "void" else args.split(",")):
            a = a.strip()      # "const double * x0": the last word is the parameter's name
            t = C.c_void_p if "*" in a else _ARG.get(a.rsplit(" ", 1)[0])
            if t is None:
                raise error(f"{header}: {name}: no ctypes type for the argument '{a}'")
            types.append(t)
        out[name] = (_RET[ret.strip()], types)
    return out


def declare(lib, protos):
    """Type every function of `protos` (prototypes()) on the loaded library; a name it does not export raises."""
    for name, (res, args) in protos.items():
        f = getattr(lib, name)
        f.restype, f.argtypes = res, args
    return lib


_PROTOTYPES = prototypes(HEADER, ObcaError)
SYMBOLS = tuple(_PROTOTYPES)      # the functions include/obca.h declares


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


_lib = None


def lib():
    """Load libobca.so (built in-tree by __graft_entry__.build()).  Raises if it is not there."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise ObcaError(f"{SO_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                            "(the OBCA hot path has no CPU fallback)")
        _lib = declare(C.CDLL(SO_PATH), _PROTOTYPES)
    return _lib


def default_opts(device=0, retry=1) -> ObcaOpts:
    o = ObcaOpts()
    lib().obca_default_opts(C.byref(o))
    o.device = device
    o.retry = retry
    return o


def opts_arg(opts):
    """The opts argument of an entry: a reference to `opts`, or NULL for None, which selects the library's defaults."""
    return None if opts is None else C.byref(opts)


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
