"""PyTorch front end of libobca.so: the parking and quadcopter solves and checkers on CUDA tensors, ordered on the current stream.

Every function here has the name and argument order of its numpy twin in obca_b200.parking / obca_b200.quadcopter and returns what
the twin returns, bit for bit, as tensors on the inputs' device:

    parking_solve_mixed / parking_solve_batch      obca.parking_solve_mixed       (obca_parking_solve_mixed_dev)
    dualmultws_batch                               obca.dualmultws                (obca_dualmultws_batch_dev)
    check_parking_batch / check_parking_mixed      obca.check_parking[_mixed]     (obca_check_parking[_mixed]_dev)
    quadcopter_solve_batch / quadcopter_solve_mixed  obca.quadcopter_solve_batch / _mixed  (obca_quadcopter_solve_*_dev)
    check_quadcopter_batch / check_quadcopter_mixed  obca.check_quadcopter[_mixed]  (obca_check_quadcopter[_mixed]_dev)

Inputs are CUDA float64 tensors (int32 for Ns) on one device, in the numpy API's shapes; a batch with different horizons comes
padded to its longest horizon Nmax (rx (B, Nmax+1), xWS (B, Nmax+1, 4), ...), and so do its outputs (xp (B, 4, Nmax+1), ...),
which read 0 past each problem's own horizon.  The layout conversion to and from the C-ABI's column-major arrays runs on the device.
Scene data (vOb, A, b, ego, XYbounds, the quadcopter's obstacles) and opts are host values.  Each op waits for the work queued on
torch's current stream of the inputs' device before it reads an input, and returns once its outputs are written: no device-wide
synchronise is needed on either side.  `time` is the solve's device time, a 0-dim float64 CPU tensor.

Each op is a torch.library custom op in the namespace `obca` with a fake implementation, so that it traces under torch.compile.
opts reaches an op flattened, as the lists of its double and of its int fields (ObcaOpts order); opts None passes NULL, the
library's defaults on device 0."""
import ctypes as C
from typing import Optional

import numpy as np
import torch

from . import _lib
from .parking import _shared

Tensor = torch.Tensor
F64, I32 = torch.float64, torch.int32
_OPT_D = [k for k, t in _lib.ObcaOpts._fields_ if t is C.c_double]
_OPT_I = [k for k, t in _lib.ObcaOpts._fields_ if t is C.c_int]


def flat_opts(opts):
    """opts (an ObcaOpts or None) as the ops take it: (its double fields, its int fields), or two empty lists for None."""
    if opts is None:
        return [], []
    return [float(getattr(opts, k)) for k in _OPT_D], [int(getattr(opts, k)) for k in _OPT_I]


def _opts(opts_d, opts_i):
    if not opts_d:
        return None
    o = _lib.ObcaOpts()
    for k, v in zip(_OPT_D, opts_d):
        setattr(o, k, v)
    for k, v in zip(_OPT_I, opts_i):
        setattr(o, k, v)
    return o


def _device(opts_i, ints=(), **tensors):
    """The device of the tensors (None entries are optional arguments left out): float64 ones, int32 for the names in `ints`, all on
    one CUDA device, the one opts selects (device 0 without opts).  Anything else raises ValueError before the library is called."""
    given = {k: t for k, t in tensors.items() if t is not None}
    for k, t in given.items():
        want = I32 if k in ints else F64
        if t.dtype != want:
            raise ValueError(f"{k}: dtype {t.dtype}, expected {want}")
    devs = sorted({str(t.device) for t in given.values()})
    if len(devs) > 1:
        raise ValueError(f"tensors on different devices: {', '.join(devs)}")
    dev = next(iter(given.values())).device
    if dev.type != "cuda":
        raise ValueError(f"tensors on {dev}: CUDA tensors expected")
    od = opts_i[_OPT_I.index("device")] if opts_i else 0
    if dev.index != od:
        raise ValueError(f"opts.device = {od}, the tensors are on {dev}")
    return dev


def _shape(name, t, *shape):
    if t is not None and tuple(t.shape) != shape:
        raise ValueError(f"{name}: shape {tuple(t.shape)}, expected {shape}")


def _c(t):
    """A tensor in the numpy API's shape (B, r, c) as the C-ABI's column-major r x c arrays, B of them; (B,) and (B, n) as they are."""
    return None if t is None else (t.transpose(1, 2) if t.dim() == 3 else t).contiguous()


def _zeros_c(like, B, shape, dtype=F64):
    """Zeroed C-ABI output for per-problem arrays of the numpy API's shape `shape` (r, c): B column-major r x c arrays."""
    return torch.zeros((B,) + tuple(reversed(shape)), dtype=dtype, device=like.device)


def _p(t):
    """The device pointer of t; the caller holds t until the library has returned."""
    return None if t is None else C.c_void_p(t.data_ptr())


def _call(dev, name, *args):
    """Call the entry `name` on dev with torch's current stream of dev as its last argument."""
    with torch.cuda.device(dev):
        _lib.check(getattr(_lib.lib(), name)(*args, C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))


def _time():
    return torch.empty((), dtype=F64, device="cpu")


def _scene(vOb, A, b, ego, XYbounds):
    """The host arrays of the scene; the caller keeps them alive across the call."""
    return (np.asarray(vOb, np.int32), np.asarray(A, np.float64), np.asarray(b, np.float64), np.asarray(ego, np.float64),
            np.asarray(XYbounds, np.float64))


# ---- parking ---------------------------------------------------------------------------------------------------------------------

def _park_out_shapes(B, N, V, nOb):
    NS = N + 1
    return (4, NS), (2, N), (NS,), (V, NS), (4 * nOb, NS), (nOb, NS)


def _check_park_solve(Ns, x0, xF, rx, ry, ryaw, xWS, uWS, lWS, nWS, vOb, opts_i):
    dev = _device(opts_i, ("Ns",), Ns=Ns, x0=x0, xF=xF, rx=rx, ry=ry, ryaw=ryaw, xWS=xWS, uWS=uWS, lWS=lWS, nWS=nWS)
    B, NS = rx.shape
    N, V, nOb = NS - 1, sum(vOb), len(vOb)
    _shape("Ns", Ns, B); _shape("x0", x0, B, 4); _shape("xF", xF, B, 4); _shape("ry", ry, B, NS); _shape("ryaw", ryaw, B, NS)
    _shape("xWS", xWS, B, NS, 4); _shape("uWS", uWS, B, N, 2); _shape("lWS", lWS, B, NS, V); _shape("nWS", nWS, B, NS, 4 * nOb)
    if (lWS is None) != (nWS is None):
        raise ValueError("lWS and nWS go together")
    return dev, B, N, V, nOb


@torch.library.custom_op("obca::parking_solve_mixed", mutates_args=())
def _parking_solve_mixed(Ns: Tensor, x0: Tensor, xF: Tensor, Ts: float, L: float, ego: list[float], XYbounds: list[float],
                         vOb: list[int], A: list[float], b: list[float], rx: Tensor, ry: Tensor, ryaw: Tensor, fixTime: int,
                         xWS: Tensor, uWS: Tensor, lWS: Optional[Tensor], nWS: Optional[Tensor], signed_dist: int,
                         opts_d: list[float], opts_i: list[int]
                         ) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    dev, B, N, V, nOb = _check_park_solve(Ns, x0, xF, rx, ry, ryaw, xWS, uWS, lWS, nWS, vOb, opts_i)
    outs = [_zeros_c(x0, B, s) for s in _park_out_shapes(B, N, V, nOb)]
    ef, it, err = torch.zeros(B, dtype=I32, device=dev), torch.zeros(B, dtype=I32, device=dev), torch.zeros(B, dtype=F64, device=dev)
    sec = np.zeros(1)
    vo, A_, b_, e_, xy = _scene(vOb, A, b, ego, XYbounds)
    ins = [_c(t) for t in (Ns, x0, xF, rx, ry, ryaw, xWS, uWS, lWS, nWS)]
    _call(dev, "obca_parking_solve_mixed_dev", B, _p(ins[0]), N, nOb, _lib.ptr(vo), _lib.ptr(A_), _lib.ptr(b_), _p(ins[1]), _p(ins[2]), Ts, L,
          _lib.ptr(e_), _lib.ptr(xy), *[_p(t) for t in ins[3:]], fixTime, signed_dist, _lib.opts_arg(_opts(opts_d, opts_i)),
          *[_p(t) for t in outs], _p(ef), _p(it), _p(err), _lib.ptr(sec))
    return (*[_c(t) for t in outs], ef, it, err, torch.tensor(sec[0], dtype=F64))


@_parking_solve_mixed.register_fake
def _(Ns, x0, xF, Ts, L, ego, XYbounds, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS, lWS, nWS, signed_dist, opts_d, opts_i):
    _, B, N, V, nOb = _check_park_solve(Ns, x0, xF, rx, ry, ryaw, xWS, uWS, lWS, nWS, vOb, opts_i)
    return (*[x0.new_empty((B,) + s) for s in _park_out_shapes(B, N, V, nOb)], x0.new_empty(B, dtype=I32), x0.new_empty(B, dtype=I32),
            x0.new_empty(B), _time())


@torch.library.custom_op("obca::dualmultws", mutates_args=())
def _dualmultws(vOb: list[int], A: list[float], b: list[float], ego: list[float], rx: Tensor, ry: Tensor, ryaw: Tensor,
                opts_d: list[float], opts_i: list[int]) -> tuple[Tensor, Tensor, Tensor]:
    dev = _device(opts_i, rx=rx, ry=ry, ryaw=ryaw)
    B, NS = rx.shape
    _shape("ry", ry, B, NS); _shape("ryaw", ryaw, B, NS)
    V, nOb = sum(vOb), len(vOb)
    lp, npp, d = (_zeros_c(rx, B, (NS, k)) for k in (V, 4 * nOb, nOb))
    vo, A_, b_, e_, _ = _scene(vOb, A, b, ego, [])
    ins = [t.contiguous() for t in (rx, ry, ryaw)]
    _call(dev, "obca_dualmultws_batch_dev", B, NS - 1, nOb, _lib.ptr(vo), _lib.ptr(A_), _lib.ptr(b_), _lib.ptr(e_), *[_p(t) for t in ins],
          _lib.opts_arg(_opts(opts_d, opts_i)), _p(lp), _p(npp), _p(d))
    return _c(lp), _c(npp), _c(d)


@_dualmultws.register_fake
def _(vOb, A, b, ego, rx, ry, ryaw, opts_d, opts_i):
    _device(opts_i, rx=rx, ry=ry, ryaw=ryaw)
    B, NS = rx.shape
    _shape("ry", ry, B, NS); _shape("ryaw", ryaw, B, NS)
    return tuple(rx.new_empty((B, NS, k)) for k in (sum(vOb), 4 * len(vOb), len(vOb)))


def _check_park_check(Ns, x0, xF, x, u, l, n, timeScale, sl, vOb, opts_i):
    dev = _device(opts_i, ("Ns",), Ns=Ns, x0=x0, xF=xF, x=x, u=u, l=l, n=n, timeScale=timeScale, sl=sl)
    B, NS = timeScale.shape
    N, V, nOb = NS - 1, sum(vOb), len(vOb)
    _shape("Ns", Ns, B); _shape("x0", x0, B, 4); _shape("xF", xF, B, 4); _shape("x", x, B, 4, NS); _shape("u", u, B, 2, N)
    _shape("l", l, B, V, NS); _shape("n", n, B, 4 * nOb, NS); _shape("sl", sl, B, nOb, NS)
    return dev, B, N, nOb


def _park_check(Ns, x0, xF, Ts, L, ego, XYbounds, vOb, A, b, x, u, l, n, timeScale, sl, fixTime, sd, opts_d, opts_i):
    dev, B, N, nOb = _check_park_check(Ns, x0, xF, x, u, l, n, timeScale, sl, vOb, opts_i)
    feas, e, strict = torch.zeros(B, dtype=I32, device=dev), torch.zeros((B, 7), dtype=I32, device=dev), torch.zeros(B, dtype=I32, device=dev)
    vo, A_, b_, e_, xy = _scene(vOb, A, b, ego, XYbounds)
    Nc, x0c, xFc, *ins = [_c(t) for t in (Ns, x0, xF, x, u, l, n, timeScale, sl)]
    head = (B, N, nOb) if Ns is None else (B, _p(Nc), N, nOb)
    _call(dev, "obca_check_parking_dev" if Ns is None else "obca_check_parking_mixed_dev", *head, _lib.ptr(vo), _lib.ptr(A_), _lib.ptr(b_),
          _p(x0c), _p(xFc), Ts, L, _lib.ptr(e_), _lib.ptr(xy), *[_p(t) for t in ins], fixTime, sd, _lib.opts_arg(_opts(opts_d, opts_i)),
          _p(feas), _p(e), _p(strict))
    return feas, e, strict


def _park_check_fake(Ns, x0, xF, Ts, L, ego, XYbounds, vOb, A, b, x, u, l, n, timeScale, sl, fixTime, sd, opts_d, opts_i):
    _, B, _, _ = _check_park_check(Ns, x0, xF, x, u, l, n, timeScale, sl, vOb, opts_i)
    return x0.new_empty(B, dtype=I32), x0.new_empty((B, 7), dtype=I32), x0.new_empty(B, dtype=I32)


@torch.library.custom_op("obca::check_parking", mutates_args=())
def _check_parking(x0: Tensor, xF: Tensor, Ts: float, L: float, ego: list[float], XYbounds: list[float], vOb: list[int], A: list[float],
                   b: list[float], x: Tensor, u: Tensor, l: Tensor, n: Tensor, timeScale: Tensor, sl: Optional[Tensor], fixTime: int,
                   sd: int, opts_d: list[float], opts_i: list[int]) -> tuple[Tensor, Tensor, Tensor]:
    return _park_check(None, x0, xF, Ts, L, ego, XYbounds, vOb, A, b, x, u, l, n, timeScale, sl, fixTime, sd, opts_d, opts_i)


@_check_parking.register_fake
def _(x0, xF, Ts, L, ego, XYbounds, vOb, A, b, x, u, l, n, timeScale, sl, fixTime, sd, opts_d, opts_i):
    return _park_check_fake(None, x0, xF, Ts, L, ego, XYbounds, vOb, A, b, x, u, l, n, timeScale, sl, fixTime, sd, opts_d, opts_i)


@torch.library.custom_op("obca::check_parking_mixed", mutates_args=())
def _check_parking_mixed(Ns: Tensor, x0: Tensor, xF: Tensor, Ts: float, L: float, ego: list[float], XYbounds: list[float],
                         vOb: list[int], A: list[float], b: list[float], x: Tensor, u: Tensor, l: Tensor, n: Tensor, timeScale: Tensor,
                         sl: Optional[Tensor], fixTime: int, sd: int, opts_d: list[float], opts_i: list[int]
                         ) -> tuple[Tensor, Tensor, Tensor]:
    return _park_check(Ns, x0, xF, Ts, L, ego, XYbounds, vOb, A, b, x, u, l, n, timeScale, sl, fixTime, sd, opts_d, opts_i)


@_check_parking_mixed.register_fake
def _(Ns, x0, xF, Ts, L, ego, XYbounds, vOb, A, b, x, u, l, n, timeScale, sl, fixTime, sd, opts_d, opts_i):
    return _park_check_fake(Ns, x0, xF, Ts, L, ego, XYbounds, vOb, A, b, x, u, l, n, timeScale, sl, fixTime, sd, opts_d, opts_i)


# ---- quadcopter ------------------------------------------------------------------------------------------------------------------

def _quad_out_shapes(N):
    NS = N + 1
    return (12, NS), (4, N), (NS,), (30, NS), (5, NS)


def _check_quad_solve(Ns, Tsb, x0, xF, xWS, opts_i):
    dev = _device(opts_i, ("Ns",), Ns=Ns, Tsb=Tsb, x0=x0, xF=xF, xWS=xWS)
    B, _, NS = xWS.shape
    _shape("Ns", Ns, B); _shape("Tsb", Tsb, B); _shape("x0", x0, B, 12); _shape("xF", xF, B, 12); _shape("xWS", xWS, B, 12, NS)
    return dev, B, NS - 1


def _quad_solve(Ns, Tsb, x0, xF, Ts, R, ob, xWS, timeWS, signed_dist, opts_d, opts_i):
    dev, B, N = _check_quad_solve(Ns, Tsb, x0, xF, xWS, opts_i)
    outs = [_zeros_c(x0, B, s) for s in _quad_out_shapes(N)]
    ef, it, err = torch.zeros(B, dtype=I32, device=dev), torch.zeros(B, dtype=I32, device=dev), torch.zeros(B, dtype=F64, device=dev)
    sec = np.zeros(1)
    obh = np.asarray(ob, np.float64)
    Nc, Tc, x0c, xFc, xWc = (_c(t) for t in (Ns, Tsb, x0, xF, xWS))
    if Ns is None:
        head = (B, N, _p(x0c), _p(xFc), Ts, R)
    else:
        head = (B, _p(Nc), N, _p(x0c), _p(xFc), _p(Tc), R)
    _call(dev, "obca_quadcopter_solve_batch_dev" if Ns is None else "obca_quadcopter_solve_mixed_dev", *head, _lib.ptr(obh), _p(xWc),
          timeWS, signed_dist, _lib.opts_arg(_opts(opts_d, opts_i)), *[_p(t) for t in outs], _p(ef), _p(it), _p(err), _lib.ptr(sec))
    return (*[_c(t) for t in outs], ef, it, err, torch.tensor(sec[0], dtype=F64))


def _quad_solve_fake(Ns, Tsb, x0, xF, xWS, opts_i):
    _, B, N = _check_quad_solve(Ns, Tsb, x0, xF, xWS, opts_i)
    return (*[x0.new_empty((B,) + s) for s in _quad_out_shapes(N)], x0.new_empty(B, dtype=I32), x0.new_empty(B, dtype=I32),
            x0.new_empty(B), _time())


@torch.library.custom_op("obca::quadcopter_solve_batch", mutates_args=())
def _quadcopter_solve_batch(x0: Tensor, xF: Tensor, Ts: float, R: float, ob: list[float], xWS: Tensor, timeWS: float, signed_dist: int,
                            opts_d: list[float], opts_i: list[int]
                            ) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    return _quad_solve(None, None, x0, xF, Ts, R, ob, xWS, timeWS, signed_dist, opts_d, opts_i)


@_quadcopter_solve_batch.register_fake
def _(x0, xF, Ts, R, ob, xWS, timeWS, signed_dist, opts_d, opts_i):
    return _quad_solve_fake(None, None, x0, xF, xWS, opts_i)


@torch.library.custom_op("obca::quadcopter_solve_mixed", mutates_args=())
def _quadcopter_solve_mixed(Ns: Tensor, x0: Tensor, xF: Tensor, Tsb: Tensor, R: float, ob: list[float], xWS: Tensor, timeWS: float,
                            signed_dist: int, opts_d: list[float], opts_i: list[int]
                            ) -> tuple[Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor]:
    return _quad_solve(Ns, Tsb, x0, xF, float("nan"), R, ob, xWS, timeWS, signed_dist, opts_d, opts_i)


@_quadcopter_solve_mixed.register_fake
def _(Ns, x0, xF, Tsb, R, ob, xWS, timeWS, signed_dist, opts_d, opts_i):
    return _quad_solve_fake(Ns, Tsb, x0, xF, xWS, opts_i)


def _check_quad_check(Ns, Tsb, x, u, timeScale, x0, xF, lam, opts_i):
    dev = _device(opts_i, ("Ns",), Ns=Ns, Tsb=Tsb, x=x, u=u, timeScale=timeScale, x0=x0, xF=xF, lam=lam)
    B, NS = timeScale.shape
    _shape("Ns", Ns, B); _shape("Tsb", Tsb, B); _shape("x", x, B, 12, NS); _shape("u", u, B, 4, NS - 1); _shape("x0", x0, B, 12)
    _shape("xF", xF, B, 12); _shape("lam", lam, B, 30, NS)
    return dev, B, NS - 1


def _quad_check(Ns, Tsb, x, u, timeScale, x0, xF, Ts, lam, ob, R, opts_d, opts_i):
    dev, B, N = _check_quad_check(Ns, Tsb, x, u, timeScale, x0, xF, lam, opts_i)
    feas, worst = torch.zeros(B, dtype=I32, device=dev), torch.zeros(B, dtype=F64, device=dev)
    Nc, Tc, xx, uu, tt, x0c, xFc, ll = (_c(t) for t in (Ns, Tsb, x, u, timeScale, x0, xF, lam))
    obh = np.asarray(ob, np.float64)
    if Ns is None:
        args = (B, N, _p(xx), _p(uu), _p(tt), _p(x0c), _p(xFc), Ts, _p(ll))
    else:
        args = (B, _p(Nc), N, _p(xx), _p(uu), _p(tt), _p(x0c), _p(xFc), _p(Tc), _p(ll))
    _call(dev, "obca_check_quadcopter_dev" if Ns is None else "obca_check_quadcopter_mixed_dev", *args, _lib.ptr(obh), R,
          _lib.opts_arg(_opts(opts_d, opts_i)), _p(feas), _p(worst))
    return feas, worst


def _quad_check_fake(Ns, Tsb, x, u, timeScale, x0, xF, lam, opts_i):
    _, B, _ = _check_quad_check(Ns, Tsb, x, u, timeScale, x0, xF, lam, opts_i)
    return x0.new_empty(B, dtype=I32), x0.new_empty(B)


@torch.library.custom_op("obca::check_quadcopter", mutates_args=())
def _check_quadcopter(x: Tensor, u: Tensor, timeScale: Tensor, x0: Tensor, xF: Tensor, Ts: float, lam: Tensor, ob: list[float], R: float,
                      opts_d: list[float], opts_i: list[int]) -> tuple[Tensor, Tensor]:
    return _quad_check(None, None, x, u, timeScale, x0, xF, Ts, lam, ob, R, opts_d, opts_i)


@_check_quadcopter.register_fake
def _(x, u, timeScale, x0, xF, Ts, lam, ob, R, opts_d, opts_i):
    return _quad_check_fake(None, None, x, u, timeScale, x0, xF, lam, opts_i)


@torch.library.custom_op("obca::check_quadcopter_mixed", mutates_args=())
def _check_quadcopter_mixed(x: Tensor, u: Tensor, timeScale: Tensor, x0: Tensor, xF: Tensor, Ns: Tensor, Tsb: Tensor, lam: Tensor,
                            ob: list[float], R: float, opts_d: list[float], opts_i: list[int]) -> tuple[Tensor, Tensor]:
    return _quad_check(Ns, Tsb, x, u, timeScale, x0, xF, float("nan"), lam, ob, R, opts_d, opts_i)


@_check_quadcopter_mixed.register_fake
def _(x, u, timeScale, x0, xF, Ns, Tsb, lam, ob, R, opts_d, opts_i):
    return _quad_check_fake(Ns, Tsb, x, u, timeScale, x0, xF, lam, opts_i)


# ---- public functions: the numpy twins' names and argument order --------------------------------------------------------------------

def _scene_lists(nOb, vOb, A, b, ego_, XYbounds=None):
    vOb, _, A, b = _shared(nOb, vOb, A, b)
    xy = [] if XYbounds is None else np.asarray(XYbounds, float).ravel().tolist()
    return vOb.tolist(), A.ravel(order="F").tolist(), b.tolist(), np.asarray(ego_, float).ravel().tolist(), xy


def _rows(t, B, n):
    """x0 / xF as (B, n): a tensor of shape (n,) or (1, n) is every problem's."""
    return t.reshape(-1, n).expand(B, n)


def parking_solve_mixed(x0, xF, Ns, Ts, L, ego_, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS,
                        signed_dist=1, lWS=None, nWS=None, opts=None):
    """parking.parking_solve_mixed on tensors padded to Nmax: x0 (B,4), xF (4,) or (B,4), Ns (B,) int32, rx / ry / ryaw (B,Nmax+1),
    xWS (B,Nmax+1,4), uWS (B,>=Nmax,2), optional lWS (B,Nmax+1,V), nWS (B,Nmax+1,4nOb).  Returns dict: xp (B,4,Nmax+1), up (B,2,Nmax),
    ts (B,Nmax+1), lp (B,V,Nmax+1), np (B,4nOb,Nmax+1), sl (B,nOb,Nmax+1), exitflag, iters, kkt_err, N (= Ns), time."""
    B, Nmax = rx.shape[0], rx.shape[1] - 1
    vo, Al, bl, eg, xy = _scene_lists(nOb, vOb, A, b, ego_, XYbounds)
    r = torch.ops.obca.parking_solve_mixed(Ns, x0, _rows(xF, B, 4), float(Ts), float(L), eg, xy, vo, Al, bl, rx, ry, ryaw, int(fixTime),
                                           xWS, uWS[:, :Nmax], lWS, nWS, int(signed_dist), *flat_opts(opts))
    return dict(zip(("xp", "up", "ts", "lp", "np", "sl", "exitflag", "iters", "kkt_err"), r[:9]), N=Ns, time=r[9])


def parking_solve_batch(x0, xF, N, Ts, L, ego_, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS,
                        signed_dist=1, lWS=None, nWS=None, opts=None):
    """parking.parking_solve_batch on tensors: every problem has the horizon N (the mixed op with Ns = N, bit for bit the uniform solve)."""
    Ns = torch.full((rx.shape[0],), int(N), dtype=I32, device=rx.device)
    return parking_solve_mixed(x0, xF, Ns, Ts, L, ego_, XYbounds, nOb, vOb, A, b, rx, ry, ryaw, fixTime, xWS, uWS, signed_dist, lWS, nWS, opts)


def dualmultws_batch(N, nOb, vOb, A, b, rx, ry, ryaw, ego_, opts=None, want_d=False):
    """parking.dualmultws_batch on tensors: rx, ry, ryaw (B,N+1) -> lp (B,N+1,V), np (B,N+1,4nOb)[, d (B,N+1,nOb)]."""
    _shape("rx", rx, rx.shape[0], N + 1)
    vo, Al, bl, eg, _ = _scene_lists(nOb, vOb, A, b, ego_)
    lp, npp, d = torch.ops.obca.dualmultws(vo, Al, bl, eg, rx, ry, ryaw, *flat_opts(opts))
    return (lp, npp, d) if want_d else (lp, npp)


def check_parking_batch(x0, xF, N, Ts, L, ego_, XYbounds, nOb, vOb, A, b, x, u, l, n, timeScale, fixTime, sd, sl=None, opts=None):
    """parking.check_parking_batch on tensors: x (B,4,N+1), u (B,2,N), l (B,V,N+1), n (B,4nOb,N+1), timeScale (B,N+1), sl (B,nOb,N+1).
    Returns feasible (B,), e (B,7), strict (B,), int32."""
    B = x.shape[0]
    _shape("timeScale", timeScale, B, N + 1)
    vo, Al, bl, eg, xy = _scene_lists(nOb, vOb, A, b, ego_, XYbounds)
    return torch.ops.obca.check_parking(_rows(x0, B, 4), _rows(xF, B, 4), float(Ts), float(L), eg, xy, vo, Al, bl, x, u, l, n, timeScale,
                                        sl, int(fixTime), int(sd), *flat_opts(opts))


def check_parking_mixed(x0, xF, Ns, Ts, L, ego_, XYbounds, nOb, vOb, A, b, x, u, l, n, timeScale, fixTime, sd, sl=None, opts=None):
    """parking.check_parking_mixed on tensors padded to Nmax, in the shapes of check_parking_batch with N = Nmax; Ns (B,) int32."""
    B = x.shape[0]
    vo, Al, bl, eg, xy = _scene_lists(nOb, vOb, A, b, ego_, XYbounds)
    return torch.ops.obca.check_parking_mixed(Ns, _rows(x0, B, 4), _rows(xF, B, 4), float(Ts), float(L), eg, xy, vo, Al, bl, x, u, l, n,
                                              timeScale, sl, int(fixTime), int(sd), *flat_opts(opts))


def _ob(obs):
    return np.asarray(obs, float).reshape(5, 6).ravel().tolist()      # rows = obstacles == the C-ABI's 6 x 5 column-major block


_QKEYS = ("xp", "up", "ts", "lp", "slack", "exitflag", "iters", "kkt_err")


def quadcopter_solve_batch(x0, xF, N, Ts, R, obs, xWS, timeWS=1.0, signed_dist=1, opts=None):
    """quadcopter.quadcopter_solve_batch on tensors: x0 (B,12), xF (12,) or (B,12), xWS (B,12,N+1).  Returns dict: xp (B,12,N+1),
    up (B,4,N), ts (B,N+1), lp (B,30,N+1), slack (B,5,N+1), exitflag, iters, kkt_err, time."""
    B = x0.shape[0]
    _shape("xWS", xWS, B, 12, N + 1)
    r = torch.ops.obca.quadcopter_solve_batch(x0, _rows(xF, B, 12), float(Ts), float(R), _ob(obs), xWS, float(timeWS), int(signed_dist),
                                              *flat_opts(opts))
    return dict(zip(_QKEYS, r[:8]), time=r[8])


def quadcopter_solve_mixed(x0, xF, Ns, Ts, R, obs, xWS, timeWS=1.0, signed_dist=1, opts=None):
    """quadcopter.quadcopter_solve_mixed on tensors padded to Nmax: x0 (B,12), xF (12,) or (B,12), Ns (B,) int32, Ts a float or (B,),
    xWS (B,12,Nmax+1).  Returns the dict of quadcopter_solve_batch at N = Nmax, with N (= Ns) and Ts (B,)."""
    B = x0.shape[0]
    Tsb = Ts if isinstance(Ts, Tensor) else torch.full((B,), float(Ts), dtype=F64, device=x0.device)
    r = torch.ops.obca.quadcopter_solve_mixed(Ns, x0, _rows(xF, B, 12), Tsb, float(R), _ob(obs), xWS, float(timeWS), int(signed_dist),
                                              *flat_opts(opts))
    return dict(zip(_QKEYS, r[:8]), N=Ns, Ts=Tsb, time=r[8])


def check_quadcopter_batch(x, u, timeScale, x0, xF, Ts, lam, obs, R, opts=None):
    """quadcopter.check_quadcopter_batch on tensors: x (B,12,N+1), u (B,4,N), timeScale (B,N+1), lam (B,30,N+1).  Returns feasible
    (B,) int32 and worst (B,)."""
    B = x.shape[0]
    return torch.ops.obca.check_quadcopter(x, u, timeScale, _rows(x0, B, 12), _rows(xF, B, 12), float(Ts), lam, _ob(obs), float(R),
                                           *flat_opts(opts))


def check_quadcopter_mixed(x, u, timeScale, x0, xF, Ns, Ts, lam, obs, R, opts=None):
    """quadcopter.check_quadcopter_mixed on tensors padded to Nmax, in the shapes of check_quadcopter_batch; Ns (B,) int32, Ts a float
    or (B,)."""
    B = x.shape[0]
    Tsb = Ts if isinstance(Ts, Tensor) else torch.full((B,), float(Ts), dtype=F64, device=x.device)
    return torch.ops.obca.check_quadcopter_mixed(x, u, timeScale, _rows(x0, B, 12), _rows(xF, B, 12), Ns, Tsb, lam, _ob(obs), float(R),
                                                 *flat_opts(opts))
