"""The device-pointer entries on the caller's stream and their PyTorch ops, without a GPU: each entry is declared, exported and typed as
its host-pointer twin plus a stream; it refuses what its twin refuses, with the same code and message, before any device work; it
stops at OBCA_ERR_NO_DEVICE without a device; the mixed twins refuse two faults in their order; the ops register, trace under FakeTensorMode with the documented shapes and dtypes, and
refuse CPU, float32 and mixed-device tensors with ValueError."""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
from torch._subclasses.fake_tensor import FakeTensorMode

from obca_b200 import _lib, scenarios

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = {"obca_parking_solve_mixed_dev": "obca_parking_solve_mixed", "obca_dualmultws_batch_dev": "obca_dualmultws_batch",
           "obca_check_parking_dev": "obca_check_parking", "obca_check_parking_mixed_dev": "obca_check_parking_mixed",
           "obca_quadcopter_solve_batch_dev": "obca_quadcopter_solve_batch", "obca_quadcopter_solve_mixed_dev": "obca_quadcopter_solve_mixed",
           "obca_check_quadcopter_dev": "obca_check_quadcopter", "obca_check_quadcopter_mixed_dev": "obca_check_quadcopter_mixed"}
# pointer arguments an entry accepts as NULL (opts: the library's defaults; stream: the default stream)
OPTIONAL = {"opts", "stream", "lWS", "nWS", "sl", "e", "strict", "d", "slack", "worst", "solve_seconds"}
B = 4


def _params(name):
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "obca.h")).read(), flags=re.S)
    m = re.search(r"\bint " + name + r"\(([^;]*)\);", src)
    assert m, name
    return [a.replace("*", " ").split()[-1] for a in m.group(1).split(",")]


def _args(name, **over):
    """Valid arguments of `name` by parameter name: the scene as host arrays, every other array a small host buffer that the host-side
    checks never read (Nb / Tsb hold B valid values, which the host-pointer twins read), then the overrides."""
    park, quad = scenarios.reverse_parking_batch(1, 80, 0), scenarios.quadcopter_batch(1, 100)
    quadcopter = "quadcopter" in name
    keep = []

    def arr(a):
        keep.append(a)
        return a.ctypes.data_as(C.c_void_p)
    scene = dict(vOb=np.asarray(park["vOb"], np.int32), A=np.asfortranarray(park["A"], dtype=np.float64), b=np.ravel(park["b"]).astype(float),
                 ego=np.asarray(park["ego"], float), XYbounds=np.asarray(park["XYbounds"], float),
                 ob=np.ascontiguousarray(quad["obs"], dtype=float).ravel(), Nb=np.full(B, 80, np.int32), Tsb=np.full(B, 0.2))
    vals = dict(B=B, N=100 if quadcopter else 80, Nmax=100 if quadcopter else 80, nOb=park["nOb"], Ts=0.2, L=park["L"], R=quad["R"],
                timeWS=1.0, fixTime=0, signed_dist=1, sd=1, opts=None, stream=None)
    vals.update(over)
    out = []
    for p in _params(name):
        v = vals[p] if p in vals else scene[p] if p in scene else np.zeros(8)
        out.append(arr(v) if isinstance(v, np.ndarray) else v)
    return out, keep


def _call(name, **over):
    args, keep = _args(name, **over)
    rc = getattr(_lib.lib(), name)(*args)
    return rc, _lib.lib().obca_last_error().decode()


def _twin(name, **over):
    over.pop("stream", None)
    return _call(ENTRIES[name], **over)


def test_entries_declared_exported_and_typed_as_their_twins_plus_a_stream():
    lib = _lib.lib()
    for dev, twin in ENTRIES.items():
        assert dev in _lib.SYMBOLS and hasattr(lib, dev)
        f, g = getattr(lib, dev), getattr(lib, twin)
        assert f.restype is C.c_int and list(f.argtypes) == list(g.argtypes) + [C.c_void_p], dev
        assert _params(dev) == _params(twin) + ["stream"]
    assert "obca_parking_solve_batch_dev" in _lib.SYMBOLS and _params("obca_parking_solve_batch_dev")[-1] == "solve_seconds"


def _null_cases():
    for name in ENTRIES:
        for p in _params(name):
            if p not in OPTIONAL and p not in ("B", "N", "Nmax", "nOb", "Ts", "L", "R", "timeWS", "fixTime", "signed_dist", "sd"):
                yield pytest.param(name, p, id=f"{name}-{p}")


@pytest.mark.parametrize("name,arg", list(_null_cases()))
def test_null_argument_refused_as_the_twin_refuses_it(name, arg):
    rc, msg = _call(name, **{arg: None})
    assert rc == -1 and msg.startswith("null argument")
    assert msg == ("null argument: " + arg if arg in ("Nb", "Tsb") else "null argument")
    assert (rc, msg) == _twin(name, **{arg: None})


@pytest.mark.parametrize("name", list(ENTRIES))
def test_empty_batch_and_shape_errors_refused_as_the_twin_refuses_them(name):
    cases = [dict(B=0)]
    if "quadcopter" in name:
        cases += [dict(N=1)] if "mixed" not in name else []
    else:
        cases += [dict(nOb=0), dict(vOb=np.array([5, 4, 4], np.int32))]
    for over in cases:
        rc, msg = _call(name, **over)
        assert rc == -1, (over, msg)
        assert (rc, msg) == _twin(name, **over), over


@pytest.mark.parametrize("name,over,bound", [("obca_parking_solve_mixed_dev", dict(Nmax=320), "N = 320 > 319"),
                                             ("obca_quadcopter_solve_batch_dev", dict(N=512), "N = 512 > 511"),
                                             ("obca_quadcopter_solve_mixed_dev", dict(Nmax=512), "N = 512 > 511")])
def test_horizon_bound_unsupported(name, over, bound):
    rc, msg = _call(name, **over)
    assert rc == -4 and bound in msg
    assert (rc, msg) == _twin(name, **over)


@pytest.mark.parametrize("name", list(ENTRIES))
def test_no_device_without_a_gpu(name):
    if _lib.lib().obca_device_count() > 0:
        pytest.skip("a CUDA device is visible")
    assert _call(name) == (-2, "no CUDA device visible")
    assert _call(name, stream=C.c_void_p(1234)) == (-2, "no CUDA device visible")      # never touched before the device check


# A bad host-resident horizon together with a second fault: the solves check their required pointers before the horizons, the
# checkers the horizons first; every mixed entry checks the horizons' values before the shape, the horizon bound and Tsb.
BAD_NB = np.array([80, 80, 1, 80], np.int32)


def _bad_nb(Nmax, q=2, n=1):
    return f"Nb[{q}] = {n} outside [2, Nmax = {Nmax}]"


@pytest.mark.parametrize("name,over,msg", [
    ("obca_parking_solve_mixed", dict(x0=None), "null argument"),
    ("obca_parking_solve_mixed", dict(nOb=0), _bad_nb(80)),
    ("obca_parking_solve_mixed", dict(vOb=np.array([5, 4, 4], np.int32)), _bad_nb(80)),
    ("obca_parking_solve_mixed", dict(Nmax=320), _bad_nb(320)),
    ("obca_check_parking_mixed", dict(x0=None), _bad_nb(80)),
    ("obca_check_parking_mixed", dict(nOb=0), _bad_nb(80)),
    ("obca_check_parking_mixed", dict(vOb=np.array([5, 4, 4], np.int32)), _bad_nb(80)),
    ("obca_quadcopter_solve_mixed", dict(x0=None), "null argument"),
    ("obca_quadcopter_solve_mixed", dict(Nmax=1), _bad_nb(1, q=0, n=80)),
    ("obca_quadcopter_solve_mixed", dict(Nmax=512), _bad_nb(512)),
    ("obca_quadcopter_solve_mixed", dict(Tsb=None), _bad_nb(100)),
    ("obca_check_quadcopter_mixed", dict(x0=None), _bad_nb(100)),
    ("obca_check_quadcopter_mixed", dict(Nmax=1), _bad_nb(1, q=0, n=80)),
    ("obca_check_quadcopter_mixed", dict(Tsb=None), _bad_nb(100)),
])
def test_mixed_host_twin_refuses_a_bad_horizon_and_a_second_fault_in_order(name, over, msg):
    assert _call(name, Nb=BAD_NB, **over) == (-1, msg)


# ---- the PyTorch ops ---------------------------------------------------------------------------------------------------------------

OPS = ("parking_solve_mixed", "dualmultws", "check_parking", "check_parking_mixed", "quadcopter_solve_batch", "quadcopter_solve_mixed",
       "check_quadcopter", "check_quadcopter_mixed")


def test_import_registers_the_ops():
    import obca_b200.torch_ops  # noqa: F401
    for op in OPS:
        assert hasattr(torch.ops.obca, op), op
        assert torch.ops.obca.__getattr__(op).default._schema.name == "obca::" + op


def _park_inputs(Bp, Nmax, dev, dtype=torch.float64, lws=False):
    sc = scenarios.reverse_parking_batch(1, 80, 0)
    V, nOb = int(np.sum(sc["vOb"])), sc["nOb"]
    z = lambda *s: torch.zeros(s, dtype=dtype, device=dev)
    ins = dict(x0=z(Bp, 4), xF=z(4), Ns=torch.full((Bp,), Nmax, dtype=torch.int32, device=dev), Ts=sc["Ts"], L=sc["L"], ego_=sc["ego"],
               XYbounds=sc["XYbounds"], nOb=nOb, vOb=sc["vOb"], A=sc["A"], b=sc["b"], rx=z(Bp, Nmax + 1), ry=z(Bp, Nmax + 1),
               ryaw=z(Bp, Nmax + 1), fixTime=0, xWS=z(Bp, Nmax + 1, 4), uWS=z(Bp, Nmax, 2))
    if lws:
        ins.update(lWS=z(Bp, Nmax + 1, V), nWS=z(Bp, Nmax + 1, 4 * nOb))
    return ins, V, nOb


def test_fake_shapes_and_dtypes():
    from obca_b200 import torch_ops as T
    Bp, Nm = 5, 37
    f64, i32 = torch.float64, torch.int32
    with FakeTensorMode():
        ins, V, nOb = _park_inputs(Bp, Nm, "cuda", lws=True)
        r = T.parking_solve_mixed(**ins)
        want = dict(xp=((Bp, 4, Nm + 1), f64), up=((Bp, 2, Nm), f64), ts=((Bp, Nm + 1), f64), lp=((Bp, V, Nm + 1), f64),
                    np=((Bp, 4 * nOb, Nm + 1), f64), sl=((Bp, nOb, Nm + 1), f64), exitflag=((Bp,), i32), iters=((Bp,), i32),
                    kkt_err=((Bp,), f64), time=((), f64))
        for k, (shape, dt) in want.items():
            assert tuple(r[k].shape) == shape and r[k].dtype == dt and r[k].is_contiguous(), k
            assert r[k].device.type == ("cpu" if k == "time" else "cuda"), k
        sc = scenarios.reverse_parking_batch(1, 80, 0)
        lp, npp, d = T.dualmultws_batch(Nm, nOb, sc["vOb"], sc["A"], sc["b"], ins["rx"], ins["ry"], ins["ryaw"], sc["ego"], want_d=True)
        assert [tuple(t.shape) for t in (lp, npp, d)] == [(Bp, Nm + 1, V), (Bp, Nm + 1, 4 * nOb), (Bp, Nm + 1, nOb)]
        x, u = r["xp"], r["up"]
        for fn, extra in ((T.check_parking_batch, dict(N=Nm)), (T.check_parking_mixed, dict(Ns=ins["Ns"]))):
            feas, e, strict = fn(ins["x0"], ins["xF"], Ts=0.2, L=sc["L"], ego_=sc["ego"], XYbounds=sc["XYbounds"], nOb=nOb, vOb=sc["vOb"],
                                 A=sc["A"], b=sc["b"], x=x, u=u, l=r["lp"], n=r["np"], timeScale=r["ts"], fixTime=0, sd=1, sl=r["sl"], **extra)
            assert [(tuple(t.shape), t.dtype) for t in (feas, e, strict)] == [((Bp,), i32), ((Bp, 7), i32), ((Bp,), i32)]
        q = scenarios.quadcopter_scenario()
        z = lambda *s: torch.zeros(s, dtype=f64, device="cuda")
        Ns = torch.full((Bp,), Nm, dtype=i32, device="cuda")
        for rq in (T.quadcopter_solve_batch(z(Bp, 12), z(12), Nm, 0.2, q["R"], q["obs"], z(Bp, 12, Nm + 1)),
                   T.quadcopter_solve_mixed(z(Bp, 12), z(Bp, 12), Ns, z(Bp), q["R"], q["obs"], z(Bp, 12, Nm + 1))):
            want = dict(xp=(Bp, 12, Nm + 1), up=(Bp, 4, Nm), ts=(Bp, Nm + 1), lp=(Bp, 30, Nm + 1), slack=(Bp, 5, Nm + 1),
                        exitflag=(Bp,), iters=(Bp,), kkt_err=(Bp,), time=())
            for k, shape in want.items():
                assert tuple(rq[k].shape) == shape and rq[k].dtype == (i32 if k in ("exitflag", "iters") else f64), k
        for feas, worst in (T.check_quadcopter_batch(rq["xp"], rq["up"], rq["ts"], z(Bp, 12), z(12), 0.2, rq["lp"], q["obs"], q["R"]),
                            T.check_quadcopter_mixed(rq["xp"], rq["up"], rq["ts"], z(Bp, 12), z(12), Ns, 0.2, rq["lp"], q["obs"], q["R"])):
            assert (tuple(feas.shape), feas.dtype, tuple(worst.shape), worst.dtype) == ((Bp,), i32, (Bp,), f64)


def test_cpu_float32_and_mixed_device_tensors_refused():
    from obca_b200 import torch_ops as T
    ins, _, _ = _park_inputs(3, 20, "cpu")
    with pytest.raises(ValueError, match="CUDA tensors expected"):
        T.parking_solve_mixed(**ins)
    ins32, _, _ = _park_inputs(3, 20, "cpu", dtype=torch.float32)
    with pytest.raises(ValueError, match="rx: dtype torch.float32"):
        T.parking_solve_mixed(**dict(ins32, x0=ins["x0"], xF=ins["xF"]))
    with pytest.raises(ValueError, match="Ns: dtype torch.int64"):
        T.parking_solve_mixed(**dict(ins, Ns=ins["Ns"].long()))
    with FakeTensorMode():
        fins, _, _ = _park_inputs(3, 20, "cuda")
        with pytest.raises(ValueError, match="different devices: cpu, cuda:0"):
            T.parking_solve_mixed(**dict(fins, rx=torch.zeros(3, 21, dtype=torch.float64)))
        fins32, _, _ = _park_inputs(3, 20, "cuda", dtype=torch.float32)
        with pytest.raises(ValueError, match="dtype torch.float32"):
            T.parking_solve_mixed(**fins32)
        o = _lib.ObcaOpts()
        o.device = 1
        with pytest.raises(ValueError, match="opts.device = 1, the tensors are on cuda:0"):
            T.parking_solve_mixed(**fins, opts=o)
        with pytest.raises(ValueError, match="xWS: shape"):
            T.parking_solve_mixed(**dict(fins, xWS=torch.zeros(3, 21, 3, dtype=torch.float64, device="cuda")))
        lins, _, _ = _park_inputs(3, 20, "cuda", lws=True)
        with pytest.raises(ValueError, match="lWS and nWS go together"):
            T.parking_solve_mixed(**dict(lins, nWS=None))
        q = scenarios.quadcopter_scenario()
        z = lambda *s: torch.zeros(s, dtype=torch.float64, device="cuda")
        with pytest.raises(ValueError, match="different devices"):
            T.check_quadcopter_batch(z(3, 12, 21), z(3, 4, 20), z(3, 21), z(3, 12), torch.zeros(12, dtype=torch.float64), 0.2,
                                     z(3, 30, 21), q["obs"], q["R"])
        with pytest.raises(ValueError, match="Tsb: dtype torch.float32"):
            T.quadcopter_solve_mixed(z(3, 12), z(12), torch.full((3,), 20, dtype=torch.int32, device="cuda"),
                                     torch.zeros(3, device="cuda"), q["R"], q["obs"], z(3, 12, 21))
