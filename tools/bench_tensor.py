"""Host-pointer entries against the PyTorch ops on CUDA tensors, alternating in one process (profiles/tensor_h100.md).

Workloads: parking mixed (reverse_parking_mixed_batch, SignedDist, N uniform over 40..80) and quadcopter mixed (quadcopter_mixed_batch,
SignedDist, N over 90..127).  Per repetition, in turn:
  host    obca_parking_solve_mixed / obca_quadcopter_solve_mixed on numpy arrays already in the C-ABI's layout: the library stages
          them to the device and back (the path a PyTorch caller takes today, less its own device <-> host copies);
  tensor  torch_ops.parking_solve_mixed / quadcopter_solve_mixed on CUDA tensors in the numpy API's shapes: on-device layout
          conversion, output allocation, the _dev entry on the current stream.
Wall time of each call (ending in a device synchronise) and the solve's device time it reports; exitflag, iters and kkt_err of the two
paths are compared in every repetition.  Prints one JSON line per workload, with the card and its power limit.
    python tools/bench_tensor.py [--reps 5] [--park-B 4096] [--quad-B 2048]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from obca_b200 import _lib, parking as pk, scenarios, torch_ops as T  # noqa: E402
from obca_b200.parking import _pad_stages  # noqa: E402

DEV = torch.device("cuda", 0)


def _t(a, dtype=torch.float64):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=DEV)


def _p(a):
    return _lib.ptr(a)


def park_case(B, seed):
    sc = scenarios.reverse_parking_mixed_batch(B, (40, 80), seed=seed)
    Ns, Nmax = sc["Ns"], int(sc["Ns"].max())
    NS = Nmax + 1
    pad = lambda arrs, cols, ext=1: _pad_stages([np.asarray(a, float).reshape(-1, cols)[:n + ext] for a, n in zip(arrs, Ns)], Nmax)
    rx, ry, ryaw = (pad(sc[k], 1)[..., 0] for k in ("rx", "ry", "ryaw"))
    xWS, uWS = pad(sc["xWS"], 4), pad(sc["uWS"], 2, 0)[:, :Nmax]
    vOb, V, A, b = pk._shared(sc["nOb"], sc["vOb"], sc["A"], sc["b"])
    nOb = sc["nOb"]
    ego, xy = np.asarray(sc["ego"], float).ravel(), np.asarray(sc["XYbounds"], float).ravel()
    x0, xF = np.ascontiguousarray(sc["x0"]), np.ascontiguousarray(np.broadcast_to(np.asarray(sc["xF"], float), (B, 4)))
    hin = [np.ascontiguousarray(a) for a in (x0, xF, rx, ry, ryaw, xWS.transpose(0, 2, 1), uWS.transpose(0, 2, 1))]
    Nsh = np.ascontiguousarray(Ns, np.int32)

    def host():
        o = [np.zeros((B, NS, 4)), np.zeros((B, Nmax, 2)), np.zeros((B, NS)), np.zeros((B, NS, V)), np.zeros((B, NS, 4 * nOb)),
             np.zeros((B, NS, nOb))]
        ef, it, err, sec = np.zeros(B, np.int32), np.zeros(B, np.int32), np.zeros(B), np.zeros(1)
        _lib.check(_lib.lib().obca_parking_solve_mixed(
            B, _p(Nsh), Nmax, nOb, _p(vOb), _p(A), _p(b), _p(hin[0]), _p(hin[1]), float(sc["Ts"]), float(sc["L"]), _p(ego), _p(xy),
            *[_p(a) for a in hin[2:]], None, None, 0, 1, None, *[_p(a) for a in o], _p(ef), _p(it), _p(err), _p(sec)))
        return ef, it, err, float(sec[0])

    tin = dict(x0=_t(x0), xF=_t(xF), Ns=_t(Ns, torch.int32), rx=_t(rx), ry=_t(ry), ryaw=_t(ryaw), xWS=_t(xWS), uWS=_t(uWS))

    def tensor():
        r = T.parking_solve_mixed(tin["x0"], tin["xF"], tin["Ns"], sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], nOb, sc["vOb"], sc["A"],
                                  sc["b"], tin["rx"], tin["ry"], tin["ryaw"], 0, tin["xWS"], tin["uWS"])
        torch.cuda.synchronize(DEV)
        return r["exitflag"].cpu().numpy(), r["iters"].cpu().numpy(), r["kkt_err"].cpu().numpy(), float(r["time"])
    return host, tensor


def quad_case(B, seed):
    sc = scenarios.quadcopter_mixed_batch(B, (90, 127), seed=seed)
    Ns, Nmax = sc["Ns"], int(sc["Ns"].max())
    NS = Nmax + 1
    xw = _pad_stages([np.asarray(w, float).T for w in sc["xWS"]], Nmax)          # (B, Nmax+1, 12): the C-ABI's 12 x (Nmax+1)
    ob = np.ascontiguousarray(sc["obs"], dtype=float).ravel()
    x0, xF, Tsb, Nsh = (np.ascontiguousarray(a) for a in (sc["x0"], sc["xF"], sc["Ts"], np.asarray(Ns, np.int32)))

    def host():
        o = [np.zeros((B, NS, 12)), np.zeros((B, Nmax, 4)), np.zeros((B, NS)), np.zeros((B, NS, 30)), np.zeros((B, NS, 5))]
        ef, it, err, sec = np.zeros(B, np.int32), np.zeros(B, np.int32), np.zeros(B), np.zeros(1)
        _lib.check(_lib.lib().obca_quadcopter_solve_mixed(B, _p(Nsh), Nmax, _p(x0), _p(xF), _p(Tsb), float(sc["R"]), _p(ob), _p(xw), 1.0, 1,
                                                          None, *[_p(a) for a in o], _p(ef), _p(it), _p(err), _p(sec)))
        return ef, it, err, float(sec[0])

    tin = dict(x0=_t(x0), xF=_t(xF), Ns=_t(Ns, torch.int32), Ts=_t(Tsb), xWS=_t(xw.transpose(0, 2, 1)))

    def tensor():
        r = T.quadcopter_solve_mixed(tin["x0"], tin["xF"], tin["Ns"], tin["Ts"], sc["R"], sc["obs"], tin["xWS"])
        torch.cuda.synchronize(DEV)
        return r["exitflag"].cpu().numpy(), r["iters"].cpu().numpy(), r["kkt_err"].cpu().numpy(), float(r["time"])
    return host, tensor


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def measure(name, B, host, tensor, reps):
    host(); tensor()      # warm-up: module load, workspace, staging buffer
    wall = {"host": [], "tensor": []}
    dev = {"host": [], "tensor": []}
    same = True
    for _ in range(reps):
        out = {}
        for k, f in (("host", host), ("tensor", tensor)):
            torch.cuda.synchronize(DEV)
            t0 = time.perf_counter()
            out[k] = f()
            wall[k].append(time.perf_counter() - t0)
            dev[k].append(out[k][3])
        same &= all(np.array_equal(a, b) for a, b in zip(out["host"][:3], out["tensor"][:3]))
    med = lambda v: float(np.median(v))
    return dict(workload=name, B=B, reps=reps, card=card(), identical=bool(same),
                host_wall_ms=[round(1e3 * v, 2) for v in wall["host"]], tensor_wall_ms=[round(1e3 * v, 2) for v in wall["tensor"]],
                host_solve_ms=round(1e3 * med(dev["host"]), 2), tensor_solve_ms=round(1e3 * med(dev["tensor"]), 2),
                median_host_wall_ms=round(1e3 * med(wall["host"]), 2), median_tensor_wall_ms=round(1e3 * med(wall["tensor"]), 2),
                host_per_s=round(B / med(wall["host"]), 1), tensor_per_s=round(B / med(wall["tensor"]), 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--park-B", type=int, default=4096)
    ap.add_argument("--quad-B", type=int, default=2048)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tensor.py measures on a CUDA device; none is visible")
    print(json.dumps(measure("parking_mixed_sd_N40-80", a.park_B, *park_case(a.park_B, 0), a.reps)), flush=True)
    print(json.dumps(measure("quadcopter_mixed_sd_N90-127", a.quad_B, *quad_case(a.quad_B, 2), a.reps)), flush=True)


if __name__ == "__main__":
    main()
