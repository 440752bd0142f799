"""Quadcopter (config 4) timing + per-phase cycle breakdown (development tool).  usage: gpu_quad.py [B] [N]   (N default 100)"""
import ctypes as C, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import obca_b200
from obca_b200 import quadcopter, scenarios
B = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
N = int(sys.argv[2]) if len(sys.argv) > 2 else 100
sc = scenarios.quadcopter_batch(B, N, seed=2)
o = obca_b200.default_opts(); o.max_iter = 3000
for sd in (1, 0):
    for rep in range(2):
        r = quadcopter.quadcopter_solve_batch(sc["x0"], sc["xF"], sc["N"], sc["Ts"], sc["R"], sc["obs"], sc["xWS"], 1.0, sd, o)
    it = r["iters"]
    print(f"sd={sd} B={B} N={N}: device {r['time']*1e3:.1f} ms -> {B/r['time']:.0f} traj/s; ok {int((r['exitflag']>=1).sum())}; iters mean {it.mean():.1f} max {it.max()}")
    prof = (C.c_ulonglong * 8)()
    obca_b200.lib().obca_last_profile(0, prof)
    p = np.array(list(prof), float); names = ["eval_K1", "kkt_K3", "recover", "merit", "update", "serial"]
    tot = p[:6].sum() or 1.0
    print("  phase share:", {n: round(p[i] / tot, 3) for i, n in enumerate(names)}, "cycles/iter", int(tot / max(it.sum(), 1)),
          "k1 evals/iter", round(p[7] / max(it.sum(), 1), 2), "merit/iter", round(p[6] / max(it.sum(), 1), 2))
    print("  cycles/iter per phase:", {n: int(p[i] / max(it.sum(), 1)) for i, n in enumerate(names)})
    L = obca_b200.lib()
    if hasattr(L, "obca_debug_qprof"):
        q = (C.c_ulonglong * 8)(); L.obca_debug_qprof(q); q = np.array(list(q), float)
        n = max(q[7], 1.0) * 100.0
        print("  sweep cycles/stage: issue+rp", int(q[0] / n), "wait", int(q[1] / n), "T", int(q[2] / n), "H", int(q[3] / n), "K", int(q[4] / n),
              "P(loop tail)", int(q[5] / n), "forward", int(q[6] / n), "sweeps", int(q[7]))
