#!/usr/bin/env python
"""tools/bench_mixed.py -- a batch of problems with different horizons: one obca_parking_solve_mixed call against one
obca_parking_solve_batch call per horizon (the path a planned batch took before per-problem horizons existed).

  python tools/bench_mixed.py [--batch B] [--steps K] [--warmup W] [--nmin 40] [--nmax 80] [--dump-outputs DIR]
  python tools/bench_mixed.py --workload quadcopter [--steps K] [--warmup W] [--dump-outputs DIR]

B reverse-parking problems (SignedDist, variable time), horizon of every problem drawn uniformly from nmin..nmax with numpy
default_rng(0) (scenarios.reverse_parking_mixed_batch).  Each step solves the batch both ways, alternating, with a 256 MB L2
flush before each.  Prints ONE JSON line: `value` = converged traj/s of the single call (device time, CUDA events inside the
library), `grouped` = the same for the per-horizon calls (their device times summed), `identical` = whether both returned the
same bits for every problem.  --dump-outputs DIR: the outputs of the last single call, padded with NaN to nmax, as .npy files
(bench.py's format).

--workload quadcopter: the same comparison for config 4 (obca_quadcopter_solve_mixed against one obca_quadcopter_solve_batch call
per horizon): B = 2048 (--batch) SignedDist problems of scenarios.quadcopter_mixed_batch(B, (90, 127), seed=0), a horizon and its
sampling time Ts = round(0.25 * 80 / N, 2) per problem (defaults --nmin 90 --nmax 127; the solver takes horizons up to
N = 511, e.g. --nmin 128 --nmax 160 for a batch of long horizons only).  `value` counts exitflag == 1."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import ClockSampler, dump_outputs      # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=("parking", "quadcopter"), default="parking")
    ap.add_argument("--batch", type=int, default=None, help="default 4096 (parking) / 2048 (quadcopter)")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--nmin", type=int, default=None, help="default 40 (parking) / 90 (quadcopter)")
    ap.add_argument("--nmax", type=int, default=None, help="default 80 (parking) / 127 (quadcopter); at most 127 (parking) / 511 (quadcopter)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    if args.steps < 1:
        ap.error("--steps must be >= 1")
    quad = args.workload == "quadcopter"
    B = args.batch if args.batch is not None else (2048 if quad else 4096)
    if args.nmin is None:
        args.nmin = 90 if quad else 40
    if args.nmax is None:
        args.nmax = 127 if quad else 80
    if quad:
        return run_quadcopter(args, B)
    import torch
    import obca_b200
    from obca_b200 import parking, scenarios
    torch.cuda.set_device(0)
    opts = obca_b200.default_opts(device=0, retry=1)
    sc = scenarios.reverse_parking_mixed_batch(B, (args.nmin, args.nmax), seed=0)
    Ns = sc["Ns"]
    groups = {int(N): np.flatnonzero(Ns == N) for N in np.unique(Ns)}
    shared = (sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], sc["nOb"], sc["vOb"], sc["A"], sc["b"])

    def run_mixed():
        return parking.parking_solve_mixed(sc["x0"], sc["xF"], Ns, *shared, sc["rx"], sc["ry"], sc["ryaw"], 0, sc["xWS"], sc["uWS"],
                                           1, None, None, opts)

    def run_grouped():
        out = []
        for N, idx in groups.items():
            st = lambda key: np.stack([sc[key][i][:N] if key == "uWS" else sc[key][i] for i in idx])
            out.append((idx, parking.parking_solve_batch(sc["x0"][idx], sc["xF"], N, *shared, st("rx"), st("ry"), st("ryaw"), 0,
                                                         st("xWS"), st("uWS"), 1, None, None, opts)))
        return out
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    for _ in range(args.warmup):
        run_mixed(); run_grouped()
    sampler = ClockSampler(0); sampler.start()
    torch.cuda.synchronize()
    t_mix = t_grp = 0.0; conv_mix = conv_grp = 0; its = 0; identical = True
    for _ in range(args.steps):
        flush.zero_(); torch.cuda.synchronize()
        r = run_mixed()
        t_mix += r["time"]; conv_mix += int((r["exitflag"] == 1).sum()); its += int(r["iters"].sum())
        flush.zero_(); torch.cuda.synchronize()
        g = run_grouped()
        t_grp += sum(x["time"] for _, x in g); conv_grp += sum(int((x["exitflag"] == 1).sum()) for _, x in g)
        for idx, x in g:
            for k, i in enumerate(idx):
                identical &= all(np.array_equal(r[key][i], x[key][k]) for key in ("xp", "up", "ts", "lp", "np", "sl"))
                identical &= bool(r["exitflag"][i] == x["exitflag"][k] and r["iters"][i] == x["iters"][k])
    sampler.stop = True; sampler.join()
    if args.dump_outputs:
        Nmax = int(Ns.max())
        padded = lambda key, ext: np.stack([np.pad(a, ((0, 0), (0, Nmax + ext - a.shape[1])), constant_values=np.nan) for a in r[key]])
        arrs = {k: padded(k, 1) for k in ("xp", "lp", "np", "sl")}
        arrs["up"] = padded("up", 0)
        arrs["ts"] = np.stack([np.pad(a, (0, Nmax + 1 - a.size), constant_values=np.nan) for a in r["ts"]])
        arrs.update(exitflag=r["exitflag"], iters=r["iters"], kkt_err=r["kkt_err"], N=Ns)
        dump_outputs(args.dump_outputs, arrs, B)
    line = {"metric": "OBCA trajs/sec, mixed-horizon batch in one call", "value": conv_mix / t_mix, "unit": "traj/s", "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * t_mix / args.steps, "higher_is_better": True,
            "dtype": "f64", "data": "synthetic",
            "config": {"workload": f"reverse-parking SD var-time, 3 obstacles, N uniform over {args.nmin}..{args.nmax} "
                                   f"(numpy default_rng(0)), {len(groups)} distinct horizons",
                       "batch_per_gpu": B, "l2": "256 MB flush before each solve", "converged_frac": conv_mix / (B * args.steps),
                       "iters_mean": its / (B * args.steps)},
            "grouped": {"value": conv_grp / t_grp, "unit": "traj/s", "ms_per_step": 1e3 * t_grp / args.steps, "calls_per_step": len(groups),
                        "converged_frac": conv_grp / (B * args.steps),
                        "note": "one parking_solve_batch call per horizon, device times summed"},
            "speedup_vs_grouped": t_grp / t_mix, "identical": bool(identical),
            "clocks": sampler.result()}
    print(json.dumps(line), flush=True)


def run_quadcopter(args, B):
    import torch
    import obca_b200
    from obca_b200 import quadcopter, scenarios
    torch.cuda.set_device(0)
    opts = obca_b200.default_opts(device=0); opts.max_iter = 3000      # as quadcopter_solve_batch without opts
    sc = scenarios.quadcopter_mixed_batch(B, (args.nmin, args.nmax), seed=0)
    Ns, Ts = sc["Ns"], sc["Ts"]
    groups = {int(N): np.flatnonzero(Ns == N) for N in np.unique(Ns)}

    def run_mixed():
        return quadcopter.quadcopter_solve_mixed(sc["x0"], sc["xF"], Ns, Ts, sc["R"], sc["obs"], sc["xWS"], 1.0, 1, opts)

    def run_grouped():
        return [(idx, quadcopter.quadcopter_solve_batch(sc["x0"][idx], sc["xF"][idx], N, float(Ts[idx[0]]), sc["R"], sc["obs"],
                                                        np.stack([sc["xWS"][i] for i in idx]), 1.0, 1, opts))
                for N, idx in groups.items()]
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    for _ in range(args.warmup):
        run_mixed(); run_grouped()
    sampler = ClockSampler(0); sampler.start()
    torch.cuda.synchronize()
    t_mix = t_grp = 0.0; conv_mix = conv_grp = 0; its = 0; identical = True
    for _ in range(args.steps):
        flush.zero_(); torch.cuda.synchronize()
        r = run_mixed()
        t_mix += r["time"]; conv_mix += int((r["exitflag"] == 1).sum()); its += int(r["iters"].sum())
        flush.zero_(); torch.cuda.synchronize()
        g = run_grouped()
        t_grp += sum(x["time"] for _, x in g); conv_grp += sum(int((x["exitflag"] == 1).sum()) for _, x in g)
        for idx, x in g:
            for k, i in enumerate(idx):
                identical &= all(np.array_equal(r[key][i], x[key][k]) for key in ("xp", "up", "ts", "lp", "slack"))
                identical &= bool(r["exitflag"][i] == x["exitflag"][k] and r["iters"][i] == x["iters"][k]
                                  and r["kkt_err"][i] == x["kkt_err"][k])
    sampler.stop = True; sampler.join()
    if args.dump_outputs:
        Nmax = int(Ns.max())
        padded = lambda key, ext: np.stack([np.pad(a, ((0, 0), (0, Nmax + ext - a.shape[1])), constant_values=np.nan) for a in r[key]])
        arrs = {k: padded(k, 1) for k in ("xp", "lp", "slack")}
        arrs["up"] = padded("up", 0)
        arrs["ts"] = np.stack([np.pad(a, (0, Nmax + 1 - a.size), constant_values=np.nan) for a in r["ts"]])
        arrs.update(exitflag=r["exitflag"], iters=r["iters"], kkt_err=r["kkt_err"], N=Ns, Ts=Ts)
        dump_outputs(args.dump_outputs, arrs, B)
    line = {"metric": "OBCA trajs/sec, mixed-horizon quadcopter batch in one call", "value": conv_mix / t_mix, "unit": "traj/s",
            "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": 1e3 * t_mix / args.steps, "higher_is_better": True,
            "dtype": "f64", "data": "synthetic",
            "config": {"workload": f"quadcopter SD (config 4), N uniform over {args.nmin}..{args.nmax} (numpy default_rng(0)), "
                                   f"Ts = round(0.25 * 80 / N, 2), {len(groups)} distinct horizons",
                       "batch_per_gpu": B, "l2": "256 MB flush before each solve", "converged_frac": conv_mix / (B * args.steps),
                       "iters_mean": its / (B * args.steps)},
            "grouped": {"value": conv_grp / t_grp, "unit": "traj/s", "ms_per_step": 1e3 * t_grp / args.steps, "calls_per_step": len(groups),
                        "converged_frac": conv_grp / (B * args.steps),
                        "note": "one quadcopter_solve_batch call per horizon, device times summed"},
            "speedup_vs_grouped": t_grp / t_mix, "identical": bool(identical),
            "clocks": sampler.result()}
    print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
