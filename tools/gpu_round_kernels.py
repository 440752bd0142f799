"""development: per-kernel CUDA-event times of one config-2 solve (reverse parking, N = 80, 3 obstacles, B = 4096), the
schedule (rounds, problems handed to the tail kernel) and the evaluation / merit counters, as one JSON line.

    OBCA_SO=build/libobca_<name>.so python tools/gpu_round_kernels.py [--tag name]

kernel_ms slots (obca_last_schedule): [0] k_pk_eval, [1] k_pk_sweep, [2] k_pk_step, [3] k_pk_tail, [4] DualMultWS.  The
timed solve launches every round separately (no CUDA graph), so its rounds / hand-over differ a little from bench.py's."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import obca_b200  # noqa: E402
from obca_b200 import parking, scenarios  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--tag", default=os.path.basename(os.environ.get("OBCA_SO", "libobca.so")))
ap.add_argument("--repeat", type=int, default=3)
args = ap.parse_args()
sc = scenarios.reverse_parking_batch(4096, 80, 0)


def run():
    return parking.parking_solve_batch(sc["x0"], sc["xF"], 80, sc["Ts"], sc["L"], sc["ego"], sc["XYbounds"], 3, sc["vOb"], sc["A"],
                                       sc["b"], sc["rx"], sc["ry"], sc["ryaw"], 0, sc["xWS"], sc["uWS"])


os.environ["OBCA_PHASE_TIMING"] = "1"
run()
for _ in range(args.repeat):
    r = run()
    rnd = C.c_int(0); hand = C.c_int(0); kms = (C.c_double * 5)(); pr = (C.c_ulonglong * 8)()
    lib = obca_b200.lib()
    lib.obca_last_schedule(C.c_int(0), C.byref(rnd), C.byref(hand), kms)
    lib.obca_last_profile(C.c_int(0), pr)
    print(json.dumps({"tag": args.tag, "solve_ms": round(r["time"] * 1e3, 2), "rounds": rnd.value, "handed_over": hand.value,
                      "kernel_ms": [round(x, 2) for x in kms],
                      "counters": {"k1_evals_rounds": pr[7], "of_which_after_barrier_update": pr[5], "merit_evals_rounds": pr[6],
                                   "k1_evals_tail": pr[4], "merit_evals_tail": pr[3]}}), flush=True)
