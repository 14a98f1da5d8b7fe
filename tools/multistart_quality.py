"""What K candidate solves per robot buy and cost (mpcb200_step_batch_multistart), on cfg 2 and cfg 3 instances of configs.generate:
one cold call per (config, B, K), every robot from the same instances for every K.  Per row:

  converged        fraction of robots whose returned solve converged
  challenger_wins  fraction of robots whose winner is a challenger (winner > 0)
  ratio_median / ratio_worst   obj(winner) / obj(incumbent) over the robots where both converged (the incumbent's objective from
                   a second handle that runs mpcb200_step_batch on the same instances; <= 1 with hysteresis 1)
  ms / ms_vs_k1    device time of the call (solve + selection, the median of --reps calls) and its ratio to K = 1

Prints one JSON line per row and a markdown table, with the card's name and power limit read in the same run.
Usage: python tools/multistart_quality.py [--batches 16 1024] [--ks 1 2 3 5] [--reps 5]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mpc_local_planner_b200 import capi, configs  # noqa: E402


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True, timeout=30)
        return q.strip().splitlines()[0]
    except Exception as e:
        return f"unknown card (nvidia-smi: {e})"


def call(s, d, K, B):
    return s.step_multistart(d["x0"], d["xf"], K, u_prev=d["u_prev"], u_prev_dt=d["u_prev_dt"], obstacles=d["obstacles"],
                             viapoints=d["viapoints"], reinit=np.ones(B, dtype=np.uint8))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[16, 1024])
    ap.add_argument("--ks", type=int, nargs="+", default=[1, 2, 3, 5])
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    rows = []
    for cid, make in ((2, configs.cfg2), (3, configs.cfg3)):
        cfg = make()
        for B in args.batches:
            data = configs.generate(cid, B)
            twin = capi.BatchSolver(cfg, B)
            inc = twin.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
            inc_obj = twin.ws_read(capi.F_SCAL, B)[:, capi.SC_OBJ]
            inc_conv = inc["status"] == capi.STATUS_CONVERGED
            twin.close()
            ms_k1 = None
            for K in args.ks:
                s = capi.BatchSolver(cfg, B * K)
                call(s, data, K, B)   # warm-up: module load, staging arrays
                times = []
                for _ in range(args.reps):
                    r = call(s, data, K, B)   # reinit = 1: every call the same cold problem
                    times.append(r["solve_time_s"] * 1e3)
                obj = s.ws_read(capi.F_SCAL, B)[:, capi.SC_OBJ]
                s.close()
                conv = r["status"] == capi.STATUS_CONVERGED
                both = conv & inc_conv & (np.abs(inc_obj) > 0)
                ratio = obj[both] / inc_obj[both]
                ms = float(np.median(times))
                ms_k1 = ms if K == 1 else ms_k1
                row = dict(config=cid, B=B, K=K, converged=float(conv.mean()), challenger_wins=float((r["winner"] > 0).mean()),
                           ratio_median=float(np.median(ratio)) if ratio.size else None,
                           ratio_worst=float(ratio.max()) if ratio.size else None, ms=ms, ms_vs_k1=ms / ms_k1 if ms_k1 else None)
                rows.append(row)
                print(json.dumps(row), flush=True)
    print("| cfg | B | K | converged | challenger wins | obj ratio median | obj ratio worst | ms | vs K=1 |")
    print("|---|---|---|---|---|---|---|---|---|")
    f = lambda v, p: "-" if v is None else f"{v:.{p}f}"   # noqa: E731
    for r in rows:
        print(f"| {r['config']} | {r['B']} | {r['K']} | {f(r['converged'], 3)} | {f(r['challenger_wins'], 3)} | {f(r['ratio_median'], 4)} | "
              f"{f(r['ratio_worst'], 4)} | {f(r['ms'], 2)} | {f(r['ms_vs_k1'], 2)} |")


if __name__ == "__main__":
    main()
