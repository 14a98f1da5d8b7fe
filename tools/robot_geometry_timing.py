"""What per-robot geometry (mpcb200_set_robot_geometry) costs and what it saves, on cfg 3 (simple car, polygon footprint, N = 80)
and on cfg 3 with a two-circles footprint, instances of configs.generate at B = 1024: cold steps (reinit = 1, every call the same
problem), the median of --reps calls after a warm-up, device time from CUDA events around the calls on one stream.  Cases:

  none        no records (solve_fused_kernel)
  equal       records equal to the configuration (solve_fused_fleet_kernel, the same results)
  groups4     four geometry groups in one launch: robot b in group b % 4, the footprint scaled by 1, 0.9, 0.8, 0.7 and the
              wheelbase by 1, 1.1, 1.2, 1.3
  handles4    the same four groups as four handles created with the group's values, one step each, back to back on one stream

Prints one JSON line per case and a markdown table, with the card's name, power limit and max SM clock read in the same run.
Usage: python tools/robot_geometry_timing.py [--batch 1024] [--reps 7]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import robot_geometry_cases as rg  # noqa: E402
from mpc_local_planner_b200 import capi, configs  # noqa: E402

FOOTPRINT = (1.0, 0.9, 0.8, 0.7)
WHEELBASE = (1.0, 1.1, 1.2, 1.3)


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True, timeout=30)
        return q.strip().splitlines()[0]
    except Exception as e:
        return f"unknown card (nvidia-smi: {e})"


def record(cfg, g=0):
    return rg.scaled(cfg, FOOTPRINT[g], WHEELBASE[g])


def two_circles():
    c = configs.cfg3()
    c.footprint_type = capi.FOOTPRINT_TWO_CIRCLES
    c.footprint_params[:] = [0.2, 0.18, 0.1, 0.18]
    return c


def dev_inputs(d, rows):
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a[rows]), device="cuda:0")   # noqa: E731
    cnt, typ, par = d["obstacles"]
    return dict(x0=t(d["x0"]), xf=t(d["xf"]), u_prev=t(d["u_prev"]), obst=(t(cnt), t(typ), t(par)),
                reinit=torch.ones(len(rows), dtype=torch.uint8, device="cuda:0"))


def timed(calls, reps):
    """median device ms of running every call of `calls` once, back to back on the current stream"""
    for c in calls:
        c()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for c in calls:
            c()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    B = args.batch
    st = torch.cuda.Stream()
    rows = []
    with torch.cuda.stream(st):
        for name, make in (("cfg3", configs.cfg3), ("cfg3_two_circles", two_circles)):
            cfg = make()
            data = configs.generate(3, B)
            groups = np.arange(B) % 4
            every = dev_inputs(data, np.arange(B))

            def step(s, inp):
                return lambda: s.step_async(inp["x0"], inp["xf"], inp["u_prev"], data["u_prev_dt"], inp["obst"], reinit=inp["reinit"])

            def solver(c, n):
                s = capi.BatchSolver(c, n)
                s.set_stream(st.cuda_stream)
                return s
            res = {}
            s = solver(cfg, B)
            res["none"] = timed([step(s, every)], args.reps)
            s.set_robot_geometry(np.tile(record(cfg), (B, 1)))
            res["equal"] = timed([step(s, every)], args.reps)
            s.set_robot_geometry(np.stack([record(cfg, g) for g in groups]))
            res["groups4"] = timed([step(s, every)], args.reps)
            s.close()
            hs, calls = [], []
            for g in range(4):
                idx = np.nonzero(groups == g)[0]
                h = solver(rg.with_geometry(cfg, record(cfg, g)), len(idx))
                hs.append(h)
                calls.append(step(h, dev_inputs(data, idx)))
            res["handles4"] = timed(calls, args.reps)
            for h in hs:
                h.close()
            row = dict(config=name, B=B, **{k + "_ms": v for k, v in res.items()}, equal_over_none=res["equal"] / res["none"],
                       groups4_over_handles4=res["groups4"] / res["handles4"])
            rows.append(row)
            print(json.dumps(row), flush=True)
    print("| cfg | B | none ms | equal ms | groups4 ms | handles4 ms | equal / none | groups4 / handles4 |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['config']} | {r['B']} | {r['none_ms']:.2f} | {r['equal_ms']:.2f} | {r['groups4_ms']:.2f} | {r['handles4_ms']:.2f} | "
              f"{r['equal_over_none']:.3f} | {r['groups4_over_handles4']:.3f} |")


if __name__ == "__main__":
    main()
