"""What per-robot models (mpcb200_set_robot_model) cost and what they save, instances of configs.generate at B = 1024: cold steps
(reinit = 1, every call the same problem), the median of --reps calls after a warm-up, device time from CUDA events around the calls
on one stream.  Cases:

  groups4     four model groups in one launch on cfg 3 (N = 80, minimum time): robot b in group b % 4 -- (unicycle, circular),
              (simple car, the polygon of cfg 3), (front-wheel car, two circles), (kinematic bicycle, line) -- each with its own
              model, geometry and limits records (solve_fused_models_kernel)
  handles4    the same four groups as four handles created with the group's configuration, one step each, back to back on one stream
  uni_none    cfg 2 (unicycle, point footprint, N = 50, fixed-dt quadratic form) without records: its own key
              (MODEL_UNI_POINT / PROBLEM_FIXED_DT_QF)
  uni_equal   cfg 2 with model records equal to its types: the same problem on the generic key, which every solve with model
              records runs

Prints one JSON line per case and a markdown table, with the card's name, power limit and max SM clock read in the same run.
Usage: python tools/robot_model_timing.py [--batch 1024] [--reps 7]"""
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
import robot_model_cases as rm  # noqa: E402
from mpc_local_planner_b200 import capi, configs  # noqa: E402


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True, timeout=30)
        return q.strip().splitlines()[0]
    except Exception as e:
        return f"unknown card (nvidia-smi: {e})"


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
    res = {}
    with torch.cuda.stream(st):
        def solver(c, n):
            s = capi.BatchSolver(c, n)
            s.set_stream(st.cuda_stream)
            return s

        def step(s, data, inp):
            return lambda: s.step_async(inp["x0"], inp["xf"], inp["u_prev"], data["u_prev_dt"], inp["obst"], reinit=inp["reinit"])

        host = configs.cfg3()
        data = configs.generate(3, B)
        model, limits, geometry = rm.fleet_records(host, B)
        s = solver(host, B)
        s.set_robot_limits(limits); s.set_robot_geometry(geometry); s.set_robot_model(model)
        res["groups4"] = timed([step(s, data, dev_inputs(data, np.arange(B)))], args.reps)
        conv = float((s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"])["status"] == 0).mean())
        s.close()
        hs, calls = [], []
        for g in range(4):
            idx = np.arange(g, B, 4)
            h = solver(rm.group_config(host, rm.GROUPS[g]), len(idx))
            hs.append(h)
            calls.append(step(h, data, dev_inputs(data, idx)))
        res["handles4"] = timed(calls, args.reps)
        for h in hs:
            h.close()
        uni = configs.cfg2()
        data2 = configs.generate(2, B)
        every2 = dev_inputs(data2, np.arange(B))
        s = solver(uni, B)
        res["uni_none"] = timed([step(s, data2, every2)], args.reps)
        key_none = (s.kernel_model(), s.kernel_problem())
        s.set_robot_model(np.tile(rm.record_of(uni), (B, 1)))
        res["uni_equal"] = timed([step(s, data2, every2)], args.reps)
        key_equal = (s.kernel_model(), s.kernel_problem())
        s.close()
    row = dict(B=B, **{k + "_ms": v for k, v in res.items()}, groups4_over_handles4=res["groups4"] / res["handles4"],
               uni_equal_over_none=res["uni_equal"] / res["uni_none"], groups4_converged=conv, uni_key_none=key_none,
               uni_key_equal=key_equal)
    print(json.dumps(row), flush=True)
    print("| B | groups4 ms | handles4 ms | groups4 / handles4 | cfg 2 none ms | cfg 2 equal ms | equal / none |")
    print("|---|---|---|---|---|---|---|")
    print(f"| {B} | {res['groups4']:.2f} | {res['handles4']:.2f} | {row['groups4_over_handles4']:.3f} | {res['uni_none']:.2f} | "
          f"{res['uni_equal']:.2f} | {row['uni_equal_over_none']:.3f} |")


if __name__ == "__main__":
    main()
