"""What per-robot weights (mpcb200_set_robot_weights) cost and what they save, on cfg 2 (the fixed-dt quadratic-form key) and on
cfg 4 (cfg 2 with via-points), instances of configs.generate at B = 1024: cold steps (reinit = 1, every call the same problem),
the median of --reps calls after a warm-up, device time from CUDA events around the calls on one stream.  Cases:

  none        no records (solve_fused_kernel)
  equal       records equal to the configuration (solve_fused_weights_kernel, the same results)
  groups4     four weight groups in one launch: robot b in group b % 4, R scaled by 1, 2, 4, 8 and Qf by 1, 0.5, 2, 4
  handles4    the same four groups as four handles created with the group's values, one step each, back to back on one stream

Then a weight sweep, the tuning use case: one obstacle-free cfg 2 instance (a goal 1.7 m ahead and to the side, close enough
that the speed bounds do not decide the plan) replicated over R scaled by 0.25 .. 4 in one launch, and per scale the converged
control energy sum_k u_k' R0 u_k (R0 the configuration's R) and the tracking term sum_k (x_k - xf)' Q (x_k - xf) (heading
difference wrapped).  A report, not a test.

Prints one JSON line per case and two markdown tables, with the card's name, power limit and max SM clock read in the same run.
Usage: python tools/robot_weights_timing.py [--batch 1024] [--reps 7]"""
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
import robot_weights_cases as rw  # noqa: E402
from mpc_local_planner_b200 import capi, configs  # noqa: E402

R_SCALE = (1.0, 2.0, 4.0, 8.0)
QF_SCALE = (1.0, 0.5, 2.0, 4.0)
SWEEP = (0.25, 0.35, 0.5, 0.71, 1.0, 1.41, 2.0, 2.83, 4.0)


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True, timeout=30)
        return q.strip().splitlines()[0]
    except Exception as e:
        return f"unknown card (nvidia-smi: {e})"


def record(cfg, g=0):
    return rw.scaled(cfg, r=R_SCALE[g], qf=QF_SCALE[g])


def dev_inputs(d, rows):
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a[rows]), device="cuda:0")   # noqa: E731
    cnt, typ, par = d["obstacles"]
    vp = None if d["viapoints"] is None else (t(d["viapoints"][0]), t(d["viapoints"][1]))
    return dict(x0=t(d["x0"]), xf=t(d["xf"]), u_prev=t(d["u_prev"]), obst=(t(cnt), t(typ), t(par)), vp=vp,
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


def sweep():
    """one obstacle-free cfg 2 instance, one robot per R scale, one launch: control energy under R0 and tracking term per scale"""
    cfg = configs.cfg2(tol=1e-8)
    n = len(SWEEP)
    data = dict(x0=np.zeros((n, 3)), xf=np.tile([1.5, 0.8, 0.6], (n, 1)), u_prev=np.zeros((n, 2)), u_prev_dt=0.2,
                obstacles=(np.zeros(n, np.int32), np.zeros((n, 1), np.int32), np.zeros((n, 1, capi.OBST_STRIDE))), viapoints=None)
    s = capi.BatchSolver(cfg, n)
    s.set_robot_weights(np.stack([rw.scaled(cfg, r=k) for k in SWEEP]))
    out = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    s.close()
    R0, Q0 = np.array(cfg.R).reshape(2, 2), np.array(cfg.Q).reshape(3, 3)
    rows = []
    for b, k in enumerate(SWEEP):
        u, x = out["u_seq"][b], out["x_seq"][b]
        d = x - data["xf"][b]
        d[:, 2] = (d[:, 2] + np.pi) % (2 * np.pi) - np.pi
        rows.append(dict(r_scale=k, status=int(out["status"][b]), iters=int(out["iters"][b]),
                         control_energy=float(np.einsum("ki,ij,kj->", u, R0, u)), tracking=float(np.einsum("ki,ij,kj->", d, Q0, d))))
        print(json.dumps(rows[-1]), flush=True)
    return rows


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
        for name, gen in (("cfg2", 2), ("cfg4", 4)):
            cfg = configs.config_for(gen)
            data = configs.generate(gen, B)
            groups = np.arange(B) % 4
            every = dev_inputs(data, np.arange(B))

            def step(s, inp):
                return lambda: s.step_async(inp["x0"], inp["xf"], inp["u_prev"], data["u_prev_dt"], inp["obst"], inp["vp"],
                                            reinit=inp["reinit"])

            def solver(c, n):
                s = capi.BatchSolver(c, n)
                s.set_stream(st.cuda_stream)
                return s
            res = {}
            s = solver(cfg, B)
            res["none"] = timed([step(s, every)], args.reps)
            s.set_robot_weights(np.tile(record(cfg), (B, 1)))
            res["equal"] = timed([step(s, every)], args.reps)
            s.set_robot_weights(np.stack([record(cfg, g) for g in groups]))
            res["groups4"] = timed([step(s, every)], args.reps)
            s.close()
            hs, calls = [], []
            for g in range(4):
                idx = np.nonzero(groups == g)[0]
                h = solver(rw.with_weights(cfg, record(cfg, g)), len(idx))
                hs.append(h)
                calls.append(step(h, dev_inputs(data, idx)))
            res["handles4"] = timed(calls, args.reps)
            for h in hs:
                h.close()
            row = dict(config=name, B=B, **{k + "_ms": v for k, v in res.items()}, equal_over_none=res["equal"] / res["none"],
                       groups4_over_handles4=res["groups4"] / res["handles4"])
            rows.append(row)
            print(json.dumps(row), flush=True)
    sw = sweep()
    print("| cfg | B | none ms | equal ms | groups4 ms | handles4 ms | equal / none | groups4 / handles4 |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['config']} | {r['B']} | {r['none_ms']:.2f} | {r['equal_ms']:.2f} | {r['groups4_ms']:.2f} | {r['handles4_ms']:.2f} | "
              f"{r['equal_over_none']:.3f} | {r['groups4_over_handles4']:.3f} |")
    print()
    print("| R scale | status | iterations | control energy sum u' R0 u | tracking sum d' Q d |")
    print("|---|---|---|---|---|")
    for r in sw:
        print(f"| {r['r_scale']:.2f} | {r['status']} | {r['iters']} | {r['control_energy']:.4f} | {r['tracking']:.3f} |")


if __name__ == "__main__":
    main()
