"""Time per planning step with host arrays against device arrays, at cfg 2 (B = 1024, every step a cold solve: reinit = 1):

  step_pageable_ms    BatchSolver.step from pageable numpy arrays (copies and a synchronise inside the call; host clock)
  step_pinned_ms      the same with page-locked input and result buffers
  step_async_ms       step_async from torch CUDA tensors: CUDA events on the stream around K steps
  graph_replay_ms     the same step captured once in a CUDA graph and replayed K times
  costmap_host_ms     step_from_costmaps with host maps (B x 400 x 400 bytes copied per step; host clock)
  costmap_device_ms   step_from_costmaps_async with device maps read in place (events around K steps)

Results must not depend on the path: the last step of every mode is compared with the pageable one bit for bit.  Prints one JSON
line (with the card's name and power limit, read in the same run).
Usage: python tools/device_io_timing.py [--batch 1024] [--steps 10] [--map 400] [--skip-costmap]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from mpc_local_planner_b200 import capi, configs  # noqa: E402

KEYS = ("u_seq", "x_seq", "dt", "status", "kkt_err", "iters")


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], text=True, timeout=30)
        return q.strip().splitlines()[0]
    except Exception as e:   # the numbers stay valid; the card is then named by torch only
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi: {e})"


def same(a, b):
    return all(np.ascontiguousarray(a[k]).tobytes() == np.ascontiguousarray(b[k]).tobytes() for k in KEYS)


def host_ms(fn, K):
    fn()   # warm-up: allocations, module loading
    t = time.perf_counter()
    for _ in range(K):
        out = fn()
    return (time.perf_counter() - t) * 1e3 / K, out


def event_ms(fn, K, stream):
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(K):
        out = fn()
    e1.record(stream)
    e1.synchronize()
    return e0.elapsed_time(e1) / K, out


def to_host(res):
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in res.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--map", type=int, default=400)
    ap.add_argument("--skip-costmap", action="store_true")
    a = ap.parse_args()
    B, K = a.batch, a.steps
    cfg = configs.cfg2()
    d = configs.generate(2, B)
    ob = d["obstacles"]
    reinit = np.ones(B, dtype=np.uint8)
    r = dict(card=card(), config=2, batch=B, steps=K)

    s = capi.BatchSolver(cfg, B, device=0)
    r["step_pageable_ms"], ref = host_ms(lambda: s.step(d["x0"], d["xf"], d["u_prev"], 0.2, ob, None, reinit=reinit), K)

    def pin(x):
        t = torch.from_numpy(np.ascontiguousarray(x)).pin_memory()
        return t.numpy(), t
    keep = []
    px0, pxf, pup, pri = (pin(x) for x in (d["x0"], d["xf"], d["u_prev"], reinit))
    pob = tuple(pin(x) for x in ob)
    keep += [px0, pxf, pup, pri, pob]
    pout = s.alloc_outputs(B, pin=pin)
    r["step_pinned_ms"], out = host_ms(lambda: s.step(px0[0], pxf[0], pup[0], 0.2, tuple(p[0] for p in pob), None, reinit=pri[0], out=pout), K)
    r["pinned_equal"] = same(out, ref)
    s.close()

    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        s = capi.BatchSolver(cfg, B, device=0)
        s.set_stream(st.cuda_stream)
        dev = lambda x: torch.as_tensor(np.ascontiguousarray(x), device="cuda:0")  # noqa: E731
        x0, xf, up, ri = dev(d["x0"]), dev(d["xf"]), dev(d["u_prev"]), dev(reinit)
        dob = tuple(dev(x) for x in ob)
        res = {k: v for k, v in zip(KEYS, (torch.empty((B, cfg.n, 2), dtype=torch.float64, device="cuda:0"),
                                           torch.empty((B, cfg.n, 3), dtype=torch.float64, device="cuda:0"),
                                           torch.empty(B, dtype=torch.float64, device="cuda:0"), torch.empty(B, dtype=torch.int32, device="cuda:0"),
                                           torch.empty(B, dtype=torch.float64, device="cuda:0"), torch.empty(B, dtype=torch.int32, device="cuda:0")))}
        step = lambda: s.step_async(x0, xf, up, 0.2, dob, reinit=ri, out=res)  # noqa: E731
        r["step_async_ms"], out = event_ms(step, K, st)
        r["async_equal"] = same(to_host(out), ref)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        gres = s.step_async(x0, xf, up, 0.2, dob, reinit=ri)
    with torch.cuda.stream(st):
        r["graph_replay_ms"], _ = event_ms(g.replay, K, st)
        r["graph_equal"] = same(to_host(gres), ref)
    torch.cuda.synchronize()
    del g
    s.close()

    if not a.skip_costmap:
        W = H = a.map
        rng = np.random.default_rng(0)
        res_m = 0.05
        cost = rng.choice(np.array([0, 1, 100, 253], dtype=np.uint8), size=(B, H, W))
        cost[rng.random((B, H, W)) < 0.002] = 254
        origin = rng.uniform(-3, 3, (B, 2))
        pose = np.concatenate([origin + 0.5 * res_m * np.array([W, H]) + rng.uniform(-2, 2, (B, 2)), rng.uniform(-np.pi, np.pi, (B, 1))], axis=1)
        goal = pose.copy(); goal[:, 0] += 4.0 * np.cos(pose[:, 2]); goal[:, 1] += 4.0 * np.sin(pose[:, 2])
        M = 512
        r.update(map_size=W, map_bytes_per_step=int(cost.nbytes))
        s = capi.BatchSolver(cfg, B, device=0)
        r["costmap_host_ms"], cref = host_ms(lambda: s.step_from_costmaps(pose, goal, cost, origin, res_m, 0.3, M, reinit=reinit), K)
        s.close()
        with torch.cuda.stream(st):
            s = capi.BatchSolver(cfg, B, device=0)
            s.set_stream(st.cuda_stream)
            dcost, dorg, dpose, dgoal, ri = (torch.as_tensor(x, device="cuda:0") for x in (cost, origin, pose, goal, reinit))
            r["costmap_device_ms"], cout = event_ms(lambda: s.step_from_costmaps_async(dpose, dgoal, dcost, dorg, res_m, 0.3, M, reinit=ri), K, st)
            r["costmap_equal"] = same(to_host(cout), cref)
            s.close()
    print(json.dumps(r), flush=True)
    out_dir = os.environ.get("DEVICE_IO_OUT")
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "device_io_timing.json"), "w") as f:
            json.dump(r, f, indent=1)


if __name__ == "__main__":
    main()
