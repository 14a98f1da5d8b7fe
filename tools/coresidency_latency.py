"""Iteration latency of one instance against the number of CTAs that share its SM.
Solves B = k x SMs copies of one heavy cfg 2 instance (every CTA does identical work, one instance each) with
MPCB200_OPT_CTAS_PER_SM = k and the phase gates at their default, for k = 1..4: cold solves, L2 flushed before each.
Reports the device time of a solve, that time per iteration, and a CTA's kernel_ms (phases) and gate wait per solve.
usage: python tools/coresidency_latency.py [reps=10] [instance (default: the heaviest of the headline batch below the cap)]"""
import subprocess
import sys; sys.path.insert(0, '.')
import numpy as np
import torch
from mpc_local_planner_b200 import capi, configs

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip()
print("card:", card)
cfg = configs.config_for(2, tol=1e-6)
n_sms = torch.cuda.get_device_properties(0).multi_processor_count
data = configs.generate(2, 1024)
s = capi.BatchSolver(cfg, 1024)
out = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
s.close()
it = out["iters"]
if len(sys.argv) > 2:
    pick = int(sys.argv[2])
else:
    below = np.where(it < cfg.max_iter, it, -1)
    pick = int(np.argmax(below))
print(f"instance {pick} of the cfg 2 batch: {it[pick]} iterations (batch: mean {it.mean():.2f}, max {it.max()})")


def copies(a, B):
    return np.repeat(a[pick:pick + 1], B, axis=0)


cnt, types, params = data["obstacles"]
rows = []
for k in (1, 2, 3, 4):
    B = k * n_sms
    s = capi.BatchSolver(cfg, B)
    s.set_option(capi.OPT_CTAS_PER_SM, k)
    s.upload(copies(data["x0"], B), copies(data["xf"], B), copies(data["u_prev"], B), data["u_prev_dt"],
             (copies(cnt, B), copies(types, B), copies(params, B)), None)
    for _ in range(3):
        s.flush_l2(); s.solve_resident(cold=True)
    s.stats_reset()
    ts = []
    for _ in range(reps):
        s.flush_l2(); ts.append(s.solve_resident(cold=True) * 1e3)
    st = s.stats()
    o = s.fetch()
    s.close()
    assert (o["iters"] == o["iters"][0]).all(), "copies of one instance must run the same iterations"
    n_it = int(o["iters"][0])
    ph = np.array(st["ms"]) / reps
    rows.append((k, B, n_it, min(ts), float(np.median(ts)), max(ts), ph, st["gate_ms"] / reps))
print(f"{'CTAs/SM':>7} {'B':>5} {'iters':>5}  {'ms min':>7} {'median':>7} {'max':>7}  {'us/iter':>7}  "
      f"{'kernel_ms':>9} (init assoc eval kkt ls)  gate_ms")
t4 = rows[-1][4] / rows[-1][2]
for k, B, n_it, lo, med, hi, ph, gate in rows:
    print(f"{k:7d} {B:5d} {n_it:5d}  {lo:7.3f} {med:7.3f} {hi:7.3f}  {med / n_it * 1e3:7.1f}  {ph.sum():9.3f} "
          f"({' '.join(f'{x:.3f}' for x in ph)})  {gate:.3f}   t_k / t_4 = {med / n_it / t4:.3f}")
