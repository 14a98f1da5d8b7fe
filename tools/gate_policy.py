"""Phase-gate policy of the persistent solve kernel (MPCB200_OPT_SM_PHASE_SYNC) on one workload, measured the way bench.py
measures its headline: cold batch solves, L2 flushed before each, queue longest-first by history, warm-up steps first.
Each round runs every setting once, so the settings alternate; results must be identical across settings (checked).
Per setting: device ms per step (min / median over the rounds), the phase split of a CTA's time per step and its gate wait.
usage: python tools/gate_policy.py [cfg=2] [B=1024] [steps=40] [rounds=3] [warmup=3] [N (cfg 5 only)=50]"""
import sys; sys.path.insert(0, '.')
import numpy as np
from mpc_local_planner_b200 import capi, configs

cid = int(sys.argv[1]) if len(sys.argv) > 1 else 2
B = int(sys.argv[2]) if len(sys.argv) > 2 else 1024
steps = int(sys.argv[3]) if len(sys.argv) > 3 else 40
rounds = int(sys.argv[4]) if len(sys.argv) > 4 else 3
warmup = int(sys.argv[5]) if len(sys.argv) > 5 else 3
n = int(sys.argv[6]) if cid == 5 and len(sys.argv) > 6 else None
SETTINGS = (("off", 0), ("2 gates", 2), ("3 gates", 1), ("default", -1))
cfg = configs.config_for(cid, n=n, tol=1e-6)
data = configs.generate(cid, B, n=n)
rows = {name: [] for name, _ in SETTINGS}
outs = {}
for r in range(rounds):
    for name, sync in SETTINGS:
        s = capi.BatchSolver(cfg, B)
        s.set_option(capi.OPT_SM_PHASE_SYNC, sync)
        s.upload(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
        for _ in range(warmup):
            s.flush_l2(); s.solve_resident(cold=True)
        s.stats_reset()
        t = 0.0
        for _ in range(steps):
            s.flush_l2(); t += s.solve_resident(cold=True)
        st = s.stats()
        rows[name].append((t / steps * 1e3, [x / steps for x in st["ms"]], st["gate_ms"] / steps))
        outs[name] = s.fetch()
        s.close()
print(f"cfg {cid} N {cfg.n} B {B}: {steps} steps x {rounds} rounds per setting")
for name, _ in SETTINGS:
    ms = [x[0] for x in rows[name]]
    ph = np.mean([x[1] for x in rows[name]], axis=0)
    gate = np.mean([x[2] for x in rows[name]])
    print(f"  {name:8s} ms/step min {min(ms):.3f} median {np.median(ms):.3f} runs {[round(x, 3) for x in ms]}  "
          f"kernel_ms init {ph[0]:.3f} assoc {ph[1]:.3f} eval {ph[2]:.3f} kkt {ph[3]:.3f} ls {ph[4]:.3f}  gate {gate:.3f}", flush=True)
a = outs["off"]
print("identical results:", all(all(np.array_equal(a[k], o[k]) for k in a) for o in outs.values()))
