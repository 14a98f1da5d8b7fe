"""Critical placement (MPCB200_OPT_CRITICAL_PLACEMENT) of one workload against its plan: the heavy-part threshold PLACE_RHO and the
co-resident cap PLACE_COTENANTS are compile-time constants of the library, so each setting is a library of its own, e.g.
  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -shared -ldl -DPLACE_RHO=1.5 \
       -DPLACE_COTENANTS=1 -o /tmp/rho15c1.so mpc_local_planner_b200/csrc/mpcb200.cu mpc_local_planner_b200/csrc/mpcb200_weights.cu
Measured the way bench.py measures its headline: cold batch solves, L2 flushed before each, queue longest-first by the history of
the warm-up solves.  Each round runs every library once with the placement on, and the in-tree library with it off, so the
settings alternate; results must be identical across settings (checked).
usage: python tools/placement_sweep.py [cfg=2] [B=1024] [steps=40] [rounds=3] label=path.so ..."""
import subprocess
import sys; sys.path.insert(0, '.')
import numpy as np
from mpc_local_planner_b200 import capi, configs

pos = [a for a in sys.argv[1:] if "=" not in a]
libs = [tuple(a.split("=", 1)) for a in sys.argv[1:] if "=" in a]
cid = int(pos[0]) if len(pos) > 0 else 2
B = int(pos[1]) if len(pos) > 1 else 1024
steps = int(pos[2]) if len(pos) > 2 else 40
rounds = int(pos[3]) if len(pos) > 3 else 3
print("card:", subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True).stdout.strip())
cfg = configs.config_for(cid, tol=1e-6)
data = configs.generate(cid, B)
settings = [("off", capi.LIB_PATH, 0), ("default", capi.LIB_PATH, 1)] + [(name, path, 1) for name, path in libs]
loaded = {}
rows = {name: [] for name, _, _ in settings}
outs = {}
for r in range(rounds):
    for name, path, on in settings:
        if path not in loaded:
            loaded[path] = capi.load_library(path)
        capi._LIB = loaded[path]
        s = capi.BatchSolver(cfg, B)
        s.set_option(capi.OPT_CRITICAL_PLACEMENT, on)
        s.upload(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
        for _ in range(3):
            s.flush_l2(); s.solve_resident(cold=True)
        s.stats_reset()
        t = 0.0
        for _ in range(steps):
            s.flush_l2(); t += s.solve_resident(cold=True)
        st = s.stats()
        rows[name].append((t / steps * 1e3, sum(st["ms"]) / steps, st["gate_ms"] / steps))
        outs[name] = s.fetch()
        s.close()
print(f"cfg {cid} N {cfg.n} B {B}: {steps} steps x {rounds} rounds per setting")
for name, _, _ in settings:
    ms = [x[0] for x in rows[name]]
    print(f"  {name:10s} ms/step min {min(ms):.3f} median {np.median(ms):.3f} runs {[round(x, 3) for x in ms]}  "
          f"kernel_ms {np.mean([x[1] for x in rows[name]]):.3f}  gate {np.mean([x[2] for x in rows[name]]):.3f}", flush=True)
a = outs["off"]
print("identical results:", all(all(np.array_equal(a[k], o[k]) for k in a if k != "solve_time_s") for o in outs.values()))
