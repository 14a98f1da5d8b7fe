"""solver/ipopt/max_cpu_time on the headline workload: cfg 2, B = 1024, cold, resident inputs (bench.py's `value` path), first
without a budget, then under budgets of 25 / 50 / 75 % of that run's own ms per step.  Per budget: solve time per step (solve_time_s
of mpcb200_solve_resident -- CUDA events around the queue-order and solve kernels, the L2 flush between steps is outside) mean and
max, the overshoot (max - budget), converged % and MAX_TIME %, mean iterations and the median KKT error of the MAX_TIME instances
(instances of the last step).  Prints one JSON object with the card's name and power limit.
usage: python tools/budget_sweep.py [steps=10] [warmup=3]"""
import json
import subprocess
import sys

sys.path.insert(0, ".")
import numpy as np  # noqa: E402

from mpc_local_planner_b200 import capi, configs  # noqa: E402


def card():
    """name and power limit (W) of GPU 0, read (not set) through nvidia-smi"""
    try:
        o = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                                    timeout=10).decode().strip().split(",")
        return {"gpu": o[0].strip(), "power_limit_w": float(o[1]), "sm_max_mhz": float(o[2])}
    except Exception as e:
        return {"gpu": None, "power_limit_w": None, "error": repr(e)}


def run(budget_s, data, B, steps, warmup):
    cfg = configs.config_for(2, tol=1e-6)
    if budget_s is not None:
        cfg.max_cpu_time = budget_s
    s = capi.BatchSolver(cfg, B, device=0)
    s.upload(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
    for _ in range(warmup):
        s.flush_l2(); s.solve_resident(cold=True)
    ms = []
    for _ in range(steps):
        s.flush_l2()
        ms.append(s.solve_resident(cold=True) * 1e3)
    r = s.fetch()
    s.close()
    mt = r["status"] == capi.STATUS_MAX_TIME
    return {"solve_ms_mean": float(np.mean(ms)), "solve_ms_max": float(np.max(ms)), "converged_pct": 100.0 * float((r["status"] == 0).mean()),
            "max_time_pct": 100.0 * float(mt.mean()), "mean_ipm_iterations": float(r["iters"].mean()),
            "median_kkt_err_max_time": float(np.median(r["kkt_err"][mt])) if mt.any() else None}


def main():
    steps = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    warmup = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    B = 1024
    data = configs.generate(2, B)
    base = run(None, data, B, steps, warmup)
    rows = []
    for frac in (0.25, 0.5, 0.75):
        budget_ms = frac * base["solve_ms_mean"]
        r = run(budget_ms * 1e-3, data, B, steps, warmup)
        rows.append(dict(budget_frac=frac, budget_ms=budget_ms, overshoot_ms=r["solve_ms_max"] - budget_ms, **r))
    print(json.dumps({"workload": "cfg 2, B = 1024, cold, resident inputs", "steps_per_budget": steps, "unbudgeted": base,
                      "budgets": rows, **card()}))


if __name__ == "__main__":
    main()
