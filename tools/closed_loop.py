"""Receding-horizon closed loop of B simulated unicycles through the C ABI: every control cycle solves all robots' OCPs warm-started
from the previous solution (shifted on the device), applies the first control for the cycle time with the exact unicycle
flow, and feeds the new state and the applied control back -- the steady state `MpcLocalPlannerROS::computeVelocityCommands`
runs in.  Prints per-cycle device time, iterations and the fraction of robots whose solve converged.
Usage: python tools/closed_loop.py [B] [cycles] [critical placement 0|1 (default: the library's, MPCB200_OPT_CRITICAL_PLACEMENT)]"""
import sys; sys.path.insert(0, '.')
import numpy as np
from mpc_local_planner_b200 import capi, configs

B = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
cycles = int(sys.argv[2]) if len(sys.argv) > 2 else 30
T = 0.2  # control period (5 Hz, EX/launch/diff_drive_quadratic_form.launch:37)
cfg = configs.config_for(2, tol=1e-6)
data = configs.generate(2, B)
s = capi.BatchSolver(cfg, B)
if len(sys.argv) > 3:
    s.set_option(capi.OPT_CRITICAL_PLACEMENT, int(sys.argv[3]))
x = data["x0"].copy(); u_prev = data["u_prev"].copy()
alive = np.ones(B, bool)
rows = []
for c in range(cycles):
    out = s.step(x, data["xf"], u_prev, T if c else data["u_prev_dt"], data["obstacles"], None,
                 reinit=(~alive).astype(np.uint8) if c else None)
    ok = (out["status"] == capi.STATUS_CONVERGED) | (out["status"] == capi.STATUS_MAX_ITER)   # Controller::step() == true
    conv = out["status"] == capi.STATUS_CONVERGED
    u0 = np.where(ok[:, None], out["u_seq"][:, 0], 0.0)          # failed solve: stop, the planner resets (mpc_local_planner_ros.cpp:394-404)
    v, w = u0[:, 0], u0[:, 1]
    th = x[:, 2]
    sw = np.abs(w) > 1e-9
    x[:, 0] += np.where(sw, v / np.where(sw, w, 1) * (np.sin(th + w * T) - np.sin(th)), v * T * np.cos(th))
    x[:, 1] += np.where(sw, -v / np.where(sw, w, 1) * (np.cos(th + w * T) - np.cos(th)), v * T * np.sin(th))
    x[:, 2] = (th + w * T + np.pi) % (2 * np.pi) - np.pi
    u_prev = u0
    alive = ok
    dist = np.linalg.norm(x[:, :2] - data["xf"][:, :2], axis=1)
    rows.append((c, out["solve_time_s"] * 1e3, conv.mean(), ok.mean(), out["iters"].mean(), int(out["iters"].max()), np.median(dist)))
print("cycle  dev_ms  converged  usable  mean_it  max_it  median dist to goal")
for r in rows:
    print("%4d  %7.2f  %8.3f  %6.3f  %7.1f  %6d  %.2f" % r)
warm = rows[3:]
print("steady state (cycles 3..): %.2f ms per cycle for %d robots = %.0f robot-solves/s, converged %.3f" % (
    np.mean([r[1] for r in warm]), B, B / np.mean([r[1] for r in warm]) * 1e3, np.mean([r[2] for r in warm])))
s.close()
