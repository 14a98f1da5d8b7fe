"""Per-robot weights (mpcb200_set_robot_weights) on the GPU: records equal to the configuration change nothing, a mixed batch is bit
for bit one handle per weight group (cold and warm, in every per-robot-weights kernel and under the execution options), parity
with the oracle, changed weights warm-start under the new values, the async setter and CUDA graphs, the validation and the refused
calls, the kernel key and the C++ mirror."""
import os
import re
import subprocess

import numpy as np
import pytest

import costmap_cases as cm
import robot_geometry_cases as rg
import robot_weights_cases as rw
from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu
OUT = ("u_seq", "x_seq", "dt", "status", "kkt_err", "iters")
WARM = (capi.F_X, capi.F_U, capi.F_NU, capi.F_S, capi.F_LAM, capi.F_OBSIDX, capi.F_SCAL)
U_TOL = 1e-4


def _rows(d, idx):
    cnt, typ, par = d["obstacles"]
    vp = None if d["viapoints"] is None else (d["viapoints"][0][idx], d["viapoints"][1][idx])
    return dict(x0=d["x0"][idx], xf=d["xf"][idx], u_prev=d["u_prev"][idx], u_prev_dt=d["u_prev_dt"],
                obstacles=(cnt[idx], typ[idx], par[idx]), viapoints=vp)


def _moved(data, t):
    d = dict(data)
    d["x0"] = data["x0"] + t * (data["xf"] - data["x0"]) * np.array([1.0, 1.0, 0.0])
    return d


def _step(s, d, K=1):
    if K > 1:
        return s.step_multistart(d["x0"], d["xf"], K, u_prev=d["u_prev"], u_prev_dt=d["u_prev_dt"], obstacles=d["obstacles"],
                                 viapoints=d["viapoints"])
    return s.step(d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], d["viapoints"])


def _same(a, b, what, rows=slice(None), rows_b=None, keys=OUT):
    for k in keys:
        x, y = np.ascontiguousarray(a[k][rows]), np.ascontiguousarray(b[k][rows if rows_b is None else rows_b])
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), f"{what}: {k} differs"


def _limits_of(cfg, B):
    return np.tile(np.array(list(cfg.u_lb) + list(cfg.u_ub) + list(cfg.du_lb) + list(cfg.du_ub) + [cfg.min_obstacle_dist]), (B, 1))


def _generic_qf():
    """cfg 3 (simple car, polygon footprint) with cfg 2's quadratic form and fixed dt: a generic-key handle that reads weights and
    geometry"""
    c, q = configs.cfg3(n=50), configs.cfg2()
    c.objective, c.variable_dt, c.xf_fixed[:] = capi.OBJ_QUADRATIC_FORM, 0, [0, 0, 0]
    c.Q[:], c.R[:], c.terminal_cost, c.Qf[:], c.dt_ref = list(q.Q), list(q.R), q.terminal_cost, list(q.Qf), q.dt_ref
    return c


# ---- 1. records equal to the configuration ----
@pytest.mark.parametrize("name", ["cfg2", "cfg4", "integral", "hybrid", "ball", "mintime_vp"])
def test_records_equal_to_the_config_change_nothing(name):
    cfg, gen = rw.variant(name)
    B = 48
    data = configs.generate(gen, B)
    a, b = capi.BatchSolver(cfg, B), capi.BatchSolver(cfg, B)
    a.set_robot_weights(rw.records_of(cfg, B))
    for t in range(3):
        d = _moved(data, 0.05 * t)
        _same(_step(a, d), _step(b, d), f"{name} call {t}")
    assert (a.kernel_model(), a.kernel_problem()) == (b.kernel_model(), b.kernel_problem())
    a.set_robot_weights(None)
    d = _moved(data, 0.15)
    _same(_step(a, d), _step(b, d), f"{name} after clearing")
    a.close(); b.close()


def test_records_equal_to_the_config_with_limits_and_geometry():
    cfg, B = _generic_qf(), 48
    data = configs.generate(3, B)
    a, b = capi.BatchSolver(cfg, B), capi.BatchSolver(cfg, B)
    a.set_robot_weights(rw.records_of(cfg, B))
    for h in (a, b):
        h.set_robot_limits(_limits_of(cfg, B))
        h.set_robot_geometry(rg.records_of(cfg, B))
    for t in range(2):
        d = _moved(data, 0.05 * t)
        _same(_step(a, d), _step(b, d), f"limits + geometry call {t}")
    a.close(); b.close()


def test_records_equal_to_the_config_multistart_costmaps_and_async():
    torch = pytest.importorskip("torch")
    cfg, B, K = configs.cfg2(), 24, 3
    data = configs.generate(2, B)
    a, b = capi.BatchSolver(cfg, B * K), capi.BatchSolver(cfg, B * K)
    a.set_robot_weights(rw.records_of(cfg, B))
    for t in range(2):   # multistart: one record per robot covers its K candidates
        d = _moved(data, 0.05 * t)
        ra, rb = _step(a, d, K), _step(b, d, K)
        _same(ra, rb, f"multistart call {t}")
        assert np.array_equal(ra["winner"], rb["winner"])
    a.close(); b.close()
    cost, origin, res, pose, goal = cm.costmap_scene(B, 0.006, 21)
    chain, plain = capi.BatchSolver(cfg, B), capi.BatchSolver(cfg, B)
    chain.set_robot_weights(rw.records_of(cfg, B))
    x0, up = pose, np.zeros((B, 2))
    for cycle in range(2):
        got = chain.step_from_costmaps(x0, goal, cost, origin, res, 0.3, 256, u_prev=up, u_prev_dt=0.2)
        want = plain.step_from_costmaps(x0, goal, cost, origin, res, 0.3, 256, u_prev=up, u_prev_dt=0.2)
        _same(got, want, f"costmap cycle {cycle}")
        x0, up = want["x_seq"][:, 1].copy(), want["u_seq"][:, 0].copy()
    chain.close(); plain.close()
    dev = lambda a_: torch.as_tensor(np.ascontiguousarray(a_), device="cuda:0")   # noqa: E731
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        s, p = capi.BatchSolver(cfg, B), capi.BatchSolver(cfg, B)
        for h in (s, p):
            h.set_stream(st.cuda_stream)
        s.set_robot_weights_async(dev(rw.records_of(cfg, B)))
        args = (dev(data["x0"]), dev(data["xf"]), dev(data["u_prev"]), data["u_prev_dt"], tuple(dev(x) for x in data["obstacles"]))
        got, want = s.step_async(*args), p.step_async(*args)
        torch.cuda.synchronize()
        _same({k: v.cpu().numpy() for k, v in got.items()}, {k: v.cpu().numpy() for k, v in want.items()}, "async")
        s.close(); p.close()


# ---- 2. a mixed batch against one handle per weight group ----
def _mixed_vs_groups(cfg, data, B, K, opts):
    rec, groups = rw.group_records(cfg, B)
    s = capi.BatchSolver(cfg, B * K)
    for o, v in opts:
        s.set_option(o, v)
    s.set_robot_weights(rec)
    hs = []
    for g, idx in enumerate(groups):
        h = capi.BatchSolver(rw.with_weights(cfg, rec[idx[0]]), len(idx) * K)
        for o, v in opts:
            h.set_option(o, v)
        hs.append(h)
    for t in range(2):   # cold, then warm
        d = _moved(data, 0.05 * t)
        r = _step(s, d, K)
        wm = {f: s.ws_read(f, B) for f in WARM}
        for g, idx in enumerate(groups):
            rh = _step(hs[g], _rows(d, idx), K)
            _same(r, rh, f"call {t} group {g}", rows=idx, rows_b=slice(None))
            if K > 1:
                assert np.array_equal(r["winner"][idx], rh["winner"])
            for f in WARM:
                assert wm[f][idx].tobytes() == hs[g].ws_read(f, len(idx)).tobytes(), f"call {t} group {g} warm field {f}"
    key = (s.kernel_model(), s.kernel_problem())
    assert all((h.kernel_model(), h.kernel_problem()) == key for h in hs)
    conv = (r["status"] == capi.STATUS_CONVERGED).mean()
    for h in hs:
        h.close()
    s.close()
    return conv, key


def _weights_case(lines, ext, small):
    """cfg 2 in each per-robot-weights kernel shape: fixed dt (the fixed-dt quadratic-form key without line obstacles) or a free dt
    in integral form (EXT), N = 40 (small CTA) or 80, with or without line obstacles (LINES, the generic key)"""
    c = configs.cfg2_integral_form(n=40 if small else 80) if ext else configs.cfg2(n=40 if small else 80)
    return c


@pytest.mark.parametrize("lines", [False, True])
@pytest.mark.parametrize("ext", [False, True])
@pytest.mark.parametrize("small", [False, True])
@pytest.mark.parametrize("K", [1, 3])
def test_mixed_batch_equals_one_handle_per_group(lines, ext, small, K):
    """B well above the CTA count, so each CTA solves robots of several groups in turn; the warm call is history-ordered (and
    placed) by default, the cold one is not"""
    cfg = _weights_case(lines, ext, small)
    B = 1200 if K == 1 else 400
    data = configs.generate(2, B)
    data = configs.with_line_obstacles(data) if lines else data
    conv, key = _mixed_vs_groups(cfg, data, B, K, ())
    assert conv > 0, conv
    want = (capi.MODEL_GENERIC, capi.PROBLEM_GENERIC) if lines else \
        (capi.MODEL_UNI_POINT, capi.PROBLEM_GENERIC if ext else capi.PROBLEM_FIXED_DT_QF)
    assert key == want


@pytest.mark.parametrize("opts", [((capi.OPT_SM_PHASE_SYNC, 1),), ((capi.OPT_CTAS_PER_SM, 2),), ((capi.OPT_ORDER_BY_HISTORY, 0),),
                                  ((capi.OPT_CRITICAL_PLACEMENT, 0),)])
def test_mixed_batch_with_execution_options(opts):
    _mixed_vs_groups(configs.cfg2(), configs.generate(2, 800), 800, 1, opts)


def test_mixed_batch_via_points_and_generic_key():
    """the via-point weights (cfg 4) and the generic key with limits and geometry records as well (all three patches per robot)"""
    cfg = configs.cfg4()
    _mixed_vs_groups(cfg, configs.generate(4, 800), 800, 1, ())
    cfg, B = _generic_qf(), 400
    data = configs.generate(3, B)
    rec, groups = rw.group_records(cfg, B)
    geo = np.stack([rg.scaled(cfg, (1.0, 0.9, 0.8, 0.7)[b % 4], 1.0) for b in range(B)])
    s = capi.BatchSolver(cfg, B)
    s.set_robot_limits(_limits_of(cfg, B)); s.set_robot_geometry(geo); s.set_robot_weights(rec)
    r = _step(s, data)
    for g, idx in enumerate(groups):
        h = capi.BatchSolver(rw.with_weights(rg.with_geometry(cfg, geo[idx[0]]), rec[idx[0]]), len(idx))
        _same(r, _step(h, _rows(data, idx)), f"limits + geometry + weights group {g}", rows=idx, rows_b=slice(None))
        h.close()
    s.close()


# ---- 3. oracle parity per robot ----
@pytest.mark.parametrize("name", ["cfg2", "cfg4"])
def test_oracle_parity_per_robot(orc, name):
    """each group against the oracle run with that group's configuration, at the thresholds of test_gpu_parity's solve parity
    (fixed dt: the controls within 1e-4 on all converged instances but one)"""
    cfg, gen = rw.variant(name)
    cfg.tol = 1e-8
    B = 32
    data = configs.generate(gen, B)
    rec, groups = rw.group_records(cfg, B)
    s = capi.BatchSolver(cfg, B)
    s.set_robot_weights(rec)
    out = _step(s, data)
    ref = {k: np.empty_like(v) for k, v in out.items() if k in OUT}
    for idx in groups:
        rr = orc.step_batch(rw.with_weights(cfg, rec[idx[0]]), _rows(data, idx), n_threads=4)
        for k in ref:
            ref[k][idx] = rr[k]
    agree = (out["status"] == ref["status"]).sum()
    both = (out["status"] == 0) & (ref["status"] == 0)
    assert agree >= B - 1, f"gpu {out['status']} oracle {ref['status']}"
    assert both.sum() >= max((ref["status"] == 0).sum(), 1) - 1
    du = np.abs(out["u_seq"][both] - ref["u_seq"][both]).max(axis=(1, 2))
    assert (du < U_TOL).sum() >= len(du) - 1, f"du {du}"
    s.close()


# ---- 4. changed weights warm-start under the new values ----
@pytest.mark.parametrize("name", ["cfg2", "cfg4"])
def test_changed_weights_warm_start_under_the_new_values(name):
    cfg, gen = rw.variant(name)
    B = 16
    data = configs.generate(gen, B)
    r1, _ = rw.group_records(cfg, B)
    r2 = r1[::-1].copy()   # every robot moves to another group
    s = capi.BatchSolver(cfg, B)
    s.set_robot_weights(r1)
    _step(s, data)
    twins = [capi.BatchSolver(rw.with_weights(cfg, r2[b]), 1) for b in range(B)]
    for b in range(B):
        _step(twins[b], _rows(data, slice(b, b + 1)))
    s.set_robot_weights(r2)
    for t in (1, 2):
        state = {f: s.ws_read(f, B) for f in WARM}
        d = _moved(data, 0.05 * t)
        r = _step(s, d)
        for b in range(B):
            for f in WARM:
                twins[b].ws_write(f, state[f][b:b + 1])
            _same(r, _step(twins[b], _rows(d, slice(b, b + 1))), f"{name} call {t + 1} robot {b}", rows=slice(b, b + 1),
                  rows_b=slice(0, 1))
    for t_ in twins:
        t_.close()
    s.close()


# ---- 5. the async setter and CUDA graphs ----
def test_async_setter_and_graph_replay():
    torch = pytest.importorskip("torch")
    cfg, B = configs.cfg2(), 64
    data = configs.generate(2, B)
    r1, _ = rw.group_records(cfg, B)
    r2 = r1[::-1].copy()
    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a), device="cuda:0")   # noqa: E731
    host = lambda res: {k: v.cpu().numpy() for k, v in res.items()}            # noqa: E731
    blocking = capi.BatchSolver(cfg, B)
    blocking.set_robot_weights(r1)
    want1 = _step(blocking, data)
    blocking.set_robot_weights(r2)
    want2 = _step(blocking, _moved(data, 0.05))
    st = torch.cuda.Stream()
    ob = tuple(dev(a) for a in data["obstacles"])
    with torch.cuda.stream(st):
        s = capi.BatchSolver(cfg, B)
        s.set_stream(st.cuda_stream)
        wgt = dev(r1)
        x0, xf, up = dev(data["x0"]), dev(data["xf"]), dev(data["u_prev"])
        s.set_robot_weights_async(wgt)
        res = s.step_async(x0, xf, up, data["u_prev_dt"], ob)
        torch.cuda.synchronize()
        _same(host(res), want1, "async setter + async step")
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            s.set_robot_weights_async(wgt)
            out = s.step_async(x0, xf, up, data["u_prev_dt"], ob)
        wgt.copy_(dev(r2))
        x0.copy_(dev(_moved(data, 0.05)["x0"]))
        g.replay()
        torch.cuda.synchronize()
        _same(host(out), want2, "graph replay with rewritten weights")
        del g
        bad = r2.copy()
        bad[5, rw.Q + 4] = np.nan   # a state weight NaN: only robot 5 is INVALID_INPUT
        bad[9, rw.QF] = np.inf      # a terminal weight inf: only robot 9
        bad[12, rw.VPP] = np.nan    # cfg 2 has no via-points: the word is not read, robot 12 is solved
        fresh = capi.BatchSolver(cfg, B)
        fresh.set_stream(st.cuda_stream)
        fresh.set_robot_weights_async(dev(bad))
        got = host(fresh.step_async(x0, xf, up, data["u_prev_dt"], ob))
        torch.cuda.synchronize()
        assert got["status"][5] == got["status"][9] == capi.STATUS_INVALID_INPUT
        ref = capi.BatchSolver(cfg, B)
        ref.set_robot_weights(r2)
        want = _step(ref, _moved(data, 0.05))
        keep = (np.arange(B) != 5) & (np.arange(B) != 9)
        _same(got, want, "the robots with valid records", rows=keep)
        fresh.close(); ref.close(); s.close()
    blocking.close()


# ---- 6. validation and refused calls ----
def test_validation_and_refused_calls_leave_the_state_alone():
    cfg, B = configs.cfg4(), 16
    data = configs.generate(4, B)
    good, _ = rw.group_records(cfg, B)
    s, twin = capi.BatchSolver(cfg, 3 * B), capi.BatchSolver(cfg, 3 * B)
    for h in (s, twin):
        h.set_robot_weights(good)
        _step(h, data)

    def refused(code, call):
        with pytest.raises(capi.SolverError, match=rf"\({code}\)"):
            call()

    def bad(i, w, v):
        r = good.copy(); r[i, w] = v
        return r
    for r in (bad(3, rw.Q, np.nan), bad(3, rw.R + 3, np.inf), bad(2, rw.QF + 8, -np.inf), bad(1, rw.VPP, np.nan),
              bad(0, rw.VPO, np.inf)):
        refused(-1, lambda: s.set_robot_weights(r))
    refused(-1, lambda: s.set_robot_weights(np.tile(good[0], (3 * B + 1, 1))))
    assert s.lib.mpcb200_set_robot_weights(s.h, -1, None) == capi.E_INVALID
    big = configs.generate(4, B + 1)
    refused(-1, lambda: _step(s, big))
    refused(-1, lambda: _step(s, big, 2))
    refused(-2, lambda: s.solve_stream(data["x0"], data["xf"]))
    s.set_option(capi.OPT_SOLVE_MODE, capi.SOLVE_PHASED)
    refused(-2, lambda: _step(s, data))
    s.set_option(capi.OPT_SOLVE_MODE, capi.SOLVE_FUSED)
    refused(-2, lambda: s.run_phase(capi.PHASE_EVAL, B))
    refused(-2, lambda: s.time_phase(capi.PHASE_EVAL, reps=1))
    d = _moved(data, 0.05)
    _same(_step(s, d), _step(twin, d), "after the refused calls")
    s.close(); twin.close()
    # the hybrid term: a record cannot switch it off on a hybrid handle, nor on on a handle whose flag fell back
    hyb = configs.cfg2_hybrid_min_time()
    h = capi.BatchSolver(hyb, B)
    h.set_robot_weights(rw.records_of(hyb, B))
    r = rw.records_of(hyb, B); r[4, rw.Q] = 1.0
    refused(-1, lambda: h.set_robot_weights(r))
    r = rw.records_of(hyb, B); r[4, rw.R:rw.R + 4] = 0.0
    refused(-1, lambda: h.set_robot_weights(r))
    h.close()
    fall = configs.cfg2_integral_form()
    fall.hybrid_cost_minimum_time = 1   # non-zero Q: the plain quadratic form
    h = capi.BatchSolver(fall, B)
    r = rw.records_of(fall, B); r[7, rw.Q:rw.Q + 9] = 0.0
    refused(-1, lambda: h.set_robot_weights(r))
    h.close()
    for c in (configs.cfg1(), configs.cfg3()):   # minimum time without terminal cost: no weight is read
        h = capi.BatchSolver(c, B)
        refused(-1, lambda: h.set_robot_weights(rw.records_of(c, B)))
        assert h.lib.mpcb200_set_robot_weights_async(h.h, B, 16) == capi.E_INVALID   # refused before the pointer is looked at
        h.set_robot_weights(None)
        h.close()


# ---- 7. the kernel key ----
@pytest.mark.parametrize("name", ["cfg2", "cfg4"])
def test_kernel_key_with_records(name):
    cfg, gen = rw.variant(name)
    B = 8
    a = capi.BatchSolver(cfg, B)
    a.set_robot_weights(rw.group_records(cfg, B)[0])
    _step(a, configs.generate(gen, B))
    assert (a.kernel_model(), a.kernel_problem()) == (capi.MODEL_UNI_POINT, capi.PROBLEM_FIXED_DT_QF)
    a.close()


# ---- 8. the C++ mirror ----
def test_cpp_mirror_weights_change_the_plan_and_survive_reset():
    """tests/robot_weights/controller_weights.cpp: R grows eightfold from the second step on (Controller::setRobotWeights); the
    first plan equals that of a controller with the configuration's weights, the later ones do not, and after reset() the cold
    plan equals that of a controller configured with the new weights"""
    from tests.conftest import ROOT
    here = os.path.join(ROOT, "tests", "robot_weights")
    out = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"controller_weights_{os.getpid()}")
    lib = os.path.join(ROOT, "mpc_local_planner_b200")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", out, os.path.join(here, "controller_weights.cpp"), f"-L{lib}",
                           "-lmpcb200", f"-Wl,-rpath,{lib}", "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"])
    p = subprocess.run([out], capture_output=True, text=True, timeout=300)
    os.unlink(out)
    assert p.returncode == 0, p.stdout + p.stderr
    rows = re.findall(r"step (\d+) status (\d+) iters (\d+) same_as_plain (\d)", p.stdout)
    assert len(rows) == 3 and all(r[1] == "0" for r in rows), p.stdout
    assert [r[3] for r in rows] == ["1", "0", "0"], p.stdout
    m = re.search(r"after reset status (\d+) same_as_heavy (\d) same_as_plain (\d)", p.stdout)
    assert m and m.groups() == ("0", "1", "0"), p.stdout
