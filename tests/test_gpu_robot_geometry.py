"""Per-robot geometry (mpcb200_set_robot_geometry) on the GPU: records equal to the configuration change nothing, a mixed batch is
bit for bit one handle per geometry group (cold and warm, in every per-robot-geometry kernel), changed geometry warm-starts under
the new values, converged plans keep their own footprint and dynamics, parity with the oracle, the async setter and CUDA graphs,
the validation, the kernel key and the C++ mirror."""
import os
import re
import subprocess

import numpy as np
import pytest

import costmap_cases as cm
import robot_geometry_cases as rg
from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu
OUT = ("u_seq", "x_seq", "dt", "status", "kkt_err", "iters")
WARM = (capi.F_X, capi.F_U, capi.F_NU, capi.F_S, capi.F_LAM, capi.F_OBSIDX, capi.F_SCAL)
GROUP_FP, GROUP_WB = (1.0, 0.9, 0.8, 0.7), (1.0, 1.1, 1.2, 1.3)


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


def _groups(cfg, B):
    """four geometry groups, robot b in group b mod 4: footprint scaled by 1, 0.9, 0.8, 0.7, wheelbase / lengths by 1 .. 1.3"""
    rec = np.stack([rg.scaled(cfg, GROUP_FP[b % 4], GROUP_WB[b % 4]) for b in range(B)])
    return rec, [np.arange(g, B, 4) for g in range(4)]


def _fleet_case(lines, ext, small):
    """cfg 3 (simple car, polygon footprint) in each per-robot-geometry kernel shape: free dt (EXT, minimum time) or fixed dt
    (quadratic form), N = 40 (small CTA) or 80, with or without line obstacles (LINES)"""
    c = configs.cfg3(n=40 if small else 80)
    if not ext:
        q = configs.cfg2()
        c.objective, c.variable_dt, c.xf_fixed[:] = capi.OBJ_QUADRATIC_FORM, 0, [0, 0, 0]
        c.Q[:], c.R[:], c.terminal_cost, c.Qf[:], c.dt_ref = list(q.Q), list(q.R), q.terminal_cost, list(q.Qf), q.dt_ref
    return c


def _data(cfg, B, lines):
    d = configs.generate(3, B)
    return configs.with_line_obstacles(d) if lines else d


@pytest.mark.parametrize("name", ["cfg3", "circular", "two_circles", "line", "bicycle"])
def test_records_equal_to_the_config_change_nothing(name):
    cfg, _ = rg.variant(name)
    B = 48
    data = configs.generate(3, B)
    a, b = capi.BatchSolver(cfg, B), capi.BatchSolver(cfg, B)
    a.set_robot_geometry(rg.records_of(cfg, B))
    for t in range(3):
        d = _moved(data, 0.05 * t)
        _same(_step(a, d), _step(b, d), f"{name} call {t}")
    assert a.kernel_model() == b.kernel_model() == capi.MODEL_GENERIC
    a.set_robot_geometry(None)
    d = _moved(data, 0.15)
    _same(_step(a, d), _step(b, d), f"{name} after clearing")
    a.close(); b.close()


def test_records_equal_to_the_config_with_limits_multistart_and_costmaps():
    cfg, B, K = configs.cfg3(), 24, 3
    data = configs.generate(3, B)
    lim = np.tile(np.array(list(cfg.u_lb) + list(cfg.u_ub) + list(cfg.du_lb) + list(cfg.du_ub) + [cfg.min_obstacle_dist]), (B, 1))
    a, b = capi.BatchSolver(cfg, B * K), capi.BatchSolver(cfg, B * K)
    a.set_robot_geometry(rg.records_of(cfg, B))
    for t in range(2):   # multistart: one record per robot covers its K candidates
        d = _moved(data, 0.05 * t)
        ra, rb = _step(a, d, K), _step(b, d, K)
        _same(ra, rb, f"multistart call {t}")
        assert np.array_equal(ra["winner"], rb["winner"])
    a.set_robot_limits(lim); b.set_robot_limits(lim)   # limits records as well: the fleet kernel applies both
    d = _moved(data, 0.1)
    _same(_step(a, d), _step(b, d), "with limits records")
    a.close(); b.close()
    cost, origin, res, pose, goal = cm.costmap_scene(B, 0.006, 21)
    chain, plain = capi.BatchSolver(cfg, B), capi.BatchSolver(cfg, B)
    chain.set_robot_geometry(rg.records_of(cfg, B))
    x0, up = pose, np.zeros((B, 2))
    for cycle in range(2):
        got = chain.step_from_costmaps(x0, goal, cost, origin, res, 0.3, 256, u_prev=up, u_prev_dt=0.2)
        want = plain.step_from_costmaps(x0, goal, cost, origin, res, 0.3, 256, u_prev=up, u_prev_dt=0.2)
        _same(got, want, f"costmap cycle {cycle}")
        x0, up = want["x_seq"][:, 1].copy(), want["u_seq"][:, 0].copy()
    chain.close(); plain.close()


def _mixed_vs_groups(cfg, data, B, K, opts):
    rec, groups = _groups(cfg, B)
    s = capi.BatchSolver(cfg, B * K)
    for o, v in opts:
        s.set_option(o, v)
    s.set_robot_geometry(rec)
    hs = []
    for g, idx in enumerate(groups):
        h = capi.BatchSolver(rg.with_geometry(cfg, rec[idx[0]]), len(idx) * K)
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
    conv = (r["status"] == capi.STATUS_CONVERGED).mean()
    for h in hs:
        h.close()
    s.close()
    return conv


@pytest.mark.parametrize("lines", [False, True])
@pytest.mark.parametrize("ext", [False, True])
@pytest.mark.parametrize("small", [False, True])
@pytest.mark.parametrize("K", [1, 3])
def test_mixed_batch_equals_one_handle_per_group(lines, ext, small, K):
    """B well above the CTA count, so each CTA solves robots of several groups in turn; the warm call is history-ordered (and
    placed) by default, the cold one is not"""
    cfg = _fleet_case(lines, ext, small)
    B = 1200 if K == 1 else 400
    data = _data(cfg, B, lines)
    conv = _mixed_vs_groups(cfg, data, B, K, ())
    assert conv > 0, conv


@pytest.mark.parametrize("opts", [((capi.OPT_ORDER_BY_HISTORY, 0),), ((capi.OPT_CRITICAL_PLACEMENT, 0),)])
def test_mixed_batch_with_execution_options(opts):
    cfg = _fleet_case(False, True, False)
    _mixed_vs_groups(cfg, configs.generate(3, 800), 800, 1, opts)


def test_polygons_of_3_to_16_vertices_in_one_launch():
    cfg, B = configs.cfg3(), 600
    data = configs.generate(3, B)
    rec = rg.random_records(cfg, B, 17)
    s = capi.BatchSolver(cfg, B)
    s.set_robot_geometry(rec)
    r = _step(s, data)
    for g in range(14):   # robots b = g mod 14 have a polygon of 3 + g vertices; check a few of each against their own handle
        for b in range(g, B, 14 * 11):
            one = capi.BatchSolver(rg.with_geometry(cfg, rec[b]), 1)
            _same(r, _step(one, _rows(data, slice(b, b + 1))), f"robot {b} ({3 + g} vertices)", rows=slice(b, b + 1),
                  rows_b=slice(0, 1))
            one.close()
    s.close()


@pytest.mark.parametrize("name", ["cfg3", "bicycle"])
def test_changed_geometry_warm_starts_under_the_new_values(name):
    cfg, _ = rg.variant(name)
    B = 16
    data = configs.generate(3, B)
    r1, r2 = rg.random_records(cfg, B, 7), rg.random_records(cfg, B, 8)
    s = capi.BatchSolver(cfg, B)
    s.set_robot_geometry(r1)
    _step(s, data)
    twins = [capi.BatchSolver(rg.with_geometry(cfg, r2[b]), 1) for b in range(B)]
    for b in range(B):
        _step(twins[b], _rows(data, slice(b, b + 1)))
    s.set_robot_geometry(r2)
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


@pytest.mark.parametrize("name", ["cfg3", "two_circles"])
def test_converged_plans_keep_their_own_geometry(orc, name):
    """every associated obstacle at least min_obstacle_dist from the robot's own footprint (oracle distance); the car's defects
    vanish with its own wheelbase and not with the handle's"""
    cfg, _ = rg.variant(name)
    B = 128
    data = configs.generate(3, B)
    rec, _ = _groups(cfg, B)
    s = capi.BatchSolver(cfg, B)
    s.set_robot_geometry(rec)
    r = _step(s, data)
    obs = s.ws_read(capi.F_OBSIDX, B)
    conv = np.nonzero(r["status"] == capi.STATUS_CONVERGED)[0]
    assert len(conv) >= B // 3
    L, tol = orc.lib(), 1e-5
    _, typ, par = data["obstacles"]
    checked, turned, others = 0, 0, 0
    for b in conv:
        own = rg.with_geometry(cfg, rec[b])
        X, U, dt = r["x_seq"][b], r["u_seq"][b], float(r["dt"][b])
        for k in range(1, cfg.n):
            for j in obs[b, :, k]:
                if j < 0:
                    continue
                j = int(j)
                dist = L.orc_footprint_distance(own, orc._dp(np.ascontiguousarray(X[k])), int(typ[b, j]),
                                                orc._dp(np.ascontiguousarray(par[b, j])), None, None)
                assert dist >= cfg.min_obstacle_dist - tol, f"robot {b} stage {k} obstacle {j}: {dist}"
                checked += 1
        if b % 4:   # a wheelbase other than the handle's
            e_own, e_cfg, worst_cfg = np.zeros(3), np.zeros(3), 0.0
            for k in range(cfg.n - 1):
                for c_, e in ((own, e_own), (cfg, e_cfg)):
                    L.orc_defect(c_, orc._dp(np.ascontiguousarray(X[k])), orc._dp(np.ascontiguousarray(U[k])),
                                 orc._dp(np.ascontiguousarray(X[k + 1])), dt, orc._dp(e))
                assert np.abs(e_own).max() < 1e-5, f"robot {b} stage {k}: {e_own}"
                worst_cfg = max(worst_cfg, np.abs(e_cfg).max())
            others += 1
            turned += worst_cfg > 1e-4   # (a plan that never steers fits every wheelbase)
    assert checked > 0 and turned >= others // 2, (checked, turned, others)
    s.close()


def test_oracle_parity_per_robot(orc):
    """each group against the oracle run with that group's configuration, at the thresholds of test_gpu_parity (minimum time)"""
    cfg = configs.cfg3(tol=1e-8)
    B = 24
    data = configs.generate(3, B)
    rec, groups = _groups(cfg, B)
    s = capi.BatchSolver(cfg, B)
    s.set_robot_geometry(rec)
    out = _step(s, data)
    ref = {k: np.empty_like(v) for k, v in out.items() if k in OUT}
    for idx in groups:
        rr = orc.step_batch(rg.with_geometry(cfg, rec[idx[0]]), _rows(data, idx), n_threads=4)
        for k in ref:
            ref[k][idx] = rr[k]
    agree = (out["status"] == ref["status"]).sum()
    both = (out["status"] == 0) & (ref["status"] == 0)
    assert agree >= B - 1, f"gpu {out['status']} oracle {ref['status']}"
    assert both.sum() >= max((ref["status"] == 0).sum(), 1) - 1
    assert np.abs(out["dt"][both] - ref["dt"][both]).max() < 1e-6
    du = np.abs(out["u_seq"][both] - ref["u_seq"][both]).max(axis=(1, 2))
    assert (du < 1e-4).mean() >= 0.8, f"du {du}"
    s.close()


def test_async_setter_and_graph_replay():
    torch = pytest.importorskip("torch")
    cfg, B = configs.cfg3(), 64
    data = configs.generate(3, B)
    r1, r2 = rg.random_records(cfg, B, 1), rg.random_records(cfg, B, 2)
    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a), device="cuda:0")   # noqa: E731
    host = lambda res: {k: v.cpu().numpy() for k, v in res.items()}            # noqa: E731
    blocking = capi.BatchSolver(cfg, B)
    blocking.set_robot_geometry(r1)
    want1 = _step(blocking, data)
    blocking.set_robot_geometry(r2)
    want2 = _step(blocking, _moved(data, 0.05))
    st = torch.cuda.Stream()
    ob = tuple(dev(a) for a in data["obstacles"])
    with torch.cuda.stream(st):
        s = capi.BatchSolver(cfg, B)
        s.set_stream(st.cuda_stream)
        geo = dev(r1)
        x0, xf, up = dev(data["x0"]), dev(data["xf"]), dev(data["u_prev"])
        s.set_robot_geometry_async(geo)
        res = s.step_async(x0, xf, up, data["u_prev_dt"], ob)
        torch.cuda.synchronize()
        _same(host(res), want1, "async setter + async step")
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            s.set_robot_geometry_async(geo)
            out = s.step_async(x0, xf, up, data["u_prev_dt"], ob)
        geo.copy_(dev(r2))
        x0.copy_(dev(_moved(data, 0.05)["x0"]))
        g.replay()
        torch.cuda.synchronize()
        _same(host(out), want2, "graph replay with rewritten geometry")
        del g
        bad = r2.copy()
        bad[5, capi.GEO_WHEELBASE] = 0.0   # a wheelbase not > 0: only robot 5 is INVALID_INPUT
        bad[9, rg.NP] = 2.5                # n_poly not integral: only robot 9
        fresh = capi.BatchSolver(cfg, B)
        fresh.set_stream(st.cuda_stream)
        fresh.set_robot_geometry_async(dev(bad))
        got = host(fresh.step_async(x0, xf, up, data["u_prev_dt"], ob))
        torch.cuda.synchronize()
        assert got["status"][5] == got["status"][9] == capi.STATUS_INVALID_INPUT
        ref = capi.BatchSolver(cfg, B)
        ref.set_robot_geometry(r2)
        want = _step(ref, _moved(data, 0.05))
        keep = (np.arange(B) != 5) & (np.arange(B) != 9)
        _same(got, want, "the robots with valid records", rows=keep)
        fresh.close(); ref.close(); s.close()
    blocking.close()


def test_validation_and_refused_calls_leave_the_state_alone():
    cfg, B = configs.cfg3(), 16
    data = configs.generate(3, B)
    good = rg.random_records(cfg, B, 3)
    s, twin = capi.BatchSolver(cfg, 3 * B), capi.BatchSolver(cfg, 3 * B)
    for h in (s, twin):
        h.set_robot_geometry(good)
        _step(h, data)

    def refused(code, call):
        with pytest.raises(capi.SolverError, match=rf"\({code}\)"):
            call()

    def bad(i, w, v):
        r = good.copy(); r[i, w] = v
        return r
    for r in (bad(3, capi.GEO_WHEELBASE, np.nan), bad(3, capi.GEO_WHEELBASE, 0.0), bad(2, capi.GEO_WHEELBASE, -np.inf),
              bad(1, rg.NP, 0.0), bad(1, rg.NP, 17.0), bad(1, rg.NP, 3.5), bad(0, rg.XY, np.inf)):
        refused(-1, lambda: s.set_robot_geometry(r))
    refused(-1, lambda: s.set_robot_geometry(np.tile(good[0], (3 * B + 1, 1))))
    assert s.lib.mpcb200_set_robot_geometry(s.h, -1, None) == capi.E_INVALID
    big = configs.generate(3, B + 1)
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
    uni = capi.BatchSolver(configs.cfg2(), B)   # a unicycle with a point footprint: nothing to vary
    rec = np.ones((B, rg.W)); rec[:, rg.NP] = 3
    refused(-1, lambda: uni.set_robot_geometry(rec))
    assert uni.lib.mpcb200_set_robot_geometry_async(uni.h, B, 16) == capi.E_INVALID   # refused before the pointer is looked at
    uni.set_robot_geometry(None)
    uni.close()


def test_kernel_key_with_records():
    cfg, B = configs.cfg3(n=40), 8
    a = capi.BatchSolver(cfg, B)
    a.set_robot_geometry(rg.random_records(cfg, B, 9))
    _step(a, configs.generate(3, B))
    assert (a.kernel_model(), a.kernel_problem()) == (capi.MODEL_GENERIC, capi.PROBLEM_GENERIC)
    a.close()


def test_cpp_mirror_footprint_grows_from_the_second_step():
    """tests/robot_geometry/controller_footprint.cpp: a circular footprint of radius 0.1 that grows to 0.35 from the second step
    on (Controller::setRobotGeometry); every step converges, the later plans keep min_obstacle_dist from the larger circle, and
    the warm-started later steps take fewer iterations than a cold solve of the same step"""
    from tests.conftest import ROOT
    here = os.path.join(ROOT, "tests", "robot_geometry")
    out = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"controller_footprint_{os.getpid()}")
    lib = os.path.join(ROOT, "mpc_local_planner_b200")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", out, os.path.join(here, "controller_footprint.cpp"), f"-L{lib}",
                           "-lmpcb200", f"-Wl,-rpath,{lib}", "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"])
    p = subprocess.run([out], capture_output=True, text=True, timeout=300)
    os.unlink(out)
    assert p.returncode == 0, p.stdout + p.stderr
    rows = re.findall(r"step (\d+) radius (\S+) status (\d+) iters (\d+) clearance (\S+) cold_iters (\d+)", p.stdout)
    assert len(rows) == 4 and all(r[2] == "0" for r in rows), p.stdout
    assert float(rows[0][1]) == 0.1 and all(float(r[1]) == 0.35 for r in rows[1:])
    for r in rows:
        assert float(r[4]) >= 0.5 - 1e-5, r   # min_obstacle_dist from the circle of that step
    for r in rows[2:]:
        assert int(r[3]) < int(r[5]), r
