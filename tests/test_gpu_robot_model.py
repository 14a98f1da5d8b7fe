"""Per-robot model (mpcb200_set_robot_model) on the GPU: records equal to the handle's types change nothing, a mixed batch of
unicycles, car-likes and bicycles of four footprint types is bit for bit one handle per model group (cold and warm, in every
per-robot-model kernel, on a car handle and on a unicycle / point handle), all four record kinds combine on the costmap chain and
the device-memory path, a model change warm-starts, converged plans keep their own footprint and dynamics, parity with the oracle,
the validation, the kernel key and the C++ mirror."""
import os
import re
import subprocess

import numpy as np
import pytest

import costmap_cases as cm
import robot_geometry_cases as rg
import robot_model_cases as rm
import robot_weights_cases as rw
from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu
OUT = ("u_seq", "x_seq", "dt", "status", "kkt_err", "iters")
WARM = (capi.F_X, capi.F_U, capi.F_NU, capi.F_S, capi.F_LAM, capi.F_OBSIDX, capi.F_SCAL)
GENERIC = (capi.MODEL_GENERIC, capi.PROBLEM_GENERIC)


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


def _key(s):
    return (s.kernel_model(), s.kernel_problem())


def _generic(cfg, B, opts=()):
    """a handle that always runs the generic key (the key every solve with model records runs)"""
    h = capi.BatchSolver(cfg, B)
    h.set_option(capi.OPT_FORCE_GENERIC_MODEL, 1)
    for o, v in opts:
        h.set_option(o, v)
    return h


@pytest.mark.parametrize("name", ["cfg3", "circular", "two_circles", "line", "bicycle"])
def test_records_equal_to_the_handle_types_change_nothing(name):
    cfg, _ = rg.variant(name)
    B = 48
    data = configs.generate(3, B)
    a, b = capi.BatchSolver(cfg, B), capi.BatchSolver(cfg, B)
    a.set_robot_model(np.tile(rm.record_of(cfg), (B, 1)))
    for t in range(3):
        d = _moved(data, 0.05 * t)
        _same(_step(a, d), _step(b, d), f"{name} call {t}")
        assert _key(a) == _key(b) == GENERIC
    ws = {f: (a.ws_read(f, B), b.ws_read(f, B)) for f in WARM}
    for f, (x, y) in ws.items():
        assert x.tobytes() == y.tobytes(), f"{name} warm field {f}"
    a.set_robot_model(None)
    d = _moved(data, 0.15)
    _same(_step(a, d), _step(b, d), f"{name} after clearing")
    a.close(); b.close()


def test_records_equal_to_the_uni_point_types_run_the_generic_key():
    """cfg 2 (the unicycle / point, fixed-dt quadratic-form key) with records of its own types is the same handle forced to the
    generic key; clearing the records brings the handle's own key back"""
    cfg, B = configs.cfg2(), 64
    data = configs.generate(2, B)
    a, b = capi.BatchSolver(cfg, B), _generic(cfg, B)
    a.set_robot_model(np.tile(rm.record_of(cfg), (B, 1)))
    for t in range(2):
        d = _moved(data, 0.05 * t)
        _same(_step(a, d), _step(b, d), f"call {t}")
        assert _key(a) == GENERIC
    for f in WARM:
        assert a.ws_read(f, B).tobytes() == b.ws_read(f, B).tobytes(), f"warm field {f}"
    a.set_robot_model(None)
    b.set_option(capi.OPT_FORCE_GENERIC_MODEL, 0)
    d = _moved(data, 0.1)
    _same(_step(a, d), _step(b, d), "after clearing")
    assert _key(a) == _key(b) == (capi.MODEL_UNI_POINT, capi.PROBLEM_FIXED_DT_QF)
    a.close(); b.close()


def _shape_host(ext, small):
    """cfg 3 in each per-robot-model kernel shape: free dt (EXT, minimum time) or fixed dt (quadratic form), N = 40 (small CTA)
    or 80"""
    c = configs.cfg3(n=40 if small else 80)
    if not ext:
        q = configs.cfg2()
        c.objective, c.variable_dt, c.xf_fixed[:] = capi.OBJ_QUADRATIC_FORM, 0, [0, 0, 0]
        c.Q[:], c.R[:], c.terminal_cost, c.Qf[:], c.dt_ref = list(q.Q), list(q.R), q.terminal_cost, list(q.Qf), q.dt_ref
    return c


def _mixed_vs_groups(host, data, B, K, opts=(), weights=None):
    """the mixed handle (model, limits and geometry records; weights records too when given) against one generic-key handle per
    group, created with the group's configuration: a cold call, then a warm one, outputs, winners and warm fields"""
    model, limits, geometry = rm.fleet_records(host, B)
    groups = [np.arange(g, B, 4) for g in range(4)]
    s = capi.BatchSolver(host, B * K)
    for o, v in opts:
        s.set_option(o, v)
    _set_fleet(s, host, model, limits, geometry)
    if weights is not None:
        s.set_robot_weights(weights)
    hs = []
    for g, idx in enumerate(groups):
        c = rm.group_config(host, rm.GROUPS[g])
        if weights is not None:
            c = rw.with_weights(c, weights[idx[0]])
        hs.append(_generic(c, len(idx) * K, opts))
    for t in range(2):
        d = _moved(data, 0.05 * t)
        r = _step(s, d, K)
        assert _key(s) == GENERIC
        wm = {f: s.ws_read(f, B) for f in WARM}
        for g, idx in enumerate(groups):
            rh = _step(hs[g], _rows(d, idx), K)
            _same(r, rh, f"call {t} group {rm.GROUPS[g]}", rows=idx, rows_b=slice(None))
            if K > 1:
                assert np.array_equal(r["winner"][idx], rh["winner"])
            for f in WARM:
                assert wm[f][idx].tobytes() == hs[g].ws_read(f, len(idx)).tobytes(), f"call {t} group {g} warm field {f}"
    conv = [(r["status"][idx] == capi.STATUS_CONVERGED).mean() for idx in groups]
    for h in hs:
        h.close()
    s.close()
    return conv


def _set_fleet(s, host, model, limits, geometry):
    """the fleet's records in an order every handle accepts: model records of the handle's own types first (valid with any
    geometry record, and they let a unicycle / point handle take geometry records), then the geometry, then the robots' models"""
    s.set_robot_limits(limits)
    s.set_robot_model(np.tile(rm.record_of(host), (len(model), 1)))
    s.set_robot_geometry(geometry)
    s.set_robot_model(model)


@pytest.mark.parametrize("lines", [False, True])
@pytest.mark.parametrize("ext", [False, True])
@pytest.mark.parametrize("small", [False, True])
@pytest.mark.parametrize("K", [1, 3])
def test_mixed_batch_equals_one_handle_per_group(lines, ext, small, K):
    """B well above the CTA count, so each CTA solves robots of several models in turn; the warm call is history-ordered (and
    placed) by default, the cold one is not"""
    host = _shape_host(ext, small)
    B = 1200 if K == 1 else 400
    data = configs.generate(3, B)
    if lines:
        data = configs.with_line_obstacles(data)
    conv = _mixed_vs_groups(host, data, B, K)
    assert min(conv) > 0, conv


@pytest.mark.parametrize("opts", [((capi.OPT_ORDER_BY_HISTORY, 0),), ((capi.OPT_CRITICAL_PLACEMENT, 0),)])
def test_mixed_batch_with_execution_options(opts):
    _mixed_vs_groups(_shape_host(True, False), configs.generate(3, 800), 800, 1, opts)


def test_mixed_batch_on_a_uni_point_handle():
    """the same mix hosted by cfg 2, whose own key is the unicycle / point fixed-dt quadratic form: it refuses geometry records
    until model records are set, and a polygon model until its robots have a geometry record with vertices"""
    host = configs.cfg2()
    s = capi.BatchSolver(host, 8)
    model, limits, geometry = rm.fleet_records(host, 8)
    with pytest.raises(capi.SolverError, match=r"\(-1\)"):
        s.set_robot_geometry(geometry)
    with pytest.raises(capi.SolverError, match=r"\(-1\)"):
        s.set_robot_model(model)   # robot 1 a polygon of the configuration's n_poly = 0
    s.close()
    conv = _mixed_vs_groups(host, configs.generate(2, 1000), 1000, 1)
    assert min(conv) > 0, conv


def test_all_four_record_kinds_on_the_costmap_chain():
    host, B = _shape_host(False, False), 24   # a quadratic form: it reads the weights
    model, limits, geometry = rm.fleet_records(host, B)
    weights = np.stack([rw.record_of(host) * (1.0 + 0.25 * (b % 4)) for b in range(B)])
    groups = [np.arange(g, B, 4) for g in range(4)]
    cost, origin, res, pose, goal = cm.costmap_scene(B, 0.006, 21)
    s = capi.BatchSolver(host, B)
    s.set_robot_limits(limits); s.set_robot_geometry(geometry); s.set_robot_model(model); s.set_robot_weights(weights)
    hs = [_generic(rw.with_weights(rm.group_config(host, rm.GROUPS[g]), weights[idx[0]]), len(idx)) for g, idx in enumerate(groups)]
    x0, up = pose.copy(), np.zeros((B, 2))
    for cycle in range(2):
        got = s.step_from_costmaps(x0, goal, cost, origin, res, 0.3, 256, u_prev=up, u_prev_dt=0.2)
        for g, idx in enumerate(groups):
            want = hs[g].step_from_costmaps(x0[idx], goal[idx], cost[idx], origin[idx], res, 0.3, 256, u_prev=up[idx], u_prev_dt=0.2)
            _same(got, want, f"costmap cycle {cycle} group {g}", rows=idx, rows_b=slice(None))
        x0, up = got["x_seq"][:, 1].copy(), got["u_seq"][:, 0].copy()
    for h in hs:
        h.close()
    s.close()


def test_all_four_record_kinds_on_the_device_path_async_setters_and_graph_replay():
    torch = pytest.importorskip("torch")
    host, B = _shape_host(False, False), 64
    data = configs.generate(3, B)
    model, limits, geometry = rm.fleet_records(host, B)
    weights = np.stack([rw.record_of(host) * (1.0 + 0.25 * (b % 4)) for b in range(B)])
    model2 = model[np.arange(B) ^ 1]   # each pair of robots swaps models (and keeps geometry records valid for both: checked below)
    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a), device="cuda:0")   # noqa: E731
    host_of = lambda res: {k: v.cpu().numpy() for k, v in res.items()}         # noqa: E731
    blocking = capi.BatchSolver(host, B)
    blocking.set_robot_limits(limits); blocking.set_robot_geometry(geometry); blocking.set_robot_weights(weights)
    blocking.set_robot_model(model)
    want1 = _step(blocking, data)
    geometry2 = geometry[np.arange(B) ^ 1]
    limits2 = limits[np.arange(B) ^ 1]
    blocking.set_robot_limits(limits2)
    blocking.set_robot_geometry(geometry2)   # (every group record holds the polygon, so a polygon model accepts any of them)
    blocking.set_robot_model(model2)
    want2 = _step(blocking, _moved(data, 0.05))
    st = torch.cuda.Stream()
    ob = tuple(dev(a) for a in data["obstacles"])
    with torch.cuda.stream(st):
        s = capi.BatchSolver(host, B)
        s.set_stream(st.cuda_stream)
        md, lm, gm, wg = dev(model), dev(limits), dev(geometry), dev(weights)
        x0, xf, up = dev(data["x0"]), dev(data["xf"]), dev(data["u_prev"])
        s.set_robot_limits_async(lm); s.set_robot_geometry_async(gm); s.set_robot_weights_async(wg); s.set_robot_model_async(md)
        res = s.step_async(x0, xf, up, data["u_prev_dt"], ob)
        torch.cuda.synchronize()
        _same(host_of(res), want1, "async setters + async step")
        assert _key(s) == GENERIC
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            s.set_robot_limits_async(lm); s.set_robot_geometry_async(gm); s.set_robot_model_async(md)
            out = s.step_async(x0, xf, up, data["u_prev_dt"], ob)
        md.copy_(dev(model2)); gm.copy_(dev(geometry2)); lm.copy_(dev(limits2))
        x0.copy_(dev(_moved(data, 0.05)["x0"]))
        g.replay()
        torch.cuda.synchronize()
        _same(host_of(out), want2, "graph replay with rewritten models")
        del g
        bad = model.copy()
        bad[5, rm.RT] = 4.0     # robot_type out of range: only robot 5 is INVALID_INPUT
        bad[9, rm.FT] = 1.5     # footprint_type not integral: only robot 9
        badg = geometry.copy()
        badg[13, rg.NP] = 0.0   # robot 13 (car, polygon): a polygon of no vertex is not valid for its model
        fresh = capi.BatchSolver(host, B)
        fresh.set_stream(st.cuda_stream)
        fresh.set_robot_limits_async(dev(limits)); fresh.set_robot_geometry_async(dev(badg)); fresh.set_robot_weights_async(wg)
        fresh.set_robot_model_async(dev(bad))
        got = host_of(fresh.step_async(x0, xf, up, data["u_prev_dt"], ob))
        torch.cuda.synchronize()
        assert got["status"][5] == got["status"][9] == got["status"][13] == capi.STATUS_INVALID_INPUT
        keep = ~np.isin(np.arange(B), [5, 9, 13])
        assert (got["status"][keep] != capi.STATUS_INVALID_INPUT).all()
        ref = capi.BatchSolver(host, B)
        ref.set_robot_limits(limits); ref.set_robot_geometry(geometry); ref.set_robot_weights(weights); ref.set_robot_model(model)
        want = _step(ref, _moved(data, 0.05))
        _same(got, want, "the robots with valid pairs", rows=keep)
        fresh.close(); ref.close(); s.close()
    blocking.close()


def test_a_model_change_warm_starts_under_the_new_model():
    """robots switch from a circular to a polygon footprint between calls (geometry record first, holding the radius and the
    polygon, then the model record): each equals a handle created with the new types whose warm fields are the mixed handle's"""
    host, B = configs.cfg3(), 16
    data = configs.generate(3, B)
    geo = np.tile(rm.group_geometry("uni_circle"), (B, 1))
    s = capi.BatchSolver(host, B)
    s.set_robot_geometry(geo)
    s.set_robot_model(np.tile(rm.record(capi.ROBOT_UNICYCLE, capi.FOOTPRINT_CIRCULAR), (B, 1)))
    _step(s, data)
    new = rm.record(capi.ROBOT_UNICYCLE, capi.FOOTPRINT_POLYGON)
    s.set_robot_model(np.tile(new, (B, 1)))
    c_new = rg.with_geometry(rm.with_model(host, new), geo[0])
    twins = [_generic(c_new, 1) for _ in range(B)]
    for b in range(B):
        _step(twins[b], _rows(data, slice(b, b + 1)))   # (a first call sizes the twin; its warm fields are rewritten below)
    for t in (1, 2):
        state = {f: s.ws_read(f, B) for f in WARM}
        d = _moved(data, 0.05 * t)
        r = _step(s, d)
        for b in range(B):
            for f in WARM:
                twins[b].ws_write(f, state[f][b:b + 1])
            _same(r, _step(twins[b], _rows(d, slice(b, b + 1))), f"call {t + 1} robot {b}", rows=slice(b, b + 1), rows_b=slice(0, 1))
    assert (r["status"] == capi.STATUS_CONVERGED).mean() >= 0.5
    for t_ in twins:
        t_.close()
    s.close()


def test_oracle_parity_and_own_model_per_group(orc):
    """each group against the oracle run with that group's configuration, at the thresholds of test_gpu_parity (minimum time);
    converged plans keep min_obstacle_dist from the robot's own footprint (oracle distance), and the defects of a car-like or a
    bicycle vanish under its own model and not under the handle's"""
    host = configs.cfg3(tol=1e-8)
    B = 32
    data = configs.generate(3, B)
    model, limits, geometry = rm.fleet_records(host, B)
    groups = [np.arange(g, B, 4) for g in range(4)]
    s = capi.BatchSolver(host, B)
    s.set_robot_limits(limits); s.set_robot_geometry(geometry); s.set_robot_model(model)
    out = _step(s, data)
    obs = s.ws_read(capi.F_OBSIDX, B)
    for g, idx in enumerate(groups):
        c = rm.group_config(host, rm.GROUPS[g])
        ref = orc.step_batch(c, _rows(data, idx), n_threads=4)
        st, rs = out["status"][idx], ref["status"]
        both = (st == 0) & (rs == 0)
        assert (st == rs).sum() >= len(idx) - 1, f"group {g}: gpu {st} oracle {rs}"
        assert both.sum() >= max((rs == 0).sum(), 1) - 1
        assert np.abs(out["dt"][idx][both] - ref["dt"][both]).max() < 1e-6
        du = np.abs(out["u_seq"][idx][both] - ref["u_seq"][both]).max(axis=(1, 2))
        assert (du < 1e-4).mean() >= 0.8, f"group {g} du {du}"
    L, tol = orc.lib(), 1e-5
    _, typ, par = data["obstacles"]
    checked, others, turned = 0, 0, 0
    for b in np.nonzero(out["status"] == capi.STATUS_CONVERGED)[0]:
        own = rm.group_config(host, rm.GROUPS[b % 4])
        X, U, dt = out["x_seq"][b], out["u_seq"][b], float(out["dt"][b])
        for k in range(1, host.n):
            for j in obs[b, :, k]:
                if j < 0:
                    continue
                j = int(j)
                dist = L.orc_footprint_distance(own, orc._dp(np.ascontiguousarray(X[k])), int(typ[b, j]),
                                                orc._dp(np.ascontiguousarray(par[b, j])), None, None)
                assert dist >= host.min_obstacle_dist - tol, f"robot {b} stage {k} obstacle {j}: {dist}"
                checked += 1
        if b % 4 != 1:   # a model other than the handle's simple car
            e_own, e_cfg, worst = np.zeros(3), np.zeros(3), 0.0
            for k in range(host.n - 1):
                for c_, e in ((own, e_own), (host, e_cfg)):
                    L.orc_defect(c_, orc._dp(np.ascontiguousarray(X[k])), orc._dp(np.ascontiguousarray(U[k])),
                                 orc._dp(np.ascontiguousarray(X[k + 1])), dt, orc._dp(e))
                assert np.abs(e_own).max() < 1e-5, f"robot {b} stage {k}: {e_own}"
                worst = max(worst, np.abs(e_cfg).max())
            others += 1
            turned += worst > 1e-4
    assert checked > 0 and turned >= others // 2, (checked, turned, others)
    s.close()


def test_validation_and_refused_calls_leave_the_state_alone():
    host, B = configs.cfg3(), 16
    data = configs.generate(3, B)
    model, limits, geometry = rm.fleet_records(host, B)
    s, twin = capi.BatchSolver(host, 3 * B), capi.BatchSolver(host, 3 * B)
    for h in (s, twin):
        h.set_robot_limits(limits); h.set_robot_geometry(geometry); h.set_robot_model(model)
        _step(h, data)

    def refused(code, call):
        with pytest.raises(capi.SolverError, match=rf"\({code}\)"):
            call()

    def bad(a, i, w, v):
        r = a.copy(); r[i, w] = v
        return r
    for r in (bad(model, 3, rm.RT, np.nan), bad(model, 3, rm.RT, 4.0), bad(model, 2, rm.FT, -1.0), bad(model, 1, rm.FT, 0.5),
              bad(model, 0, rm.RT, np.inf)):
        refused(-1, lambda: s.set_robot_model(r))
    # the interplay, in both orders: a geometry record the robot's model refuses, a model the robot's geometry record refuses
    refused(-1, lambda: s.set_robot_geometry(bad(geometry, 1, rg.NP, 0.0)))            # robot 1 is a car with a polygon
    refused(-1, lambda: s.set_robot_geometry(bad(geometry, 2, capi.GEO_WHEELBASE, 0.0)))  # robot 2 a front-wheel car
    g0 = geometry.copy(); g0[0, capi.GEO_WHEELBASE] = np.nan   # robot 0 (a unicycle) does not read its wheelbase ...
    s.set_robot_geometry(g0); twin.set_robot_geometry(g0)
    refused(-1, lambda: s.set_robot_model(bad(model, 0, rm.RT, capi.ROBOT_SIMPLE_CAR)))   # ... so it cannot become a car
    g3 = geometry.copy(); g3[3, rg.NP] = 0.0                   # robot 3 (a bicycle with a line) does not read n_poly ...
    s.set_robot_geometry(g3); twin.set_robot_geometry(g3)
    refused(-1, lambda: s.set_robot_model(bad(model, 3, rm.FT, capi.FOOTPRINT_POLYGON)))  # ... so it cannot get a polygon
    refused(-1, lambda: s.set_robot_model(np.tile(model[0], (3 * B + 1, 1))))
    assert s.lib.mpcb200_set_robot_model(s.h, -1, None) == capi.E_INVALID
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
    for f in WARM:
        assert s.ws_read(f, B).tobytes() == twin.ws_read(f, B).tobytes(), f"warm field {f}"
    s.close(); twin.close()
    # clearing: the model records of a geometry record that only their types accept; the geometry records of a model that needs them
    uni = capi.BatchSolver(configs.cfg2(), B)   # a unicycle with a point footprint, n_poly 0
    rec = np.tile(rm.group_geometry("car_polygon"), (B, 1))
    refused(-1, lambda: uni.set_robot_geometry(rec))   # no model records: nothing to vary
    assert uni.lib.mpcb200_set_robot_geometry_async(uni.h, B, 16) == capi.E_INVALID
    refused(-1, lambda: uni.set_robot_model(np.tile(rm.record(capi.ROBOT_UNICYCLE, capi.FOOTPRINT_POLYGON), (B, 1))))   # n_poly 0
    uni.set_robot_model(np.tile(rm.record(capi.ROBOT_UNICYCLE, capi.FOOTPRINT_CIRCULAR), (B, 1)))   # radius 0 of the configuration
    uni.set_robot_geometry(rec)   # accepted now: checked for the robots' types
    uni.set_robot_model(np.tile(rm.record(capi.ROBOT_SIMPLE_CAR, capi.FOOTPRINT_POLYGON), (B, 1)))
    refused(-1, lambda: uni.set_robot_geometry(None))   # the polygon of the configuration has no vertex
    refused(-1, lambda: uni.set_robot_model(None))      # the handle's own types refuse geometry records
    r = _step(uni, configs.generate(2, B))
    assert _key(uni) == GENERIC and (r["status"] == capi.STATUS_CONVERGED).any()
    uni.set_robot_model(np.tile(rm.record(capi.ROBOT_UNICYCLE, capi.FOOTPRINT_CIRCULAR), (B, 1)))
    uni.set_robot_geometry(None)
    uni.set_robot_model(None)
    _step(uni, configs.generate(2, B))
    assert _key(uni) == (capi.MODEL_UNI_POINT, capi.PROBLEM_FIXED_DT_QF)
    uni.close()


def test_cpp_mirror_circular_robot_gets_a_polygon_from_the_second_step():
    """tests/robot_model/controller_model.cpp: a circular robot gets a polygon footprint from the second step on
    (Controller::setRobotGeometry, then setRobotModel); every step converges, the later plans keep min_obstacle_dist from the
    polygon, and the warm-started later steps take fewer iterations than a cold solve of the same step"""
    from tests.conftest import ROOT
    here = os.path.join(ROOT, "tests", "robot_model")
    out = os.path.join(os.environ.get("TMPDIR", "/tmp"), f"controller_model_{os.getpid()}")
    lib = os.path.join(ROOT, "mpc_local_planner_b200")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", out, os.path.join(here, "controller_model.cpp"), f"-L{lib}",
                           "-lmpcb200", f"-Wl,-rpath,{lib}", "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64", "-lcudart"])
    p = subprocess.run([out], capture_output=True, text=True, timeout=300)
    os.unlink(out)
    assert p.returncode == 0, p.stdout + p.stderr
    rows = re.findall(r"step (\d+) footprint (\d+) status (\d+) iters (\d+) clearance (\S+) cold_iters (\d+)", p.stdout)
    assert len(rows) == 4 and all(r[2] == "0" for r in rows), p.stdout
    assert rows[0][1] == "1" and all(r[1] == "4" for r in rows[1:])
    for r in rows:
        assert float(r[4]) >= 0.5 - 1e-5, r   # min_obstacle_dist from the footprint of that step
    for r in rows[2:]:
        assert int(r[3]) < int(r[5]), r
