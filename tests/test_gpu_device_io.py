"""The device-memory entry points (mpcb200_step_batch_async, _step_batch_costmap_async, _check_feasible_async) through
BatchSolver.step_async / step_from_costmaps_async / check_feasible_async on torch CUDA tensors: the same results as the blocking
calls bit for bit, shared batch state, CUDA graph capture, the line-obstacle guard and the pointer checks."""
import ctypes as C

import numpy as np
import pytest

import costmap_cases as cm
from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
KEYS = ("u_seq", "x_seq", "dt", "status", "kkt_err", "iters")


def _dev(a):
    return None if a is None else torch.as_tensor(np.ascontiguousarray(a), device="cuda:0")


def _host(res):
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in res.items()}


def _same_bits(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.dtype == b.dtype and a.shape == b.shape, (what, a.dtype, b.dtype, a.shape, b.shape)
    if a.tobytes() != b.tobytes():
        bad = np.argwhere(a.view(np.uint8).reshape(a.shape[0], -1) != b.view(np.uint8).reshape(b.shape[0], -1))[:, 0]
        raise AssertionError(f"{what}: not bit-identical, instances {np.unique(bad)[:10]}")


def _same_results(got, want, what, keys=KEYS, rows=slice(None)):
    for k in keys:
        _same_bits(got[k][rows], want[k][rows], f"{what} {k}")


def _async_solver(cfg, B, stream):
    s = capi.BatchSolver(cfg, B, device=0)
    s.set_stream(stream.cuda_stream)
    return s


def _dev_obstacles(obst):
    return None if obst is None else tuple(_dev(a) for a in obst)


def _step_async(s, x0, xf, u_prev, u_prev_dt, obst, vp, **kw):
    return s.step_async(_dev(x0), _dev(xf), _dev(u_prev), u_prev_dt, _dev_obstacles(obst), _dev_obstacles(vp), **kw)


def _long_list_case(B):
    M = 250
    cost, origin, res, pose, goal = cm.costmap_scene(B, 0.006, 11)
    s = capi.BatchSolver(configs.cfg2(), B, device=0)
    (count, typ, par), _ = s.costmap_obstacles(cost, origin, res, pose, 0.3, M)
    s.close()
    assert count.max() >= 100 and count.max() <= M
    return dict(x0=pose, xf=goal, u_prev=np.zeros((B, 2)), u_prev_dt=0.2, obstacles=(count, typ, par), viapoints=None)


def _case(name, B):
    if name == "cfg2":
        return configs.cfg2(), configs.generate(2, B), False
    if name == "cfg3":
        return configs.cfg3(), configs.generate(3, B), False
    if name == "cfg4":
        return configs.cfg4(), configs.generate(4, B), False
    if name == "lines":
        return configs.cfg2(), configs.with_line_obstacles(configs.generate(2, B)), True
    if name == "long_lists":
        return configs.cfg2(), _long_list_case(B), False
    raise ValueError(name)


def _next_inputs(d, out):
    """the next cycle of a receding horizon: the robots moved one stage along their plans"""
    return dict(d, x0=out["x_seq"][:, 1].copy(), u_prev=out["u_seq"][:, 0].copy())


@pytest.mark.parametrize("name", ["cfg2", "cfg3", "cfg4", "lines", "long_lists"])
def test_step_async_equals_step(cuda_lib, name):
    """cold, warm, warm: step_async on tensors equals step on the same numpy arrays, all six results bit for bit"""
    B = 48
    cfg, d, lines = _case(name, B)
    st = torch.cuda.Stream()
    blocking = capi.BatchSolver(cfg, B, device=0)
    with torch.cuda.stream(st):
        s = _async_solver(cfg, B, st)
        for cycle in range(3):
            want = blocking.step(d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], d["viapoints"])
            got = _host(_step_async(s, d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], d["viapoints"], line_obstacles=lines))
            _same_results(got, want, f"{name} cycle {cycle}")
            assert s.kernel_model() == blocking.kernel_model() and s.kernel_problem() == blocking.kernel_problem()
            d = _next_inputs(d, want)
        assert (want["status"] == 0).sum() >= B // 2
        if name == "cfg2":
            assert s.kernel_problem() == capi.PROBLEM_FIXED_DT_QF
        s.close()
    blocking.close()


def test_mixed_sequence_shares_the_batch_state(cuda_lib):
    """blocking cold, async warm, blocking warm on one handle equals the all-blocking sequence (B above the SM count: the
    queue is ordered by the previous solve's iteration counts); the async step moves no bytes through the host, and the counters
    of launches with different grids fold into the same statistics as the blocking calls"""
    B = 200
    cfg, d0, _ = _case("cfg2", B)
    st = torch.cuda.Stream()
    ref = capi.BatchSolver(cfg, B, device=0)
    seq, d = [], d0
    for _ in range(3):
        seq.append(ref.step(d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], None))
        d = _next_inputs(d, seq[-1])
    with torch.cuda.stream(st):
        s = _async_solver(cfg, B, st)
        d = d0
        out = s.step(d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], None)
        _same_results(out, seq[0], "blocking cold")
        d = _next_inputs(d, out)
        before = s.stats()
        out = _host(_step_async(s, d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], None))
        after = s.stats()
        assert (after["h2d_bytes"], after["d2h_bytes"]) == (before["h2d_bytes"], before["d2h_bytes"])
        assert after["launches_total"] > before["launches_total"]
        _same_results(out, seq[1], "async warm")
        d = _next_inputs(d, out)
        out = s.step(d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], None)
        _same_results(out, seq[2], "blocking warm")
        s.close()
    ref.close()
    # statistics: async launches of two grids (B = 40 and B = 200) accumulate before one read.  The iteration counts of the KKT
    # phase are the blocking sequence's, and the per-CTA phase means agree with the blocking ones (each launch averaged over its
    # own grid: averaging both over the last grid would shrink the B = 40 launch's share five times)
    ref = capi.BatchSolver(cfg, B, device=0)
    with torch.cuda.stream(st):
        s = _async_solver(cfg, B, st)
        for sub in (40, B):
            dd = {k: (v[:sub] if isinstance(v, np.ndarray) else v) for k, v in d0.items() if k not in ("obstacles", "viapoints")}
            ob = tuple(a[:sub] for a in d0["obstacles"])
            ref.step(dd["x0"], dd["xf"], dd["u_prev"], dd["u_prev_dt"], ob, None)
            ref.reset()
            _step_async(s, dd["x0"], dd["xf"], dd["u_prev"], dd["u_prev_dt"], ob, None)
            s.reset()
        sa, sb = s.stats(), ref.stats()
        assert (sa["kkt_instances"], sa["kkt_sweeps"]) == (sb["kkt_instances"], sb["kkt_sweeps"])
        for p in (capi.PHASE_EVAL, capi.PHASE_KKT, capi.PHASE_LINESEARCH):
            assert sb["ms"][p] > 0 and 0.75 < sa["ms"][p] / sb["ms"][p] < 1.33, (p, sa["ms"], sb["ms"])
        s.close()
    ref.close()


def _scene(B, W, H, seed):
    rng = np.random.default_rng(seed)
    res = 0.05
    cost = np.stack([cm.random_costmap(rng, W, H, 0.006) for _ in range(B)])
    origin = rng.uniform(-3, 3, (B, 2))
    pose = np.concatenate([origin + rng.uniform(2.5, 4.0, (B, 2)), rng.uniform(-np.pi, np.pi, (B, 1))], axis=1)
    goal = pose.copy(); goal[:, 0] += 3.0 * np.cos(pose[:, 2]); goal[:, 1] += 3.0 * np.sin(pose[:, 2])
    yy, xx = np.mgrid[0:H, 0:W]
    for b in range(B):
        cx, cy = origin[b, 0] + (xx + 0.5) * res, origin[b, 1] + (yy + 0.5) * res
        for p in (pose[b], goal[b]):
            cost[b][(cx - p[0]) ** 2 + (cy - p[1]) ** 2 < 0.7 ** 2] = 0
    return cost, origin, res, pose, goal


def _offset_map(cost, offset):
    """the maps inside a larger tensor, `offset` bytes past its (aligned) start"""
    flat = torch.as_tensor(cost.reshape(-1), device="cuda:0")
    big = torch.zeros(flat.numel() + 16, dtype=torch.uint8, device="cuda:0")
    big[offset:offset + flat.numel()].copy_(flat)
    t = big[offset:offset + flat.numel()].view(cost.shape)
    assert t.is_contiguous() and t.data_ptr() % 16 == offset % 16
    return t


@pytest.mark.parametrize("W,offset", [(208, 0), (204, 0), (201, 0), (208, 1), (208, 4)])
def test_costmap_chain_async_equals_blocking(cuda_lib, W, offset):
    """step_from_costmaps_async on device maps (read in place: 16-byte, 4-byte and byte loads by width and alignment) equals
    step_from_costmaps, obst_found included, cold and warm"""
    B, H, M = 24, 160, 512
    cfg = configs.cfg2()
    cost, origin, res, pose, goal = _scene(B, W, H, 7 + W)
    st = torch.cuda.Stream()
    blocking = capi.BatchSolver(cfg, B, device=0)
    with torch.cuda.stream(st):
        s = _async_solver(cfg, B, st)
        dcost, dorg = _offset_map(cost, offset), _dev(origin)
        x0, up = pose, np.zeros((B, 2))
        for cycle in range(2):
            want = blocking.step_from_costmaps(x0, goal, cost, origin, res, 0.3, M, u_prev=up, u_prev_dt=0.2)
            got = _host(s.step_from_costmaps_async(_dev(x0), _dev(goal), dcost, dorg, res, 0.3, M, u_prev=_dev(up), u_prev_dt=0.2))
            _same_results(got, want, f"W={W} offset={offset} cycle {cycle}", KEYS + ("obst_found",))
            x0, up = want["x_seq"][:, 1].copy(), want["u_seq"][:, 0].copy()
        assert want["obst_found"].max() > 64 and (want["status"] == 0).sum() >= B // 2
        s.close()
    blocking.close()


@pytest.mark.parametrize("footprint", ["polygon", "two_points"])
def test_check_feasible_async_equals_blocking(cuda_lib, footprint):
    rng = np.random.default_rng(5)
    fp = np.array(configs.CARLIKE_POLYGON) if footprint == "polygon" else np.array([[0.1, 0.0], [-0.1, 0.0]])
    B = 96
    cases = cm.feasibility_cases(rng, B)
    cost = np.stack([c[0] for c in cases]); origin = np.stack([c[1] for c in cases]); xs = np.stack([c[2] for c in cases])
    cfg = configs.cfg2()
    st = torch.cuda.Stream()
    blocking = capi.BatchSolver(cfg, B, device=0)
    with torch.cuda.stream(st):
        s = _async_solver(cfg, B, st)
        for look in (-1, 5):
            want = blocking.check_feasible(cost, origin, 0.05, fp, 0.18, 0.3, look, x_seq=xs)
            got = _host(s.check_feasible_async(_dev(cost), _dev(origin), 0.05, _dev(fp), 0.18, 0.3, look, x_seq=_dev(xs)))["feasible"]
            np.testing.assert_array_equal(got.astype(bool), want)
            assert want.any() and not want.all()
        # the trajectories of the last solve (an async solve here, a blocking one on the other handle), read on the device
        d = configs.generate(2, B)
        out = blocking.step(d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], None)
        _step_async(s, d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], None)
        H, Wm, res = 200, 200, 0.05
        maps = np.zeros((B, H, Wm), dtype=np.uint8)
        org = np.tile(np.array([-2.0, -5.0]), (B, 1))
        cnt, _, par = d["obstacles"]
        for b in range(B):
            for j in range(cnt[b]):
                mx, my = int((par[b, j, 0] - org[b, 0]) / res), int((par[b, j, 1] - org[b, 1]) / res)
                if 0 <= mx < Wm and 0 <= my < H:
                    maps[b, my, mx] = 254
        want = blocking.check_feasible(maps, org, res, fp, 0.18, 0.3, -1)
        got = _host(s.check_feasible_async(_dev(maps), _dev(org), res, _dev(fp), 0.18, 0.3, -1))["feasible"]
        np.testing.assert_array_equal(got.astype(bool), want)
        assert want.any() and (out["status"] == 0).sum() >= B // 2
        s.close()
    blocking.close()


def _moved(d, k):
    """inputs of cycle k: every robot a little further along"""
    x0 = d["x0"].copy()
    x0[:, 0] += 0.02 * k; x0[:, 2] += 0.01 * k
    return x0


def test_cuda_graph_replay_equals_eager(cuda_lib):
    """warm-up, capture step_async in torch.cuda.graph on the handle's stream, replay twice with new inputs written into the
    static tensors: the results equal an eager async sequence bit for bit"""
    B = 200
    cfg, d, _ = _case("cfg2", B)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        eager = _async_solver(cfg, B, st)
        want = [_host(_step_async(eager, _moved(d, k), d["xf"], d["u_prev"], 0.2, d["obstacles"], None)) for k in range(3)]
        eager.close()
        s = _async_solver(cfg, B, st)
        x0, xf, up, ob = _dev(_moved(d, 0)), _dev(d["xf"]), _dev(d["u_prev"]), _dev_obstacles(d["obstacles"])
        _same_results(_host(s.step_async(x0, xf, up, 0.2, ob)), want[0], "warm-up")
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        res = s.step_async(x0, xf, up, 0.2, ob)
    with torch.cuda.stream(st):
        for k in (1, 2):
            x0.copy_(torch.as_tensor(_moved(d, k), device="cuda:0"))
            g.replay()
            _same_results(_host(res), want[k], f"replay {k}")
    torch.cuda.synchronize()
    del g
    s.close()


def test_cuda_graph_replay_of_the_costmap_chain(cuda_lib):
    B, W, H, M = 24, 208, 160, 512
    cfg = configs.cfg2()
    cost, origin, res, pose, goal = _scene(B, W, H, 3)
    st = torch.cuda.Stream()

    def maps_of(k):
        c = cost.copy()
        c[:, :, 10 + 5 * k] = 254 * (k % 2)   # a wall that comes and goes
        return c
    with torch.cuda.stream(st):
        eager = _async_solver(cfg, B, st)
        want = [_host(eager.step_from_costmaps_async(_dev(pose), _dev(goal), _dev(maps_of(k)), _dev(origin), res, 0.3, M)) for k in range(3)]
        eager.close()
        s = _async_solver(cfg, B, st)
        dcost, x0, xf, org = _dev(maps_of(0)), _dev(pose), _dev(goal), _dev(origin)
        _same_results(_host(s.step_from_costmaps_async(x0, xf, dcost, org, res, 0.3, M)), want[0], "warm-up", KEYS + ("obst_found",))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        out = s.step_from_costmaps_async(x0, xf, dcost, org, res, 0.3, M)
    with torch.cuda.stream(st):
        for k in (1, 2):
            dcost.copy_(torch.as_tensor(maps_of(k), device="cuda:0"))
            g.replay()
            _same_results(_host(out), want[k], f"replay {k}", KEYS + ("obst_found",))
    torch.cuda.synchronize()
    del g
    s.close()


@pytest.mark.filterwarnings("ignore:The CUDA Graph is empty")   # the failed call captured nothing, by design
def test_capture_that_needs_growth_fails_cleanly(cuda_lib):
    """a capture whose call would grow the staging arrays (a longer obstacle list than the warm-up's) returns E_INVALID and the
    capture ends cleanly; outside the capture the same call grows the arrays and solves"""
    B = 16
    cfg, d, _ = _case("cfg2", B)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        s = _async_solver(cfg, B, st)
        x0, xf = _dev(d["x0"]), _dev(d["xf"])
        _host(s.step_async(x0, xf, None, 0.2, _dev_obstacles(d["obstacles"])))
        cnt, typ, par = d["obstacles"]
        M = 100
        typ2 = np.zeros((B, M), dtype=np.int32); typ2[:, :typ.shape[1]] = typ
        par2 = np.zeros((B, M, capi.OBST_STRIDE)); par2[:, :par.shape[1]] = par
        ob2 = (_dev(cnt), _dev(typ2), _dev(par2))
    g = torch.cuda.CUDAGraph()
    with pytest.raises(capi.SolverError, match=r"\(-1\).*warm-up"):
        with torch.cuda.graph(g, stream=st):
            s.step_async(x0, xf, None, 0.2, ob2)
    assert not torch.cuda.is_current_stream_capturing()
    with torch.cuda.stream(st):
        s.reset()
        got = _host(s.step_async(x0, xf, None, 0.2, ob2))
        ref = capi.BatchSolver(cfg, B, device=0)
        want = ref.step(d["x0"], d["xf"], None, 0.2, (cnt, typ2, par2), None)
        _same_results(got, want, "after the failed capture")
        ref.close()
        s.close()


def test_undeclared_line_obstacle_is_invalid_input(cuda_lib):
    """a line obstacle on a launch without the line paths: INVALID_INPUT for its instance only, the others bit-identical to the
    batch without it"""
    B, bad = 32, 5
    cfg, d, _ = _case("cfg2", B)
    cnt, typ, par = (a.copy() for a in d["obstacles"])
    typ2, par2 = typ.copy(), par.copy()
    typ2[bad, 1] = capi.OBST_LINE
    par2[bad, 1, 2:4] = par2[bad, 1, 0:2] + 0.3
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        s = _async_solver(cfg, B, st)
        got = _host(_step_async(s, d["x0"], d["xf"], d["u_prev"], 0.2, (cnt, typ2, par2), None))
        assert s.kernel_problem() == capi.PROBLEM_FIXED_DT_QF
        s.close()
        s = _async_solver(cfg, B, st)
        want = _host(_step_async(s, d["x0"], d["xf"], d["u_prev"], 0.2, (cnt, typ, par), None))
        s.close()
    assert got["status"][bad] == capi.STATUS_INVALID_INPUT and (want["status"] != capi.STATUS_INVALID_INPUT).all()
    others = np.arange(B) != bad
    _same_results(got, want, "other instances", rows=others)


def test_host_pointers_are_rejected(cuda_lib):
    """a host (numpy) map behind the device-memory entry points: E_INVALID, nothing launched"""
    B = 4
    cfg, d, _ = _case("cfg2", B)
    cost, origin, res, pose, goal = _scene(B, 64, 48, 1)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        s = _async_solver(cfg, B, st)
        org, x0, xf = _dev(origin), _dev(pose), _dev(goal)
        m = capi.Costmaps(64, 48, res, C.cast(C.c_void_p(org.data_ptr()), C.POINTER(C.c_double)), cost.ctypes.data_as(C.POINTER(C.c_ubyte)))
        outs = s._async_outputs(torch, B, None, KEYS + ("obst_found", "feasible"))
        n0 = s.stats()["launches_total"]
        rc = s.lib.mpcb200_step_batch_costmap_async(s.h, B, x0.data_ptr(), xf.data_ptr(), None, 0.2, C.byref(m), 0.3, 64, None, None, None,
                                                    *(outs[k].data_ptr() for k in KEYS + ("obst_found",)))
        assert rc == capi.E_INVALID and b"device memory" in s.lib.mpcb200_last_error(s.h)
        fp = _dev(np.array(configs.CARLIKE_POLYGON))
        rc = s.lib.mpcb200_check_feasible_async(s.h, B, C.byref(m), None, 0, fp.data_ptr(), fp.shape[0], 0.18, 0.0, 0.3, -1,
                                                outs["feasible"].data_ptr())
        assert rc == capi.E_INVALID
        rc = s.lib.mpcb200_step_batch_async(s.h, B, d["x0"].ctypes.data, xf.data_ptr(), None, 0.2, None, None, None, None, 0,
                                            *(outs[k].data_ptr() for k in KEYS))
        assert rc == capi.E_INVALID
        assert s.stats()["launches_total"] == n0
        with pytest.raises(ValueError):
            s.step_async(d["x0"], xf)
        s.close()


def test_async_needs_the_current_stream_and_the_fused_mode(cuda_lib):
    B = 4
    cfg, d, _ = _case("cfg2", B)
    s = capi.BatchSolver(cfg, B, device=0)
    x0, xf = _dev(d["x0"]), _dev(d["xf"])
    with pytest.raises(capi.SolverError, match="current_stream"):
        s.step_async(x0, xf)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        s.set_stream(st.cuda_stream)
        s.set_option(capi.OPT_SOLVE_MODE, capi.SOLVE_PHASED)
        with pytest.raises(capi.SolverError, match=r"\(-2\)"):
            s.step_async(x0, xf)
    s.close()
