"""Per-robot limits (mpcb200_set_robot_limits) on the GPU: records equal to the configuration change nothing, robot b of a mixed
batch is bit for bit a one-robot handle created with its values (cold, warm, and after its limits changed), converged plans keep
their own bounds, the costmap chain, the async setter and CUDA graphs, the validation, the kernel key, the execution options and
the C++ mirror."""
import os
import re
import subprocess

import numpy as np
import pytest

import costmap_cases as cm
from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu
OUT = ("u_seq", "x_seq", "dt", "status", "kkt_err", "iters")
WARM = (capi.F_X, capi.F_U, capi.F_NU, capi.F_S, capi.F_LAM, capi.F_OBSIDX, capi.F_SCAL)


def _record(cfg):
    return np.array(list(cfg.u_lb) + list(cfg.u_ub) + list(cfg.du_lb) + list(cfg.du_ub) + [cfg.min_obstacle_dist])


def _records_of_config(cfg, B):
    return np.tile(_record(cfg), (B, 1))


def _random_records(cfg, B, seed):
    """seeded per-robot limits with the configuration's row pattern: every finite bound scaled by U(0.5, 1.5), clearance U(0.1, 0.4)"""
    rng = np.random.default_rng(seed)
    r = _records_of_config(cfg, B)
    finite = np.abs(r[:, :8]) < capi.INF
    r[:, :8] = np.where(finite, r[:, :8] * rng.uniform(0.5, 1.5, (B, 8)), r[:, :8])
    r[:, 8] = rng.uniform(0.1, 0.4, B)
    return r


def _with(cfg, rec):
    """a configuration with a record's values: what a handle of its own for that robot is created with"""
    c = cfg.copy()
    c.u_lb[:] = rec[0:2]; c.u_ub[:] = rec[2:4]; c.du_lb[:] = rec[4:6]; c.du_ub[:] = rec[6:8]
    c.min_obstacle_dist = float(rec[8])
    return c


def _row(d, b):
    cnt, typ, par = d["obstacles"]
    vp = None if d["viapoints"] is None else (d["viapoints"][0][b:b + 1], d["viapoints"][1][b:b + 1])
    return dict(x0=d["x0"][b:b + 1], xf=d["xf"][b:b + 1], u_prev=d["u_prev"][b:b + 1], u_prev_dt=d["u_prev_dt"],
                obstacles=(cnt[b:b + 1], typ[b:b + 1], par[b:b + 1]), viapoints=vp)


def _moved(data, t):
    d = dict(data)
    d["x0"] = data["x0"] + t * (data["xf"] - data["x0"]) * np.array([1.0, 1.0, 0.0])
    return d


def _step(s, d, **kw):
    return s.step(d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], d["viapoints"], **kw)


def _ms(s, d, K):
    return s.step_multistart(d["x0"], d["xf"], K, u_prev=d["u_prev"], u_prev_dt=d["u_prev_dt"], obstacles=d["obstacles"],
                             viapoints=d["viapoints"])


def _same(a, b, what, rows=slice(None), rows_b=None):
    """rows `rows` of a and rows `rows_b` (default: the same) of b, bit for bit"""
    for k in OUT:
        x, y = np.ascontiguousarray(a[k][rows]), np.ascontiguousarray(b[k][rows if rows_b is None else rows_b])
        assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), f"{what}: {k} differs"


def _case(name, B):
    if name == "lines_midpoint":   # the line-obstacle kernels (LINES), chosen by midpoint differences and line obstacles
        cfg = configs.cfg2()
        cfg.collocation = capi.COLLOC_MIDPOINT
        return cfg, configs.with_line_obstacles(configs.generate(2, B))
    if name == "cfg5":
        return configs.cfg5(100), configs.generate(5, B, n=100)
    cid = int(name[3:])
    return configs.config_for(cid), configs.generate(cid, B)


@pytest.mark.parametrize("name", ["cfg2", "cfg3", "cfg4", "cfg5", "lines_midpoint"])
def test_records_equal_to_the_config_change_nothing(name):
    B = 48
    cfg, data = _case(name, B)
    a, b = capi.BatchSolver(cfg, B), capi.BatchSolver(cfg, B)
    a.set_robot_limits(_records_of_config(cfg, B))
    for t in range(3):
        d = _moved(data, 0.05 * t)
        _same(_step(a, d), _step(b, d), f"{name} call {t}")
    assert a.kernel_model() == b.kernel_model() and a.kernel_problem() == b.kernel_problem()
    a.set_robot_limits(None)   # cleared: the handle is one that never had records
    for t in range(3, 5):
        d = _moved(data, 0.05 * t)
        _same(_step(a, d), _step(b, d), f"{name} call {t} after clearing")
    a.close(); b.close()


def test_multistart_with_records_equal_to_the_config():
    cfg, B, K = configs.cfg2(), 32, 3
    data = configs.generate(2, B)
    a, b = capi.BatchSolver(cfg, B * K), capi.BatchSolver(cfg, B * K)
    a.set_robot_limits(_records_of_config(cfg, B))   # one record per robot covers its K candidates
    for t in range(2):
        d = _moved(data, 0.05 * t)
        ra, rb = _ms(a, d, K), _ms(b, d, K)
        _same(ra, rb, f"multistart call {t}")
        assert np.array_equal(ra["winner"], rb["winner"])
    a.close(); b.close()


@pytest.mark.parametrize("cid", [2, 3, 4])
def test_mixed_batch_equals_one_handle_per_robot(cid):
    cfg, B = configs.config_for(cid), 64
    data = configs.generate(cid, B)
    rec = _random_records(cfg, B, 100 + cid)
    s = capi.BatchSolver(cfg, B)
    s.set_robot_limits(rec)
    r = _step(s, data)
    assert (r["status"] == capi.STATUS_CONVERGED).sum() >= B // 2
    for b in range(B):
        one = capi.BatchSolver(_with(cfg, rec[b]), 1)
        _same(r, _step(one, _row(data, b)), f"cfg{cid} robot {b}", rows=slice(b, b + 1), rows_b=slice(0, 1))
        one.close()
    s.close()


@pytest.mark.parametrize("cid", [2, 3])
def test_changed_limits_warm_start_under_the_new_values(cid):
    """three warm calls, the records changed before the second: robot b of calls 2 and 3 equals a one-robot twin created with its
    new values whose warm state was copied from slot b"""
    cfg, B = configs.config_for(cid), 16
    data = configs.generate(cid, B)
    r1, r2 = _random_records(cfg, B, 7), _random_records(cfg, B, 8)
    s = capi.BatchSolver(cfg, B)
    s.set_robot_limits(r1)
    _step(s, data)
    twins = [capi.BatchSolver(_with(cfg, r2[b]), 1) for b in range(B)]
    for b in range(B):
        _step(twins[b], _row(data, b))   # the twin's layout; its warm state is overwritten below
    s.set_robot_limits(r2)
    for t in (1, 2):
        state = {f: s.ws_read(f, B) for f in WARM}
        d = _moved(data, 0.05 * t)
        r = _step(s, d)
        for b in range(B):
            for f in WARM:
                twins[b].ws_write(f, state[f][b:b + 1])
            _same(r, _step(twins[b], _row(d, b)), f"cfg{cid} call {t + 1} robot {b}", rows=slice(b, b + 1), rows_b=slice(0, 1))
    for t_ in twins:
        t_.close()
    s.close()


@pytest.mark.parametrize("cid", [2, 3])
def test_converged_plans_keep_their_own_bounds(cid):
    cfg, B = configs.config_for(cid), 256
    data = configs.generate(cid, B)
    rec = _random_records(cfg, B, 31 + cid)
    s = capi.BatchSolver(cfg, B)
    s.set_robot_limits(rec)
    r = _step(s, data)
    conv = np.nonzero(r["status"] == capi.STATUS_CONVERGED)[0]
    assert len(conv) >= B // 2
    tol = 1e-6
    for b in conv:
        u = r["u_seq"][b, :-1]
        assert (u >= rec[b, 0:2] - tol).all() and (u <= rec[b, 2:4] + tol).all(), f"robot {b}"
        rate = np.diff(u, axis=0) / r["dt"][b]
        assert (rate >= rec[b, 4:6] - tol).all() and (rate <= rec[b, 6:8] + tol).all(), f"robot {b}"
    s.close()


def test_costmap_chain_with_records_equals_extraction_then_step():
    B, M = 24, 512
    cfg = configs.cfg2()
    cost, origin, res, pose, goal = cm.costmap_scene(B, 0.006, 21)
    rec = _random_records(cfg, B, 5)
    chain, ext, step = capi.BatchSolver(cfg, B), capi.BatchSolver(cfg, B), capi.BatchSolver(cfg, B)
    chain.set_robot_limits(rec); step.set_robot_limits(rec)
    x0, up = pose, np.zeros((B, 2))
    for cycle in range(2):
        got = chain.step_from_costmaps(x0, goal, cost, origin, res, 0.3, M, u_prev=up, u_prev_dt=0.2)
        obst, _ = ext.costmap_obstacles(cost, origin, res, x0, 0.3, M)
        want = step.step(x0, goal, up, 0.2, obst)
        _same(got, want, f"cycle {cycle}")
        x0, up = want["x_seq"][:, 1].copy(), want["u_seq"][:, 0].copy()
    for s_ in (chain, ext, step):
        s_.close()


def test_async_setter_and_graph_replay():
    torch = pytest.importorskip("torch")
    cfg, B = configs.cfg2(), 64
    data = configs.generate(2, B)
    r1, r2 = _random_records(cfg, B, 1), _random_records(cfg, B, 2)
    dev = lambda a: torch.as_tensor(np.ascontiguousarray(a), device="cuda:0")   # noqa: E731
    host = lambda res: {k: v.cpu().numpy() for k, v in res.items()}            # noqa: E731
    blocking = capi.BatchSolver(cfg, B)
    blocking.set_robot_limits(r1)
    want1 = _step(blocking, data)
    blocking.set_robot_limits(r2)
    want2 = _step(blocking, _moved(data, 0.05))
    st = torch.cuda.Stream()
    ob = tuple(dev(a) for a in data["obstacles"])
    with torch.cuda.stream(st):
        s = capi.BatchSolver(cfg, B)
        s.set_stream(st.cuda_stream)
        lim = dev(r1)
        x0, xf, up = dev(data["x0"]), dev(data["xf"]), dev(data["u_prev"])
        s.set_robot_limits_async(lim)
        res = s.step_async(x0, xf, up, data["u_prev_dt"], ob)
        torch.cuda.synchronize()
        _same(host(res), want1, "async setter + async step")
        # the captured pair reads the limit tensor at replay
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            s.set_robot_limits_async(lim)
            out = s.step_async(x0, xf, up, data["u_prev_dt"], ob)
        lim.copy_(dev(r2))
        x0.copy_(dev(_moved(data, 0.05)["x0"]))
        g.replay()
        torch.cuda.synchronize()
        _same(host(out), want2, "graph replay with rewritten limits")
        del g
        # an invalid device record: only its robot is INVALID_INPUT
        bad = r2.copy()
        bad[5, 2] = bad[5, 0] - 0.1   # u_ub <= u_lb
        fresh = capi.BatchSolver(cfg, B)
        fresh.set_stream(st.cuda_stream)
        fresh.set_robot_limits_async(dev(bad))
        got = host(fresh.step_async(x0, xf, up, data["u_prev_dt"], ob))
        torch.cuda.synchronize()
        assert got["status"][5] == capi.STATUS_INVALID_INPUT
        ref = capi.BatchSolver(cfg, B)
        ref.set_robot_limits(r2)
        want = _step(ref, _moved(data, 0.05))
        keep = np.arange(B) != 5
        _same(got, want, "the robots with valid records", rows=keep)
        fresh.close(); ref.close(); s.close()
    blocking.close()


def test_validation_and_refused_calls_leave_the_state_alone():
    cfg, B = configs.cfg2(), 16
    data = configs.generate(2, B)
    good = _random_records(cfg, B, 3)
    s, twin = capi.BatchSolver(cfg, 3 * B), capi.BatchSolver(cfg, 3 * B)
    for h in (s, twin):
        h.set_robot_limits(good)
        _step(h, data)

    def refused(code, call):
        with pytest.raises(capi.SolverError, match=rf"\({code}\)"):
            call()

    def bad(i, w, v):
        r = good.copy(); r[i, w] = v
        return r
    for r in (bad(3, 0, np.nan), bad(3, 8, np.nan), bad(2, 2, good[2, 0]), bad(2, 3, good[2, 1] - 1.0), bad(1, 0, -np.inf),
              bad(1, 7, capi.INF), bad(0, 6, np.inf), bad(4, 8, -0.01), bad(4, 8, np.inf)):
        refused(-1, lambda: s.set_robot_limits(r))
    refused(-1, lambda: s.set_robot_limits(np.zeros((3 * B + 1, capi.LIMIT_WORDS)) + good[0]))
    assert s.lib.mpcb200_set_robot_limits(s.h, -1, None) == capi.E_INVALID
    big = configs.generate(2, B + 1)
    refused(-1, lambda: _step(s, big))
    refused(-1, lambda: _ms(s, big, 2))
    refused(-2, lambda: s.solve_stream(data["x0"], data["xf"]))
    s.set_option(capi.OPT_SOLVE_MODE, capi.SOLVE_PHASED)
    refused(-2, lambda: _step(s, data))
    s.set_option(capi.OPT_SOLVE_MODE, capi.SOLVE_FUSED)
    refused(-2, lambda: s.run_phase(capi.PHASE_EVAL, B))
    refused(-2, lambda: s.time_phase(capi.PHASE_EVAL, reps=1))
    d = _moved(data, 0.05)
    _same(_step(s, d), _step(twin, d), "after the refused calls")
    s.close(); twin.close()


@pytest.mark.parametrize("cid", [2, 3])
def test_kernel_key_is_the_same_with_records(cid):
    cfg, B = configs.config_for(cid), 8
    data = configs.generate(cid, B)
    a, b = capi.BatchSolver(cfg, B), capi.BatchSolver(cfg, B)
    a.set_robot_limits(_random_records(cfg, B, 9))
    _step(a, data); _step(b, data)
    assert (a.kernel_model(), a.kernel_problem()) == (b.kernel_model(), b.kernel_problem())
    if cid == 2:
        assert (a.kernel_model(), a.kernel_problem()) == (capi.MODEL_UNI_POINT, capi.PROBLEM_FIXED_DT_QF)
    a.close(); b.close()


def test_execution_options_do_not_change_results():
    cfg, B = configs.cfg2(), 400
    data = configs.generate(2, B)
    rec = _random_records(cfg, B, 11)
    ref = None
    for opt, val in ((capi.OPT_ORDER_BY_HISTORY, 0), (capi.OPT_ORDER_BY_HISTORY, 1), (capi.OPT_CRITICAL_PLACEMENT, 0),
                     (capi.OPT_CTAS_PER_SM, 1), (capi.OPT_CTAS_PER_SM, 2), (capi.OPT_SM_PHASE_SYNC, 0), (capi.OPT_SM_PHASE_SYNC, 2)):
        s = capi.BatchSolver(cfg, B)
        s.set_option(opt, val)
        s.set_robot_limits(rec)
        outs = [_step(s, _moved(data, 0.05 * t)) for t in range(2)]   # the second call is ordered by the first's history
        if ref is None:
            ref = outs
        for o, r in zip(outs, ref):
            _same(o, r, f"option {opt}={val}")
        s.close()


def test_cpp_mirror_lowers_max_vel_x_from_the_second_step():
    """the demo with max_vel_x = 0.3 from its second step on (Controller::setRobotLimits): the first step keeps scenario G1's known
    answer, the later ones converge with u0 <= 0.3"""
    from tests.conftest import ROOT
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples"), "-B", "test_mpc_optim_demo"], stdout=subprocess.DEVNULL)
    p = subprocess.run([os.path.join(ROOT, "examples", "test_mpc_optim_demo"), "4", "0", "-1", "1", "0.3"], capture_output=True,
                       text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    rows = re.findall(r"step (\d+) ok 1 status (\d+) iters (\d+) dt (\S+) u0 (\S+) (\S+)", p.stdout)
    assert len(rows) == 4 and all(r[1] == "0" for r in rows), p.stdout
    assert abs(float(rows[0][3]) - 0.71287734) < 5e-8 and abs(float(rows[0][4]) - 0.4) < 1e-6
    for r in rows[1:]:
        assert float(r[4]) <= 0.3 + 1e-6, r
    assert float(rows[-1][3]) > float(rows[0][3])   # slower: the same path takes longer
