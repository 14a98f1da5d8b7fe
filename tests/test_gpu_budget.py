"""solver/ipopt/max_cpu_time (src/controller.cpp:395-397) on the device: a budget of device time per solve call, counted from the
start of the solve kernel.  No budget (or one that never runs out) changes nothing; an instance that the budget stops after j
iterations returns MAX_TIME and bit for bit what a solve with max_iter = j returns; instances the queue hands out after the deadline
return their initial guess; the queue order of the next batch takes those first."""
import os
import re
import subprocess

import numpy as np
import pytest

from mpc_local_planner_b200 import capi, configs
from tests.conftest import ROOT

pytestmark = pytest.mark.gpu
FIELDS = ("u_seq", "x_seq", "dt", "status", "kkt_err", "iters")


def _with_budget(cfg, t):
    c = cfg.copy()
    c.max_cpu_time = t
    return c


def _step(cfg, data, idx=None, ctas_per_sm=0):
    """one cold batch solve on a fresh handle (queue in index order); idx: a subset of the instances"""
    d = data if idx is None else _subset(data, idx)
    B = d["x0"].shape[0]
    s = capi.BatchSolver(cfg, B, device=0)
    if ctas_per_sm:
        s.set_option(capi.OPT_CTAS_PER_SM, ctas_per_sm)
    out = s.step(d["x0"], d["xf"], d["u_prev"], d["u_prev_dt"], d["obstacles"], d["viapoints"])
    s.close()
    return out


def _subset(data, idx):
    out = dict(data)
    for k in ("x0", "xf", "u_prev"):
        out[k] = data[k][idx]
    if data["obstacles"] is not None:
        out["obstacles"] = tuple(a[idx] for a in data["obstacles"])
    if data["viapoints"] is not None:
        out["viapoints"] = tuple(a[idx] for a in data["viapoints"])
    return out


def _assert_same(a, b, idx=None, fields=FIELDS):
    for f in fields:
        x, y = (a[f], b[f]) if idx is None else (a[f][idx], b[f][idx])
        np.testing.assert_array_equal(x, y, err_msg=f)


def _midpoint():
    c = configs.cfg2(tol=1e-6)
    c.collocation = capi.COLLOC_MIDPOINT
    return c


@pytest.fixture(scope="module")
def cfg2_run():
    """cfg 2, B = 1024, cold: the unbudgeted outputs and the solve time t of a warmed-up handle"""
    cfg = configs.cfg2(tol=1e-6)
    B = 1024
    data = configs.generate(2, B)
    s = capi.BatchSolver(cfg, B, device=0)
    s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    s.reset()
    base = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    s.close()
    return cfg, data, base, base["solve_time_s"]


# ---- 1. no budget / a budget that never runs out: bit-identical to the default config --------------------------------
@pytest.mark.parametrize("case", ["cfg2_b1024", "cfg3", "midpoint"])
def test_no_budget_changes_nothing(cuda_lib, case):
    if case == "cfg2_b1024":
        cfg, data = configs.cfg2(tol=1e-6), configs.generate(2, 1024)
    elif case == "cfg3":
        cfg, data = configs.cfg3(tol=1e-6), configs.generate(3, 256)
    else:
        cfg, data = _midpoint(), configs.generate(2, 128)
    base = _step(cfg, data)
    for t in (-1.0, 1e6):
        _assert_same(_step(_with_budget(cfg, t), data), base)


def test_no_budget_changes_nothing_in_the_queue_and_the_costmap_cycle(cuda_lib):
    from test_gpu_variants import _costmap_scene
    cfg = configs.cfg2(tol=1e-6)
    data = configs.generate(2, 1536)
    res = {}
    for t in (None, -1.0, 1e6):
        s = capi.BatchSolver(cfg if t is None else _with_budget(cfg, t), 512, device=0)
        res[t] = s.solve_stream(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
        s.close()
    _assert_same(res[-1.0], res[None]); _assert_same(res[1e6], res[None])
    B, M = 32, 512
    cost, origin, r, pose, goal = _costmap_scene(B, 0.006, 11)
    for t in (None, -1.0, 1e6):
        s = capi.BatchSolver(cfg if t is None else _with_budget(cfg, t), B, device=0)
        res[t] = s.step_from_costmaps(pose, goal, cost, origin, r, 0.3, M, u_prev=np.zeros((B, 2)), u_prev_dt=0.2)
        s.close()
    _assert_same(res[-1.0], res[None], fields=FIELDS + ("obst_found",)); _assert_same(res[1e6], res[None], fields=FIELDS + ("obst_found",))


# ---- 2. a budget that has run out before the first evaluation: every instance returns its initial guess ----------------
TINY = 1e-9


def _bad_inputs(data):
    d = dict(data)
    d["x0"] = data["x0"].copy(); d["xf"] = data["xf"].copy()
    d["x0"][3, 1] = np.nan
    d["xf"][17, 0] = np.inf
    return d, [3, 17]


def _initial_guess(cfg, data):
    """x, u after the phases INIT + ASSOCIATE (run one by one through the kernel-level API)"""
    B = data["x0"].shape[0]
    s = capi.BatchSolver(cfg, B, device=0)
    s.upload(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
    s.run_phase(capi.PHASE_INIT); s.run_phase(capi.PHASE_ASSOCIATE)
    X, U = s.ws_read(capi.F_X), s.ws_read(capi.F_U)
    s.close()
    return X, U


def _assert_initial_guess(out, X, U, ok, bad):
    N = X.shape[2]
    assert (out["status"][ok] == capi.STATUS_MAX_TIME).all(), out["status"]
    assert (out["iters"][ok] == 0).all()
    assert (out["status"][bad] == capi.STATUS_INVALID_INPUT).all()
    kk = np.minimum(np.arange(N), N - 2)
    np.testing.assert_array_equal(out["u_seq"][ok], np.transpose(U[ok][:, :, kk], (0, 2, 1)))
    np.testing.assert_array_equal(out["x_seq"][ok][:, :, :2], np.transpose(X[ok][:, :2, :], (0, 2, 1)))
    dth = out["x_seq"][ok][:, :, 2] - X[ok][:, 2, :]
    assert np.abs(np.arctan2(np.sin(dth), np.cos(dth))).max() < 1e-12   # headings are returned normalised


def test_tiny_budget_returns_the_initial_guess(cuda_lib):
    cfg = configs.cfg2(tol=1e-6)
    B = 256
    data, bad = _bad_inputs(configs.generate(2, B))
    ok = np.array([b for b in range(B) if b not in bad])
    X, U = _initial_guess(cfg, data)
    s = capi.BatchSolver(_with_budget(cfg, TINY), B, device=0)
    out = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    _assert_initial_guess(out, X, U, ok, bad)
    # MAX_TIME keeps the instance warm (only NUMERICAL_ERROR and invalid inputs leave it cold)
    assert (s.ws_read(capi.F_SCAL)[ok, capi.SC_COLD] == 0).all()
    s.close()
    # the budget spans the outer iterations: five of them stop where one stops
    c5 = _with_budget(cfg, TINY); c5.outer_iterations = 5
    _assert_same(_step(c5, data), out)
    # the queue entry point: one budget for the whole queue
    s = capi.BatchSolver(_with_budget(cfg, TINY), 64, device=0)
    q = s.solve_stream(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    s.close()
    _assert_initial_guess(q, X, U, ok, bad)


# ---- 3. truncation: the budget stops an instance exactly where max_iter = j would ---------------------------------------
def test_truncated_instances_equal_max_iter_solves(cuda_lib, cfg2_run):
    cfg, data, base, t = cfg2_run
    checked = False
    for frac in (0.2, 0.4, 0.6):
        budget = frac * t
        out = _step(_with_budget(cfg, budget), data)
        assert out["solve_time_s"] <= budget + 2e-3, (budget, out["solve_time_s"])
        mt = out["status"] == capi.STATUS_MAX_TIME
        if not ((out["status"] == capi.STATUS_CONVERGED).any() and (mt & (out["iters"] >= 1)).any()):
            continue
        # every instance the budget did not stop ended as without it
        _assert_same(out, base, np.where(~mt)[0])
        # every stopped one holds what a solve with max_iter = its iteration count holds
        for j in np.unique(out["iters"][mt]):
            idx = np.where(mt & (out["iters"] == j))[0]
            if j == 0:
                continue   # never started (test_tiny_budget_returns_the_initial_guess); max_iter >= 1
            capped = cfg.copy(); capped.max_iter = int(j)
            ref = _step(capped, data, idx)
            assert (ref["status"] == capi.STATUS_MAX_ITER).all()
            _assert_same({f: out[f][idx] for f in FIELDS}, ref, fields=("u_seq", "x_seq", "dt", "kkt_err", "iters"))
        checked = True
        break
    assert checked, "no budget in the list stopped some instances after >= 1 iteration while others converged"


# ---- 4. wall time ----------------------------------------------------------------------------------------------------
def test_solve_time_stays_near_the_budget(cuda_lib, cfg2_run):
    cfg, data, base, t = cfg2_run
    budget = 0.3 * t
    out = _step(_with_budget(cfg, budget), data)
    assert (out["status"] == capi.STATUS_MAX_TIME).any()
    assert out["solve_time_s"] <= budget + 2e-3, (budget, out["solve_time_s"], t)


# ---- 5. the queue order of the next batch does not starve the instances the budget never reached -----------------------
def test_never_started_instances_go_first_next_time(cuda_lib):
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per_sm = 2                      # resident CTAs of the solve kernel: 2 x SMs
    B = 2 * per_sm * sms            # two instances per resident CTA
    cfg = configs.cfg2(tol=1e-6)
    data = configs.generate(2, B)
    t = _step(cfg, data, ctas_per_sm=per_sm)["solve_time_s"]
    for frac in (0.6, 0.5, 0.4, 0.3, 0.2, 0.1):
        s = capi.BatchSolver(_with_budget(cfg, frac * t), B, device=0)
        s.set_option(capi.OPT_CTAS_PER_SM, per_sm)
        out1 = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
        never = np.where((out1["status"] == capi.STATUS_MAX_TIME) & (out1["iters"] == 0))[0]
        if len(never) == 0:
            s.close()
            continue
        out2 = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None, reinit=np.ones(B, np.uint8))
        s.close()
        assert (out2["iters"][never] >= 1).all(), (frac, never, out2["iters"][never])
        return
    pytest.fail("no budget in the list left instances unstarted")


# ---- 6. the phased solve mode has no budget ------------------------------------------------------------------------------
def test_phased_mode_with_a_budget_is_unsupported(cuda_lib):
    cfg = _with_budget(configs.cfg2(tol=1e-6), 0.01)
    data = configs.generate(2, 8)
    s = capi.BatchSolver(cfg, 8, device=0)
    s.set_option(capi.OPT_SOLVE_MODE, capi.SOLVE_PHASED)
    with pytest.raises(capi.SolverError, match=r"\(-2\).*max_cpu_time"):
        s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    s.upload(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    with pytest.raises(capi.SolverError, match=r"\(-2\)"):
        s.solve_resident(cold=True)
    s.set_option(capi.OPT_SOLVE_MODE, capi.SOLVE_FUSED)
    s.solve_resident(cold=True)
    s.close()


# ---- 7. the C++ controller: a step the budget stopped still succeeds ----------------------------------------------------
def test_controller_step_succeeds_when_the_budget_runs_out(cuda_lib):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "examples"), "-B", "test_mpc_optim_demo"], stdout=subprocess.DEVNULL)
    p = subprocess.run([os.path.join(ROOT, "examples", "test_mpc_optim_demo"), "3", "0", "1e-9"], capture_output=True, text=True, timeout=300)
    assert p.returncode == 0, p.stdout + p.stderr
    lines = [l for l in p.stdout.splitlines() if l.startswith("step")]
    assert len(lines) == 3
    for l in lines:
        assert re.search(r"ok 1 status 4 iters 0 ", l), l
