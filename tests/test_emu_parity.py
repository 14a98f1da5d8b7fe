"""The device code (the host/device headers the CUDA kernels are compiled from) replayed by the CPU warp emulator
(tests/emu, test infrastructure) against the CPU oracle.  Runs without a GPU; the real kernels are checked by
tests/test_gpu_parity.py on the GPU."""
import numpy as np
import pytest

import parity as par
from mpc_local_planner_b200 import capi, configs


def _data(cid, B):
    return configs.g1_instance() if cid == 1 else configs.generate(cid, B)


@pytest.mark.parametrize("cid,b", [(1, 0), (2, 0), (2, 2), (3, 2), (4, 1)])
def test_phases_match_oracle(orc, emu, cid, b):
    cfg = configs.config_for(cid, tol=1e-8)
    data = _data(cid, b + 1)
    o = par.oracle_init(orc, cfg, data, b)
    e = emu.instance_from_batch(cfg, data, b)
    e.init(); e.associate()
    par.assert_init(*par.emu_init_fields(e), o, par.EMU)
    steps = marginal = 0
    for it in range(4):
        s, m = par.emu_iterate(o, e, cfg, f"cfg {cid}, iteration {it}")
        steps += s; marginal += m
    assert steps >= 1 and marginal <= 1, (steps, marginal)


@pytest.mark.parametrize("cid,B", [(1, 1), (2, 16), (3, 8), (4, 8), (5, 12)])
def test_full_solve_matches_oracle(orc, emu, cid, B):
    """Whole solves of the device code against the oracle: statuses, dt, controls and the iteration counts.  The counts
    agreed on every instance both solvers converge on, 107 of 107 measured over these batches and a cfg-2 batch of 64; a
    line search that costs iterations shows here first.  The bound leaves one instance per batch."""
    cfg = configs.config_for(cid, tol=1e-8)
    data = _data(cid, B)
    ref = orc.step_batch(cfg, data, n_threads=2)
    n_both = 0
    agree = 0
    same_iters = 0
    for b in range(B):
        e = emu.instance_from_batch(cfg, data, b)
        st = e.solve()
        u, x = e.outputs()
        agree += (st == ref["status"][b])
        if st == 0 and ref["status"][b] == 0:
            n_both += 1
            same_iters += e.field(capi.F_SCAL)[capi.SC_ITER] == ref["iters"][b]
            assert abs(e.field(capi.F_SCAL)[capi.SC_DT] - ref["dt"][b]) < 1e-8
            if not cfg.variable_dt or B == 1:
                assert np.abs(u - ref["u_seq"][b]).max() < 1e-6
    assert n_both >= 1
    assert agree >= 0.8 * B
    assert same_iters >= n_both - 1, (same_iters, n_both)


def test_warm_start_shift_matches_oracle(orc, emu):
    cfg = configs.cfg2(tol=1e-8)
    data = configs.generate(2, 3)
    for b in range(3):
        o = orc.instance_from_batch(cfg, data, b)
        u1, x1, r1 = o.step()
        e = emu.instance_from_batch(cfg, data, b)
        assert e.solve() == r1.status
        ue, xe = e.outputs()
        if r1.status != 0:
            continue
        assert np.abs(ue - u1).max() < 1e-6
        # next control cycle: measured state = second grid state, previous control = applied control
        o.set_measurement(x1[1], data["xf"][b], u1[0], cfg.dt_ref)
        u2, x2, r2 = o.step()
        e.u_prev_dt = cfg.dt_ref
        cnt, types, params = data["obstacles"]
        e.set_inputs(xe[1], data["xf"][b], ue[0], types[b, :cnt[b]], params[b, :cnt[b]])
        st2 = e.solve()
        assert st2 == r2.status
        if st2 == 0:
            u2e, _ = e.outputs()
            assert np.abs(u2e - u2).max() < 1e-6


@pytest.mark.parametrize("cid,B", [(2, 10), (3, 6)])
def test_line_obstacles_match_oracle(orc, emu, cid, B):
    """LineObstacle rows (every second obstacle of the batch turned into a wall segment): association, condensed records
    and whole solves of the device code against the oracle."""
    cfg = configs.config_for(cid, tol=1e-8)
    data = configs.with_line_obstacles(configs.generate(cid, B))
    ref = orc.step_batch(cfg, data, n_threads=2)
    agree = 0
    for b in range(B):
        o = par.oracle_init(orc, cfg, data, b)
        e = emu.instance_from_batch(cfg, data, b)
        e.init(); e.associate()
        par.assert_init(*par.emu_init_fields(e), o, par.EMU)
        par.emu_assert_eval(o, e)
        st = e.solve()
        u, x = e.outputs()
        agree += st == ref["status"][b]
        if st == 0 and ref["status"][b] == 0:
            assert abs(e.field(capi.F_SCAL)[capi.SC_DT] - ref["dt"][b]) < 1e-7
            if not cfg.variable_dt:
                assert np.abs(u - ref["u_seq"][b]).max() < 1e-5
    assert agree >= B - 1


@pytest.mark.parametrize("rule", ["left_sum", "trapezoidal", "hybrid_min_time"])
def test_integral_form_cost_matches_oracle(orc, emu, rule):
    """quadratic_form/integral_form (left sum or trapezoidal rule) with a free dt, and the hybrid minimum-time + quadratic
    control cost: records of the first evaluation and whole solves."""
    cfg = {"left_sum": configs.cfg2_integral_form, "trapezoidal": configs.cfg2_trapezoidal, "hybrid_min_time": configs.cfg2_hybrid_min_time}[rule](tol=1e-8)
    B = 8
    data = configs.generate(2, B)
    ref = orc.step_batch(cfg, data, n_threads=2)
    n_both = 0
    for b in range(B):
        o = par.oracle_init(orc, cfg, data, b)
        e = emu.instance_from_batch(cfg, data, b)
        e.init(); e.associate()
        par.assert_init(*par.emu_init_fields(e), o, par.EMU)
        par.emu_assert_eval(o, e)
        st = e.solve()
        u, x = e.outputs()
        if st == 0 and ref["status"][b] == 0:
            n_both += 1
            assert abs(e.field(capi.F_SCAL)[capi.SC_DT] - ref["dt"][b]) < 1e-7
            assert np.abs(u - ref["u_seq"][b]).max() < 1e-5
    assert n_both >= 2


def test_terminal_ball_matches_oracle(orc, emu):
    """terminal_constraint l2_ball (TerminalBallSE2): records of the first evaluation and whole solves; the ball is
    active on some instances (final state on its boundary) and inactive on others."""
    cfg = configs.cfg2_terminal_ball(tol=1e-8)
    B = 14
    data = configs.generate(2, B)
    ref = orc.step_batch(cfg, data, n_threads=2)
    n_both = n_active = 0
    for b in range(B):
        o = par.oracle_init(orc, cfg, data, b)
        e = emu.instance_from_batch(cfg, data, b)
        e.init(); e.associate()
        par.assert_init(*par.emu_init_fields(e), o, par.EMU)
        par.emu_assert_eval(o, e)
        st = e.solve()
        u, x = e.outputs()
        if st == 0 and ref["status"][b] == 0:
            n_both += 1
            assert np.abs(u - ref["u_seq"][b]).max() < 1e-5
            d = x[-1] - data["xf"][b]
            d[2] = (d[2] + np.pi) % (2 * np.pi) - np.pi
            val = d[0] ** 2 + d[1] ** 2 + 0.5 * d[2] ** 2
            assert val <= cfg.terminal_ball_gamma + 1e-7
            n_active += abs(val - cfg.terminal_ball_gamma) < 1e-6
    assert n_both >= 3 and n_active >= 1


@pytest.mark.parametrize("free_dt", [False, True])
def test_dynamic_obstacles_match_oracle(orc, emu, free_dt):
    """enable_dynamic_obstacles: every obstacle moves with a constant velocity; rows use the predicted positions at t = k dt
    (with a free dt they depend on dt as well)."""
    cfg = configs.cfg2_integral_form(tol=1e-8) if free_dt else configs.cfg2(tol=1e-8)
    cfg.enable_dynamic_obstacles = 1
    B = 8
    data = configs.with_moving_obstacles(configs.generate(2, B))
    ref = orc.step_batch(cfg, data, n_threads=2)
    n_both = 0
    for b in range(B):
        o = par.oracle_init(orc, cfg, data, b)
        e = emu.instance_from_batch(cfg, data, b)
        e.init(); e.associate()
        par.assert_init(*par.emu_init_fields(e), o, par.EMU)
        assert (o.arr("OBSIDX")[:, 1:-1] >= 0).all()  # all (moving) obstacles are kept at every stage
        par.emu_assert_eval(o, e)
        st = e.solve()
        u, x = e.outputs()
        if st == 0 and ref["status"][b] == 0:
            n_both += 1
            assert abs(e.field(capi.F_SCAL)[capi.SC_DT] - ref["dt"][b]) < 1e-7
            assert np.abs(u - ref["u_seq"][b]).max() < 1e-5
    assert n_both >= 2


@pytest.mark.parametrize("n,n_new", [(20, 21), (20, 19), (50, 43), (7, 30), (4, 3)])
def test_resample_matches_oracle(orc, emu, n, n_new):
    """the device's horizon change (resample_serial, behind mpcb200_resample) against the oracle's resampleTrajectory"""
    rng = np.random.default_rng(n + 1000 * n_new)
    X = np.cumsum(rng.normal(0, 0.3, (3, n)), axis=1)
    U = rng.normal(0, 0.3, (2, n)); U[:, n - 1] = 0
    for dt in (0.3, 0.71287734, 1e-3):
        a = emu.resample(X, U, dt, n_new); b = orc.resample_trajectory(X, U, dt, n_new)
        np.testing.assert_array_equal(a[0], b[0]); np.testing.assert_array_equal(a[1], b[1])
        assert a[2] == b[2]


@pytest.mark.parametrize("base", ["cfg2", "cfg2_integral_free_dt", "cfg3"])
def test_midpoint_differences_match_oracle(orc, emu, base):
    """grid/collocation_method midpoint_differences (fd_collocation_se2.h:91-108): records of the first evaluation
    (transformed to the explicit form, cross Hessian block condensed) and whole solves, device code against the oracle."""
    cid = 3 if base == "cfg3" else 2
    n = 30 if base == "cfg3" else 50
    cfg = {"cfg2": configs.cfg2, "cfg2_integral_free_dt": configs.cfg2_integral_form, "cfg3": configs.cfg3}[base](n=n, tol=1e-8)
    cfg.collocation = capi.COLLOC_MIDPOINT
    B = 6
    data = configs.generate(cid, B, n=n)
    ref = orc.step_batch(cfg, data, n_threads=2)
    n_both = 0
    n_other_optimum = 0
    for b in range(B):
        o = par.oracle_init(orc, cfg, data, b)
        e = emu.instance_from_batch(cfg, data, b)
        e.init(); e.associate()
        par.assert_init(*par.emu_init_fields(e), o, par.EMU)
        par.emu_assert_eval(o, e)
        st = e.solve()
        u, x = e.outputs()
        if st == 0 and ref["status"][b] == 0:
            if abs(e.field(capi.F_SCAL)[capi.SC_DT] - ref["dt"][b]) >= 1e-7:
                # non-convex problem, 80+ regularised iterations: rounding differences between the dense (oracle) and the
                # structured (device) factorisation may end in another KKT point -- tolerated once, and it must be one
                n_other_optimum += 1
                assert e.field(capi.F_SCAL)[capi.SC_ERR0] <= cfg.tol
            else:
                n_both += 1
                if base != "cfg3":   # minimum-time optima need not be strict in the controls
                    assert np.abs(u - ref["u_seq"][b]).max() < 1e-5
            # the converged trajectory satisfies the reference's midpoint defect
            dt = e.field(capi.F_SCAL)[capi.SC_DT]
            for k in range(n - 1):
                d = np.zeros(3)
                orc.lib().orc_defect_reference(cfg, x[k].copy().ctypes.data_as(orc.C.POINTER(orc.C.c_double)), u[k].copy().ctypes.data_as(orc.C.POINTER(orc.C.c_double)),
                                               x[k + 1].copy().ctypes.data_as(orc.C.POINTER(orc.C.c_double)), float(dt), d.ctypes.data_as(orc.C.POINTER(orc.C.c_double)))
                assert np.abs(d).max() * dt < 1e-6
    assert n_both >= 2 and n_other_optimum <= 1
