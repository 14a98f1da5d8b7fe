"""grid/xf_fixed component by component (controller.cpp:282-292), with a fixed or a free dt: the oracle's Newton step against the
dense KKT system, the device code (replayed by the CPU warp emulator) against the oracle phase by phase and in whole solves, the
warm start with a moved goal, the golden fixtures, and fixed components that stay exactly at the goal.  Runs without a GPU;
tests/test_gpu_fixed_final_state.py runs the same cases on the CUDA kernels.

Which code each case reaches: the root Cholesky of the pi block with 1, 2 or 3 fixed components, with or without a d(dt)
pivot (riccati_root); mixed fixed / free entries of the terminal block and its dt border (rw_terminal); the bordered KKT with
no d(dt) unknown (fixed dt, some component fixed); the terminal cost and ball beside fixed components."""
import numpy as np
import pytest

import dense_kkt as dk
import golden_checks as gc
import parity as par
from fixed_cases import FIXED_CASES, GOLDEN_CASES, SHIPPED, assert_fixed_components_exact, case, moved_goal
from mpc_local_planner_b200 import capi


def assert_same_status(cfg, st_a, it_a, st_b, it_b, what):
    """Equal statuses, except on an instance that one solver finishes within the last 3 iterations of the budget and the other
    does not finish at all (the iterates agree to rounding, the iteration counts need not)."""
    if st_a == st_b:
        return
    marginal = {int(st_a), int(st_b)} == {capi.STATUS_CONVERGED, capi.STATUS_MAX_ITER} and min(it_a, it_b) >= cfg.max_iter - 3
    assert marginal, f"{what}: status {st_a} ({it_a} iterations) vs {st_b} ({it_b} iterations)"


# ---- the oracle's Newton step against the dense KKT system ----
@pytest.mark.parametrize("name", list(FIXED_CASES))
def test_newton_step_matches_dense_kkt(orc, name):
    """Analytic Lagrangian gradient vs finite differences and the Riccati step (terminal block with fixed and free entries,
    the pi multipliers, the dt border where dt is free) vs a dense numpy solve, at multipliers of size 1 and 0.05."""
    cfg, make_data = case(name)
    data = make_data(2)
    compared = 0
    for nu_scale in (1.0, 0.05):
        compared += dk.check_gradient_and_newton_step(orc, None, nu_scale, cfg=cfg, data=data, b=0)
    if compared == 0:   # every regularisation hit the conservative pivot test on this iterate: another instance and seed
        compared += dk.check_gradient_and_newton_step(orc, None, 0.05, cfg=cfg, data=data, b=1, seed=1)
    assert compared >= 1


# ---- the device code (CPU warp emulator) against the oracle ----
@pytest.mark.parametrize("name", list(FIXED_CASES))
def test_phases_match_oracle(orc, emu, name):
    """Four interior-point iterations: records, scalars and the association after each evaluation; the step (states,
    controls and multiplier rows) and d(dt) after each factorisation."""
    cfg, make_data = case(name)
    b = 1
    data = make_data(b + 1)
    o = par.oracle_init(orc, cfg, data, b)
    e = emu.instance_from_batch(cfg, data, b)
    e.init(); e.associate()
    par.assert_init(*par.emu_init_fields(e), o, par.EMU)
    steps = marginal = 0
    for it in range(4):
        s, m = par.emu_iterate(o, e, cfg, f"{name}, iteration {it}")
        steps += s; marginal += m
    assert steps >= 1 and marginal <= 1, (steps, marginal)


def _emu_solves(emu, cfg, data, B):
    out = dict(status=np.zeros(B, dtype=np.int32), u_seq=np.zeros((B, cfg.n, 2)), x_seq=np.zeros((B, cfg.n, 3)), dt=np.zeros(B))
    for b in range(B):
        e = emu.instance_from_batch(cfg, data, b)
        out["status"][b] = e.solve()
        out["u_seq"][b], out["x_seq"][b] = e.outputs()
        out["dt"][b] = e.field(capi.F_SCAL)[capi.SC_DT]
    return out


@pytest.mark.parametrize("name", list(FIXED_CASES))
def test_whole_solves_match_oracle(orc, emu, name):
    cfg, make_data = case(name)
    B = 4 if name == "car_heading_free" else 6
    data = make_data(B)
    ref = orc.step_batch(cfg, data, n_threads=4)
    out = _emu_solves(emu, cfg, data, B)
    np.testing.assert_array_equal(out["status"], ref["status"])
    both = (out["status"] == 0) & (ref["status"] == 0)
    assert both.sum() >= 1, ref["status"]
    assert np.abs(out["dt"][both] - ref["dt"][both]).max() < 1e-8
    assert np.abs(out["u_seq"][both] - ref["u_seq"][both]).max() < 1e-6
    for b in np.flatnonzero(both):
        assert_fixed_components_exact(cfg, out["x_seq"][b, -1], data["xf"][b], f"{name} emulator instance {b}")
        assert_fixed_components_exact(cfg, ref["x_seq"][b, -1], data["xf"][b], f"{name} oracle instance {b}")


@pytest.mark.parametrize("name", ["qf_position_fixed", "mt_heading_free"])
def test_warm_step_with_a_moved_goal(orc, emu, name):
    """Two receding-horizon steps, the goal moved by 0.2 m / 0.1 rad between them: the warm start (the shift with a fixed dt,
    the plain warm path with a free dt) must put the fixed components on the new goal."""
    cfg, make_data = case(name)
    B = 4
    data = make_data(B)
    n_warm = 0
    for b in range(B):
        o = orc.instance_from_batch(cfg, data, b)
        u1, x1, r1 = o.step()
        e = emu.instance_from_batch(cfg, data, b)
        assert e.solve() == r1.status
        ue, xe = e.outputs()
        if r1.status != 0:
            continue
        assert np.abs(ue - u1).max() < 1e-6
        xf2 = moved_goal(data["xf"][b])
        o.set_measurement(x1[1], xf2, u1[0], cfg.dt_ref)
        u2, x2, r2 = o.step()
        e.u_prev_dt = cfg.dt_ref
        cnt, types, params = data["obstacles"]
        e.set_inputs(xe[1], xf2, ue[0], types[b, :cnt[b]], params[b, :cnt[b]])
        st2 = e.solve()
        u2e, x2e = e.outputs()
        assert_same_status(cfg, st2, e.field(capi.F_SCAL)[capi.SC_ITER], r2.status, r2.iters, f"{name} warm, instance {b}")
        if r2.status == 0 and st2 == 0:
            n_warm += 1
            assert np.abs(u2e - u2).max() < 1e-6
            assert_fixed_components_exact(cfg, x2[-1], xf2, f"{name} oracle, warm, instance {b}")
            assert_fixed_components_exact(cfg, x2e[-1], xf2, f"{name} emulator, warm, instance {b}")
    assert n_warm >= 1


# ---- fixed components stay exactly at the goal ----
@pytest.mark.parametrize("name", list(FIXED_CASES) + list(SHIPPED))
def test_fixed_components_stay_exactly_at_the_goal(orc, emu, name):
    """In the reference a fixed component of the final state is not a variable (full_discretization_grid_base_se2.cpp:104-110):
    it equals the goal.  Here it is a row of the KKT system; its step must be exactly zero, or the forward substitution's rounding
    residue is added at every accepted step.  Oracle and device code, cold and after a warm step with a moved goal."""
    cfg, make_data = case(name)
    B = 3 if name.startswith("car") or name == "cfg3" else 4
    data = make_data(B)
    assert (np.abs(data["xf"][:, 2]) < np.pi).all()
    n_conv = 0
    for b in range(B):
        o = orc.instance_from_batch(cfg, data, b)
        u1, x1, r1 = o.step()
        e = emu.instance_from_batch(cfg, data, b)
        st = e.solve()
        ue, xe = e.outputs()
        # every final state the solver returns, converged or not, keeps the fixed components
        assert_fixed_components_exact(cfg, x1[-1], data["xf"][b], f"{name} oracle, cold, instance {b} (status {r1.status})")
        assert_fixed_components_exact(cfg, xe[-1], data["xf"][b], f"{name} emulator, cold, instance {b} (status {st})")
        n_conv += r1.status == 0
        xf2 = moved_goal(data["xf"][b])
        o.set_measurement(x1[1], xf2, u1[0], cfg.dt_ref)
        _, x2, r2 = o.step()
        e.u_prev_dt = cfg.dt_ref
        cnt, types, params = data["obstacles"]
        e.set_inputs(xe[1], xf2, ue[0], types[b, :cnt[b]], params[b, :cnt[b]])
        st2 = e.solve()
        _, x2e = e.outputs()
        assert_fixed_components_exact(cfg, x2[-1], xf2, f"{name} oracle, warm, instance {b} (status {r2.status})")
        assert_fixed_components_exact(cfg, x2e[-1], xf2, f"{name} emulator, warm, instance {b} (status {st2})")
    assert n_conv >= 1


# ---- golden fixtures (SLSQP on the independent numpy restatement) ----
@pytest.mark.parametrize("gcase", GOLDEN_CASES)
def test_golden_cases(orc, gcase):
    matched, other = gc.check_case(gcase, lambda cfg, data: orc.step_batch(cfg, data, n_threads=4))
    assert matched >= 1
