"""The robot models, footprints and via-point objectives of tests/model_cases.py phase by phase on the CPU: the oracle's
Newton step against the dense KKT system, and the device code (replayed by the CPU warp emulator) against the oracle in
lockstep -- initialisation and association (the via-point stages included), four interior-point iterations from a shared
state, a re-association from a later iterate (the association of the outer iterations after the first), whole solves with
their iteration counts, and the geometric edge states.  tests/test_gpu_model_phases.py runs the same cases on the CUDA phase
kernels."""
import numpy as np
import pytest

import dense_kkt as dk
import model_cases as mc
import parity as par
from mpc_local_planner_b200 import capi

B0 = mc.INSTANCE
INIT_SCAL = (capi.SC_DT, capi.SC_MU)


def _n_vp(data, b):
    return int(data["viapoints"][0][b]) if data.get("viapoints") is not None else 0


def assert_association(o, e, cfg, data, b, what):
    """INIT / ASSOCIATE (states, controls, association, slacks, multipliers), the via-point stages, dt and mu"""
    par.assert_init(*par.emu_init_fields(e), o, par.EMU, what)
    if mc.has_viapoints(cfg):
        np.testing.assert_array_equal(e.vp_stage(_n_vp(data, b)), o.vp_stage(), err_msg=what)
    np.testing.assert_allclose(e.field(capi.F_SCAL)[list(INIT_SCAL)], o.arr("SCAL")[list(INIT_SCAL)], rtol=1e-12, err_msg=what)


# ---- the oracle's Newton step against the dense KKT system ----
@pytest.mark.parametrize("name", list(mc.CASES))
def test_newton_step_matches_dense_kkt(orc, name):
    """Analytic Lagrangian gradient vs finite differences and the Riccati step vs a dense numpy solve of the KKT system
    assembled by finite differences, at multipliers of size 1 and 0.05 (tests/dense_kkt.py).  N = 20 keeps the dense system
    small."""
    cfg, data, _ = mc.case(name, n=20, B=2)
    compared = 0
    for nu_scale in (1.0, 0.05):
        compared += dk.check_gradient_and_newton_step(orc, None, nu_scale, cfg=cfg, data=data, b=B0)
    if compared == 0:   # every regularisation gave the wrong inertia on this iterate: another instance and seed
        compared += dk.check_gradient_and_newton_step(orc, None, 0.05, cfg=cfg, data=data, b=0, seed=1)
    assert compared >= 1


# ---- the device code against the oracle, phase by phase ----
@pytest.mark.parametrize("name", list(mc.CASES))
def test_phases_match_oracle(orc, emu, name):
    """INIT and ASSOCIATE (states, controls, association, via-point stages, slacks, multipliers, mu), then four iterations
    in lockstep; then the oracle's iterate 10 re-associated on both sides (no cold-start repair: the association of every
    outer iteration after the first) and four more iterations from there."""
    cfg, data, _ = mc.case(name)
    o = par.oracle_init(orc, cfg, data, B0)
    e = emu.instance_from_batch(cfg, data, B0)
    e.init(); e.associate()
    assert_association(o, e, cfg, data, B0, "cold")
    steps = marginal = 0
    for it in range(4):
        s, m = par.emu_iterate(o, e, cfg, f"{name}, iteration {it}")
        steps += s; marginal += m
    o, converged = par.oracle_iterate(orc, cfg, data, B0, 10)
    par.emu_set_state(e, o)
    o.associate(); o.init_duals()
    e.associate(first_outer=False)
    assert_association(o, e, cfg, data, B0, "iterate 10, re-associated")
    if not converged:
        for it in range(4):
            s, m = par.emu_iterate(o, e, cfg, f"{name}, re-associated, iteration {it}")
            steps += s; marginal += m
    assert steps >= 3 and marginal <= 1, (steps, marginal)


def _emu_solve(emu, cfg, data, b):
    """emu_solve, with the iterations of every outer iteration summed as the oracle counts them"""
    e = emu.instance_from_batch(cfg, data, b)
    e.init()
    iters = 0
    for oi in range(max(cfg.outer_iterations, 1)):
        e.associate(first_outer=oi == 0)
        for it in range(cfg.max_iter + 1):
            if e.eval() or it == cfg.max_iter or e.kkt():
                break
            e.linesearch()
        iters += int(e.field(capi.F_SCAL)[capi.SC_ITER])
    st = e.field(capi.F_SCAL)[capi.SC_STATUS]
    return (capi.STATUS_MAX_ITER if st < 0 else int(st)), iters, e


@pytest.mark.parametrize("name", list(mc.CASES))
def test_whole_solves_match_oracle(orc, emu, name):
    """Whole solves of the device code against the oracle: statuses, dt, controls (fixed dt) and iteration counts.  A wrong
    Hessian term leaves the solution where it is and costs iterations: the counts must agree on all but one instance that
    both solvers converge on."""
    make_cfg, make_data, _ = mc.CASES[name]
    cfg = make_cfg()
    B = 6
    data = make_data(B)
    ref = orc.step_batch(cfg, data, n_threads=4)
    agree = n_both = same_iters = 0
    for b in range(B):
        st, iters, e = _emu_solve(emu, cfg, data, b)
        agree += st == ref["status"][b]
        if st == 0 and ref["status"][b] == 0:
            n_both += 1
            same_iters += iters == ref["iters"][b]
            assert abs(e.field(capi.F_SCAL)[capi.SC_DT] - ref["dt"][b]) < 1e-8
            if not cfg.variable_dt:
                u, _ = e.outputs()
                assert np.abs(u - ref["u_seq"][b]).max() < 1e-6
    assert n_both >= 2, ref["status"]
    assert agree >= B - 1, (agree, ref["status"])
    assert same_iters >= n_both - 1, (same_iters, n_both, ref["iters"])


# ---- geometric edge states ----
def _edge_state(orc, name, B):
    """the oracle's iterate EDGE_ITERATE of instance B-1 of the edge state's batch, the stage placed; (cfg, data, o, stage)"""
    b = B - 1
    if name in mc.STEERING_EDGES:
        base, bound = mc.STEERING_EDGES[name]
        cfg, data, _ = mc.case(base, B=B)
        o, _ = par.oracle_iterate(orc, cfg, data, b, mc.EDGE_ITERATE)
        return cfg, data, o, mc.steer_stage(o, cfg, bound)
    cfg, data = mc.edge_data(name, B)
    _, _, otype, pose = mc.EDGES[name]
    o, _ = par.oracle_iterate(orc, cfg, data, b, mc.EDGE_ITERATE)
    cnt, typ, prm = data["obstacles"]
    return cfg, data, o, mc.place_stage(o, otype, pose, typ[b, :cnt[b]], prm[b, :cnt[b]])


@pytest.mark.parametrize("name", list(mc.EDGES) + list(mc.STEERING_EDGES))
def test_edge_states_match_oracle(orc, emu, name):
    """EVAL and KKT of the device code against the oracle at a geometric edge state (model_cases.EDGES: ties of two features,
    projections at a segment's end, an obstacle on the footprint, crossing, parallel and zero-length line obstacles, headings
    of +-pi; the steering control at its bound), on two instances.  The record of the placed stage is compared at 1e-12 of
    the records' scale as well: the arithmetic of its obstacle rows is exact."""
    for B in (1, 2):
        cfg, data, o, k = _edge_state(orc, name, B)
        e = par.emu_from_oracle(emu, cfg, data, B - 1, o)
        par.eval_and_kkt(o, e, cfg)
        scale = np.abs(o.arr("KKT")).max()
        np.testing.assert_allclose(e.field(capi.F_KKT)[:, k], o.arr("KKT")[:, k], atol=1e-12 * scale, err_msg=f"stage {k}")


@pytest.mark.parametrize("name", mc.VP_CASES)
@pytest.mark.parametrize("n", [30, 50])
def test_via_point_ties_match_oracle(orc, emu, name, n):
    """Stages of the oracle's iterate 3 put on a via-point (model_cases.via_point_tie), then re-associated on both sides: the
    first of the equal minima gets the via-point, then EVAL and KKT"""
    make_cfg, make_data, _ = mc.CASES[name]
    cfg = make_cfg(n)
    data = make_data(2, n)
    for b in range(2):
        o, _ = par.oracle_iterate(orc, cfg, data, b, 3)
        stages = mc.via_point_tie(o, data, b)
        e = par.emu_from_oracle(emu, cfg, data, b, o)
        o.associate(); o.init_duals()
        e.associate(first_outer=False)
        assert_association(o, e, cfg, data, b, f"instance {b}")
        assert o.vp_stage()[0] == stages[0], (o.vp_stage(), stages)
        par.eval_and_kkt(o, e, cfg)


@pytest.mark.parametrize("name", ["front_quadratic", "front_min_time", "bicycle_quadratic", "bicycle_min_time"])
def test_init_controls_of_a_standing_plan(orc, emu, name):
    """The cold start from an initial plan that stands still while it turns (and moves 1.5e-4 m in one interval): the
    dynamics are not inverted where |v| <= 1e-3 (init_controls_stage).  States, controls and duals after INIT and ASSOCIATE."""
    cfg, data, _ = mc.case(name, B=2)
    for b in range(2):
        xi = mc.standing_plan(cfg, data, b)
        o = par.oracle_init(orc, cfg, data, b, x_init=xi)
        e = emu.instance_from_batch(cfg, data, b, x_init=xi)
        e.init(); e.associate()
        assert_association(o, e, cfg, data, b, f"instance {b}")
        assert (o.arr("U")[1, 0:3] == 0.0).all(), o.arr("U")[:, :4]   # the branch is taken: no steering while standing
