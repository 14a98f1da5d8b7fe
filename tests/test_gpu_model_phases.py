"""The robot models, footprints and via-point objectives of tests/model_cases.py on the CUDA phase kernels, field by field against
the oracle, and the fused solve kernel of each case against the phase kernels bit for bit.

- INIT and ASSOCIATE of a cold start (the CUDA tolerances of tests/parity.py), and ASSOCIATE again from the oracle's
  iterate 10: the association of the outer iterations after the first, with the device's warp argmin over the via-points.  The
  via-point stage has no workspace field; a wrong one shows in the gradient records of the EVAL that follows.
- EVAL, KKT and the line search from the oracle's iterates (parity.compare_at), with the kernel keys.
- Horizons of one warp with idle lanes, several warps, the 4-warp shape and threads that own two stages.
- The geometric edge states of model_cases.EDGES: EVAL and KKT at exact arithmetic.
- Fused == phased: the persistent kernel each case launches (<LINES, EXT, WARPS, MODEL>) computes what the phase kernels
  compute, cold and warm, at N = 20, 50, 100 and 160."""
import numpy as np
import pytest

import linesearch_cases as lc
import model_cases as mc
import parity as par
from mpc_local_planner_b200 import capi

pytestmark = pytest.mark.gpu
B = 4


def _read(s, *fields):
    return [s.ws_read(f) for f in fields]


@pytest.mark.parametrize("name", list(mc.CASES))
def test_init_and_associate_match_oracle(cuda_lib, orc, name):
    make_cfg, make_data, keys = mc.CASES[name]
    cfg = make_cfg()
    data = make_data(B)
    s = par.phase_solver(cfg, data, B)
    s.run_phase(capi.PHASE_INIT); s.run_phase(capi.PHASE_ASSOCIATE)
    assert (s.kernel_model(), s.kernel_problem()) == keys
    init = _read(s, *par.INIT_FIELDS)
    s.run_phase(capi.PHASE_EVAL)
    KKT, SC = _read(s, capi.F_KKT, capi.F_SCAL)
    for b in range(B):
        o = par.oracle_init(orc, cfg, data, b)
        par.assert_init(*(a[b] for a in init), o, par.CUDA, f"cold, instance {b}")
        o.eval()
        par.assert_eval(KKT[b], SC[b], o, par.CUDA, f"cold, instance {b}")
    # re-association from the oracle's iterate 10 (the device's cold start is done: no repair of the guess)
    inst = [par.oracle_iterate(orc, cfg, data, b, 10)[0] for b in range(B)]
    par.write_state(s, inst)
    s.run_phase(capi.PHASE_ASSOCIATE)
    init = _read(s, *par.INIT_FIELDS)
    s.run_phase(capi.PHASE_EVAL)
    KKT, SC = _read(s, capi.F_KKT, capi.F_SCAL)
    s.close()
    for b, o in enumerate(inst):
        o.associate(); o.init_duals()
        par.assert_init(*(a[b] for a in init), o, par.CUDA, f"iterate 10 re-associated, instance {b}")
        np.testing.assert_allclose(SC[b][capi.SC_MU], o.arr("SCAL")[capi.SC_MU], rtol=1e-12)
        o.eval()
        par.assert_eval(KKT[b], SC[b], o, par.CUDA, f"iterate 10 re-associated, instance {b}")


@pytest.mark.parametrize("name", list(mc.CASES))
def test_phases_match_oracle(cuda_lib, orc, name):
    """EVAL, KKT and the line search from the oracle's iterates 0, 1, 3, 10, 25 and the last one, B instances each: at least
    12 of them compared, at most 2 decisions excused as marginal"""
    make_cfg, make_data, keys = mc.CASES[name]
    cfg = make_cfg()
    data = make_data(B)
    compared = marginal = 0
    for j in lc.ITERATES:
        c, m = par.compare_at(orc, cfg, data, B, j, 0, keys)
        compared += c; marginal += m
    print(f"\n{name}: {compared} instance iterates compared, {marginal} marginal")
    assert compared >= 12 and marginal <= 2, (compared, marginal)


@pytest.mark.parametrize("name", ["bicycle_min_time", "line_lines"])
@pytest.mark.parametrize("n", [20, 33, 100, 160])
def test_phases_match_oracle_at_horizons(cuda_lib, orc, name, n):
    make_cfg, make_data, keys = mc.CASES[name]
    cfg = make_cfg(n)
    Bn = 3
    data = make_data(Bn, n)
    compared = marginal = 0
    for j in (0, 3, 10):
        c, m = par.compare_at(orc, cfg, data, Bn, j, 0, keys)
        compared += c; marginal += m
    print(f"\n{name} N={n}: {compared} compared, {marginal} marginal")
    assert compared >= 3 and marginal <= 1, (compared, marginal)


def _edge_states(orc, name, Bn):
    """(cfg, data, the oracle's instances with the stage placed, the stages)"""
    inst, stages = [], []
    for b in range(Bn):
        if name in mc.STEERING_EDGES:
            base, bound = mc.STEERING_EDGES[name]
            cfg, data, _ = mc.case(base, B=Bn)
            o, _ = par.oracle_iterate(orc, cfg, data, b, mc.EDGE_ITERATE)
            k = mc.steer_stage(o, cfg, bound)
        else:
            cfg, data = mc.edge_data(name, Bn)
            _, _, otype, pose = mc.EDGES[name]
            o, _ = par.oracle_iterate(orc, cfg, data, b, mc.EDGE_ITERATE)
            cnt, typ, prm = data["obstacles"]
            k = mc.place_stage(o, otype, pose, typ[b, :cnt[b]], prm[b, :cnt[b]])
        inst.append(o); stages.append(k)
    return cfg, data, inst, stages


@pytest.mark.parametrize("name", list(mc.EDGES) + list(mc.STEERING_EDGES))
def test_edge_states_match_oracle(cuda_lib, orc, name):
    """EVAL and KKT of the phase kernels at the edge states of tests/test_model_phases.py; the placed stage's record at 1e-12
    of the records' scale"""
    Bn = 2
    cfg, data, inst, stages = _edge_states(orc, name, Bn)
    s = par.phase_solver(cfg, data, Bn)
    s.run_phase(capi.PHASE_INIT); s.run_phase(capi.PHASE_ASSOCIATE)
    OBS = s.ws_read(capi.F_OBSIDX)
    for b, o in enumerate(inst):
        np.testing.assert_array_equal(OBS[b], o.arr("OBSIDX"))
    par.write_state(s, inst)
    s.run_phase(capi.PHASE_EVAL)
    KKT, SC = _read(s, capi.F_KKT, capi.F_SCAL)
    s.run_phase(capi.PHASE_KKT)
    STEP, SC2 = _read(s, capi.F_STEP, capi.F_SCAL)
    s.close()
    for b, (o, k) in enumerate(zip(inst, stages)):
        o.eval()
        par.assert_eval(KKT[b], SC[b], o, par.CUDA, f"instance {b}")
        scale = np.abs(o.arr("KKT")).max()
        np.testing.assert_allclose(KKT[b][:, k], o.arr("KKT")[:, k], rtol=0, atol=1e-12 * scale, err_msg=f"stage {k}")
        if SC2[b][capi.SC_DEFER] != 0.0:
            continue
        assert o.kkt_solve(SC2[b][capi.SC_DELTA]) == 0
        par.assert_step(cfg, STEP[b], SC2[b][capi.SC_DDT], o, par.LATE_STEP, f"instance {b}")


@pytest.mark.parametrize("name", mc.VP_CASES)
@pytest.mark.parametrize("n", [30, 50])
def test_via_point_ties_match_oracle(cuda_lib, orc, name, n):
    """Stages of the oracle's iterate 3 put on a via-point (model_cases.via_point_tie) and re-associated: the device's warp
    argmin must give the via-point to the first of the equal minima, as the oracle's loop does.  The via-point stage has no
    workspace field; its terms (Hessian 2 w_p I, the orientation gradient) show in the records of the EVAL that follows."""
    make_cfg, make_data, _ = mc.CASES[name]
    cfg = make_cfg(n)
    Bn = 2
    data = make_data(Bn, n)
    s = par.phase_solver(cfg, data, Bn)
    s.run_phase(capi.PHASE_INIT); s.run_phase(capi.PHASE_ASSOCIATE)
    inst = [par.oracle_iterate(orc, cfg, data, b, 3)[0] for b in range(Bn)]
    stages = [mc.via_point_tie(o, data, b) for b, o in enumerate(inst)]
    par.write_state(s, inst)
    s.run_phase(capi.PHASE_ASSOCIATE)
    init = _read(s, *par.INIT_FIELDS)
    s.run_phase(capi.PHASE_EVAL)
    KKT, SC = _read(s, capi.F_KKT, capi.F_SCAL)
    s.close()
    for b, o in enumerate(inst):
        o.associate(); o.init_duals()
        assert o.vp_stage()[0] == stages[b][0], (o.vp_stage(), stages[b])
        par.assert_init(*(a[b] for a in init), o, par.CUDA, f"instance {b}")
        o.eval()
        par.assert_eval(KKT[b], SC[b], o, par.CUDA, f"instance {b}")


@pytest.mark.parametrize("name", list(mc.CASES))
@pytest.mark.parametrize("n", [20, 50, 100, 160])
def test_fused_and_phased_solves_are_identical(cuda_lib, name, n):
    """the same batch solved cold, then warm, by the persistent kernel and by the phase kernels: every output bit for bit"""
    make_cfg, make_data, keys = mc.CASES[name]
    cfg = make_cfg(n)
    Bn = 16
    data = make_data(Bn, n)
    fused, keys_f = par.solve_twice(cfg, data, Bn, capi.SOLVE_FUSED)
    phased, keys_p = par.solve_twice(cfg, data, Bn, capi.SOLVE_PHASED)
    assert keys_f == keys_p == keys
    assert (fused[0]["status"] == capi.STATUS_CONVERGED).sum() >= Bn // 4, fused[0]["status"]
    par.assert_same_solves(fused, phased, "the fused and the phased solve")
