"""The robot models, footprints and via-point objectives of tests/model_cases.py on the CUDA phase kernels, field by field against
the oracle, and the fused solve kernel of each case against the phase kernels bit for bit.

- INIT and ASSOCIATE of a cold start (tolerances of test_gpu_parity.test_phase_parity), and ASSOCIATE again from the oracle's
  iterate 10: the association of the outer iterations after the first, with the device's warp argmin over the via-points.  The
  via-point stage has no workspace field; a wrong one shows in the gradient records of the EVAL that follows.
- EVAL, KKT and the line search from the oracle's iterates (test_gpu_linesearch._compare_at), with the kernel keys.
- Horizons of one warp with idle lanes, several warps, the 4-warp shape and threads that own two stages.
- The geometric edge states of model_cases.EDGES: EVAL and KKT at exact arithmetic.
- Fused == phased: the persistent kernel each case launches (<LINES, EXT, WARPS, MODEL>) computes what the phase kernels
  compute, cold and warm, at N = 20, 50, 100 and 160."""
import numpy as np
import pytest

import linesearch_cases as lc
import model_cases as mc
import test_gpu_linesearch as tgl
import test_gpu_model_variants as tmv
from mpc_local_planner_b200 import capi

pytestmark = pytest.mark.gpu
B = 4


def _solver(cfg, data, Bn):
    s = capi.BatchSolver(cfg, Bn, device=0)
    s.upload(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
    return s


def _assert_init(X, U, S, LAM, OBS, o, what):
    np.testing.assert_allclose(X, o.arr("X"), rtol=0, atol=1e-12, err_msg=what)
    np.testing.assert_allclose(U, o.arr("U"), rtol=0, atol=1e-12, err_msg=what)
    np.testing.assert_array_equal(OBS, o.arr("OBSIDX"), err_msg=what)
    np.testing.assert_allclose(S, o.arr("S"), rtol=1e-11, atol=1e-13, err_msg=what)
    np.testing.assert_allclose(LAM, o.arr("LAM"), rtol=1e-10, atol=1e-13, err_msg=what)


def _assert_eval(KKT, SC, o, what):
    o.eval()
    scale = np.abs(o.arr("KKT")).max()
    np.testing.assert_allclose(KKT, o.arr("KKT"), rtol=0, atol=1e-11 * scale, err_msg=what)
    idx = list(lc.EVAL_SCAL)
    np.testing.assert_allclose(SC[idx], o.arr("SCAL")[idx], rtol=1e-10, atol=1e-12, err_msg=what)


def _read(s, *fields):
    return [s.ws_read(f) for f in fields]


@pytest.mark.parametrize("name", list(mc.CASES))
def test_init_and_associate_match_oracle(cuda_lib, orc, name):
    make_cfg, make_data, keys = mc.CASES[name]
    cfg = make_cfg()
    data = make_data(B)
    s = _solver(cfg, data, B)
    s.run_phase(capi.PHASE_INIT); s.run_phase(capi.PHASE_ASSOCIATE)
    assert (s.kernel_model(), s.kernel_problem()) == keys
    X, U, S, LAM, OBS = _read(s, capi.F_X, capi.F_U, capi.F_S, capi.F_LAM, capi.F_OBSIDX)
    s.run_phase(capi.PHASE_EVAL)
    KKT, SC = _read(s, capi.F_KKT, capi.F_SCAL)
    for b in range(B):
        o = lc.oracle_init(orc, cfg, data, b)
        _assert_init(X[b], U[b], S[b], LAM[b], OBS[b], o, f"cold, instance {b}")
        _assert_eval(KKT[b], SC[b], o, f"cold, instance {b}")
    # re-association from the oracle's iterate 10 (the device's cold start is done: no repair of the guess)
    inst = [lc.oracle_iterate(orc, cfg, data, b, 10)[0] for b in range(B)]
    for nm, f in lc.STATE_FIELDS:
        s.ws_write(f, np.stack([o.arr(nm) for o in inst]))
    SC = s.ws_read(capi.F_SCAL)
    s.ws_write(capi.F_SCAL, np.stack([lc.merged_scal(SC[b], inst[b].arr("SCAL")) for b in range(B)]))
    s.run_phase(capi.PHASE_ASSOCIATE)
    X, U, S, LAM, OBS = _read(s, capi.F_X, capi.F_U, capi.F_S, capi.F_LAM, capi.F_OBSIDX)
    s.run_phase(capi.PHASE_EVAL)
    KKT, SC = _read(s, capi.F_KKT, capi.F_SCAL)
    s.close()
    for b, o in enumerate(inst):
        o.associate(); o.init_duals()
        _assert_init(X[b], U[b], S[b], LAM[b], OBS[b], o, f"iterate 10 re-associated, instance {b}")
        np.testing.assert_allclose(SC[b][capi.SC_MU], o.arr("SCAL")[capi.SC_MU], rtol=1e-12)
        _assert_eval(KKT[b], SC[b], o, f"iterate 10 re-associated, instance {b}")


@pytest.mark.parametrize("name", list(mc.CASES))
def test_phases_match_oracle(cuda_lib, orc, name):
    """EVAL, KKT and the line search from the oracle's iterates 0, 1, 3, 10, 25 and the last one, B instances each: at least
    12 of them compared, at most 2 decisions excused as marginal"""
    make_cfg, make_data, keys = mc.CASES[name]
    cfg = make_cfg()
    data = make_data(B)
    compared = marginal = 0
    for j in lc.ITERATES:
        c, m = tgl._compare_at(orc, cfg, data, B, j, 0, keys)
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
        c, m = tgl._compare_at(orc, cfg, data, Bn, j, 0, keys)
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
            o, _ = lc.oracle_iterate(orc, cfg, data, b, mc.EDGE_ITERATE)
            k = mc.steer_stage(o, cfg, bound)
        else:
            cfg, data = mc.edge_data(name, Bn)
            _, _, otype, pose = mc.EDGES[name]
            o, _ = lc.oracle_iterate(orc, cfg, data, b, mc.EDGE_ITERATE)
            cnt, typ, par = data["obstacles"]
            k = mc.place_stage(o, otype, pose, typ[b, :cnt[b]], par[b, :cnt[b]])
        inst.append(o); stages.append(k)
    return cfg, data, inst, stages


@pytest.mark.parametrize("name", list(mc.EDGES) + list(mc.STEERING_EDGES))
def test_edge_states_match_oracle(cuda_lib, orc, name):
    """EVAL and KKT of the phase kernels at the edge states of tests/test_model_phases.py; the placed stage's record at 1e-12
    of the records' scale"""
    Bn = 2
    cfg, data, inst, stages = _edge_states(orc, name, Bn)
    s = _solver(cfg, data, Bn)
    s.run_phase(capi.PHASE_INIT); s.run_phase(capi.PHASE_ASSOCIATE)
    OBS = s.ws_read(capi.F_OBSIDX)
    for b, o in enumerate(inst):
        np.testing.assert_array_equal(OBS[b], o.arr("OBSIDX"))
    for nm, f in lc.STATE_FIELDS:
        s.ws_write(f, np.stack([o.arr(nm) for o in inst]))
    SC = s.ws_read(capi.F_SCAL)
    s.ws_write(capi.F_SCAL, np.stack([lc.merged_scal(SC[b], inst[b].arr("SCAL")) for b in range(Bn)]))
    s.run_phase(capi.PHASE_EVAL)
    KKT, SC = _read(s, capi.F_KKT, capi.F_SCAL)
    s.run_phase(capi.PHASE_KKT)
    STEP, SC2 = _read(s, capi.F_STEP, capi.F_SCAL)
    s.close()
    rows = lc.step_rows(cfg)
    for b, (o, k) in enumerate(zip(inst, stages)):
        _assert_eval(KKT[b], SC[b], o, f"instance {b}")
        scale = np.abs(o.arr("KKT")).max()
        np.testing.assert_allclose(KKT[b][:, k], o.arr("KKT")[:, k], rtol=0, atol=1e-12 * scale, err_msg=f"stage {k}")
        if SC2[b][capi.SC_DEFER] != 0.0:
            continue
        assert o.kkt_solve(SC2[b][capi.SC_DELTA]) == 0
        sscale = max(np.abs(o.arr("STEP")).max(), 1.0)
        np.testing.assert_allclose(STEP[b][:rows], o.arr("STEP")[:rows], rtol=0, atol=1e-7 * sscale)


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
    s = _solver(cfg, data, Bn)
    s.run_phase(capi.PHASE_INIT); s.run_phase(capi.PHASE_ASSOCIATE)
    inst = [lc.oracle_iterate(orc, cfg, data, b, 3)[0] for b in range(Bn)]
    stages = [mc.via_point_tie(o, data, b) for b, o in enumerate(inst)]
    for nm, f in lc.STATE_FIELDS:
        s.ws_write(f, np.stack([o.arr(nm) for o in inst]))
    SC = s.ws_read(capi.F_SCAL)
    s.ws_write(capi.F_SCAL, np.stack([lc.merged_scal(SC[b], inst[b].arr("SCAL")) for b in range(Bn)]))
    s.run_phase(capi.PHASE_ASSOCIATE)
    X, U, S, LAM, OBS = _read(s, capi.F_X, capi.F_U, capi.F_S, capi.F_LAM, capi.F_OBSIDX)
    s.run_phase(capi.PHASE_EVAL)
    KKT, SC = _read(s, capi.F_KKT, capi.F_SCAL)
    s.close()
    for b, o in enumerate(inst):
        o.associate(); o.init_duals()
        assert o.vp_stage()[0] == stages[b][0], (o.vp_stage(), stages[b])
        _assert_init(X[b], U[b], S[b], LAM[b], OBS[b], o, f"instance {b}")
        _assert_eval(KKT[b], SC[b], o, f"instance {b}")


@pytest.mark.parametrize("name", list(mc.CASES))
@pytest.mark.parametrize("n", [20, 50, 100, 160])
def test_fused_and_phased_solves_are_identical(cuda_lib, name, n):
    """the same batch solved cold, then warm, by the persistent kernel and by the phase kernels: every output bit for bit"""
    make_cfg, make_data, keys = mc.CASES[name]
    cfg = make_cfg(n)
    Bn = 16
    data = make_data(Bn, n)
    fused, model_f = tmv._solve_twice(cfg, data, Bn, 0, capi.SOLVE_FUSED)
    phased, model_p = tmv._solve_twice(cfg, data, Bn, 0, capi.SOLVE_PHASED)
    assert model_f == model_p == keys[0]
    assert (fused[0]["status"] == capi.STATUS_CONVERGED).sum() >= Bn // 4, fused[0]["status"]
    for step, (a, b) in enumerate(zip(fused, phased)):
        for f in tmv.FIELDS:
            assert np.array_equal(tmv._bits(a[f]), tmv._bits(b[f])), f"step {step}: {f} differs between the fused and the phased solve"
