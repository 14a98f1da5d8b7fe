"""GPU parity of the device variants that the BASELINE configurations do not exercise: front-drive car and kinematic bicycle
(include/mpc_local_planner/systems/simple_car.h:131-141, kinematic_bicycle_model.h:65-77), circular / two-circles / line
footprints (src/mpc_local_planner_ros.cpp:890-1044), the reference's own via-point objective with ordered association and the
linear orientation term (src/optimal_control/min_time_via_points_cost.cpp:40-145), several outer OCP iterations
(controller/outer_ocp_iterations = 5 in the shipped minimum-time configuration), and the error statuses of the batch ABI.
Each case: the CUDA path through the C ABI against the CPU oracle on the same seeded instances."""
import numpy as np
import pytest

import costmap_cases as cm
from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu
U_TOL = 1e-4


def _compare(cfg, data, orc, min_both, strict_controls=True, status_agree=0.9):
    B = data["x0"].shape[0]
    s = capi.BatchSolver(cfg, B, device=0)
    out = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
    s.close()
    ref = orc.step_batch(cfg, data, n_threads=4)
    agree = (out["status"] == ref["status"]).mean()
    assert agree >= status_agree, f"status agreement {agree}: gpu {out['status']} oracle {ref['status']}"
    both = (out["status"] == 0) & (ref["status"] == 0)
    assert both.sum() >= min_both, f"gpu {out['status']} oracle {ref['status']}"
    assert np.abs(out["dt"][both] - ref["dt"][both]).max() < 1e-6
    du = np.abs(out["u_seq"][both] - ref["u_seq"][both]).max(axis=(1, 2))
    if strict_controls:
        assert (du < U_TOL).mean() >= 0.95, f"du {du}"
    else:   # minimum-time optima need not be strict in the controls (SURVEY 7, hard part 3): the optimal time is
        assert (du < U_TOL).mean() >= 0.8, f"du {du}"
    assert (out["kkt_err"][both] <= cfg.tol).all()
    return out, ref


@pytest.mark.parametrize("robot", ["simple_car_front", "kinematic_bicycle"])
@pytest.mark.parametrize("objective", ["quadratic", "min_time"])
def test_robot_models(cuda_lib, orc, robot, objective):
    """a2 (front wheel driving) and a3 (kinematic bicycle, velocity input) on the device."""
    if objective == "quadratic":
        cfg = configs.cfg2(tol=1e-8)
        data = configs.generate(2, 24)
    else:
        cfg = configs.cfg3(n=40, tol=1e-8)
        cfg.footprint_type = capi.FOOTPRINT_POINT
        data = configs.generate(3, 16, n=40)
    if robot == "simple_car_front":
        cfg.robot_type = capi.ROBOT_SIMPLE_CAR_FRONT
        cfg.wheelbase = 0.4
    else:
        cfg.robot_type = capi.ROBOT_KIN_BICYCLE
        cfg.length_rear, cfg.length_front = 0.2, 0.25
    cfg.u_lb[:] = [-0.2, -1.2]
    cfg.u_ub[:] = [0.4, 1.2]
    cfg.du_lb[:] = [-0.5, -0.5]
    cfg.du_ub[:] = [0.5, 0.5]
    _compare(cfg, data, orc, min_both=6, strict_controls=(objective == "quadratic"), status_agree=0.85)


@pytest.mark.parametrize("footprint", ["circular", "two_circles", "line"])
@pytest.mark.parametrize("with_lines", [False, True])
def test_footprint_models(cuda_lib, orc, footprint, with_lines):
    """a13: circular, two-circles and line footprints against point / circle (and line) obstacles on the device."""
    cfg = configs.cfg2(tol=1e-8)
    if footprint == "circular":
        cfg.footprint_type = capi.FOOTPRINT_CIRCULAR
        cfg.footprint_params[0] = 0.15
        cfg.min_obstacle_dist = 0.1
    elif footprint == "two_circles":
        cfg.footprint_type = capi.FOOTPRINT_TWO_CIRCLES
        cfg.footprint_params[:] = [0.2, 0.12, 0.15, 0.1]
        cfg.min_obstacle_dist = 0.1
    else:
        cfg.footprint_type = capi.FOOTPRINT_LINE
        cfg.footprint_params[:] = [-0.15, 0.0, 0.2, 0.0]
        cfg.min_obstacle_dist = 0.15
    data = configs.generate(2, 24)
    if with_lines:
        data = configs.with_line_obstacles(data)
    _compare(cfg, data, orc, min_both=8, status_agree=0.85)


@pytest.mark.parametrize("ordered", [0, 1])
@pytest.mark.parametrize("ori_weight", [0.0, 0.3])
def test_minimum_time_via_points_objective(cuda_lib, orc, ordered, ori_weight):
    """a11: objective minimum_time_via_points itself (not the quadratic-form extension): (N-1) dt + w_p |p_vp - p_k|^2
    (+ w_th wrap(th_vp - th_k), LINEAR as coded in the reference), association with via_points_ordered on and off."""
    cfg = configs.cfg1(tol=1e-8)
    cfg.n = 30
    cfg.objective = capi.OBJ_MINIMUM_TIME_VIA_POINTS
    cfg.vp_position_weight = 1.5
    cfg.vp_orientation_weight = ori_weight
    cfg.vp_ordered = ordered
    cfg.du_lb[:] = [-0.3, -0.4]
    cfg.du_ub[:] = [0.3, 0.4]
    cfg.min_obstacle_dist = 0.2
    cfg.k_max_obstacles_per_stage = 5
    data = configs.generate(4, 16)
    # the via-point list in REVERSE order of the path (ordered association then differs from the closest-pose association:
    # it only searches behind the previous via-point's pose) and with headings along the start -> goal line
    vc, vp = data["viapoints"]
    vp = vp[:, ::-1].copy()
    vp[:, :, 2] = np.arctan2(data["xf"][:, 1], data["xf"][:, 0])[:, None]
    data["viapoints"] = (vc, vp)
    _compare(cfg, data, orc, min_both=5, strict_controls=False, status_agree=0.85)


def test_five_outer_iterations(cuda_lib, orc):
    """controller/outer_ocp_iterations = 5 (EX/cfg/diff_drive/mpc_local_planner_params_minimum_time.yaml:73): every outer
    iteration re-associates obstacles and via-points on the new trajectory and solves again from it."""
    cfg = configs.cfg1(tol=1e-8)
    cfg.n = 30
    cfg.outer_iterations = 5
    cfg.min_obstacle_dist = 0.25
    cfg.k_max_obstacles_per_stage = 4
    data = configs.generate(2, 16)
    out, ref = _compare(cfg, data, orc, min_both=5, strict_controls=False, status_agree=0.85)
    # and both solve modes run the same outer loop
    s = capi.BatchSolver(cfg, 16, device=0)
    s.set_option(capi.OPT_SOLVE_MODE, capi.SOLVE_PHASED)
    ph = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    s.close()
    np.testing.assert_array_equal(out["status"], ph["status"])
    np.testing.assert_array_equal(out["u_seq"], ph["u_seq"])


def test_invalid_inputs_are_reported_per_instance(cuda_lib):
    """NaN / inf in the inputs of an instance: status INVALID_INPUT, zero outputs, no iteration; the others are untouched;
    the instance starts cold the next time."""
    cfg = configs.cfg2(tol=1e-6)
    B = 12
    data = configs.generate(2, B)
    x0 = data["x0"].copy(); xf = data["xf"].copy()
    cnt, typ, par = (a.copy() for a in data["obstacles"])
    x0[3, 1] = np.nan
    xf[5, 0] = np.inf
    par[7, 2, 0] = np.nan          # an obstacle in use
    par[9, 4, 1] = np.nan; cnt[9] = 4   # NaN in a padding slot: never read
    s = capi.BatchSolver(cfg, B, device=0)
    out = s.step(x0, xf, data["u_prev"], data["u_prev_dt"], (cnt, typ, par), None)
    clean = s2 = None
    bad = [3, 5, 7]
    assert (out["status"][bad] == capi.STATUS_INVALID_INPUT).all(), out["status"]
    assert (out["u_seq"][bad] == 0).all() and (out["x_seq"][bad] == 0).all() and (out["iters"][bad] == 0).all()
    ok = [b for b in range(B) if b not in bad]
    assert np.isfinite(out["u_seq"][ok]).all() and (out["status"][ok] != capi.STATUS_INVALID_INPUT).all()
    # the healthy instances got what they get in a clean batch
    s2 = capi.BatchSolver(cfg, B, device=0)
    cnt9 = data["obstacles"][0].copy(); cnt9[9] = 4
    clean = s2.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], (cnt9, typ, data["obstacles"][2]), None)
    keep = [b for b in ok]
    np.testing.assert_array_equal(out["u_seq"][keep], clean["u_seq"][keep])
    # repaired inputs: the instance is solved from a cold start
    out2 = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], (cnt9, typ, data["obstacles"][2]), None)
    assert (out2["status"][bad] != capi.STATUS_INVALID_INPUT).all()
    np.testing.assert_array_equal(out2["u_seq"][bad], clean["u_seq"][bad])
    s.close(); s2.close()


def test_failed_instance_restarts_cold(cuda_lib):
    """An instance that ends with NUMERICAL_ERROR keeps nothing to warm-start from: the next step solves it from the cold
    initial guess (the reference's planner resets the controller after a failed step, mpc_local_planner_ros.cpp:394-404)."""
    cfg = configs.cfg2(tol=1e-8)
    cfg.max_iter = 100
    B = 256
    data = configs.generate(2, B)
    s = capi.BatchSolver(cfg, B, device=0)
    out = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    failed = np.where(out["status"] == capi.STATUS_NUMERICAL_ERROR)[0]
    sc = s.ws_read(capi.F_SCAL)
    assert (sc[failed, capi.SC_COLD] == 1.0).all()
    healthy = np.where(out["status"] != capi.STATUS_NUMERICAL_ERROR)[0]
    assert (sc[healthy, capi.SC_COLD] == 0.0).all()
    if len(failed):
        out2 = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
        np.testing.assert_array_equal(out2["status"][failed], out["status"][failed])     # same cold solve, same outcome
        np.testing.assert_array_equal(out2["u_seq"][failed], out["u_seq"][failed])
    s.close()


@pytest.mark.parametrize("footprint", ["polygon", "two_points"])
def test_check_feasible_matches_the_oracle(cuda_lib, orc, footprint):
    """mpcb200_check_feasible (Controller::isPoseTrajectoryFeasible, controller.cpp:859-917) for a batch of robots: accept /
    reject byte for byte as the oracle's plain-C loop, on random maps, trajectories that turn and leave the map, both look-ahead
    settings -- and on the trajectories of a solve that are still on the device."""
    rng = np.random.default_rng(5)
    fp = np.array(configs.CARLIKE_POLYGON) if footprint == "polygon" else np.array([[0.1, 0.0], [-0.1, 0.0]])
    cases = cm.feasibility_cases(rng, 96)
    cost = np.stack([c[0] for c in cases]); origin = np.stack([c[1] for c in cases]); xs = np.stack([c[2] for c in cases])
    cfg = configs.cfg2(tol=1e-6)
    s = capi.BatchSolver(cfg, 96, device=0)
    for look in (-1, 5):
        got = s.check_feasible(cost, origin, 0.05, fp, 0.18, 0.3, look, x_seq=xs)
        want = np.array([orc.pose_trajectory_feasible(cost[b], origin[b], 0.05, xs[b], fp, 0.18, 0.3, look) for b in range(96)])
        np.testing.assert_array_equal(got, want)
        assert want.any() and not want.all()
    # the trajectories of the last solve, checked where they are (device)
    data = configs.generate(2, 96)
    out = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    H, W, res = 200, 200, 0.05
    maps = np.zeros((96, H, W), dtype=np.uint8)
    org = np.tile(np.array([-2.0, -5.0]), (96, 1))
    cnt, typ, par = data["obstacles"]
    for b in range(96):      # the obstacle centres of the instance as lethal cells
        for j in range(cnt[b]):
            mx, my = int((par[b, j, 0] - org[b, 0]) / res), int((par[b, j, 1] - org[b, 1]) / res)
            if 0 <= mx < W and 0 <= my < H:
                maps[b, my, mx] = 254
    got = s.check_feasible(maps, org, res, fp, 0.18, 0.3, -1)
    want = np.array([orc.pose_trajectory_feasible(maps[b], org[b], res, out["x_seq"][b], fp, 0.18, 0.3, -1) for b in range(96)])
    np.testing.assert_array_equal(got, want)
    s.close()


def test_multi_device_handle_equals_single_device(cuda_lib):
    """mpcb200_create_multi / mpcb200_step_batch_multi (SURVEY 8e): contiguous blocks over the devices, one NCCL all-gather of
    u*.  The G-device results equal the 1-device results bit for bit, and every device holds the controls of all instances."""
    import torch
    G = torch.cuda.device_count()
    if G < 2:
        pytest.skip("needs at least two devices")
    G = min(G, 8)
    cfg = configs.cfg2(tol=1e-6)
    B = 64 * G - 5          # ragged last block
    data = configs.generate(2, B)
    s = capi.BatchSolver(cfg, B, device=0)
    one = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    s.close()
    m = capi.MultiSolver(cfg, B, list(range(G)))
    many = m.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    for k in ("status", "iters", "u_seq", "x_seq", "dt"):
        np.testing.assert_array_equal(one[k], many[k])
    per = (B + G - 1) // G
    for rank in (0, G - 1):
        g = m.gathered_controls(rank).reshape(G * per, cfg.n - 1, 2)[:B]
        np.testing.assert_array_equal(g, one["u_seq"][:, :-1, :])
    m.close()


def test_long_obstacle_lists_stay_in_global_memory(cuda_lib, orc):
    """SURVEY 8 f-1, second half: the raw costmap list of a robot (hundreds of point obstacles, far beyond the 64 resident
    slots) goes into step() as it is.  The association runs over the list in global memory (StageInequalitySE2::update,
    stage_inequality_se2.cpp:73-147) and only what it selects becomes resident: same rows per stage as the oracle's loop over the
    full list, same cold start (the bumps look at the full list as well), same solves."""
    B, M = 16, 512
    cost, origin, res, pose, goal = cm.costmap_scene(B, 0.006, 11)
    cfg = configs.cfg2(tol=1e-6)
    s = capi.BatchSolver(cfg, B, device=0)
    (count, typ, par), found = s.costmap_obstacles(cost, origin, res, pose, 0.3, M)
    assert count.max() > 100 and (found <= M).all()
    data = dict(x0=pose, xf=goal, u_prev=np.zeros((B, 2)), u_prev_dt=0.2, obstacles=(count, typ, par), viapoints=None)
    s.upload(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    s.run_phase(capi.PHASE_INIT); s.run_phase(capi.PHASE_ASSOCIATE)
    X, OBS, GIDX, SC = (s.ws_read(f) for f in (capi.F_X, capi.F_OBSIDX, capi.F_OBSGIDX, capi.F_SCAL))
    rows = 0
    for b in range(B):
        o = orc.instance_from_batch(cfg, data, b)
        o.init_cold(); o.associate()
        want = o.arr("OBSIDX")
        slot = OBS[b].astype(int)
        got = np.where(slot >= 0, GIDX[b].astype(int)[np.clip(slot, 0, None)], -1)
        np.testing.assert_array_equal(got, want.astype(int))
        used = np.unique(slot[slot >= 0])
        assert len(used) == (GIDX[b] >= 0).sum() and SC[b][capi.SC_OBST_DROPPED] == 0     # every resident slot is referenced, each obstacle once
        assert len(np.unique(GIDX[b][GIDX[b] >= 0])) == len(used)
        o.L.orc_project_init(orc.C.byref(o.p), o.ws)
        np.testing.assert_allclose(X[b], o.arr("X"), rtol=0, atol=1e-12)
        rows += (want >= 0).sum()
    assert rows > 20 * B
    s.close()
    # whole solves, fused and phased
    ref = orc.step_batch(cfg, data, n_threads=8)
    for mode in (capi.SOLVE_FUSED, capi.SOLVE_PHASED):
        s = capi.BatchSolver(cfg, B, device=0)
        s.set_option(capi.OPT_SOLVE_MODE, mode)
        out = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
        assert (out["status"] == ref["status"]).mean() >= 0.8
        both = (out["status"] == 0) & (ref["status"] == 0)
        assert both.sum() >= B // 2
        du = np.abs(out["u_seq"][both] - ref["u_seq"][both]).reshape(both.sum(), -1).max(axis=1)
        assert (du < U_TOL).mean() >= 0.8
        # a second, warm step with the same lists
        out2 = s.step(out["x_seq"][:, 1], data["xf"], out["u_seq"][:, 0], 0.2, data["obstacles"], None)
        assert (out2["status"][both] == 0).mean() >= 0.8
        s.close()
    # the chained entry point (maps in, controls out; the lists never leave the device) gives the same results bit for bit
    s = capi.BatchSolver(cfg, B, device=0)
    out = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    s.close()
    s = capi.BatchSolver(cfg, B, device=0)
    outc = s.step_from_costmaps(pose, goal, cost, origin, res, 0.3, M, u_prev=data["u_prev"], u_prev_dt=0.2)
    np.testing.assert_array_equal(outc["obst_found"], found)
    np.testing.assert_array_equal(outc["status"], out["status"])
    np.testing.assert_array_equal(outc["u_seq"], out["u_seq"])
    s.close()
    # the queue entry point takes the same lists
    s = capi.BatchSolver(cfg, B, device=0)
    outq = s.solve_stream(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    both = (outq["status"] == 0) & (ref["status"] == 0)
    assert both.sum() >= B // 2
    s.close()


def test_resident_list_overflow_is_counted(cuda_lib):
    """a map so dense that the union of the selected obstacles exceeds the resident list: rows are dropped, counted, and the
    solve still ends in a defined status"""
    B, M = 4, 2048
    cost, origin, res, pose, goal = cm.costmap_scene(B, 0.12, 12, ahead=4.5)
    cfg = configs.cfg2(tol=1e-6)
    cfg.k_max_obstacles_per_stage = 8
    s = capi.BatchSolver(cfg, B, device=0)
    (count, typ, par), found = s.costmap_obstacles(cost, origin, res, pose, 0.3, M)
    assert count.max() > 1000
    s.upload(pose, goal, None, 0.2, (count, typ, par), None)
    s.run_phase(capi.PHASE_INIT); s.run_phase(capi.PHASE_ASSOCIATE)
    SC, G, O = (s.ws_read(f) for f in (capi.F_SCAL, capi.F_OBSGIDX, capi.F_OBSIDX))
    assert (SC[:, capi.SC_OBST_DROPPED] > 0).any()
    full = SC[:, capi.SC_OBST_DROPPED] > 0
    assert ((G >= 0).sum(axis=1)[full] == 64).all() and O.max() <= 63
    out = s.step(pose, goal, None, 0.2, (count, typ, par), None)
    assert np.isin(out["status"], [0, 1, 2]).all() and np.isfinite(out["u_seq"][out["status"] == 0]).all()
    s.close()


def test_execution_options_do_not_change_results(cuda_lib):
    """MPCB200_OPT_SM_PHASE_SYNC (phase alignment of the CTAs that share an SM: off / three gates / two gates),
    MPCB200_OPT_CTAS_PER_SM and MPCB200_OPT_ORDER_BY_HISTORY (queue longest-first by the previous solve's iteration counts) only
    change WHEN a CTA runs WHICH instance: every instance gets bit for bit the same result.  The batch is large enough for
    several CTAs per SM and a second wave, so the gates really wait and the order really matters; every solver runs the batch
    twice (cold) so that the second solve has a history."""
    cfg = configs.cfg2(tol=1e-6)
    B = 900
    data = configs.generate(2, B)
    ref = None
    times = {}
    for sync, cap, order in ((0, 0, 0), (1, 0, 0), (2, 0, 0), (1, 2, 1), (-1, 0, 1), (-1, 0, 0)):
        s = capi.BatchSolver(cfg, B, device=0)
        s.set_option(capi.OPT_SM_PHASE_SYNC, sync)
        s.set_option(capi.OPT_CTAS_PER_SM, cap)
        s.set_option(capi.OPT_ORDER_BY_HISTORY, order)
        for rep in range(2):
            s.reset()
            out = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
            st = s.stats()
            if sync > 0:
                assert st["gate_ms"] > 0.0
            if sync == 0:
                assert st["gate_ms"] == 0.0
            if ref is None:
                ref = out
            else:
                for k in ("status", "iters", "u_seq", "x_seq", "dt", "kkt_err"):
                    np.testing.assert_array_equal(out[k], ref[k])
        times[(sync, cap, order)] = out["solve_time_s"]
        # a queue through the aligned kernel as well
        if sync == 1 and cap == 0:
            q = s.solve_stream(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
            np.testing.assert_array_equal(q["u_seq"], ref["u_seq"])
        s.close()
    assert (ref["status"] == 0).mean() > 0.95
    # with the history the second solve starts its longest instances first: it must not be clearly slower than index order
    # (loose bound: a timing, not a result)
    assert times[(-1, 0, 1)] <= 1.3 * times[(-1, 0, 0)]


def test_queue_job_leaves_resident_batch_alone(cuda_lib):
    """The batch and the queue job have inputs of their own: a queue solve without obstacles and with another u_prev_dt
    between two cold solves of the resident batch does not change what the resident batch is solved with."""
    cfg = configs.cfg2(tol=1e-6)
    B = 64
    data = configs.generate(2, B)
    other = configs.generate(2, B, first=B)
    s = capi.BatchSolver(cfg, B, device=0)
    s.upload(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], None)
    s.solve_resident(cold=True)
    r1 = s.fetch()
    s.solve_stream(other["x0"], other["xf"], other["u_prev"], other["u_prev_dt"] + 0.1, None, None)
    s.solve_resident(cold=True)
    r2 = s.fetch()
    s.close()
    for k in ("status", "iters", "u_seq", "x_seq", "dt", "kkt_err"):
        np.testing.assert_array_equal(r2[k], r1[k], err_msg=k)
