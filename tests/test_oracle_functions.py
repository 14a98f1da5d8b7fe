"""The CPU oracle's restatement of the reference's elementary functions + analytic derivatives (CPU, no GPU)."""
import ctypes as C
import math

import numpy as np
import pytest

import costmap_cases as cm
import dense_kkt as dk
from mpc_local_planner_b200 import capi, configs


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def test_normalize_theta_matches_reference_rule(orc):
    """math_utils.h:81-91: identity on [-pi, pi), else floor-mod then +-2pi."""
    L = orc.lib()
    for th in (-math.pi, -3.0, 0.0, 3.0, math.pi - 1e-12):
        assert L.orc_normalize_theta(th) == th
    assert L.orc_normalize_theta(math.pi) == pytest.approx(-math.pi)
    rng = np.random.default_rng(0)
    for th in rng.uniform(-50, 50, 200):
        w = L.orc_normalize_theta(th)
        assert -math.pi <= w < math.pi
        assert math.isclose(math.sin(w), math.sin(th), abs_tol=1e-12) and math.isclose(math.cos(w), math.cos(th), abs_tol=1e-12)
    assert L.orc_interpolate_angle(3.0, -3.0, 0.5) == pytest.approx(L.orc_normalize_theta(3.0 + 0.5 * (2 * math.pi - 6.0)))


@pytest.mark.parametrize("robot", [capi.ROBOT_UNICYCLE, capi.ROBOT_SIMPLE_CAR, capi.ROBOT_SIMPLE_CAR_FRONT, capi.ROBOT_KIN_BICYCLE])
def test_dynamics_values_and_derivatives(orc, robot):
    """systems/*.h dynamics; analytic Jacobian/Hessian vs central differences."""
    L = orc.lib()
    cfg = capi.default_config()
    cfg.robot_type = robot
    cfg.wheelbase, cfg.length_rear, cfg.length_front = 0.4, 0.7, 0.9
    rng = np.random.default_rng(robot)
    for _ in range(10):
        x = rng.uniform(-2, 2, 3); u = np.array([rng.uniform(-0.3, 0.5), rng.uniform(-1.0, 1.0)]); nu = rng.standard_normal(3)
        f = np.zeros(3); J = np.zeros(9); Hc = np.zeros(6); f2 = np.zeros(3)
        L.orc_dynamics(C.byref(cfg), _dp(x), _dp(u), _dp(f2))
        L.orc_dynamics_derivs(C.byref(cfg), _dp(x), _dp(u), _dp(nu), _dp(f), _dp(J), _dp(Hc))
        np.testing.assert_allclose(f, f2, atol=1e-15)
        th, v, w = x[2], u[0], u[1]
        if robot == capi.ROBOT_UNICYCLE:
            np.testing.assert_allclose(f, [v * math.cos(th), v * math.sin(th), w], atol=1e-15)
        elif robot == capi.ROBOT_SIMPLE_CAR:
            np.testing.assert_allclose(f, [v * math.cos(th), v * math.sin(th), v * math.tan(w) / 0.4], atol=1e-14)
        elif robot == capi.ROBOT_SIMPLE_CAR_FRONT:
            np.testing.assert_allclose(f, [v * math.cos(th), v * math.sin(th), v * math.sin(w) / 0.4], atol=1e-14)
        else:
            beta = math.atan(0.7 / 1.6 * math.tan(w))
            np.testing.assert_allclose(f, [v * math.cos(th + beta), v * math.sin(th + beta), v * math.sin(beta) / 0.7], atol=1e-14)

        def fq(q):
            xx = x.copy(); xx[2] = q[0]; uu = np.array([q[1], q[2]]); o = np.zeros(3)
            L.orc_dynamics(C.byref(cfg), _dp(xx), _dp(uu), _dp(o)); return o
        q0 = np.array([th, v, w]); h = 1e-6
        Jfd = np.zeros((3, 3))
        for i in range(3):
            e = np.zeros(3); e[i] = h
            Jfd[:, i] = (fq(q0 + e) - fq(q0 - e)) / (2 * h)
        np.testing.assert_allclose(J.reshape(3, 3), Jfd, atol=1e-8)
        # Hessian of nu^T f
        def g(q): return nu @ fq(q)
        H = np.zeros((3, 3)); hh = 1e-4
        for i in range(3):
            for j in range(3):
                ei = np.zeros(3); ej = np.zeros(3); ei[i] = hh; ej[j] = hh
                H[i, j] = (g(q0 + ei + ej) - g(q0 + ei - ej) - g(q0 - ei + ej) + g(q0 - ei - ej)) / (4 * hh * hh)
        Hpk = np.array([[Hc[0], Hc[1], Hc[2]], [Hc[1], Hc[3], Hc[4]], [Hc[2], Hc[4], Hc[5]]])
        np.testing.assert_allclose(Hpk, H, atol=2e-6)


def test_defect_is_dt_times_reference_defect(orc):
    """fd_collocation_se2.h:54-69 as coded (divides by dt) vs the multiplied form used by the solvers."""
    L = orc.lib()
    cfg = capi.default_config()
    rng = np.random.default_rng(1)
    for _ in range(50):
        x1 = rng.uniform(-3, 3, 3); x2 = x1 + rng.uniform(-0.3, 0.3, 3); u = rng.uniform(-0.4, 0.4, 2); dt = rng.uniform(0.05, 1.0)
        x2[2] += rng.integers(-2, 3) * 2 * math.pi  # periodic in theta
        e_ref = np.zeros(3); e = np.zeros(3)
        L.orc_defect_reference(C.byref(cfg), _dp(x1), _dp(u), _dp(x2), dt, _dp(e_ref))
        L.orc_defect(C.byref(cfg), _dp(x1), _dp(u), _dp(x2), dt, _dp(e))
        np.testing.assert_allclose(e, dt * e_ref, atol=1e-13)


def _fp_cfg(kind):
    c = capi.default_config()
    c.footprint_type = kind
    if kind == capi.FOOTPRINT_CIRCULAR:
        c.footprint_params[0] = 0.25
    elif kind == capi.FOOTPRINT_TWO_CIRCLES:
        c.footprint_params[:] = [0.2, 0.15, 0.25, 0.2]
    elif kind == capi.FOOTPRINT_LINE:
        c.footprint_params[:] = [-0.1, 0.05, 0.4, -0.02]
    elif kind == capi.FOOTPRINT_POLYGON:
        c.n_poly = len(configs.CARLIKE_POLYGON)
        for i, (x, y) in enumerate(configs.CARLIKE_POLYGON):
            c.poly_xy[2 * i], c.poly_xy[2 * i + 1] = x, y
    return c


@pytest.mark.parametrize("kind", [capi.FOOTPRINT_POINT, capi.FOOTPRINT_CIRCULAR, capi.FOOTPRINT_TWO_CIRCLES, capi.FOOTPRINT_LINE,
                                  capi.FOOTPRINT_POLYGON])
def test_footprint_distance(orc, kind):
    """teb RobotFootprintModel::calculateDistance semantics (SURVEY App. B.3): values by brute force in the world frame,
    gradient / Hessian of the active feature by finite differences."""
    L = orc.lib()
    cfg = _fp_cfg(kind)
    rng = np.random.default_rng(kind)

    def dist(pose, otype, op):
        return L.orc_footprint_distance(C.byref(cfg), _dp(np.ascontiguousarray(pose)), otype, _dp(op), None, None)

    def brute(pose, otype, op):
        c, s = math.cos(pose[2]), math.sin(pose[2])
        R = np.array([[c, -s], [s, c]])
        o = op[:2]
        def seg_d(a, b):
            a = pose[:2] + R @ a; b = pose[:2] + R @ b
            ab = b - a; sq = ab @ ab
            t = 0.0 if sq == 0 else min(1.0, max(0.0, ((o - a) @ ab) / sq))
            return np.linalg.norm(o - (a + t * ab))
        if kind == capi.FOOTPRINT_POINT:
            d = np.linalg.norm(o - pose[:2])
        elif kind == capi.FOOTPRINT_CIRCULAR:
            d = np.linalg.norm(o - pose[:2]) - 0.25
        elif kind == capi.FOOTPRINT_TWO_CIRCLES:
            h = np.array([c, s])
            d = min(np.linalg.norm(o - (pose[:2] + 0.2 * h)) - 0.15, np.linalg.norm(o - (pose[:2] - 0.25 * h)) - 0.2)
        elif kind == capi.FOOTPRINT_LINE:
            d = seg_d(np.array([-0.1, 0.05]), np.array([0.4, -0.02]))
        else:
            P = np.array(configs.CARLIKE_POLYGON)
            d = min(seg_d(P[i], P[(i + 1) % len(P)]) for i in range(len(P)))
        return d - (op[4] if otype == capi.OBST_CIRCLE else 0.0)

    for _ in range(40):
        pose = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(-3, 3)])
        op = np.array([rng.uniform(-2, 2), rng.uniform(-2, 2), 0, 0, rng.uniform(0.05, 0.3)])
        otype = int(rng.integers(0, 2))
        d = dist(pose, otype, op)
        assert d == pytest.approx(brute(pose, otype, op), abs=1e-12)
        g = np.zeros(3); H = np.zeros(6)
        L.orc_footprint_distance(C.byref(cfg), _dp(pose), otype, _dp(op), _dp(g), _dp(H))
        h = 1e-6
        gfd = np.array([(dist(pose + h * e, otype, op) - dist(pose - h * e, otype, op)) / (2 * h) for e in np.eye(3)])
        np.testing.assert_allclose(g, gfd, atol=1e-7)
        hh = 1e-4
        Hfd = np.zeros((3, 3))
        for i in range(3):
            for j in range(3):
                ei, ej = np.eye(3)[i] * hh, np.eye(3)[j] * hh
                Hfd[i, j] = (dist(pose + ei + ej, otype, op) - dist(pose + ei - ej, otype, op) - dist(pose - ei + ej, otype, op)
                             + dist(pose - ei - ej, otype, op)) / (4 * hh * hh)
        Hm = np.array([[H[0], H[1], H[2]], [H[1], H[3], H[4]], [H[2], H[4], H[5]]])
        if np.abs(Hfd - Hm).max() > 1e-4:  # feature switch inside the FD stencil: skip (piecewise smooth distance)
            continue
        np.testing.assert_allclose(Hm, Hfd, atol=1e-4)


@pytest.mark.parametrize("kind", [capi.FOOTPRINT_POINT, capi.FOOTPRINT_CIRCULAR, capi.FOOTPRINT_TWO_CIRCLES, capi.FOOTPRINT_LINE,
                                  capi.FOOTPRINT_POLYGON])
def test_footprint_distance_to_line_obstacle(orc, kind):
    """LineObstacle (SURVEY App. B.3): value by brute force (teb's segment / segment rule written independently with
    numpy), gradient / Hessian by finite differences."""
    L = orc.lib()
    cfg = _fp_cfg(kind)
    rng = np.random.default_rng(100 + kind)

    def dist(pose, op):
        return L.orc_footprint_distance(C.byref(cfg), _dp(np.ascontiguousarray(pose)), capi.OBST_LINE, _dp(op), None, None)

    def pt_seg(q, a, b):
        ab = b - a; sq = ab @ ab
        t = 0.0 if sq == 0 else min(1.0, max(0.0, ((q - a) @ ab) / sq))
        return np.linalg.norm(q - (a + t * ab))

    def cross(o, a, b):
        return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])

    def seg_seg(a, b, c_, d):
        if (a == b).all():
            return pt_seg(a, c_, d)
        # proper crossing via orientation tests
        if cross(a, b, c_) * cross(a, b, d) <= 0 and cross(c_, d, a) * cross(c_, d, b) <= 0 and abs(cross(a, b, c_)) + abs(cross(a, b, d)) > 0:
            return 0.0
        return min(pt_seg(a, c_, d), pt_seg(b, c_, d), pt_seg(c_, a, b), pt_seg(d, a, b))

    def features():
        if kind == capi.FOOTPRINT_POINT:
            return [(np.zeros(2), np.zeros(2), 0.0)]
        if kind == capi.FOOTPRINT_CIRCULAR:
            return [(np.zeros(2), np.zeros(2), 0.25)]
        if kind == capi.FOOTPRINT_TWO_CIRCLES:
            return [(np.array([0.2, 0.0]),) * 2 + (0.15,), (np.array([-0.25, 0.0]),) * 2 + (0.2,)]
        if kind == capi.FOOTPRINT_LINE:
            return [(np.array([-0.1, 0.05]), np.array([0.4, -0.02]), 0.0)]
        P = np.array(configs.CARLIKE_POLYGON)
        return [(P[i], P[(i + 1) % len(P)], 0.0) for i in range(len(P))]

    def brute(pose, op):
        c, s = math.cos(pose[2]), math.sin(pose[2])
        R = np.array([[c, -s], [s, c]])
        a, b = op[0:2], op[2:4]
        return min(seg_seg(pose[:2] + R @ f0, pose[:2] + R @ f1, a, b) - r for f0, f1, r in features())

    checked = 0
    for _ in range(60):
        pose = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(-3, 3)])
        a = rng.uniform(-2, 2, 2)
        ang = rng.uniform(0, 2 * math.pi)
        b = a + rng.uniform(0.2, 2.0) * np.array([math.cos(ang), math.sin(ang)])
        op = np.array([a[0], a[1], b[0], b[1], 0.0])
        d = dist(pose, op)
        assert d == pytest.approx(brute(pose, op), abs=1e-12)
        if d < 1e-3:
            continue  # crossing / touching: the distance is clamped at 0 there
        g = np.zeros(3); H = np.zeros(6)
        L.orc_footprint_distance(C.byref(cfg), _dp(pose), capi.OBST_LINE, _dp(op), _dp(g), _dp(H))
        h = 1e-6
        gfd = np.array([(dist(pose + h * e, op) - dist(pose - h * e, op)) / (2 * h) for e in np.eye(3)])
        np.testing.assert_allclose(g, gfd, atol=1e-7)
        hh = 1e-4
        Hfd = np.zeros((3, 3))
        for i in range(3):
            for j in range(3):
                ei, ej = np.eye(3)[i] * hh, np.eye(3)[j] * hh
                Hfd[i, j] = (dist(pose + ei + ej, op) - dist(pose + ei - ej, op) - dist(pose - ei + ej, op) + dist(pose - ei - ej, op)) / (4 * hh * hh)
        Hm = np.array([[H[0], H[1], H[2]], [H[1], H[3], H[4]], [H[2], H[4], H[5]]])
        if np.abs(Hfd - Hm).max() > 1e-4:  # feature switch inside the FD stencil (piecewise smooth distance)
            continue
        np.testing.assert_allclose(Hm, Hfd, atol=1e-4)
        checked += 1
    assert checked >= 30



@pytest.mark.parametrize("rule", ["left_sum", "trapezoidal"])
def test_integral_form_objective_is_the_edge_sum(orc, rule):
    """The objective of the integral form against the sum of the reference's per-interval cost edges written out in numpy
    (finite_differences_grid_se2.cpp:57-72): left sum dt l(x_k, u_k); trapezoid dt/2 (l(x_k, u_k) + l(x_{k+1}, u_k))."""
    inst, cfg = dk.random_iterate(orc, 24 if rule == "trapezoidal" else 21, 1, 3)
    inst.eval()
    N = inst.N
    X = inst.arr("X"); U = inst.arr("U"); dt = inst.arr("SCAL")[capi.SC_DT]
    xf = configs.generate(2, 2)["xf"][1]
    Q = np.array(cfg.Q[:]).reshape(3, 3); R = np.array(cfg.R[:]).reshape(2, 2); Qf = np.array(cfg.Qf[:]).reshape(3, 3)

    def d(k):
        v = X[:, k] - xf
        v[2] = (v[2] + np.pi) % (2 * np.pi) - np.pi
        return v
    l = lambda k, j: d(k) @ Q @ d(k) + U[:, j] @ R @ U[:, j]
    J = 0.0
    for k in range(N - 1):
        J += dt * l(k, k) if rule == "left_sum" else 0.5 * dt * (l(k, k) + l(k + 1, k))
    J += d(N - 1) @ Qf @ d(N - 1)
    assert abs(inst.arr("SCAL")[capi.SC_OBJ] - J) < 1e-10 * max(1.0, abs(J))


@pytest.mark.parametrize("cid", [1, 2, 3, 4, 21, 22, 23, 24, 25, 26, 27, 31, 41, 42, 43])
def test_lagrangian_gradient_and_newton_step(orc, cid):
    """Analytic Lagrangian gradient vs finite differences; the Riccati Newton step (incl. the dt border and the fixed
    terminal state) vs a dense numpy solve of the full KKT system assembled by finite differences.  Two random iterates:
    multipliers of size 1 (indefinite Hessians: the inertia test must fire) and of size 0.05 (the step is compared)."""
    compared = dk.check_gradient_and_newton_step(orc, cid, 1.0) + dk.check_gradient_and_newton_step(orc, cid, 0.05)
    assert compared >= 1



@pytest.mark.parametrize("n,n_new", [(20, 21), (20, 19), (50, 57), (33, 12), (5, 3), (3, 8)])
def test_resample_trajectory_properties(orc, n, n_new):
    """resampleTrajectory (full_discretization_grid_base_se2.cpp:440-524) against numpy's piecewise-linear interpolation of
    the old polyline at the new sample times: horizon time kept, first sample and final state carried over, headings
    interpolated on the short way round, controls taken from the old interval a new sample falls into."""
    rng = np.random.default_rng(n * 100 + n_new)
    dt = 0.37
    X = np.cumsum(rng.normal(0, 0.2, (3, n)), axis=1)
    X[2] = (X[2] + np.pi) % (2 * np.pi) - np.pi
    U = rng.normal(0, 0.3, (2, n)); U[:, n - 1] = 0
    Xn, Un, dt_new = orc.resample_trajectory(X, U, dt, n_new)
    assert abs(dt_new * (n_new - 1) - dt * (n - 1)) < 1e-12
    np.testing.assert_array_equal(Xn[:, 0], X[:, 0]); np.testing.assert_array_equal(Xn[:, -1], X[:, -1])
    np.testing.assert_array_equal(Un[:, 0], U[:, 0])
    t_old = dt * np.arange(n); t_new = dt_new * np.arange(n_new)
    for c in range(2):
        np.testing.assert_allclose(Xn[c, 1:-1], np.interp(t_new[1:-1], t_old, X[c]), atol=1e-12)
    th = np.unwrap(X[2])
    d = Xn[2, 1:-1] - np.interp(t_new[1:-1], t_old, th)
    assert np.abs((d + np.pi) % (2 * np.pi) - np.pi).max() < 1e-12
    assert (Xn[2] >= -np.pi).all() and (Xn[2] < np.pi).all()
    # controls: the old interval that ends at or after t_new (a sample exactly on an old grid point takes the interval before it)
    idx = np.minimum(np.ceil(t_new[1:-1] / dt - 1e-12).astype(int), n - 1)
    np.testing.assert_array_equal(Un[:, 1:-1], U[:, np.minimum(idx - 1, n - 2)])


@pytest.mark.parametrize("W,H", [(60, 40), (33, 77), (2, 2), (128, 3)])
def test_costmap_obstacles_against_numpy(orc, W, H):
    """updateObstacleContainerWithCostmap (mpc_local_planner_ros.cpp:474-499): the oracle's loops against a vectorised numpy
    restatement -- which cells qualify, their world coordinates, the reference's push_back order, the cut at max_out."""
    rng = np.random.default_rng(W * 1000 + H)
    cost = cm.random_costmap(rng, W, H, 0.05)
    origin = rng.uniform(-5, 5, 2); res = 0.05
    pose = np.array([origin[0] + 0.5 * W * res, origin[1] + 0.5 * H * res, rng.uniform(-np.pi, np.pi)])
    behind = 0.4
    mx, my = np.meshgrid(np.arange(W - 1), np.arange(H - 1), indexing="ij")          # [mx, my]: mx outer, my inner
    wx = origin[0] + (mx + 0.5) * res; wy = origin[1] + (my + 0.5) * res
    dx, dy = wx - pose[0], wy - pose[1]
    keep = (cost[:H - 1, :W - 1].T == 254) & ~((dx * np.cos(pose[2]) + dy * np.sin(pose[2]) < 0) & (np.hypot(dx, dy) > behind))
    want = np.stack([wx[keep], wy[keep]], -1)                                         # boolean indexing walks mx-major
    xy, found = orc.costmap_obstacles(cost, origin, res, pose, behind, max_out=10000)
    assert found == len(want)
    np.testing.assert_allclose(xy, want, atol=1e-12)
    if found > 3:
        xy3, found3 = orc.costmap_obstacles(cost, origin, res, pose, behind, max_out=3)
        assert found3 == found and len(xy3) == 3
        np.testing.assert_array_equal(xy3, xy[:3])


# ---- the independent numpy restatement (tests/golden/ocp_numpy.py, written from the reference's lines without the oracle)
#      against the oracle, function by function, on random iterates ----
def _np_problem(cfg, data, b):
    import os, sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import ocp_numpy as on
    return on, on.problem_from_batch(cfg, data, b)


@pytest.mark.parametrize("variant", ["cfg2", "cfg3_polygon", "cfg4_viapoints", "two_circles_lines", "line_footprint", "min_time_via_points_ordered", "midpoint"])
def test_numpy_restatement_agrees_with_the_oracle(orc, variant):
    """Association (StageInequalitySE2::update incl. the world-centroid side test), via-point association, obstacle rows,
    control-rate rows (the oracle keeps them multiplied by dt), collocation defects (ditto) and the objective."""
    rng = np.random.default_rng(11)
    if variant == "cfg2":
        cfg = configs.cfg2(n=20); data = configs.generate(5, 6, n=20)
    elif variant == "cfg3_polygon":
        cfg = configs.cfg3(n=16); data = configs.generate(3, 6, n=16)
    elif variant == "cfg4_viapoints":
        cfg = configs.cfg4(n=20); data = configs.generate(4, 6)
    elif variant == "two_circles_lines":
        cfg = configs.cfg2(n=16); cfg.footprint_type = capi.FOOTPRINT_TWO_CIRCLES; cfg.footprint_params[:] = [0.2, 0.12, 0.15, 0.1]
        data = configs.with_line_obstacles(configs.generate(5, 6, n=16))
    elif variant == "line_footprint":
        cfg = configs.cfg2(n=16); cfg.footprint_type = capi.FOOTPRINT_LINE; cfg.footprint_params[:] = [-0.15, 0.0, 0.2, 0.0]
        data = configs.with_line_obstacles(configs.generate(5, 6, n=16))
    elif variant == "min_time_via_points_ordered":
        cfg = configs.cfg1(); cfg.objective = capi.OBJ_MINIMUM_TIME_VIA_POINTS; cfg.vp_ordered = 1; cfg.vp_orientation_weight = 0.3
        cfg.vp_position_weight = 1.5; cfg.du_lb[:] = [-0.3, -0.4]; cfg.du_ub[:] = [0.3, 0.4]; cfg.k_max_obstacles_per_stage = 5
        data = configs.generate(4, 6)
        vc, vp = data["viapoints"]; data["viapoints"] = (vc, vp[:, ::-1].copy())
    else:
        cfg = configs.cfg2(n=16); cfg.collocation = capi.COLLOC_MIDPOINT; data = configs.generate(5, 6, n=16)
    cfg.reference_initial_guess = 1
    N = cfg.n
    for b in range(6):
        on, p = _np_problem(cfg, data, b)
        o = orc.instance_from_batch(cfg, data, b)
        o.init_cold()
        # a wiggled trajectory (so that sides, forced inclusions and the via-point association are not trivial)
        X = o.arr("X"); U = o.arr("U")
        X[:2, 1:N - 1] += rng.normal(0, 0.15, (2, N - 2)); X[2, 1:N - 1] += rng.normal(0, 0.4, N - 2)
        U[:, :N - 1] = rng.uniform(-0.15, 0.25, (2, N - 1))
        dt = float(o.arr("SCAL")[capi.SC_DT])
        if cfg.variable_dt:
            dt = 0.37; o.arr("SCAL")[capi.SC_DT] = dt
        o.associate(); o.init_duals(); o.eval()
        Xn = X.T.copy(); Un = U[:, :N - 1].T.copy()
        # association: same obstacles per stage, same order
        assoc = on.associate(cfg, Xn, p.ot, p.op, dt)
        OBS = o.arr("OBSIDX")
        for k in range(N):
            mine = assoc[k]
            theirs = [int(v) for v in OBS[:, k] if v >= 0]
            assert mine == theirs, f"{variant} instance {b} stage {k}: numpy {mine} oracle {theirs}"
        if p.vps:
            assert on.associate_viapoints(cfg, Xn, p.vps) == list(o.vp_stage()), variant
        # defects: oracle keeps e = x_k + dt f - x_{k+1} = -dt * (reference defect)
        e_np = on.defects(cfg, Xn, Un, dt).reshape(N - 1, 3)
        np.testing.assert_allclose(o.defects().T, -dt * e_np, atol=1e-12)
        # rows: obstacle rows as they are, control-rate rows multiplied by the interval length
        G = o.arr("G")
        for k in range(1, N - 1):
            for j, oi in enumerate(assoc[k]):
                row = cfg.min_obstacle_dist - on.footprint_distance(cfg, Xn[k], p.ot[oi], p.op[oi], t=k * dt)
                assert G[8 + j, k] == pytest.approx(row, abs=1e-12)
        for k in range(N):
            uk = Un[k] if k <= N - 2 else np.zeros(2)
            um = Un[k - 1] if k >= 1 else data["u_prev"][b]
            T = dt if k >= 1 else data["u_prev_dt"]
            for i in range(2):
                if cfg.du_lb[i] > -1e29:
                    assert G[4 + 2 * i, k] == pytest.approx(T * (cfg.du_lb[i] - (uk[i] - um[i]) / T), abs=1e-12)
                if cfg.du_ub[i] < 1e29:
                    assert G[5 + 2 * i, k] == pytest.approx(T * ((uk[i] - um[i]) / T - cfg.du_ub[i]), abs=1e-12)
        # objective
        vp_stage = on.associate_viapoints(cfg, Xn, p.vps) if p.vps else []
        f_np = on.objective(cfg, Xn, Un, dt, data["xf"][b], p.vps, vp_stage)
        assert o.arr("SCAL")[capi.SC_OBJ] == pytest.approx(f_np, rel=1e-12, abs=1e-12)


# ---- Controller::isPoseTrajectoryFeasible (controller.cpp:859-917): the oracle's C loop against a plain-Python restatement ----
def _py_feasible(cost, origin, res, xs, fp, inscribed, min_ang, look):
    H, W = cost.shape

    def w2m(wx, wy):
        if wx < origin[0] or wy < origin[1]:
            return None
        mx, my = int((wx - origin[0]) / res), int((wy - origin[1]) / res)
        return (mx, my) if (mx < W and my < H) else None

    def line_cost(x0, x1, y0, y1):
        dx, dy = abs(x1 - x0), abs(y1 - y0)
        x, y = x0, y0
        xi1 = xi2 = 1 if x1 >= x0 else -1
        yi1 = yi2 = 1 if y1 >= y0 else -1
        if dx >= dy:
            xi1 = 0; yi2 = 0; den = dx; num = dx // 2; numadd = dy; npx = dx
        else:
            xi2 = 0; yi1 = 0; den = dy; num = dy // 2; numadd = dx; npx = dy
        lc = 0.0
        for _ in range(npx + 1):
            c = int(cost[y, x])
            pc = -2.0 if c == 255 else (-1.0 if c == 254 else float(c))
            if pc < 0:
                return pc
            lc = max(lc, pc)
            num += numadd
            if num >= den:
                num -= den; x += xi1; y += yi1
            x += xi2; y += yi2
        return lc

    def fcost(px, py, th):
        c = w2m(px, py)
        if c is None:
            return -1.0
        if len(fp) < 3:
            v = int(cost[c[1], c[0]])
            return -2.0 if v == 255 else (-1.0 if v in (254, 253) else float(v))
        co, si = math.cos(th), math.sin(th)
        pts = [(px + (fx * co - fy * si), py + (fx * si + fy * co)) for fx, fy in fp]
        fc = 0.0
        for i in range(len(pts)):
            a, b = pts[i], pts[(i + 1) % len(pts)]
            ca, cb = w2m(*a), w2m(*b)
            if ca is None or cb is None:
                return -3.0
            lc = line_cost(ca[0], cb[0], ca[1], cb[1])
            fc = max(fc, lc)
            if lc < 0:
                return lc
        return fc

    def norm(t):
        if -math.pi <= t < math.pi:
            return t
        t = t - math.floor(t / (2 * math.pi)) * 2 * math.pi
        if t >= math.pi:
            t -= 2 * math.pi
        if t < -math.pi:
            t += 2 * math.pi
        return t
    n = len(xs)
    if n < 2:
        return False
    if look < 0 or look >= n:
        look = n - 1
    for i in range(look + 1):
        if fcost(*xs[i]) == -1.0:
            return False
        if i < look:
            drot = norm(xs[i + 1][2] - xs[i][2]); dx = xs[i + 1][0] - xs[i][0]; dy = xs[i + 1][1] - xs[i][1]
            dist = math.sqrt(dx * dx + dy * dy)
            if abs(drot) > min_ang or dist > inscribed:
                nadd = int(max(math.ceil(abs(drot) / min_ang), math.ceil(dist / inscribed))) - 1
                ix, iy, ith = xs[i]
                for _ in range(nadd):
                    ix += dx / (nadd + 1.0); iy += dy / (nadd + 1.0); ith = norm(ith + drot / (nadd + 1.0))
                    if fcost(ix, iy, ith) == -1.0:
                        return False
    return True


@pytest.mark.parametrize("footprint", ["polygon", "two_points"])
def test_pose_trajectory_feasibility_against_python(orc, footprint):
    rng = np.random.default_rng(5)
    fp = np.array(configs.CARLIKE_POLYGON) if footprint == "polygon" else np.array([[0.1, 0.0], [-0.1, 0.0]])
    seen = set()
    for look in (-1, 5):
        for cost, origin, xs in cm.feasibility_cases(rng, 40):
            a = orc.pose_trajectory_feasible(cost, origin, 0.05, xs, fp, 0.18, 0.3, look)
            b = _py_feasible(cost, origin, 0.05, [tuple(r) for r in xs], [tuple(p) for p in fp], 0.18, 0.3, look)
            assert a == b
            seen.add(a)
    assert seen == {True, False}   # the cases exercise both outcomes
