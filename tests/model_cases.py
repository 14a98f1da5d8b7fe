"""Cases of the phase tests of the robot models, footprints and via-point objectives (tests/test_model_phases.py on the CPU,
tests/test_gpu_model_phases.py on the CUDA phase kernels).

CASES: name -> (configuration(n), data(B, n), the kernel keys (model, problem) of a default launch).  Every case reaches device
code that the BASELINE configurations leave out: the front-drive car and the kinematic bicycle (dynamics_derivs and the
inversion of init_controls_stage), the circular, two-circles and line footprints and the degenerate polygons of one and two
vertices (footprint_distance_point / footprint_distance_line), the minimum_time_via_points objective with ordered association and
an orientation weight (the device's warp argmin in dev_associate), five outer iterations (re-association from a solved
trajectory) and a scene turned by pi, whose headings cross the +-pi seam.

EDGES: geometric edge states.  The pose of one stage is put at dyadic coordinates relative to an obstacle that stage is
associated with (the obstacles themselves on a dyadic grid), with theta = 0, so that the distance arithmetic is exact: a
different branch on the two sides (the first of equal minima wins, with a strict <) shows as a difference of the size of the
record itself, not of rounding."""
import math

import numpy as np

import linesearch_cases as lc
from mpc_local_planner_b200 import capi, configs
from parity import GEN, UNI, UNI_QF


# ---- robot models (the bounds of test_gpu_variants.test_robot_models) ----
def _robot(robot, objective):
    def f(n=None):
        if objective == "quadratic":
            c = configs.cfg2(n or 50, tol=1e-8)
        else:   # minimum time: free dt, fixed final state
            c = configs.cfg3(n or 40, tol=1e-8)
            c.footprint_type = capi.FOOTPRINT_POINT
        if robot == "front":
            c.robot_type = capi.ROBOT_SIMPLE_CAR_FRONT
            c.wheelbase = 0.4
        else:
            c.robot_type = capi.ROBOT_KIN_BICYCLE
            c.length_rear, c.length_front = 0.2, 0.25
        c.u_lb[:] = [-0.2, -1.2]
        c.u_ub[:] = [0.4, 1.2]
        c.du_lb[:] = [-0.5, -0.5]
        c.du_ub[:] = [0.5, 0.5]
        return c
    return f


# ---- footprints (the parameters of test_gpu_variants.test_footprint_models) ----
def _footprint(kind, params=None):
    def f(n=None):
        c = configs.cfg2(n or 50, tol=1e-8)
        if kind == "circular":
            c.footprint_type = capi.FOOTPRINT_CIRCULAR
            c.footprint_params[0] = 0.15
            c.min_obstacle_dist = 0.1
        elif kind == "two_circles":
            c.footprint_type = capi.FOOTPRINT_TWO_CIRCLES
            c.footprint_params[:] = params or [0.2, 0.12, 0.15, 0.1]
            c.min_obstacle_dist = 0.1
        else:
            c.footprint_type = capi.FOOTPRINT_LINE
            c.footprint_params[:] = params or [-0.15, 0.0, 0.2, 0.0]
            c.min_obstacle_dist = 0.15
        return c
    return f


def _polygon(vertices):
    """the car-like minimum-time problem of cfg 3 with a degenerate polygon: one vertex (a point off the origin) or two (a
    segment; the polygon's closing edge is not repeated)"""
    def f(n=None):
        c = configs.cfg3(n or 40, tol=1e-8)
        c.n_poly = len(vertices)
        for i, (x, y) in enumerate(vertices):
            c.poly_xy[2 * i], c.poly_xy[2 * i + 1] = x, y
        return c
    return f


# ---- the minimum_time_via_points objective (test_gpu_variants.test_minimum_time_via_points_objective) ----
def _via_points(ordered, ori_weight):
    def f(n=None):
        c = configs.cfg1(tol=1e-8)
        c.n = n or 30
        c.objective = capi.OBJ_MINIMUM_TIME_VIA_POINTS
        c.vp_position_weight = 1.5
        c.vp_orientation_weight = ori_weight
        c.vp_ordered = ordered
        c.du_lb[:] = [-0.3, -0.4]
        c.du_ub[:] = [0.3, 0.4]
        c.min_obstacle_dist = 0.2
        c.k_max_obstacles_per_stage = 5
        return c
    return f


def _reversed_via_points(B, n=None):
    """the via-point list in reverse order of the path, headings along the start -> goal line: ordered association then differs
    from the closest-pose association"""
    d = configs.generate(4, B)
    vc, vp = d["viapoints"]
    vp = vp[:, ::-1].copy()
    vp[:, :, 2] = np.arctan2(d["xf"][:, 1], d["xf"][:, 0])[:, None]
    d["viapoints"] = (vc, vp)
    return d


def _five_outer(n=None):
    c = configs.cfg1(tol=1e-8)
    c.n = n or 30
    c.outer_iterations = 5
    c.min_obstacle_dist = 0.25
    c.k_max_obstacles_per_stage = 4
    return c


def _wrap(a):
    return (np.asarray(a) + np.pi) % (2 * np.pi) - np.pi


def rotated_by_pi(data):
    """the scene turned by pi about the origin: start and goal headings (within +-pi/4 and +-pi/2 of 0 before) lie near +-pi,
    and the path between them crosses the seam"""
    out = dict(data)
    for key in ("x0", "xf"):
        x = data[key].copy()
        x[:, :2] *= -1.0
        x[:, 2] = _wrap(x[:, 2] + np.pi)
        out[key] = x
    cnt, typ, par = (a.copy() for a in data["obstacles"])
    par[:, :, 0:4] *= -1.0
    par[:, :, 5:7] *= -1.0
    out["obstacles"] = (cnt, typ, par)
    return out


def _gen(cid, transform=None):
    def f(B, n=None):
        d = configs.generate(cid, B, n=n if cid == 5 else None)
        return transform(d) if transform else d
    return f


_LINES = configs.with_line_obstacles

# name -> (configuration(n), data(B, n), kernel keys)
CASES = {
    "front_quadratic": (_robot("front", "quadratic"), _gen(2), GEN),
    "front_min_time": (_robot("front", "min_time"), _gen(3), GEN),
    "bicycle_quadratic": (_robot("bicycle", "quadratic"), _gen(2), GEN),
    "bicycle_min_time": (_robot("bicycle", "min_time"), _gen(3), GEN),
    "circular": (_footprint("circular"), _gen(2), GEN),
    "circular_lines": (_footprint("circular"), _gen(2, _LINES), GEN),
    "two_circles": (_footprint("two_circles"), _gen(2), GEN),
    "two_circles_lines": (_footprint("two_circles"), _gen(2, _LINES), GEN),
    "line": (_footprint("line"), _gen(2), GEN),
    "line_lines": (_footprint("line"), _gen(2, _LINES), GEN),
    "polygon_1": (_polygon([[0.1, 0.05]]), _gen(3, _LINES), GEN),
    "polygon_2": (_polygon([[0.25, 0.0], [-0.2, 0.0]]), _gen(3, _LINES), GEN),
    "vp_unordered": (_via_points(0, 0.0), _reversed_via_points, UNI),
    "vp_ordered": (_via_points(1, 0.0), _reversed_via_points, UNI),
    "vp_unordered_orientation": (_via_points(0, 0.3), _reversed_via_points, UNI),
    "vp_ordered_orientation": (_via_points(1, 0.3), _reversed_via_points, UNI),
    "cfg4_ordered_orientation": (lc.CASES["vp_ordered_orientation"][0], _gen(4), UNI_QF),
    "five_outer": (_five_outer, _gen(2), UNI),
    "rotated_pi": (lambda n=None: configs.cfg2(n or 50, tol=1e-8), _gen(2, rotated_by_pi), UNI_QF),
}
# instance of each batch the single-instance tests use
INSTANCE = 1


def case(name, n=None, B=None):
    make_cfg, make_data, keys = CASES[name]
    return make_cfg(n), make_data(B or INSTANCE + 1, n), keys


def has_viapoints(cfg):
    return cfg.objective == capi.OBJ_MINIMUM_TIME_VIA_POINTS or cfg.vp_attraction_with_quadratic


# ---- geometric edge states ----
def _dyadic(a, q=1.0 / 16.0):
    return np.round(np.asarray(a) / q) * q


def _vertical_lines(par, typ, b):
    """every line obstacle of instance b a vertical segment of length 1 through its (dyadic) midpoint"""
    for j in np.flatnonzero(typ[b] == capi.OBST_LINE):
        c = _dyadic(0.5 * (par[b, j, 0:2] + par[b, j, 2:4]))
        par[b, j, 0:4] = [c[0], c[1] - 0.5, c[0], c[1] + 0.5]


def _horizontal_lines(par, typ, b):
    for j in np.flatnonzero(typ[b] == capi.OBST_LINE):
        c = _dyadic(0.5 * (par[b, j, 0:2] + par[b, j, 2:4]))
        par[b, j, 0:4] = [c[0] - 0.5, c[1], c[0] + 0.5, c[1]]


def _zero_length_lines(par, typ, b):
    for j in np.flatnonzero(typ[b] == capi.OBST_LINE):
        c = _dyadic(0.5 * (par[b, j, 0:2] + par[b, j, 2:4]))
        par[b, j, 0:4] = [c[0], c[1], c[0], c[1]]


# robot-frame offsets q = R(theta)'(w - p) of the obstacle point from the stage's pose (theta = 0: q = w - p)
def _at(qx, qy, th=0.0):
    return lambda w: (w[0] - qx, w[1] - qy, th)


# line footprint of the edge states: a segment from (-1/4, 0) to (1/4, 0)
_LINE_FP = [-0.25, 0.0, 0.25, 0.0]
_TIE_FP = [0.25, 0.125, 0.25, 0.125]

# name -> (configuration(n), the change of the obstacle data of the instance, the obstacle type the stage is associated with,
#          the pose of the stage from the obstacle's first point, or a change of the stage's controls)
EDGES = {
    # the obstacle on the perpendicular bisector of the two circles: equal distances, the first circle wins
    "two_circles_tie": (_footprint("two_circles", _TIE_FP), None, capi.OBST_POINT, _at(0.0, 0.5)),
    "two_circles_tie_circle_obstacle": (_footprint("two_circles", _TIE_FP), None, capi.OBST_CIRCLE, _at(0.0, -0.5)),
    # projections onto the line footprint exactly at t = 1 and t = 0
    "line_endpoint_t1": (_footprint("line", _LINE_FP), None, capi.OBST_POINT, _at(0.25, 0.5)),
    "line_endpoint_t0": (_footprint("line", _LINE_FP), None, capi.OBST_CIRCLE, _at(-0.25, -0.5)),
    # the obstacle on the footprint segment / at the circle's centre: rho = 0, the 1e-12 clamp
    "line_on_feature": (_footprint("line", _LINE_FP), None, capi.OBST_POINT, _at(0.125, 0.0)),
    "circular_on_centre": (_footprint("circular"), None, capi.OBST_CIRCLE, _at(0.0, 0.0)),
    # a line obstacle crossing the line footprint at both midpoints: distance 0, zero derivatives
    "line_crossing": (_footprint("line", _LINE_FP), _vertical_lines, capi.OBST_LINE, _at(0.0, -0.5)),
    # a line obstacle parallel to the line footprint (den = 0): both vertices at the same distance to its interior
    "line_parallel": (_footprint("line", _LINE_FP), _horizontal_lines, capi.OBST_LINE, _at(-0.5, -0.25)),
    # a line obstacle of zero length: the point-obstacle path from its first point
    "line_zero_length": (_footprint("line", _LINE_FP), _zero_length_lines, capi.OBST_LINE, _at(0.5, 0.25)),
    # headings on the seam
    "heading_pi": (_footprint("line", _LINE_FP), None, capi.OBST_POINT, _at(0.0, 0.5, math.pi)),
    "heading_minus_pi": (_footprint("line", _LINE_FP), None, capi.OBST_POINT, _at(0.125, -0.5, -math.pi)),
}
# name -> (robot case, the steering control of the stage): controls at the steering bound
STEERING_EDGES = {
    "front_steering_upper": ("front_quadratic", "ub"),
    "front_steering_lower": ("front_min_time", "lb"),
    "bicycle_steering_upper": ("bicycle_min_time", "ub"),
    "bicycle_steering_lower": ("bicycle_quadratic", "lb"),
}
EDGE_ITERATE = 3


def edge_data(name, B):
    """the batch of an edge state: the obstacles of cfg 2 on a dyadic grid with dyadic radii; every other one a point or a
    line where the state is about points or lines"""
    make_cfg, change, otype, _ = EDGES[name]
    d = configs.generate(2, B)
    if otype == capi.OBST_LINE:
        d = configs.with_line_obstacles(d)
    cnt, typ, par = (a.copy() for a in d["obstacles"])
    if otype == capi.OBST_POINT:   # (the generated obstacles are circles)
        typ[:, 1::2] = capi.OBST_POINT
        par[:, 1::2, 4] = 0.0
    par[:, :, 0:5] = _dyadic(par[:, :, 0:5])
    if change is not None:
        for b in range(B):
            change(par, typ, b)
    d["obstacles"] = (cnt, typ, par)
    return make_cfg(), d


def place_stage(o, otype, pose, b_types, b_params):
    """Put the pose of the first inner stage associated with an obstacle of type otype at pose(first point of the obstacle);
    returns the stage.  o: an oracle instance after the association; b_types / b_params: the instance's obstacle list."""
    OBS = o.arr("OBSIDX")
    N = o.N
    for k in range(1, N - 1):
        for j in OBS[:, k]:
            j = int(j)
            if j >= 0 and b_types[j] == otype:
                o.arr("X")[:, k] = pose(b_params[j])
                return k
    raise AssertionError(f"no stage is associated with an obstacle of type {otype}")


def steer_stage(o, cfg, bound):
    """the steering control of the middle stage (and of the next one) at its bound"""
    k = o.N // 2
    v = cfg.u_ub[1] if bound == "ub" else cfg.u_lb[1]
    o.arr("U")[1, k] = v
    o.arr("U")[1, k + 1] = v
    return k


VP_CASES = [nm for nm in CASES if has_viapoints(CASES[nm][0]())]


def via_point_tie(o, data, b):
    """Stages k, k + 7 and (N > 40) k + 32 of an oracle iterate put exactly on the first via-point of the list: equal distances
    in the association's argmin over the stages, in two lanes of the device's warp and (k + 32) twice in one lane.  The first
    stage must win.  Returns the stages."""
    vp = data["viapoints"][1][b][0]
    k = 4
    stages = [k, k + 7] + ([k + 32] if o.N > 40 else [])
    for kk in stages:
        o.arr("X")[:2, kk] = vp[:2]
    return stages


def standing_plan(cfg, data, b):
    """an initial plan (x_init) whose first stages stand still while the heading turns: |v| = 0 at those stages, the branch of
    init_controls_stage that does not invert the dynamics (|v| <= 1e-3)"""
    N = int(cfg.n)
    x0, xf = data["x0"][b], data["xf"][b]
    t = np.linspace(0.0, 1.0, N)
    X = np.stack([x0[0] + t * (xf[0] - x0[0]), x0[1] + t * (xf[1] - x0[1]), x0[2] + t * _wrap(xf[2] - x0[2])], axis=1)
    X[:4, :2] = x0[:2]
    X[:4, 2] = x0[2] + 0.05 * np.arange(4)
    X[N // 2, :2] = X[N // 2 - 1, :2] + 5e-4 * cfg.dt_ref   # |v| just below the threshold
    return X
