"""Per-robot model records (mpcb200_set_robot_model) for the tests: the configuration a record makes (restated from
include/mpcb200.h, the expected result of apply_robot_model), the validity rule restated on top of the geometry rule of
robot_geometry_cases, and the four model groups of a mixed fleet with their configurations, limits and geometry."""
import numpy as np

import robot_geometry_cases as rg
from mpc_local_planner_b200 import capi, configs

W = capi.MODEL_WORDS
RT, FT = capi.MOD_ROBOT_TYPE, capi.MOD_FOOTPRINT_TYPE
TYPES = [(r, f) for r in range(4) for f in range(5)]


def record(robot, footprint):
    r = np.zeros(W)
    r[RT], r[FT] = robot, footprint
    return r


def record_of(cfg):
    """the record holding the configuration's own types"""
    return record(cfg.robot_type, cfg.footprint_type)


def with_model(cfg, rec):
    """the configuration of a robot with record `rec`: its two types, every other field as in cfg"""
    c = cfg.copy()
    c.robot_type, c.footprint_type = int(rec[RT]), int(rec[FT])
    return c


def _word_ok(v, hi):
    return bool(np.isfinite(v)) and 0 <= v <= hi and v == np.floor(v)


def rule(cfg, rec, geo=None):
    """the validity rule of include/mpcb200.h restated: both words integers in range, and the robot's geometry (its record, else
    the configuration's values) valid for the record's types"""
    if not (_word_ok(rec[RT], 3) and _word_ok(rec[FT], 4)):
        return False
    c = with_model(cfg, rec)
    return rg.rule(c, rg.record_of(cfg) if geo is None else geo)


# ---- the four model groups of a mixed fleet: robot b is in group b % 4 ----
GROUPS = ("uni_circle", "car_polygon", "front_two_circles", "bicycle_line")
GROUP_TYPES = {"uni_circle": (capi.ROBOT_UNICYCLE, capi.FOOTPRINT_CIRCULAR), "car_polygon": (capi.ROBOT_SIMPLE_CAR, capi.FOOTPRINT_POLYGON),
               "front_two_circles": (capi.ROBOT_SIMPLE_CAR_FRONT, capi.FOOTPRINT_TWO_CIRCLES),
               "bicycle_line": (capi.ROBOT_KIN_BICYCLE, capi.FOOTPRINT_LINE)}
# control bounds (v, omega) of the unicycle, (v, steering angle) of the others
GROUP_U = {"uni_circle": ([-0.2, -0.6], [0.4, 0.6]), "car_polygon": ([-0.2, -1.4], [0.4, 1.4]),
           "front_two_circles": ([-0.15, -1.2], [0.35, 1.2]), "bicycle_line": ([-0.15, -0.5], [0.35, 0.5])}


def group_geometry(g):
    """the geometry record of group g: the polygon of cfg 3 (car_polygon), two circles, a line or a circle of the group's size, a
    wheelbase of 0.4 / 0.45 and the bicycle's lengths 0.2 / 0.25"""
    c3 = configs.cfg3()
    r = rg.record_of(c3)
    r[capi.GEO_WHEELBASE] = 0.45 if g == "front_two_circles" else 0.4
    r[capi.GEO_LENGTH_REAR], r[capi.GEO_LENGTH_FRONT] = 0.2, 0.25
    r[rg.FP:rg.FP + 4] = {"uni_circle": [0.25, 0.0, 0.0, 0.0], "car_polygon": [0.0, 0.0, 0.0, 0.0],
                          "front_two_circles": [0.2, 0.18, 0.1, 0.15], "bicycle_line": [0.25, 0.0, -0.1, 0.0]}[g]
    return r


def group_limits(host, g):
    """the limits record of group g on a handle: the group's control bounds, the handle's rate bounds and clearance"""
    r = np.zeros(capi.LIMIT_WORDS)
    r[capi.LIM_U_LB:capi.LIM_U_LB + 2], r[capi.LIM_U_UB:capi.LIM_U_UB + 2] = GROUP_U[g]
    r[capi.LIM_DU_LB:capi.LIM_DU_LB + 2], r[capi.LIM_DU_UB:capi.LIM_DU_UB + 2] = list(host.du_lb), list(host.du_ub)
    r[capi.LIM_MIN_OBSTACLE_DIST] = host.min_obstacle_dist
    return r


def group_config(host, g):
    """the configuration of a robot of group g on the handle `host`: its types, geometry and limits, everything else the host's"""
    c = rg.with_geometry(with_model(host, record(*GROUP_TYPES[g])), group_geometry(g))
    lim = group_limits(host, g)
    c.u_lb[:], c.u_ub[:] = [float(v) for v in lim[0:2]], [float(v) for v in lim[2:4]]
    return c


def fleet_records(host, B):
    """(model, limits, geometry) records of a mixed fleet of B robots on `host`, robot b in group b % 4"""
    gs = [GROUPS[b % 4] for b in range(B)]
    model = np.stack([record(*GROUP_TYPES[g]) for g in gs])
    limits = np.stack([group_limits(host, g) for g in gs])
    geometry = np.stack([group_geometry(g) for g in gs])
    return model, limits, geometry
