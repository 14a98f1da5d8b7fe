"""Per-robot geometry records (mpcb200_set_robot_geometry) for the tests: the record of a configuration, the configuration a
record makes (restated from include/mpcb200.h, the expected result of apply_robot_geometry), the validity rules restated, scaled
and random records, and the configurations of every robot / footprint type the records apply to."""
import numpy as np

from mpc_local_planner_b200 import capi, configs

W = capi.GEOMETRY_WORDS
FP, NP, XY = capi.GEO_FOOTPRINT, capi.GEO_N_POLY, capi.GEO_POLY_XY
CARS = (capi.ROBOT_SIMPLE_CAR, capi.ROBOT_SIMPLE_CAR_FRONT)


def record_of(cfg):
    """the record holding the configuration's own values in every word"""
    r = np.zeros(W)
    r[capi.GEO_WHEELBASE], r[capi.GEO_LENGTH_REAR], r[capi.GEO_LENGTH_FRONT] = cfg.wheelbase, cfg.length_rear, cfg.length_front
    r[FP:FP + 4] = list(cfg.footprint_params)
    r[NP] = cfg.n_poly
    r[XY:XY + 2 * capi.MAX_POLY] = list(cfg.poly_xy)
    return r


def records_of(cfg, B):
    return np.tile(record_of(cfg), (B, 1))


def with_geometry(cfg, rec):
    """the configuration of a robot with record `rec`: the words its robot and footprint types read, every other field as in cfg"""
    c = cfg.copy()
    if c.robot_type in CARS:
        c.wheelbase = float(rec[capi.GEO_WHEELBASE])
    elif c.robot_type == capi.ROBOT_KIN_BICYCLE:
        c.length_rear, c.length_front = float(rec[capi.GEO_LENGTH_REAR]), float(rec[capi.GEO_LENGTH_FRONT])
    if c.footprint_type == capi.FOOTPRINT_CIRCULAR:
        c.footprint_params[0] = float(rec[FP])
    elif c.footprint_type in (capi.FOOTPRINT_TWO_CIRCLES, capi.FOOTPRINT_LINE):
        c.footprint_params[:] = [float(v) for v in rec[FP:FP + 4]]
    elif c.footprint_type == capi.FOOTPRINT_POLYGON:
        c.n_poly = int(rec[NP])
        for i in range(2 * c.n_poly):
            c.poly_xy[i] = float(rec[XY + i])
    return c


def rule(cfg, r):
    """the validity rules of include/mpcb200.h restated, on the words the handle's two types read"""
    fin = lambda v: bool(np.isfinite(v))   # noqa: E731
    if cfg.robot_type in CARS and not (fin(r[0]) and r[0] > 0):
        return False
    if cfg.robot_type == capi.ROBOT_KIN_BICYCLE and not (fin(r[1]) and r[1] > 0 and fin(r[2]) and r[2] >= 0):
        return False
    f = r[FP:FP + 4]
    if cfg.footprint_type == capi.FOOTPRINT_CIRCULAR:
        return fin(f[0]) and f[0] >= 0
    if cfg.footprint_type == capi.FOOTPRINT_TWO_CIRCLES:
        return all(fin(v) for v in f) and f[1] >= 0 and f[3] >= 0
    if cfg.footprint_type == capi.FOOTPRINT_LINE:
        return all(fin(v) for v in f)
    if cfg.footprint_type == capi.FOOTPRINT_POLYGON:
        n = r[NP]
        if not (1 <= n <= capi.MAX_POLY) or n != np.floor(n):
            return False
        return all(fin(v) for v in r[XY:XY + 2 * int(n)])
    return True


def scaled(cfg, fp, wb):
    """the configuration's record with the footprint scaled by fp (offsets, radii, end points, vertices) and the wheelbase or the
    bicycle's lengths by wb"""
    r = record_of(cfg)
    r[0:3] *= wb
    r[FP:FP + 4] *= fp
    r[XY:] *= fp
    return r


def polygon(n, rng, size=1.0):
    """a convex polygon of n vertices around the origin (a robot footprint in its own frame), radius about 0.2 * size"""
    ang = np.sort(rng.uniform(0, 2 * np.pi, n)) if n > 3 else np.array([0.0, 2.1, 4.2])
    rad = size * rng.uniform(0.15, 0.25, n)
    return np.stack([rad * np.cos(ang) + 0.05 * size, rad * np.sin(ang)], axis=1)


def random_records(cfg, B, seed):
    """seeded records valid for cfg: footprints scaled by U(0.6, 1.2), wheelbases and lengths by U(0.8, 1.4), and for a polygon
    footprint a fresh convex polygon of 3 to 16 vertices per robot (its unused words NaN: nothing may read them)"""
    rng = np.random.default_rng(seed)
    r = np.stack([scaled(cfg, rng.uniform(0.6, 1.2), rng.uniform(0.8, 1.4)) for _ in range(B)])
    if cfg.footprint_type == capi.FOOTPRINT_POLYGON:
        for b in range(B):
            n = 3 + b % 14
            r[b, NP] = n
            r[b, XY:] = np.nan
            r[b, XY:XY + 2 * n] = polygon(n, rng).ravel()
    return r


def variant(name):
    """(configuration, generator id) of the geometry test cases: cfg 3 (simple car, polygon) and cfg 3 with another footprint or
    the kinematic bicycle"""
    c = configs.cfg3()
    if name == "cfg3":
        return c, 3
    if name == "circular":
        c.footprint_type = capi.FOOTPRINT_CIRCULAR
        c.footprint_params[:] = [0.25, 0.0, 0.0, 0.0]
    elif name == "two_circles":
        c.footprint_type = capi.FOOTPRINT_TWO_CIRCLES
        c.footprint_params[:] = [0.2, 0.18, 0.1, 0.18]
    elif name == "line":
        c.footprint_type = capi.FOOTPRINT_LINE
        c.footprint_params[:] = [0.25, 0.0, -0.1, 0.0]
    elif name == "bicycle":
        c.robot_type = capi.ROBOT_KIN_BICYCLE
        c.length_rear, c.length_front = 0.2, 0.25
    else:
        raise ValueError(name)
    return c, 3
