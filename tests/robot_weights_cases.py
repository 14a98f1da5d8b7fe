"""Per-robot weights records (mpcb200_set_robot_weights) for the tests: the record of a configuration, the configuration a record
makes (restated from include/mpcb200.h, the expected result of apply_robot_weights), the validity rules restated, the words a
handle reads, scaled records, and the configurations of every objective the records apply to."""
import numpy as np

from mpc_local_planner_b200 import capi, configs

W = capi.WEIGHT_WORDS
Q, R, QF, VPP, VPO = capi.WGT_Q, capi.WGT_R, capi.WGT_QF, capi.WGT_VP_POSITION, capi.WGT_VP_ORIENTATION


def quadratic(cfg):
    return cfg.objective == capi.OBJ_QUADRATIC_FORM


def terminal(cfg):
    return bool(cfg.terminal_cost) and not all(cfg.xf_fixed)


def viapoints(cfg):
    return cfg.objective == capi.OBJ_MINIMUM_TIME_VIA_POINTS or (quadratic(cfg) and bool(cfg.vp_attraction_with_quadratic))


def hybrid(cfg, q, r):
    """the hybrid minimum-time term of a quadratic form with state weights q and control weights r"""
    return bool(cfg.hybrid_cost_minimum_time) and quadratic(cfg) and all(v == 0 for v in q) and not all(v == 0 for v in r)


def words_read(cfg):
    w = []
    if quadratic(cfg):
        w += list(range(Q, Q + 9)) + list(range(R, R + 4))
    if terminal(cfg):
        w += list(range(QF, QF + 9))
    if viapoints(cfg):
        w += [VPP, VPO]
    return w


def record_of(cfg):
    """the record holding the configuration's own values in every word"""
    r = np.zeros(W)
    r[Q:Q + 9], r[R:R + 4], r[QF:QF + 9] = list(cfg.Q), list(cfg.R), list(cfg.Qf)
    r[VPP], r[VPO] = cfg.vp_position_weight, cfg.vp_orientation_weight
    return r


def records_of(cfg, B):
    return np.tile(record_of(cfg), (B, 1))


def with_weights(cfg, rec):
    """the configuration of a robot with record `rec`: the words its objective reads, every other field as in cfg"""
    c = cfg.copy()
    if quadratic(cfg):
        c.Q[:] = [float(v) for v in rec[Q:Q + 9]]
        c.R[:] = [float(v) for v in rec[R:R + 4]]
    if terminal(cfg):
        c.Qf[:] = [float(v) for v in rec[QF:QF + 9]]
    if viapoints(cfg):
        c.vp_position_weight, c.vp_orientation_weight = float(rec[VPP]), float(rec[VPO])
    return c


def rule(cfg, r):
    """the validity rules of include/mpcb200.h restated: every word read finite, the hybrid term as the handle has it"""
    if not all(np.isfinite(r[w]) for w in words_read(cfg)):
        return False
    if quadratic(cfg) and hybrid(cfg, r[Q:Q + 9], r[R:R + 4]) != hybrid(cfg, list(cfg.Q), list(cfg.R)):
        return False
    return True


def scaled(cfg, q=1.0, r=1.0, qf=1.0, vp=1.0):
    """the configuration's record with Q, R, Qf and both via-point weights scaled"""
    rec = record_of(cfg)
    rec[Q:Q + 9] *= q
    rec[R:R + 4] *= r
    rec[QF:QF + 9] *= qf
    rec[VPP:VPO + 1] *= vp
    return rec


# four weight groups of the mixed-batch tests, robot b in group b mod 4: R x 1, 2, 4, 8 and Qf x 1, 0.5, 2, 4 (Q and the via-point
# weights too on the objectives where R alone would not change anything)
GROUP_R, GROUP_QF, GROUP_Q, GROUP_VP = (1.0, 2.0, 4.0, 8.0), (1.0, 0.5, 2.0, 4.0), (1.0, 1.5, 0.75, 1.25), (1.0, 0.5, 2.0, 1.5)


def group_records(cfg, B):
    q = (1.0,) * 4 if hybrid(cfg, list(cfg.Q), list(cfg.R)) else GROUP_Q   # (a hybrid handle keeps Q zero either way)
    rec = np.stack([scaled(cfg, q[b % 4], GROUP_R[b % 4], GROUP_QF[b % 4], GROUP_VP[b % 4]) for b in range(B)])
    return rec, [np.arange(g, B, 4) for g in range(4)]


def variant(name):
    """(configuration, generator id) of the weights test cases"""
    if name == "cfg2":
        return configs.cfg2(), 2
    if name == "cfg4":
        return configs.cfg4(), 4
    if name == "integral":
        return configs.cfg2_integral_form(), 2
    if name == "hybrid":
        return configs.cfg2_hybrid_min_time(), 2
    if name == "ball":
        return configs.cfg2_terminal_ball(), 2
    if name == "mintime_vp":   # minimum time with via-points, an orientation weight and a terminal cost (free final heading)
        c = configs.cfg1()
        c.n, c.objective = 50, capi.OBJ_MINIMUM_TIME_VIA_POINTS
        c.vp_position_weight, c.vp_orientation_weight = 8.0, 0.5
        c.xf_fixed[:] = [1, 1, 0]
        c.terminal_cost = 1
        c.Qf[:] = [0.0] * 8 + [1.0]
        return c, 4
    raise ValueError(name)
