"""The solve kernels compiled for one robot / footprint model and for the fixed-dt quadratic-form problem (the kernel keys
(model, problem), ModelTraits in mpc_core.h) compute what the kernels that read the model and the problem from the
configuration compute, bit for bit: the same seeded batch, solved cold and then warm, with the specialised kernels allowed and
forced off (MPCB200_OPT_FORCE_GENERIC_MODEL).  Configurations that are the unicycle / point-footprint model but not that problem
keep the generic problem key and match too; a fixed dt with a fixed goal component runs the unicycle / point kernel of the
bordered KKT system.  Floats are compared as bit patterns, so a -0.0 against 0.0 or a differently contracted expression is a
failure."""
import pytest

import parity as par
from fixed_cases import case as fixed_case
from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu

BOTH = (capi.SOLVE_FUSED, capi.SOLVE_PHASED)


def _circular_footprint():
    cfg = configs.cfg2(tol=1e-8)
    cfg.footprint_type = capi.FOOTPRINT_CIRCULAR
    cfg.footprint_params[0] = 0.15
    cfg.min_obstacle_dist = 0.1
    return cfg


def _one_rate_limit_removed():
    cfg = configs.cfg2(tol=1e-8)
    cfg.du_ub[1] = capi.INF
    return cfg


# name: (configuration, data(B), batch, keys of the default launch, converged instances the first solve must reach, solve modes)
CASES = {
    "cfg2": (lambda: configs.cfg2(tol=1e-8), lambda B: configs.generate(2, B), 256, par.UNI_QF, 128, BOTH),
    "cfg4": (lambda: configs.cfg4(tol=1e-8), lambda B: configs.generate(4, B), 256, par.UNI_QF, 128, BOTH),
    "cfg5_n20": (lambda: configs.cfg5(20, tol=1e-8), lambda B: configs.generate(5, B, n=20), 128, par.UNI_QF, 64, BOTH),
    "cfg5_n200": (lambda: configs.cfg5(200, tol=1e-8), lambda B: configs.generate(5, B, n=200), 32, par.UNI_QF, 16, BOTH),
    "cfg2_circular_footprint": (_circular_footprint, lambda B: configs.generate(2, B), 64, par.GEN, 32, BOTH),
    # the unicycle / point footprint, but not the fixed-dt quadratic-form problem
    "cfg2_integral_form": (lambda: configs.cfg2_integral_form(tol=1e-8), lambda B: configs.generate(2, B), 64, par.UNI, 32,
                           BOTH),
    # (the terminal ball leaves fewer of these instances a KKT point within the iteration cap, with either kernel)
    "cfg2_terminal_ball": (lambda: configs.cfg2_terminal_ball(tol=1e-8), lambda B: configs.generate(2, B), 64, par.UNI, 16,
                           BOTH),
    "cfg2_one_rate_limit_removed": (_one_rate_limit_removed, lambda B: configs.generate(2, B), 64, par.UNI, 32, BOTH),
    # a fixed dt with a fixed goal component: the bordered KKT system with the generic problem code
    "qf_position_fixed": (lambda: fixed_case("qf_position_fixed")[0], lambda B: fixed_case("qf_position_fixed")[1](B), 64,
                          par.UNI, 16, (capi.SOLVE_FUSED,)),
    "qf_goal_fixed": (lambda: fixed_case("qf_goal_fixed")[0], lambda B: fixed_case("qf_goal_fixed")[1](B), 64, par.UNI, 16,
                      (capi.SOLVE_FUSED,)),
}
MODE_NAMES = {capi.SOLVE_FUSED: "fused", capi.SOLVE_PHASED: "phased"}


@pytest.mark.parametrize("name,mode", [pytest.param(name, mode, id=f"{name}-{MODE_NAMES[mode]}")
                                       for name, c in CASES.items() for mode in c[5]])
def test_specialised_kernels_match_the_generic_ones(cuda_lib, name, mode):
    make_cfg, make_data, B, keys, min_converged, _ = CASES[name]
    cfg = make_cfg()
    data = make_data(B)
    spec, keys_spec = par.solve_twice(cfg, data, B, mode, force_generic=0)
    gen, keys_gen = par.solve_twice(cfg, data, B, mode, force_generic=1)
    assert keys_spec == keys
    assert keys_gen == par.GEN
    assert (spec[0]["status"] == capi.STATUS_CONVERGED).sum() >= min_converged, spec[0]["status"]
    par.assert_same_solves(spec, gen, "the specialised and the generic kernels")


def test_problem_key_before_the_first_solve_and_with_line_obstacles(cuda_lib):
    """Before any solve the handle reports the generic keys; the specialised variants leave the line-obstacle path out: a
    unicycle / point batch with line obstacles runs the generic kernels, model and problem key."""
    cfg = configs.cfg2(tol=1e-8)
    B = 16
    data = configs.with_line_obstacles(configs.generate(2, B))
    s = capi.BatchSolver(cfg, B, device=0)
    assert (s.kernel_model(), s.kernel_problem()) == par.GEN
    s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
    assert (s.kernel_model(), s.kernel_problem()) == par.GEN
    s.close()
