"""The solve kernels compiled for the fixed-dt quadratic-form problem (problem key MPCB200_PROBLEM_FIXED_DT_QF, ModelTraits in
mpc_core.h) compute what the kernels that read the model and the problem from the configuration compute, bit for bit: the same
seeded batch, solved cold and then warm, with the specialised kernels allowed and forced off (MPCB200_OPT_FORCE_GENERIC_MODEL).
Configurations that are the unicycle / point-footprint model but not that problem keep the generic problem key and match too.
Floats are compared as bit patterns."""
import numpy as np
import pytest

from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu

FIELDS = ("status", "iters", "u_seq", "x_seq", "dt", "kkt_err")


def _one_rate_limit_removed():
    cfg = configs.cfg2(tol=1e-8)
    cfg.du_ub[1] = capi.INF
    return cfg


# name: (configuration, data, batch, problem key the default launch picks, converged instances the first solve must reach)
CASES = {
    "cfg2": (lambda: configs.cfg2(tol=1e-8), lambda B: configs.generate(2, B), 256, capi.PROBLEM_FIXED_DT_QF, 128),
    "cfg4": (lambda: configs.cfg4(tol=1e-8), lambda B: configs.generate(4, B), 256, capi.PROBLEM_FIXED_DT_QF, 128),
    "cfg5_n20": (lambda: configs.cfg5(20, tol=1e-8), lambda B: configs.generate(5, B, n=20), 128, capi.PROBLEM_FIXED_DT_QF, 64),
    "cfg5_n200": (lambda: configs.cfg5(200, tol=1e-8), lambda B: configs.generate(5, B, n=200), 32, capi.PROBLEM_FIXED_DT_QF, 16),
    # the unicycle / point footprint, but not the fixed-dt quadratic-form problem
    "cfg2_integral_form": (lambda: configs.cfg2_integral_form(tol=1e-8), lambda B: configs.generate(2, B), 64,
                           capi.PROBLEM_GENERIC, 32),
    # (the terminal ball leaves fewer of these instances a KKT point within the iteration cap, with either kernel)
    "cfg2_terminal_ball": (lambda: configs.cfg2_terminal_ball(tol=1e-8), lambda B: configs.generate(2, B), 64,
                           capi.PROBLEM_GENERIC, 16),
    "cfg2_one_rate_limit_removed": (_one_rate_limit_removed, lambda B: configs.generate(2, B), 64, capi.PROBLEM_GENERIC, 32),
}


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def _solve_twice(cfg, data, B, force_generic, mode):
    s = capi.BatchSolver(cfg, B, device=0)
    s.set_option(capi.OPT_SOLVE_MODE, mode)
    s.set_option(capi.OPT_FORCE_GENERIC_MODEL, force_generic)
    outs = []
    for _ in range(2):   # cold, then warm from the first solve
        out = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
        outs.append({f: np.array(out[f], copy=True) for f in FIELDS})
    keys = (s.kernel_model(), s.kernel_problem())
    s.close()
    return outs, keys


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("mode", [capi.SOLVE_FUSED, capi.SOLVE_PHASED])
def test_fixed_dt_problem_kernels_match_the_generic_ones(cuda_lib, case, mode):
    make_cfg, make_data, B, expected, min_converged = CASES[case]
    cfg = make_cfg()
    data = make_data(B)
    spec, keys_spec = _solve_twice(cfg, data, B, 0, mode)
    gen, keys_gen = _solve_twice(cfg, data, B, 1, mode)
    assert keys_spec == (capi.MODEL_UNI_POINT, expected)
    assert keys_gen == (capi.MODEL_GENERIC, capi.PROBLEM_GENERIC)
    assert (spec[0]["status"] == capi.STATUS_CONVERGED).sum() >= min_converged, spec[0]["status"]
    for step, (a, b) in enumerate(zip(spec, gen)):
        for f in FIELDS:
            assert np.array_equal(_bits(a[f]), _bits(b[f])), f"step {step}: {f} differs between the specialised and the generic kernels"


def test_problem_key_before_the_first_solve_and_with_line_obstacles(cuda_lib):
    """Before any solve the handle reports the generic keys; line obstacles keep the generic kernels, problem key included."""
    cfg = configs.cfg2(tol=1e-8)
    B = 16
    data = configs.with_line_obstacles(configs.generate(2, B))
    s = capi.BatchSolver(cfg, B, device=0)
    assert (s.kernel_model(), s.kernel_problem()) == (capi.MODEL_GENERIC, capi.PROBLEM_GENERIC)
    s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
    assert (s.kernel_model(), s.kernel_problem()) == (capi.MODEL_GENERIC, capi.PROBLEM_GENERIC)
    s.close()
