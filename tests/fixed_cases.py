"""Cases of the fixed final state tests (grid/xf_fixed component by component, with a fixed or a free dt):
tests/test_fixed_final_state.py on the CPU, tests/test_gpu_fixed_final_state.py on the CUDA kernels."""
import numpy as np
import pytest

from mpc_local_planner_b200 import capi, configs


def _stack(a, b):
    """one batch of the instances of a, then those of b (obstacle lists padded to the longer one)"""
    ca, ta, pa = a["obstacles"]; cb, tb, pb = b["obstacles"]
    M = max(ta.shape[1], tb.shape[1])
    pad_t = lambda t: np.pad(t, ((0, 0), (0, M - t.shape[1])))
    pad_p = lambda p: np.pad(p, ((0, 0), (0, M - p.shape[1]), (0, 0)))
    return dict(x0=np.concatenate([a["x0"], b["x0"]]), xf=np.concatenate([a["xf"], b["xf"]]),
                u_prev=np.concatenate([a["u_prev"], b["u_prev"]]), u_prev_dt=b["u_prev_dt"],
                obstacles=(np.concatenate([ca, cb]).astype(np.int32), np.concatenate([pad_t(ta), pad_t(tb)]),
                           np.concatenate([pad_p(pa), pad_p(pb)])), viapoints=None)


def _g1_then_generated(B):
    """G1 (the reference's own scenario) first, then cfg-2 style instances at N = 20"""
    g1 = configs.g1_instance()
    if B == 1:
        return g1
    gen = configs.generate(5, B - 1, n=20)
    g1["u_prev_dt"] = gen["u_prev_dt"]
    return _stack(g1, gen)


def _with_mask(make, mask, **kw):
    def f():
        c = make(tol=1e-8, **kw)
        c.xf_fixed[:] = mask
        # a fixed goal with a fixed dt: the reference's cold guess (zero controls) leaves the linearised fixed-goal rows rank
        # deficient (see tests/golden/golden_cases.py); start from the solver's seeded guess
        if not c.variable_dt:
            c.reference_initial_guess = 0
        return c
    return f


def _midpoint_integral(tol):
    c = configs.cfg2_integral_form(tol=tol)
    c.collocation = capi.COLLOC_MIDPOINT
    return c


# Fixed-dt fixed-goal cases run on cfg-2 style instances with goals 2.1 - 4.2 m away (generate(5, ., n=35)), all reachable in
# 14.7 s.  Reachability is not what limits convergence here: closer goals (more spare time) converge LESS often, and with the
# whole goal pose fixed the oracle converges on 18 of the first 48.  The cause is not established; the interior-point method
# here has no constraint regularisation (Ipopt's delta_c).
_QF_DATA = lambda B: configs.generate(5, B, n=35)
# name -> (configuration, data(B))
FIXED_CASES = {
    "mt_heading_free": (_with_mask(configs.cfg1, [1, 1, 0]), _g1_then_generated),
    "mt_x_only": (_with_mask(configs.cfg1, [1, 0, 0]), _g1_then_generated),
    "qf_goal_fixed": (_with_mask(configs.cfg2, [1, 1, 1]), _QF_DATA),
    "qf_position_fixed": (_with_mask(configs.cfg2, [1, 1, 0]), _QF_DATA),
    "qf_heading_fixed": (_with_mask(configs.cfg2, [0, 0, 1]), _QF_DATA),
    "trap_position_fixed": (_with_mask(configs.cfg2_trapezoidal, [1, 1, 0], variable_dt=True), lambda B: configs.generate(2, B)),
    "midpoint_position_fixed": (_with_mask(_midpoint_integral, [1, 1, 0]), lambda B: configs.generate(2, B)),
    "ball_y_fixed": (_with_mask(configs.cfg2_terminal_ball, [0, 1, 0]), lambda B: configs.generate(2, B)),
    "car_heading_free": (_with_mask(configs.cfg3, [1, 1, 0], n=80), lambda B: configs.generate(3, B)),
}
SHIPPED = {
    "cfg1": (lambda: configs.cfg1(tol=1e-8), _g1_then_generated),
    "cfg3": (lambda: configs.cfg3(tol=1e-8), lambda B: configs.generate(3, B)),
}

# golden fixtures (SLSQP on the independent numpy restatement).  With a fixed dt and a fixed goal position the interior-point
# method fails (maximum iterations or numerical error) on instances where SLSQP finds a feasible optimum; expected to fail until
# that is fixed.
_NOT_SOLVED = pytest.mark.xfail(strict=True, reason="fixed dt + fixed goal position: the interior-point solve does not converge "
                                                     "on most instances SLSQP solves")
GOLDEN_CASES = ["g1_heading_free", pytest.param("cfg2_goal_fixed", marks=_NOT_SOLVED), pytest.param("cfg2_position_fixed", marks=_NOT_SOLVED)]


def case(name):
    make_cfg, make_data = {**FIXED_CASES, **SHIPPED}[name]
    return make_cfg(), make_data


def fixed_components(cfg):
    return [i for i in range(3) if cfg.xf_fixed[i]]


def assert_fixed_components_exact(cfg, x_last, xf, what):
    """every fixed component of the final state equals the goal bit for bit (headings of the goals lie in [-pi, pi), where the
    output normalisation is the identity)"""
    for i in fixed_components(cfg):
        assert x_last[i] == xf[i], f"{what}: x_(N-1),{i} - xf_{i} = {x_last[i] - xf[i]:.3e}"


def moved_goal(xf):
    g = np.array(xf, dtype=np.float64).copy()
    g[0] += 0.2; g[1] -= 0.2; g[2] = g[2] + 0.1 if g[2] + 0.1 < np.pi else g[2] - 0.1
    return g
