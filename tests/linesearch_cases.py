"""States of the line-search tests (tests/test_linesearch.py, tests/test_gpu_linesearch.py): the cases, the iterates and the
edge changes.  A state is the oracle's own interior-point iterate j of one instance (its solve run with max_iter = j,
parity.oracle_iterate), optionally changed at the edges of the line search."""
import numpy as np

from mpc_local_planner_b200 import capi, configs

ITERATES = (0, 1, 3, 10, 25, "last")


def _cfg2_variant(**kw):
    def f(n=None):
        c = configs.cfg2(n or 50, tol=1e-8)
        for k, v in kw.items():
            setattr(c, k, v)
        return c
    return f


def _cfg4_ordered_orientation(n=None):
    c = configs.cfg4(n or 50, tol=1e-8)
    c.vp_ordered = 1
    c.vp_orientation_weight = 0.5
    return c


def _with(make, **kw):
    def f(n=None):
        c = make(n)
        for k, v in kw.items():
            setattr(c, k, v)
        return c
    return f


def _midpoint(make):
    return _with(make, collocation=capi.COLLOC_MIDPOINT)


def _gen(cid, transform=None):
    def f(B, n=None):
        d = configs.generate(cid, B, n=n)
        return transform(d) if transform else d
    return f


# name -> (configuration(n), data(B, n), instance)
CASES = {
    "cfg1": (lambda n=None: configs.cfg1(tol=1e-8), lambda B, n=None: configs.g1_instance(), 0),
    "cfg2": (lambda n=None: configs.cfg2(n or 50, tol=1e-8), _gen(2), 1),
    "cfg3": (lambda n=None: configs.cfg3(n or 80, tol=1e-8), _gen(3), 1),
    "cfg4": (lambda n=None: configs.cfg4(n or 50, tol=1e-8), _gen(4), 1),
    "cfg5": (lambda n=None: configs.cfg5(n or 50, tol=1e-8), _gen(5), 0),
    "vp_ordered_orientation": (_cfg4_ordered_orientation, _gen(4), 1),
    "integral_fixed_dt": (_cfg2_variant(quadratic_integral_form=1), _gen(2), 1),
    "integral_free_dt": (lambda n=None: configs.cfg2_integral_form(n or 50, tol=1e-8), _gen(2), 1),
    "trapezoid_fixed_dt": (lambda n=None: configs.cfg2_trapezoidal(n or 50, tol=1e-8, variable_dt=False), _gen(2), 1),
    "trapezoid_free_dt": (lambda n=None: configs.cfg2_trapezoidal(n or 50, tol=1e-8), _gen(2), 1),
    "hybrid_min_time": (lambda n=None: configs.cfg2_hybrid_min_time(n or 50, tol=1e-8), _gen(2), 1),
    "terminal_ball": (lambda n=None: configs.cfg2_terminal_ball(n or 50, tol=1e-8), _gen(2), 1),
    "dynamic_fixed_dt": (_cfg2_variant(enable_dynamic_obstacles=1), _gen(2, configs.with_moving_obstacles), 1),
    "dynamic_free_dt": (_with(lambda n=None: configs.cfg2_integral_form(n or 50, tol=1e-8), enable_dynamic_obstacles=1),
                        _gen(2, configs.with_moving_obstacles), 1),
    "line_obstacles": (lambda n=None: configs.cfg2(n or 50, tol=1e-8), _gen(2, configs.with_line_obstacles), 1),
    "midpoint": (_midpoint(lambda n=None: configs.cfg2(n or 50, tol=1e-8)), _gen(2), 1),
    "midpoint_free_dt": (_midpoint(lambda n=None: configs.cfg2_integral_form(n or 50, tol=1e-8)), _gen(2), 1),
}


def case(name, n=None):
    make_cfg, make_data, b = CASES[name]
    cfg = make_cfg(n)
    return cfg, make_data(b + 1, n), b


# ---- edge states: applied to the oracle's state, then written into the device's -----------------------------------------
def scale_step(f):
    def mod(o):
        o.arr("STEP")[:5] *= f
        o.arr("SCAL")[capi.SC_DDT] *= f
    return mod


def negate_step(o):
    o.arr("STEP")[:5] *= -1.0
    o.arr("SCAL")[capi.SC_DDT] *= -1.0


def jam(tiny):
    def mod(o):
        scale_step(1e10)(o)
        o.arr("SCAL")[capi.SC_TINY] = tiny
    return mod


def feasible_merit(o):
    o.arr("SCAL")[capi.SC_INF] = 1e-15


def defer(o):
    o.arr("SCAL")[capi.SC_DEFER] = 1.0


def stopped(o):
    o.arr("SCAL")[capi.SC_STATUS] = float(capi.STATUS_MAX_ITER)


def extreme_multipliers(o):
    """before EVAL: a few rows' multipliers far above and below mu / s, so that the kappa-sigma clamp of the update bites"""
    LAM = o.arr("LAM")
    rows = np.argwhere(LAM > 0)
    for i, (sl, k) in enumerate(rows[:: max(len(rows) // 6, 1)][:6]):
        LAM[sl, k] *= 1e12 if i % 2 == 0 else 1e-12


# name -> (changed before EVAL, changed after the KKT solve)
EDGES = {
    "saturated": (None, scale_step(1e3)),
    "no_blocking_row": (None, scale_step(1e-3)),
    "backtracking_exhausted": (None, negate_step),
    # iterate 60 of a solve that does not stop (tol 1e-15): the step is of rounding size, the first trial is refused and the
    # second one accepted as flat (a scaled step does not get there: the slack steps of the rows stay of full size)
    "flat_merit": (None, None),
    "jam": (None, jam(1.0)),
    "first_tiny_step": (None, jam(0.0)),
    "kappa_sigma": (extreme_multipliers, None),
    "feasible": (None, feasible_merit),
    "null_step": (None, defer),
    "stopped": (None, stopped),
}


def check_edge(name, d, before, after):
    """what each edge state must show in the oracle's diagnostics and scalars (before / after: SCAL around the line search)"""
    if name == "saturated":
        assert d["hist"].sum() > d["m"] // 8 and d["jt"] < 40, (d["hist"].sum(), d["m"], d["jt"])
    elif name == "no_blocking_row":
        assert d["a_p"] == 1.0
    elif name == "backtracking_exhausted":   # (a negated step may still decrease the merit: asserted on one state at least)
        assert d["nbt"] < 3 or (d["alpha"] == d["a_p"] / 8 and d["branch"] == 0)
    elif name == "jam":
        assert after[capi.SC_STATUS] == capi.STATUS_NUMERICAL_ERROR and after[capi.SC_TINY] == 2.0
    elif name == "first_tiny_step":
        assert after[capi.SC_TINY] == 1.0 and after[capi.SC_STATUS] == -1.0
    elif name == "feasible":
        assert d["rho"] == 1.0
    elif name == "null_step":
        assert after[capi.SC_ITER] == before[capi.SC_ITER] + 1 and after[capi.SC_ALPHA] == 0.0 and after[capi.SC_DEFER] == 0.0
        for i in range(capi.SCAL_WORDS):
            if i not in (capi.SC_ITER, capi.SC_ALPHA, capi.SC_DEFER):
                assert after[i] == before[i] or (np.isnan(after[i]) and np.isnan(before[i])), i
    elif name == "stopped":
        np.testing.assert_array_equal(after, before)
