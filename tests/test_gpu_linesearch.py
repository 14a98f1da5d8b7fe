"""PHASE_LINESEARCH of the CUDA phase kernels against the oracle's line search (orc_linesearch), field by field.

Every comparison starts from one shared state: the oracle's own iterate j of each instance of the batch, written into the
device workspace after the device's own INIT and ASSOCIATE (the association must be the oracle's).  EVAL and KKT run on the
device and are checked with the tolerances of the phase tests; then the oracle's records, step and scalars are written, so
that both line searches start from the same inputs, and the iterate, the slacks, the multipliers and DT, ALPHA, RHO, NBT, ITER,
TINY, STATUS are compared (tests/parity.py has the tolerances and the rule for decisions at their threshold).

Every phase-kernel variant is reached, and the launch reports its model / problem key: <false, MODEL_UNI_POINT_QF>,
<false, MODEL_UNI_POINT>, <false, MODEL_GENERIC> and <true, MODEL_GENERIC> (line obstacles, moving obstacles, midpoint
differences), with the unbordered and the bordered KKT (free dt, fixed final-state components).  The horizons cover idle lanes
of the warp reductions, the cross-warp merges (N > 32) and threads that own two stages (N > 128).  The fused solve kernel is
not stepped phase by phase: the fused == phased and specialised == generic bit-identity tests (test_gpu_parity,
test_gpu_model_phases, test_gpu_kernel_keys) tie it to these phase kernels."""
import pytest

import linesearch_cases as lc
from fixed_cases import case as fixed_case
from mpc_local_planner_b200 import configs
from parity import GEN, UNI, UNI_QF, compare_at

pytestmark = pytest.mark.gpu


# name -> (configuration, data(B), force the generic kernels, expected keys)
VARIANTS = {
    "qf_cfg2": (lambda: lc.case("cfg2")[0], lambda B: configs.generate(2, B), 0, UNI_QF),
    "qf_cfg5": (lambda: lc.case("cfg5")[0], lambda B: configs.generate(5, B), 0, UNI_QF),
    "uni_integral_free_dt": (lambda: lc.case("integral_free_dt")[0], lambda B: configs.generate(2, B), 0, UNI),
    "uni_terminal_ball": (lambda: lc.case("terminal_ball")[0], lambda B: configs.generate(2, B), 0, UNI),
    "uni_qf_position_fixed": (lambda: fixed_case("qf_position_fixed")[0], lambda B: fixed_case("qf_position_fixed")[1](B), 0, UNI),
    "generic_cfg3": (lambda: lc.case("cfg3")[0], lambda B: configs.generate(3, B), 0, GEN),
    "generic_forced_cfg2": (lambda: lc.case("cfg2")[0], lambda B: configs.generate(2, B), 1, GEN),
    "generic_trap_position_fixed": (lambda: fixed_case("trap_position_fixed")[0], lambda B: fixed_case("trap_position_fixed")[1](B), 1, GEN),
    "lines": (lambda: lc.case("line_obstacles")[0], lambda B: configs.with_line_obstacles(configs.generate(2, B)), 0, GEN),
    "lines_dynamic_fixed_dt": (lambda: lc.case("dynamic_fixed_dt")[0],
                               lambda B: configs.with_moving_obstacles(configs.generate(2, B)), 0, GEN),
    "lines_dynamic_free_dt": (lambda: lc.case("dynamic_free_dt")[0],
                              lambda B: configs.with_moving_obstacles(configs.generate(2, B)), 0, GEN),
    "lines_midpoint": (lambda: lc.case("midpoint")[0], lambda B: configs.generate(2, B), 0, GEN),
    "lines_midpoint_free_dt": (lambda: lc.case("midpoint_free_dt")[0], lambda B: configs.generate(2, B), 0, GEN),
}


@pytest.mark.parametrize("variant", list(VARIANTS))
def test_linesearch_matches_oracle(cuda_lib, orc, variant):
    make_cfg, make_data, force_generic, keys = VARIANTS[variant]
    cfg = make_cfg()
    B = 4
    data = make_data(B)
    compared = marginal = 0
    for j in lc.ITERATES:
        c, m = compare_at(orc, cfg, data, B, j, force_generic, keys)
        compared += c; marginal += m
    assert compared >= 12 and marginal <= 2, (compared, marginal)


@pytest.mark.parametrize("cid,n", [(5, n) for n in (3, 20, 31, 32, 33, 64, 65, 97, 128, 129, 200)] +
                                  [(3, n) for n in (33, 65, 129, 160)])
def test_linesearch_horizons(cuda_lib, orc, cid, n):
    """cfg 5 (fixed-dt quadratic-form kernels) and cfg 3 (generic kernels, bordered KKT) at horizons around the warp and CTA
    boundaries: one warp with idle lanes, several warps (cross-warp merges of a_p, a_d, the sums and the trial accumulators),
    and more stages than threads (cfg 3 at N = 200 does not fit the shared-memory image of an instance; 160 is the same shape)"""
    cfg = configs.config_for(cid, n=n, tol=1e-8)
    B = 3
    data = configs.generate(cid, B, n=n)
    compared = marginal = 0
    for j in (0, 3, 10):
        c, m = compare_at(orc, cfg, data, B, j, 0, UNI_QF if cid == 5 else GEN)
        compared += c; marginal += m
    assert compared >= 3 and marginal <= 1, (compared, marginal)


@pytest.mark.parametrize("edge", [e for e in lc.EDGES if e not in ("kappa_sigma", "flat_merit")])
def test_linesearch_edge_states(cuda_lib, orc, edge):
    """the edge states of tests/test_linesearch.py on the fixed-dt quadratic-form and the generic kernels, from iterate 3: no
    deferred step, the inertia right at the device's regularisation"""
    _, post = lc.EDGES[edge]
    for variant in ("qf_cfg2", "generic_cfg3"):
        make_cfg, make_data, force_generic, keys = VARIANTS[variant]
        cfg = make_cfg()
        B = 2
        data = make_data(B)
        c, m = compare_at(orc, cfg, data, B, 3, force_generic, keys, post)
        assert c >= 1 and m == 0
