"""The solve kernels compiled for one robot / footprint model (MPCB200_OPT_FORCE_GENERIC_MODEL, ModelTraits in mpc_core.h)
compute what the kernels that read the model from the configuration compute, bit for bit: the same seeded batch, solved cold and
then warm, with the specialised variant allowed and forced off.  Floats are compared as bit patterns, so a -0.0 against 0.0 or
a differently contracted expression is a failure."""
import numpy as np
import pytest

from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu

FIELDS = ("status", "iters", "u_seq", "x_seq", "dt", "kkt_err")


def _circular_footprint():
    cfg = configs.cfg2(tol=1e-8)
    cfg.footprint_type = capi.FOOTPRINT_CIRCULAR
    cfg.footprint_params[0] = 0.15
    cfg.min_obstacle_dist = 0.1
    return cfg


# name: (configuration, data, batch, model key the default launch picks)
CASES = {
    "cfg2": (lambda: configs.cfg2(tol=1e-8), lambda B: configs.generate(2, B), 256, capi.MODEL_UNI_POINT),
    "cfg4": (lambda: configs.cfg4(tol=1e-8), lambda B: configs.generate(4, B), 256, capi.MODEL_UNI_POINT),
    "cfg2_circular_footprint": (_circular_footprint, lambda B: configs.generate(2, B), 64, capi.MODEL_GENERIC),
    "cfg5_n20": (lambda: configs.cfg5(20, tol=1e-8), lambda B: configs.generate(5, B, n=20), 128, capi.MODEL_UNI_POINT),
    "cfg5_n200": (lambda: configs.cfg5(200, tol=1e-8), lambda B: configs.generate(5, B, n=200), 32, capi.MODEL_UNI_POINT),
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
    model = s.kernel_model()
    s.close()
    return outs, model


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("mode", [capi.SOLVE_FUSED, capi.SOLVE_PHASED])
def test_specialised_model_kernels_match_the_generic_ones(cuda_lib, case, mode):
    if mode == capi.SOLVE_PHASED and case.startswith("cfg5"):
        pytest.skip("the phased mode runs the same phase functions; cfg 2 / 4 cover it")
    make_cfg, make_data, B, expected = CASES[case]
    cfg = make_cfg()
    data = make_data(B)
    spec, model_spec = _solve_twice(cfg, data, B, 0, mode)
    gen, model_gen = _solve_twice(cfg, data, B, 1, mode)
    assert model_spec == expected
    assert model_gen == capi.MODEL_GENERIC
    assert (spec[0]["status"] == capi.STATUS_CONVERGED).sum() >= B // 2, spec[0]["status"]
    for step, (a, b) in enumerate(zip(spec, gen)):
        for f in FIELDS:
            assert np.array_equal(_bits(a[f]), _bits(b[f])), f"step {step}: {f} differs between the specialised and the generic kernels"


def test_line_obstacles_keep_the_generic_kernels(cuda_lib):
    """The specialised variants leave the line-obstacle path out: a unicycle / point batch with line obstacles runs the generic
    kernels."""
    cfg = configs.cfg2(tol=1e-8)
    B = 16
    data = configs.with_line_obstacles(configs.generate(2, B))
    s = capi.BatchSolver(cfg, B, device=0)
    s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
    assert s.kernel_model() == capi.MODEL_GENERIC
    s.close()
