"""grid/xf_fixed component by component on the CUDA kernels (the cases of tests/test_fixed_final_state.py): phase parity at the
first iterate, whole solves through the C ABI in both solve modes, the golden fixtures, and fixed components that stay exactly at
the goal.  The specialised unicycle / point kernels with a fixed dt and a fixed goal are compared with the generic ones in
tests/test_gpu_kernel_keys.py."""
import numpy as np
import pytest

import golden_checks as gc
import parity as par
from fixed_cases import FIXED_CASES, GOLDEN_CASES, SHIPPED, assert_fixed_components_exact, case, moved_goal
from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu
U_TOL = 1e-4


def _step(s, data, x0=None, xf=None, u_prev=None, u_prev_dt=None):
    return s.step(data["x0"] if x0 is None else x0, data["xf"] if xf is None else xf, data["u_prev"] if u_prev is None else u_prev,
                  data["u_prev_dt"] if u_prev_dt is None else u_prev_dt, data["obstacles"], data["viapoints"])


@pytest.mark.parametrize("name", list(FIXED_CASES))
def test_phase_parity(cuda_lib, orc, name):
    """INIT / ASSOCIATE / EVAL / KKT of the kernels against the oracle at the first iterate; the step and d(dt) at the
    regularisation the kernel settled on (delta = 0 where the inertia was right)."""
    cfg, make_data = case(name)
    B = 6
    data = make_data(B)
    n_steps = par.check_first_iterate(orc, cfg, data, B)
    # the car's cold start needs more regularisation than one iteration's factorisation budget on every instance (its steps are
    # compared over four iterations on the emulator, tests/test_fixed_final_state.py)
    assert n_steps >= (0 if name == "car_heading_free" else 1)


# (case, N or None for the case's own horizon, batch)
SOLVE_CASES = [(n, None, 48) for n in FIXED_CASES if n != "car_heading_free"] + [("car_heading_free", None, 32),
                                                                                  ("qf_position_fixed", 100, 32)]


@pytest.mark.parametrize("mode", [capi.SOLVE_FUSED, capi.SOLVE_PHASED])
@pytest.mark.parametrize("name,n,B", SOLVE_CASES)
def test_solve_parity(cuda_lib, orc, name, n, B, mode):
    """Whole solves through the C ABI against the oracle (cfg 2's N = 50 and N = 100 run the two CTA shapes with the bordered
    KKT system and no d(dt))."""
    cfg, make_data = case(name)
    if n is not None:
        cfg.n = n
        data = configs.generate(5, B, n=int(0.7 * n))   # goals 0.042 n - 0.084 n m away, as the case's own batch at N = 50
    else:
        data = make_data(B)
    s = capi.BatchSolver(cfg, B, device=0)
    s.set_option(capi.OPT_SOLVE_MODE, mode)
    out = _step(s, data)
    s.close()
    ref = orc.step_batch(cfg, data, n_threads=8)
    agree = (out["status"] == ref["status"]).sum()
    both = (out["status"] == 0) & (ref["status"] == 0)
    assert agree >= B - 1, f"status agreement {agree}/{B}: gpu {out['status']} oracle {ref['status']}"
    assert both.sum() >= max(2, (ref["status"] == 0).sum() - 1), f"gpu {out['status']} oracle {ref['status']}"
    assert np.abs(out["dt"][both] - ref["dt"][both]).max() < 1e-6
    du = np.abs(out["u_seq"][both] - ref["u_seq"][both]).max(axis=(1, 2))
    if cfg.variable_dt:   # minimum-time optima need not be strict in the controls
        assert (du < U_TOL).mean() >= 0.8, f"du {du}"
    else:
        assert (du < U_TOL).sum() >= len(du) - 1, f"du {du}"
    assert (out["kkt_err"][both] <= cfg.tol).all()
    for b in range(B):   # converged or not
        assert_fixed_components_exact(cfg, out["x_seq"][b, -1], data["xf"][b], f"{name} instance {b} (status {out['status'][b]})")


def _cuda_solve(cfg, data):
    B = data["x0"].shape[0]
    s = capi.BatchSolver(cfg, B, device=0)
    out = _step(s, data)
    s.close()
    return out


@pytest.mark.parametrize("gcase", GOLDEN_CASES)
def test_golden_cases(cuda_lib, gcase):
    matched, other = gc.check_case(gcase, _cuda_solve)
    assert matched >= 1


@pytest.mark.parametrize("name", list(FIXED_CASES) + list(SHIPPED))
def test_fixed_components_stay_exactly_at_the_goal(cuda_lib, orc, name):
    """Cold, then a warm step with the goal moved by 0.2 m / 0.1 rad: every fixed component of every returned final state is
    the goal, bit for bit; the warm controls agree with the oracle's."""
    cfg, make_data = case(name)
    B = 16
    data = make_data(B)
    s = capi.BatchSolver(cfg, B, device=0)
    out1 = _step(s, data)
    for b in range(B):
        assert_fixed_components_exact(cfg, out1["x_seq"][b, -1], data["xf"][b], f"{name} cold, instance {b}")
    x0b = out1["x_seq"][:, 1, :].copy()
    uprev = out1["u_seq"][:, 0, :].copy()
    xf2 = np.stack([moved_goal(g) for g in data["xf"]])
    out2 = _step(s, data, x0=x0b, xf=xf2, u_prev=uprev, u_prev_dt=cfg.dt_ref)
    s.close()
    for b in range(B):
        assert_fixed_components_exact(cfg, out2["x_seq"][b, -1], xf2[b], f"{name} warm, instance {b}")
        if b >= 4:
            continue
        o = orc.instance_from_batch(cfg, data, b)
        u1, x1, r1 = o.step()
        o.set_measurement(x1[1], xf2[b], u1[0], cfg.dt_ref)
        u2, x2, r2 = o.step()
        if r1.status == 0 and r2.status == 0 and out1["status"][b] == 0 and out2["status"][b] == 0 and not cfg.variable_dt:
            assert np.abs(u2 - out2["u_seq"][b]).max() < U_TOL   # (minimum-time optima need not be strict in the controls)
    assert (out1["status"] == 0).sum() >= 1
