"""The KKT phase as an operator on synthetic stage records (tests/kkt_cases.py), on the CPU warp emulator of
mpc_riccati_warp.h and on the oracle's serial sweep, against the dense KKT system of the same records solved in extended
precision: every horizon shape of the forward substitution, every configuration that changes what the sweep reads, the
words it must ignore, the inertia test and the regularisation schedule.

TOL = (normwise backward error in long double, forward error relative to the largest unknown).  Measured maxima on the
generated cases (emulator: g++ -O2 -march=x86-64-v3):
    emulator, fixed / free dt, every horizon     backward 1.2e-16 / 4.0e-17   forward 2.3e-15 / 2.6e-15
    emulator, other variants, reduced horizons   backward 5.1e-16 (free dt, final state fixed, N = 3; the rest <= 8.4e-17)
                                                 forward 5.4e-15
    emulator, regularised steps (inertia cases)  backward 8.1e-17             forward 2.3e-15
    oracle, non-midpoint variants                backward 6.7e-17             forward 3.8e-15
The bounds leave about 10x over the largest of them."""
import functools

import numpy as np
import pytest

import kkt_cases as kc
from mpc_local_planner_b200 import capi

TOL = (5e-15, 6e-14)


def check_emulator(emu, name, xf, N, tol=TOL):
    """One case on the emulator: solved at delta = 0 with the bookkeeping of a step, the exact properties, bit for bit the
    same with the ignored words zeroed, and accurate against the dense solution.  Returns (backward, forward)."""
    cfg = kc.variant_config(name, xf)
    cfg.n = N
    R, htt, gt = kc.make_records(cfg, N, kc.seed_of(name, xf, N))
    what = f"{name} xf={xf} N={N}"
    STEP, SC = kc.run_emulator(emu, cfg, R, htt, gt, nreg=2.0)
    d = kc.Dense(cfg, R, htt, gt)
    z = d.solve(0.0)
    kc.assert_outcome(SC, kc.store_outcome(kc.scal_words(htt, gt, 0.0, 2.0), True, d.unpack(z)[1], 0.0, 0), what)
    kc.assert_exact_properties(cfg, STEP, SC, what)
    R0, htt0, gt0 = kc.zero_ignored(cfg, R, htt, gt)
    STEP0, SC0 = kc.run_emulator(emu, cfg, R0, htt0, gt0, nreg=2.0)
    SC0[capi.SC_HTT], SC0[capi.SC_GT] = SC[capi.SC_HTT], SC[capi.SC_GT]
    assert (STEP0 == STEP).all() and (SC0 == SC).all(), f"{what}: the step depends on words the sweep must ignore"
    return kc.assert_accuracy(d, 0.0, STEP, SC[capi.SC_DDT], z, tol, what)


@pytest.mark.parametrize("name", ["fixed", "free_dt"])
def test_every_horizon(emu, cuda_lib, name):
    """Both sweep templates (fixed dt and free final state: unbordered; free dt: bordered) at every horizon shape of the
    forward substitution -- N = 3 .. 70, the chunk transitions around 96, 128, 160 and 192, and the largest horizon
    mpcb200_create accepts -- against the dense solution."""
    hs = kc.horizons(name)
    assert hs[-1] == kc.n_max(name) and kc.chunk(hs[-1]) >= 7
    for N in hs:
        check_emulator(emu, name, (0, 0, 0), N)


@pytest.mark.parametrize("name,xf", kc.CROSS)
def test_variants(emu, cuda_lib, name, xf):
    """Every configuration that changes what the sweep reads (terminal dt border: trapezoidal cost, midpoint differences;
    each fixed final state pattern with a fixed and a free dt) at the reduced horizon list."""
    for N in kc.horizons(name, xf):
        check_emulator(emu, name, xf, N)


def test_inertia(emu):
    """Indefinite records: the sweep never solves at a wrong inertia; with a free final state every word of SCAL follows
    the schedule driven by the dense inertia.  Conservative failures with a fixed final state stay rare (measured: 9 of the
    300 phases)."""
    run = functools.partial(kc.run_emulator, emu)
    cases = kc.inertia_cases()
    conservative = sum(kc.check_inertia(run, TOL, *case, dlast) for case in cases for dlast in kc.INERTIA_DLASTS)
    assert conservative <= len(cases) // 10, f"{conservative} conservative failures"


def test_positive_definite_solves_without_regularisation(emu):
    """A free final state and a Hessian whose eigenvalues spread over six decades: solved at delta = 0 (the pivot test is
    not stricter than the inertia)."""
    for name in ("fixed", "free_dt", "trap"):
        for lam_min, lam_max in ((1e-3, 1e3), (1e-6, 1.0), (1.0, 1e6)):
            for N in (3, 34, 97):
                cfg = kc.variant_config(name)
                cfg.n = N
                R, htt, gt = kc.make_records(cfg, N, kc.seed_of(name, (0, 0, 0), N, 5), lam_min=lam_min, lam_max=lam_max)
                _, SC = kc.run_emulator(emu, cfg, R, htt, gt)
                assert SC[capi.SC_DEFER] == 0.0 and SC[capi.SC_DELTA] == 0.0 and SC[capi.SC_NREG] == 0.0, \
                    f"{name} N={N} eigenvalues in [{lam_min}, {lam_max}]"


def test_schedule(emu):
    """DEFER, DELTA, DELTA_LAST, NREG, DDT and STATUS against the Python schedule driven by the dense inertia, for every last
    regularisation and indefiniteness whose threshold is clear of the candidates.  The cases reach a solve at the first and
    at the second attempt, a deferral and NUMERICAL_ERROR."""
    run = functools.partial(kc.run_emulator, emu)
    outcomes = {kc.check_schedule(run, *case) for case in kc.schedule_cases()}
    assert outcomes == kc.SCHEDULE_OUTCOMES, outcomes


@pytest.mark.parametrize("name,xf", [("fixed", (0, 0, 0)), ("free_dt", (0, 0, 0)), ("trap", (0, 0, 0))]
                         + [("xf_fixed", p) for p in kc.XF_PATTERNS] + [("xf_fixed_dt", p) for p in kc.XF_PATTERNS])
def test_oracle_sweep(orc, cuda_lib, name, xf):
    """orc_kkt_solve, the serial Riccati sweep the device steps are compared with elsewhere, on the same records against the
    dense solution (not midpoint differences: the oracle's Newton step post-processes the heading multiplier from the
    iterate).  A fault here is in the recursion both implementations share, not in the warp sweep."""
    for N in kc.reduced_horizons(kc.n_max(name, xf)):
        cfg = kc.variant_config(name, xf)
        cfg.n = N
        R, htt, gt = kc.make_records(cfg, N, kc.seed_of(name, xf, N))
        ok, STEP, ddt = kc.run_oracle(orc, cfg, R, htt, gt, 0.0)
        what = f"{name} xf={xf} N={N}"
        assert ok, what
        d = kc.Dense(cfg, R, htt, gt)
        kc.assert_accuracy(d, 0.0, STEP, ddt, d.solve(0.0), TOL, what)
        assert all(STEP[i, -1] == 0.0 for i in range(3) if cfg.xf_fixed[i]) and (cfg.variable_dt or ddt == 0.0), what
