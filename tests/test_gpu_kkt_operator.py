"""The KKT phase kernel (kkt_warp_kernel, one warp per instance) as an operator on synthetic stage records
(tests/kkt_cases.py): against the dense solution of the records at every horizon shape and variant of the CPU tests
(tests/test_kkt_operator.py), against the CPU warp emulator of the same header, the inertia and schedule cases, skipped
instances, and the fused solve kernel (whose warp 0 runs the same sweep) against the phased one at the new horizons.

CUDA_TOL = (normwise backward error, forward error relative to the largest unknown).  Measured maxima on an NVIDIA H100
80GB HBM3 (700 W power limit), B = 4 instances per horizon:
    backward 1.8e-16 (fixed dt, final state fixed; every other variant <= 1.1e-16)
    forward  1.2e-14 (the same variant; every other variant <= 2.9e-15)
EMU_TOL: the kernel against the emulator on the same records, relative to the largest entry of the step.  g++ and nvcc
contract multiply-adds differently, so the two agree to rounding, not bit for bit: measured 1.1e-14 (the same variant, whose
steps are the worst conditioned), <= 3.9e-15 elsewhere.  Both bounds leave about 10x."""
import numpy as np
import pytest

import kkt_cases as kc
import parity as par
from mpc_local_planner_b200 import capi, configs

pytestmark = pytest.mark.gpu

CUDA_TOL = (2e-15, 1.2e-13)
EMU_TOL = 1.2e-13
B = 4


class Phase:
    """one handle per variant, created at the variant's largest horizon and moved to shorter ones with resample()"""

    def __init__(self, cfg, n_cap, B):
        c = cfg.copy()
        c.n = n_cap
        self.s = capi.BatchSolver(c, B)

    def run(self, recs, scals, steps):
        """the KKT phase on instances with records recs [b][KW][N], SCAL scals and STEP steps; (STEP, SCAL) after it"""
        N = recs[0].shape[1]
        if self.s.N != N:
            self.s.resample(N)
        Bn = len(recs)
        self.s.ws_write(capi.F_KKT, np.stack(recs))
        self.s.ws_write(capi.F_SCAL, np.stack(scals))
        self.s.ws_write(capi.F_STEP, np.stack(steps))
        self.s.run_phase(capi.PHASE_KKT, Bn)
        return self.s.ws_read(capi.F_STEP, Bn), self.s.ws_read(capi.F_SCAL, Bn)

    def run_one(self, cfg, R, htt, gt, dlast=0.0, nreg=0.0):
        STEP, SC = self.run([R], [kc.scal_words(htt, gt, dlast, nreg)], [kc.step_sentinel(R.shape[1])])
        return STEP[0], SC[0]

    def close(self):
        self.s.close()


_phases = {}


def phase_for(name, xf=(0, 0, 0)):
    if (name, xf) not in _phases:
        _phases[(name, xf)] = Phase(kc.variant_config(name, xf), kc.n_max(name, xf), B)
    return _phases[(name, xf)]


@pytest.fixture(scope="module", autouse=True)
def _close_handles():
    yield
    for ph in _phases.values():
        ph.close()
    _phases.clear()


def instance_seed(name, xf, b):
    """the seed of instance b of a variant's batch: the same at every horizon"""
    return kc.seed_of(name, xf, 0, 1 + b)


def check_batch(emu, name, xf):
    """The KKT phase on a batch of B instances at every horizon of the variant: each against the dense solution, the exact
    properties, the bookkeeping of a solve at delta = 0, and the emulator.  Returns the worst (backward, forward, kernel -
    emulator)."""
    ph = phase_for(name, xf)
    worst = np.zeros(3)
    for N in kc.horizons(name, xf):
        cfg = kc.variant_config(name, xf)
        cfg.n = N
        cases = [kc.make_records(cfg, N, instance_seed(name, xf, b)) for b in range(B)]
        STEP, SC = ph.run([c[0] for c in cases], [kc.scal_words(c[1], c[2], 0.0, 2.0) for c in cases], [kc.step_sentinel(N)] * B)
        for b, (R, htt, gt) in enumerate(cases):
            what = f"{name} xf={xf} N={N} instance {b}"
            d = kc.Dense(cfg, R, htt, gt)
            z = d.solve(0.0)
            kc.assert_outcome(SC[b], kc.store_outcome(kc.scal_words(htt, gt, 0.0, 2.0), True, d.unpack(z)[1], 0.0, 0), what)
            kc.assert_exact_properties(cfg, STEP[b], SC[b], what)
            bwd, fwd = kc.assert_accuracy(d, 0.0, STEP[b], SC[b][capi.SC_DDT], z, CUDA_TOL, what)
            ESTEP, ESC = kc.run_emulator(emu, cfg, R, htt, gt, nreg=2.0)
            scale = np.abs(ESTEP).max()
            de = max(np.abs(STEP[b] - ESTEP).max(), abs(SC[b][capi.SC_DDT] - ESC[capi.SC_DDT])) / scale
            assert de <= EMU_TOL, f"{what}: kernel and emulator differ by {de:.2e} of the step"
            assert all(SC[b][i] == ESC[i] for i in range(capi.SCAL_WORDS) if i != capi.SC_DDT), what
            worst = np.maximum(worst, (bwd, fwd, de))
    return worst


@pytest.mark.parametrize("name", ["fixed", "free_dt"])
def test_every_horizon(cuda_lib, emu, name):
    """Both sweep templates at every horizon shape of the forward substitution, up to the largest horizon that fits."""
    check_batch(emu, name, (0, 0, 0))


@pytest.mark.parametrize("name,xf", kc.CROSS)
def test_variants(cuda_lib, emu, name, xf):
    """Every configuration that changes what the sweep reads, at the reduced horizon list."""
    check_batch(emu, name, xf)


def test_inertia(cuda_lib):
    """The inertia cases of the CPU tests: never a solve at a wrong inertia; with a free final state the schedule's outcome."""
    cases = kc.inertia_cases()
    conservative = 0
    for case in cases:
        name, xf = case[0], case[1]
        run = phase_for(name, xf).run_one
        conservative += sum(kc.check_inertia(run, CUDA_TOL, *case, dlast) for dlast in kc.INERTIA_DLASTS)
    assert conservative <= len(cases) // 10, f"{conservative} conservative failures"


def test_schedule(cuda_lib):
    """The schedule cases of the CPU tests: every word of SCAL, and STEP untouched without a solve."""
    outcomes = {kc.check_schedule(phase_for(case[0]).run_one, *case) for case in kc.schedule_cases()}
    assert outcomes == kc.SCHEDULE_OUTCOMES, outcomes


def test_skipped_instances(cuda_lib):
    """Instances with SC_VALID = 0 or a final status (SC_STATUS >= 0) mixed into a batch keep STEP and SCAL bit for bit; the
    live instances give the results of a batch without them."""
    for name in ("fixed", "free_dt"):
        ph = phase_for(name)
        for N in (5, 34, kc.n_max(name)):
            cfg = kc.variant_config(name)
            cfg.n = N
            live = [kc.make_records(cfg, N, instance_seed(name, (0, 0, 0), b)) for b in range(2)]
            recs = [c[0] for c in live]
            scals = [kc.scal_words(c[1], c[2], 0.0) for c in live]
            steps = [kc.step_sentinel(N)] * 2
            ref_step, ref_sc = ph.run(recs, scals, steps)
            dead = kc.make_records(cfg, N, instance_seed(name, (0, 0, 0), 7))
            invalid = kc.scal_words(dead[1], dead[2], 0.0); invalid[capi.SC_VALID] = 0.0
            done = kc.scal_words(dead[1], dead[2], 0.0); done[capi.SC_STATUS] = float(capi.STATUS_CONVERGED)
            order = [("live", 0), ("skip", invalid), ("live", 1), ("skip", done)]
            mixed = [(recs[x], scals[x], steps[x]) if kind == "live" else (dead[0], x, kc.step_sentinel(N) + 0.5) for kind, x in order]
            STEP, SC = ph.run(*zip(*mixed))
            for j, (kind, x) in enumerate(order):
                if kind == "live":
                    assert np.array_equal(par.bits(STEP[j]), par.bits(ref_step[x])) and np.array_equal(par.bits(SC[j]), par.bits(ref_sc[x]))
                else:
                    assert np.array_equal(par.bits(STEP[j]), par.bits(mixed[j][2])) and np.array_equal(par.bits(SC[j]), par.bits(x))


@pytest.mark.parametrize("case", ["uni_qf", "free_dt_fixed_final_state"])
def test_fused_equals_phased_at_new_horizons(cuda_lib, case):
    """The fused solve kernel runs the sweep on warp 0: its cold and warm solves equal the phased ones bit for bit at
    N = 3, 34, 65 and the largest horizon the configuration fits -- a fixed-dt quadratic-form unicycle with a point footprint
    (the UNI_QF kernel key, unbordered sweep) and a free dt with a fixed final state (bordered sweep)."""
    cfg = configs.cfg2(tol=1e-8) if case == "uni_qf" else configs.cfg1(tol=1e-8)
    Bn = 8
    for N in (3, 34, 65, kc.largest_horizon(cuda_lib, cfg)):
        c = cfg.copy()
        c.n = N
        data = configs.generate(2, Bn, n=N)
        fused, keys_f = par.solve_twice(c, data, Bn, capi.SOLVE_FUSED)
        phased, keys_p = par.solve_twice(c, data, Bn, capi.SOLVE_PHASED)
        assert keys_f == keys_p and (case != "uni_qf" or keys_f == par.UNI_QF), keys_f
        par.assert_same_solves(fused, phased, f"the fused and the phased solve at N = {N}")
