"""The parity harness of the phase tests: the oracle's cold start and iterates, the shared state written into the device's
workspace or the emulator's, the phase tolerances of the CUDA kernels and of the CPU warp emulator against the oracle, one
emulator iteration in lockstep with the oracle, one line search from the oracle's iterates on the CUDA phase kernels, and the
cold-then-warm solve whose outputs are compared as bit patterns.

A state is the oracle's own iterate of one instance.  Every comparison starts from one such state on both sides, so the two
solvers never drift apart."""
import numpy as np

from fixed_cases import fixed_components
from mpc_local_planner_b200 import capi

# kernel keys (model, problem) of a launch
UNI_QF = (capi.MODEL_UNI_POINT, capi.PROBLEM_FIXED_DT_QF)
UNI = (capi.MODEL_UNI_POINT, capi.PROBLEM_GENERIC)
GEN = (capi.MODEL_GENERIC, capi.PROBLEM_GENERIC)

# the device's own bookkeeping words of SCAL: kept when the oracle's state is written into the device's workspace
DEVICE_OWN_SCAL = (capi.SC_COLD, capi.SC_VALID, capi.SC_OBST_DROPPED)
STATE_FIELDS = (("X", capi.F_X), ("U", capi.F_U), ("NU", capi.F_NU), ("S", capi.F_S), ("LAM", capi.F_LAM))
INIT_FIELDS = (capi.F_X, capi.F_U, capi.F_S, capi.F_LAM, capi.F_OBSIDX)
EVAL_SCAL = (capi.SC_MU, capi.SC_HTT, capi.SC_GT, capi.SC_ERR0, capi.SC_ERRMU, capi.SC_OBJ, capi.SC_INF, capi.SC_BLOG)

# ---- tolerances of INIT / ASSOCIATE (x: X and U absolute; s, lam: (rtol, atol)) and EVAL (kkt: the records, relative to
# their largest entry; scal: EVAL_SCAL (rtol, atol)) ----
# the CUDA kernels against the oracle
CUDA = dict(x=1e-12, s=(1e-11, 1e-13), lam=(1e-10, 1e-13), kkt=1e-11, scal=(1e-10, 1e-12))
# the CPU warp emulator against the oracle
EMU = dict(x=1e-13, s=(1e-9, 0.0), lam=(1e-9, 0.0), kkt=1e-9, scal=(1e-8, 1e-10))
# the Newton step of KKT, relative to the step's size: (tolerance, floor of the size).  At the first iterate of a cold start the
# step is well conditioned; the steps of later iterates are not (6e-8 of their size measured on the CUDA kernels), and a
# rounding-sized late step is compared against a size of 1
FIRST_STEP = (1e-9, 0.0)
LATE_STEP = (1e-7, 1.0)
# d(dt), relative to max(1, |d(dt)|)
DDT_TOL = 1e-9
# a decision (Armijo test, bin of a blocking ratio) closer than this to its threshold may go either way between two codes
DECISION_MARGIN = 1e-9


def is_midpoint(cfg):
    return cfg.collocation == capi.COLLOC_MIDPOINT


def step_rows(cfg):
    """STEP rows that the KKT phase and the oracle's Newton step share: with midpoint differences the heading multiplier row
    becomes nu+ only in the line search (ls_stage_midpoint_fix), in the oracle at the end of its Newton step"""
    return 7 if is_midpoint(cfg) else 8


def merged_scal(device_scal, oracle_scal):
    """the oracle's solver scalars with the device's own bookkeeping words"""
    s = np.array(oracle_scal, dtype=np.float64, copy=True)
    for i in DEVICE_OWN_SCAL:
        s[i] = device_scal[i]
    return s


# ---- the oracle's states ----
def oracle_init(orc, cfg, data, b, x_init=None):
    """the oracle's cold start of instance b (initial guess, association, projection, controls, duals)"""
    o = orc.instance_from_batch(cfg, data, b)
    o.init_cold(x_init); o.associate()
    o.L.orc_project_init(orc.C.byref(o.p), o.ws); o.L.orc_init_controls(orc.C.byref(o.p), o.ws)
    o.init_duals()
    return o


def oracle_iterate(orc, cfg, data, b, j):
    """The oracle's iterate j (its own solve, stopped by max_iter = j), or the last iterate before convergence (j = "last").
    Returns the instance, ready for eval(), and whether the solve converged before iterate j."""
    if j == "last":
        o = oracle_init(orc, cfg, data, b)
        r = o.solve()
        j = max(int(r.iters) - 1, 0)
    o = oracle_init(orc, cfg, data, b)
    o.cfg.max_iter = j
    r = o.solve()
    o.cfg.max_iter = cfg.max_iter
    o.arr("SCAL")[capi.SC_STATUS] = -1.0
    return o, r.status == capi.STATUS_CONVERGED


# ---- phase comparisons (one instance; the device's fields as numpy arrays) ----
def assert_init(X, U, S, LAM, OBS, o, tol, what=""):
    """INIT / ASSOCIATE: states, controls, association, slacks and multipliers (read in the order of INIT_FIELDS)"""
    np.testing.assert_allclose(X, o.arr("X"), rtol=0, atol=tol["x"], err_msg=what)
    np.testing.assert_allclose(U, o.arr("U"), rtol=0, atol=tol["x"], err_msg=what)
    np.testing.assert_array_equal(OBS, o.arr("OBSIDX"), err_msg=what)
    np.testing.assert_allclose(S, o.arr("S"), rtol=tol["s"][0], atol=tol["s"][1], err_msg=what)
    np.testing.assert_allclose(LAM, o.arr("LAM"), rtol=tol["lam"][0], atol=tol["lam"][1], err_msg=what)


def assert_eval(KKT, SC, o, tol, what="", scal=EVAL_SCAL):
    """EVAL, after o.eval(): the stage records and the solver scalars `scal`"""
    scale = np.abs(o.arr("KKT")).max()
    np.testing.assert_allclose(KKT, o.arr("KKT"), rtol=0, atol=tol["kkt"] * scale, err_msg=what)
    idx = list(scal)
    np.testing.assert_allclose(SC[idx], o.arr("SCAL")[idx], rtol=tol["scal"][0], atol=tol["scal"][1], err_msg=what)


def assert_step(cfg, STEP, ddt, o, step_tol, what="", ddt_tol=DDT_TOL):
    """KKT, after the oracle's kkt_solve at the device's regularisation: the step rows both share (step_rows), d(dt), no step
    on a fixed component of the final state (it is not a variable) and no d(dt) with a fixed dt"""
    rows = step_rows(cfg)
    tol, floor = step_tol
    sscale = max(np.abs(o.arr("STEP")).max(), floor)
    np.testing.assert_allclose(STEP[:rows], o.arr("STEP")[:rows], rtol=0, atol=tol * sscale, err_msg=what)
    for i in fixed_components(cfg):
        assert STEP[i, -1] == 0.0 and o.arr("STEP")[i, -1] == 0.0, f"{what}: step of fixed component {i}"
    ddt_o = o.arr("SCAL")[capi.SC_DDT]
    assert abs(ddt - ddt_o) <= ddt_tol * max(1.0, abs(ddt_o)), f"{what}: d(dt) {ddt!r} vs oracle {ddt_o!r}"
    if not cfg.variable_dt:
        assert ddt == 0.0 and ddt_o == 0.0, f"{what}: d(dt) {ddt!r}, oracle {ddt_o!r} with a fixed dt"


# ---- the line search of the device code against the oracle's from the same inputs ----
def near_threshold(d):
    """the oracle's diagnostics show a discrete decision within DECISION_MARGIN of its threshold: a blocking ratio's
    -2 log2(r) that close to a bin boundary, or a trial's merit that close (relative to the change of the merit it tests)
    to the Armijo or flat-merit bound.  The merit itself is a sum of terms of the size of phi0 that two codes round
    differently, by about 1e-13 phi0 measured: that much is added to the margin."""
    if len(d["phi"]) == 0:   # a null step or a stopped instance: no decision taken
        return False
    rnd = 1e-12 * (1.0 + abs(d["phi0"]))
    armijo = any(abs(p - a) <= DECISION_MARGIN * abs(p - d["phi0"]) + rnd for p, a in zip(d["phi"], d["armijo"]))
    flat_bound = 1e-13 * (1.0 + abs(d["phi0"]))
    flat = any(abs(abs(p - d["phi0"]) - flat_bound) <= DECISION_MARGIN * flat_bound + rnd for p in d["phi"][1:])
    return armijo or flat or d["bin_margin"] <= DECISION_MARGIN


def row_sensitivity(pre, G, DS, d):
    """Absolute tolerances (S, LAM per row; rho) for the inputs that each side computes itself at the shared iterate: the row
    values and gradients (the obstacle rows by each side's EVAL, the linear rows by each side's own arithmetic in the line
    search).  They differ by rounding, taken as dg = 1e-14 (1 + |g| + |g' dz|) per row.  The line search multiplies that by
    alpha in the slack, by a_dual lambda / s in the multiplier, and by (mu + 2 lambda |ds|) / s / (0.9 inf1) in rho: near
    convergence an active row's slack is of the size of mu, and these factors reach 1e8 (measured on the CUDA kernels: LAM
    1.5e-5, rho 1.3e-4 relative, both on obstacle rows; 1.2e-9 absolute on a control-rate row at k = 0).
    pre: S, LAM and SCAL before the line search; G, DS: the oracle's row values and slack steps; d: its diagnostics."""
    S, LAM = pre["S"], pre["LAM"]
    obst = LAM > 0
    gdz = -(DS + G + S)
    dg = np.where(obst, 1e-14 * (1.0 + np.abs(G) + np.abs(gdz)), 0.0)
    sig = np.where(obst, LAM / np.where(obst, S, 1.0), 0.0)
    tol_s = d["alpha"] * dg
    tol_lam = d["a_dual"] * sig * dg
    inf1 = pre["SCAL"][capi.SC_INF]
    mu = pre["SCAL"][capi.SC_MU]
    num = (np.where(obst, mu / np.where(obst, S, 1.0), 0.0) * dg + 2.0 * sig * np.abs(DS) * dg).sum()
    tol_rho = num / (0.9 * inf1) if inf1 > 1e-14 else 0.0
    return dict(S=tol_s, LAM=tol_lam, rho=tol_rho)


def assert_same_outcome(cfg, d, o_arrs, o_scal, dev_arrs, dev_scal, what, rtol=1e-13, rho_tol=1e-10, sens=None):
    """The line search of the device code against the oracle's from the same inputs.  The discrete outcomes must be equal;
    a different decision is excused only when the oracle's diagnostics put it within DECISION_MARGIN of its threshold, and
    then nothing else is compared (returns True).  When both sides decided alike, everything is compared (returns False).
    sens: row_sensitivity, for the inputs that each side computes itself."""
    same = all(dev_scal[i] == o_scal[i] for i in (capi.SC_NBT, capi.SC_ITER, capi.SC_TINY, capi.SC_STATUS))
    if not same and d is not None and near_threshold(d):
        return True
    for i in (capi.SC_NBT, capi.SC_ITER, capi.SC_TINY, capi.SC_STATUS):
        assert dev_scal[i] == o_scal[i], f"{what}: SCAL[{i}] {dev_scal[i]} vs oracle {o_scal[i]}"
    # rho = (dJ + dphi_bar + curv / 2) / (0.9 inf1) + 1: sums over the rows and stages, accumulated in another order, whose
    # terms cancel and whose quotient by a small inf1 near convergence magnifies that rounding (up to 1e-12 measured)
    for i, tol, extra in ((capi.SC_DT, rtol, 0.0), (capi.SC_ALPHA, rtol, 0.0),
                          (capi.SC_RHO, rho_tol, sens["rho"] if sens else 0.0)):
        assert abs(dev_scal[i] - o_scal[i]) <= tol * abs(o_scal[i]) + extra, \
            f"{what}: SCAL[{i}] {dev_scal[i]!r} vs oracle {o_scal[i]!r}"
    for nm, _ in STATE_FIELDS:
        a, b = dev_arrs[nm], o_arrs[nm]
        # with midpoint differences the heading multiplier row of the step is the device's own (see step_rows), so NU agrees
        # to the tolerance of the Newton step only
        tol = LATE_STEP[0] if nm == "NU" and is_midpoint(cfg) else rtol
        bound = tol * max(1.0, np.abs(b).max()) + (sens[nm] if sens and nm in sens else 0.0)
        excess = np.abs(a - b) - bound
        assert (excess <= 0).all(), \
            f"{what}: {nm} differs by {np.abs(a - b).max():.3e}, worst at {np.unravel_index(np.argmax(excess), a.shape)}"
    return False


def oracle_linesearch_and_compare(cfg, o, dev_arrs, dev_scal, what, rho_tol=1e-10):
    """the oracle's line search on its state, then the device's result against it; returns (diagnostics, marginal)"""
    pre = {nm: o.arr(nm).copy() for nm in ("S", "LAM", "SCAL")}
    d = o.linesearch()
    sens = row_sensitivity(pre, o.arr("G"), o.arr("DS"), d)
    marginal = assert_same_outcome(cfg, d, {nm: o.arr(nm) for nm, _ in STATE_FIELDS}, o.arr("SCAL"), dev_arrs, dev_scal,
                                   what, rho_tol=rho_tol, sens=sens)
    return d, marginal


# ---- the CPU warp emulator ----
def emu_set_state(e, o):
    """the oracle's iterate into the emulator's workspace"""
    for nm, f in STATE_FIELDS:
        e.set_field(f, o.arr(nm))
    e.set_field(capi.F_SCAL, merged_scal(e.field(capi.F_SCAL), o.arr("SCAL")))


def emu_from_oracle(emu, cfg, data, b, o):
    """an emulator instance with the device's own initialisation and association, then the oracle's iterate"""
    e = emu.instance_from_batch(cfg, data, b)
    e.init(); e.associate()
    np.testing.assert_array_equal(e.field(capi.F_OBSIDX), o.arr("OBSIDX"))
    emu_set_state(e, o)
    return e


def emu_init_fields(e):
    return [e.field(f) for f in INIT_FIELDS]


def emu_assert_eval(o, e, what="", scal=EVAL_SCAL):
    """EVAL on both sides, compared"""
    o.eval(); e.eval()
    assert_eval(e.field(capi.F_KKT), e.field(capi.F_SCAL), o, EMU, what, scal)


def eval_and_kkt(o, e, cfg, step_tol=LATE_STEP, ddt_tol=DDT_TOL):
    """EVAL and KKT on both sides, compared; False when the device defers the step"""
    emu_assert_eval(o, e)
    assert e.kkt() == 0
    if e.field(capi.F_SCAL)[capi.SC_DEFER] != 0.0:
        return False
    if o.kkt_solve(e.field(capi.F_SCAL)[capi.SC_DELTA]) != 0:
        # an inertia decision at the margin (seen on rounding-sized steps): the line search gets the oracle's step anyway
        assert step_tol[0] > LATE_STEP[0] and any(o.kkt_solve(dl) == 0 for dl in (1e-4, 1e-2, 1.0, 100.0))
        return True
    assert_step(cfg, e.field(capi.F_STEP), e.field(capi.F_SCAL)[capi.SC_DDT], o, step_tol, ddt_tol=ddt_tol)
    return True


def share_inputs(o, e, cfg):
    """the oracle's records, step and scalars into the emulator: both line searches start from bit-identical inputs"""
    e.set_field(capi.F_KKT, o.arr("KKT"))
    rows = step_rows(cfg)
    STEP = e.field(capi.F_STEP).copy()
    STEP[:rows] = o.arr("STEP")[:rows]
    e.set_field(capi.F_STEP, STEP)
    e.set_field(capi.F_SCAL, merged_scal(e.field(capi.F_SCAL), o.arr("SCAL")))


def run_both(o, e, cfg, what, post=None, rho_tol=1e-10):
    """share the inputs, run one line search on each side, compare; returns (diagnostics, marginal, SCAL before)"""
    if post is not None:
        post(o)
    share_inputs(o, e, cfg)
    before = o.arr("SCAL").copy()
    e.linesearch()
    d, marginal = oracle_linesearch_and_compare(cfg, o, {nm: e.field(f) for nm, f in STATE_FIELDS}, e.field(capi.F_SCAL),
                                                what, rho_tol)
    return d, marginal, before


def emu_iterate(o, e, cfg, what):
    """One interior-point iteration of the emulator in lockstep with the oracle from a shared state: records, scalars (dt
    included) and the association after EVAL; the step after KKT (the emulator's regularisation bookkeeping is the one both
    continue with; a deferred step is a null step on both sides); one line search each from the oracle's records, step and
    scalars, and the step rows the line search finishes; then the oracle's iterate is the shared state.  Returns (stepped,
    marginal)."""
    emu_assert_eval(o, e, what, (capi.SC_DT,) + EVAL_SCAL)
    np.testing.assert_array_equal(e.field(capi.F_OBSIDX), o.arr("OBSIDX"), err_msg=what)
    assert e.kkt() == 0
    for i in (capi.SC_DELTA_LAST, capi.SC_NREG):
        o.arr("SCAL")[i] = e.field(capi.F_SCAL)[i]
    stepped = e.field(capi.F_SCAL)[capi.SC_DEFER] == 0.0
    if not stepped:
        # factorisation budget spent: null step, the escalation resumes at DELTA_LAST / 3 in the next iteration
        nxt = e.field(capi.F_SCAL)[capi.SC_DELTA_LAST] / 3.0
        assert o.kkt_solve(nxt / 8.0) == 1 or o.kkt_solve(nxt / 100.0) == 1
        o.arr("SCAL")[capi.SC_DEFER] = 1.0
        _, marginal, _ = run_both(o, e, cfg, f"{what} (null step)")
    else:
        assert o.kkt_solve(e.field(capi.F_SCAL)[capi.SC_DELTA]) == 0
        assert_step(cfg, e.field(capi.F_STEP), e.field(capi.F_SCAL)[capi.SC_DDT], o, LATE_STEP, what)
        _, marginal, _ = run_both(o, e, cfg, what)
        # midpoint differences: the device turns the heading multiplier of the condensed system into nu+ at the start of the
        # line search (ls_stage_midpoint_fix), the oracle at the end of its solve; that row is compared after it
        rows = step_rows(cfg)
        sscale = max(np.abs(o.arr("STEP")).max(), LATE_STEP[1])
        np.testing.assert_allclose(e.field(capi.F_STEP)[rows:], o.arr("STEP")[rows:], atol=LATE_STEP[0] * sscale,
                                   err_msg=what)
    emu_set_state(e, o)
    return stepped, marginal


# ---- the CUDA phase kernels ----
def phase_solver(cfg, data, B, force_generic=0):
    """a BatchSolver for the phase API with the batch uploaded"""
    s = capi.BatchSolver(cfg, B, device=0)
    s.set_option(capi.OPT_FORCE_GENERIC_MODEL, force_generic)
    s.upload(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
    return s


def write_state(s, inst):
    """the oracle's iterates (one per instance) into the device's workspace"""
    for nm, f in STATE_FIELDS:
        s.ws_write(f, np.stack([o.arr(nm) for o in inst]))
    SC = s.ws_read(capi.F_SCAL)
    s.ws_write(capi.F_SCAL, np.stack([merged_scal(SC[b], o.arr("SCAL")) for b, o in enumerate(inst)]))


def compare_at(orc, cfg, data, B, j, force_generic=0, keys=None, post=None):
    """One line search on B instances from the oracle's iterate j; returns (compared, marginal) instance counts.  The
    device's INIT and ASSOCIATE must give the oracle's association; EVAL and KKT run on the device from the oracle's state and
    are compared; then both line searches start from the oracle's records, step and scalars.  post: an edge change applied to
    the oracle's state after its Newton step; every instance must then take a step at the right inertia."""
    s = phase_solver(cfg, data, B, force_generic)
    s.run_phase(capi.PHASE_INIT); s.run_phase(capi.PHASE_ASSOCIATE)
    if keys is not None:
        assert (s.kernel_model(), s.kernel_problem()) == keys
    OBS = s.ws_read(capi.F_OBSIDX)
    inst, live = [], []
    for b in range(B):
        o, converged = oracle_iterate(orc, cfg, data, b, j)
        np.testing.assert_array_equal(OBS[b], o.arr("OBSIDX"))
        inst.append(o)
        live.append(not converged)
    write_state(s, inst)
    s.run_phase(capi.PHASE_EVAL)
    KKT, SC = s.ws_read(capi.F_KKT), s.ws_read(capi.F_SCAL)
    s.run_phase(capi.PHASE_KKT)
    STEP, SC2 = s.ws_read(capi.F_STEP).copy(), s.ws_read(capi.F_SCAL)
    rows = step_rows(cfg)
    for b, o in enumerate(inst):
        o.eval()
        if post is not None:
            assert live[b] and SC2[b][capi.SC_DEFER] == 0.0, f"instance {b}: no step to change"
        if not live[b]:
            continue
        assert_eval(KKT[b], SC[b], o, CUDA, f"instance {b}, iterate {j}")
        if SC2[b][capi.SC_DEFER] != 0.0:
            o.arr("SCAL")[capi.SC_DEFER] = 1.0   # both take the null step
            continue
        if o.kkt_solve(SC2[b][capi.SC_DELTA]) != 0:
            # an inertia decision at the margin: the line search gets the oracle's own step anyway
            assert post is None and any(o.kkt_solve(dl) == 0 for dl in (1e-4, 1e-2, 1.0, 100.0))
            continue
        assert_step(cfg, STEP[b], SC2[b][capi.SC_DDT], o, LATE_STEP, f"instance {b}, iterate {j}")
        if post is not None:
            post(o)
    # identical line-search inputs: the oracle's records, step (the device's heading multiplier row with midpoint
    # differences) and scalars
    s.ws_write(capi.F_KKT, np.stack([o.arr("KKT") for o in inst]))
    for b, o in enumerate(inst):
        STEP[b][:rows] = o.arr("STEP")[:rows]
    s.ws_write(capi.F_STEP, STEP)
    for b, o in enumerate(inst):
        if not live[b]:
            o.arr("SCAL")[capi.SC_STATUS] = SC2[b][capi.SC_STATUS]   # converged on both sides: nothing may change
    s.ws_write(capi.F_SCAL, np.stack([merged_scal(SC2[b], o.arr("SCAL")) for b, o in enumerate(inst)]))
    s.run_phase(capi.PHASE_LINESEARCH)
    dev = {nm: s.ws_read(f) for nm, f in STATE_FIELDS}
    DSC = s.ws_read(capi.F_SCAL)
    if keys is not None:
        assert (s.kernel_model(), s.kernel_problem()) == keys
    s.close()
    compared = marginal = 0
    for b, o in enumerate(inst):
        _, m = oracle_linesearch_and_compare(cfg, o, {nm: dev[nm][b] for nm, _ in STATE_FIELDS}, DSC[b],
                                             f"instance {b}, iterate {j}")
        compared += live[b]
        marginal += m
    return compared, marginal


def check_first_iterate(orc, cfg, data, B):
    """INIT / ASSOCIATE / EVAL / KKT of the phase kernels against the oracle's cold start; the step and d(dt) at the
    regularisation the kernel settled on (delta = 0 where the inertia was right).  Returns the number of instances whose
    steps were compared."""
    s = phase_solver(cfg, data, B)
    s.run_phase(capi.PHASE_INIT); s.run_phase(capi.PHASE_ASSOCIATE)
    init = [s.ws_read(f) for f in INIT_FIELDS]
    s.run_phase(capi.PHASE_EVAL)
    KKT, SC = s.ws_read(capi.F_KKT), s.ws_read(capi.F_SCAL)
    s.run_phase(capi.PHASE_KKT)
    STEP, SC2 = s.ws_read(capi.F_STEP), s.ws_read(capi.F_SCAL)
    s.close()
    n_steps = 0
    for b in range(B):
        o = oracle_init(orc, cfg, data, b)
        assert_init(*(a[b] for a in init), o, CUDA, f"instance {b}")
        o.eval()
        assert_eval(KKT[b], SC[b], o, CUDA, f"instance {b}")
        if SC2[b][capi.SC_DEFER] != 0.0:
            assert o.kkt_solve(0.0) == 1   # factorisation budget spent at this iterate: wrong inertia at delta = 0 for both
            continue
        delta = SC2[b][capi.SC_DELTA]
        if delta != 0.0:
            assert o.kkt_solve(0.0) == 1   # both see the wrong inertia at delta = 0; the regularised steps are compared
        assert o.kkt_solve(delta) == 0
        assert_step(cfg, STEP[b], SC2[b][capi.SC_DDT], o, FIRST_STEP, f"instance {b}")
        n_steps += 1
    return n_steps


# ---- whole solves compared bit for bit ----
SOLVE_FIELDS = ("status", "iters", "u_seq", "x_seq", "dt", "kkt_err")


def bits(a):
    """floats as their bit patterns: a -0.0 against 0.0 or a differently contracted expression is a difference"""
    a = np.ascontiguousarray(a)
    return a.view(np.uint64) if a.dtype == np.float64 else a


def solve_twice(cfg, data, B, mode=capi.SOLVE_FUSED, force_generic=0):
    """the batch solved cold, then warm from the first solve; returns (the two outputs, (kernel_model, kernel_problem))"""
    s = capi.BatchSolver(cfg, B, device=0)
    s.set_option(capi.OPT_SOLVE_MODE, mode)
    s.set_option(capi.OPT_FORCE_GENERIC_MODEL, force_generic)
    outs = []
    for _ in range(2):
        out = s.step(data["x0"], data["xf"], data["u_prev"], data["u_prev_dt"], data["obstacles"], data["viapoints"])
        outs.append({f: np.array(out[f], copy=True) for f in SOLVE_FIELDS})
    keys = (s.kernel_model(), s.kernel_problem())
    s.close()
    return outs, keys


def assert_same_solves(outs_a, outs_b, what):
    for step, (a, b) in enumerate(zip(outs_a, outs_b)):
        for f in SOLVE_FIELDS:
            assert np.array_equal(bits(a[f]), bits(b[f])), f"step {step}: {f} differs between {what}"
