"""The interior-point line search (step lengths, clip histogram, l1 merit, backtracking, update) on the CPU.

- The oracle's line search (orc_linesearch) against independent checks: its directional derivative dJ against a central
  difference of the objective itself, its curvature against the dense Hessian, and its step-length rules and update
  recomputed in numpy.  The dJ check is the one that does not rest on a second restatement of the same formula.
- The device code (the host/device headers, replayed by the CPU warp emulator) against the oracle, from one shared state:
  the oracle's own iterate j, written into the emulator's workspace, evaluated and factorised on both sides, and then given
  bit-identical line-search inputs (records, step, scalars)."""
import numpy as np
import pytest

import dense_kkt as dk
import linesearch_cases as lc
import parity as par
from mpc_local_planner_b200 import capi

# ---- the oracle's line search against independent checks -------------------------------------------------------------

DJ_CASES = ["cfg2", "integral_fixed_dt", "integral_free_dt", "trapezoid_fixed_dt", "trapezoid_free_dt", "hybrid_min_time",
            "cfg1", "cfg3", "cfg4", "vp_ordered_orientation"]


def _oracle_step(orc, cfg, data, b, j):
    """the oracle's iterate j, evaluated and factorised (the solve's first inertia attempt, else the next regularisations)"""
    o, _ = par.oracle_iterate(orc, cfg, data, b, j)
    o.eval()
    dl = o.arr("SCAL")[capi.SC_DELTA_LAST]
    for delta in ([dl / 3.0] if dl > 0 else []) + [0.0, 1e-4, 1e-2, 1.0, 100.0]:
        if o.kkt_solve(delta) == 0:
            return o
    pytest.fail("no regularisation gave the right inertia")


@pytest.mark.parametrize("name", DJ_CASES)
def test_dJ_is_the_derivative_of_the_objective(orc, name):
    """dJ (the objective's directional derivative along (dX, dU, d(dt))) against a central difference of orc_objective.
    Objective variants: quadratic form with terminal cost, integral form (left sum and trapezoid) with a fixed and a free dt,
    hybrid minimum time, minimum time, via-points unordered and ordered with an orientation weight."""
    cfg, data, b = lc.case(name)
    for j in (0, 1, 3):
        o = _oracle_step(orc, cfg, data, b, j)
        X, U = o.arr("X").copy(), o.arr("U").copy()
        dt, ddt = o.arr("SCAL")[capi.SC_DT], o.arr("SCAL")[capi.SC_DDT]
        dX, dU = o.arr("STEP")[:3].copy(), o.arr("STEP")[3:5].copy()
        dU[:, -1] = 0.0
        scale = max(np.abs(dX).max(), np.abs(dU).max(), abs(ddt))
        h = 1e-5 / scale
        J = lambda t: o.objective(X + t * dX, U + t * dU, dt + t * ddt)
        fd = (J(h) - J(-h)) / (2 * h)
        d = o.linesearch()
        # central differences are exact for the quadratic terms; the dt-weighted ones leave O(h^2) terms
        assert abs(d["dJ"] - fd) <= 1e-6 * max(1.0, abs(fd)) + 1e-9 * abs(J(0.0)) / (h * scale), \
            f"{name} iterate {j}: dJ {d['dJ']!r} vs central difference {fd!r}"


@pytest.mark.parametrize("cid", [2, 21, 24, 26, 3])
def test_curvature_matches_the_dense_hessian(orc, cid):
    """curv = dz'(H + delta I)dz + sum sigma ds^2, with H the condensed Hessian of the dense KKT system (finite differences of
    the analytic gradient, the same assembly the Newton-step test uses): the block, the control-rate cross blocks and the dt
    border of the stage records."""
    inst, cfg = dk.random_iterate(orc, cid, 1, 0, 0.05)
    Hc, _, _, _, free = dk.dense_kkt(inst, cfg)
    N = inst.N
    for delta in (0.0, 1e-2, 1.0, 100.0):
        if inst.kkt_solve(delta) == 0:
            break
    else:
        pytest.fail("no regularisation gave the right inertia")
    STEP, ddt = inst.arr("STEP").copy(), inst.arr("SCAL")[capi.SC_DDT]
    sig = np.where(inst.arr("LAM") > 0, inst.arr("LAM") / inst.arr("S"), 0.0)
    dz = np.zeros(5 * N + 1); dz[:3 * N] = STEP[:3].ravel(); dz[3 * N:5 * N] = STEP[3:5].ravel(); dz[5 * N] = ddt
    dz[3 * N + N - 1] = dz[4 * N + N - 1] = 0.0
    d = inst.linesearch()
    dzf = dz[free]
    ds = inst.arr("DS")
    expected = dzf @ (Hc[np.ix_(free, free)] + delta * np.eye(len(free))) @ dzf + (sig * ds * ds).sum()
    scale = np.abs(dzf) @ (np.abs(Hc[np.ix_(free, free)]) + delta * np.eye(len(free))) @ np.abs(dzf) + (sig * ds * ds).sum()
    assert abs(d["curv"] - expected) <= 1e-5 * scale, (d["curv"], expected, scale)


def _step_rules(o, pre, d, cfg):
    """the oracle's step lengths and update recomputed in numpy from DS, DLAM and the state before the line search"""
    N = o.N
    mu = pre["SCAL"][capi.SC_MU]
    S, LAM, DS, DLAM = pre["S"], pre["LAM"], o.arr("DS"), o.arr("DLAM")
    act = LAM > 0
    assert d["m"] == act.sum()
    tau = max(1.0 - mu, 0.99)
    blk = act & (DS < 0)
    r = np.full(S.shape, np.inf)
    r[blk] = -tau * S[blk] / DS[blk]
    blocking = blk & (r < 1.0)
    bins = np.clip(np.floor(-2.0 * np.log2(r[blocking])).astype(int), 0, 39)
    hist = np.bincount(bins, minlength=40)
    np.testing.assert_array_equal(d["hist"], hist)
    cum, jt = 0, 40
    for j in range(39, -1, -1):
        if cum + hist[j] > d["m"] // 8:
            break
        cum += hist[j]; jt = j
    assert d["jt"] == jt
    assert hist[jt:].sum() <= d["m"] // 8           # at most m / 8 rows are clipped
    allbins = np.clip(np.floor(-2.0 * np.log2(np.where(blk, r, 1.0))).astype(int), 0, 39)
    cand = r[blk & (allbins < jt)]
    assert d["a_p"] == min(1.0, cand.min() if cand.size else 1.0)
    dneg = act & (DLAM < 0)
    a_d = min(1.0, (-tau * LAM[dneg] / DLAM[dneg]).min()) if dneg.any() else 1.0
    assert d["a_d"] == pytest.approx(a_d, rel=1e-15, abs=0)
    assert d["dphi_bar"] == pytest.approx((-mu * DS[act] / S[act]).sum(), rel=1e-12, abs=1e-14)
    assert d["alpha"] == d["a_p"] * 2.0 ** -d["nbt"]
    assert d["a_dual"] == min(d["a_d"], d["alpha"])
    al, ad = d["alpha"], d["a_dual"]
    s_new = np.maximum(S + al * DS, 0.01 * S)
    lam = np.clip(LAM + ad * DLAM, mu / (1e10 * s_new), 1e10 * mu / s_new)
    tight = dict(rtol=1e-14, atol=0)
    np.testing.assert_allclose(o.arr("S")[act], s_new[act], **tight)
    np.testing.assert_allclose(o.arr("LAM")[act], lam[act], **tight)
    np.testing.assert_array_equal(o.arr("S")[~act], S[~act])
    STEP = pre["STEP"]
    np.testing.assert_allclose(o.arr("X"), pre["X"] + al * STEP[:3], rtol=1e-14, atol=1e-15)
    np.testing.assert_allclose(o.arr("U")[:, :N - 1], pre["U"][:, :N - 1] + al * STEP[3:5, :N - 1], rtol=1e-14, atol=1e-15)
    np.testing.assert_allclose(o.arr("NU")[:, :N - 1], pre["NU"][:, :N - 1] + al * (STEP[5:8, :N - 1] - pre["NU"][:, :N - 1]),
                               rtol=1e-13, atol=1e-15)
    dt_new = pre["SCAL"][capi.SC_DT] + (al * pre["SCAL"][capi.SC_DDT] if cfg.variable_dt else 0.0)
    assert o.arr("SCAL")[capi.SC_DT] == pytest.approx(dt_new, rel=1e-15)


def _snapshot(o):
    return {nm: o.arr(nm).copy() for nm in ("X", "U", "NU", "S", "LAM", "STEP", "SCAL")}


@pytest.mark.parametrize("name", ["cfg1", "cfg2", "cfg3", "cfg4", "integral_free_dt", "terminal_ball", "dynamic_free_dt",
                                  "line_obstacles", "midpoint"])
def test_step_length_rules(orc, name):
    """Histogram, threshold bin, a_p, a_d, dphi_bar, at most m/8 clipped rows, alpha = a_p 2^-nbt, a_dual = min(a_d, alpha), and
    the update (1 % slack floor, kappa-sigma clamp of the multipliers, nu, x, u, dt) recomputed in numpy."""
    cfg, data, b = lc.case(name)
    for j in (0, 1, 3, 10, "last"):
        o = _oracle_step(orc, cfg, data, b, j)
        pre = _snapshot(o)
        d = o.linesearch()
        _step_rules(o, pre, d, cfg)


# ---- the device code (CPU warp emulator) against the oracle -----------------------------------------------------------

@pytest.mark.parametrize("name", list(lc.CASES))
def test_device_linesearch_matches_oracle(orc, emu, name):
    """Iterates 0, 1, 3, 10, 25 and the last before convergence of one instance; at most one of the six may put a discrete
    decision within 1e-9 of its threshold (then only the continuous outputs are not compared)."""
    cfg, data, b = lc.case(name)
    n_marginal = n_compared = 0
    for j in lc.ITERATES:
        o, converged = par.oracle_iterate(orc, cfg, data, b, j)
        if converged:   # before iterate j
            continue
        e = par.emu_from_oracle(emu, cfg, data, b, o)
        if not par.eval_and_kkt(o, e, cfg):
            continue
        _, marginal, _ = par.run_both(o, e, cfg, f"{name} iterate {j}")
        n_marginal += marginal
        n_compared += 1
    assert n_compared >= 3 and n_marginal <= 1, (n_compared, n_marginal)


# (not midpoint differences: the heading multiplier row of their step is the device's own, and a changed step would leave it
# inconsistent with the oracle's)
EDGE_CASES = ["cfg1", "cfg2", "cfg3", "integral_free_dt"]
# multipliers 1e12 times too large (kappa_sigma) make the Newton step ill-conditioned, and so is the rounding-sized step of
# iterate 60 (flat_merit); the line search gets the oracle's step anyway
ILL_CONDITIONED_STEP = (1e-4, 1.0)
ILL_CONDITIONED_DDT = 1e-6


@pytest.mark.parametrize("edge", list(lc.EDGES))
def test_device_linesearch_edge_states(orc, emu, edge):
    """Edge states made identically on both sides from iterate 3 (saturated histogram, no blocking row, backtracking
    exhausted, flat merit, jam, first tiny step, kappa-sigma clamp, inf1 <= 1e-14, null step, stopped instance)."""
    pre, post = lc.EDGES[edge]
    branches = []
    for name in EDGE_CASES:
        cfg, data, b = lc.case(name)
        j = 3
        if edge == "flat_merit":
            cfg.tol, j = 1e-15, 60
        o, _ = par.oracle_iterate(orc, cfg, data, b, j)
        if pre is not None:
            pre(o)
        e = par.emu_from_oracle(emu, cfg, data, b, o)
        if edge in ("kappa_sigma", "flat_merit"):
            assert par.eval_and_kkt(o, e, cfg, ILL_CONDITIONED_STEP, ILL_CONDITIONED_DDT)
        else:
            assert par.eval_and_kkt(o, e, cfg)
        # (rho sums sigma ds^2: multipliers 1e12 times too large magnify the rounding of ds by as much)
        d, marginal, before = par.run_both(o, e, cfg, f"{name}, {edge}", post, rho_tol=1e-5 if edge == "kappa_sigma" else 1e-10)
        # the flat-merit test compares a rounding-sized merit change with its bound: that decision is marginal by design
        assert not marginal or edge == "flat_merit"
        lc.check_edge(edge, d, before, o.arr("SCAL"))
        branches.append(d["branch"])
    if edge == "flat_merit":
        assert orc.LS_BRANCH_FLAT in branches, branches
    if edge == "backtracking_exhausted":
        assert orc.LS_BRANCH_NONE in branches, branches


def _threshold_scale(orc, cfg, data, b):
    """A step scale f at which the blocking rows of bins j..39 number exactly m // 8 for some bin j with rows in it: the bin
    is clipped, one more row would make it block.  The slack steps are affine in f, ds(f) = ds(0) + f (ds(1) - ds(0)); the
    scale is searched in numpy on that model and then checked on the oracle's diagnostics."""
    ds = {}
    for f in (0.0, 1.0):
        o = _oracle_step(orc, cfg, data, b, 3)
        lc.scale_step(f)(o)
        S, LAM, mu = o.arr("S").copy(), o.arr("LAM").copy(), o.arr("SCAL")[capi.SC_MU]
        o.linesearch()
        ds[f] = o.arr("DS").copy()
    act = LAM > 0
    m, tau = act.sum(), max(1.0 - mu, 0.99)
    for f in np.geomspace(0.3, 300.0, 4000):
        DS = ds[0.0] + f * (ds[1.0] - ds[0.0])
        blk = act & (DS < 0)
        r = -tau * S[blk] / DS[blk]
        t = -2.0 * np.log2(r[r < 1.0])
        if t.size == 0 or np.abs(t - np.round(t)).min() < 1e-6:
            continue
        hist = np.bincount(np.clip(np.floor(t).astype(int), 0, 39), minlength=40)
        tail = np.cumsum(hist[::-1])[::-1]
        if any(tail[j] == m // 8 and hist[j] > 0 for j in range(40)):
            return f
    return None


def test_threshold_bin_with_exactly_m_over_8_clipped_rows(orc, emu):
    """The threshold bin where the rows of bins j..39 are exactly m // 8: bin j is clipped (cum + hist[j] > m // 8 is false),
    one more row would make it block.  An off-by-one in the threshold rule changes a_p here and nowhere else."""
    hit = 0
    for name in ["cfg1", "cfg2", "cfg3", "cfg4", "integral_free_dt", "terminal_ball"]:
        cfg, data, b = lc.case(name)
        f = _threshold_scale(orc, cfg, data, b)
        if f is None:
            continue
        o, _ = par.oracle_iterate(orc, cfg, data, b, 3)
        e = par.emu_from_oracle(emu, cfg, data, b, o)
        assert par.eval_and_kkt(o, e, cfg)
        d, marginal, _ = par.run_both(o, e, cfg, f"{name}, step x {f:.6g}", lc.scale_step(f))
        assert not marginal
        # (the search used the oracle's own regularisation; where the device's differs, the step and the counts do too)
        jt = d["jt"]
        hit += jt < 40 and d["hist"][jt:].sum() == d["m"] // 8 and d["hist"][jt] > 0
    assert hit >= 2, hit
