"""The oracle's Newton step against the dense KKT system: random iterates of the oracle, the condensed KKT system assembled
by finite differences of the analytic gradient, and the check of the gradient and the Riccati step against a dense solve
(tests/test_oracle_functions.py, tests/test_linesearch.py, tests/test_fixed_final_state.py, tests/test_model_phases.py)."""
import numpy as np

from mpc_local_planner_b200 import capi, configs

def random_iterate(orc, cid, b, seed, nu_scale=1.0, cfg=None, data=None):
    """cid 21 / 22 / 23: cfg 2 with the integral-form cost + free dt / the terminal ball / moving obstacles + free dt;
    cid 24 / 25: integral form integrated by the trapezoidal rule, free / fixed dt;
    cid 26 / 27: hybrid minimum-time + quadratic control cost (Q = 0, fixed final state), point / integral form;
    cid 41 / 42 / 43: midpoint differences on cfg 2 (fixed dt), cfg 2 in integral form (free dt, free final state) and
    cfg 3 (car-like minimum time, fixed final state);
    cid 31: cfg 3 (car-like minimum time, polygon footprint) with moving obstacles;
    cid None: the configuration `cfg` on instance b of the batch `data`"""
    if cid is None:
        return _perturbed_iterate(orc, cfg, orc.instance_from_batch(cfg, data, b), seed, nu_scale), cfg
    moving = cid in (23, 31)
    if cid in (24, 25):
        cfg = configs.cfg2_trapezoidal(tol=1e-8, variable_dt=cid == 24)
    elif cid in (26, 27):
        cfg = configs.cfg2_hybrid_min_time(tol=1e-8, integral_form=cid == 27)
    elif cid in (41, 42, 43):
        cfg = {41: configs.cfg2, 42: configs.cfg2_integral_form, 43: configs.cfg3}[cid](tol=1e-8)
        cfg.collocation = capi.COLLOC_MIDPOINT
    else:
        cfg = configs.cfg2_integral_form(tol=1e-8) if cid in (21, 23) else (configs.cfg2_terminal_ball(tol=1e-8) if cid == 22 else configs.config_for(3 if cid == 31 else cid, tol=1e-8))
    cid = 2 if cid in (21, 22, 23, 24, 25, 26, 27, 41, 42) else (3 if cid in (31, 43) else cid)
    data = configs.g1_instance() if cid == 1 else configs.generate(cid, b + 1)
    if moving:
        cfg.enable_dynamic_obstacles = 1
        data = configs.with_moving_obstacles(data)
    inst = orc.instance_from_batch(cfg, data, 0 if cid == 1 else b)
    return _perturbed_iterate(orc, cfg, inst, seed, nu_scale), cfg


def _perturbed_iterate(orc, cfg, inst, seed, nu_scale):
    """cold start, perturbed states and controls, random multipliers of size nu_scale, mu = 0.1"""
    N = inst.N
    inst.init_cold()
    rng = np.random.default_rng(seed)
    inst.arr("X")[:, 1:] += 0.05 * rng.standard_normal((3, N - 1))
    inst.arr("U")[:] = 0.1 * rng.standard_normal((2, N)); inst.arr("U")[:, N - 1] = 0
    inst.associate(); inst.init_duals()
    inst.arr("NU")[:] = nu_scale * rng.standard_normal((3, N)); inst.arr("NU")[:, N - 1] = 0
    act = inst.arr("LAM") > 0
    inst.arr("LAM")[:] = np.where(act, rng.uniform(0.5, 2, act.shape), 0)
    inst.arr("SCAL")[capi.SC_MU] = 0.1
    return inst


def _pack(inst):
    return np.concatenate([inst.arr("X").ravel(), inst.arr("U").ravel(), [inst.arr("SCAL")[capi.SC_DT]]])


def _unpack(inst, z):
    N = inst.N
    inst.arr("X")[:] = z[:3 * N].reshape(3, N); inst.arr("U")[:] = z[3 * N:5 * N].reshape(2, N); inst.arr("SCAL")[capi.SC_DT] = z[5 * N]


def _lagrangian(inst):
    inst.eval()
    S = inst.arr("SCAL"); K = inst.arr("KKT"); N = inst.N
    e = inst.defects()   # (the record holds them too, transformed to the explicit form for midpoint differences)
    return S[capi.SC_OBJ] + (inst.arr("NU")[:, :N - 1] * e).sum() + (inst.arr("LAM") * (inst.arr("G") + inst.arr("S")) * (inst.arr("LAM") > 0)).sum()

def dense_kkt(inst, cfg, h=1e-6):
    """The condensed KKT system of the oracle instance's current iterate, dense, by finite differences of the analytic
    gradient: Hc = W + Jg' Sigma Jg over z = (X, U, dt), the defect Jacobian Jc, the condensed gradient gt, the defects e and
    the indices of the free variables in z.  Leaves the instance evaluated at its iterate."""
    N = inst.N
    z0 = _pack(inst)
    n = len(z0)
    free = []
    for k in range(1, N):
        for i in range(3):
            if k == N - 1 and cfg.xf_fixed[i]:
                continue
            free.append(i * N + k)
    for k in range(N - 1):
        for i in range(2):
            free.append(3 * N + i * N + k)
    if cfg.variable_dt:
        free.append(5 * N)
    free = np.array(free)

    def grads(z):
        _unpack(inst, z); inst.eval()
        G_ = inst.arr("GL")
        g = np.concatenate([G_[:3].ravel(), G_[3:5].ravel(), [inst.ws.contents.gl_dt]])
        return g, inst.defects().T.ravel().copy(), inst.arr("G").copy()
    m = 3 * (N - 1); RS = inst.RS
    W = np.zeros((n, n)); Jc = np.zeros((m, n)); Jg = np.zeros((RS * N, n))
    for i in range(n):
        zp = z0.copy(); zp[i] += h; gp, ep, Gp = grads(zp)
        zm = z0.copy(); zm[i] -= h; gm, em, Gm = grads(zm)
        W[:, i] = (gp - gm) / (2 * h); Jc[:, i] = (ep - em) / (2 * h); Jg[:, i] = ((Gp - Gm) / (2 * h)).ravel()
    _unpack(inst, z0); inst.eval()
    S = inst.arr("S").ravel(); LAM = inst.arr("LAM").ravel(); G = inst.arr("G").ravel()
    act = LAM > 0
    sig = np.where(act, LAM / S, 0.0)
    mu = inst.arr("SCAL")[capi.SC_MU]
    Hc = W + Jg.T @ np.diag(sig) @ Jg
    gl, _, _ = grads(z0)
    nu = inst.arr("NU")[:, :N - 1].T.ravel()
    gJ = gl - Jc.T @ nu - Jg.T @ np.where(act, LAM, 0)
    r = np.where(act, G + S, 0)
    gt = gJ + Jg.T @ (np.where(act, mu / S, 0) + sig * r)
    e = inst.defects().T.ravel()
    return Hc, Jc, gt, e, free


def check_gradient_and_newton_step(orc, cid, nu_scale, cfg=None, data=None, b=0, seed=0):
    """cid: a case of random_iterate, or None for the configuration `cfg` on instance b of the batch `data`.  Returns the
    number of regularisations at which the Riccati step was compared with the dense solve."""
    inst, cfg = random_iterate(orc, cid, b, seed, nu_scale, cfg, data)
    compared = 0
    N = inst.N
    z0 = _pack(inst)
    n = len(z0)
    inst.eval()
    GL = inst.arr("GL").copy(); gl_dt = inst.ws.contents.gl_dt
    h = 1e-6
    g_fd = np.zeros(n)
    for i in range(n):
        zp = z0.copy(); zp[i] += h; _unpack(inst, zp); Lp = _lagrangian(inst)
        zm = z0.copy(); zm[i] -= h; _unpack(inst, zm); Lm = _lagrangian(inst)
        g_fd[i] = (Lp - Lm) / (2 * h)
    _unpack(inst, z0)
    gx = g_fd[:3 * N].reshape(3, N); gu = g_fd[3 * N:5 * N].reshape(2, N)
    assert np.abs(gx[:, 1:] - GL[:3, 1:]).max() < 5e-6
    assert np.abs(gu[:, :N - 1] - GL[3:5, :N - 1]).max() < 5e-6
    if cfg.variable_dt:
        assert abs(g_fd[5 * N] - gl_dt) < 5e-6 * max(1, abs(gl_dt))
    Hc, Jc, gt, e, free = dense_kkt(inst, cfg)
    m = Jc.shape[0]
    nf = len(free)
    for delta in (0.0, 1e-2, 1.0, 100.0):   # (free-dt problems are indefinite away from the solution: large shifts get compared)
        Kmat = np.zeros((nf + m, nf + m))
        Kmat[:nf, :nf] = Hc[np.ix_(free, free)] + delta * np.eye(nf); Kmat[:nf, nf:] = Jc[:, free].T; Kmat[nf:, :nf] = Jc[:, free]
        ev = np.linalg.eigvalsh(Kmat)
        rc = inst.kkt_solve(delta)
        if (ev > 0).sum() != nf or (ev < 0).sum() != m:
            assert rc == 1  # wrong inertia must be detected
            continue
        if rc == 1 and any(cfg.xf_fixed[i] for i in range(3)):
            # the Riccati pivot test is sufficient, not necessary, when terminal components are fixed: it asks for positive
            # curvature before the terminal constraint is imposed (the constraint enters through the multiplier block at the
            # root); a conservative "wrong inertia" only costs a regularised step
            continue
        assert rc == 0
        sol = np.linalg.solve(Kmat, np.concatenate([-gt[free], -e]))
        STEP = inst.arr("STEP"); ddt = inst.arr("SCAL")[capi.SC_DDT]
        dz = np.zeros(n); dz[:3 * N] = STEP[:3].ravel(); dz[3 * N:5 * N] = STEP[3:5].ravel(); dz[5 * N] = ddt
        nup = STEP[5:8, :N - 1].T.ravel()
        assert np.abs(dz[free] - sol[:nf]).max() < 1e-5 * max(1.0, np.abs(sol[:nf]).max())
        assert np.abs(nup - sol[nf:]).max() < 1e-5 * max(1.0, np.abs(sol[nf:]).max())
        compared += 1
    return compared
