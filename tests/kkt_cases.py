"""The KKT phase as a pure operator: synthetic stage records, the dense KKT system they describe, solved in float64 and
refined in extended precision, and the regularisation schedule of the warp solve restated in plain Python
(tests/test_kkt_operator.py, tests/test_gpu_kkt_operator.py).

The records follow include/mpcb200.h ("offsets inside one KKT stage record"); the sweep that reads them is
mpc_riccati_warp.h, run by kkt_warp_kernel, by warp 0 of the solve kernel and by the CPU warp emulator."""
import ctypes as C
import functools

import numpy as np
import scipy.linalg
import scipy.sparse as sp
import scipy.sparse.linalg as spla

from mpc_local_planner_b200 import capi, configs

KW = capi.KKT_WORDS


def hidx(i, j):
    """packed index of entry (i, j), i <= j, of the upper triangle (row-major) of a 5x5 block (mpc_core.h hidx)"""
    return i * 5 - (i * (i - 1)) // 2 + (j - i)


# ---- configurations: every case that changes what the sweep reads ----
def variant_config(name, xf=(0, 0, 0)):
    """name: "fixed" (fixed dt, free final state: the unbordered sweep, EXT = false), "free_dt" (free dt, left-sum integral
    cost: no terminal dt border), "trap" (free dt, trapezoidal integral cost) or "mid" (free dt, midpoint differences): the
    last two read the terminal K_HB.  "xf_fixed" / "xf_fixed_dt": fixed final state components xf with a fixed / a free dt.
    No obstacle rows: the records do not depend on them, and without them the instance fits the largest horizon."""
    if name in ("fixed", "xf_fixed"):
        c = configs.cfg2()
    elif name in ("free_dt", "xf_fixed_dt"):
        c = configs.cfg2_integral_form()
    elif name == "trap":
        c = configs.cfg2_trapezoidal(variable_dt=True)
    elif name == "mid":
        c = configs.cfg2_integral_form()
        c.collocation = capi.COLLOC_MIDPOINT
    else:
        raise ValueError(name)
    c.xf_fixed[:] = list(xf)
    c.k_max_obstacles_per_stage = 0
    return c


def is_ext(cfg):
    """the bordered sweep (RW<true>): a free dt or a fixed final state component (mpc_layout.h kkt_is_ext)"""
    return bool(cfg.variable_dt or any(cfg.xf_fixed))


def terminal_border(cfg):
    """the terminal record's K_HB x part enters the system (rw_terminal, cc == 1)"""
    return bool(cfg.variable_dt) and (
        (cfg.objective == capi.OBJ_QUADRATIC_FORM and cfg.quadratic_integral_form and cfg.cost_integration == capi.COST_TRAPEZOIDAL)
        or cfg.collocation == capi.COLLOC_MIDPOINT)


def accepted_horizon(lib, cfg, n):
    """mpcb200_create accepts the configuration at horizon n (the configuration is validated before a device is looked for:
    E_NODEVICE on a machine without one means accepted)"""
    c = cfg.copy()
    c.n = n
    h = C.c_void_p()
    rc = lib.mpcb200_create(C.byref(c), 1, 0, C.byref(h))
    if rc == 0:
        lib.mpcb200_destroy(h)
    assert rc != capi.E_INVALID, lib.mpcb200_last_error(None).decode()
    return rc != capi.E_UNSUPPORTED


def largest_horizon(lib, cfg):
    """the largest n in [3, 512] that mpcb200_create accepts for cfg (bisection on E_UNSUPPORTED)"""
    lo, hi = 3, 513
    assert accepted_horizon(lib, cfg, lo)
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if accepted_horizon(lib, cfg, mid) else (lo, mid)
    return lo


# ---- synthetic records ----
def ignored_words(cfg, N):
    """Boolean mask [KW][N] of the record words the sweep must not read:
      stage 0: its x parts (dx_0 = 0 is not a variable): the x rows of K_H, K_G[0:3], K_HB[0:3], K_A; and K_C (du_{-1} is
               not a variable);
      stage N-1: everything but the x Hessian block and the x gradient: the u part of K_H and K_G, K_C, K_A, K_B, K_E, K_D,
               and K_HB (its x part is read by the trapezoidal and the midpoint configurations with a free dt);
      a fixed dt: K_HB and K_D of every stage (and HTT, GT of SCAL, see scal_words)."""
    m = np.zeros((KW, N), dtype=bool)
    for i in range(3):
        for j in range(i, 5):
            m[capi.K_H + hidx(i, j), 0] = True
    m[capi.K_G:capi.K_G + 3, 0] = True
    m[capi.K_HB:capi.K_HB + 3, 0] = True
    m[capi.K_A:capi.K_A + 3, 0] = True
    m[capi.K_C:capi.K_C + 2, 0] = True
    last = np.ones(KW, dtype=bool)
    for i in range(3):
        for j in range(i, 3):
            last[capi.K_H + hidx(i, j)] = False
    last[capi.K_G:capi.K_G + 3] = False
    if terminal_border(cfg):
        last[capi.K_HB:capi.K_HB + 3] = False
    m[:, N - 1] |= last
    if not cfg.variable_dt:
        m[capi.K_HB:capi.K_HB + 5, :] = True
        m[capi.K_D:capi.K_D + 3, :] = True
    return m


def make_records(cfg, N, seed, lam_min=0.1, lam_max=10.0, neg_u=None, neg_htt=None, garbage=True):
    """Synthetic stage records [KW][N] and (HTT, GT) for cfg at horizon N from `seed`.
      K_H   SPD 5x5 blocks, eigenvalues log-uniform in [lam_min, lam_max] (random eigenvectors);
      K_C   |c| <= lam_min / 4: the control-rate couplings (each control couples with two neighbours) keep the Hessian of
            (x, u) positive definite with its smallest eigenvalue >= lam_min / 2;
      K_G   N(0, 1); K_A (a0, a1) U(-0.3, 0.3), a2 U(-2e-3, 2e-3) (A_k = I + a e_theta': products over 500 stages stay
            moderate); K_B U(-0.3, 0.3); K_E N(0, 0.1); K_D N(0, 0.3); K_HB N(0, 0.1);
      HTT   1 + 2 sum_k |K_HB_k|^2 / lam_min (the dt row keeps the Hessian positive definite), GT N(0, 1).
    The words of ignored_words() get finite garbage U(-5, 5) unless garbage is False (then 0).
    neg_u = (k, s, "dir" | "def"): the u block of stage k gets curvature -s along a random direction ("dir") or becomes
    negative definite with its eigenvalues <= -s ("def"); neg_htt = s: HTT = -s."""
    rng = np.random.default_rng(seed)
    R = np.zeros((KW, N))
    for k in range(N):
        Q, _ = np.linalg.qr(rng.standard_normal((5, 5)))
        H = (Q * np.exp(rng.uniform(np.log(lam_min), np.log(lam_max), 5))) @ Q.T
        if neg_u is not None and neg_u[0] == k:
            _, s, mode = neg_u
            Huu = H[3:5, 3:5]
            if mode == "dir":
                v = rng.standard_normal(2); v /= np.linalg.norm(v)
                H[3:5, 3:5] = Huu - (v @ Huu @ v + s) * np.outer(v, v)
            else:
                H[3:5, 3:5] = Huu - (np.linalg.eigvalsh(Huu)[-1] + s) * np.eye(2)
        for i in range(5):
            for j in range(i, 5):
                R[capi.K_H + hidx(i, j), k] = H[i, j]
        R[capi.K_C:capi.K_C + 2, k] = rng.uniform(-0.25, 0.25, 2) * lam_min
        R[capi.K_G:capi.K_G + 5, k] = rng.standard_normal(5)
        R[capi.K_A:capi.K_A + 2, k] = rng.uniform(-0.3, 0.3, 2)
        R[capi.K_A + 2, k] = rng.uniform(-2e-3, 2e-3)
        R[capi.K_B:capi.K_B + 6, k] = rng.uniform(-0.3, 0.3, 6)
        R[capi.K_E:capi.K_E + 3, k] = 0.1 * rng.standard_normal(3)
        R[capi.K_D:capi.K_D + 3, k] = 0.3 * rng.standard_normal(3)
        R[capi.K_HB:capi.K_HB + 5, k] = 0.1 * rng.standard_normal(5)
    htt = 1.0 + 2.0 * (R[capi.K_HB:capi.K_HB + 5] ** 2).sum() / lam_min
    if neg_htt is not None:
        htt = -neg_htt
    gt = rng.standard_normal()
    ign = ignored_words(cfg, N)
    R[ign] = rng.uniform(-5.0, 5.0, ign.sum()) if garbage else 0.0
    if not cfg.variable_dt:   # HTT and GT are read with a free dt only
        htt, gt = (rng.uniform(-5.0, 5.0), rng.uniform(-5.0, 5.0)) if garbage else (0.0, 0.0)
    return R, htt, gt


def zero_ignored(cfg, R, htt, gt):
    """the records with the ignored words zeroed"""
    R = R.copy()
    R[ignored_words(cfg, R.shape[1])] = 0.0
    if not cfg.variable_dt:
        htt = gt = 0.0
    return R, htt, gt


def scal_words(htt, gt, dlast, nreg=0.0):
    """SCAL of a live instance whose KKT phase is pending: HTT, GT, DELTA_LAST, a previous NREG, VALID = 1, STATUS = -1;
    the words the KKT phase may write hold sentinels"""
    s = np.zeros(capi.SCAL_WORDS)
    s[capi.SC_HTT], s[capi.SC_GT], s[capi.SC_DELTA_LAST], s[capi.SC_NREG] = htt, gt, dlast, nreg
    s[capi.SC_VALID], s[capi.SC_STATUS] = 1.0, -1.0
    s[capi.SC_DELTA], s[capi.SC_DDT], s[capi.SC_DEFER] = 7.25, -3.5, 0.0
    return s


def step_sentinel(N):
    """a STEP pattern the KKT phase overwrites only when it solves"""
    return np.arange(8 * N, dtype=np.float64).reshape(8, N) * 0.125 - 1000.0


# ---- the dense reference ----
class Dense:
    """The KKT system the records describe, assembled directly from the record words (no oracle, no finite differences):
        [[H + delta I, Jc'], [Jc, 0]] (dz, nu+) = (-g, -e).
    Unknowns z: dx_1 .. dx_{N-1} without the fixed components of dx_{N-1}, du_0 .. du_{N-2}, and d(dt) when dt is free;
    nu+_k (k = 0 .. N-2) are the multipliers of the defect rows (the conventions of tests/dense_kkt.py).  Terms:
      H[w_k, w_k]      K_H (upper triangle, hidx) over w_k = (dx_k, du_k), k = 0 .. N-2; stage 0 without its x rows
      H[x_N-1, x_N-1]  K_H x block of stage N-1 (fixed components dropped)
      H[du_k-1, du_k]  K_C[i] of stage k (k = 1 .. N-2), on the same control component i
      H[w_k, dt]       K_HB of stage k (dt free; k = 0 .. N-2, stage 0 without x), K_HB[0:3] of stage N-1 when
                       terminal_border(cfg)
      H[dt, dt]        HTT (SCAL);  delta is added on every diagonal entry of H, dt included
      g                K_G of w_k (as H), K_G[0:3] of stage N-1, GT (SCAL) for dt
      Jc row (k, i)    A_k dx_k + B_k du_k + d_k d(dt) - dx_{k+1} = -e_k: A_k = I + K_A e_theta' (k >= 1), B_k = K_B
                       (row-major 3x2), d_k = K_D (dt free), e_k = K_E."""

    def __init__(self, cfg, R, htt, gt):
        N = R.shape[1]
        self.cfg, self.N, self.R, self.htt, self.gt = cfg, N, R, htt, gt
        fixed = [bool(f) for f in cfg.xf_fixed]
        dt_free = bool(cfg.variable_dt)
        xcol = -np.ones((3, N), dtype=np.int64); ucol = -np.ones((2, N), dtype=np.int64)
        n = 0
        for k in range(1, N):
            for i in range(3):
                if k == N - 1 and fixed[i]:
                    continue
                xcol[i, k] = n; n += 1
        for k in range(N - 1):
            for i in range(2):
                ucol[i, k] = n; n += 1
        tcol = -1
        if dt_free:
            tcol = n; n += 1
        self.xcol, self.ucol, self.tcol, self.n, self.m = xcol, ucol, tcol, n, 3 * (N - 1)
        rows, cols, vals = [], [], []
        rhs = np.zeros(n + self.m)

        def sym(a, b, v):
            rows.append(a); cols.append(b); vals.append(v)
            if a != b:
                rows.append(b); cols.append(a); vals.append(v)

        for k in range(N):
            w = [xcol[0, k], xcol[1, k], xcol[2, k], ucol[0, k], ucol[1, k]]
            for a in range(5):
                if w[a] < 0:
                    continue
                for b in range(a, 5):
                    if w[b] >= 0:
                        sym(w[a], w[b], R[capi.K_H + hidx(a, b), k])
                rhs[w[a]] = -R[capi.K_G + a, k]
                if dt_free and (k < N - 1 or (a < 3 and terminal_border(cfg))):
                    sym(w[a], tcol, R[capi.K_HB + a, k])
            if 1 <= k <= N - 2:
                for i in range(2):
                    sym(ucol[i, k - 1], ucol[i, k], R[capi.K_C + i, k])
        if dt_free:
            sym(tcol, tcol, htt)
            rhs[tcol] = -gt
        for k in range(N - 1):
            for i in range(3):
                r = n + 3 * k + i
                if k >= 1:
                    sym(r, xcol[i, k], 1.0)
                    sym(r, xcol[2, k], R[capi.K_A + i, k])
                for j in range(2):
                    sym(r, ucol[j, k], R[capi.K_B + 2 * i + j, k])
                if dt_free:
                    sym(r, tcol, R[capi.K_D + i, k])
                if xcol[i, k + 1] >= 0:
                    sym(r, xcol[i, k + 1], -1.0)
                rhs[r] = -R[capi.K_E + i, k]
        self.rows = np.array(rows, dtype=np.int64); self.cols = np.array(cols, dtype=np.int64)
        self.vals = np.array(vals, dtype=np.float64)
        self.diag = np.arange(n, dtype=np.int64)   # delta on the unknowns z
        self.rhs = rhs

    def _coo(self, delta):
        rows = np.concatenate([self.rows, self.diag]); cols = np.concatenate([self.cols, self.diag])
        vals = np.concatenate([self.vals, np.full(len(self.diag), float(delta))])
        return rows, cols, vals

    def matrix(self, delta):
        rows, cols, vals = self._coo(delta)
        sz = self.n + self.m
        return sp.csc_matrix((vals, (rows, cols)), shape=(sz, sz))

    def residual(self, delta, z):
        """r - K z in long double (z: any float array of the system's size)"""
        rows, cols, vals = self._coo(delta)
        zl = np.asarray(z, dtype=np.longdouble)
        out = self.rhs.astype(np.longdouble)
        np.subtract.at(out, rows, vals.astype(np.longdouble) * zl[cols])
        return out

    def norm(self, delta):
        """infinity norm of K"""
        rows, _, vals = self._coo(delta)
        return np.bincount(rows, weights=np.abs(vals), minlength=self.n + self.m).max()

    def solve(self, delta):
        """float64 sparse LU, refined twice with residuals in long double; the solution in long double"""
        lu = spla.splu(self.matrix(delta))
        z = lu.solve(self.rhs).astype(np.longdouble)
        for _ in range(2):
            z = z + lu.solve(self.residual(delta, z).astype(np.float64))
        return z

    def reduced_eigenvalues(self):
        """eigenvalues of the reduced Hessian Z' H Z (Z: an orthonormal basis of the null space of Jc, dense: small horizons
        only).  Jc has full row rank, so the inertia of K at delta is that of Z' H Z + delta I plus (m, m, 0) (Gould): it is
        right iff delta > -min(eigenvalues)."""
        if getattr(self, "_red", None) is None:
            A = self.matrix(0.0).toarray()
            H, J = A[:self.n, :self.n], A[self.n:, :self.n]
            Z = scipy.linalg.null_space(J)
            assert Z.shape[1] == self.n - self.m   # full row rank
            self._red = np.linalg.eigvalsh(Z.T @ H @ Z)
        return self._red

    def right_inertia(self, delta):
        return bool(self.reduced_eigenvalues()[0] + delta > 0.0)

    def threshold_delta(self):
        """the regularisation above which the inertia is right (0 when it is right without)"""
        return max(0.0, -float(self.reduced_eigenvalues()[0]))

    # STEP layout [8][N]: dx (3), du (2), nu+ (3); d(dt)
    def pack(self, STEP, ddt):
        """the unknowns of the system from a STEP field and d(dt)"""
        N = self.N
        z = np.zeros(self.n + self.m)
        for i in range(3):
            sel = self.xcol[i] >= 0
            z[self.xcol[i, sel]] = STEP[i, sel]
        for i in range(2):
            z[self.ucol[i, :N - 1]] = STEP[3 + i, :N - 1]
        if self.tcol >= 0:
            z[self.tcol] = ddt
        z[self.n:] = STEP[5:8, :N - 1].T.ravel()
        return z

    def unpack(self, z):
        """(STEP [8][N], d(dt)) of a solution (zeros where the system has no unknown)"""
        N = self.N
        z = np.asarray(z, dtype=np.float64)
        STEP = np.zeros((8, N))
        for i in range(3):
            sel = self.xcol[i] >= 0
            STEP[i, sel] = z[self.xcol[i, sel]]
        for i in range(2):
            STEP[3 + i, :N - 1] = z[self.ucol[i, :N - 1]]
        STEP[5:8, :N - 1] = z[self.n:].reshape(N - 1, 3).T
        return STEP, (float(z[self.tcol]) if self.tcol >= 0 else 0.0)

    def errors(self, delta, STEP, ddt, zref):
        """(normwise backward error |K z - r| / (|K| |z| + |r|), forward error |z - zref| / |zref|) of a computed step,
        infinity norms, in long double"""
        z = self.pack(STEP, ddt)
        res = np.abs(self.residual(delta, z)).max()
        bwd = res / (np.longdouble(self.norm(delta)) * np.abs(z).max() + np.abs(self.rhs).max())
        fwd = np.abs(z.astype(np.longdouble) - zref).max() / np.abs(zref).max()
        return float(bwd), float(fwd)


# ---- the regularisation schedule (mpc_riccati_warp.h kkt_first_delta, kkt_escalate, kkt_warp_solve, kkt_store_outcome;
#      the constants of mpc_core.h) ----
MAX_INERTIA_TRIES = 2
MAX_DELTA = 1e8
DELTA_FLOOR = 1e-5


def first_delta(dlast):
    """the regularisation of the first attempt of an iteration: a third of the last one, none below the floor"""
    return dlast / 3.0 if dlast > 0.0 and dlast / 3.0 >= DELTA_FLOOR else 0.0


def escalate(delta, dlast):
    """the regularisation of the next attempt after a wrong inertia at delta"""
    if delta == 0.0:
        return 1e-4 if dlast == 0.0 else max(dlast / 3.0, 1e-20)
    return delta * (100.0 if dlast == 0.0 else 8.0)


def candidates(dlast):
    """the regularisations one iteration may try, in order"""
    out, delta = [], first_delta(dlast)
    while len(out) < MAX_INERTIA_TRIES and delta <= MAX_DELTA:
        out.append(delta)
        delta = escalate(delta, dlast)
    return out


def schedule(solves, dlast):
    """the attempts of one iteration; solves(delta) -> whether the attempt at delta solves.  Returns (ok, delta, nreg): delta
    is the regularisation of the solve, or the next one after the last failure"""
    delta, nreg, ok = first_delta(dlast), 0, False
    for _ in range(MAX_INERTIA_TRIES):
        if ok or delta > MAX_DELTA:
            break
        ok = solves(delta)
        if not ok:
            nreg += 1
            delta = escalate(delta, dlast)
    return ok, delta, nreg


def store_outcome(scal, ok, ddt, delta, nreg):
    """the bookkeeping words of SCAL after the KKT phase: a step (DEFER 0, DDT, DELTA, DELTA_LAST = delta), a null step
    that resumes the escalation in the next iteration (DEFER 1, DELTA_LAST = 3 delta), or NUMERICAL_ERROR past MAX_DELTA;
    NREG counts the failed attempts"""
    s = np.array(scal, dtype=np.float64, copy=True)
    s[capi.SC_NREG] += nreg
    if not ok and delta <= MAX_DELTA:
        s[capi.SC_DELTA_LAST] = 3.0 * delta
        s[capi.SC_DEFER] = 1.0
    elif not ok:
        s[capi.SC_STATUS] = float(capi.STATUS_NUMERICAL_ERROR)
    else:
        s[capi.SC_DEFER] = 0.0
        s[capi.SC_DDT] = ddt
        s[capi.SC_DELTA] = delta
        s[capi.SC_DELTA_LAST] = delta
    return s


# ---- horizons ----
def full_horizons(n_max):
    """every N from 3 to 70, the chunk-count transitions 95-99, 127-131, 159-163, 190-200 (CH = ceil((N-1)/32)), and the
    largest horizon that fits"""
    hs = list(range(3, 71)) + list(range(95, 100)) + list(range(127, 132)) + list(range(159, 164)) + list(range(190, 201))
    return [n for n in hs if n <= n_max] + ([n_max] if n_max > 200 else [])


def reduced_horizons(n_max):
    """the horizons of the cross product of the variants: one and two stages per lane, a partial and a full last chunk,
    and the largest horizon"""
    return [n for n in (3, 4, 5, 32, 33, 34, 35, 65, 97, 129, 193) if n <= n_max] + [n_max]


def run_emulator(emu, cfg, R, htt, gt, dlast=0.0, nreg=0.0):
    """the KKT phase of the CPU warp emulator on the records: (STEP, SCAL) after it, from step_sentinel() and
    scal_words()"""
    N = R.shape[1]
    c = cfg.copy()
    c.n = N
    e = emu.EmuInstance(c, np.zeros(3), np.zeros(3))
    e.set_field(capi.F_KKT, R)
    e.set_field(capi.F_SCAL, scal_words(htt, gt, dlast, nreg))
    e.set_field(capi.F_STEP, step_sentinel(N))
    e.kkt()
    return e.field(capi.F_STEP).copy(), e.field(capi.F_SCAL).copy()


def run_oracle(orc, cfg, R, htt, gt, delta):
    """the oracle's serial Riccati sweep (orc_kkt_solve) on the records at delta: (solved, STEP, d(dt))"""
    N = R.shape[1]
    c = cfg.copy()
    c.n = N
    o = orc.Instance(c, np.zeros(3), np.zeros(3))
    o.arr("KKT")[:] = R
    o.arr("SCAL")[capi.SC_HTT], o.arr("SCAL")[capi.SC_GT] = htt, gt
    ok = o.kkt_solve(delta) == 0
    return ok, o.arr("STEP").copy(), float(o.arr("SCAL")[capi.SC_DDT])


def chunk(N):
    """stages per lane of the forward substitution"""
    return (N - 1 + 31) // 32


# ---- the cases the CPU and the GPU tests share ----
VARIANTS = ("fixed", "free_dt", "trap", "mid", "xf_fixed", "xf_fixed_dt")
XF_PATTERNS = [(i & 1, (i >> 1) & 1, (i >> 2) & 1) for i in range(1, 8)]
# every configuration that changes what the sweep reads besides the template: (name, fixed final state components)
CROSS = [("trap", (0, 0, 0)), ("mid", (0, 0, 0))] + [("xf_fixed", p) for p in XF_PATTERNS] + [("xf_fixed_dt", p) for p in XF_PATTERNS]


@functools.lru_cache(maxsize=None)
def n_max(name, xf=(0, 0, 0)):
    """the largest horizon of a variant"""
    return largest_horizon(capi.load_library(), variant_config(name, xf))


def horizons(name, xf=(0, 0, 0)):
    """every horizon shape for the two templates, the reduced list for the other variants"""
    return full_horizons(n_max(name)) if name in ("fixed", "free_dt") else reduced_horizons(n_max(name, xf))


def seed_of(name, xf, N, extra=0):
    """the seed of a case"""
    return 1000003 * N + 7919 * (xf[0] + 2 * xf[1] + 4 * xf[2]) + 104729 * VARIANTS.index(name) + extra


def assert_exact_properties(cfg, STEP, SC, what):
    """no step on a fixed final state component, no d(dt) with a fixed dt, dx_0 = 0, no du and nu+ at N-1"""
    for i in range(3):
        if cfg.xf_fixed[i]:
            assert STEP[i, -1] == 0.0, f"{what}: step of fixed component {i}"
    if not cfg.variable_dt:
        assert SC[capi.SC_DDT] == 0.0, f"{what}: d(dt) {SC[capi.SC_DDT]!r} with a fixed dt"
    assert (STEP[0:3, 0] == 0.0).all(), f"{what}: dx_0"
    assert (STEP[3:8, -1] == 0.0).all(), f"{what}: du / nu+ at N-1"


def assert_outcome(SC, exp, what, ddt_tol=1e-12):
    """the words of SCAL exactly, d(dt) relative to max(1, |d(dt)|)"""
    for i in range(capi.SCAL_WORDS):
        if i == capi.SC_DDT:
            assert abs(SC[i] - exp[i]) <= ddt_tol * max(1.0, abs(exp[i])), f"{what}: d(dt) {SC[i]!r} vs {exp[i]!r}"
        else:
            assert SC[i] == exp[i], f"{what}: SCAL[{i}] {SC[i]!r} vs {exp[i]!r}"


def assert_accuracy(d, delta, STEP, ddt, z, tol, what):
    """backward and forward error of a step within tol = (backward, forward); returns them"""
    bwd, fwd = d.errors(delta, STEP, ddt, z)
    assert bwd <= tol[0] and fwd <= tol[1], f"{what}: backward error {bwd:.2e}, forward error {fwd:.2e}"
    return bwd, fwd


# inertia: (variant, xf, N, neg_u, neg_htt)
def inertia_cases():
    """negative curvature along one u direction ("dir") or a negative definite u block ("def") at stage 0, at N-2 and at a
    chunk boundary k = CH j of the forward substitution; a negative HTT (free dt)"""
    out = []
    for name, xf in (("fixed", (0, 0, 0)), ("free_dt", (0, 0, 0)), ("xf_fixed", (1, 1, 0)), ("xf_fixed_dt", (1, 1, 1))):
        for N in (20, 67):
            ch = chunk(N)
            for k in (0, N - 2, ch * (N // (2 * ch))):
                for mode in ("dir", "def"):
                    for s in (0.05, 3.0, 300.0):
                        out.append((name, xf, N, (k, s, mode), None))
        if name in ("free_dt", "xf_fixed_dt"):
            for s in (1e-3, 1.0, 1e3):
                out.append((name, xf, 20, None, s))
    return out


INERTIA_DLASTS = (0.0, 1.0)


def check_inertia(run, tol, name, xf, N, neg_u, neg_htt, dlast):
    """The attempts of one KKT phase against the dense inertia at each regularisation tried: a solve at a wrong inertia is
    a bug (the pivot test is sufficient).  With a free final state the test is also necessary, so every word of SCAL must be
    the schedule's (and the step accurate to tol, or STEP untouched); with fixed components a conservative failure is
    allowed.  run(cfg, R, htt, gt, dlast, nreg) -> (STEP, SCAL).  Returns whether the failure was conservative."""
    cfg = variant_config(name, xf)
    cfg.n = N
    R, htt, gt = make_records(cfg, N, seed_of(name, xf, N, 17), neg_u=neg_u, neg_htt=neg_htt)
    d = Dense(cfg, R, htt, gt)
    right = {delta: d.right_inertia(delta) for delta in candidates(dlast)}
    STEP, SC = run(cfg, R, htt, gt, dlast, 0.0)
    what = f"{name} xf={xf} N={N} neg_u={neg_u} neg_htt={neg_htt} dlast={dlast}"
    ok = SC[capi.SC_DEFER] == 0.0 and SC[capi.SC_STATUS] < 0.0
    tried = candidates(dlast)[:int(SC[capi.SC_NREG]) + ok]
    if ok:
        assert right[tried[-1]], f"{what}: solved at delta = {tried[-1]} with the wrong inertia"
    conservative = any(right[delta] for delta in tried[:len(tried) - ok])
    if conservative and any(cfg.xf_fixed):
        return True
    exp_ok, exp_delta, exp_nreg = schedule(lambda delta: right[delta], dlast)
    z = d.solve(exp_delta) if exp_ok else None
    exp = store_outcome(scal_words(htt, gt, dlast), exp_ok, d.unpack(z)[1] if exp_ok else 0.0, exp_delta, exp_nreg)
    assert_outcome(SC, exp, what)
    if exp_ok:
        assert_accuracy(d, exp_delta, STEP, SC[capi.SC_DDT], z, tol, what)
    else:
        np.testing.assert_array_equal(STEP, step_sentinel(N), err_msg=f"{what}: STEP written without a solve")
    return False


# schedule: (variant, s, where, dlast)
SCHEDULE_DLASTS = (0.0, 5e-6, 3e-5, 1.0, 1e7, 5e8)
SCHEDULE_S = tuple(10.0 ** e for e in np.arange(-7.0, 9.5, 0.5))
SCHEDULE_N = 12


@functools.lru_cache(maxsize=None)
def schedule_case(name, s, where):
    """records whose dense inertia turns right at a delta that grows with the indefiniteness s of one u direction at stage 5
    (where = "u") or of HTT ("htt"), and that delta"""
    cfg = variant_config(name)
    cfg.n = SCHEDULE_N
    neg_u, neg_htt = ((5, s, "dir"), None) if where == "u" else (None, s)
    R, htt, gt = make_records(cfg, SCHEDULE_N, seed_of(name, (0, 0, 0), SCHEDULE_N, 31), neg_u=neg_u, neg_htt=neg_htt)
    d = Dense(cfg, R, htt, gt)
    return cfg, R, htt, gt, d, d.threshold_delta()


def schedule_cases():
    """the cases whose threshold delta lies at least a factor 2 from every candidate of their last regularisation, so that
    no decision of the schedule is marginal"""
    out = []
    for name, where in (("fixed", "u"), ("free_dt", "u"), ("free_dt", "htt")):
        for s in SCHEDULE_S:
            thr = schedule_case(name, s, where)[-1]
            for dlast in SCHEDULE_DLASTS:
                if thr > 1e-9 and all(c == 0.0 or not 0.5 < thr / c < 2.0 for c in candidates(dlast)):
                    out.append((name, s, where, dlast))
    return out


def check_schedule(run, name, s, where, dlast):
    """SCAL after the KKT phase against the schedule driven by the dense inertia; STEP untouched without a solve.  Returns
    the outcome: "solved after <failed attempts>", "defer" or "error"."""
    cfg, R, htt, gt, d, thr = schedule_case(name, s, where)
    exp_ok, exp_delta, exp_nreg = schedule(lambda delta: delta > thr, dlast)
    ddt = d.unpack(d.solve(exp_delta))[1] if exp_ok else 0.0
    exp = store_outcome(scal_words(htt, gt, dlast, 1.0), exp_ok, ddt, exp_delta, exp_nreg)
    STEP, SC = run(cfg, R, htt, gt, dlast, 1.0)
    what = f"{name} s={s:g} ({where}) threshold {thr:.3g} dlast={dlast:g}"
    assert_outcome(SC, exp, what)
    if not exp_ok:
        np.testing.assert_array_equal(STEP, step_sentinel(cfg.n), err_msg=f"{what}: STEP written without a solve")
        return "error" if SC[capi.SC_STATUS] >= 0 else "defer"
    return f"solved after {exp_nreg}"


SCHEDULE_OUTCOMES = {"solved after 0", "solved after 1", "defer", "error"}
