// emu.cpp -- CPU WARP EMULATOR of the device code (TEST INFRASTRUCTURE, not product code).
//
// Compiles the SAME host/device headers that the CUDA kernels are made of (mpc_core.h, mpc_stage.h, mpc_riccati_warp.h,
// mpc_layout.h) with g++ and replays the kernels' warp-level orchestration (lane loops, reductions, passes) serially
// for ONE instance.  Purpose: `-m "not gpu"` tests can check the device algorithm (stage bodies, Riccati task tables,
// line search) against the oracle on a box without a GPU.  It is never loaded by the product package; the product
// path exists only as CUDA kernels (mpcb200.cu) and fails loudly without a GPU.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "../../mpc_local_planner_b200/csrc/mpc_core.h"
#include "../../mpc_local_planner_b200/csrc/mpc_riccati_warp.h"
#include "../../mpc_local_planner_b200/csrc/mpc_stage.h"
#include "../../mpc_local_planner_b200/csrc/mpc_layout.h"

// serial replay of a warp: every "phase" between two warp barriers runs lane after lane on 32 lane states
template <bool EXT>
struct SerialWarp
{
    RwLane<EXT> ls[32];
    template <class F> void each(const F& f) { for (int l = 0; l < 32; ++l) f(l, ls[l]); }
    void sync() {}
    bool all(bool p) const { return p; }   // the driver only votes on values that are the same in every lane
    void shift_up(int d) { for (int l = 31; l >= d; --l) ls[l].in = ls[l - d].out; }
};

extern "C" {

// words of the emulator buffer: one instance block
long long emu_stride(const Cfg* c)
{
    WsLayout L;
    make_layout(c, MAX_OBST, MAX_VP, L);
    return (long long)L.stride;
}

int emu_field_offset(const Cfg* c, int field, int* cnt)
{
    WsLayout L;
    make_layout(c, MAX_OBST, MAX_VP, L);
    switch (field)
    {
        case MPCB200_F_X: *cnt = 3; return L.oX;
        case MPCB200_F_U: *cnt = 2; return L.oU;
        case MPCB200_F_NU: *cnt = 3; return L.oNU;
        case MPCB200_F_S: *cnt = L.RS; return L.oS;
        case MPCB200_F_LAM: *cnt = L.RS; return L.oLAM;
        case MPCB200_F_KKT: *cnt = KW; return L.oKKT;  /* records [k][RSTR]: element (k, f) at k * RSTR + f */
        case MPCB200_F_STEP: *cnt = 8; return L.oSTEP;
        case MPCB200_F_SCAL: *cnt = MPCB200_SCAL_WORDS; return L.oSCAL;
        case MPCB200_F_OBSIDX: *cnt = L.K > 0 ? L.K : 1; return L.oOBS;
    }
    return -1;
}

// the via-point stages of the last association (not a workspace field of the C ABI); returns their number
int emu_vp_stage(const Cfg* c, const double* W, int* out)
{
    WsLayout L;
    make_layout(c, MAX_OBST, MAX_VP, L);
    for (int j = 0; j < L.V; ++j) out[j] = (int)W[L.oVPST + j];
    return L.V;
}

void emu_scatter(const Cfg* c, double* W, const double* x0, const double* xf, const double* u_prev, int nobst, const int* types,
                 const double* params, int nvp, const double* vp, const double* x_init, int reinit)
{
    WsLayout L;
    make_layout(c, MAX_OBST, MAX_VP, L);
    const int N = L.N;
    (void)N;
    for (int i = 0; i < 3; ++i) { AIN(IN_X0 + i) = x0[i]; AIN(IN_XF + i) = xf[i]; }
    for (int i = 0; i < 2; ++i) AIN(IN_UPREV + i) = u_prev ? u_prev[i] : 0.0;
    AIN(IN_NOBST) = nobst; AIN(IN_NVP) = nvp; AIN(IN_HASXINIT) = x_init ? 1.0 : 0.0; AIN(IN_REINIT) = reinit ? 1.0 : 0.0;
    for (int i = 0; i < nobst * MPCB200_OBST_STRIDE; ++i) W[L.oOBST + i] = params[i];
    for (int i = 0; i < nobst; ++i) W[L.oOTYPE + i] = (double)types[i];
    for (int i = 0; i < nvp * 3; ++i) W[L.oVP + i] = vp[i];
    if (x_init)
        for (int i = 0; i < 3 * L.N; ++i) W[L.oXINIT + i] = x_init[i];
}

void emu_reset(const Cfg* c, double* W)
{
    WsLayout L;
    make_layout(c, MAX_OBST, MAX_VP, L);
    ASC(MPCB200_SC_COLD) = 1.0;
    ASC(MPCB200_SC_STATUS) = -1.0;
}

void emu_init(const Cfg* cp, double* W, int force_cold)
{
    const Cfg& c = *cp;
    WsLayout L;
    make_layout(cp, MAX_OBST, MAX_VP, L);
    const int N = L.N;
    const bool cold = force_cold || ASC(MPCB200_SC_COLD) != 0.0 || AIN(IN_REINIT) != 0.0;
    if (cold)
    {
        for (int k = 0; k < N; ++k) init_cold_stage(c, L, W, k, W + L.oXINIT);
        bump_select_serial(c, L, W);
        ASC(MPCB200_SC_DT) = c.dt_ref;
        ASC(MPCB200_SC_COLD) = 2.0;
    }
    else
    {
        if (c.warm_start && !c.variable_dt) warm_shift_serial(c, L, W);
        else
        {
            for (int i = 0; i < 3; ++i) AX(i, 0) = AIN(IN_X0 + i);
            for (int i = 0; i < 3; ++i)
                if (c.xf_fixed[i]) AX(i, N - 1) = AIN(IN_XF + i);
        }
        ASC(MPCB200_SC_COLD) = 0.0;
    }
}

void emu_associate(const Cfg* cp, double* W, double uprev_dt, int first_outer)
{
    const Cfg& c = *cp;
    WsLayout L;
    make_layout(cp, MAX_OBST, MAX_VP, L);
    const int N = L.N;
    const bool cold_pending = first_outer && ASC(MPCB200_SC_COLD) == 2.0;
    const bool repair = cold_pending && !c.reference_initial_guess;
    for (int k = 0; k < N; ++k) associate_stage(c, L, W, k);
    if (has_viapoints(c))
    {
        const int nvp = (int)AIN(IN_NVP);
        int start_idx = 0;
        for (int j = 0; j < nvp && j < L.V; ++j)
        {
            const double vx = W[L.oVP + 3 * j], vy = W[L.oVP + 3 * j + 1];
            double best = 1e300;
            int bidx = -1;
            for (int i = start_idx; i < N - 1; ++i)
            {
                const double dx = AX(0, i) - vx, dy = AX(1, i) - vy, d = sqrt(dx * dx + dy * dy);
                if (d < best) { best = d; bidx = i; }
            }
            {
                const double dx = AX(0, N - 1) - vx, dy = AX(1, N - 1) - vy, d = sqrt(dx * dx + dy * dy);
                if (d < best) { best = d; bidx = N - 1; }
            }
            int idx = bidx;
            if (c.vp_ordered) start_idx = idx + 2;
            if (idx > N - 2) idx = N - 2;
            if (idx < 1) idx = c.vp_ordered ? 1 : -1;
            W[L.oVPST + j] = (double)idx;
        }
        for (int j = nvp; j < L.V; ++j) W[L.oVPST + j] = -1.0;
    }
    if (repair)
    {
        for (int k = 0; k < N; ++k) project_stage(c, L, W, k);
        repair_lateral_serial(c, L, W);
        for (int k = 0; k < N; ++k) init_controls_stage(c, L, W, k);
        clip_rates_serial(c, L, W, uprev_dt);
    }
    double mu = c.mu_init;
    if (!(mu > 0.0))
    {
        double obj = 0.0, rows = 0.0;
        for (int k = 0; k < N; ++k) auto_mu_stage(c, L, W, uprev_dt, k, &obj, &rows);
        mu = auto_mu(obj, rows);
    }
    for (int k = 0; k < N; ++k) init_duals_stage(c, L, W, uprev_dt, k, mu);
    ASC(MPCB200_SC_MU) = mu; ASC(MPCB200_SC_RHO) = 1.0; ASC(MPCB200_SC_DELTA) = 0.0; ASC(MPCB200_SC_DELTA_LAST) = 0.0;
    ASC(MPCB200_SC_ITER) = 0.0; ASC(MPCB200_SC_STATUS) = -1.0; ASC(MPCB200_SC_NREG) = 0.0; ASC(MPCB200_SC_NBT) = 0.0;
    ASC(MPCB200_SC_DDT) = 0.0; ASC(MPCB200_SC_ALPHA) = 0.0; ASC(MPCB200_SC_TINY) = 0.0; ASC(MPCB200_SC_DEFER) = 0.0;
    if (cold_pending) ASC(MPCB200_SC_COLD) = 0.0;
}

// lanes accumulate their own stages, then a tree reduction in the same xor order as the shuffles
static void reduce_eval(EvalAcc* a)
{
    for (int o = 16; o > 0; o >>= 1)
        for (int l = 0; l < 32; ++l)
            if ((l & o) == 0) { EvalAcc t = a[l]; evalacc_merge(t, a[l ^ o]); a[l] = t; a[l ^ o] = t; }
}

int emu_eval(const Cfg* cp, double* W, double uprev_dt)
{
    const Cfg& c = *cp;
    WsLayout L;
    make_layout(cp, MAX_OBST, MAX_VP, L);
    const int N = L.N;
    if (ASC(MPCB200_SC_STATUS) >= 0.0) return 1;
    EvalAcc a[32];
    for (int l = 0; l < 32; ++l)
    {
        evalacc_init(a[l]);
        for (int k = l; k < N; k += 32) eval_stage(c, L, W, W, uprev_dt, k, a[l]);
    }
    reduce_eval(a);
    int fin = 0;
    const double mu = eval_finish(c, L, W, a[0], true, &fin);
    if (fin) return 1;
    for (int k = 0; k < N; ++k) eval_finalize_stage(L, W, k, mu);
    return 0;
}

int emu_kkt(const Cfg* cp, double* W)
{
    const Cfg& c = *cp;
    WsLayout L;
    make_layout(cp, MAX_OBST, MAX_VP, L);
    const int N = L.N;
    if (ASC(MPCB200_SC_STATUS) >= 0.0) return 1;
    double ddt = 0.0, delta = 0.0;
    int nreg = 0, ok;
    if (kkt_is_ext(c))
    {
        SerialWarp<true> ex;
        kkt_warp_setup<true>(ex, c.variable_dt);
        ok = kkt_warp_solve<true>(ex, c, N, W + L.oKKT, W + L.oMM, W + L.oSTEP, ASC(MPCB200_SC_HTT), ASC(MPCB200_SC_GT), ASC(MPCB200_SC_DELTA_LAST), &ddt, &delta, &nreg);
    }
    else
    {
        SerialWarp<false> ex;
        kkt_warp_setup<false>(ex, c.variable_dt);
        ok = kkt_warp_solve<false>(ex, c, N, W + L.oKKT, W + L.oMM, W + L.oSTEP, ASC(MPCB200_SC_HTT), ASC(MPCB200_SC_GT), ASC(MPCB200_SC_DELTA_LAST), &ddt, &delta, &nreg);
    }
    kkt_store_outcome(W + L.oSCAL, ok, ddt, delta, nreg);
    return ASC(MPCB200_SC_STATUS) >= 0.0 ? 1 : 0;
}

void emu_linesearch(const Cfg* cp, double* W, double uprev_dt)
{
    const Cfg& c = *cp;
    WsLayout L;
    make_layout(cp, MAX_OBST, MAX_VP, L);
    const int N = L.N;
    if (ASC(MPCB200_SC_STATUS) >= 0.0) return;
    if (ASC(MPCB200_SC_DEFER) != 0.0) { ASC(MPCB200_SC_DEFER) = 0.0; ASC(MPCB200_SC_ITER) += 1.0; ASC(MPCB200_SC_ALPHA) = 0.0; return; }
    LsAcc a;
    lsacc_init(a);
    int hist[CLIP_BINS + 1];
    for (int j = 0; j <= CLIP_BINS; ++j) hist[j] = 0;
    for (int l = 0; l < 32; ++l)
    {
        LsAcc t;
        lsacc_init(t);
        for (int k = l; k < N; k += 32) ls_stage_steps(c, L, W, W, uprev_dt, k, t, hist);
        a.a_d = fmin(a.a_d, t.a_d);
        a.dphi_bar += t.dphi_bar; a.curv += t.curv; a.dJ += t.dJ;
    }
    const int jt = clip_threshold_bin(hist, hist[CLIP_BINS]);
    for (int k = 0; k < N; ++k) a.a_p = fmin(a.a_p, ls_stage_ap(L, W, k, jt));
    const double mu = ASC(MPCB200_SC_MU), inf1 = ASC(MPCB200_SC_INF), obj = ASC(MPCB200_SC_OBJ), blog = ASC(MPCB200_SC_BLOG);
    const double ddt = ASC(MPCB200_SC_DDT), dt = ASC(MPCB200_SC_DT);
    double rho = 1.0;
    {
        const double num = a.dJ + a.dphi_bar + 0.5 * (a.curv > 0 ? a.curv : 0.0);
        if (inf1 > 1e-14)
        {
            const double rho_trial = num / ((1.0 - 0.1) * inf1);
            if (rho < rho_trial) rho = rho_trial + 1.0;
        }
    }
    const double phi0 = obj - mu * blog + rho * inf1;
    const double dphi = a.dJ + a.dphi_bar - rho * inf1;
    double alpha = a.a_p;
    int nbt = 0;
    for (int bt = 0; bt < MAX_BACKTRACK; ++bt)
    {
        TrialAcc t;
        t.obj = t.inf1 = t.blog = 0.0;
        for (int k = 0; k < N; ++k) ls_stage_trial(c, L, W, W, uprev_dt, k, alpha, t);
        const double phi = t.obj - mu * t.blog + rho * t.inf1;
        if (phi <= phi0 + ARMIJO * alpha * dphi || (bt > 0 && fabs(phi - phi0) <= 1e-13 * (1.0 + fabs(phi0)))) break;
        alpha *= 0.5;
        ++nbt;
    }
    const double a_dual = a.a_d > alpha ? alpha : a.a_d;
    if (is_midpoint(c))
        for (int k = 0; k < N; ++k) ls_stage_midpoint_fix(c, L, W, k);
    for (int k = 0; k < N; ++k) ls_stage_update(c, L, W, W, uprev_dt, k, alpha, a_dual);
    if (c.variable_dt) ASC(MPCB200_SC_DT) = dt + alpha * ddt;
    ASC(MPCB200_SC_ALPHA) = alpha;
    ASC(MPCB200_SC_RHO) = rho;
    ASC(MPCB200_SC_ITER) += 1.0;
    ASC(MPCB200_SC_NBT) += (double)nbt;
    const double tiny = alpha < TINY_STEP ? ASC(MPCB200_SC_TINY) + 1.0 : 0.0;
    ASC(MPCB200_SC_TINY) = tiny;
    if (tiny >= (double)TINY_STEP_COUNT) ASC(MPCB200_SC_STATUS) = (double)MPCB200_STATUS_NUMERICAL_ERROR;  /* jammed: give up */
}

// whole Controller::step of one instance, same launch sequence as solve_phased() in mpcb200.cu
int emu_solve(const Cfg* cp, double* W, double uprev_dt, int force_cold)
{
    const Cfg& c = *cp;
    WsLayout L;
    make_layout(cp, MAX_OBST, MAX_VP, L);
    emu_init(cp, W, force_cold);
    const int outer = c.outer_iterations > 0 ? c.outer_iterations : 1;
    for (int oi = 0; oi < outer; ++oi)
    {
        emu_associate(cp, W, uprev_dt, oi == 0);
        for (int it = 0; it <= c.max_iter; ++it)
        {
            if (emu_eval(cp, W, uprev_dt)) break;
            if (it == c.max_iter) break;
            if (emu_kkt(cp, W)) break;
            emu_linesearch(cp, W, uprev_dt);
        }
    }
    const double st = ASC(MPCB200_SC_STATUS);
    return st < 0 ? MPCB200_STATUS_MAX_ITER : (int)st;
}

void emu_outputs(const Cfg* cp, const double* W, double* u_seq, double* x_seq)
{
    WsLayout L;
    make_layout(cp, MAX_OBST, MAX_VP, L);
    const int N = L.N;
    for (int k = 0; k < N; ++k)
    {
        const int kk = k <= N - 2 ? k : N - 2;
        u_seq[2 * k] = AU(0, kk); u_seq[2 * k + 1] = AU(1, kk);
        x_seq[3 * k] = AX(0, k); x_seq[3 * k + 1] = AX(1, k); x_seq[3 * k + 2] = normalize_theta(AX(2, k));
    }
}

// the device's horizon change (mpcb200_resample) on one trajectory
double emu_resample(int n, const double* X, const double* U, double dt, int n_new, double* Xn, double* Un)
{
    return resample_serial(n, X, U, dt, n_new, Xn, Un);
}

}  // extern "C"
