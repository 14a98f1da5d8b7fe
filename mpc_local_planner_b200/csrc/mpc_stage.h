// mpc_stage.h -- per-stage (= per-lane) bodies of the solver phases.  A group of lanes (a CTA of ceil(N/32) warps in the
// eval / line-search kernels, one warp in the init kernels) owns one OCP instance and each lane handles the stages
// k = t, t + group size, ...  Each function below is the work of ONE stage; the kernels in mpcb200.cu (and the CPU
// warp emulator in tests/emu, test infrastructure) loop over a lane's stages and combine the accumulators with
// shuffle / shared-memory reductions.  All functions are host/device.
//
// Reference structure restated here:
//   which term attaches to which stage      R/src/optimal_control/finite_differences_grid_se2.cpp:36-152
//   quadratic costs                         R/src/optimal_control/quadratic_cost_se2.cpp:31-52, final_state_conditions_se2.cpp:31-52
//   via-point cost                          R/src/optimal_control/min_time_via_points_cost.cpp:120-145
//   obstacle / control-rate rows            R/src/optimal_control/stage_inequality_se2.cpp:164-222
//   obstacle association                    R/src/optimal_control/stage_inequality_se2.cpp:50-162
//   cold init / warm start                  R/src/optimal_control/full_discretization_grid_base_se2.cpp:192-339
#pragma once
#include "mpc_core.h"

// Where the FULL obstacle list of an instance is read from: the resident image (lists of at most MAX_OBST obstacles are copied
// there and list index = resident slot) or the caller's compact arrays in global memory (longer lists, e.g. the point obstacles of
// a raw costmap: only the obstacles the association selects enter the image).
struct ObstSrc
{
    const double* par;   // [n][MPCB200_OBST_STRIDE]
    const double* td;    // types as doubles (image) ...
    const int* ti;       // ... or as ints (compact input arrays)
    HD int type(int j) const { return ti ? ti[j] : (int)td[j]; }
    HD const double* p(int j) const { return par + (size_t)j * MPCB200_OBST_STRIDE; }
};
#define AX(c_, k_) W[L.oX + (c_) * N + (k_)]
#define AU(c_, k_) W[L.oU + (c_) * N + (k_)]
#define ANU(c_, k_) W[L.oNU + (c_) * N + (k_)]
#define AS(c_, k_) W[L.oS + (c_) * N + (k_)]
#define ALAM(c_, k_) W[L.oLAM + (c_) * N + (k_)]
#define AKKT(c_, k_) W[L.oKKT + (k_) * RSTR + (c_)]  /* stage records [k][RSTR] (odd stride: lane-per-stage accesses without bank conflicts) */
#define ASTEP(c_, k_) W[L.oSTEP + (c_) * N + (k_)]
// associated obstacle per row slot: one signed byte per (slot, stage) -- the RESIDENT slot of the obstacle, -1 = empty
#define AOBS(c_, k_) ((signed char*)(W + L.oOBS))[(c_) * N + (k_)]
#define ADS(c_, k_) W[L.oDS + (c_) * N + (k_)]
// W addresses the instance image: the leading part of the workspace (scalars, inputs, iterate, steps, obstacles), which the
// eval / line-search kernels stage in shared memory; G always addresses the instance's workspace in global memory (fields
// outside the image, and every result that must outlive the kernel).  Host emulator and the init kernels pass W == G.
#define GR0(c_, k_) G[L.oR0 + (c_) * N + (k_)]
#define GOG(c_, k_) G[L.oOG + (c_) * N + (k_)]
#define GX(c_, k_) G[L.oX + (c_) * N + (k_)]
#define GU(c_, k_) G[L.oU + (c_) * N + (k_)]
#define GNU(c_, k_) G[L.oNU + (c_) * N + (k_)]
#define GS(c_, k_) G[L.oS + (c_) * N + (k_)]
#define GLAM(c_, k_) G[L.oLAM + (c_) * N + (k_)]
#define ASC(i_) W[L.oSCAL + (i_)]
#define AIN(i_) W[L.oIN + (i_)]

// ------------------------------------------------------------------------------------------------------
// EVAL
// ------------------------------------------------------------------------------------------------------
struct EvalAcc
{
    double dual_inf, prim_inf, sl_max, sl_min;        // max / max / max / min
    double sum_nu, sum_lam, inf1, blog, gt0, gt1, gldt, htt, obj;  // sums
    double m_ineq, m_eq;                               // counts (as double so that one reduction routine serves all)
};
HD inline void evalacc_init(EvalAcc& a)
{
    a.dual_inf = 0; a.prim_inf = 0; a.sl_max = -1e300; a.sl_min = 1e300;
    a.sum_nu = a.sum_lam = a.inf1 = a.blog = a.gt0 = a.gt1 = a.gldt = a.htt = a.obj = 0.0;
    a.m_ineq = a.m_eq = 0.0;
}
HD inline void evalacc_merge(EvalAcc& a, const EvalAcc& b)
{
    a.dual_inf = fmax(a.dual_inf, b.dual_inf); a.prim_inf = fmax(a.prim_inf, b.prim_inf);
    a.sl_max = fmax(a.sl_max, b.sl_max); a.sl_min = fmin(a.sl_min, b.sl_min);
    a.sum_nu += b.sum_nu; a.sum_lam += b.sum_lam; a.inf1 += b.inf1; a.blog += b.blog; a.gt0 += b.gt0; a.gt1 += b.gt1;
    a.gldt += b.gldt; a.htt += b.htt; a.obj += b.obj; a.m_ineq += b.m_ineq; a.m_eq += b.m_eq;
}

// bookkeeping of one inequality row (owner side): errors + barrier terms.  The barrier term sum(log s) is accumulated
// as a running product that is flushed through one log() every few rows (fp64 log costs ~60 instructions).
struct RowProd { double p; int n; };
HD NOINL inline double log_call(double x) { return log(x); }   // one copy of the fp64 logarithm instead of one per call site
HD inline void rowprod_add(RowProd& rp, double s, double& blog)
{
    rp.p *= s;
    if (++rp.n >= 4) { blog += log_call(rp.p); rp.p = 1.0; rp.n = 0; }
}
HD inline void rowprod_flush(RowProd& rp, double& blog)
{
    if (rp.n > 0) { blog += log_call(rp.p); rp.p = 1.0; rp.n = 0; }
}
HD inline void row_stats(EvalAcc& acc, RowProd& rp, double r, double s, double lam)
{
    acc.prim_inf = fmax(acc.prim_inf, fabs(r));
    acc.inf1 += fabs(r);
    acc.sl_max = fmax(acc.sl_max, s * lam);
    acc.sl_min = fmin(acc.sl_min, s * lam);
    acc.sum_lam += fabs(lam);
    rowprod_add(rp, s, acc.blog);
    acc.m_ineq += 1.0;
}

// One linear row (control bound / control-rate row) seen from stage k's control component I.
//   g: row value, (s, lam): slack / multiplier, gmine: d g / d u_k[I], gdt: d g / d(dt), own: the row belongs to stage k
//   (bookkeeping of errors and dt terms is done once, by the owner), gcross: d g / d u_{k-1}[I] (own rate rows only).
// The arithmetic of a row is ONE function on the device (twelve call sites per stage): the products come back by value.
struct LinTerms { double r, rs, c0g, rsg, lamg, sgg, sgt, sgc, c0t, rst, lamt, sgtt; };
HD NOINL inline LinTerms lin_row_terms(double g, double s, double lam, double gmine, double gdt, double gcross)
{
    LinTerms t;
    const double rs = 1.0 / s;
    const double r = g + s, sig = lam * rs, c0 = sig * r;
    t.r = r; t.rs = rs;
    t.c0g = c0 * gmine; t.rsg = rs * gmine; t.lamg = lam * gmine;
    t.sgg = sig * gmine * gmine; t.sgt = sig * gmine * gdt; t.sgc = sig * gmine * gcross;
    t.c0t = c0 * gdt; t.rst = rs * gdt; t.lamt = lam * gdt; t.sgtt = sig * gdt * gdt;
    return t;
}
// the same row with dt fixed: the terms that do not involve gdt, each formed as in lin_row_terms
struct LinTermsFixed { double r, rs, c0g, rsg, lamg, sgg, sgc; };
HD NOINL inline LinTermsFixed lin_row_terms_fixed(double g, double s, double lam, double gmine, double gcross)
{
    LinTermsFixed t;
    const double rs = 1.0 / s;
    const double r = g + s, sig = lam * rs, c0 = sig * r;
    t.r = r; t.rs = rs;
    t.c0g = c0 * gmine; t.rsg = rs * gmine; t.lamg = lam * gmine;
    t.sgg = sig * gmine * gmine; t.sgc = sig * gmine * gcross;
    return t;
}
// DT = false: dt is fixed (gdt is not read); the dt terms are zero and are not accumulated
template <int I, bool DT>
HD inline void lin_row_accum(double g, double s, double lam, double gmine, double gdt, bool own, double gcross, double* H, double* g0,
                             double* g1, double* GL, double* hb, double* Cc, EvalAcc& acc, RowProd& rp)
{
    if (DT)
    {
        const LinTerms t = lin_row_terms(g, s, lam, gmine, gdt, gcross);
        g0[3 + I] += t.c0g; g1[3 + I] += t.rsg; GL[3 + I] += t.lamg;
        H[hidx(3 + I, 3 + I)] += t.sgg;
        hb[3 + I] += t.sgt;
        if (own)
        {
            Cc[I] += t.sgc;
            row_stats(acc, rp, t.r, s, lam);
            acc.gt0 += t.c0t; acc.gt1 += t.rst; acc.gldt += t.lamt; acc.htt += t.sgtt;
        }
    }
    else
    {
        const LinTermsFixed t = lin_row_terms_fixed(g, s, lam, gmine, gcross);
        g0[3 + I] += t.c0g; g1[3 + I] += t.rsg; GL[3 + I] += t.lamg;
        H[hidx(3 + I, 3 + I)] += t.sgg;
        if (own)
        {
            Cc[I] += t.sgc;
            row_stats(acc, rp, t.r, s, lam);
        }
    }
}

// all linear rows that touch control component I of stage k <= N-2: bounds (slots 2I, 2I+1), own rate rows
// (slots 4+2I, 5+2I) and the rate rows of stage k+1 (gather: their derivative wrt u_k)
template <int I, int MODEL>
HD inline void lin_rows_component(const Cfg& c, const WsLayout& L, const double* W, double uprev_dt, int k, double dt, double u_i, double* H,
                                  double* g0, double* g1, double* GL, double* hb, double* Cc, EvalAcc& acc, RowProd& rp)
{
    using T_ = ModelTraits<MODEL>;
    constexpr bool DT = T_::DT_TERMS;
    const int N = L.N;
    // control bounds
    if (T_::row_finite(c, 2 * I)) lin_row_accum<I, DT>(c.u_lb[I] - u_i, AS(2 * I, k), ALAM(2 * I, k), -1.0, 0.0, true, 0.0, H, g0, g1, GL, hb, Cc, acc, rp);
    if (T_::row_finite(c, 2 * I + 1)) lin_row_accum<I, DT>(u_i - c.u_ub[I], AS(2 * I + 1, k), ALAM(2 * I + 1, k), 1.0, 0.0, true, 0.0, H, g0, g1, GL, hb, Cc, acc, rp);
    const bool has_lb = T_::row_finite(c, 4 + 2 * I), has_ub = T_::row_finite(c, 5 + 2 * I);
    if (!has_lb && !has_ub) return;
    // own rate rows: Delta = u_k - u_{k-1}; k = 0 uses (u_prev, dt_prev) and is absent when dt_prev == 0
    if (!(k == 0 && uprev_dt == 0.0))
    {
        const double um = (k >= 1) ? AU(I, k - 1) : AIN(IN_UPREV + I);
        const double T = (k >= 1) ? dt : uprev_dt;
        const double delta = u_i - um;
        const double cross = (k >= 1) ? 1.0 : 0.0;             // d/du_{k-1} exists only for k >= 1
        const double dtf = (k >= 1 && T_::variable_dt(c)) ? 1.0 : 0.0;
        if (has_lb) lin_row_accum<I, DT>(-(delta - c.du_lb[I] * T), AS(4 + 2 * I, k), ALAM(4 + 2 * I, k), -1.0, dtf * c.du_lb[I], true, cross * 1.0, H, g0, g1, GL, hb, Cc, acc, rp);
        if (has_ub) lin_row_accum<I, DT>(delta - c.du_ub[I] * T, AS(5 + 2 * I, k), ALAM(5 + 2 * I, k), 1.0, -dtf * c.du_ub[I], true, cross * -1.0, H, g0, g1, GL, hb, Cc, acc, rp);
    }
    // rate rows of stage k+1: Delta' = u_{k+1} - u_k (u_{N-1} := u_ref = 0); derivative wrt u_k is -sgn
    {
        const int kk = k + 1;
        const double un = (kk <= N - 2) ? AU(I, kk) : 0.0;
        const double delta = un - u_i;
        const double dtf = T_::variable_dt(c) ? 1.0 : 0.0;
        if (has_lb) lin_row_accum<I, DT>(-(delta - c.du_lb[I] * dt), AS(4 + 2 * I, kk), ALAM(4 + 2 * I, kk), 1.0, dtf * c.du_lb[I], false, 0.0, H, g0, g1, GL, hb, Cc, acc, rp);
        if (has_ub) lin_row_accum<I, DT>(delta - c.du_ub[I] * dt, AS(5 + 2 * I, kk), ALAM(5 + 2 * I, kk), -1.0, -dtf * c.du_ub[I], false, 0.0, H, g0, g1, GL, hb, Cc, acc, rp);
    }
}

// Stage functions + derivatives of stage k -> condensed KKT record (G holds the mu-independent part g0, the
// coefficient of mu is parked in STEP[0..4][k] until the barrier parameter is decided), error accumulators.
// LINES = false compiles the rarely used obstacle kinds out (line obstacles, moving obstacles): see footprint_distance_sc;
// MODEL fixes the robot and footprint model at compile time (ModelTraits)
template <bool LINES = true, int MODEL = MODEL_GENERIC>
HD inline void eval_stage(const Cfg& c, const WsLayout& L, double* W, double* G, double uprev_dt, int k, EvalAcc& acc)
{
    using T_ = ModelTraits<MODEL>;
    const int N = L.N, K = L.K;
    const double dt = ASC(MPCB200_SC_DT);
    const bool vdt = T_::variable_dt(c);
    double H[15], g0[5], g1[5], GL[5], a3[3], Bm[6], e[3], Cc[2], hb[5], dvec[3];
#pragma unroll
    for (int i = 0; i < 15; ++i) H[i] = 0.0;
#pragma unroll
    for (int i = 0; i < 5; ++i) { g0[i] = 0; g1[i] = 0; GL[i] = 0; hb[i] = 0; }
#pragma unroll
    for (int i = 0; i < 3; ++i) { a3[i] = 0; e[i] = 0; dvec[i] = 0; }
#pragma unroll
    for (int i = 0; i < 6; ++i) Bm[i] = 0;
    Cc[0] = Cc[1] = 0.0;
    RowProd rp; rp.p = 1.0; rp.n = 0;
    const double x[3] = {AX(0, k), AX(1, k), AX(2, k)};
    const double xf[3] = {AIN(IN_XF), AIN(IN_XF + 1), AIN(IN_XF + 2)};
    double sc[2];
    sincos(x[2], &sc[0], &sc[1]);  // shared by the dynamics and every footprint distance of this stage

    if (k <= N - 2)
    {
        const double u[2] = {AU(0, k), AU(1, k)};
        const double nu[3] = {ANU(0, k), ANU(1, k), ANU(2, k)};
        double f[3], J[9], Hc[6];
        // midpoint differences (fd_collocation_se2.h:91-108) evaluate f at the mean heading of the interval; see midpoint_* below
        const bool mid = LINES && is_midpoint(c);
        const double dth = normalize_theta(AX(2, k + 1) - x[2]);
        if (mid) dynamics_derivs<MODEL>(c, x[2] + 0.5 * dth, u[0], u[1], nu, f, J, Hc, nullptr);
        else dynamics_derivs<MODEL>(c, x[2], u[0], u[1], nu, f, J, Hc, sc);
        e[0] = x[0] + dt * f[0] - AX(0, k + 1);
        e[1] = x[1] + dt * f[1] - AX(1, k + 1);
        e[2] = dt * f[2] - dth;
#pragma unroll
        for (int i = 0; i < 3; ++i)
        {
            dvec[i] = f[i];
            a3[i] = dt * J[i * 3 + 0];
            Bm[2 * i] = dt * J[i * 3 + 1];
            Bm[2 * i + 1] = dt * J[i * 3 + 2];
            acc.prim_inf = fmax(acc.prim_inf, fabs(e[i]));
            acc.inf1 += fabs(e[i]);
            acc.sum_nu += fabs(nu[i]);
        }
        acc.m_eq += 3.0;
        if (mid)
        {
            // the defect depends on x_{k+1} through the mean heading: de/dx_k = I + a e_th', de/dx_{k+1} = -(I - a e_th'),
            // a = dt/2 f_theta (a_theta = 0 for every model).  Multiplying the linearised row by (I - a e_th')^{-1} = I + a e_th'
            // restores the explicit form dx_{k+1} = (I + 2a e_th') dx_k + B~ du + d~ d(dt) + e~ the Riccati sweep expects
            // (a3 above is already 2a); the multiplier it returns belongs to the transformed row (ls_stage_update undoes this).
#pragma unroll
            for (int i = 0; i < 2; ++i)
            {
                const double ai = 0.5 * a3[i];
                Bm[2 * i] += ai * Bm[4]; Bm[2 * i + 1] += ai * Bm[5];
                dvec[i] += ai * dvec[2];
                e[i] += ai * e[2];
            }
        }
        // quadratic running cost (k = 0 state term is a constant: its gradient is never used since x_0 is fixed)
        if (T_::quadratic(c))
        {
            // integral form: dt * (w_k l_x(x_k) + l_u(u_k)), w_k the state weight of the integration rule (left sum or
            // trapezoid, integral_state_weight); then the dt-gradient is w_k l_x + l_u and the w-dt cross Hessian its gradient
            const bool integ = T_::integral(c);
            const double fx = integ ? integral_state_weight(c, N, k) : 1.0;
            const double wx = integ ? dt * fx : 1.0, wu = integ ? dt : 1.0;
            const double d[3] = {x[0] - xf[0], x[1] - xf[1], normalize_theta(x[2] - xf[2])};
            double ox = 0.0, ou = 0.0;
#pragma unroll
            for (int i = 0; i < 3; ++i)
            {
                double gi = 0.0;
#pragma unroll
                for (int j = 0; j < 3; ++j)
                {
                    gi += (c.Q[i * 3 + j] + c.Q[j * 3 + i]) * d[j];
                    ox += d[i] * c.Q[i * 3 + j] * d[j];
                    if (j >= i) H[hidx(i, j)] += wx * (c.Q[i * 3 + j] + c.Q[j * 3 + i]);
                }
                g0[i] += wx * gi; GL[i] += wx * gi;
                if (integ && vdt) hb[i] += fx * gi;
            }
#pragma unroll
            for (int i = 0; i < 2; ++i)
            {
                double gi = 0.0;
#pragma unroll
                for (int j = 0; j < 2; ++j)
                {
                    gi += (c.R[i * 2 + j] + c.R[j * 2 + i]) * u[j];
                    ou += u[i] * c.R[i * 2 + j] * u[j];
                    if (j >= i) H[hidx(3 + i, 3 + j)] += wu * (c.R[i * 2 + j] + c.R[j * 2 + i]);
                }
                g0[3 + i] += wu * gi; GL[3 + i] += wu * gi;
                if (integ && vdt) hb[3 + i] += gi;
            }
            acc.obj += wx * ox + wu * ou;
            if (integ && vdt) { acc.gt0 += fx * ox + ou; acc.gldt += fx * ox + ou; }
        }
        // Lagrangian terms of nu_k^T e_k
        const double fx_nu = nu[0] * J[0] + nu[1] * J[3] + nu[2] * J[6];
        const double fu_nu0 = nu[0] * J[1] + nu[1] * J[4] + nu[2] * J[7];
        const double fu_nu1 = nu[0] * J[2] + nu[1] * J[5] + nu[2] * J[8];
        acc.gldt += nu[0] * f[0] + nu[1] * f[1] + nu[2] * f[2];
        GL[0] += nu[0]; GL[1] += nu[1];
        GL[3] += dt * fu_nu0; GL[4] += dt * fu_nu1;
        H[hidx(3, 3)] += dt * Hc[3]; H[hidx(3, 4)] += dt * Hc[4]; H[hidx(4, 4)] += dt * Hc[5];
        if (vdt) { hb[3] += fu_nu0; hb[4] += fu_nu1; }
        if (!mid)
        {
            GL[2] += nu[2] + dt * fx_nu;
            H[hidx(2, 2)] += dt * Hc[0]; H[hidx(2, 3)] += dt * Hc[1]; H[hidx(2, 4)] += dt * Hc[2];
            if (vdt) hb[2] += fx_nu;
        }
        else
        {
            // theta_k enters through the mean heading with weight 1/2
            GL[2] += nu[2] + 0.5 * dt * fx_nu;
            H[hidx(2, 2)] += 0.25 * dt * Hc[0]; H[hidx(2, 3)] += 0.5 * dt * Hc[1]; H[hidx(2, 4)] += 0.5 * dt * Hc[2];
            if (vdt) hb[2] += 0.5 * fx_nu;
            // Hessian block between theta_{k+1} and (theta_k, u_k): q = (dt/4 Hc_tt, dt/2 Hc_t0, dt/2 Hc_t1).  It is condensed
            // into this stage with the linearised heading row d(theta_{k+1}) = r' dw_k + e~_2 + d~_2 d(dt), r = (1, B~_20, B~_21):
            // H += q r' + r q', Newton gradient += q e~_2, dt border += q d~_2 (exact; DESIGN.md "midpoint differences")
            const double q[3] = {0.25 * dt * Hc[0], 0.5 * dt * Hc[1], 0.5 * dt * Hc[2]};
            const double r[3] = {1.0, Bm[4], Bm[5]};
#pragma unroll
            for (int i = 0; i < 3; ++i)
            {
#pragma unroll
                for (int j = i; j < 3; ++j) H[hidx(2 + i, 2 + j)] += q[i] * r[j] + r[i] * q[j];
                g0[2 + i] += q[i] * e[2];
                if (vdt) hb[2 + i] += q[i] * dvec[2];
            }
        }
        // linear rows touching u_k (own bounds, own rate rows, rate rows of stage k+1)
        lin_rows_component<0, MODEL>(c, L, W, uprev_dt, k, dt, u[0], H, g0, g1, GL, hb, Cc, acc, rp);
        lin_rows_component<1, MODEL>(c, L, W, uprev_dt, k, dt, u[1], H, g0, g1, GL, hb, Cc, acc, rp);
    }
    else
    {
        // terminal stage k = N-1: terminal cost, dt-bound rows (slots 0,1), final control-rate rows (slots 4..7; their
        // contribution to u_{N-2} is gathered by stage N-2 above), minimum-time term
        if (has_terminal_cost(c))
        {
            const double d[3] = {x[0] - xf[0], x[1] - xf[1], normalize_theta(x[2] - xf[2])};
            double o = 0.0;
#pragma unroll
            for (int i = 0; i < 3; ++i)
            {
                double gi = 0.0;
#pragma unroll
                for (int j = 0; j < 3; ++j)
                {
                    gi += (c.Qf[i * 3 + j] + c.Qf[j * 3 + i]) * d[j];
                    o += d[i] * c.Qf[i * 3 + j] * d[j];
                    if (j >= i) H[hidx(i, j)] += c.Qf[i * 3 + j] + c.Qf[j * 3 + i];
                }
                g0[i] += gi; GL[i] += gi;
            }
            acc.obj += o;
        }
        if (T_::trapezoid(c))
        {
            // end term of the trapezoidal rule: dt/2 * l_x(x_{N-1})
            const double fx = integral_state_weight(c, N, k);
            const double d[3] = {x[0] - xf[0], x[1] - xf[1], normalize_theta(x[2] - xf[2])};
            double ox = 0.0;
#pragma unroll
            for (int i = 0; i < 3; ++i)
            {
                double gi = 0.0;
#pragma unroll
                for (int j = 0; j < 3; ++j)
                {
                    gi += (c.Q[i * 3 + j] + c.Q[j * 3 + i]) * d[j];
                    ox += d[i] * c.Q[i * 3 + j] * d[j];
                    if (j >= i) H[hidx(i, j)] += dt * fx * (c.Q[i * 3 + j] + c.Q[j * 3 + i]);
                }
                g0[i] += dt * fx * gi; GL[i] += dt * fx * gi;
                if (vdt) hb[i] += fx * gi;
            }
            acc.obj += dt * fx * ox;
            if (vdt) { acc.gt0 += fx * ox; acc.gldt += fx * ox; }
        }
        if (T_::mintime(c)) { acc.gt0 += (double)(N - 1); acc.gldt += (double)(N - 1); acc.obj += (double)(N - 1) * dt; }
        for (int sl = 0; sl < 8; ++sl)
        {
            if (!lin_row_active<MODEL>(c, N, k, sl, uprev_dt)) continue;
            const int i = (sl < 4) ? (sl >> 1) : ((sl - 4) >> 1);
            double gu, gum, gdt;
            const double um = (sl >= 4) ? AU(i, k - 1) : 0.0;
            const double g = lin_row<MODEL>(c, N, k, sl, 0.0, um, dt, uprev_dt, gu, gum, gdt);
            const double s = AS(sl, k), lam = ALAM(sl, k);
            const double rs = 1.0 / s, r = g + s, sig = lam * rs, c0 = sig * r;
            row_stats(acc, rp, r, s, lam);
            if (T_::DT_TERMS) { acc.gt0 += c0 * gdt; acc.gt1 += rs * gdt; acc.gldt += lam * gdt; acc.htt += sig * gdt * gdt; }
        }
        if (T_::ball(c))
        {
            // terminal ball on x_{N-1} (slot BALL_SLOT): a nonlinear state row, handled like an obstacle row
            double gr[3], hd[6];
            const double g = ball_row(c, x, xf, gr, hd);
            const double s = AS(BALL_SLOT, k), lam = ALAM(BALL_SLOT, k);
            const double rs = 1.0 / s, r = g + s, sig = lam * rs, c0 = sig * r;
            row_stats(acc, rp, r, s, lam);
            int q = 0;
#pragma unroll
            for (int i = 0; i < 3; ++i)
            {
                g0[i] += c0 * gr[i]; g1[i] += rs * gr[i]; GL[i] += lam * gr[i];
#pragma unroll
                for (int jj = i; jj < 3; ++jj, ++q) H[hidx(i, jj)] += lam * hd[q] + sig * gr[i] * gr[jj];
            }
        }
    }
    // multiplier of the previous defect: d/dx_k ( nu_{k-1}^T e_{k-1} ) = -nu_{k-1}
    if (k >= 1) { GL[0] -= ANU(0, k - 1); GL[1] -= ANU(1, k - 1); GL[2] -= ANU(2, k - 1); }
    if (LINES && is_midpoint(c) && k >= 1)
    {
        // midpoint differences: theta_k is also the far end of interval k-1 (weight 1/2 in its mean heading)
        const double nup[3] = {ANU(0, k - 1), ANU(1, k - 1), ANU(2, k - 1)};
        double fp[3], Jp[9], Hp[6];
        dynamics_derivs<MODEL>(c, AX(2, k - 1) + 0.5 * normalize_theta(x[2] - AX(2, k - 1)), AU(0, k - 1), AU(1, k - 1), nup, fp, Jp, Hp, nullptr);
        const double fx_nu_p = nup[0] * Jp[0] + nup[1] * Jp[3] + nup[2] * Jp[6];
        GL[2] += 0.5 * dt * fx_nu_p;
        H[hidx(2, 2)] += 0.25 * dt * Hp[0];
        if (vdt) hb[2] += 0.5 * fx_nu_p;
    }
    // via-points attached to this stage
    if (has_viapoints(c) && k >= 1 && k <= N - 2)
    {
        const int nvp = (int)AIN(IN_NVP);
        for (int j = 0; j < nvp && j < L.V; ++j)
        {
            if ((int)W[L.oVPST + j] != k) continue;
            const double w = c.vp_position_weight;
            const double ex = W[L.oVP + 3 * j] - x[0], ey = W[L.oVP + 3 * j + 1] - x[1];
            g0[0] += -2 * w * ex; GL[0] += -2 * w * ex;
            g0[1] += -2 * w * ey; GL[1] += -2 * w * ey;
            H[hidx(0, 0)] += 2 * w; H[hidx(1, 1)] += 2 * w;
            acc.obj += w * (ex * ex + ey * ey);
            if (c.vp_orientation_weight > 0)
            {
                g0[2] += -c.vp_orientation_weight; GL[2] += -c.vp_orientation_weight;
                acc.obj += c.vp_orientation_weight * normalize_theta(W[L.oVP + 3 * j + 2] - x[2]);
            }
        }
    }
    // obstacle rows (k = 1..N-2); value and gradient are kept for the line-search kernel
    if (k >= 1 && k <= N - 2)
    {
        for (int j = 0; j < K; ++j)
        {
            const int oi = (int)AOBS(j, k);
            if (oi < 0) continue;
            double gd[3], hd[6], ob[5];
            const double* op = W + L.oOBST + oi * MPCB200_OBST_STRIDE;
            const double dist = footprint_distance_sc<true, true, LINES, MODEL>(c, x[0], x[1], sc[0], sc[1], (int)W[L.oOTYPE + oi],
                                                                  LINES ? obstacle_at(c, op, k, dt, ob) : op, gd, hd);
            const double g = c.min_obstacle_dist - dist;
            const double s = AS(8 + j, k), lam = ALAM(8 + j, k);
            const double rs = 1.0 / s, r = g + s, sig = lam * rs, c0 = sig * r;
            row_stats(acc, rp, r, s, lam);
            const double gr[3] = {-gd[0], -gd[1], -gd[2]};
            if (LINES && vdt && obstacle_is_dynamic(c, op))
            {
                // g = G(p - o - k dt v, theta): dg/ddt = -k grad_p g . v, d2g/dpose ddt = -k H_g v, d2g/ddt2 = k^2 v'H_g v  (H_g = -hd)
                const double kk = (double)k, vx = op[5], vy = op[6];
                const double gdt = -kk * (gr[0] * vx + gr[1] * vy);
                const double hx = -(hd[0] * vx + hd[1] * vy), hy = -(hd[1] * vx + hd[3] * vy), ht = -(hd[2] * vx + hd[4] * vy);
                hb[0] += lam * (-kk * hx) + sig * gr[0] * gdt;
                hb[1] += lam * (-kk * hy) + sig * gr[1] * gdt;
                hb[2] += lam * (-kk * ht) + sig * gr[2] * gdt;
                acc.htt += lam * (kk * kk * (vx * hx + vy * hy)) + sig * gdt * gdt;
                acc.gt0 += c0 * gdt; acc.gt1 += rs * gdt; acc.gldt += lam * gdt;
            }
            GOG(4 * j + 0, k) = g; GOG(4 * j + 1, k) = gr[0]; GOG(4 * j + 2, k) = gr[1]; GOG(4 * j + 3, k) = gr[2];
            int q = 0;
#pragma unroll
            for (int i = 0; i < 3; ++i)
            {
                g0[i] += c0 * gr[i]; g1[i] += rs * gr[i]; GL[i] += lam * gr[i];
#pragma unroll
                for (int jj = i; jj < 3; ++jj, ++q) H[hidx(i, jj)] += lam * (-hd[q]) + sig * gr[i] * gr[jj];
            }
        }
    }
    rowprod_flush(rp, acc.blog);
    // dual infeasibility over the free variables of this stage
#pragma unroll
    for (int i = 0; i < 5; ++i)
    {
        if (i < 3 && k == 0) continue;
        if (i < 3 && k == N - 1 && c.xf_fixed[i]) continue;
        if (i >= 3 && k == N - 1) continue;
        acc.dual_inf = fmax(acc.dual_inf, fabs(GL[i]));
    }
    // store the record
#pragma unroll
    for (int i = 0; i < 15; ++i) AKKT(MPCB200_K_H + i, k) = H[i];
#pragma unroll
    for (int i = 0; i < 5; ++i) { ADS(i, k) = g0[i]; ASTEP(i, k) = g1[i]; AKKT(MPCB200_K_HB + i, k) = hb[i]; }  // g = g0 + mu g1 is stored by eval_finalize_stage
    // (g0, g1 wait in the image -- DS / STEP are free during the evaluation -- so that the record is written exactly once)
#pragma unroll
    for (int i = 0; i < 3; ++i) { AKKT(MPCB200_K_A + i, k) = a3[i]; AKKT(MPCB200_K_E + i, k) = e[i]; AKKT(MPCB200_K_D + i, k) = dvec[i]; }
#pragma unroll
    for (int i = 0; i < 6; ++i) AKKT(MPCB200_K_B + i, k) = Bm[i];
    AKKT(MPCB200_K_C + 0, k) = Cc[0];
    AKKT(MPCB200_K_C + 1, k) = Cc[1];
}

// After the warp reduction: convergence test, monotone barrier update (Ipopt's Fiacco-McCormick rule), scalars.
// Returns the barrier parameter to finalise the gradients with; *finished is set when the instance terminates.
// expired: the time budget of the solve (max_cpu_time) has run out.  It is tested after the iteration cap, so an instance stopped
// here at iteration j holds exactly what a solve with max_iter = j leaves; only the status differs.
template <int MODEL = MODEL_GENERIC>
HD inline double eval_finish(const Cfg& c, const WsLayout& L, double* W, const EvalAcc& a, bool write, int* finished, bool expired = false)
{
    double mu = ASC(MPCB200_SC_MU);
    const double tol = c.tol, mu_min = tol / 10.0;
    const int m_eq = (int)a.m_eq, m_in = (int)a.m_ineq;
    double dual_inf = a.dual_inf;
    if (ModelTraits<MODEL>::variable_dt(c)) dual_inf = fmax(dual_inf, fabs(a.gldt));
    const double e0 = scaled_error(dual_inf, a.prim_inf, a.sl_max, a.sl_min, a.sum_nu, a.sum_lam, m_eq, m_in, 0.0);
    double emu = scaled_error(dual_inf, a.prim_inf, a.sl_max, a.sl_min, a.sum_nu, a.sum_lam, m_eq, m_in, mu);
    const int iter = (int)ASC(MPCB200_SC_ITER);
    int fin = 0, status = -1;
    if (e0 <= tol) { fin = 1; status = MPCB200_STATUS_CONVERGED; }
    else if (iter >= c.max_iter) { fin = 1; status = MPCB200_STATUS_MAX_ITER; }
    else if (expired) { fin = 1; status = MPCB200_STATUS_MAX_TIME; }
    if (!(e0 == e0)) { fin = 1; status = MPCB200_STATUS_NUMERICAL_ERROR; }
    if (!fin)
    {
        while (emu <= KAPPA_EPS * mu && mu > mu_min)
        {
            double m1 = KAPPA_MU * mu, m2 = pow(mu, THETA_MU);
            mu = m1 < m2 ? m1 : m2;
            if (mu < mu_min) mu = mu_min;
            emu = scaled_error(dual_inf, a.prim_inf, a.sl_max, a.sl_min, a.sum_nu, a.sum_lam, m_eq, m_in, mu);
        }
    }
    if (write)
    {
        ASC(MPCB200_SC_MU) = mu;
        ASC(MPCB200_SC_ERR0) = e0;
        ASC(MPCB200_SC_ERRMU) = emu;
        ASC(MPCB200_SC_HTT) = a.htt;
        ASC(MPCB200_SC_GT) = a.gt0 + mu * a.gt1;
        ASC(MPCB200_SC_GLDT) = a.gldt;
        ASC(MPCB200_SC_OBJ) = a.obj;
        ASC(MPCB200_SC_INF) = a.inf1;
        ASC(MPCB200_SC_BLOG) = a.blog;
        if (fin) ASC(MPCB200_SC_STATUS) = (double)status;
    }
    *finished = fin;
    return mu;
}
HD inline void eval_finalize_stage(const WsLayout& L, double* W, int k, double mu)
{
    const int N = L.N;
#pragma unroll
    for (int i = 0; i < 5; ++i) AKKT(MPCB200_K_G + i, k) = ADS(i, k) + mu * ASTEP(i, k);
}

// ------------------------------------------------------------------------------------------------------
// LINE SEARCH
// ------------------------------------------------------------------------------------------------------
struct LsAcc
{
    double a_p, a_d;                 // min
    double dphi_bar, curv, dJ;       // sums
};
HD inline void lsacc_init(LsAcc& a) { a.a_p = 1.0; a.a_d = 1.0; a.dphi_bar = a.curv = a.dJ = 0.0; }

// slack / multiplier steps of the rows owned by stage k, fraction to the boundary, directional derivatives
// hist: CLIP_BINS counters of the blocking step ratios + one counter of the active rows (shared memory in the kernel)
#ifdef __CUDA_ARCH__
#define HIST_ADD(p_) atomicAdd((p_), 1)
#else
#define HIST_ADD(p_) (++*(p_))
#endif
// part: PART_BASE = the linear rows, the terminal ball, the objective and curvature terms; PART_OBST = the obstacle rows
#define PART_BASE 1
#define PART_OBST 2
#define PART_ALL 3
template <int MODEL = MODEL_GENERIC>
HD inline void ls_stage_steps(const Cfg& c, const WsLayout& L, double* W, double* G, double uprev_dt, int k, LsAcc& acc, int* hist, int part = PART_ALL)
{
    using T_ = ModelTraits<MODEL>;
    const int N = L.N, K = L.K;
    const bool vdt = T_::variable_dt(c);
    const double dt = ASC(MPCB200_SC_DT), mu = ASC(MPCB200_SC_MU), ddt = ASC(MPCB200_SC_DDT);
    const double delta = ASC(MPCB200_SC_DELTA);
    const double tau = (1.0 - mu > TAU_MIN) ? 1.0 - mu : TAU_MIN;
    const double x[3] = {AX(0, k), AX(1, k), AX(2, k)};
    const double dx[3] = {ASTEP(0, k), ASTEP(1, k), ASTEP(2, k)};
    const double xf[3] = {AIN(IN_XF), AIN(IN_XF + 1), AIN(IN_XF + 2)};
    double du[2] = {0, 0};
    if (k <= N - 2) { du[0] = ASTEP(3, k); du[1] = ASTEP(4, k); }
    // rows: slack / multiplier steps.  Linear rows are re-evaluated (pure arithmetic); obstacle rows reuse the value and
    // gradient stored by the EVAL kernel at this very point.  r0 = g + s is kept for the analytic trial evaluation.
    for (int sl = (part & PART_BASE) ? 0 : 8; sl < ((part & PART_OBST) ? 8 + K : 8); ++sl)
    {
        double g, gdz;
        if (sl == BALL_SLOT && k == N - 1 && T_::ball(c))
        {
            double gr[3];
            g = ball_row(c, x, xf, gr, nullptr);
            gdz = gr[0] * dx[0] + gr[1] * dx[1] + gr[2] * dx[2];
        }
        else if (sl < 8)
        {
            if (!lin_row_active<MODEL>(c, N, k, sl, uprev_dt)) { ADS(sl, k) = 0.0; GR0(sl, k) = 0.0; continue; }
            const int i = (sl < 4) ? (sl >> 1) : ((sl - 4) >> 1);
            const double uk = (k <= N - 2) ? AU(i, k) : 0.0;
            const double um = (sl >= 4) ? ((k >= 1) ? AU(i, k - 1) : AIN(IN_UPREV + i)) : 0.0;
            double gu, gum, gdt;
            g = lin_row<MODEL>(c, N, k, sl, uk, um, dt, uprev_dt, gu, gum, gdt);
            gdz = gu * du[i] + gdt * ddt;
            if (gum != 0.0) gdz += gum * ASTEP(3 + i, k - 1);
        }
        else
        {
            const int j = sl - 8;
            const int oi = (k >= 1 && k <= N - 2) ? (int)AOBS(j, k) : -1;
            if (oi < 0) { ADS(sl, k) = 0.0; GR0(sl, k) = 0.0; continue; }
            g = GOG(4 * j + 0, k);
            gdz = GOG(4 * j + 1, k) * dx[0] + GOG(4 * j + 2, k) * dx[1] + GOG(4 * j + 3, k) * dx[2];
            const double* op = W + L.oOBST + oi * MPCB200_OBST_STRIDE;
            if (vdt && obstacle_is_dynamic(c, op)) gdz += -(double)k * (GOG(4 * j + 1, k) * op[5] + GOG(4 * j + 2, k) * op[6]) * ddt;
        }
        const double s = AS(sl, k), lam = ALAM(sl, k);
        const double rs = 1.0 / s;
        const double r0 = g + s;
        const double ds = -r0 - gdz;
        // explicit fused multiply-adds: left to the compiler, the contraction of this expression differed between the solve
        // kernel and the phase kernels (sm_90a), and with it the dual step length of the two execution modes
        const double dl = fma(-(lam * rs), ds, fma(mu, rs, -lam));
        ADS(sl, k) = ds;
        GR0(sl, k) = r0;
        HIST_ADD(hist + CLIP_BINS);
        // (cross-multiplied tests first: the fp64 divisions are paid by the blocking rows only)
        if (ds < 0 && tau * s < -ds) { const double r = -tau * s / ds; if (r < 1.0) HIST_ADD(hist + clip_bin(r)); }
        if (dl < 0 && tau * lam < -dl * acc.a_d) acc.a_d = fmin(acc.a_d, -tau * lam / dl);
        acc.dphi_bar += -mu * ds * rs;
        acc.curv += (lam * rs) * ds * ds;
    }
    if (!(part & PART_BASE)) return;
    // directional derivative of the objective
    double dJ = 0.0;
    if (k <= N - 2)
    {
        if (T_::quadratic(c))
        {
            const double d[3] = {x[0] - xf[0], x[1] - xf[1], normalize_theta(x[2] - xf[2])};
            const double u[2] = {AU(0, k), AU(1, k)};
            const bool integ = T_::integral(c);
            const double fx = integ ? integral_state_weight(c, N, k) : 1.0;
            const double wx = integ ? ASC(MPCB200_SC_DT) * fx : 1.0, wu = integ ? ASC(MPCB200_SC_DT) : 1.0;
            double dlx = 0.0, dlu = 0.0, lx = 0.0, lu = 0.0;
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) { dlx += (c.Q[i * 3 + j] + c.Q[j * 3 + i]) * d[j] * dx[i]; lx += d[i] * c.Q[i * 3 + j] * d[j]; }
            for (int i = 0; i < 2; ++i)
                for (int j = 0; j < 2; ++j) { dlu += (c.R[i * 2 + j] + c.R[j * 2 + i]) * u[j] * du[i]; lu += u[i] * c.R[i * 2 + j] * u[j]; }
            dJ += wx * dlx + wu * dlu + ((integ && vdt) ? (fx * lx + lu) * ddt : 0.0);
        }
    }
    else
    {
        if (T_::mintime(c)) dJ += (double)(N - 1) * ddt;
        if (has_terminal_cost(c))
        {
            const double d[3] = {x[0] - xf[0], x[1] - xf[1], normalize_theta(x[2] - xf[2])};
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) dJ += (c.Qf[i * 3 + j] + c.Qf[j * 3 + i]) * d[j] * dx[i];
        }
        if (T_::trapezoid(c))
        {
            const double fx = integral_state_weight(c, N, k);
            const double d[3] = {x[0] - xf[0], x[1] - xf[1], normalize_theta(x[2] - xf[2])};
            double dlx = 0.0, lx = 0.0;
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) { dlx += (c.Q[i * 3 + j] + c.Q[j * 3 + i]) * d[j] * dx[i]; lx += d[i] * c.Q[i * 3 + j] * d[j]; }
            dJ += ASC(MPCB200_SC_DT) * fx * dlx + (vdt ? fx * lx * ddt : 0.0);
        }
    }
    if (has_viapoints(c) && k >= 1 && k <= N - 2)
    {
        const int nvp = (int)AIN(IN_NVP);
        for (int j = 0; j < nvp && j < L.V; ++j)
        {
            if ((int)W[L.oVPST + j] != k) continue;
            const double w = c.vp_position_weight;
            dJ += -2 * w * (W[L.oVP + 3 * j] - x[0]) * dx[0];
            dJ += -2 * w * (W[L.oVP + 3 * j + 1] - x[1]) * dx[1];
            if (c.vp_orientation_weight > 0) dJ += -c.vp_orientation_weight * dx[2];
        }
    }
    acc.dJ += dJ;
    // curvature dz' H dz of this stage's block (+ cross block with stage k-1, + border)
    {
        // (unrolled over the largest block with the bound as a condition: st stays in registers)
        const int nv = (k <= N - 2) ? 5 : 3;
        const double st[5] = {dx[0], dx[1], dx[2], du[0], du[1]};
        double cv = 0.0;
#pragma unroll
        for (int i = 0; i < 5; ++i)
#pragma unroll
            for (int j = 0; j < 5; ++j)
            {
                if (i >= nv || j >= nv) continue;
                const int a = i < j ? i : j, b = i < j ? j : i;
                cv += st[i] * (AKKT(MPCB200_K_H + hidx(a, b), k) + (a == b ? delta : 0.0)) * st[j];
            }
        if (k >= 1 && k <= N - 2)
            for (int i = 0; i < 2; ++i) cv += 2.0 * ASTEP(3 + i, k - 1) * AKKT(MPCB200_K_C + i, k) * du[i];
        if (vdt)  // border (the terminal record carries one only with the trapezoidal rule)
#pragma unroll
            for (int i = 0; i < 5; ++i)
                if (i < nv) cv += 2.0 * ddt * AKKT(MPCB200_K_HB + i, k) * st[i];
        if (vdt && k == N - 1) cv += ddt * ddt * (ASC(MPCB200_SC_HTT) + delta);
        acc.curv += cv;
    }
}

// primal step length: smallest step ratio over the rows of stage k that are not clipped (bins below jt)
HD inline double ls_stage_ap(const WsLayout& L, const double* W, int k, int jt, int part = PART_ALL)
{
    const int N = L.N, RS = L.RS;
    const double mu = ASC(MPCB200_SC_MU);
    const double tau = (1.0 - mu > TAU_MIN) ? 1.0 - mu : TAU_MIN;
    double a_p = 1.0;
    for (int sl = (part & PART_BASE) ? 0 : 8; sl < ((part & PART_OBST) ? RS : 8); ++sl)
    {
        const double ds = ADS(sl, k);  // 0 for inactive rows
        if (!(ds < 0)) continue;
        const double s0 = AS(sl, k);
        if (!(tau * s0 < -ds * a_p)) continue;   // r >= a_p: not blocking (decided without the division)
        const double r = -tau * s0 / ds;
        if (r < a_p && clip_bin(r) < jt) a_p = r;
    }
    return a_p;
}

// objective contribution of stage k at (x, u, dt): quadratic running cost (k <= N-2; dt-weighted in integral form), terminal
// cost and minimum-time term (k = N-1), via-points attached to the stage.  u is read for k <= N-2 only.
template <int MODEL = MODEL_GENERIC>
HD NOINL inline double stage_objective(const Cfg& c, const WsLayout& L, const double* W, int k, const double* x, const double* u, double dtt)
{
    using T_ = ModelTraits<MODEL>;
    const int N = L.N;
    const double xf[3] = {AIN(IN_XF), AIN(IN_XF + 1), AIN(IN_XF + 2)};
    double obj = 0.0;
    if (k <= N - 2)
    {
        if (T_::quadratic(c))
        {
            const double d[3] = {x[0] - xf[0], x[1] - xf[1], normalize_theta(x[2] - xf[2])};
            double ox = 0.0, ou = 0.0;
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
                for (int j = 0; j < 3; ++j) ox += d[i] * c.Q[i * 3 + j] * d[j];
#pragma unroll
            for (int i = 0; i < 2; ++i)
#pragma unroll
                for (int j = 0; j < 2; ++j) ou += u[i] * c.R[i * 2 + j] * u[j];
            const bool integ = T_::integral(c);
            obj += (integ ? dtt * integral_state_weight(c, N, k) : 1.0) * ox + (integ ? dtt : 1.0) * ou;
        }
    }
    else
    {
        if (T_::trapezoid(c))
        {
            const double d[3] = {x[0] - xf[0], x[1] - xf[1], normalize_theta(x[2] - xf[2])};
            double ox = 0.0;
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
                for (int j = 0; j < 3; ++j) ox += d[i] * c.Q[i * 3 + j] * d[j];
            obj += dtt * integral_state_weight(c, N, k) * ox;
        }
        if (T_::mintime(c)) obj += (double)(N - 1) * dtt;
        if (has_terminal_cost(c))
        {
            const double d[3] = {x[0] - xf[0], x[1] - xf[1], normalize_theta(x[2] - xf[2])};
            double o = 0.0;
#pragma unroll
            for (int i = 0; i < 3; ++i)
#pragma unroll
                for (int j = 0; j < 3; ++j) o += d[i] * c.Qf[i * 3 + j] * d[j];
            obj += o;
        }
    }
    if (has_viapoints(c) && k >= 1 && k <= N - 2)
    {
        const int nvp = (int)AIN(IN_NVP);
        for (int j = 0; j < nvp && j < L.V; ++j)
        {
            if ((int)W[L.oVPST + j] != k) continue;
            const double ex = W[L.oVP + 3 * j] - x[0], ey = W[L.oVP + 3 * j + 1] - x[1];
            obj += c.vp_position_weight * (ex * ex + ey * ey);
            if (c.vp_orientation_weight > 0)
                obj += c.vp_orientation_weight * normalize_theta(W[L.oVP + 3 * j + 2] - x[2]);
        }
    }
    return obj;
}

struct TrialAcc { double obj, inf1, blog; };
// merit pieces of stage k at the trial point z + alpha dz, s + alpha ds.  Linear rows are exact in alpha:
// g(alpha) + s(alpha) = (1 - alpha) r0, so only the dynamics defect, the objective and the obstacle rows are re-evaluated.
template <bool LINES = true, int MODEL = MODEL_GENERIC>
HD inline void ls_stage_trial(const Cfg& c, const WsLayout& L, const double* W, const double* G, double uprev_dt, int k, double alpha, TrialAcc& acc, int part = PART_ALL)
{
    using T_ = ModelTraits<MODEL>;
    const int N = L.N, K = L.K;
    const double dtt = ASC(MPCB200_SC_DT) + (T_::variable_dt(c) ? alpha * ASC(MPCB200_SC_DDT) : 0.0);
    const double x[3] = {AX(0, k) + alpha * ASTEP(0, k), AX(1, k) + alpha * ASTEP(1, k), AX(2, k) + alpha * ASTEP(2, k)};
    const double xf[3] = {AIN(IN_XF), AIN(IN_XF + 1), AIN(IN_XF + 2)};
    double sc[2];
    sincos(x[2], &sc[0], &sc[1]);
    if (!(part & PART_BASE)) {}
    else if (k <= N - 2)
    {
        const double u[2] = {AU(0, k) + alpha * ASTEP(3, k), AU(1, k) + alpha * ASTEP(4, k)};
        double f[3];
        const double xn2 = AX(2, k + 1) + alpha * ASTEP(2, k + 1);
        const int robot = ModelTraits<MODEL>::robot(c);
        if (LINES && is_midpoint(c)) dynamics_value(c, x[2] + 0.5 * normalize_theta(xn2 - x[2]), u[0], u[1], f);
        else if (robot == MPCB200_ROBOT_KIN_BICYCLE) dynamics_value(c, x[2], u[0], u[1], f);
        else
        {
            f[0] = u[0] * sc[1]; f[1] = u[0] * sc[0];
            f[2] = robot == MPCB200_ROBOT_UNICYCLE ? u[1]
                 : (robot == MPCB200_ROBOT_SIMPLE_CAR ? u[0] * tan(u[1]) / c.wheelbase : u[0] * sin(u[1]) / c.wheelbase);
        }
        const double xn[3] = {AX(0, k + 1) + alpha * ASTEP(0, k + 1), AX(1, k + 1) + alpha * ASTEP(1, k + 1),
                              AX(2, k + 1) + alpha * ASTEP(2, k + 1)};
        acc.inf1 += fabs(x[0] + dtt * f[0] - xn[0]) + fabs(x[1] + dtt * f[1] - xn[1]) +
                    fabs(dtt * f[2] - normalize_theta(xn[2] - x[2]));
        acc.obj += stage_objective<MODEL>(c, L, W, k, x, u, dtt);
    }
    else acc.obj += stage_objective<MODEL>(c, L, W, k, x, nullptr, dtt);
    RowProd rp; rp.p = 1.0; rp.n = 0;
    const double oma = 1.0 - alpha;
    for (int sl = (part & PART_BASE) ? 0 : 8; sl < 8; ++sl)
    {
        if (!lin_row_active<MODEL>(c, N, k, sl, uprev_dt)) continue;
        const double s0 = AS(sl, k), ds = ADS(sl, k);
        double sn = s0 + alpha * ds;
        double res = oma * GR0(sl, k);           // g(alpha) + s + alpha ds, exact for linear rows
        if (sn < CLIP_FLOOR * s0) { res += CLIP_FLOOR * s0 - sn; sn = CLIP_FLOOR * s0; }  // clipped slack: the residual keeps the difference
        acc.inf1 += fabs(res);
        rowprod_add(rp, sn, acc.blog);
    }
    if ((part & PART_OBST) && k >= 1 && k <= N - 2)
        for (int j = 0; j < K; ++j)
        {
            const int oi = (int)AOBS(j, k);
            if (oi < 0) continue;
            double ob[5];
            const double dist = footprint_distance_sc<false, false, LINES, MODEL>(c, x[0], x[1], sc[0], sc[1], (int)W[L.oOTYPE + oi],
                                                                    LINES ? obstacle_at(c, W + L.oOBST + oi * MPCB200_OBST_STRIDE, k, dtt, ob) : W + L.oOBST + oi * MPCB200_OBST_STRIDE,
                                                                    nullptr, nullptr);
            double sn = AS(8 + j, k) + alpha * ADS(8 + j, k);
            if (sn < CLIP_FLOOR * AS(8 + j, k)) sn = CLIP_FLOOR * AS(8 + j, k);
            acc.inf1 += fabs(c.min_obstacle_dist - dist + sn);
            rowprod_add(rp, sn, acc.blog);
        }
    if ((part & PART_BASE) && k == N - 1 && T_::ball(c))
    {
        double sn = AS(BALL_SLOT, k) + alpha * ADS(BALL_SLOT, k);
        if (sn < CLIP_FLOOR * AS(BALL_SLOT, k)) sn = CLIP_FLOOR * AS(BALL_SLOT, k);
        acc.inf1 += fabs(ball_row(c, x, xf, nullptr, nullptr) + sn);
        rowprod_add(rp, sn, acc.blog);
    }
    rowprod_flush(rp, acc.blog);
}

// midpoint differences: the sweep solved the transformed, condensed system (eval_stage): nu+ = (I + e_th a') nu~ + e_th (q' dw_k).
// Rewrites STEP(7, k) in place; reads the heading of stage k+1, so it runs for all stages BEFORE any stage is updated.
HD inline void ls_stage_midpoint_fix(const Cfg& c, const WsLayout& L, double* W, int k)
{
    const int N = L.N;
    if (k > N - 2) return;
    const double nu[3] = {ANU(0, k), ANU(1, k), ANU(2, k)};
    const double dt = ASC(MPCB200_SC_DT);
    double f[3], J[9], Hc[6];
    dynamics_derivs(c, AX(2, k) + 0.5 * normalize_theta(AX(2, k + 1) - AX(2, k)), AU(0, k), AU(1, k), nu, f, J, Hc, nullptr);
    double n2 = ASTEP(7, k);
    n2 += 0.5 * dt * (J[0] * ASTEP(5, k) + J[3] * ASTEP(6, k));
    n2 += 0.25 * dt * Hc[0] * ASTEP(2, k) + 0.5 * dt * (Hc[1] * ASTEP(3, k) + Hc[2] * ASTEP(4, k));
    ASTEP(7, k) = n2;
}

// accept the step: z, s, lambda, nu of stage k (reads and writes stage k only: safe to run lane-parallel in place)
template <int MODEL = MODEL_GENERIC>
HD inline void ls_stage_update(const Cfg& c, const WsLayout& L, const double* W, double* G, double uprev_dt, int k, double alpha, double a_dual, int part = PART_ALL)
{
    const int N = L.N, K = L.K;
    const double mu = ASC(MPCB200_SC_MU);
    const double d0 = ASTEP(0, k), d1 = ASTEP(1, k), d2 = ASTEP(2, k);
    double nup[3] = {0.0, 0.0, 0.0};
    if (k <= N - 2) { nup[0] = ASTEP(5, k); nup[1] = ASTEP(6, k); nup[2] = ASTEP(7, k); }
    if (part & PART_BASE) { GX(0, k) = AX(0, k) + alpha * d0; GX(1, k) = AX(1, k) + alpha * d1; GX(2, k) = AX(2, k) + alpha * d2; }
    if ((part & PART_BASE) && k <= N - 2)
    {
        GU(0, k) = AU(0, k) + alpha * ASTEP(3, k);
        GU(1, k) = AU(1, k) + alpha * ASTEP(4, k);
        for (int i = 0; i < 3; ++i) GNU(i, k) = ANU(i, k) + alpha * (nup[i] - ANU(i, k));
    }
    for (int sl = (part & PART_BASE) ? 0 : 8; sl < ((part & PART_OBST) ? 8 + K : 8); ++sl)
    {
        bool act;
        if (sl < 8) act = lin_row_active<MODEL>(c, N, k, sl, uprev_dt) || (sl == BALL_SLOT && k == N - 1 && ModelTraits<MODEL>::ball(c));
        else act = (k >= 1 && k <= N - 2) && AOBS(sl - 8, k) >= 0;
        if (!act) continue;
        const double s0 = AS(sl, k), ds = ADS(sl, k), lam0 = ALAM(sl, k);
        const double rs = 1.0 / s0;
        const double dl = fma(-(lam0 * rs), ds, fma(mu, rs, -lam0));   // multiplier step of the row (as in ls_stage_steps)
        double s = s0 + alpha * ds;
        if (s < CLIP_FLOOR * s0) s = CLIP_FLOOR * s0;
        double lam = lam0 + a_dual * dl;
        const double lo = mu / (KAPPA_SIGMA * s), hi = KAPPA_SIGMA * mu / s;
        if (lam < lo) lam = lo;
        if (lam > hi) lam = hi;
        GS(sl, k) = s;
        GLAM(sl, k) = lam;
    }
}

// ------------------------------------------------------------------------------------------------------
// INITIALISATION / ASSOCIATION
// ------------------------------------------------------------------------------------------------------
// cold initial guess of stage k (SURVEY App. A.6)
HD inline void init_cold_stage(const Cfg& c, const WsLayout& L, double* W, int k, const double* xinit /* [N][3] initial plan samples of this instance, read when IN_HASXINIT */)
{
    const int N = L.N;
    const double* x0 = &AIN(IN_X0);
    const double* xf = &AIN(IN_XF);
    if (k == 0) { for (int i = 0; i < 3; ++i) AX(i, k) = x0[i]; }
    else if (k == N - 1) { for (int i = 0; i < 3; ++i) AX(i, k) = xf[i]; }
    else if (AIN(IN_HASXINIT) != 0.0) { for (int i = 0; i < 3; ++i) AX(i, k) = xinit[3 * k + i]; }
    else
    {
        const double frac = (double)k / (double)(N - 1);
        AX(0, k) = x0[0] + frac * (xf[0] - x0[0]);
        AX(1, k) = x0[1] + frac * (xf[1] - x0[1]);
        AX(2, k) = interpolate_angle(x0[2], xf[2], frac);
    }
    AU(0, k) = 0.0;
    AU(1, k) = 0.0;
}

// Choice of the cold initial guess (solver-side, DESIGN.md "cold initial guess"): among the laterally bumped straight lines
// p_k + A sin(pi k/(N-1)) n_perp, A = BUMP_STEP * m, |m| <= initial_guess_bumps, the one that violates the obstacle clearances
// least is taken; 1e-3 |A| breaks ties.  bump_stage_violation: contribution of stage k for one candidate.
#define BUMP_STEP 0.4
#define BUMP_MARGIN 0.05
HD inline bool bump_enabled(const Cfg& c, const WsLayout& L, const double* W)
{
    return c.initial_guess_bumps > 0 && !c.reference_initial_guess && AIN(IN_HASXINIT) == 0.0 && (int)AIN(IN_NOBST) > 0;
}
HD inline bool bump_normal(const WsLayout& L, const double* W, double* nx, double* ny)
{
    double ax = -(AIN(IN_XF + 1) - AIN(IN_X0 + 1)), ay = AIN(IN_XF) - AIN(IN_X0);
    const double nn = sqrt(ax * ax + ay * ay);
    if (!(nn > 1e-9)) return false;
    *nx = ax / nn; *ny = ay / nn;
    return true;
}
HD inline double bump_offset(int N, int k, double A) { return A * sin(M_PI * (double)k / (double)(N - 1)); }
HD inline double bump_stage_violation(const Cfg& c, const WsLayout& L, const double* W, const ObstSrc& os, int k, double A, double nx, double ny)
{
    const int N = L.N;
    if (k < 1 || k > N - 2) return 0.0;
    const double o = bump_offset(N, k, A);
    const double px = AX(0, k) + o * nx, py = AX(1, k) + o * ny;
    double sn, cs;
    sincos(AX(2, k), &sn, &cs);
    const int nobst = (int)AIN(IN_NOBST);
    double v = 0.0;
    for (int j = 0; j < nobst; ++j)
    {
        double ob[5];
        const double* op = obstacle_at(c, os.p(j), k, c.dt_ref, ob);
        const double d = footprint_distance_sc<false, false, true>(c, px, py, sn, cs, os.type(j), op, nullptr, nullptr);
        const double viol = c.min_obstacle_dist + BUMP_MARGIN - d;
        if (viol > 0.0) v += viol;
    }
    return v;
}
// car-like models cannot turn on the spot: on a bumped line their headings follow the path (central differences of the positions)
HD inline bool bump_align_headings(const Cfg& c, double A) { return A != 0.0 && c.robot_type != MPCB200_ROBOT_UNICYCLE; }
HD inline double bump_heading(const WsLayout& L, const double* W, int k)
{
    const int N = L.N;
    return atan2(AX(1, k + 1) - AX(1, k - 1), AX(0, k + 1) - AX(0, k - 1));
}
// candidate m is better than the best so far only beyond rounding noise: the order of the candidates decides exact ties
HD inline bool bump_better(double score, double best) { return score < best - 1e-9 * (1.0 + best); }
// Amplitude of the bumped line of rank `rank` (multistart: challenger k starts from rank k): repeated selection with bump_better
// over the lines the earlier rounds left, lower m first, so rank 0 is the cold start's choice.  score(A): the line's score,
// 1e-3 |A| + its clearance violation.  Ranks above 0 need 2 initial_guess_bumps + 1 <= 64 (the lines taken are a bit mask).
template <class Score>
HD inline double bump_ranked_amplitude(const Cfg& c, int rank, const Score& score)
{
    const int nb = c.initial_guess_bumps;
    unsigned long long taken = 0ull;
    double best_a = 0.0;
    for (int r = 0; r <= rank; ++r)
    {
        double best = 1e300;
        int best_i = -1;
        for (int m = -nb; m <= nb; ++m)
        {
            if (r > 0 && ((taken >> (m + nb)) & 1ull)) continue;
            const double A = BUMP_STEP * (double)m;
            const double s = score(A);
            if (bump_better(s, best)) { best = s; best_a = A; best_i = m + nb; }
        }
        if (best_i < 0 || r == rank) break;   // (scores that are not finite: the earlier round's line stays)
        taken |= 1ull << best_i;
    }
    return best_a;
}
// serial form (host emulator; the CUDA kernel spreads the stages of a candidate over the lanes of the warp)
HD inline void bump_select_serial(const Cfg& c, const WsLayout& L, double* W, int rank = 0)
{
    const int N = L.N;
    double nx, ny;
    if (!bump_enabled(c, L, W) || !bump_normal(L, W, &nx, &ny)) return;
    const ObstSrc os{W + L.oOBST, W + L.oOTYPE, nullptr};
    const double best_a = bump_ranked_amplitude(c, rank, [&](double A) {
        double score = 1e-3 * fabs(A);
        for (int k = 1; k <= N - 2; ++k) score += bump_stage_violation(c, L, W, os, k, A, nx, ny);
        return score;
    });
    for (int k = 1; k <= N - 2; ++k) { const double o = bump_offset(N, k, best_a); AX(0, k) += o * nx; AX(1, k) += o * ny; }
    if (bump_align_headings(c, best_a))
        for (int k = 1; k <= N - 2; ++k) AX(2, k) = bump_heading(L, W, k);
}

// warm start shift (serial; run by one lane): FullDiscretizationGridBaseSE2::warmStartShifting + findNearestState
HD inline void warm_shift_serial(const Cfg& c, const WsLayout& L, double* W)
{
    const int N = L.N;
    const double* x0 = &AIN(IN_X0);
    const double* xf = &AIN(IN_XF);
    int num_shift = 0;
    {
        double d0 = 0;
        for (int i = 0; i < 3; ++i) { double e = x0[i] - AX(i, 0); d0 += e * e; }
        d0 = sqrt(d0);
        if (fabs(d0) >= 1e-12)
        {
            const int num_interv = N - 1, lookahead = num_interv - 1 < 20 ? num_interv - 1 : 20;
            double cache = d0;
            for (int i = 1; i <= lookahead; ++i)
            {
                double d = 0;
                for (int j = 0; j < 3; ++j) { double e = x0[j] - AX(j, i); d += e * e; }
                d = sqrt(d);
                if (d < cache) { cache = d; num_shift = i; }
                else break;
            }
        }
    }
    if (num_shift > 0 && num_shift <= N - 2)
    {
        for (int i = 0; i < N - num_shift; ++i)
        {
            const int idx = i + num_shift;
            for (int j = 0; j < 3; ++j) AX(j, i) = AX(j, idx);
            if (idx != N - 1)
                for (int j = 0; j < 2; ++j) AU(j, i) = AU(j, idx);
        }
        int idx = N - num_shift;
        for (int i = 0; i < num_shift; ++i, ++idx)
        {
            for (int j = 0; j < 2; ++j) AX(j, idx) = AX(j, idx - 2) + 2.0 * (AX(j, idx - 1) - AX(j, idx - 2));
            AX(2, idx) = interpolate_angle(AX(2, idx - 2), AX(2, idx - 1), 2.0);
            for (int j = 0; j < 2; ++j) AU(j, idx - 1) = AU(j, idx - 2);
        }
    }
    for (int i = 0; i < 3; ++i) AX(i, 0) = x0[i];
    for (int i = 0; i < 3; ++i)
        if (c.xf_fixed[i]) AX(i, N - 1) = xf[i];
}

// Horizon change of a warm trajectory (FullDiscretizationGridBaseSE2::resampleTrajectory,
// full_discretization_grid_base_se2.cpp:440-524; the grid adaptation of the variable grid calls it with n +- 1,
// finite_differences_variable_grid_se2.cpp:99-121).  The horizon time is kept, dt_new = dt (n-1)/(n_new-1); sample
// idx_new sits at t = idx_new dt_new on the old polyline (positions linear, heading by interpolate_angle), its control is
// the one of the old interval it falls into; the first sample and the final state are carried over.
// Xo/Uo: old trajectory, component-major with n columns (column n-1 of Xo = the final-state vertex); Xn/Un: n_new columns.
// A non-positive old dt (never produced by a solve with dt_lb > 0) would divide by zero in the reference; here the new
// samples then collapse onto the old sample 0.  Returns dt_new.
HD inline double resample_serial(int n, const double* Xo, const double* Uo, double dt_old, int n_new, double* Xn, double* Un)
{
    const double dt_new = dt_old * (double)(n - 1) / (double)(n_new - 1);
    for (int i = 0; i < 3; ++i) { Xn[i * n_new] = Xo[i * n]; Xn[i * n_new + n_new - 1] = Xo[i * n + n - 1]; }
    for (int j = 0; j < 2; ++j) { Un[j * n_new] = Uo[j * n]; Un[j * n_new + n_new - 1] = 0.0; }
    int idx_old = 1;
    for (int idx_new = 1; idx_new < n_new - 1; ++idx_new)
    {
        const double t_new = dt_new * (double)idx_new;
        while (t_new > (double)idx_old * dt_old && idx_old < n) ++idx_old;  // old sample that follows t_new
        const double t_old_p1 = (double)idx_old * dt_old;
        const double f = dt_old > 0.0 ? (t_new - (t_old_p1 - dt_old)) / dt_old : 0.0;
        const int p = idx_old - 1 < n - 1 ? idx_old - 1 : n - 1, q = idx_old < n - 1 ? idx_old : n - 1;
        for (int i = 0; i < 2; ++i) Xn[i * n_new + idx_new] = Xo[i * n + p] + f * (Xo[i * n + q] - Xo[i * n + p]);
        Xn[2 * n_new + idx_new] = interpolate_angle(Xo[2 * n + p], Xo[2 * n + q], f);
        const int pu = idx_old - 1 < n - 2 ? idx_old - 1 : n - 2;  // the time series repeats the last control at sample n-1
        for (int j = 0; j < 2; ++j) Un[j * n_new + idx_new] = Uo[j * n + pu];
    }
    return dt_new;
}

// obstacle association of stage k
HD inline void associate_stage(const Cfg& c, const WsLayout& L, double* W, int k)
{
    const int N = L.N, K = L.K;
    for (int j = 0; j < K; ++j) AOBS(j, k) = -1;
    if (k < 1 || k > N - 2 || K <= 0) return;
    const double px = AX(0, k), py = AX(1, k), pth = AX(2, k);
    const double ox = cos(pth), oy = sin(pth);
    double left_min = 1e300, right_min = 1e300;
    int left = -1, right = -1, cnt = 0;
    double dists[16];
    const int nobst = (int)AIN(IN_NOBST);
    const int KK = K < 16 ? K : 16;
    for (int pass = 0; pass < 3; ++pass)
    {
        // pass 0: forced inclusions in obstacle order; pass 1: left; pass 2: right (reference order)
        const int jb = pass == 0 ? 0 : (pass == 1 ? left : right);
        const int je = pass == 0 ? nobst : jb + 1;
        if (pass > 0 && jb < 0) continue;
        for (int j = jb; j < je; ++j)
        {
            double ob[5];
            const double* op0 = W + L.oOBST + j * MPCB200_OBST_STRIDE;
            const double* op = obstacle_at(c, op0, k, ASC(MPCB200_SC_DT), ob);
            double dist;
            if (pass == 0)
            {
                dist = footprint_distance<false, false>(c, px, py, pth, (int)W[L.oOTYPE + j], op, nullptr, nullptr);
                // dynamic obstacles are kept at every stage (stage_inequality_se2.cpp:99-106)
                if (!(dist < c.force_inclusion_dist) && !obstacle_is_dynamic(c, op0))
                {
                    if (dist > c.cutoff_dist) continue;
                    double ccx, ccy;
                    obstacle_centroid((int)W[L.oOTYPE + j], op, &ccx, &ccy);
                    if (ox * ccy - ccx * oy > 0) { if (dist < left_min) { left_min = dist; left = j; } }
                    else { if (dist < right_min) { right_min = dist; right = j; } }
                    continue;
                }
            }
            else dist = pass == 1 ? left_min : right_min;
            // insert into the K-slot list (append; when full replace the farthest if nearer)
            if (cnt < KK) { AOBS(cnt, k) = (signed char)j; dists[cnt] = dist; ++cnt; }
            else
            {
                int far = 0;
                for (int i = 1; i < KK; ++i)
                    if (dists[i] > dists[far]) far = i;
                if (dist < dists[far]) { AOBS(far, k) = (signed char)j; dists[far] = dist; }
            }
        }
    }
}

// initial-guess repair (see DESIGN.md), step 1, stage k: push the pose out of violated obstacle rows, one row after the other.
// Leaves the pose before the repair in STEP(0..1,k) and the largest remaining row value in STEP(2,k) for step 2.
HD inline double stage_max_obstacle_row(const Cfg& c, const WsLayout& L, const double* W, int k, double px, double py)
{
    const int N = L.N, K = L.K;
    double m = -1e300;
    for (int j = 0; j < K; ++j)
    {
        const int oi = (int)AOBS(j, k);
        if (oi < 0) continue;
        double ob[5];
        const double dist = footprint_distance<false, false>(c, px, py, AX(2, k), (int)W[L.oOTYPE + oi],
                                                             obstacle_at(c, W + L.oOBST + oi * MPCB200_OBST_STRIDE, k, ASC(MPCB200_SC_DT), ob), nullptr, nullptr);
        const double g = c.min_obstacle_dist - dist;
        if (g > m) m = g;
    }
    return m;
}
HD inline void project_stage(const Cfg& c, const WsLayout& L, double* W, int k)
{
    const int N = L.N, K = L.K;
    ASTEP(0, k) = AX(0, k); ASTEP(1, k) = AX(1, k); ASTEP(2, k) = -1e300;
    if (k < 1 || k > N - 2) return;
    for (int sweep = 0; sweep < PROJ_SWEEPS; ++sweep)
    {
        int moved = 0;
        for (int j = 0; j < K; ++j)
        {
            const int oi = (int)AOBS(j, k);
            if (oi < 0) continue;
            double gd[3];
            double ob[5];
            const double dist = footprint_distance<true, false>(c, AX(0, k), AX(1, k), AX(2, k), (int)W[L.oOTYPE + oi],
                                                                obstacle_at(c, W + L.oOBST + oi * MPCB200_OBST_STRIDE, k, ASC(MPCB200_SC_DT), ob), gd, nullptr);
            const double g = c.min_obstacle_dist - dist;
            if (g <= -PROJ_MARGIN) continue;
            double gx = -gd[0], gy = -gd[1];
            double n2 = gx * gx + gy * gy;
            if (n2 < 1e-16) { gx = 1.0; gy = 0.0; n2 = 1.0; }
            const double step = (g + PROJ_MARGIN) / n2;
            AX(0, k) -= step * gx;
            AX(1, k) -= step * gy;
            moved = 1;
        }
        if (!moved) break;
    }
    ASTEP(2, k) = stage_max_obstacle_row(c, L, W, k, AX(0, k), AX(1, k));
}
// Step 2 (stages in order): a pose that is still pinched between obstacles after step 1 is moved sideways -- along the
// normal (nx, ny) of the start -> goal line, in LAT_STEP increments up to +-LAT_MAX_STEPS -- to the clear position whose
// lateral offset is closest to the one of the previous stage (keeps the guess on one side of an obstacle).
// lateral_candidate: cost of candidate m for stage k (1e300 = not clear).
#define LAT_STEP 0.1
#define LAT_MAX_STEPS 25
HD inline void lateral_normal(const WsLayout& L, const double* W, double* nx, double* ny)
{
    const int N = L.N;
    double ax = -(ASTEP(1, N - 1) - ASTEP(1, 0)), ay = ASTEP(0, N - 1) - ASTEP(0, 0);
    const double nn = sqrt(ax * ax + ay * ay);
    if (nn < 1e-12) { ax = 0.0; ay = 1.0; } else { ax /= nn; ay /= nn; }
    *nx = ax; *ny = ay;
}
HD inline bool lateral_needed(const WsLayout& L, const double* W, int k) { const int N = L.N; return ASTEP(2, k) > -0.5 * PROJ_MARGIN; }
HD inline double lateral_offset(const WsLayout& L, const double* W, int k, double nx, double ny)
{
    const int N = L.N;
    return (AX(0, k) - ASTEP(0, k)) * nx + (AX(1, k) - ASTEP(1, k)) * ny;
}
HD inline double lateral_candidate(const Cfg& c, const WsLayout& L, const double* W, int k, int m, double o_prev, double nx, double ny)
{
    const int N = L.N;
    const double o = LAT_STEP * (double)m;
    if (stage_max_obstacle_row(c, L, W, k, ASTEP(0, k) + o * nx, ASTEP(1, k) + o * ny) > -PROJ_MARGIN) return 1e300;
    return fabs(o - o_prev) + 1e-3 * fabs(o);
}
HD inline void lateral_apply(const WsLayout& L, double* W, int k, int m, bool found, double nx, double ny)
{
    const int N = L.N;
    const double o = found ? LAT_STEP * (double)m : 0.0;
    AX(0, k) = ASTEP(0, k) + o * nx;
    AX(1, k) = ASTEP(1, k) + o * ny;
}
// serial form (host emulator; the CUDA kernel spreads the candidates of a stage over the lanes of the warp)
HD inline void repair_lateral_serial(const Cfg& c, const WsLayout& L, double* W)
{
    const int N = L.N;
    double nx, ny;
    lateral_normal(L, W, &nx, &ny);
    for (int k = 1; k <= N - 2; ++k)
    {
        if (!lateral_needed(L, W, k)) continue;
        const double o_prev = lateral_offset(L, W, k - 1, nx, ny);
        double best = 1e300;
        int best_m = 0;
        for (int m = -LAT_MAX_STEPS; m <= LAT_MAX_STEPS; ++m)
        {
            const double cost = lateral_candidate(c, L, W, k, m, o_prev, nx, ny);
            if (cost < best) { best = cost; best_m = m; }
        }
        lateral_apply(L, W, k, best_m, best < 1e299, nx, ny);
    }
}

// initial controls of stage k by inverting the dynamics along the state guess, clipped inside the bounds
HD inline void init_controls_stage(const Cfg& c, const WsLayout& L, double* W, int k)
{
    const int N = L.N;
    if (k > N - 2) return;
    const double dt = ASC(MPCB200_SC_DT);
    const double th = AX(2, k);
    const double dx = AX(0, k + 1) - AX(0, k), dy = AX(1, k + 1) - AX(1, k);
    const double dth = normalize_theta(AX(2, k + 1) - th);
    const double v = (dx * cos(th) + dy * sin(th)) / dt, w = dth / dt;
    double u1 = 0.0;
    switch (c.robot_type)
    {
        case MPCB200_ROBOT_UNICYCLE: u1 = w; break;
        case MPCB200_ROBOT_SIMPLE_CAR: u1 = fabs(v) > 1e-3 ? atan(c.wheelbase * w / v) : 0.0; break;
        case MPCB200_ROBOT_SIMPLE_CAR_FRONT:
        {
            double a = fabs(v) > 1e-3 ? c.wheelbase * w / v : 0.0;
            u1 = asin(a > 1 ? 1 : (a < -1 ? -1 : a));
            break;
        }
        default:
        {
            double a = fabs(v) > 1e-3 ? c.length_rear * w / v : 0.0;
            double beta = asin(a > 0.99 ? 0.99 : (a < -0.99 ? -0.99 : a));
            u1 = atan(tan(beta) * (c.length_front + c.length_rear) / c.length_rear);
        }
    }
    double uu[2] = {v, u1};
    for (int i = 0; i < 2; ++i)
    {
        const double l = c.u_lb[i] > -MPCB200_INF ? c.u_lb[i] : -1e6, h = c.u_ub[i] < MPCB200_INF ? c.u_ub[i] : 1e6;
        const double mid = 0.5 * (l + h), half = 0.5 * (h - l) * INIT_SHRINK;
        const double lo = mid - half, hi = mid + half;
        AU(i, k) = uu[i] < lo ? lo : (uu[i] > hi ? hi : uu[i]);
    }
}
// serial clipping of the controls into the control-rate rows (forward from u_prev, backward from u_ref = 0)
HD inline void clip_rates_serial(const Cfg& c, const WsLayout& L, double* W, double uprev_dt)
{
    const int N = L.N;
    const double dt = ASC(MPCB200_SC_DT);
    for (int i = 0; i < 2; ++i)
    {
        const double dl = c.du_lb[i] > -MPCB200_INF ? c.du_lb[i] * INIT_SHRINK : -1e6;
        const double dh = c.du_ub[i] < MPCB200_INF ? c.du_ub[i] * INIT_SHRINK : 1e6;
        double prev = AIN(IN_UPREV + i), T = uprev_dt;
        for (int k = 0; k <= N - 2; ++k)
        {
            if (!(k == 0 && T == 0.0))
            {
                const double a = prev + dl * T, b = prev + dh * T, u = AU(i, k);
                AU(i, k) = u < a ? a : (u > b ? b : u);
            }
            prev = AU(i, k);
            T = dt;
        }
        double next = 0.0;
        for (int k = N - 2; k >= 0; --k)
        {
            const double a = next - dh * dt, b = next - dl * dt, u = AU(i, k);
            AU(i, k) = u < a ? a : (u > b ? b : u);
            next = AU(i, k);
        }
    }
}

// Automatic initial barrier parameter (mu_init <= 0): the barrier has one term per inequality row; it is balanced against the
// objective at the initial guess, mu_0 = |f(x_0)| / m clamped to [MU_AUTO_MIN, MU_AUTO_MAX] (0.1 = Ipopt's mu_init).
// auto_mu_stage: objective value and number of active rows of stage k.
#define MU_AUTO_MIN 0.1
#define MU_AUTO_MAX 1.0
HD inline void auto_mu_stage(const Cfg& c, const WsLayout& L, const double* W, double uprev_dt, int k, double* obj, double* rows)
{
    const int N = L.N, K = L.K;
    const double x[3] = {AX(0, k), AX(1, k), AX(2, k)};
    const double u[2] = {k <= N - 2 ? AU(0, k) : 0.0, k <= N - 2 ? AU(1, k) : 0.0};
    *obj += stage_objective(c, L, W, k, x, u, ASC(MPCB200_SC_DT));
    int m = 0;
    for (int sl = 0; sl < 8; ++sl) m += lin_row_active(c, N, k, sl, uprev_dt) || (sl == BALL_SLOT && k == N - 1 && ball_active(c));
    if (k >= 1 && k <= N - 2)
        for (int j = 0; j < K; ++j) m += AOBS(j, k) >= 0;
    *rows += (double)m;
}
HD inline double auto_mu(double obj, double rows)
{
    double mu = rows > 0.0 ? fabs(obj) / rows : MU_AUTO_MIN;
    if (mu < MU_AUTO_MIN) mu = MU_AUTO_MIN;
    if (mu > MU_AUTO_MAX) mu = MU_AUTO_MAX;
    return mu;
}

// slack / multiplier initialisation of stage k
HD inline void init_duals_stage(const Cfg& c, const WsLayout& L, double* W, double uprev_dt, int k, double mu)
{
    const int N = L.N, K = L.K;
    const double dt = ASC(MPCB200_SC_DT);
    for (int sl = 0; sl < 8 + K; ++sl)
    {
        double s = 1.0, lam = 0.0, g = 0.0;
        bool act;
        if (sl == BALL_SLOT && k == N - 1 && ball_active(c))
        {
            const double xk[3] = {AX(0, k), AX(1, k), AX(2, k)}, xf[3] = {AIN(IN_XF), AIN(IN_XF + 1), AIN(IN_XF + 2)};
            act = true;
            g = ball_row(c, xk, xf, nullptr, nullptr);
        }
        else if (sl < 8)
        {
            act = lin_row_active(c, N, k, sl, uprev_dt);
            if (act)
            {
                const int i = (sl < 4) ? (sl >> 1) : ((sl - 4) >> 1);
                const double uk = (k <= N - 2) ? AU(i, k) : 0.0;
                const double um = (sl >= 4) ? ((k >= 1) ? AU(i, k - 1) : AIN(IN_UPREV + i)) : 0.0;
                double gu, gum, gdt;
                g = lin_row(c, N, k, sl, uk, um, dt, uprev_dt, gu, gum, gdt);
            }
        }
        else
        {
            const int oi = (k >= 1 && k <= N - 2) ? (int)AOBS(sl - 8, k) : -1;
            act = oi >= 0;
            double ob[5];
            if (act)
                g = c.min_obstacle_dist - footprint_distance<false, false>(c, AX(0, k), AX(1, k), AX(2, k), (int)W[L.oOTYPE + oi],
                                                                           obstacle_at(c, W + L.oOBST + oi * MPCB200_OBST_STRIDE, k, dt, ob), nullptr, nullptr);
        }
        if (act) { s = -g > SLACK_PUSH ? -g : SLACK_PUSH; lam = mu / s; }
        AS(sl, k) = s;
        ALAM(sl, k) = lam;
    }
    for (int i = 0; i < 3; ++i) ANU(i, k) = 0.0;
}
