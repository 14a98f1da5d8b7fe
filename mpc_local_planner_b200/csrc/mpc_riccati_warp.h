// mpc_riccati_warp.h -- warp-cooperative factorisation + solve of the bordered block-tridiagonal KKT system of ONE OCP
// instance (the replacement of MUMPS' general sparse LDL^T inside Ipopt, R/src/controller.cpp:380-421), executed by ONE
// WARP on data in shared memory: the lanes own the ENTRIES of the stage matrix, the horizon is walked stage by stage with
// ONE warp barrier per stage.
//
// Unknowns: dw_k = (dx_k, du_k), nu+_k, d(dt);  dx_{k+1} = A_k dx_k + B_k du_k + d_k d(dt) + e_k,  dx_0 = 0,
// dx_{N-1,j} = 0 for fixed terminal components.  Stage variables r = (x (3), p (2) = du_{k-1}, th^ (NC)), v = du_k (2);
// parameters th^ = (1, d(dt), pi_0, pi_1, pi_2) (pi = multipliers of fixed terminal components); NC = 1 when dt is fixed and
// the terminal state free (EXT = false), else 5.
//
// The recursion keeps, per stage, the symmetric matrix BEFORE the controls are eliminated,
//     MM_k = HH_k + FF_k' V_{k+1} FF_k      over (x, p, v, th^),      V_{k+1} = MM_{k+1} / v  (Schur complement of the v block),
// instead of the value function V_k itself: substituting the Schur complement,
//     MM_k[i][j] = HH_k[i][j] + phi_i' MM_{k+1} phi_j - (phi_i' MM_{k+1,.v}) inv(MM_{k+1,vv}) (MM_{k+1,v.} phi_j),
// where phi_i = column i of FF_k has at most 4 non-zeros (3 coefficients on x+ and a unit on its "own" successor variable).
// One lane computes one entry (i, j): the first term does not depend on the 2x2 pivot, so its multiply-adds overlap the
// reciprocal of the determinant, and a stage costs one shared-memory round trip (read MM_{k+1}, write MM_k, __syncwarp)
// with ~10 dependent FP64 operations -- against ~600 dependent operations per stage when one thread owns an instance.
// Inertia: MM_{k,vv} must be positive definite at every stage (=> the reduced Hessian is, => correct KKT inertia); at the
// root the pi block must be negative definite and the reduced d(dt) pivot positive (riccati_root).
//
// Everything the forward substitution needs is a function of MM_k alone, so after the root the gains of ALL stages are
// formed in parallel (lane = stage), one lane runs the 5-dimensional affine recursion, and the multipliers
//     nu+_k = MM_{k+1,xx} dx_{k+1} + MM_{k+1,xv} du_{k+1} + MM_{k+1,x th^} th^
// are again formed for all stages in parallel.
//
// The functions below are "phases" in the bulk-synchronous sense: rw_*(..., lane) is the work of one lane between two
// warp barriers, reading only what earlier phases wrote.  kkt_warp_solve() (CUDA) strings them together with __syncwarp();
// the CPU warp emulator (tests/emu, test infrastructure) replays the same phase functions lane after lane.
#pragma once
#include "mpc_core.h"

#define RSTR 43        // words per stage record in memory: MPCB200_KKT_WORDS + one zero word (odd stride: lane-per-stage accesses are bank-conflict free)
#define REC_ZERO 42    // index of the zero word of a record
#define GAIN_WORDS 12  // per stage: KGx (2x3), KGp (2x2), kappa (2)

// Regularisation schedule of one IPM iteration (Ipopt's algorithm IC, at most MAX_INERTIA_TRIES attempts per iteration):
// attempt 0 uses kkt_first_delta(), attempt t+1 uses kkt_escalate(delta_t).
HD inline double kkt_first_delta(double dlast) { return (dlast > 0.0 && dlast / 3.0 >= DELTA_FLOOR) ? dlast / 3.0 : 0.0; }
HD inline double kkt_escalate(double delta, double dlast)
{
    if (delta == 0.0) return (dlast == 0.0) ? 1e-4 : fmax(dlast / 3.0, 1e-20);
    return delta * (dlast == 0.0 ? 100.0 : 8.0);
}

// root: y_0 = 0 -> stationarity of 1/2 th' TH th over the active parameters: pi block (negative definite) first,
// then d(dt) (must leave a positive pivot).  Returns 0 on wrong inertia.
HD inline int riccati_root(const Cfg& c, const double TH[5][5], double* th)
{
    th[0] = 1.0; th[1] = th[2] = th[3] = th[4] = 0.0;
    int act[3], na = 0;
    for (int j = 0; j < 3; ++j)
        if (c.xf_fixed[j]) act[na++] = 2 + j;
    double Lm[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    for (int i = 0; i < na; ++i)
        for (int j = 0; j <= i; ++j)
        {
            double s = -0.5 * (TH[act[i]][act[j]] + TH[act[j]][act[i]]);
            for (int l = 0; l < j; ++l) s -= Lm[i][l] * Lm[j][l];
            if (i == j) { if (!(s > 0.0)) return 0; Lm[i][i] = sqrt(s); }
            else Lm[i][j] = s / Lm[j][j];
        }
    double sol0[3] = {0, 0, 0}, sol1[3] = {0, 0, 0};
    for (int pass = 0; pass < 2; ++pass)
    {
        double* sl = pass ? sol1 : sol0;
        double y[3] = {0, 0, 0};
        for (int i = 0; i < na; ++i)
        {
            double t = TH[act[i]][pass];
            for (int l = 0; l < i; ++l) t -= Lm[i][l] * y[l];
            y[i] = t / Lm[i][i];
        }
        for (int i = na - 1; i >= 0; --i)
        {
            double t = y[i];
            for (int l = i + 1; l < na; ++l) t -= Lm[l][i] * sl[l];
            sl[i] = t / Lm[i][i];
        }
    }
    double ddt = 0.0;
    if (c.variable_dt)
    {
        double htt = TH[1][1], gt = TH[1][0];
        for (int i = 0; i < na; ++i) { htt += TH[1][act[i]] * sol1[i]; gt += TH[1][act[i]] * sol0[i]; }
        if (!(htt > 0.0)) return 0;
        ddt = -gt / htt;
    }
    th[1] = ddt;
    for (int i = 0; i < na; ++i) th[act[i]] = sol0[i] + sol1[i] * ddt;
    return 1;
}

// ---- packed storage of the symmetric stage matrix MM over the variables x0 x1 x2 | p0 p1 | v0 v1 | th^0 .. th^(NC-1) ----
// Only the structurally non-zero entries are kept (p couples with nothing but its own v through the control-rate rows):
//   xx (6)  xv (6)  pv (2)  vv (3)  x th^ (3 NC)  v th^ (2 NC)  th^ th^ (NC (NC+1) / 2);   index NE = a constant zero word.
template <bool EXT>
struct RW
{
    static constexpr int NC = EXT ? 5 : 1;
    static constexpr int NE = 17 + 5 * NC + NC * (NC + 1) / 2;          // 23 / 57 entries
    static constexpr int EPL = (NE + 31) / 32;                          // entries per lane: 1 / 2
    static constexpr int ZERO = NE;
    static constexpr int MSTR = EXT ? NE + 1 : NE + 5;                  // words per stage (even): entries, zero word, (NC = 1: 4 gain words)
    static constexpr int oXV = 6, oPV = 12, oVV = 14, oXT = 17, oVT = 17 + 3 * NC, oTT = 17 + 5 * NC;
    // The 12 gain words of a stage overwrite entries that are dead once the root is known (pv, vv, v th^, th^ th^: the
    // multipliers only need xx, xv, x th^); NC = 1 has 8 of those and 4 extra words behind the zero word.
    HD static constexpr int gslot(int i) { return i < 5 ? oPV + i : (EXT ? oVT - 5 + i : (i < 8 ? 15 + i : 16 + i)); }
    // variable numbering: x 0..2, p 3..4, v 5..6, th^ 7..
    HD static int idx(int i, int j)
    {
        if (i < 0 || j < 0) return ZERO;
        if (i > j) { const int t = i; i = j; j = t; }
        if (j < 3) return i * 3 - (i * (i - 1)) / 2 + (j - i);
        if (i < 3) return j < 5 ? ZERO : (j < 7 ? oXV + i * 2 + (j - 5) : oXT + i * NC + (j - 7));
        if (i < 5) return (j >= 5 && j < 7 && j - 5 == i - 3) ? oPV + (i - 3) : ZERO;
        if (i < 7) return j < 7 ? oVV + (i - 5) + (j - 5) : oVT + (i - 5) * NC + (j - 7);
        const int a = i - 7, b = j - 7;
        return oTT + a * NC - (a * (a - 1)) / 2 + (b - a);
    }
    // inverse map: entry e -> (i, j), i <= j
    HD static void pair(int e, int* i, int* j)
    {
        if (e < oXV) { int a = 0, r = e; while (r >= 3 - a) { r -= 3 - a; ++a; } *i = a; *j = a + r; return; }
        if (e < oPV) { *i = (e - oXV) >> 1; *j = 5 + ((e - oXV) & 1); return; }
        if (e < oVV) { *i = 3 + (e - oPV); *j = 5 + (e - oPV); return; }
        if (e < oXT) { const int r = e - oVV; *i = r == 2 ? 6 : 5; *j = r == 0 ? 5 : 6; return; }
        if (e < oVT) { *i = (e - oXT) / NC; *j = 7 + (e - oXT) % NC; return; }
        if (e < oTT) { *i = 5 + (e - oVT) / NC; *j = 7 + (e - oVT) % NC; return; }
        int a = 0, r = e - oTT;
        while (r >= NC - a) { r -= NC - a; ++a; }
        *i = 7 + a; *j = 7 + a + r;
    }
};

// ---- the stage recursion in two bulk-synchronous phases, every operand at a FIXED shared-memory address ----
//   cur  : the latest stage matrix MM_{k+1} (packed entries + a zero word), rewritten every stage
//   tt   : the column products T[c][r] = (MM_{k+1} phi_c)[r] over the variables x0 x1 x2 v0 v1 th^.. (dense (5+NC)^2 table)
// Phase A (one lane per needed (c, r)): T[c][r] = sum_b MM'[r][b] f_c[b] + MM'[r][own_c]; every lane also inverts the pivot
// MM'_vv (inertia test).  Phase B (one lane per entry (i, j)):
//   MM_k[i][j] = HH_k[i][j] + sum_a f_i[a] T[j][x_a] + T[j][own_i] - w_i' inv(MM'_vv) w_j,   w_c = (T[c][v0], T[c][v1]),
// written to `cur` (nobody reads it in phase B) and to the archive of stage k (gains and multipliers are formed from it later).
template <bool EXT>
struct RW2
{
    typedef RW<EXT> T;
    static constexpr int NC = T::NC;
    static constexpr int NV = 5 + NC;                 // variables with a column / row in the table: x0 x1 x2 v0 v1 th^..
    static constexpr int TTW = NV * NV;
    static constexpr int TZERO = TTW;                 // a zero word behind the table: the slot of "no operand"
    static constexpr int CURW = (T::NE + 2) & ~1;     // entries + zero word
    static constexpr int SCRATCH = CURW + ((TTW + 2) & ~1);
    // needed (column, row) pairs: all rows of the columns with coefficients (x2, v0, v1, th^0, th^1); of the unit columns
    // only what the upper triangle of MM_k reads
    static constexpr int NTA = EXT ? 84 : 31;
    static constexpr int SLA = (NTA + 31) / 32;       // phase-A slots per lane
    HD static int var_of(int t) { return t < 3 ? t : t + 2; }   // table index -> variable number (x 0..2, v 5..6, th^ 7..)
    HD static int tab_of(int var) { return var < 3 ? var : var - 2; }
    HD static bool need(int c, int r)
    {
        if (c == 2 || c == 3 || c == 4 || c == 5 || (EXT && c == 6)) return true;
        if (c == 0) return r == 0 || r == 3 || r == 4;
        if (c == 1) return r == 0 || r == 1 || r == 3 || r == 4;
        return r <= c;   // th^c, c >= 2: rows x, v, th^0..th^c
    }
    // the t-th needed pair
    HD static bool pair(int t, int* c, int* r)
    {
        int n = 0;
        for (int cc = 0; cc < NV; ++cc)
            for (int rr = 0; rr < NV; ++rr)
                if (need(cc, rr)) { if (n == t) { *c = cc; *r = rr; return true; } ++n; }
        return false;
    }
};

struct RwColProg   // phase A: one (column, row) product
{
    int active;
    int out;               // slot in tt
    int fo[3]; double fc[3];   // coefficients of the column on x+: constant + record word (BYTE offset into the record)
    int m[3], mo;          // BYTE offsets into cur of MM'[r][x_b], MM'[r][own_c]
};
struct RwEntProg   // phase B: one entry
{
    int active;
    int e;                 // packed index of the entry
    int hoff, hdiag;       // record word of HH[i][j] (REC_ZERO: none); delta is added on the x and v diagonal
    int fo[3]; double fc[3];   // coefficients of column i
    int t[3], to;          // BYTE offsets into tt of T[j][x_a], T[j][own_i] (TZERO: no operand)
    int wi[2], wj[2];      // ... of T[i][v_m], T[j][v_m]
};

template <bool EXT>
HD inline void rw_column(int var, int dt_free, int* fo, double* fc, int* own)
{
    // column `var` of FF_k: x+ = x + a x_2 + B v + e th^0 + d th^1,  p+ = v,  th^ = th^
    // (no runtime index into fo / fc: the lane programs live in the warp's lane state, which must stay in registers)
    for (int a = 0; a < 3; ++a) { fo[a] = REC_ZERO; fc[a] = (var < 2 && a == var) ? 1.0 : 0.0; }
    *own = -1;
    if (var < 2) {}
    else if (var == 2) { for (int a = 0; a < 3; ++a) fo[a] = MPCB200_K_A + a; fc[2] = 1.0; }
    else if (var < 5) {}
    else if (var < 7) { for (int a = 0; a < 3; ++a) fo[a] = MPCB200_K_B + 2 * a + (var - 5); *own = 3 + (var - 5); }
    else if (var == 7) { for (int a = 0; a < 3; ++a) fo[a] = MPCB200_K_E + a; *own = 7; }
    else if (var == 8) { if (dt_free) for (int a = 0; a < 3; ++a) fo[a] = MPCB200_K_D + a; *own = 8; }
    else *own = var;
}

template <bool EXT>
HD inline void rw_colprog_setup(int t, int dt_free, RwColProg& cp)
{
    typedef RW<EXT> T;
    typedef RW2<EXT> T2;
    int c = 0, r = 0;
    cp.active = t < T2::NTA && T2::pair(t, &c, &r);
    if (!cp.active) { c = 0; r = 0; }
    const int cv = T2::var_of(c), rv = T2::var_of(r);
    int own;
    rw_column<EXT>(cv, dt_free, cp.fo, cp.fc, &own);
    for (int b = 0; b < 3; ++b) { cp.m[b] = 8 * T::idx(rv, b); cp.fo[b] *= 8; }
    cp.mo = 8 * T::idx(rv, own);
    cp.out = c * T2::NV + r;
}

template <bool EXT>
HD inline void rw_entprog_setup(int e, int dt_free, RwEntProg& en)
{
    typedef RW<EXT> T;
    typedef RW2<EXT> T2;
    en.active = e < T::NE;
    en.e = en.active ? e : T::ZERO;
    int i = 3, j = 4;   // (p0, p1): structurally zero
    if (en.active) T::pair(e, &i, &j);
    int own_i;
    rw_column<EXT>(i, dt_free, en.fo, en.fc, &own_i);
    const bool jp = j >= 3 && j < 5, ip = i >= 3 && i < 5;   // p columns are zero
    const int tj = jp ? -1 : T2::tab_of(j), ti = ip ? -1 : T2::tab_of(i);
    for (int a = 0; a < 3; ++a) en.t[a] = 8 * (tj < 0 ? T2::TZERO : tj * T2::NV + a);
    en.to = 8 * ((tj < 0 || own_i < 7) ? T2::TZERO : tj * T2::NV + T2::tab_of(own_i));   // own = p contributes nothing (MM'[p][.] phi_j = 0)
    for (int m = 0; m < 2; ++m) { en.wi[m] = 8 * (ti < 0 ? T2::TZERO : ti * T2::NV + 3 + m); en.wj[m] = 8 * (tj < 0 ? T2::TZERO : tj * T2::NV + 3 + m); }
    // HH entry of the record (5x5 block of w = (x, u) in hidx order, gradient, dt border, cross block)
    en.hoff = REC_ZERO; en.hdiag = 0;
    const int wi_ = i < 3 ? i : (i >= 5 && i < 7 ? i - 2 : -1), wj_ = j < 3 ? j : (j >= 5 && j < 7 ? j - 2 : -1);
    if (wi_ >= 0 && wj_ >= 0) { en.hoff = MPCB200_K_H + hidx(wi_, wj_); en.hdiag = wi_ == wj_; }
    else if (ip && j == i + 2) en.hoff = MPCB200_K_C + (i - 3);
    else if (wi_ >= 0 && j == 7) en.hoff = MPCB200_K_G + wi_;
    else if (wi_ >= 0 && j == 8 && dt_free) en.hoff = MPCB200_K_HB + wi_;
    if (!en.active) en.hoff = REC_ZERO;
    en.hoff *= 8;
    for (int a = 0; a < 3; ++a) en.fo[a] *= 8;
}

// ---- phase T: the terminal value function as a stage matrix with an identity v block (MM_{N-1}) ----
// rec = record of stage N-1 (terminal cost block in the x entries).  Returns the value of entry e.
template <bool EXT>
HD inline double rw_terminal(const Cfg& c, const double* rec, int e, double delta, double htt, double gt)
{
    typedef RW<EXT> T;
    int i, j;
    T::pair(e, &i, &j);
    double v = 0.0;
    if (j < 3)
    {
        if (!(c.xf_fixed[i] || c.xf_fixed[j])) v = rec[MPCB200_K_H + hidx(i, j)] + (i == j ? delta : 0.0);
    }
    else if (i >= 5 && j < 7) v = (i == j) ? 1.0 : 0.0;
    else if (i < 3 && j >= 7)
    {
        const int cc = j - 7;
        if (cc == 0) v = c.xf_fixed[i] ? 0.0 : rec[MPCB200_K_G + i];
        else if (cc == 1) v = (c.variable_dt && (has_trapezoid(c) || is_midpoint(c)) && !c.xf_fixed[i]) ? rec[MPCB200_K_HB + i] : 0.0;
        else v = (c.xf_fixed[i] && cc == 2 + i) ? 1.0 : 0.0;
    }
    else if (i >= 7)
    {
        const int a = i - 7, b = j - 7;
        if (a == 0 && b == 1) v = gt;
        else if (a == 1 && b == 1) v = htt + delta;
    }
    return v;
}

// pivot of a stage: inverse determinant of MM_vv with the inertia test (same value in every lane)
HD inline bool rw_pivot(double la, double lb, double ld, double* idet)
{
    const double det = la * ld - lb * lb;
    *idet = 1.0 / det;
    return la > 0.0 && ld > 0.0 && det > 1e-14 * la * ld;
}

struct RwColCoef { double f[3]; };
struct RwEntCoef { double f[3], h; };
// word at a BYTE offset (the programs hold premultiplied offsets: base + offset is the whole address computation)
HD inline double rw_at(const double* base, int byte_off) { return *reinterpret_cast<const double*>(reinterpret_cast<const char*>(base) + byte_off); }
// The coefficients of a stage are fetched one stage ahead as RAW record words (the loads are issued at the end of the previous
// stage and nothing consumes them there: a warp issues in order, a consumer right behind the load would expose its latency);
// rw_coef_* adds the constants when the stage begins.
HD inline void rw_fetch_col(const double* rec, const RwColProg& cp, RwColCoef& raw)
{
#pragma unroll
    for (int a = 0; a < 3; ++a) raw.f[a] = rw_at(rec, cp.fo[a]);
}
HD inline void rw_fetch_ent(const double* rec, const RwEntProg& en, RwEntCoef& raw)
{
#pragma unroll
    for (int a = 0; a < 3; ++a) raw.f[a] = rw_at(rec, en.fo[a]);
    raw.h = rw_at(rec, en.hoff);
}
HD inline void rw_coef_col(const RwColProg& cp, const RwColCoef& raw, RwColCoef& co)
{
#pragma unroll
    for (int a = 0; a < 3; ++a) co.f[a] = cp.fc[a] + raw.f[a];
}
HD inline void rw_coef_ent(const RwEntProg& en, const RwEntCoef& raw, double delta, RwEntCoef& co)
{
#pragma unroll
    for (int a = 0; a < 3; ++a) co.f[a] = en.fc[a] + raw.f[a];
    co.h = raw.h + (en.hdiag ? delta : 0.0);
}
// phase A: one column product
HD inline double rw_colprod(const double* cur, const RwColProg& cp, const RwColCoef& co)
{
    return (rw_at(cur, cp.m[0]) * co.f[0] + rw_at(cur, cp.m[1]) * co.f[1]) + (rw_at(cur, cp.m[2]) * co.f[2] + rw_at(cur, cp.mo));
}
// phase B: one entry from the table.  la, lb, ld = MM'_vv and idet = 1 / det(MM'_vv) (formed in phase A, while `cur` still
// holds MM').
template <bool EXT>
HD inline double rw_entry(const double* tt, const RwEntProg& en, const RwEntCoef& co, double la, double lb, double ld, double idet)
{
#define RWT(s_) rw_at(tt, s_)
    const double t0 = RWT(en.t[0]), t1 = RWT(en.t[1]), t2 = RWT(en.t[2]), to = RWT(en.to);
    const double wi0 = RWT(en.wi[0]), wi1 = RWT(en.wi[1]), wj0 = RWT(en.wj[0]), wj1 = RWT(en.wj[1]);
#undef RWT
    const double s1 = (co.f[0] * t0 + co.f[1] * t1) + (co.f[2] * t2 + to);
    const double q = wi0 * (ld * wj0 - lb * wj1) + wi1 * (la * wj1 - lb * wj0);
    return (co.h + s1) - q * idet;
}

// ---- phase R: Schur complement of the root stage on th^ and its stationary point.  Returns 0 on wrong inertia. ----
template <bool EXT>
HD inline int rw_root(const Cfg& c, const double* m0, double* th)
{
    typedef RW<EXT> T;
    constexpr int NC = T::NC;
    th[0] = 1.0; th[1] = th[2] = th[3] = th[4] = 0.0;
    const double la = m0[T::oVV], lb = m0[T::oVV + 1], ld = m0[T::oVV + 2];
    double idet;
    if (!rw_pivot(la, lb, ld, &idet)) return 0;
    if (!EXT) return 1;
    double TH[5][5];
    for (int a = 0; a < 5; ++a)
        for (int b = 0; b < 5; ++b)
        {
            if (a >= NC || b >= NC) { TH[a][b] = 0.0; continue; }
            const double wa0 = m0[T::oVT + a], wa1 = m0[T::oVT + NC + a], wb0 = m0[T::oVT + b], wb1 = m0[T::oVT + NC + b];
            const double q = wa0 * (ld * wb0 - lb * wb1) + wa1 * (la * wb1 - lb * wb0);
            TH[a][b] = m0[T::idx(7 + a, 7 + b)] - q * idet;
        }
    return riccati_root(c, TH, th);
}

// ---- phase G (lane = stage): feedback gains of stage k from MM_k, written over its dead entries (gslot) ----
//      g0..5 = KGx (2x3), g6..9 = KGp (2x2), g10..11 = kappa = Lambda MM_{v th^} th^
template <bool EXT>
HD inline void rw_gains(double* mm, const double* th)
{
    typedef RW<EXT> T;
    constexpr int NC = T::NC;
    const double la = mm[T::oVV], lb = mm[T::oVV + 1], ld = mm[T::oVV + 2];
    const double idet = 1.0 / (la * ld - lb * lb);
    const double L00 = ld * idet, L01 = -lb * idet, L11 = la * idet;
    double g[GAIN_WORDS];
#pragma unroll
    for (int a = 0; a < 3; ++a)
    {
        const double m0 = mm[T::oXV + 2 * a], m1 = mm[T::oXV + 2 * a + 1];
        g[a] = L00 * m0 + L01 * m1;
        g[3 + a] = L01 * m0 + L11 * m1;
    }
    const double c0 = mm[T::oPV], c1 = mm[T::oPV + 1];
    g[6] = L00 * c0; g[7] = L01 * c1; g[8] = L01 * c0; g[9] = L11 * c1;
    double n0 = 0.0, n1 = 0.0;
#pragma unroll
    for (int cc = 0; cc < NC; ++cc) { n0 += mm[T::oVT + cc] * th[cc]; n1 += mm[T::oVT + NC + cc] * th[cc]; }
    g[10] = L00 * n0 + L01 * n1;
    g[11] = L01 * n0 + L11 * n1;
#pragma unroll
    for (int i = 0; i < GAIN_WORDS; ++i) mm[T::gslot(i)] = g[i];   // every input has been read
}

// ---- phase F: forward substitution, parallel in time -------------------------------------------------------------
// Stage k maps y_k = (x_k, p_k) to y_{k+1} = PHI_k y_k + phi_k with v_k = -(Kx x + Kp p + kappa),
//   x+ = (A - B Kx) x - B Kp p + (e^ - B kappa),   p+ = v_k.
// Each lane composes the maps of its CH consecutive stages, an inclusive warp scan (5 levels of 5x5 products, operands
// exchanged by shuffles) composes the chunks, and each lane replays its stages from the state at the start of its chunk.
struct RwMap { double M[5][5], b[5]; };   // y -> M y + b

template <bool EXT>
HD inline void rw_stage_map(const double* rec, const double* mm, int dt_free, double ddt, RwMap& q)
{
    typedef RW<EXT> T;
    double g[GAIN_WORDS];
#pragma unroll
    for (int i = 0; i < GAIN_WORDS; ++i) g[i] = mm[T::gslot(i)];
    double e[3] = {rec[MPCB200_K_E], rec[MPCB200_K_E + 1], rec[MPCB200_K_E + 2]};
    if (EXT && dt_free) { e[0] += rec[MPCB200_K_D] * ddt; e[1] += rec[MPCB200_K_D + 1] * ddt; e[2] += rec[MPCB200_K_D + 2] * ddt; }
#pragma unroll
    for (int i = 0; i < 3; ++i)
    {
        const double b0 = rec[MPCB200_K_B + 2 * i], b1 = rec[MPCB200_K_B + 2 * i + 1];
#pragma unroll
        for (int j = 0; j < 3; ++j) q.M[i][j] = (i == j ? 1.0 : 0.0) - (b0 * g[j] + b1 * g[3 + j]);
        q.M[i][2] += rec[MPCB200_K_A + i];
        q.M[i][3] = -(b0 * g[6] + b1 * g[8]);
        q.M[i][4] = -(b0 * g[7] + b1 * g[9]);
        q.b[i] = e[i] - (b0 * g[10] + b1 * g[11]);
    }
#pragma unroll
    for (int j = 0; j < 3; ++j) { q.M[3][j] = -g[j]; q.M[4][j] = -g[3 + j]; }
    q.M[3][3] = -g[6]; q.M[3][4] = -g[7]; q.M[4][3] = -g[8]; q.M[4][4] = -g[9];
    q.b[3] = -g[10]; q.b[4] = -g[11];
}
// Composition a o b (first b, then a):  M = Ma Mb,  b = Ma bb + ba.  Two in-place forms, so that no third map is live: the
// scan operands stay in registers.  Both form every entry by the same expression.
HD inline double rw_dot5(const double* r, double c0, double c1, double c2, double c3, double c4)
{
    return ((r[0] * c0 + r[1] * c1) + (r[2] * c2 + r[3] * c3)) + r[4] * c4;
}
// a <- a o b, row by row (row i of the result needs row i of a only)
HD inline void rw_compose(RwMap& a, const RwMap& b)
{
#pragma unroll
    for (int i = 0; i < 5; ++i)
    {
        double r[5];
#pragma unroll
        for (int j = 0; j < 5; ++j) r[j] = rw_dot5(a.M[i], b.M[0][j], b.M[1][j], b.M[2][j], b.M[3][j], b.M[4][j]);
        a.b[i] = rw_dot5(a.M[i], b.b[0], b.b[1], b.b[2], b.b[3], b.b[4]) + a.b[i];
#pragma unroll
        for (int j = 0; j < 5; ++j) a.M[i][j] = r[j];
    }
}
// b <- a o b, column by column (column j of the result needs column j of b only)
HD inline void rw_compose_onto(const RwMap& a, RwMap& b)
{
    double r[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) r[i] = rw_dot5(a.M[i], b.b[0], b.b[1], b.b[2], b.b[3], b.b[4]) + a.b[i];
#pragma unroll
    for (int i = 0; i < 5; ++i) b.b[i] = r[i];
#pragma unroll
    for (int j = 0; j < 5; ++j)
    {
#pragma unroll
        for (int i = 0; i < 5; ++i) r[i] = rw_dot5(a.M[i], b.M[0][j], b.M[1][j], b.M[2][j], b.M[3][j], b.M[4][j]);
#pragma unroll
        for (int i = 0; i < 5; ++i) b.M[i][j] = r[i];
    }
}
// replay the stages [k0, k1) from the state y at stage k0: dw_k -> stp; returns the state at k1 in y
template <bool EXT>
HD inline void rw_replay(const double* recs, const double* mms, int N, int k0, int k1, int dt_free, double ddt, double* y, double* stp)
{
    typedef RW<EXT> T;
    double x0 = y[0], x1 = y[1], x2 = y[2], p0 = y[3], p1 = y[4];
    for (int k = k0; k < k1; ++k)
    {
        const double* m = mms + (size_t)k * T::MSTR;
        const double* r = recs + (size_t)k * RSTR;
#define RWG(i_) m[T::gslot(i_)]
        const double v0 = -(((RWG(0) * x0 + RWG(1) * x1) + (RWG(2) * x2 + RWG(6) * p0)) + (RWG(7) * p1 + RWG(10)));
        const double v1 = -(((RWG(3) * x0 + RWG(4) * x1) + (RWG(5) * x2 + RWG(8) * p0)) + (RWG(9) * p1 + RWG(11)));
#undef RWG
        stp[k] = x0; stp[N + k] = x1; stp[2 * N + k] = x2; stp[3 * N + k] = v0; stp[4 * N + k] = v1;
        double e0 = r[MPCB200_K_E], e1 = r[MPCB200_K_E + 1], e2 = r[MPCB200_K_E + 2];
        if (EXT && dt_free) { e0 += r[MPCB200_K_D] * ddt; e1 += r[MPCB200_K_D + 1] * ddt; e2 += r[MPCB200_K_D + 2] * ddt; }
        const double n0 = (x0 + r[MPCB200_K_A] * x2 + e0) + (r[MPCB200_K_B] * v0 + r[MPCB200_K_B + 1] * v1);
        const double n1 = (x1 + r[MPCB200_K_A + 1] * x2 + e1) + (r[MPCB200_K_B + 2] * v0 + r[MPCB200_K_B + 3] * v1);
        const double n2 = (x2 + r[MPCB200_K_A + 2] * x2 + e2) + (r[MPCB200_K_B + 4] * v0 + r[MPCB200_K_B + 5] * v1);
        x0 = n0; x1 = n1; x2 = n2; p0 = v0; p1 = v1;
    }
    y[0] = x0; y[1] = x1; y[2] = x2; y[3] = p0; y[4] = p1;
}

// ---- phase O (lane = stage): nu+_k (k <= N-2) from MM_{k+1} and the step of stage k+1; zeros at k = N-1 ----
template <bool EXT>
HD inline void rw_multiplier(const double* mms, int N, int k, const double* th, double* stp)
{
    typedef RW<EXT> T;
    constexpr int NC = T::NC;
    if (k >= N - 1) { stp[5 * N + k] = 0.0; stp[6 * N + k] = 0.0; stp[7 * N + k] = 0.0; return; }
    const double* mn = mms + (size_t)(k + 1) * T::MSTR;
    const double xn[3] = {stp[k + 1], stp[N + k + 1], stp[2 * N + k + 1]}, vn[2] = {stp[3 * N + k + 1], stp[4 * N + k + 1]};
#pragma unroll
    for (int i = 0; i < 3; ++i)
    {
        double s = mn[T::idx(i, 0)] * xn[0] + mn[T::idx(i, 1)] * xn[1] + mn[T::idx(i, 2)] * xn[2];
        s += mn[T::oXV + 2 * i] * vn[0] + mn[T::oXV + 2 * i + 1] * vn[1];
#pragma unroll
        for (int cc = 0; cc < NC; ++cc) s += mn[T::oXT + i * NC + cc] * th[cc];
        stp[(5 + i) * N + k] = s;
    }
}

// words of scratch for a horizon of N grid points: the archive of stage matrices (+ gains), the current stage matrix, the table
template <bool EXT>
HD inline int rw_scratch_words(int N) { return N * RW<EXT>::MSTR + RW2<EXT>::SCRATCH; }

// ---- the driver -------------------------------------------------------------------------------------------------
// Exec abstracts the warp: ex.each(f) runs f(lane, lane_state) for every lane (CUDA: the calling lane; emulator: a loop over
// 32 lane states), ex.sync() is the warp barrier, ex.all(p) the warp vote, ex.shift_up(d) delivers every lane's `out` map to
// lane + d as `in`.
template <bool EXT>
struct RwLane
{
    RwColProg cp[RW2<EXT>::SLA];
    RwColCoef cc[RW2<EXT>::SLA];   // raw record words of the coming stage
    RwEntProg en[RW<EXT>::EPL];
    RwEntCoef ec[RW<EXT>::EPL];
    double la, lb, ld;         // pivot block of the stage matrix in `cur`
    double idet;               // ... the reciprocal of its determinant
    bool pok;                  // ... and its inertia test
    RwMap out, in;             // scan operands
    double y[5];
};

template <bool EXT, class Exec>
HD inline void kkt_warp_setup(Exec& ex, int dt_free)
{
    ex.each([&](int lane, RwLane<EXT>& ls) {
#pragma unroll
        for (int s = 0; s < RW2<EXT>::SLA; ++s) rw_colprog_setup<EXT>(lane + 32 * s, dt_free, ls.cp[s]);
#pragma unroll
        for (int s = 0; s < RW<EXT>::EPL; ++s) rw_entprog_setup<EXT>(lane + 32 * s, dt_free, ls.en[s]);
    });
}

// One attempt with regularisation delta on the records recs ([k][RSTR]) with scratch mms (rw_scratch_words); the step goes to
// stp ([8][N]).  Returns 1 if the system was solved, 0 on wrong inertia.
template <bool EXT, class Exec>
HD inline int kkt_warp_attempt(Exec& ex, const Cfg& c, int N, double* recs, double* mms, double* stp, double delta, double htt, double gt, double* ddt_out)
{
    typedef RW<EXT> T;
    typedef RW2<EXT> T2;
    double* cur = mms + (size_t)N * T::MSTR;
    double* tt = cur + T2::CURW;
    // terminal stage matrix into `cur` and the archive; zero words; table cleared (slots nobody writes are read with zero coefficients)
    ex.each([&](int lane, RwLane<EXT>& ls) {
        for (int k = lane; k < N; k += 32) recs[(size_t)k * RSTR + REC_ZERO] = 0.0;
        for (int i = lane; i <= T2::TZERO; i += 32) tt[i] = 0.0;
        if (lane == 0) cur[T::ZERO] = 0.0;
#pragma unroll
        for (int s = 0; s < T::EPL; ++s)
            if (ls.en[s].active)
            {
                const double v = rw_terminal<EXT>(c, recs + (size_t)(N - 1) * RSTR, ls.en[s].e, delta, htt, gt);
                cur[ls.en[s].e] = v;
                mms[(size_t)(N - 1) * T::MSTR + ls.en[s].e] = v;
            }
    });
    ex.sync();
    ex.each([&](int lane, RwLane<EXT>& ls) {
#pragma unroll
        for (int s = 0; s < T2::SLA; ++s) rw_fetch_col(recs + (size_t)(N - 2) * RSTR, ls.cp[s], ls.cc[s]);
#pragma unroll
        for (int s = 0; s < T::EPL; ++s) rw_fetch_ent(recs + (size_t)(N - 2) * RSTR, ls.en[s], ls.ec[s]);
    });
    bool ok = true;
    for (int k = N - 2; k >= 0; --k)
    {
        // ---- phase A: column products of MM_{k+1}; the pivot block is read while `cur` still holds MM_{k+1}, and the
        //      reciprocal of its determinant is formed here: its latency overlaps the column products and the barrier
        //      instead of delaying the last operation of every entry in phase B ----
        ex.each([&](int lane, RwLane<EXT>& ls) {
            ls.la = cur[T::oVV]; ls.lb = cur[T::oVV + 1]; ls.ld = cur[T::oVV + 2];
            ls.pok = rw_pivot(ls.la, ls.lb, ls.ld, &ls.idet);
#pragma unroll
            for (int s = 0; s < T2::SLA; ++s)
            {
                RwColCoef co;
                rw_coef_col(ls.cp[s], ls.cc[s], co);
                const double v = rw_colprod(cur, ls.cp[s], co);
                if (ls.cp[s].active) tt[ls.cp[s].out] = v;
            }
        });
        ex.sync();
        // ---- phase B: entries of MM_k; raw coefficients of the next stage ----
        double* mk = mms + (size_t)k * T::MSTR;
        const double* rnext = recs + (size_t)(k > 0 ? k - 1 : 0) * RSTR;
        ex.each([&](int lane, RwLane<EXT>& ls) {
            ok = ok && ls.pok;
#pragma unroll
            for (int s = 0; s < T::EPL; ++s)
            {
                RwEntCoef co;
                rw_coef_ent(ls.en[s], ls.ec[s], delta, co);
                const double v = rw_entry<EXT>(tt, ls.en[s], co, ls.la, ls.lb, ls.ld, ls.idet);
                if (ls.en[s].active) { cur[ls.en[s].e] = v; mk[ls.en[s].e] = v; }
            }
#pragma unroll
            for (int s = 0; s < T::EPL; ++s) rw_fetch_ent(rnext, ls.en[s], ls.ec[s]);
#pragma unroll
            for (int s = 0; s < T2::SLA; ++s) rw_fetch_col(rnext, ls.cp[s], ls.cc[s]);
        });
        if (!ex.all(ok)) break;   // every lane evaluates the same pivot; the vote keeps the loop uniform for the compiler
                                  // (a failed stage wrote garbage nobody will read)
        ex.sync();
    }
    ex.sync();
    if (!ex.all(ok)) return 0;
    double th[5];
    if (!rw_root<EXT>(c, mms, th)) return 0;   // uniform (reads the archive of stage 0)
    *ddt_out = th[1];
    // ---- gains of all stages (lane = stage) ----
    ex.each([&](int lane, RwLane<EXT>& ls) {
        for (int k = lane; k <= N - 2; k += 32) rw_gains<EXT>(mms + (size_t)k * T::MSTR, th);
    });
    ex.sync();
    // ---- forward substitution: chunk maps, warp scan, replay ----
    const int S = N - 1, CH = (S + 31) / 32;
    const int dt_free = c.variable_dt;
    ex.each([&](int lane, RwLane<EXT>& ls) {
        const int k0 = lane * CH < S ? lane * CH : S, k1 = (lane + 1) * CH < S ? (lane + 1) * CH : S;
#pragma unroll
        for (int i = 0; i < 5; ++i)
        {
#pragma unroll
            for (int j = 0; j < 5; ++j) ls.out.M[i][j] = i == j ? 1.0 : 0.0;
            ls.out.b[i] = 0.0;
        }
        for (int k = k0; k < k1; ++k)
        {
            RwMap q;
            rw_stage_map<EXT>(recs + (size_t)k * RSTR, mms + (size_t)k * T::MSTR, dt_free, th[1], q);
            rw_compose_onto(q, ls.out);
        }
    });
    for (int d = 1; d < 32; d <<= 1)
    {
        ex.shift_up(d);
        ex.each([&](int lane, RwLane<EXT>& ls) {
            if (lane >= d) rw_compose(ls.out, ls.in);
        });
    }
    ex.shift_up(1);   // state at the start of a chunk = offset of the prefix map of the lanes before it (y_0 = 0)
    ex.each([&](int lane, RwLane<EXT>& ls) {
        const int k0 = lane * CH < S ? lane * CH : S, k1 = (lane + 1) * CH < S ? (lane + 1) * CH : S;
#pragma unroll
        for (int i = 0; i < 5; ++i) ls.y[i] = lane > 0 ? ls.in.b[i] : 0.0;
        rw_replay<EXT>(recs, mms, N, k0, k1, dt_free, th[1], ls.y, stp);
        if (k1 == S && k0 < S)   // the owner of the last stage writes the final state
        {
            // a fixed terminal component is not a variable: its step is exactly zero, so x_{N-1,i} stays at the goal (the
            // composed stage maps would leave a rounding residue that every accepted step adds to it)
            stp[N - 1] = (EXT && c.xf_fixed[0]) ? 0.0 : ls.y[0];
            stp[N + N - 1] = (EXT && c.xf_fixed[1]) ? 0.0 : ls.y[1];
            stp[2 * N + N - 1] = (EXT && c.xf_fixed[2]) ? 0.0 : ls.y[2];
            stp[3 * N + N - 1] = 0.0; stp[4 * N + N - 1] = 0.0;
        }
    });
    ex.sync();
    ex.each([&](int lane, RwLane<EXT>& ls) {
        for (int k = lane; k < N; k += 32) rw_multiplier<EXT>(mms, N, k, th, stp);
    });
    ex.sync();
    return 1;
}

// Factorisation + solve with the inertia-correcting regularisation schedule (at most MAX_INERTIA_TRIES attempts; the
// escalation resumes in the next IPM iteration).  *delta_out: the regularisation used, or the next one after a failure.
template <bool EXT, class Exec>
HD inline int kkt_warp_solve(Exec& ex, const Cfg& c, int N, double* recs, double* mms, double* stp, double htt, double gt, double dlast,
                             double* ddt_out, double* delta_out, int* nreg_out)
{
    double delta = kkt_first_delta(dlast), ddt = 0.0;
    int ok = 0, nreg = 0;
    for (int tries = 0; tries < MAX_INERTIA_TRIES && !ok && delta <= MAX_DELTA; ++tries)
    {
        ok = kkt_warp_attempt<EXT>(ex, c, N, recs, mms, stp, delta, htt, gt, &ddt);
        if (!ok) { ++nreg; delta = kkt_escalate(delta, dlast); }
    }
    *ddt_out = ddt; *delta_out = delta; *nreg_out = nreg;
    return ok;
}

// bookkeeping of the KKT phase in the instance scalars (sc = SCAL words of the instance): Newton step accepted, null
// step (factorisation budget of this iteration spent), or give up
HD inline void kkt_store_outcome(double* sc, int ok, double ddt, double delta, int nreg)
{
    sc[MPCB200_SC_NREG] += (double)nreg;
    if (!ok && delta <= MAX_DELTA)
    {
        sc[MPCB200_SC_DELTA_LAST] = 3.0 * delta;   // the next iteration resumes at this delta (DELTA_LAST / 3)
        sc[MPCB200_SC_DEFER] = 1.0;
        return;
    }
    if (!ok) { sc[MPCB200_SC_STATUS] = (double)MPCB200_STATUS_NUMERICAL_ERROR; return; }
    sc[MPCB200_SC_DEFER] = 0.0;
    sc[MPCB200_SC_DDT] = ddt;
    sc[MPCB200_SC_DELTA] = delta;
    sc[MPCB200_SC_DELTA_LAST] = delta;
}
