// mpc_device.cuh -- device side of the solver: the phases of one interior-point solve as functions of ONE CTA that owns ONE
// instance whose resident prefix (mpc_layout.h) sits in shared memory.  The fused solve kernel (mpcb200.cu) calls them in a
// loop until the instance terminates; the per-phase kernels (kernel-level API: parity tests, roofline measurement) stage the
// prefix, call one of them, and write it back.  CUDA only (the CPU warp emulator of tests/emu replays the same stage bodies
// of mpc_stage.h / mpc_riccati_warp.h with its own serial orchestration).
#pragma once
#include <cuda_runtime.h>

#include "mpc_core.h"
#include "mpc_riccati_warp.h"
#include "mpc_stage.h"
#include "mpc_layout.h"

#define FULLMASK 0xffffffffu
#define MAX_GROUP_WARPS 4   // warps of the CTA that owns one instance (lane per stage; longer horizons wrap)

// ---- warp reductions (fp64 via two 32-bit shuffles each) ------------------------------------------------
__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(FULLMASK, v, o);
    return v;
}
__device__ __forceinline__ double warp_max(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(FULLMASK, v, o));
    return v;
}
__device__ __forceinline__ double warp_min(double v)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmin(v, __shfl_xor_sync(FULLMASK, v, o));
    return v;
}

// ---- bulk-async (TMA) copies and mbarriers ----------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(bar), "r"(parity) : "memory");
    __syncwarp();   // lanes may leave the spin in different turns: converge before any warp collective that follows
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* dst, uint32_t src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_commit_wait()
{
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}
// generic-proxy writes (ordinary stores) before async-proxy reads of the same shared / global memory
__device__ __forceinline__ void fence_async() { asm volatile("fence.proxy.async;" ::: "memory"); }

// ---- the warp as an executor of the KKT driver (mpc_riccati_warp.h) ----
template <bool EXT>
struct CudaWarp
{
    RwLane<EXT> ls;
    int lane;
    template <class F> __device__ __forceinline__ void each(const F& f) { f(lane, ls); }
    __device__ __forceinline__ void sync() { __syncwarp(); }
    __device__ __forceinline__ bool all(bool p) const { return __all_sync(FULLMASK, p) != 0; }
    __device__ __forceinline__ void shift_up(int d)
    {
#pragma unroll
        for (int i = 0; i < 5; ++i)
        {
#pragma unroll
            for (int j = 0; j < 5; ++j) ls.in.M[i][j] = __shfl_up_sync(FULLMASK, ls.out.M[i][j], d);
            ls.in.b[i] = __shfl_up_sync(FULLMASK, ls.out.b[i], d);
        }
    }
};

struct InputPtrs
{
    const double* x0; const double* xf; const double* u_prev;      // [B][3],[B][3],[B][2]
    const int* obst_count; const int* obst_type; const double* obst_params; int obst_max;
    const int* vp_count; const double* vp_poses; int vp_max;
    const double* x_init;                                          // [B][N][3] or null
    const unsigned char* reinit;                                   // [B] or null
};
struct OutputPtrs { double* u_seq; double* x_seq; double* dt; int* status; double* kkt; int* iters; double* u_packed; };

// ---- multistart (mpcb200_step_batch_multistart): candidate k of robot b is instance k * B + b ----
// A challenger (k >= 1) starts cold from the bumped line of rank k: it has none without obstacles or without a start -> goal normal
__device__ __forceinline__ bool challenger_has_guess(const Cfg& c, const WsLayout& L, const double* W)
{
    double nx, ny;
    return bump_enabled(c, L, W) && bump_normal(L, W, &nx, &ny);
}
// The winner among the K candidates of one robot from their SCAL words (status < 0, an unfinished solve, counts as MAX_ITER):
// the converged challenger with the least objective (lower k on ties) replaces a converged incumbent only when
// obj(c*) < obj(0) - (1 - hysteresis) |obj(0)|, and always one that did not converge; with none converged, the incumbent stays
// when it ran out of iterations or time, else the challenger stopped that way with the least infeasibility wins.  Else: 0.
// scal(k, w): word w of candidate k's SCAL words.
template <class Scal>
__device__ __forceinline__ int multistart_winner(const Scal& scal, int K, double hysteresis)
{
    auto st = [&](int k) { const double s = scal(k, MPCB200_SC_STATUS); return s < 0 ? MPCB200_STATUS_MAX_ITER : (int)s; };
    auto stopped = [&](int k) { return st(k) == MPCB200_STATUS_MAX_ITER || st(k) == MPCB200_STATUS_MAX_TIME; };
    int cs = -1;
    for (int k = 1; k < K; ++k)
        if (st(k) == MPCB200_STATUS_CONVERGED && (cs < 0 || scal(k, MPCB200_SC_OBJ) < scal(cs, MPCB200_SC_OBJ))) cs = k;
    if (st(0) == MPCB200_STATUS_CONVERGED)
    {
        if (cs < 0) return 0;
        const double o0 = scal(0, MPCB200_SC_OBJ);
        return scal(cs, MPCB200_SC_OBJ) < o0 - (1.0 - hysteresis) * fabs(o0) ? cs : 0;
    }
    if (cs >= 0) return cs;
    if (stopped(0)) return 0;
    int best = 0;
    for (int k = 1; k < K; ++k)
        if (stopped(k) && (best == 0 || scal(k, MPCB200_SC_INF) < scal(best, MPCB200_SC_INF))) best = k;
    return best;
}

// ---- scatter the compact input arrays into an instance block (inputs of instance `src`), one warp.  Returns false
//      (warp-uniform) when an input that will be used is not finite: the instance is reported as INVALID_INPUT.  Kernels
//      compiled without the line-obstacle paths (LINES = false) also reject a line obstacle: they would take its distance as
//      that of a point.  The blocking entry points never launch them on lines (they scan the types on the host); the
//      device-memory entry points choose the variant from what the caller declares, so an undeclared line ends here. ----
template <bool LINES>
__device__ __forceinline__ bool scatter_one(const WsLayout& L, double* W, const InputPtrs& in, int64_t src, int lane, double* xinit_dst)
{
    const int N = L.N;
    bool ok = true;
    if (lane < 3)
    {
        const double a = in.x0[src * 3 + lane], b = in.xf[src * 3 + lane];
        AIN(IN_X0 + lane) = a; AIN(IN_XF + lane) = b;
        ok = isfinite(a) && isfinite(b);
    }
    if (lane < 2) { const double u = in.u_prev ? in.u_prev[src * 2 + lane] : 0.0; AIN(IN_UPREV + lane) = u; ok = ok && isfinite(u); }
    int nob = 0, nvp = 0;
    const bool long_list = in.obst_max > L.M;   // the list stays in global memory, the association copies what it selects
    if (in.obst_count) nob = min(max(in.obst_count[src], 0), in.obst_max);
    if (in.vp_count) nvp = min(max(in.vp_count[src], 0), min(in.vp_max, L.V));
    if (lane == 0)
    {
        AIN(IN_NOBST) = (double)nob; AIN(IN_NVP) = (double)nvp;
        AIN(IN_NRES) = long_list ? 0.0 : (double)nob;
        AIN(IN_HASXINIT) = in.x_init ? 1.0 : 0.0;
        AIN(IN_REINIT) = (in.reinit && in.reinit[src]) ? 1.0 : 0.0;
    }
    for (int i = lane; i < nob * MPCB200_OBST_STRIDE; i += 32)
    {
        const double v = in.obst_params[src * in.obst_max * MPCB200_OBST_STRIDE + i];
        if (!long_list) W[L.oOBST + i] = v;
        ok = ok && isfinite(v);
    }
    // (unrolled as the compiler unrolls the check with line obstacles: the cheaper check without them was unrolled 16 times,
    // which moved all code behind it in the instruction-fetch-bound solve kernels and cost 0.5 % of a cold solve)
#pragma unroll 4
    for (int i = lane; i < nob; i += 32)
    {
        const int t = in.obst_type[src * in.obst_max + i];
        if (!long_list) W[L.oOTYPE + i] = (double)t;
        ok = ok && t >= MPCB200_OBST_POINT && t <= (LINES ? MPCB200_OBST_LINE : MPCB200_OBST_CIRCLE);
    }
    for (int i = lane; i < nvp * 3; i += 32) { const double v = in.vp_poses[src * in.vp_max * 3 + i]; W[L.oVP + i] = v; ok = ok && isfinite(v); }
    if (in.x_init && xinit_dst)
        for (int i = lane; i < 3 * N; i += 32) xinit_dst[i] = in.x_init[src * 3 * N + i];
    return __all_sync(FULLMASK, ok) != 0;
}

// the full obstacle list of instance `src`: the image (short lists) or the caller's arrays
__device__ __forceinline__ ObstSrc obstacle_source(const WsLayout& L, const double* W, const InputPtrs& in, int64_t src)
{
    if (in.obst_count && in.obst_max > L.M)
        return ObstSrc{in.obst_params + src * in.obst_max * MPCB200_OBST_STRIDE, nullptr, in.obst_type + src * in.obst_max};
    return ObstSrc{W + L.oOBST, W + L.oOTYPE, nullptr};
}

// results of one instance into the compact output arrays (threads t, t + nt, ... of the owner)
__device__ __forceinline__ void gather_one(const WsLayout& L, const double* W, const OutputPtrs& o, int64_t dst, int t, int nt)
{
    const int N = L.N;
    const double st = ASC(MPCB200_SC_STATUS);
    const bool bad = st == (double)MPCB200_STATUS_INVALID_INPUT;   // outputs of an invalid instance are zeros
    for (int k = t; k < N; k += nt)
    {
        const int kk = k <= N - 2 ? k : N - 2;
        const double u0 = bad ? 0.0 : AU(0, kk), u1 = bad ? 0.0 : AU(1, kk);
        if (o.u_seq) { o.u_seq[(dst * N + k) * 2 + 0] = u0; o.u_seq[(dst * N + k) * 2 + 1] = u1; }
        if (o.x_seq)
        {
            o.x_seq[(dst * N + k) * 3 + 0] = bad ? 0.0 : AX(0, k);
            o.x_seq[(dst * N + k) * 3 + 1] = bad ? 0.0 : AX(1, k);
            o.x_seq[(dst * N + k) * 3 + 2] = bad ? 0.0 : normalize_theta(AX(2, k));
        }
        if (k <= N - 2 && o.u_packed) { o.u_packed[(dst * (N - 1) + k) * 2 + 0] = u0; o.u_packed[(dst * (N - 1) + k) * 2 + 1] = u1; }
    }
    if (t == 0)
    {
        if (o.dt) o.dt[dst] = ASC(MPCB200_SC_DT);
        if (o.status) o.status[dst] = st < 0 ? MPCB200_STATUS_MAX_ITER : (int)st;
        if (o.kkt) o.kkt[dst] = ASC(MPCB200_SC_ERR0);
        if (o.iters) o.iters[dst] = (int)ASC(MPCB200_SC_ITER);
    }
}

// ---- PHASE_INIT (one warp): cold initial guess or warm-start shift ----------------------------------------
// xinit: the instance's initial plan samples [N][3] (read when IN_HASXINIT); rank: the bumped line a cold start takes (0: the best,
// k: a multistart challenger's, bump_ranked_amplitude)
__device__ __forceinline__ void dev_init(const Cfg& c, const WsLayout& L, double* W, const ObstSrc& os, const double* xinit, int force_cold, int lane,
                                         int rank)
{
    const int N = L.N;
    __syncwarp();   // (see dev_kkt)
    const bool cold = force_cold || ASC(MPCB200_SC_COLD) != 0.0 || AIN(IN_REINIT) != 0.0;
    __syncwarp();
    if (cold)
    {
        for (int k = lane; k < N; k += 32) init_cold_stage(c, L, W, k, xinit);
        __syncwarp();
        double nx, ny;
        if (bump_enabled(c, L, W) && bump_normal(L, W, &nx, &ny))
        {
            // choice of the cold initial guess: candidates one after the other, their stages spread over the lanes
            const double best_a = bump_ranked_amplitude(c, rank, [&](double A) {
                double v = 0.0;
                for (int k = lane; k < N; k += 32) v += bump_stage_violation(c, L, W, os, k, A, nx, ny);
                return 1e-3 * fabs(A) + warp_sum(v);
            });
            for (int k = lane; k < N; k += 32)
                if (k >= 1 && k <= N - 2) { const double o = bump_offset(N, k, best_a); AX(0, k) += o * nx; AX(1, k) += o * ny; }
            __syncwarp();
            if (bump_align_headings(c, best_a))   // headings from the positions of the neighbours (positions are final)
                for (int k = lane; k < N; k += 32)
                    if (k >= 1 && k <= N - 2) AX(2, k) = bump_heading(L, W, k);
        }
        __syncwarp();
        if (lane == 0) { ASC(MPCB200_SC_DT) = c.dt_ref; ASC(MPCB200_SC_COLD) = 2.0; /* 2: cold init done, repair pending */ }
    }
    else
    {
        if (lane == 0)
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
    __syncwarp();
}

// ---- PHASE_ASSOCIATE (one warp): obstacle / via-point association, initial-guess repair, dual initialisation ----
// Association over a LONG obstacle list (StageInequalitySE2::update, stage_inequality_se2.cpp:73-147, for the hundreds of point
// obstacles of a raw costmap): the stages one after the other, the lanes over the obstacles of the list in global memory.  Per
// stage the same selection as associate_stage -- forced inclusions in list order, then the nearest left and the nearest right
// obstacle within the cut-off, into the K row slots with the same replacement rule -- and only the selected obstacles are copied
// into the resident list (each once: `gidx` = list index of every resident slot; a full list drops and counts).
__device__ __forceinline__ void kslot_insert(int* idx, double* dst, int& cnt, int KK, int j, double dist)
{
    if (cnt < KK) { idx[cnt] = j; dst[cnt] = dist; ++cnt; return; }
    int far = 0;
    for (int i = 1; i < KK; ++i)
        if (dst[i] > dst[far]) far = i;
    if (dist < dst[far]) { idx[far] = j; dst[far] = dist; }
}
__device__ __forceinline__ void dev_associate_list(const Cfg& c, const WsLayout& L, double* W, const ObstSrc& os, double* gidx /* [L.M] scratch */, int lane)
{
    const int N = L.N, K = L.K, KK = K < 16 ? K : 16;
    const int nobst = (int)AIN(IN_NOBST);
    int nres = 0, dropped = 0;
    for (int i = lane; i < L.M; i += 32) gidx[i] = -1.0;
    for (int k = lane; k < N; k += 32)
        for (int j = 0; j < K; ++j) AOBS(j, k) = -1;
    __syncwarp();
    for (int k = 1; k <= N - 2 && K > 0; ++k)
    {
        const double px = AX(0, k), py = AX(1, k), pth = AX(2, k);
        const double ox = cos(pth), oy = sin(pth);
        int sidx[16]; double sdst[16]; int cnt = 0;
        double lmin = 1e300, rmin = 1e300; int left = -1, right = -1;
        for (int base = 0; base < nobst; base += 32)
        {
            const int j = base + lane;
            double dist = 1e300; bool forced = false;
            if (j < nobst)
            {
                double ob[5];
                const double* op0 = os.p(j);
                const int ot = os.type(j);
                const double* op = obstacle_at(c, op0, k, ASC(MPCB200_SC_DT), ob);
                dist = footprint_distance<false, false>(c, px, py, pth, ot, op, nullptr, nullptr);
                forced = dist < c.force_inclusion_dist || obstacle_is_dynamic(c, op0);
                if (!forced && !(dist > c.cutoff_dist))
                {
                    double ccx, ccy;
                    obstacle_centroid(ot, op, &ccx, &ccy);
                    if (ox * ccy - ccx * oy > 0) { if (dist < lmin) { lmin = dist; left = j; } }
                    else { if (dist < rmin) { rmin = dist; right = j; } }
                }
            }
            unsigned m = __ballot_sync(FULLMASK, forced);
            while (m)   // forced inclusions in list order (uniform: every lane keeps the same slot list)
            {
                const int src = __ffs(m) - 1;
                m &= m - 1;
                kslot_insert(sidx, sdst, cnt, KK, base + src, __shfl_sync(FULLMASK, dist, src));
            }
        }
        // nearest left / right over the lanes: smallest distance, the earliest obstacle on ties (the reference's strict <)
        for (int o = 16; o > 0; o >>= 1)
        {
            const double ol = __shfl_xor_sync(FULLMASK, lmin, o); const int il = __shfl_xor_sync(FULLMASK, left, o);
            if (il >= 0 && (left < 0 || ol < lmin || (ol == lmin && il < left))) { lmin = ol; left = il; }
            const double orr = __shfl_xor_sync(FULLMASK, rmin, o); const int ir = __shfl_xor_sync(FULLMASK, right, o);
            if (ir >= 0 && (right < 0 || orr < rmin || (orr == rmin && ir < right))) { rmin = orr; right = ir; }
        }
        if (left >= 0) kslot_insert(sidx, sdst, cnt, KK, left, lmin);
        if (right >= 0) kslot_insert(sidx, sdst, cnt, KK, right, rmin);
        // resident slots of the selected obstacles
        for (int s_ = 0; s_ < cnt; ++s_)
        {
            const int g = sidx[s_];
            int slot = -1;
            for (int b0 = 0; b0 < L.M; b0 += 32)
            {
                const unsigned hit = __ballot_sync(FULLMASK, b0 + lane < nres && (int)gidx[b0 + lane] == g);
                if (hit) { slot = b0 + __ffs(hit) - 1; break; }
            }
            if (slot < 0)
            {
                if (nres < L.M)
                {
                    slot = nres++;
                    if (lane < MPCB200_OBST_STRIDE) W[L.oOBST + slot * MPCB200_OBST_STRIDE + lane] = os.p(g)[lane];
                    if (lane == 0) { W[L.oOTYPE + slot] = (double)os.type(g); gidx[slot] = (double)g; }
                    __syncwarp();
                }
                else ++dropped;
            }
            if (lane == 0 && slot >= 0) AOBS(s_, k) = (signed char)slot;
        }
    }
    __syncwarp();
    if (lane == 0) { AIN(IN_NRES) = (double)nres; ASC(MPCB200_SC_OBST_DROPPED) = (double)dropped; }
    __syncwarp();
}

// os / gidx: the instance's full obstacle list and, for a list in global memory (long_list), scratch for the list index of every
// resident slot
__device__ __forceinline__ void dev_associate(const Cfg& c, const WsLayout& L, double* W, double uprev_dt, int first_outer, int lane,
                                              const ObstSrc& os, bool long_list, double* gidx)
{
    const int N = L.N;
    const bool cold_pending = first_outer && ASC(MPCB200_SC_COLD) == 2.0;
    const bool repair = cold_pending && !c.reference_initial_guess;   // solver-side preprocessing of a cold guess (off: the reference's guess)
    __syncwarp();
    if (long_list) dev_associate_list(c, L, W, os, gidx, lane);
    else
        for (int k = lane; k < N; k += 32) associate_stage(c, L, W, k);
    // via-points: MinTimeViaPointsCost::update with findClosestPose (argmin over the grid, first minimum wins)
    if (has_viapoints(c))
    {
        const int nvp = (int)AIN(IN_NVP);
        int start_idx = 0;
        for (int j = 0; j < nvp && j < L.V; ++j)
        {
            const double vx = W[L.oVP + 3 * j], vy = W[L.oVP + 3 * j + 1];
            double best = 1e300; int bidx = -1;
            for (int i = start_idx + lane; i < N - 1; i += 32)
            {
                const double dx = AX(0, i) - vx, dy = AX(1, i) - vy;
                const double d = sqrt(dx * dx + dy * dy);
                if (d < best) { best = d; bidx = i; }
            }
            // warp argmin with smallest index on ties
            for (int o = 16; o > 0; o >>= 1)
            {
                const double ob = __shfl_xor_sync(FULLMASK, best, o);
                const int oi = __shfl_xor_sync(FULLMASK, bidx, o);
                if (ob < best || (ob == best && oi >= 0 && (bidx < 0 || oi < bidx))) { best = ob; bidx = oi; }
            }
            {
                const double dx = AX(0, N - 1) - vx, dy = AX(1, N - 1) - vy;
                const double d = sqrt(dx * dx + dy * dy);
                if (d < best) { best = d; bidx = N - 1; }
            }
            int idx = bidx;
            if (c.vp_ordered) start_idx = idx + 2;
            if (idx > N - 2) idx = N - 2;
            if (idx < 1) idx = c.vp_ordered ? 1 : -1;
            if (lane == 0) W[L.oVPST + j] = (double)idx;
        }
        for (int j = nvp + lane; j < L.V; j += 32) W[L.oVPST + j] = -1.0;
    }
    __syncwarp();
    if (repair)
    {
        for (int k = lane; k < N; k += 32) project_stage(c, L, W, k);
        __syncwarp();
        {
            // step 2 of the repair: stages in order, the lateral candidates of a pinched stage spread over the lanes
            double nx, ny;
            lateral_normal(L, W, &nx, &ny);
            for (int k = 1; k <= N - 2; ++k)
            {
                if (!lateral_needed(L, W, k)) continue;  // warp-uniform
                const double o_prev = lateral_offset(L, W, k - 1, nx, ny);
                double best = 1e300;
                int best_m = 0;
                for (int m = -LAT_MAX_STEPS + lane; m <= LAT_MAX_STEPS; m += 32)
                {
                    const double cost = lateral_candidate(c, L, W, k, m, o_prev, nx, ny);
                    if (cost < best) { best = cost; best_m = m; }
                }
                for (int o = 16; o > 0; o >>= 1)
                {
                    const double oc = __shfl_xor_sync(FULLMASK, best, o);
                    const int om = __shfl_xor_sync(FULLMASK, best_m, o);
                    if (oc < best || (oc == best && om < best_m)) { best = oc; best_m = om; }
                }
                __syncwarp();
                if (lane == 0) lateral_apply(L, W, k, best_m, best < 1e299, nx, ny);
                __syncwarp();
            }
        }
        // controls by inverting the dynamics along the guess: every stage reads its successor's pose, nothing writes poses here
        for (int k = lane; k < N; k += 32) init_controls_stage(c, L, W, k);
        __syncwarp();
        if (lane == 0) clip_rates_serial(c, L, W, uprev_dt);
        __syncwarp();
    }
    double mu = c.mu_init;
    if (!(mu > 0.0))
    {
        double obj = 0.0, rows = 0.0;
        for (int k = lane; k < N; k += 32) auto_mu_stage(c, L, W, uprev_dt, k, &obj, &rows);
        mu = auto_mu(warp_sum(obj), warp_sum(rows));
    }
    for (int k = lane; k < N; k += 32) init_duals_stage(c, L, W, uprev_dt, k, mu);
    __syncwarp();
    if (lane == 0)
    {
        ASC(MPCB200_SC_MU) = mu; ASC(MPCB200_SC_RHO) = 1.0; ASC(MPCB200_SC_DELTA) = 0.0; ASC(MPCB200_SC_DELTA_LAST) = 0.0;
        ASC(MPCB200_SC_ITER) = 0.0; ASC(MPCB200_SC_NREG) = 0.0; ASC(MPCB200_SC_NBT) = 0.0;
        ASC(MPCB200_SC_DDT) = 0.0; ASC(MPCB200_SC_ALPHA) = 0.0; ASC(MPCB200_SC_TINY) = 0.0; ASC(MPCB200_SC_DEFER) = 0.0;
        if (cold_pending) ASC(MPCB200_SC_COLD) = 0.0;
        ASC(MPCB200_SC_STATUS) = -1.0;
    }
    __syncwarp();
}

// ---- time budget of a solve (mpcb200_config.max_cpu_time) ----
// %globaltimer: nanoseconds of one clock for the whole device (clock64 counts cycles of one SM, at whatever clock it runs).
#define NO_DEADLINE 0xFFFFFFFFFFFFFFFFull
__device__ __forceinline__ unsigned long long global_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ bool budget_expired(unsigned long long deadline) { return deadline != NO_DEADLINE && global_ns() >= deadline; }

// ---- shared scratch of the CTA-wide phases ----
struct CtaShared
{
    EvalAcc eacc[MAX_GROUP_WARPS];
    LsAcc lacc[MAX_GROUP_WARPS];
    TrialAcc tr[MAX_GROUP_WARPS];
    int hist[CLIP_BINS + 1];
    double mu, alpha, a_dual;
    int fin, accept;
    unsigned long long deadline;   // %globaltimer value at which the solve's time budget runs out (NO_DEADLINE: none)
};

__device__ __forceinline__ double shfl_xor_d(double v, int o) { return __shfl_xor_sync(FULLMASK, v, o); }
// butterfly over the lanes, level by level for all fields (a loop over the levels: a fifth of the code of fifteen unrolled
// reductions; per field the same order of operations)
__device__ __forceinline__ void evalacc_warp_reduce(EvalAcc& a)
{
#pragma unroll 1
    for (int o = 16; o > 0; o >>= 1)
    {
        a.dual_inf = fmax(a.dual_inf, shfl_xor_d(a.dual_inf, o)); a.prim_inf = fmax(a.prim_inf, shfl_xor_d(a.prim_inf, o));
        a.sl_max = fmax(a.sl_max, shfl_xor_d(a.sl_max, o)); a.sl_min = fmin(a.sl_min, shfl_xor_d(a.sl_min, o));
        a.sum_nu += shfl_xor_d(a.sum_nu, o); a.sum_lam += shfl_xor_d(a.sum_lam, o); a.inf1 += shfl_xor_d(a.inf1, o); a.blog += shfl_xor_d(a.blog, o);
        a.gt0 += shfl_xor_d(a.gt0, o); a.gt1 += shfl_xor_d(a.gt1, o); a.gldt += shfl_xor_d(a.gldt, o); a.htt += shfl_xor_d(a.htt, o);
        a.obj += shfl_xor_d(a.obj, o); a.m_ineq += shfl_xor_d(a.m_ineq, o); a.m_eq += shfl_xor_d(a.m_eq, o);
    }
}

// ---- PHASE_EVAL (whole CTA, lane per stage): stage functions + derivatives -> condensed KKT records, KKT error,
//      convergence test (and the time budget: thread 0 reads the clock, sh.fin broadcasts its decision) and barrier update.
//      Returns 1 (uniform) when the instance terminates. ----
template <bool LINES, int MODEL>
__device__ __forceinline__ int dev_eval(const Cfg& c, const WsLayout& L, double* W, double uprev_dt, CtaShared& sh, int tid, int nt)
{
    const int N = L.N, lane = tid & 31, wid = tid >> 5, nw = nt >> 5;
    EvalAcc a;
    evalacc_init(a);
    for (int k = tid; k < N; k += nt) eval_stage<LINES, MODEL>(c, L, W, W, uprev_dt, k, a);
    __syncwarp();
    evalacc_warp_reduce(a);
    if (lane == 0) sh.eacc[wid] = a;
    __syncthreads();
    if (tid == 0)
    {
        for (int w = 1; w < nw; ++w) evalacc_merge(a, sh.eacc[w]);
        int fin = 0;
        sh.mu = eval_finish<MODEL>(c, L, W, a, true, &fin, budget_expired(sh.deadline));
        sh.fin = fin;
    }
    __syncthreads();
    if (sh.fin) return 1;
    const double mu = sh.mu;
    for (int k = tid; k < N; k += nt) eval_finalize_stage(L, W, k, mu);
    __syncthreads();
    return 0;
}

// ---- PHASE_KKT (one warp): Newton step by the warp-cooperative Riccati sweep ----
template <bool EXT>
__device__ __forceinline__ void dev_kkt(const Cfg& c, const WsLayout& L, double* W, CudaWarp<EXT>& ex, unsigned long long* sweeps)
{
    __syncwarp();   // the warp enters its collectives converged, whatever thread-0-only code ran before
    double ddt = 0.0, delta = 0.0;
    int nreg = 0;
    const int ok = kkt_warp_solve<EXT>(ex, c, L.N, W + L.oKKT, W + L.oMM, W + L.oSTEP, ASC(MPCB200_SC_HTT), ASC(MPCB200_SC_GT), ASC(MPCB200_SC_DELTA_LAST),
                                       &ddt, &delta, &nreg);
    __syncwarp();
    if (ex.lane == 0)
    {
        kkt_store_outcome(W + L.oSCAL, ok, ddt, delta, nreg);
        if (sweeps) *sweeps += (unsigned long long)(nreg + (ok ? 1 : 0));
    }
    __syncwarp();
}

// ---- PHASE_LINESEARCH (whole CTA, lane per stage): step lengths, l1-merit backtracking, iterate update ----
template <bool LINES, int MODEL>
__device__ __forceinline__ void dev_linesearch(const Cfg& c, const WsLayout& L, double* W, double uprev_dt, CtaShared& sh, int tid, int nt)
{
    const int N = L.N, lane = tid & 31, wid = tid >> 5, nw = nt >> 5;
    if (ASC(MPCB200_SC_STATUS) >= 0.0) return;   // the KKT phase gave the instance up
    if (ASC(MPCB200_SC_DEFER) != 0.0)
    {
        // the KKT phase spent its factorisation budget: null step
        __syncthreads();
        if (tid == 0) { ASC(MPCB200_SC_DEFER) = 0.0; ASC(MPCB200_SC_ITER) += 1.0; ASC(MPCB200_SC_ALPHA) = 0.0; }
        __syncthreads();
        return;
    }
    LsAcc a;
    lsacc_init(a);
    // histogram of the blocking step ratios (+ row count) -> threshold bin of the clipped rows -> primal step length
    for (int j = tid; j <= CLIP_BINS; j += nt) sh.hist[j] = 0;
    __syncthreads();
    for (int k = tid; k < N; k += nt) ls_stage_steps<MODEL>(c, L, W, W, uprev_dt, k, a, sh.hist);
    __syncthreads();
    const int jt = clip_threshold_bin(sh.hist, sh.hist[CLIP_BINS]);  // same value in every thread
    for (int k = tid; k < N; k += nt) a.a_p = fmin(a.a_p, ls_stage_ap(L, W, k, jt));
    __syncwarp();
    a.a_p = warp_min(a.a_p); a.a_d = warp_min(a.a_d);
    a.dphi_bar = warp_sum(a.dphi_bar); a.curv = warp_sum(a.curv); a.dJ = warp_sum(a.dJ);
    if (lane == 0) sh.lacc[wid] = a;
    __syncthreads();
    // scalars of the merit function (thread 0 only)
    double mu = 0.0, rho = 1.0, phi0 = 0.0, dphi = 0.0, a_d = 1.0;
    if (tid == 0)
    {
        for (int w = 1; w < nw; ++w)
        {
            const LsAcc& o = sh.lacc[w];
            a.a_p = fmin(a.a_p, o.a_p); a.a_d = fmin(a.a_d, o.a_d);
            a.dphi_bar += o.dphi_bar; a.curv += o.curv; a.dJ += o.dJ;
        }
        mu = ASC(MPCB200_SC_MU);
        const double inf1 = ASC(MPCB200_SC_INF), obj = ASC(MPCB200_SC_OBJ), blog = ASC(MPCB200_SC_BLOG);
        const double num = a.dJ + a.dphi_bar + 0.5 * (a.curv > 0 ? a.curv : 0.0);
        if (inf1 > 1e-14)
        {
            const double rho_trial = num / ((1.0 - 0.1) * inf1);
            if (rho < rho_trial) rho = rho_trial + 1.0;
        }
        phi0 = obj - mu * blog + rho * inf1;
        dphi = a.dJ + a.dphi_bar - rho * inf1;
        a_d = a.a_d;
        sh.alpha = a.a_p;
    }
    __syncthreads();
    double alpha = sh.alpha;
    int nbt = 0;
#pragma unroll 1
    for (int bt = 0; bt < MAX_BACKTRACK; ++bt)
    {
        TrialAcc t;
        t.obj = t.inf1 = t.blog = 0.0;
        for (int k = tid; k < N; k += nt) ls_stage_trial<LINES, MODEL>(c, L, W, W, uprev_dt, k, alpha, t);
        __syncwarp();
        t.obj = warp_sum(t.obj); t.inf1 = warp_sum(t.inf1); t.blog = warp_sum(t.blog);
        if (lane == 0) sh.tr[wid] = t;
        __syncthreads();
        if (tid == 0)
        {
            for (int w = 1; w < nw; ++w) { t.obj += sh.tr[w].obj; t.inf1 += sh.tr[w].inf1; t.blog += sh.tr[w].blog; }
            const double phi = t.obj - mu * t.blog + rho * t.inf1;
            sh.accept = (phi <= phi0 + ARMIJO * alpha * dphi || (bt > 0 && fabs(phi - phi0) <= 1e-13 * (1.0 + fabs(phi0)))) ? 1 : 0;
        }
        __syncthreads();
        const int accept = sh.accept;
        __syncthreads();  // sh.accept / sh.tr are rewritten by the next trial
        if (accept) break;
        alpha *= 0.5;
        ++nbt;
    }
    if (tid == 0) sh.a_dual = a_d > alpha ? alpha : a_d;
    if (LINES && is_midpoint(c))
        for (int k = tid; k < N; k += nt) ls_stage_midpoint_fix(c, L, W, k);   // reads the old heading of stage k+1
    __syncthreads();
    const double a_dual = sh.a_dual;
    for (int k = tid; k < N; k += nt) ls_stage_update<MODEL>(c, L, W, W, uprev_dt, k, alpha, a_dual);
    if (tid == 0)
    {
        if (ModelTraits<MODEL>::variable_dt(c)) ASC(MPCB200_SC_DT) = ASC(MPCB200_SC_DT) + alpha * ASC(MPCB200_SC_DDT);
        ASC(MPCB200_SC_ALPHA) = alpha;
        ASC(MPCB200_SC_RHO) = rho;
        ASC(MPCB200_SC_ITER) = ASC(MPCB200_SC_ITER) + 1.0;
        ASC(MPCB200_SC_NBT) = ASC(MPCB200_SC_NBT) + (double)nbt;
        const double tiny = alpha < TINY_STEP ? ASC(MPCB200_SC_TINY) + 1.0 : 0.0;
        ASC(MPCB200_SC_TINY) = tiny;
        if (tiny >= (double)TINY_STEP_COUNT) ASC(MPCB200_SC_STATUS) = (double)MPCB200_STATUS_NUMERICAL_ERROR;  /* jammed: give up */
    }
    __syncthreads();
}
