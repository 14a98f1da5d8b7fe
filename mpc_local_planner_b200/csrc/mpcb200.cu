// mpcb200.cu -- sm_90a kernels + C-ABI host side of the batched receding-horizon OCP solver (include/mpcb200.h).
//
// Execution model.  ONE CTA OWNS ONE INSTANCE FOR ITS WHOLE SOLVE: solve_fused_kernel is a persistent kernel whose CTAs take
// instances from a queue (atomic counter), keep the instance's resident prefix (mpc_layout.h: iterate, slacks, multipliers,
// KKT stage records, KKT stage matrices, obstacles -- 50-70 KB) in shared memory, and run initial guess, association and the
// interior-point iterations (eval -> KKT -> line search, mpc_device.cuh) back to back until the instance converges or gives
// up; then the results are written and the CTA takes the next instance.  No launch chain, no HBM round trip of records or
// gains between the phases, and no instance waits for the slowest one of its batch.  Thread mapping inside the CTA: the
// stage-parallel phases (eval, line search) put one lane on one horizon stage (ceil(N/32) warps); the KKT phase is the
// warp-cooperative Riccati sweep of mpc_riccati_warp.h on warp 0 (lanes = entries of the stage matrix, one barrier per stage).
//
// The same device functions are exposed phase by phase (mpcb200_run_phase / mpcb200_time_phase, and the "phased" solve mode)
// through phase_kernel (stages the prefix, runs one phase, writes it back) and kkt_warp_kernel (one warp per instance:
// bulk-async copy of the stage records into shared memory, sweep, Newton step back to HBM) -- the kernel the HBM roofline of
// the KKT factorisation is measured on (SURVEY 8d).
//
// This file is the ONLY implementation of the hot path: there is no CPU fallback.  Every entry point fails with
// MPCB200_E_NODEVICE / MPCB200_E_CUDA when no CUDA device is usable.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <cmath>
#include <initializer_list>
#include <string>
#include <vector>

#include "mpc_device.cuh"
#ifndef MPCB200_ENTRY_UNIT
#include "mpc_costmap.cuh"
#endif
#include "mpc_gate.h"
#include "mpc_place.h"

#define WARPS_PER_CTA 4
#define MAX_IMG_SMEM (227 * 1024 - 2048)  // dynamic shared memory a CTA may request
#define IMG_HEAD 16                        // bytes in front of the resident prefix in dynamic shared memory (mbarrier)

// device-side counters of a handle (unsigned long long each)
#define CNT_KKT_INST 0     // (instance, iteration) pairs the KKT phase factorised
#define CNT_KKT_SWEEPS 1   // backward sweeps incl. inertia-correction refactorisations
#define CNT_CYC 2          // +phase: SM cycles CTAs spent in each phase of the fused kernel (thread 0's clock64)
#define CNT_CYC_TOTAL 7    // SM cycles CTAs spent on instances in the fused kernel
#define CNT_INST 8         // instances solved by the fused kernel
#define CNT_GATE 9         // SM cycles CTAs waited at the phase gates (MPCB200_OPT_SM_PHASE_SYNC)
#define CNT_WORDS 16
// behind the CNT_WORDS counters: CNT_WORDS doubles, the counters of the device-memory solves already folded per launch
// (fold_counters_kernel): cycle words as cycles per CTA of their own launch, the other words as counts
#define CNT_BYTES (CNT_WORDS * 8 * 2)

// mpcb200_weights.cu and mpcb200_models.cu compile this file with MPCB200_ENTRY_UNIT defined: the device code the solve kernel is
// made of and the kernel-variant tables, without the other kernels and the host side, for the solve entries each instantiates (the
// per-robot-weights and the per-robot-model entries).
#ifndef MPCB200_ENTRY_UNIT
// ---- kernel: inputs of a batch into the instance blocks (phased path; the fused kernel scatters into shared memory itself) ----
__global__ void scatter_inputs_kernel(WsLayout L, double* ws, int B, InputPtrs in)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= B) return;
    double* W = ws + (int64_t)warp * L.stride;
    const bool ok = scatter_one<true>(L, W, in, warp, lane, W + L.oXINIT);   // (the phased mode serves the blocking calls only)
    if (lane == 0) ASC(MPCB200_SC_VALID) = ok ? 1.0 : 0.0;
}
#endif

// stage [0, words) of an instance block in shared memory (one bulk-async copy) / write [0, words) back
__device__ __forceinline__ void stage_in(double* W, const double* Gp, int words, uint32_t bar, uint32_t parity, int tid)
{
    if (tid == 0)
    {
        fence_async();
        mbar_expect_tx(bar, (uint32_t)words * 8u);
        bulk_g2s(smem_addr(W), Gp, (uint32_t)words * 8u, bar);
    }
    mbar_wait(bar, parity);
}
__device__ __forceinline__ void stage_out(double* Gp, const double* W, int words, int tid)
{
    __syncthreads();
    if (tid == 0)
    {
        fence_async();   // the CTA's ordinary stores to shared memory before the async-proxy read
        bulk_s2g(Gp, smem_addr(W), (uint32_t)words * 8u);
        bulk_commit_wait();
    }
    __syncthreads();
}

// an instance whose inputs are not finite: reported, never iterated, starts cold next time
__device__ __forceinline__ void mark_invalid(const WsLayout& L, double* W)
{
    ASC(MPCB200_SC_STATUS) = (double)MPCB200_STATUS_INVALID_INPUT;
    ASC(MPCB200_SC_COLD) = 1.0; ASC(MPCB200_SC_ITER) = 0.0; ASC(MPCB200_SC_ERR0) = 0.0; ASC(MPCB200_SC_DT) = 0.0;
}

// ---- kernel: ONE PHASE of the solve for every instance of a batch (kernel-level API and the phased solve mode) ----
template <bool LINES, int MODEL>
__global__ void __launch_bounds__(MAX_GROUP_WARPS * 32, 3) phase_kernel(const __grid_constant__ Cfg c, const __grid_constant__ WsLayout L, double* ws, int B, int phase,
                                                                       double uprev_dt, int force_cold, int first_outer, int* n_active, int img_words, InputPtrs in)
{
    extern __shared__ __align__(128) unsigned char dyn_smem[];
    __shared__ CtaShared sh;
    const int inst = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nt = blockDim.x;
    double* Gp = ws + (int64_t)inst * L.stride;
    if (Gp[L.oSCAL + MPCB200_SC_VALID] == 0.0)
    {
        if (tid == 0 && phase == MPCB200_PHASE_INIT) mark_invalid(L, Gp);
        return;
    }
    if (phase >= MPCB200_PHASE_EVAL && Gp[L.oSCAL + MPCB200_SC_STATUS] >= 0.0) return;  // finished instance: exact no-op (uniform over the CTA)
    double* W = reinterpret_cast<double*>(dyn_smem + IMG_HEAD);
    const uint32_t bar = smem_addr(dyn_smem);
    if (tid == 0)
    {
        mbar_init(bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        sh.deadline = NO_DEADLINE;   // one phase for every instance: no solve, no clock of a solve (max_cpu_time: fused kernel only)
    }
    __syncthreads();
    stage_in(W, Gp, img_words, bar, 0, tid);
    switch (phase)
    {
        case MPCB200_PHASE_INIT: if (wid == 0) dev_init(c, L, W, obstacle_source(L, W, in, inst), Gp + L.oXINIT, force_cold, lane, 0); break;
        case MPCB200_PHASE_ASSOCIATE:
            if (wid == 0)
            {
                const bool long_list = in.obst_count && in.obst_max > L.M;
                dev_associate(c, L, W, uprev_dt, first_outer, lane, obstacle_source(L, W, in, inst), long_list, Gp + L.oOGIDX);
            }
            break;
        case MPCB200_PHASE_EVAL:
        {
            const int fin = dev_eval<LINES, MODEL>(c, L, W, uprev_dt, sh, tid, nt);
            if (!fin && n_active && tid == 0) atomicAdd(n_active, 1);
            break;
        }
        case MPCB200_PHASE_LINESEARCH: dev_linesearch<LINES, MODEL>(c, L, W, uprev_dt, sh, tid, nt); break;
        default: break;
    }
    // everything but the inputs -- except after the association over a long list, which fills the resident obstacles
    const bool wrote_obstacles = phase == MPCB200_PHASE_ASSOCIATE && in.obst_count && in.obst_max > L.M;
    stage_out(Gp, W, wrote_obstacles ? img_words : L.oOTYPE, tid);
}

// ---- kernel: PHASE_KKT -- one warp per instance: records HBM -> shared memory (one bulk-async copy), warp-cooperative
//      Riccati sweep (mpc_riccati_warp.h), Newton step -> HBM.  Algorithmic traffic: the records in, 8 words per stage out. ----
template <bool EXT>
__global__ void __launch_bounds__(32) kkt_warp_kernel(const __grid_constant__ Cfg c, const __grid_constant__ WsLayout L, double* ws, int B, unsigned long long* counters)
{
    extern __shared__ __align__(128) unsigned char dyn_smem[];
    const int inst = blockIdx.x, lane = threadIdx.x;
    const int N = L.N;
    double* Gp = ws + (int64_t)inst * L.stride;
    if (Gp[L.oSCAL + MPCB200_SC_VALID] == 0.0 || Gp[L.oSCAL + MPCB200_SC_STATUS] >= 0.0) return;
    const int rec_words = (N * RSTR + 1) & ~1;
    double* recs = reinterpret_cast<double*>(dyn_smem + IMG_HEAD);
    double* mms = recs + rec_words;
    double* stp = mms + rw_scratch_words<EXT>(N);
    const uint32_t bar = smem_addr(dyn_smem);
    if (lane == 0)
    {
        mbar_init(bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_expect_tx(bar, (uint32_t)rec_words * 8u);
        bulk_g2s(smem_addr(recs), Gp + L.oKKT, (uint32_t)rec_words * 8u, bar);
    }
    CudaWarp<EXT> ex;
    ex.lane = lane;
    kkt_warp_setup<EXT>(ex, c.variable_dt);   // beside the copy
    const double htt = Gp[L.oSCAL + MPCB200_SC_HTT], gt = Gp[L.oSCAL + MPCB200_SC_GT], dlast = Gp[L.oSCAL + MPCB200_SC_DELTA_LAST];
    __syncwarp();
    mbar_wait(bar, 0);
    double ddt = 0.0, delta = 0.0;
    int nreg = 0;
    const int ok = kkt_warp_solve<EXT>(ex, c, N, recs, mms, stp, htt, gt, dlast, &ddt, &delta, &nreg);
    __syncwarp();
    if (ok)
        for (int i = lane; i < 8 * N; i += 32) Gp[L.oSTEP + i] = stp[i];
    if (lane == 0)
    {
        kkt_store_outcome(Gp + L.oSCAL, ok, ddt, delta, nreg);
        if (counters) { atomicAdd(counters + CNT_KKT_INST, 1ull); atomicAdd(counters + CNT_KKT_SWEEPS, (unsigned long long)(nreg + (ok ? 1 : 0))); }
    }
}
template <bool EXT>
static size_t kkt_smem_bytes(int N) { return IMG_HEAD + (size_t)(((N * RSTR + 1) & ~1) + rw_scratch_words<EXT>(N) + 8 * N) * 8; }

// ---- kernel: THE SOLVE.  Persistent CTAs take instances from a queue and own them until they terminate. ----
struct FusedArgs
{
    double* ws;              // instance blocks (batch mode: instance i <-> block i, warm state in / out); unused in queue mode
    InputPtrs in;
    OutputPtrs out;
    int total;               // instances in the queue
    int queue_mode;          // 1: a queue of cold instances without blocks (mpcb200_solve_stream)
    int force_cold;
    int cand_stride;         // multistart kernel: instance i is candidate i / cand_stride of robot i % cand_stride, whose inputs it reads
    double uprev_dt;
    int img_words;           // resident prefix
    int* queue;              // next instance
    const int* order;        // queue position -> instance (nullptr: identity)
    unsigned long long* counters;
    unsigned long long* sm_sync;   // [sm_words * SMS_WORD_STRIDE] phase alignment words, one line per SM (nullptr: off)
    int sm_words;                  // SMs with a word
    int sm_gates;                  // 3: gates before eval, KKT and line search; 2: before KKT and line search only
    unsigned long long budget_ns;  // time budget of the launch (max_cpu_time), 0: none
    unsigned long long* origin;    // %globaltimer at the start of the launch: the first CTA sets it (zeroed before the launch)
    int* place;                    // critical placement (nullptr: off): [0] heavy instances H, [1] heavy claims (mpc_place.h)
    unsigned long long* place_sm;  // admission word of each SM (sm_words of them): word 1 of its phase-alignment line
    int place_cotenants;           // CTAs a heavy instance shares its SM with, at most
};
// ---- phase alignment of the CTAs that share an SM ---------------------------------------------------------------------------
// The solve kernel's iteration is ~128 KB of straight fp64 code, several times an SM's instruction cache: CTAs that sit on the
// same SM in different phases evict each other's code and every warp streams its instructions from the next cache level.
// The co-resident CTAs therefore enter each phase of the iteration together, through a barrier per SM with changing membership
// (mpc_gate.h).  Each SM's word has a 128-byte line of its own, so the CTAs of different SMs never contend for a line.
// Timing only -- no data crosses CTAs.
#define SMS_POLL_NS 128   // pause between two polls of the barrier word (the polling thread shares its scheduler with working warps)
#define SMS_WORD_STRIDE 16   // words: one 128-byte line per SM
// Critical placement (mpc_place.h; DESIGN.md 4, measured on an H100): the heavy part is the instances whose predicted count exceeds
// PLACE_RHO x the mean per CTA slot, and each shares its SM with at most PLACE_COTENANTS other CTAs (compile-time, so that
// tools/placement_sweep.py can compare settings as libraries of their own).
#ifndef PLACE_RHO
#define PLACE_RHO 1.3
#endif
#ifndef PLACE_COTENANTS
#define PLACE_COTENANTS 0
#endif
struct DevAtomics
{
    typedef unsigned long long Word;
    static __device__ __forceinline__ Word add(Word* w, Word v) { return atomicAdd(w, v); }
    static __device__ __forceinline__ int add(int* w, int v) { return atomicAdd(w, v); }
    static __device__ __forceinline__ Word cas(Word* w, Word expected, Word desired) { return atomicCAS(w, expected, desired); }
    // relaxed, not acquire: no data crosses CTAs, and on sm_90a an acquire load is followed by an invalidation of the whole L1
    // (CCTL.IVALL), so every poll would throw away the cached global data of the CTAs that share the SM
    static __device__ __forceinline__ Word load(Word* w)
    {
        Word v;
        asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(w));
        return v;
    }
    static __device__ __forceinline__ void pause() { __nanosleep(SMS_POLL_NS); }
};
__device__ __forceinline__ unsigned sm_index() { unsigned r; asm volatile("mov.u32 %0, %%smid;" : "=r"(r)); return r; }

// ---- kernel: queue order of a batch = longest first by the iteration counts of the PREVIOUS solve of the same slots ----
// A batch costs its slowest instance: an instance that needs 100 iterations and is taken from the queue when the first slots free
// up (2-3 ms into the step) ends 2-3 ms later than if it had been among the first.  Nothing predicts the iteration count of a cold
// instance from its geometry (correlations < 0.2 on the BASELINE instances), but a robot that was hard in the last cycle tends to be
// hard in this one, so the history is the hint.  Counting sort (descending, stable) by min(iters, 1023) in one CTA.
// An instance the time budget stopped (MPCB200_STATUS_MAX_TIME) counts as needing max_iter iterations whatever it ran: otherwise
// the instances the queue never reached (iters 0) would go last again and stay unsolved in every cycle.
// With the critical placement (place != nullptr) the kernel also plans the heavy part of mpc_place.h: the H leading instances whose
// count exceeds rho x the mean count per CTA slot (the batch's total over `slots`), at most max_heavy; it writes H and a zero
// claim count to place[0..1] and starts the queue counter (the light part) at H.
__device__ __forceinline__ int history_key(const int* prev_iters, const int* prev_status, int max_iter, int i)
{
    const int k = prev_status[i] == MPCB200_STATUS_MAX_TIME ? max_iter : prev_iters[i];
    return k < 0 ? 0 : (k > 1023 ? 1023 : k);
}
#ifndef MPCB200_ENTRY_UNIT
__global__ void __launch_bounds__(1024) order_by_history_kernel(const int* __restrict__ prev_iters, const int* __restrict__ prev_status, int max_iter,
                                                                int B, int* __restrict__ order, int* place, int slots, double rho,
                                                                int max_heavy, int* queue)
{
    __shared__ int hist[1024];
    __shared__ int warp_tot[32];
    __shared__ unsigned long long s_work;
    __shared__ int s_heavy;
    const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
    hist[t] = 0;
    __syncthreads();
    for (int i = t; i < B; i += 1024) atomicAdd(&hist[1023 - history_key(prev_iters, prev_status, max_iter, i)], 1);
    __syncthreads();
    // exclusive scan of hist (bucket 0 = the longest)
    const int v = hist[t];
    if (place)
    {
        if (t == 0) { s_work = 0ull; s_heavy = 0; }
        __syncthreads();
        atomicAdd(&s_work, (unsigned long long)v * (unsigned long long)(1023 - t));
        __syncthreads();
        if (v > 0 && (double)(1023 - t) > rho * (double)s_work / (double)slots) atomicAdd(&s_heavy, v);
        __syncthreads();
        if (t == 0) { const int H = s_heavy < max_heavy ? s_heavy : max_heavy; place[0] = H; place[1] = 0; *queue = H; }
    }
    int incl = v;
    for (int o = 1; o < 32; o <<= 1) { const int u = __shfl_up_sync(FULLMASK, incl, o); if (lane >= o) incl += u; }
    if (lane == 31) warp_tot[wid] = incl;
    __syncthreads();
    int woff = 0;
    for (int w = 0; w < wid; ++w) woff += warp_tot[w];
    __syncthreads();
    hist[t] = woff + incl - v;   // first position of bucket t
    __syncthreads();
    // stable placement: the thread that owns a bucket walks the instances in index order (buckets are few and short in practice;
    // the walk is B loads per non-empty bucket owner -- done by the warps in parallel over the buckets)
    if (v > 0)
    {
        int pos = hist[t];
        const int key = 1023 - t;
        for (int i = 0; i < B; ++i)
            if (history_key(prev_iters, prev_status, max_iter, i) == key) order[pos++] = i;
    }
}
#endif

// CTA shapes of the solve kernel.  The launch bound sets the register budget of a thread (255 in both shapes), so it follows
// the shape a launch uses: horizons up to 64 grid points run 1-2 warps, and their shared-memory image (about 55 KB at N = 50)
// lets 4 CTAs share an SM; longer horizons run 3-4 warps with an image of about 70 KB and more (90 KB at N = 80), so
// shared memory allows 2 CTAs per SM from N = 80 on, and the bound keeps them at 2 below that.  A budget set for a shape a
// launch does not use spills the iteration's operands to local memory.
#define SMALL_GROUP_WARPS 2
template <int WARPS> struct FusedShape;
template <> struct FusedShape<SMALL_GROUP_WARPS> { static constexpr int MIN_CTAS = 4; };
template <> struct FusedShape<MAX_GROUP_WARPS> { static constexpr int MIN_CTAS = 2; };

// Per-robot limits (mpcb200_set_robot_limits): the records, and one configuration per CTA in global memory -- the handle's
// configuration with the record of the CTA's current instance applied.  (A copy in shared memory would cost cfg 2 one of its
// four CTAs per SM: 848 bytes more than the 56 KB images leave.)
struct RobotArgs
{
    const double* limits;   // [robots][MPCB200_LIMIT_WORDS]
    Cfg* cfg;               // [grid] the configuration CTA blockIdx.x presents to the phases
};

// The solve of the persistent kernel.  c0 is the handle's configuration.  MULTI: the multistart form (mpcb200_step_batch_multistart);
// ROBOT: the per-robot-limits form.  Either only changes the prologue of an instance (MULTI: its inputs, its bump rank; ROBOT: the
// configuration the phases read), and each is an instantiation of its own, so that the solve kernels of the other calls keep their
// registers and local memory.
// FLEET (with ROBOT): the per-robot-geometry form -- the limits records are optional (r.limits may be null), and the geometry
// record of each robot (mpcb200_set_robot_geometry, `geo`) is applied to the CTA's configuration after them.
// WEIGHTS (with ROBOT): the per-robot-weights form -- the limits and geometry records are optional (r.limits, geo may be null; geometry
// only in the MODEL_GENERIC instantiations), and the weights record of each robot (mpcb200_set_robot_weights, `wgt`) is applied last.
// MODELS (with ROBOT, MODEL_GENERIC only): the per-robot-model form -- the model record of each robot (mpcb200_set_robot_model, `mdl`)
// is applied first, then the limits, geometry and weights records of the kinds that are set (r.limits, geo, wgt may be null).
template <bool LINES, bool EXT, int WARPS, int MODEL, bool MULTI, bool ROBOT, bool FLEET = false, bool WEIGHTS = false, bool MODELS = false>
__device__ __forceinline__ void solve_fused(const Cfg& c0, const WsLayout& L, const FusedArgs& a, const RobotArgs& r, const double* geo = nullptr,
                                            const double* wgt = nullptr, const double* mdl = nullptr)
{
    const Cfg& c = ROBOT ? r.cfg[blockIdx.x] : c0;
    extern __shared__ __align__(128) unsigned char dyn_smem[];
    __shared__ CtaShared sh;
    __shared__ int s_inst, s_valid, s_solo, s_next;
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nt = blockDim.x;
    const int N = L.N;
    double* W = reinterpret_cast<double*>(dyn_smem + IMG_HEAD);
    const uint32_t bar = smem_addr(dyn_smem);
    if (tid == 0)
    {
        mbar_init(bar, 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        // the time budget: one origin for the whole launch, the %globaltimer reading of the CTA that starts first
        unsigned long long deadline = NO_DEADLINE;
        if (a.budget_ns)
        {
            const unsigned long long now = global_ns(), prev = atomicCAS(a.origin, 0ull, now), t0 = prev ? prev : now;
            deadline = t0 + a.budget_ns;
            if (deadline < t0 || deadline == NO_DEADLINE) deadline = NO_DEADLINE - 1;   // saturate
        }
        sh.deadline = deadline;
        s_solo = 0;
        s_next = place::ADMIT;
    }
    if (ROBOT)
    {
        const unsigned long long* src = reinterpret_cast<const unsigned long long*>(&c0);
        unsigned long long* dst = reinterpret_cast<unsigned long long*>(r.cfg + blockIdx.x);
        for (int i = tid; i < (int)(sizeof(Cfg) / 8); i += nt) dst[i] = src[i];
    }
    CudaWarp<EXT> ex;
    ex.lane = lane;
    if (wid == 0) kkt_warp_setup<EXT>(ex, c0.variable_dt);
    __syncthreads();
    uint32_t parity = 0;
    unsigned long long cyc[MPCB200_NUM_PHASES] = {0, 0, 0, 0, 0}, cyc_total = 0, n_kkt = 0, n_sweeps = 0, n_inst = 0;
    const unsigned nph = (unsigned)a.sm_gates;
    unsigned long long gate_cyc = 0;   // waiting at the phase gates (included in the phase that follows the gate)
    unsigned long long* sms = nullptr;
    // (PTX does not promise %smid < the SM count: a CTA without a word runs without gates)
    if (a.sm_sync) { const unsigned smid = sm_index(); if (smid < (unsigned)a.sm_words) sms = a.sm_sync + (size_t)smid * SMS_WORD_STRIDE; }
    const int outer = c0.outer_iterations > 0 ? c0.outer_iterations : 1;
// Phase clocks: EVERY thread keeps them (thread 0's are reported).  Not `if (tid == 0)`: a thread-0-only block directly in front of
// warp-collective code (shuffles, votes) made the compiler split the paths of thread 0 and of lanes 1..31 through the KKT phase in
// one build variant -- lanes 1..31 ran their shuffles on the converged fast path, thread 0 waited in the collective slow path for
// ever.  Branch-free bookkeeping leaves nothing to split.
#define TICK(p_) do { const long long t_ = clock64(); cyc[p_] += (unsigned long long)(t_ - t_mark); t_mark = t_; } while (0)
    for (;;)
    {
        if (tid == 0)
        {
            if (!a.place) { const int q = atomicAdd(a.queue, 1); s_inst = (q < a.total && a.order) ? a.order[q] : q; }
            else
            {
                int nx = s_next;   // (admission here rather than in the prologue: it leaves every variant's registers and spills alone)
                if (nx == place::ADMIT)
                {
                    nx = place::TAKE;
                    const unsigned smid = sm_index();
                    if (smid < (unsigned)a.sm_words)
                    {
                        nx = place::admit<DevAtomics>(a.place_sm + (size_t)smid * SMS_WORD_STRIDE, a.place, a.order, (unsigned)a.place_cotenants);
                        s_solo = nx >= 0 && a.place_cotenants == 0;   // a heavy instance alone on its SM: no gates
                    }
                }
                s_next = place::TAKE;
                s_inst = nx >= 0 ? nx : (nx == place::LEAVE ? a.total : place::take<DevAtomics>(a.queue, a.place, a.order, a.total));
            }
        }
        __syncthreads();
        const int inst = s_inst;
        if (inst >= a.total) break;
        long long t_mark = clock64();
        const long long t_begin = t_mark;
        double* Gp = a.queue_mode ? nullptr : a.ws + (int64_t)inst * L.stride;
        const int src = MULTI ? inst % a.cand_stride : inst, rank = MULTI ? inst / a.cand_stride : 0;   // inputs, bump rank
        // ---- state: warm trajectory and scalars of the block, or a fresh cold slot ----
        if (!a.queue_mode) { stage_in(W, Gp, L.oNU, bar, parity, tid); parity ^= 1u; }
        else if (tid < MPCB200_SCAL_WORDS) W[L.oSCAL + tid] = tid == MPCB200_SC_COLD ? 1.0 : (tid == MPCB200_SC_STATUS ? -1.0 : 0.0);
        __syncthreads();
        // ---- inputs ----
        if (wid == 0)
        {
            bool ok = scatter_one<LINES>(L, W, a.in, src, lane, nullptr);
            if (lane == 0)
            {
                if (ROBOT && ok)   // the robot's configuration: its record, checked as the blocking setter checks it
                {
                    if constexpr (MODELS)
                    {
                        // the types first: the geometry (its record, or the configuration's values) is checked for them, and the
                        // geometry record's patch writes the fields they read.  Each record rewrites every field it touches, per instance.
                        Cfg& rc = r.cfg[blockIdx.x];
                        const double* m = mdl + (int64_t)src * MPCB200_MODEL_WORDS;
                        const double* g = geo ? geo + (int64_t)src * MPCB200_GEOMETRY_WORDS : nullptr;
                        ok = robot_model_valid(c0, m, g);
                        if (ok) apply_robot_model(rc, m);
                        if (ok && r.limits)
                        {
                            const double* rec = r.limits + (int64_t)src * MPCB200_LIMIT_WORDS;
                            ok = robot_limits_valid(c0, rec);
                            if (ok) apply_robot_limits(rc, rec);
                        }
                        if (ok && g) apply_robot_geometry(rc, g);
                        if (ok && wgt)
                        {
                            const double* w = wgt + (int64_t)src * MPCB200_WEIGHT_WORDS;
                            ok = robot_weights_valid(c0, w);
                            if (ok) apply_robot_weights(rc, w);
                        }
                    }
                    else if constexpr (FLEET)
                    {
                        // every field a phase reads is rewritten here for each instance: nothing of the CTA's previous robot is left
                        Cfg& rc = r.cfg[blockIdx.x];
                        if (r.limits)
                        {
                            const double* rec = r.limits + (int64_t)src * MPCB200_LIMIT_WORDS;
                            ok = robot_limits_valid(c0, rec);
                            if (ok) apply_robot_limits(rc, rec);
                        }
                        if (ok)
                        {
                            const double* g = geo + (int64_t)src * MPCB200_GEOMETRY_WORDS;
                            ok = robot_geometry_valid(c0, g);
                            if (ok) apply_robot_geometry(rc, g);
                        }
                    }
                    else if constexpr (WEIGHTS)
                    {
                        // as FLEET: the limits, the geometry and the weights record each rewrite every field they touch, per instance
                        Cfg& rc = r.cfg[blockIdx.x];
                        if (r.limits)
                        {
                            const double* rec = r.limits + (int64_t)src * MPCB200_LIMIT_WORDS;
                            ok = robot_limits_valid(c0, rec);
                            if (ok) apply_robot_limits(rc, rec);
                        }
                        if constexpr (MODEL == MODEL_GENERIC)
                            if (ok && geo)
                            {
                                const double* g = geo + (int64_t)src * MPCB200_GEOMETRY_WORDS;
                                ok = robot_geometry_valid(c0, g);
                                if (ok) apply_robot_geometry(rc, g);
                            }
                        if (ok)
                        {
                            const double* w = wgt + (int64_t)src * MPCB200_WEIGHT_WORDS;
                            ok = robot_weights_valid(c0, w);
                            if (ok) apply_robot_weights(rc, w);
                        }
                    }
                    else
                    {
                        const double* rec = r.limits + (int64_t)src * MPCB200_LIMIT_WORDS;
                        ok = robot_limits_valid(c0, rec);
                        if (ok) apply_robot_limits(r.cfg[blockIdx.x], rec);
                    }
                }
                s_valid = ok; ASC(MPCB200_SC_VALID) = ok ? 1.0 : 0.0; if (!ok) mark_invalid(L, W);
                if (MULTI && ok && rank > 0)   // a challenger: the straight line bumped by its rank, whatever the incumbent's plan
                {
                    AIN(IN_HASXINIT) = 0.0;
                    if (!challenger_has_guess(c, L, W)) { s_valid = 0; mark_invalid(L, W); ASC(MPCB200_SC_STATUS) = (double)MPCB200_STATUS_SKIPPED; }
                }
            }
        }
        __syncthreads();
        if (s_valid)
        {
            const bool long_list = a.in.obst_count && a.in.obst_max > L.M;
            const ObstSrc os = obstacle_source(L, W, a.in, src);
            double* gidx = W + L.oMM;   // scratch of the KKT / line-search phases, free while the association runs
            if (wid == 0) dev_init(c, L, W, os, a.in.x_init ? a.in.x_init + (int64_t)src * 3 * N : nullptr, MULTI && rank > 0 ? 1 : a.force_cold, lane, rank);
            __syncthreads();
            TICK(MPCB200_PHASE_INIT);
            for (int oi = 0; oi < outer; ++oi)
            {
                if (wid == 0)
                {
                    dev_associate(c, L, W, a.uprev_dt, oi == 0, lane, os, long_list, gidx);
                    if (long_list && Gp)
                        for (int i = lane; i < L.M; i += 32) Gp[L.oOGIDX + i] = gidx[i];
                }
                __syncthreads();
                TICK(MPCB200_PHASE_ASSOCIATE);
                if (sms) { if (tid == 0 && !s_solo) gate::join<DevAtomics>(sms); __syncthreads(); }
// The tail of a launch, once the queue is drained, runs without gates.  With the queue longest first by history (a.order) the
// instances still running then are the longest ones, started first, and the step ends with the slowest of them: waiting for its
// SM neighbours at every phase costs it more than their code in its instruction cache (H100, DESIGN.md 4).  In index order the
// tail holds instances that started late, and it stays aligned; there a CTA leaves only once it is alone on its SM (every CTA of
// the SM that could still join holds an instance already).  Thread 0 keeps the flag in shared memory: the iteration loop has
// no register to spare.
#define PHASE_GATE(p_) do { if (sms) { if (tid == 0 && !s_solo) { const long long g0_ = clock64(); \
        const bool drained_ = *(volatile const int*)a.queue >= a.total; \
        if ((gate::arrive<DevAtomics>(sms, p_, nph) == 1u || a.order) && drained_) { gate::leave<DevAtomics>(sms); s_solo = 1; } \
        gate_cyc += (unsigned long long)(clock64() - g0_); } __syncthreads(); } } while (0)
                for (;;)
                {
                    if (nph == 3u) PHASE_GATE(0u);
                    const int fin = dev_eval<LINES, MODEL>(c, L, W, a.uprev_dt, sh, tid, nt);
                    TICK(MPCB200_PHASE_EVAL);
                    if (fin) break;
                    PHASE_GATE(nph - 2u);
                    if (wid == 0) dev_kkt<EXT>(c, L, W, ex, &n_sweeps);
                    __syncthreads();
                    TICK(MPCB200_PHASE_KKT);
                    ++n_kkt;
                    if (ASC(MPCB200_SC_STATUS) >= 0.0) break;   // inertia correction failed: given up
                    PHASE_GATE(nph - 1u);
                    dev_linesearch<LINES, MODEL>(c, L, W, a.uprev_dt, sh, tid, nt);
                    TICK(MPCB200_PHASE_LINESEARCH);
                    if (ASC(MPCB200_SC_STATUS) >= 0.0) break;   // jammed: given up
                }
#undef PHASE_GATE
                if (sms) { if (tid == 0 && !s_solo) gate::leave<DevAtomics>(sms); __syncthreads(); }
                if (ASC(MPCB200_SC_STATUS) == (double)MPCB200_STATUS_MAX_TIME) break;   // the budget spans the outer iterations
            }
            // a failed solve leaves nothing to warm-start from
            if (tid == 0 && ASC(MPCB200_SC_STATUS) == (double)MPCB200_STATUS_NUMERICAL_ERROR) ASC(MPCB200_SC_COLD) = 1.0;
        }
        __syncthreads();
        gather_one(L, W, a.out, inst, tid, nt);
        if (!a.queue_mode) stage_out(Gp, W, L.oSTATE_END, tid);   // state (and what the kernel-level API reads back)
        else __syncthreads();
        cyc_total += (unsigned long long)(clock64() - t_begin); ++n_inst;
    }
#undef TICK
    if (tid == 0 && a.counters)
    {
        for (int p = 0; p < MPCB200_NUM_PHASES; ++p) atomicAdd(a.counters + CNT_CYC + p, cyc[p]);
        atomicAdd(a.counters + CNT_GATE, gate_cyc);
        atomicAdd(a.counters + CNT_CYC_TOTAL, cyc_total);
        atomicAdd(a.counters + CNT_KKT_INST, n_kkt);
        atomicAdd(a.counters + CNT_KKT_SWEEPS, n_sweeps);
        atomicAdd(a.counters + CNT_INST, n_inst);
    }
}
template <bool LINES, bool EXT, int WARPS, int MODEL, bool MULTI>
__global__ void __launch_bounds__(WARPS * 32, FusedShape<WARPS>::MIN_CTAS) solve_fused_kernel(const __grid_constant__ Cfg c, const __grid_constant__ WsLayout L, const __grid_constant__ FusedArgs a)
{
    solve_fused<LINES, EXT, WARPS, MODEL, MULTI, false>(c, L, a, RobotArgs{nullptr, nullptr});
}
// the per-robot-limits form: the same solve, the phases read the configuration of the CTA's current robot (RobotArgs)
template <bool LINES, bool EXT, int WARPS, int MODEL, bool MULTI>
__global__ void __launch_bounds__(WARPS * 32, FusedShape<WARPS>::MIN_CTAS) solve_fused_robot_kernel(const __grid_constant__ Cfg c, const __grid_constant__ WsLayout L,
                                                                                                   const __grid_constant__ FusedArgs a, const __grid_constant__ RobotArgs r)
{
    solve_fused<LINES, EXT, WARPS, MODEL, MULTI, true>(c, L, a, r);
}
// the per-robot-geometry form (built for MODEL_GENERIC only: a handle with geometry records never has the unicycle / point key):
// the same solve, the CTA's configuration patched with its current robot's limits record, if any, and geometry record
template <bool LINES, bool EXT, int WARPS, int MODEL, bool MULTI>
__global__ void __launch_bounds__(WARPS * 32, FusedShape<WARPS>::MIN_CTAS) solve_fused_fleet_kernel(const __grid_constant__ Cfg c, const __grid_constant__ WsLayout L,
                                                                                                   const __grid_constant__ FusedArgs a, const __grid_constant__ RobotArgs r,
                                                                                                   const double* geometry)
{
    solve_fused<LINES, EXT, WARPS, MODEL, MULTI, true, true>(c, L, a, r, geometry);
}
// the per-robot-weights form (every key: weights are values of the quadratic-form terms the fixed-dt key keeps): the same solve, the
// CTA's configuration patched with its current robot's limits record, if any, geometry record, if any, and weights record
template <bool LINES, bool EXT, int WARPS, int MODEL, bool MULTI>
__global__ void __launch_bounds__(WARPS * 32, FusedShape<WARPS>::MIN_CTAS) solve_fused_weights_kernel(const __grid_constant__ Cfg c, const __grid_constant__ WsLayout L,
                                                                                                     const __grid_constant__ FusedArgs a, const __grid_constant__ RobotArgs r,
                                                                                                     const double* geometry, const double* weights)
{
    solve_fused<LINES, EXT, WARPS, MODEL, MULTI, true, false, true>(c, L, a, r, geometry, weights);
}
// the per-robot-model form (built for MODEL_GENERIC only, which reads both types from the configuration): the same solve, the CTA's
// configuration patched with its current robot's model record, then its limits, geometry and weights records where those are set
template <bool LINES, bool EXT, int WARPS, int MODEL, bool MULTI>
__global__ void __launch_bounds__(WARPS * 32, FusedShape<WARPS>::MIN_CTAS) solve_fused_models_kernel(const __grid_constant__ Cfg c, const __grid_constant__ WsLayout L,
                                                                                                    const __grid_constant__ FusedArgs a, const __grid_constant__ RobotArgs r,
                                                                                                    const double* geometry, const double* weights, const double* model)
{
    solve_fused<LINES, EXT, WARPS, MODEL, MULTI, true, false, false, true>(c, L, a, r, geometry, weights, model);
}

#ifndef MPCB200_ENTRY_UNIT
// ---- kernel: multistart selection, one warp per robot: the winner among the K candidates (multistart_winner), its state into
//      slot b (and the resident obstacles' list indices of a long list), its results into output row b ----
__global__ void multistart_select_kernel(WsLayout L, double* ws, int B, int K, double hysteresis, int long_list, OutputPtrs o, int* winner)
{
    const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (b >= B) return;
    double* W = ws + (int64_t)b * L.stride;
    int w = 0;
    if (lane == 0) w = multistart_winner([&](int k, int f) { return ws[((int64_t)k * B + b) * L.stride + L.oSCAL + f]; }, K, hysteresis);
    w = __shfl_sync(FULLMASK, w, 0);
    if (w > 0)
    {
        const double* Wc = ws + ((int64_t)w * B + b) * L.stride;
        for (int i = lane; i < L.oSTATE_END; i += 32) W[i] = Wc[i];
        if (long_list)
            for (int i = lane; i < L.M; i += 32) W[L.oOGIDX + i] = Wc[L.oOGIDX + i];
    }
    __syncwarp();
    gather_one(L, W, o, b, lane, 32);
    if (lane == 0 && winner) winner[b] = w;
}

// ---- kernel: gather results into compact arrays (phased path) ----------------------------------------------------------------
__global__ void gather_outputs_kernel(WsLayout L, double* ws, int B, OutputPtrs o)
{
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= B) return;
    double* W = ws + (int64_t)warp * L.stride;
    if (lane == 0 && ASC(MPCB200_SC_STATUS) == (double)MPCB200_STATUS_NUMERICAL_ERROR) ASC(MPCB200_SC_COLD) = 1.0;
    __syncwarp();
    gather_one(L, W, o, warp, lane, 32);
}

__global__ void reset_kernel(WsLayout L, double* ws, int B, const unsigned char* which)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    if (which && !which[b]) return;
    double* W = ws + (int64_t)b * L.stride;
    ASC(MPCB200_SC_COLD) = 1.0;
    ASC(MPCB200_SC_STATUS) = -1.0;
}

// ---- horizon change (grid adaptation): pack the warm trajectories, switch the layout, resample into the new one ----
// record per instance: SCAL words, X (3 x n_old), U (2 x n_old)
__global__ void resample_pack_kernel(WsLayout L, const double* ws, double* rec, int rec_words, int B)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const double* W = ws + (int64_t)b * L.stride;
    double* r = rec + (size_t)b * rec_words;
    const int N = L.N;
    for (int i = 0; i < MPCB200_SCAL_WORDS; ++i) r[i] = W[L.oSCAL + i];
    for (int i = 0; i < 3 * N; ++i) r[MPCB200_SCAL_WORDS + i] = W[L.oX + i];
    for (int i = 0; i < 2 * N; ++i) r[MPCB200_SCAL_WORDS + 3 * N + i] = W[L.oU + i];
}
__global__ void resample_unpack_kernel(WsLayout L, double* ws, const double* rec, int rec_words, int n_old, int B)
{
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    double* W = ws + (int64_t)b * L.stride;
    const double* r = rec + (size_t)b * rec_words;
    for (int i = 0; i < MPCB200_SCAL_WORDS; ++i) W[L.oSCAL + i] = r[i];
    if (ASC(MPCB200_SC_COLD) != 0.0) return;  // empty grid: the next step initialises it at the new horizon
    ASC(MPCB200_SC_DT) = resample_serial(n_old, r + MPCB200_SCAL_WORDS, r + MPCB200_SCAL_WORDS + 3 * n_old, r[MPCB200_SC_DT], L.N, W + L.oX, W + L.oU);
}


// ---- the counters of a solve launch that no host synchronise follows: a mean per CTA needs the grid of its own launch, and
//      launches of different grids may accumulate before the next synchronising call reads them ----
__global__ void fold_counters_kernel(unsigned long long* raw, int grid)
{
    const int i = threadIdx.x;
    if (i >= CNT_WORDS) return;
    double* fold = reinterpret_cast<double*>(raw + CNT_WORDS);
    const bool cycles = (i >= CNT_CYC && i < CNT_CYC + MPCB200_NUM_PHASES) || i == CNT_GATE;
    fold[i] += cycles ? (double)raw[i] / (double)grid : (double)raw[i];
    raw[i] = 0ull;
}

__global__ void flush_kernel(double* buf, size_t n)
{
    size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    for (; i < n; i += (size_t)gridDim.x * blockDim.x) buf[i] = buf[i] * 0.999 + 1.0;
}

// =================================================================================================================
// host side
// =================================================================================================================
// Compact device arrays of the inputs and outputs of `rows` instances: the batch's (instance i <-> block i) and the queue job's
// (mpcb200_solve_stream).  `in`, `uprev_dt` and `has_lines` describe what load_inputs last put in them: the launches on these
// arrays read nothing else.
struct IoBuffers
{
    size_t rows = 0;     // instances the arrays hold
    int obst_m = 0;      // obstacles per instance the obstacle arrays hold
    double *x0 = nullptr, *xf = nullptr, *uprev = nullptr, *obst = nullptr, *vp = nullptr, *xinit = nullptr;
    int *obst_count = nullptr, *obst_type = nullptr, *vp_count = nullptr;
    unsigned char* reinit = nullptr;
    double *useq = nullptr, *xseq = nullptr, *dt = nullptr, *kkt = nullptr, *upacked = nullptr;
    int *status = nullptr, *iters = nullptr;
    InputPtrs in{};
    double uprev_dt = 0.0;
    int has_lines = 0;   // line obstacles, moving obstacles or midpoint differences: the kernel variants with those (rarely used) paths
    OutputPtrs out() const { return OutputPtrs{useq, xseq, dt, status, kkt, iters, upacked}; }
};

struct mpcb200_handle
{
    Cfg cfg{};
    WsLayout L{};
    int max_batch = 0, device = 0, B = 0;
    int n_cap = 0;                   // horizon the buffers were sized for at create (mpcb200_resample moves cfg.n within [3, n_cap])
    double* d_resample = nullptr;    // scratch of mpcb200_resample, allocated on first use
    void* d_cm = nullptr; size_t cm_cap = 0; double costmap_ms = 0.0;   // scratch of mpcb200_costmap_obstacles (grown on demand), device ms of its last call
    void* d_fz = nullptr; size_t fz_cap = 0;   // scratch of mpcb200_check_feasible (maps, trajectories, footprint, flags)
    double* ws = nullptr;
    int num_sms = 0, clock_khz = 0;
    int solve_mode = 0;              // MPCB200_OPT_SOLVE_MODE: 0 fused persistent kernel (default), 1 one kernel per phase
    unsigned timing_mask = 1u << MPCB200_PHASE_KKT;   // phased mode: phases bracketed by CUDA events inside solve (bit = phase id)
    cudaStream_t stream = nullptr, own_stream = nullptr;   // stream in use / the stream the handle created
    IoBuffers batch;                 // sized for max_batch at create
    IoBuffers queue;                 // the queue job's: inputs / outputs of the whole queue (grown on demand)
    int *d_nactive = nullptr, *d_queue = nullptr;
    unsigned long long* d_counters = nullptr;
    int* h_nactive = nullptr;        // pinned, two poll slots
    cudaEvent_t poll_ev[2] = {nullptr, nullptr}, t0 = nullptr, t1 = nullptr, c0 = nullptr, c1 = nullptr;   // t: around a solve, c: around the costmap kernels
    double* d_flush = nullptr; size_t flush_n = 0;
    int fused_grid = 0;              // CTAs of the last fused launch
    int order_by_history = 1;        // MPCB200_OPT_ORDER_BY_HISTORY: batch queue longest-first by the previous solve's iteration counts
    int critical_placement = 1;      // MPCB200_OPT_CRITICAL_PLACEMENT: the heaviest instances of a history order get SMs of their own
    int hist_B = 0;                  // batch size of the last batch solve whose iteration counts are in batch.iters (0: none)
    int *d_prev_iters = nullptr, *d_prev_status = nullptr, *d_order = nullptr;
    int* d_winner = nullptr;         // [max_batch] candidate index of each robot's winner (mpcb200_step_batch_multistart)
    int robot_limits_n = 0;          // records of per-robot limits in d_limits (0: none, the solves run solve_fused_kernel)
    double* d_limits = nullptr;      // [max_batch][MPCB200_LIMIT_WORDS]
    int robot_geometry_n = 0;        // records of per-robot geometry in d_geometry (0: none; > 0: the solves run solve_fused_fleet_kernel)
    double* d_geometry = nullptr;    // [max_batch][MPCB200_GEOMETRY_WORDS]
    int robot_weights_n = 0;         // records of per-robot weights in d_weights (0: none; > 0: the solves run solve_fused_weights_kernel)
    double* d_weights = nullptr;     // [max_batch][MPCB200_WEIGHT_WORDS]
    int robot_model_n = 0;           // records of per-robot models in d_model (0: none; > 0: the solves run solve_fused_models_kernel)
    double* d_model = nullptr;       // [max_batch][MPCB200_MODEL_WORDS]
    // host copies of the model and geometry records of the blocking setters, which check each kind against the other (empty, and
    // *_host false, after an async setter: the solve checks those pairs)
    std::vector<double> h_model, h_geometry;
    bool model_host = true, geometry_host = true;
    Cfg* d_robot_cfg = nullptr;      // [robot_cfg_slots] configuration of each CTA of a solve_fused_robot / _fleet / _weights / _models_kernel launch
    int robot_cfg_slots = 0;         // CTAs a solve launch can have: min(max_batch, 32 per SM)
    unsigned long long budget_ns = 0;          // max_cpu_time in ns (0: no budget)
    unsigned long long* d_origin = nullptr;    // start of the current solve launch (%globaltimer), see FusedArgs
    int sm_phase_sync = -1;          // MPCB200_OPT_SM_PHASE_SYNC: co-resident CTAs of the solve kernel enter the phases together
    unsigned long long* d_smsync = nullptr;
    int max_ctas_per_sm = 0;         // MPCB200_OPT_CTAS_PER_SM: cap on the resident CTAs per SM of the solve kernel (0 = what fits)
    int force_generic_model = 0;     // MPCB200_OPT_FORCE_GENERIC_MODEL: never launch the variants compiled for one robot / footprint model
    int last_model = MODEL_GENERIC;  // kernel key of the last solve launch (mpcb200_kernel_model / mpcb200_kernel_problem)
    mpcb200_stats stats{};
    std::vector<cudaEvent_t> ev;     // pool of event pairs
    std::vector<int> ev_phase;
    size_t ev_used = 0;
    std::string err;
};

static std::string g_create_err = "";

static int set_err(mpcb200_handle* h, int code, const std::string& msg)
{
    if (h) h->err = msg; else g_create_err = msg;
    return code;
}
#define CK(call)                                                                                                   \
    do {                                                                                                           \
        cudaError_t e_ = (call);                                                                                   \
        if (e_ != cudaSuccess)                                                                                     \
            return set_err(h, MPCB200_E_CUDA, std::string(#call) + ": " + cudaGetErrorString(e_));                 \
    } while (0)

extern "C" void mpcb200_default_config(mpcb200_config* c)
{
    memset(c, 0, sizeof(*c));
    c->robot_type = MPCB200_ROBOT_UNICYCLE;
    c->wheelbase = 0.5; c->length_rear = 1.0; c->length_front = 1.0;
    c->u_lb[0] = -0.2; c->u_lb[1] = -0.3; c->u_ub[0] = 0.4; c->u_ub[1] = 0.3;
    c->du_lb[0] = c->du_lb[1] = -MPCB200_INF; c->du_ub[0] = c->du_ub[1] = MPCB200_INF;
    c->n = 20; c->dt_ref = 0.3; c->variable_dt = 1; c->dt_lb = 0.0; c->dt_ub = 10.0;
    c->xf_fixed[0] = c->xf_fixed[1] = c->xf_fixed[2] = 1;
    c->collocation = MPCB200_COLLOC_FORWARD; c->warm_start = 1;
    c->objective = MPCB200_OBJ_MINIMUM_TIME;
    c->vp_position_weight = 1.0; c->vp_orientation_weight = 0.0;
    c->min_obstacle_dist = 0.5; c->force_inclusion_dist = 0.5; c->cutoff_dist = 2.0;
    c->footprint_type = MPCB200_FOOTPRINT_POINT;
    c->k_max_obstacles_per_stage = 5;
    c->max_iter = 100; c->tol = 1e-6; c->mu_init = 0.0; c->outer_iterations = 1; c->quadratic_integral_form = 0;
    c->initial_guess_bumps = 4;
    c->enable_dynamic_obstacles = 0;
    c->terminal_ball = 0; c->terminal_ball_gamma = 5.0;
    for (int i = 0; i < 9; ++i) c->terminal_ball_S[i] = (i % 4 == 0) ? 1.0 : 0.0;
    c->cost_integration = MPCB200_COST_LEFT_SUM;
    c->hybrid_cost_minimum_time = 0;
    c->max_cpu_time = -1.0;
}


// doubles of the resident prefix with the largest obstacle list the handle accepts
static size_t max_resident_bytes(const WsLayout& L) { return IMG_HEAD + (size_t)resident_words(L, L.M) * 8; }

static int validate_config(const mpcb200_config* c, std::string& why)
{
    if (c->n < 3 || c->n > 512) { why = "n must be in [3, 512]"; return MPCB200_E_INVALID; }
    if (c->robot_type < 0 || c->robot_type > 3) { why = "unknown robot_type"; return MPCB200_E_INVALID; }
    if (c->collocation != MPCB200_COLLOC_FORWARD && c->collocation != MPCB200_COLLOC_MIDPOINT)
    { why = "collocation: forward_differences and midpoint_differences are implemented, crank_nicolson is not"; return MPCB200_E_UNSUPPORTED; }
    if (c->objective < 0 || c->objective > 2) { why = "unknown objective"; return MPCB200_E_INVALID; }
    if (c->cost_integration != MPCB200_COST_LEFT_SUM && c->cost_integration != MPCB200_COST_TRAPEZOIDAL)
    { why = "unknown cost_integration"; return MPCB200_E_INVALID; }
    if (c->footprint_type < 0 || c->footprint_type > 4) { why = "unknown footprint_type"; return MPCB200_E_INVALID; }
    if (c->footprint_type == MPCB200_FOOTPRINT_POLYGON && (c->n_poly < 1 || c->n_poly > MPCB200_MAX_POLY))
    { why = "polygon footprint needs 1..16 vertices"; return MPCB200_E_INVALID; }
    if (c->k_max_obstacles_per_stage < 0 || c->k_max_obstacles_per_stage > 16) { why = "k_max_obstacles_per_stage must be in [0,16]"; return MPCB200_E_INVALID; }
    if (!(c->dt_ref > 0)) { why = "dt_ref must be > 0"; return MPCB200_E_INVALID; }
    if (c->variable_dt && !(c->dt_ub > c->dt_lb)) { why = "dt_ub must exceed dt_lb"; return MPCB200_E_INVALID; }
    if (has_mintime(*c) && !c->variable_dt) { why = "minimum_time objectives need variable_dt"; return MPCB200_E_INVALID; }
    if (!(c->tol > 0) || c->max_iter < 1) { why = "tol > 0 and max_iter >= 1 required"; return MPCB200_E_INVALID; }
    if (c->max_cpu_time != c->max_cpu_time) { why = "max_cpu_time is NaN (a budget in seconds; <= 0 or +inf: none)"; return MPCB200_E_INVALID; }
    for (int i = 0; i < 2; ++i)
        if (!(c->u_ub[i] > c->u_lb[i])) { why = "u_ub must exceed u_lb"; return MPCB200_E_INVALID; }
    // one CTA keeps the instance's resident prefix in shared memory: that bounds the horizon (about (56 + 6 RS + 4 K) N words)
    WsLayout L;
    make_layout(c, MAX_OBST, MAX_VP, L);
    if (max_resident_bytes(L) > MAX_IMG_SMEM)
    {
        why = "horizon too long for this row budget: the instance does not fit in shared memory (n = " + std::to_string(c->n) + " needs " +
              std::to_string(max_resident_bytes(L)) + " bytes of " + std::to_string((size_t)MAX_IMG_SMEM) + ")";
        return MPCB200_E_UNSUPPORTED;
    }
    return 0;
}

template <class K>
static cudaError_t allow_smem(K kernel) { return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, MAX_IMG_SMEM); }
#endif

// ---- the kernel variants: one table per kernel.  The variants compiled for one robot / footprint model (MODEL_UNI_POINT) exist
//      without the line-obstacle paths only (LINES = false); a request for one with them gets the generic variant.  The fixed-dt
//      quadratic-form key (MODEL_UNI_POINT_QF) exists for the unbordered KKT only (EXT = false). ----
//      The per-robot-limits entries (solve_fused_robot_kernel) form a second table of the same variants, the per-robot-geometry
//      entries (solve_fused_fleet_kernel) a third one of the MODEL_GENERIC variants, the per-robot-weights entries
//      (solve_fused_weights_kernel) a fourth one of all the variants, compiled in mpcb200_weights.cu (weights_kernel_variant).
struct FusedEntry
{
    template <bool LINES, bool EXT, int WARPS, int MODEL, bool MULTI> static constexpr auto get() { return solve_fused_kernel<LINES, EXT, WARPS, MODEL, MULTI>; }
};
struct RobotEntry
{
    template <bool LINES, bool EXT, int WARPS, int MODEL, bool MULTI> static constexpr auto get() { return solve_fused_robot_kernel<LINES, EXT, WARPS, MODEL, MULTI>; }
};
// the per-robot-geometry entries (solve_fused_fleet_kernel) exist for MODEL_GENERIC only: every key maps to it
struct FleetEntry
{
    template <bool LINES, bool EXT, int WARPS, int MODEL, bool MULTI> static constexpr auto get() { return solve_fused_fleet_kernel<LINES, EXT, WARPS, MODEL_GENERIC, MULTI>; }
};
template <class E> using EntryKernel = decltype(E::template get<false, false, SMALL_GROUP_WARPS, MODEL_GENERIC, false>());
template <class E, int WARPS, bool MULTI>
static EntryKernel<E> fused_shape_variant(bool lines, bool ext, int model)
{
    if (lines) return ext ? E::template get<true, true, WARPS, MODEL_GENERIC, MULTI>() : E::template get<true, false, WARPS, MODEL_GENERIC, MULTI>();
    if (model == MODEL_UNI_POINT_QF && !ext) return E::template get<false, false, WARPS, MODEL_UNI_POINT_QF, MULTI>();
    if (model == MODEL_UNI_POINT) return ext ? E::template get<false, true, WARPS, MODEL_UNI_POINT, MULTI>() : E::template get<false, false, WARPS, MODEL_UNI_POINT, MULTI>();
    return ext ? E::template get<false, true, WARPS, MODEL_GENERIC, MULTI>() : E::template get<false, false, WARPS, MODEL_GENERIC, MULTI>();
}
template <class E = FusedEntry>
static EntryKernel<E> fused_variant(bool lines, bool ext, bool small, int model, bool multi)
{
    if (multi) return small ? fused_shape_variant<E, SMALL_GROUP_WARPS, true>(lines, ext, model) : fused_shape_variant<E, MAX_GROUP_WARPS, true>(lines, ext, model);
    return small ? fused_shape_variant<E, SMALL_GROUP_WARPS, false>(lines, ext, model) : fused_shape_variant<E, MAX_GROUP_WARPS, false>(lines, ext, model);
}
// the per-robot-weights entry of a variant (mpcb200_weights.cu): its host function, for cudaFuncSetAttribute, the occupancy query
// and cudaLaunchKernel
const void* weights_kernel_variant(bool lines, bool ext, bool small, int model, bool multi);
// the per-robot-model entry of a variant (mpcb200_models.cu; MODEL_GENERIC only), for the same uses
const void* models_kernel_variant(bool lines, bool ext, bool small, bool multi);
#ifndef MPCB200_ENTRY_UNIT
using FusedKernel = EntryKernel<FusedEntry>;
using RobotKernel = EntryKernel<RobotEntry>;
using FleetKernel = EntryKernel<FleetEntry>;
using PhaseKernel = decltype(&phase_kernel<false, MODEL_GENERIC>);
static PhaseKernel phase_variant(bool lines, int model)
{
    if (lines) return phase_kernel<true, MODEL_GENERIC>;
    if (model == MODEL_UNI_POINT_QF) return phase_kernel<false, MODEL_UNI_POINT_QF>;
    return model == MODEL_UNI_POINT ? phase_kernel<false, MODEL_UNI_POINT> : phase_kernel<false, MODEL_GENERIC>;
}

// Where the arrays of a call live.  Host: the blocking calls copy them in and out and synchronise the stream.  Device: the
// _async calls copy device to device on the stream, read no array content on the host and do not wait.
enum class Mem { Host, Device };

// A buffer of the handle has to grow: allocating (and the synchronise before freeing) would end a CUDA graph capture on the
// handle's stream, so a call that needs it during a capture fails instead and asks for a warm-up.
static int check_growth_allowed(mpcb200_handle* h, const char* what)
{
    cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
    CK(cudaStreamIsCapturing(h->stream, &st));
    if (st != cudaStreamCaptureStatusNone)
        return set_err(h, MPCB200_E_INVALID, std::string(what) + " must grow while the stream is capturing a CUDA graph: make the same call "
                                             "once with the same shapes before the capture (warm-up)");
    return 0;
}

// The arrays a device-memory entry point takes must be device (or managed) memory of the handle's device: the kernels read the
// maps, footprints and trajectories in place, where a host pointer would be a fault rather than an error.  Null entries are the
// optional arrays the caller left out.
static int check_device_arrays(mpcb200_handle* h, const char* what, std::initializer_list<const void*> arrays)
{
    for (const void* p : arrays)
    {
        if (!p) continue;
        cudaPointerAttributes a{};
        if (cudaPointerGetAttributes(&a, p) != cudaSuccess)
        {
            cudaGetLastError();   // (not sticky; cleared so that no later check reports it)
            return set_err(h, MPCB200_E_INVALID, std::string(what) + ": an array pointer is not known to CUDA");
        }
        if ((a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) || a.device != h->device)
            return set_err(h, MPCB200_E_INVALID, std::string(what) + ": every array must be device memory of the handle's device (device " +
                                                 std::to_string(h->device) + ")");
    }
    return 0;
}

// frees the arrays of `io` and empties it (nothing held)
static void io_release(IoBuffers& io)
{
    void* arrays[] = {io.x0, io.xf, io.uprev, io.obst, io.vp, io.xinit, io.obst_count, io.obst_type, io.vp_count, io.reinit,
                      io.useq, io.xseq, io.dt, io.kkt, io.upacked, io.status, io.iters};
    for (void* p : arrays) cudaFree(p);   // (no-op for the null ones)
    io = IoBuffers{};
}
// Grows `io` to hold `rows` instances and `obst_per_instance` obstacles per instance (at least MAX_OBST: longer lists get arrays
// of their length on first use).  Only the obstacle arrays move when only the obstacle list grows, so the outputs of the last
// solve stay where they are.  Rows are sized for the largest horizon the handle can be resampled to.  x_init / reinit: the
// batch only (the queue's instances start cold).
static int io_reserve(mpcb200_handle* h, IoBuffers& io, size_t rows, int obst_per_instance)
{
    const int m = (obst_per_instance > MAX_OBST && obst_per_instance <= MAX_OBST_LIST) ? obst_per_instance : MAX_OBST;
    if (rows <= io.rows && m <= io.obst_m) return 0;
    if (int rc = check_growth_allowed(h, "the staging arrays")) return rc;
    CK(cudaStreamSynchronize(h->stream));   // work queued on the stream may still read the arrays
    if (rows > io.rows)
    {
        io_release(io);
        const size_t T = rows, N = (size_t)h->n_cap;
        CK(cudaMalloc(&io.x0, T * 3 * 8)); CK(cudaMalloc(&io.xf, T * 3 * 8)); CK(cudaMalloc(&io.uprev, T * 2 * 8));
        CK(cudaMalloc(&io.obst_count, T * 4)); CK(cudaMalloc(&io.vp, T * MAX_VP * 3 * 8)); CK(cudaMalloc(&io.vp_count, T * 4));
        if (&io == &h->batch) { CK(cudaMalloc(&io.xinit, T * N * 3 * 8)); CK(cudaMalloc(&io.reinit, T)); }
        CK(cudaMalloc(&io.useq, T * N * 2 * 8)); CK(cudaMalloc(&io.xseq, T * N * 3 * 8)); CK(cudaMalloc(&io.dt, T * 8));
        CK(cudaMalloc(&io.kkt, T * 8)); CK(cudaMalloc(&io.upacked, T * (N - 1) * 2 * 8));
        CK(cudaMalloc(&io.status, T * 4)); CK(cudaMalloc(&io.iters, T * 4));
        io.rows = rows;
    }
    if (m > io.obst_m)
    {
        cudaFree(io.obst); cudaFree(io.obst_type);
        io.obst = nullptr; io.obst_type = nullptr; io.obst_m = 0;
        CK(cudaMalloc(&io.obst, io.rows * m * MPCB200_OBST_STRIDE * 8));
        CK(cudaMalloc(&io.obst_type, io.rows * m * 4));
        io.obst_m = m;
    }
    return 0;
}

extern "C" int mpcb200_create(const mpcb200_config* cfg, int max_batch, int device, mpcb200_handle** out)
{
    mpcb200_handle* h = nullptr;
    if (!cfg || !out || max_batch < 1) return set_err(nullptr, MPCB200_E_INVALID, "bad arguments");
    std::string why;
    int rc = validate_config(cfg, why);
    if (rc) return set_err(nullptr, rc, why);
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return set_err(nullptr, MPCB200_E_NODEVICE, std::string("no CUDA device (") + cudaGetErrorString(e) + "): this solver has no CPU fallback");
    if (device < 0 || device >= ndev) return set_err(nullptr, MPCB200_E_INVALID, "device index out of range");
    h = new mpcb200_handle();
    h->cfg = *cfg; h->max_batch = max_batch; h->device = device; h->n_cap = cfg->n;
    make_layout(cfg, MAX_OBST, MAX_VP, h->L);
    // seconds -> ns, rounded up; a budget beyond 2^62 ns (146 years) is no budget
    h->budget_ns = (cfg->max_cpu_time > 0.0 && cfg->max_cpu_time * 1e9 < 4611686018427387904.0) ? (unsigned long long)ceil(cfg->max_cpu_time * 1e9) : 0ull;
#define CKC(call)                                                                                                  \
    do {                                                                                                           \
        cudaError_t e_ = (call);                                                                                   \
        if (e_ != cudaSuccess) { std::string m = std::string(#call) + ": " + cudaGetErrorString(e_); mpcb200_destroy(h); return set_err(nullptr, MPCB200_E_CUDA, m); } \
    } while (0)
    CKC(cudaSetDevice(device));
    CKC(cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
    h->stream = h->own_stream;
    const size_t B = (size_t)max_batch;
    CKC(cudaMalloc(&h->ws, B * h->L.stride * sizeof(double)));
    CKC(cudaMemsetAsync(h->ws, 0, B * h->L.stride * sizeof(double), h->stream));
    CKC(cudaDeviceGetAttribute(&h->num_sms, cudaDevAttrMultiProcessorCount, device));
    CKC(cudaDeviceGetAttribute(&h->clock_khz, cudaDevAttrClockRate, device));
    if (io_reserve(h, h->batch, B, 0))
    {
        const std::string m = h->err;
        mpcb200_destroy(h);
        return set_err(nullptr, MPCB200_E_CUDA, m);
    }
    CKC(cudaMalloc(&h->d_nactive, 8)); CKC(cudaMalloc(&h->d_queue, 4)); CKC(cudaMalloc(&h->d_smsync, (size_t)h->num_sms * SMS_WORD_STRIDE * 8)); CKC(cudaMalloc(&h->d_prev_iters, B * 4)); CKC(cudaMalloc(&h->d_prev_status, B * 4)); CKC(cudaMalloc(&h->d_order, (B + 2) * 4));
    CKC(cudaMalloc(&h->d_origin, 8)); CKC(cudaMalloc(&h->d_winner, B * 4));
    h->robot_cfg_slots = max_batch < 32 * h->num_sms ? max_batch : 32 * h->num_sms;
    CKC(cudaMalloc(&h->d_limits, B * MPCB200_LIMIT_WORDS * 8)); CKC(cudaMalloc(&h->d_robot_cfg, (size_t)h->robot_cfg_slots * sizeof(Cfg)));
    CKC(cudaMalloc(&h->d_geometry, B * MPCB200_GEOMETRY_WORDS * 8));
    CKC(cudaMalloc(&h->d_weights, B * MPCB200_WEIGHT_WORDS * 8));
    CKC(cudaMalloc(&h->d_model, B * MPCB200_MODEL_WORDS * 8));
    CKC(cudaMalloc(&h->d_counters, CNT_BYTES)); CKC(cudaMemsetAsync(h->d_counters, 0, CNT_BYTES, h->stream));
    CKC(allow_smem(kkt_warp_kernel<false>)); CKC(allow_smem(kkt_warp_kernel<true>));
    for (const bool lines : {false, true})
        for (const int model : {MODEL_GENERIC, MODEL_UNI_POINT, MODEL_UNI_POINT_QF})
        {
            CKC(allow_smem(phase_variant(lines, model)));
            for (const bool ext : {false, true})
                for (const bool small : {false, true})
                    for (const bool multi : {false, true})
                    {
                        CKC(allow_smem(fused_variant(lines, ext, small, model, multi)));
                        CKC(allow_smem(fused_variant<RobotEntry>(lines, ext, small, model, multi)));
                        if (model == MODEL_GENERIC) CKC(allow_smem(fused_variant<FleetEntry>(lines, ext, small, model, multi)));
                        CKC(allow_smem(weights_kernel_variant(lines, ext, small, model, multi)));
                        if (model == MODEL_GENERIC) CKC(allow_smem(models_kernel_variant(lines, ext, small, multi)));
                    }
        }
    CKC(cudaMallocHost(&h->h_nactive, 8));
    CKC(cudaEventCreateWithFlags(&h->poll_ev[0], cudaEventDisableTiming)); CKC(cudaEventCreateWithFlags(&h->poll_ev[1], cudaEventDisableTiming));
    CKC(cudaEventCreate(&h->t0)); CKC(cudaEventCreate(&h->t1)); CKC(cudaEventCreate(&h->c0)); CKC(cudaEventCreate(&h->c1));
    int l2_bytes = 0;
    CKC(cudaDeviceGetAttribute(&l2_bytes, cudaDevAttrL2CacheSize, device));
    h->flush_n = (size_t)l2_bytes * 3 / 8;  // doubles: three times the L2 (150 MB on an H100's 50 MB)
    CKC(cudaMalloc(&h->d_flush, h->flush_n * 8));
    CKC(cudaMemsetAsync(h->d_flush, 0, h->flush_n * 8, h->stream));
    {
        // all instances start cold
        reset_kernel<<<(max_batch + 127) / 128, 128, 0, h->stream>>>(h->L, h->ws, max_batch, nullptr);
        CKC(cudaGetLastError());
    }
    CKC(cudaStreamSynchronize(h->stream));
    *out = h;
    return MPCB200_OK;
}

extern "C" void mpcb200_destroy(mpcb200_handle* h)
{
    if (!h) return;
    // (also the failure path of mpcb200_create: whatever was not created yet is null)
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    io_release(h->batch);
    io_release(h->queue);
    void* ptrs[] = {h->ws, h->d_nactive, h->d_queue, h->d_flush, h->d_counters, h->d_smsync, h->d_prev_iters, h->d_prev_status, h->d_order,
                    h->d_origin, h->d_winner, h->d_resample, h->d_cm, h->d_fz, h->d_limits, h->d_robot_cfg,
                    h->d_geometry, h->d_weights, h->d_model};
    for (void* p : ptrs) if (p) cudaFree(p);
    if (h->h_nactive) cudaFreeHost(h->h_nactive);
    for (auto& e : h->ev) cudaEventDestroy(e);
    for (cudaEvent_t e : {h->poll_ev[0], h->poll_ev[1], h->t0, h->t1, h->c0, h->c1}) if (e) cudaEventDestroy(e);
    if (h->own_stream) cudaStreamDestroy(h->own_stream);
    delete h;
}

extern "C" const char* mpcb200_last_error(const mpcb200_handle* h) { return h ? h->err.c_str() : g_create_err.c_str(); }

static inline int grid_for(int B, int wpc) { return (B + wpc - 1) / wpc; }

// event-pair pool: device time per phase launch (CUDA events on the solver stream)
static int ev_begin(mpcb200_handle* h, int phase)
{
    if (h->ev_used + 2 > h->ev.size())
    {
        for (int i = 0; i < 256; ++i) { cudaEvent_t e; if (cudaEventCreate(&e) != cudaSuccess) return -1; h->ev.push_back(e); }
        h->ev_phase.resize(h->ev.size() / 2);
    }
    h->ev_phase[h->ev_used / 2] = phase;
    cudaEventRecord(h->ev[h->ev_used], h->stream);
    return 0;
}
static void ev_end(mpcb200_handle* h)
{
    cudaEventRecord(h->ev[h->ev_used + 1], h->stream);
    h->ev_used += 2;
}
static void ev_collect(mpcb200_handle* h)
{
    for (size_t i = 0; i + 1 < h->ev_used; i += 2)
    {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, h->ev[i], h->ev[i + 1]) == cudaSuccess)
        {
            const int p = h->ev_phase[i / 2];
            h->stats.ms[p] += ms; h->stats.launches[p] += 1;
        }
    }
    h->ev_used = 0;
}

// threads of the CTA that owns an instance
static int group_threads(const mpcb200_handle* h)
{
    const int gw = (h->cfg.n + 31) / 32;
    return 32 * (gw < MAX_GROUP_WARPS ? gw : MAX_GROUP_WARPS);   // a lane per stage
}
// robot model / footprint / problem key of the evaluation and line-search code a launch runs (ModelTraits).  The specialised variants
// exist for the kernels without the rarely used obstacle paths only (LINES = false).
static int kernel_model(const mpcb200_handle* h, const IoBuffers& io)
{
    if (io.has_lines || h->force_generic_model || h->robot_model_n > 0) return MODEL_GENERIC;   // (model records: types per robot)
    if (qf_key_matches(h->cfg)) return MODEL_UNI_POINT_QF;
    const bool uni_point = h->cfg.robot_type == MPCB200_ROBOT_UNICYCLE && h->cfg.footprint_type == MPCB200_FOOTPRINT_POINT;
    return uni_point ? MODEL_UNI_POINT : MODEL_GENERIC;
}
static int image_words(const mpcb200_handle* h, const InputPtrs& in)
{
    return resident_words(h->L, in.obst_count ? (in.obst_max < h->L.M ? in.obst_max : h->L.M) : 0);
}

// one phase kernel over the instance blocks of the batch
static int launch_phase(mpcb200_handle* h, int phase, int B, int force_cold, int first_outer, int* n_active, bool timed)
{
    const IoBuffers& io = h->batch;
    const int img_words = image_words(h, io.in);
    const size_t img_smem = IMG_HEAD + (size_t)img_words * 8;
    if (img_smem > MAX_IMG_SMEM) return set_err(h, MPCB200_E_UNSUPPORTED, "the instance does not fit in shared memory");
    if (timed && ev_begin(h, phase)) return set_err(h, MPCB200_E_CUDA, "cudaEventCreate failed");
    if (phase == MPCB200_PHASE_KKT)
    {
        if (kkt_is_ext(h->cfg)) kkt_warp_kernel<true><<<B, 32, kkt_smem_bytes<true>(h->cfg.n), h->stream>>>(h->cfg, h->L, h->ws, B, h->d_counters);
        else kkt_warp_kernel<false><<<B, 32, kkt_smem_bytes<false>(h->cfg.n), h->stream>>>(h->cfg, h->L, h->ws, B, h->d_counters);
    }
    else if (phase >= 0 && phase < MPCB200_NUM_PHASES)
    {
        const int model = kernel_model(h, io);
        phase_variant(io.has_lines, model)<<<B, group_threads(h), img_smem, h->stream>>>(h->cfg, h->L, h->ws, B, phase, io.uprev_dt, force_cold,
                                                                                         first_outer, n_active, img_words, io.in);
        h->last_model = model;
    }
    else return set_err(h, MPCB200_E_INVALID, "unknown phase");
    if (timed) ev_end(h);
    h->stats.launches_total += 1;
    CK(cudaGetLastError());
    return 0;
}

static int check_batch(mpcb200_handle* h, int B)
{
    if (!h) return MPCB200_E_INVALID;
    if (B < 1 || B > h->max_batch) return set_err(h, MPCB200_E_INVALID, "batch size out of range");
    return 0;
}

// line obstacles among the obstacles in use (padding slots are never read)
static bool has_line_obstacles(size_t B, const mpcb200_obstacles* obst)
{
    const size_t M = (size_t)obst->max_per_instance;
    for (size_t b = 0; b < B; ++b)
    {
        const int cnt = obst->count[b] < (int)M ? obst->count[b] : (int)M;
        for (int i = 0; i < cnt; ++i)
            if (obst->type[b * M + i] == MPCB200_OBST_LINE) return true;
    }
    return false;
}

// copies of the inputs of `B` instances into `io` (host -> device, or device -> device: `mem`), and the description of what it now
// holds (io.in, io.uprev_dt, io.has_lines).  The arguments are checked before anything is copied.  The line-obstacle kernel
// variant follows the configuration and the obstacle types: scanned on the host for host arrays, declared by the caller
// (`flags & MPCB200_ASYNC_LINE_OBSTACLES`) for device arrays.  h2d_bytes counts the host copies only.
static int load_inputs(mpcb200_handle* h, IoBuffers& io, int B, const double* x0, const double* xf, const double* u_prev, double u_prev_dt,
                       const mpcb200_obstacles* obst, const mpcb200_viapoints* vp, const double* x_init, const unsigned char* reinit,
                       Mem mem = Mem::Host, unsigned flags = 0u)
{
    const cudaMemcpyKind kind = mem == Mem::Host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice;
    const long long counted = mem == Mem::Host ? 1 : 0;
    if (!x0 || !xf) return set_err(h, MPCB200_E_INVALID, "x0 and xf are required");
    const bool with_obst = obst && obst->count && obst->max_per_instance > 0, with_vp = vp && vp->count && vp->max_per_instance > 0;
    if (with_obst && obst->max_per_instance > MAX_OBST_LIST) return set_err(h, MPCB200_E_UNSUPPORTED, "more than 2048 obstacles per instance");
    if (with_obst && (!obst->type || !obst->params)) return set_err(h, MPCB200_E_INVALID, "obstacle types and parameters are required");
    if (with_vp && vp->max_per_instance > MAX_VP) return set_err(h, MPCB200_E_UNSUPPORTED, "more than 8 via-points per instance");
    if (int rc = io_reserve(h, io, io.rows, with_obst ? obst->max_per_instance : 0)) return rc;
    const size_t n = (size_t)B, N = (size_t)h->cfg.n;
    InputPtrs in{io.x0, io.xf, io.uprev, nullptr, io.obst_type, io.obst, 0, nullptr, io.vp, 0, nullptr, nullptr};
    if (u_prev) { CK(cudaMemcpyAsync(io.uprev, u_prev, n * 2 * 8, kind, h->stream)); h->stats.h2d_bytes += counted * (long long)(n * 16); }
    else CK(cudaMemsetAsync(io.uprev, 0, n * 2 * 8, h->stream));
    CK(cudaMemcpyAsync(io.x0, x0, n * 3 * 8, kind, h->stream));
    CK(cudaMemcpyAsync(io.xf, xf, n * 3 * 8, kind, h->stream));
    h->stats.h2d_bytes += counted * (long long)(n * 6 * 8);
    bool lines = is_midpoint(h->cfg);
    if (with_obst)
    {
        const size_t M = (size_t)obst->max_per_instance;
        CK(cudaMemcpyAsync(io.obst_count, obst->count, n * 4, kind, h->stream));
        CK(cudaMemcpyAsync(io.obst_type, obst->type, n * M * 4, kind, h->stream));
        CK(cudaMemcpyAsync(io.obst, obst->params, n * M * MPCB200_OBST_STRIDE * 8, kind, h->stream));
        h->stats.h2d_bytes += counted * (long long)(n * 4 + n * M * 4 + n * M * MPCB200_OBST_STRIDE * 8);
        in.obst_count = io.obst_count; in.obst_max = (int)M;
        const bool line_obstacles = mem == Mem::Host ? has_line_obstacles(n, obst) : (flags & MPCB200_ASYNC_LINE_OBSTACLES) != 0u;
        lines = lines || h->cfg.enable_dynamic_obstacles || line_obstacles;
    }
    if (with_vp)
    {
        const size_t V = (size_t)vp->max_per_instance;
        CK(cudaMemcpyAsync(io.vp_count, vp->count, n * 4, kind, h->stream));
        CK(cudaMemcpyAsync(io.vp, vp->poses, n * V * 3 * 8, kind, h->stream));
        h->stats.h2d_bytes += counted * (long long)(n * 4 + n * V * 24);
        in.vp_count = io.vp_count; in.vp_max = (int)V;
    }
    if (x_init && io.xinit) { CK(cudaMemcpyAsync(io.xinit, x_init, n * N * 3 * 8, kind, h->stream)); in.x_init = io.xinit; h->stats.h2d_bytes += counted * (long long)(n * N * 24); }
    if (reinit && io.reinit) { CK(cudaMemcpyAsync(io.reinit, reinit, n, kind, h->stream)); in.reinit = io.reinit; h->stats.h2d_bytes += counted * (long long)n; }
    io.in = in;
    io.uprev_dt = u_prev_dt;
    io.has_lines = lines;
    return 0;
}

// the batch's inputs into the instance blocks as well: the kernel-level API and the phased solve work on the blocks
static int scatter_to_blocks(mpcb200_handle* h, int B)
{
    scatter_inputs_kernel<<<grid_for(B, WARPS_PER_CTA), WARPS_PER_CTA * 32, 0, h->stream>>>(h->L, h->ws, B, h->batch.in);
    h->stats.launches_total += 1;
    CK(cudaGetLastError());
    return 0;
}

// ---- the solve: one launch of the persistent kernel over a queue of `total` instances ----
static int launch_fused(mpcb200_handle* h, const IoBuffers& io, int total, int queue_mode, int force_cold, int cand_stride = 0 /* multistart: B */)
{
    FusedArgs a;
    a.ws = h->ws; a.in = io.in; a.out = io.out(); a.total = total; a.queue_mode = queue_mode; a.force_cold = force_cold; a.uprev_dt = io.uprev_dt;
    a.cand_stride = cand_stride;
    a.img_words = image_words(h, io.in); a.queue = h->d_queue; a.counters = h->d_counters;
    a.sm_sync = nullptr; a.sm_words = 0; a.sm_gates = h->sm_phase_sync == 2 ? 2 : 3;
    a.order = nullptr; a.place = nullptr; a.place_sm = nullptr; a.place_cotenants = PLACE_COTENANTS;
    a.budget_ns = h->budget_ns; a.origin = h->d_origin;
    if (h->budget_ns) CK(cudaMemsetAsync(h->d_origin, 0, 8, h->stream));
    const size_t smem = IMG_HEAD + (size_t)a.img_words * 8;
    if (smem > MAX_IMG_SMEM) return set_err(h, MPCB200_E_UNSUPPORTED, "the instance does not fit in shared memory");
    const int threads = group_threads(h), model = kernel_model(h, io);
    const bool ext = kkt_is_ext(h->cfg), small = threads <= SMALL_GROUP_WARPS * 32, robot = h->robot_limits_n > 0 && !queue_mode;
    // geometry records: the fleet entry, which applies the limits records too when there are any
    const bool geometry = h->robot_geometry_n > 0 && !queue_mode;
    if (geometry && model != MODEL_GENERIC) return set_err(h, MPCB200_E_UNSUPPORTED, "per-robot geometry needs the generic kernel variant");
    // model records: the models entry, which applies the limits, geometry and weights records too when there are any (the model
    // records make the key MODEL_GENERIC, kernel_model); else weights records: the weights entry, which applies the limits and
    // geometry records too when there are any
    const bool models = h->robot_model_n > 0 && !queue_mode;
    const bool weights = h->robot_weights_n > 0 && !queue_mode && !models, fleet = geometry && !weights && !models;
    const bool per_robot = robot || geometry || weights || models;
    const FusedKernel kernel = per_robot ? nullptr : fused_variant(io.has_lines, ext, small, model, cand_stride > 0);
    const RobotKernel robot_kernel = robot && !geometry && !weights && !models ? fused_variant<RobotEntry>(io.has_lines, ext, small, model, cand_stride > 0) : nullptr;
    const FleetKernel fleet_kernel = fleet ? fused_variant<FleetEntry>(io.has_lines, ext, small, model, cand_stride > 0) : nullptr;
    const void* weights_kernel = weights ? weights_kernel_variant(io.has_lines, ext, small, model, cand_stride > 0) : nullptr;
    const void* models_kernel = models ? models_kernel_variant(io.has_lines, ext, small, cand_stride > 0) : nullptr;
    int per_sm = 0;
    if (models) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, models_kernel, threads, smem));
    else if (weights) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, weights_kernel, threads, smem));
    else if (fleet) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fleet_kernel, threads, smem));
    else if (robot) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, robot_kernel, threads, smem));
    else CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem));
    if (per_sm < 1) return set_err(h, MPCB200_E_UNSUPPORTED, "the solve kernel does not fit on an SM with this configuration");
    if (h->max_ctas_per_sm > 0 && per_sm > h->max_ctas_per_sm) per_sm = h->max_ctas_per_sm;
    const int grid = total < per_sm * h->num_sms ? total : per_sm * h->num_sms;
    if (per_robot && grid > h->robot_cfg_slots) return set_err(h, MPCB200_E_UNSUPPORTED, "more CTAs than per-robot configuration slots");
    h->fused_grid = grid;
    CK(cudaMemsetAsync(h->d_queue, 0, 4, h->stream));
    if (!queue_mode && h->order_by_history && h->hist_B == total && total > h->num_sms)
    {
        // The critical placement needs SMs that a heavy instance could share, and a batch of at most two instances per CTA slot:
        // with more, the heavy part is empty or nearly so (its threshold is 1.3 x the mean count per slot), and the placed
        // launch measured 2-3 % slower there (cfg 4 at B = 16 384, cfg 5 at B = 2048; H100, DESIGN.md 4).
        const bool placing = h->critical_placement && per_sm >= 2 && total <= 2 * grid;
        if (placing) { a.place = h->d_order + total; a.place_sm = h->d_smsync + 1; a.sm_words = h->num_sms; }
        // (the iteration counts and statuses are rewritten by this solve: order from copies)
        CK(cudaMemcpyAsync(h->d_prev_iters, io.iters, (size_t)total * 4, cudaMemcpyDeviceToDevice, h->stream));
        CK(cudaMemcpyAsync(h->d_prev_status, io.status, (size_t)total * 4, cudaMemcpyDeviceToDevice, h->stream));
        order_by_history_kernel<<<1, 1024, 0, h->stream>>>(h->d_prev_iters, h->d_prev_status, h->cfg.max_iter, total, h->d_order,
                                                            a.place, grid, PLACE_RHO, h->num_sms, h->d_queue);
        h->stats.launches_total += 1;
        a.order = h->d_order;
    }
    if (!queue_mode) h->hist_B = total;
    // phase alignment pays when several CTAs share an SM (auto: from three CTAs per SM)
    if (h->sm_phase_sync > 0 || (h->sm_phase_sync < 0 && per_sm >= 3 && grid > h->num_sms)) { a.sm_sync = h->d_smsync; a.sm_words = h->num_sms; }
    if (a.sm_sync || a.place) CK(cudaMemsetAsync(h->d_smsync, 0, (size_t)h->num_sms * SMS_WORD_STRIDE * 8, h->stream));
    if (models)
    {
        RobotArgs ra{robot ? h->d_limits : nullptr, h->d_robot_cfg};
        const double *geo = geometry ? h->d_geometry : nullptr, *wgt = h->robot_weights_n > 0 ? h->d_weights : nullptr, *mdl = h->d_model;
        void* args[] = {&h->cfg, &h->L, &a, &ra, &geo, &wgt, &mdl};
        CK(cudaLaunchKernel(models_kernel, dim3(grid), dim3(threads), args, smem, h->stream));
    }
    else if (weights)
    {
        RobotArgs ra{robot ? h->d_limits : nullptr, h->d_robot_cfg};
        const double *geo = geometry ? h->d_geometry : nullptr, *wgt = h->d_weights;
        void* args[] = {&h->cfg, &h->L, &a, &ra, &geo, &wgt};
        CK(cudaLaunchKernel(weights_kernel, dim3(grid), dim3(threads), args, smem, h->stream));
    }
    else if (fleet)
        fleet_kernel<<<grid, threads, smem, h->stream>>>(h->cfg, h->L, a, RobotArgs{robot ? h->d_limits : nullptr, h->d_robot_cfg}, h->d_geometry);
    else if (robot) robot_kernel<<<grid, threads, smem, h->stream>>>(h->cfg, h->L, a, RobotArgs{h->d_limits, h->d_robot_cfg});
    else kernel<<<grid, threads, smem, h->stream>>>(h->cfg, h->L, a);
    h->last_model = model;
    h->stats.launches_total += 1;
    CK(cudaGetLastError());
    return 0;
}

// the phased form of the same solve (MPCB200_OPT_SOLVE_MODE 1): one kernel per phase, the host queues the iterations
static int solve_phased(mpcb200_handle* h, int B, int force_cold)
{
    const unsigned tm = h->timing_mask;
    auto timed = [&](int phase) { return ((tm >> phase) & 1u) != 0; };
    int rc = launch_phase(h, MPCB200_PHASE_INIT, B, force_cold, 0, nullptr, timed(MPCB200_PHASE_INIT));
    if (rc) return rc;
    const int outer = h->cfg.outer_iterations > 0 ? h->cfg.outer_iterations : 1;
    for (int oi = 0; oi < outer; ++oi)
    {
        if ((rc = launch_phase(h, MPCB200_PHASE_ASSOCIATE, B, 0, oi == 0, nullptr, timed(MPCB200_PHASE_ASSOCIATE)))) return rc;
        // The number of unfinished instances is polled every POLL iterations, one poll behind: the host keeps queueing
        // iterations while the count of the previous poll travels back (a finished instance makes every kernel a no-op).
        const int POLL = 4;
        int pending = -1;  // slot of the poll in flight
        bool done = false;
        for (int it = 0; it <= h->cfg.max_iter && !done; ++it)
        {
            const bool poll = (it % POLL == POLL - 1) || it == h->cfg.max_iter;
            const int slot = (it / POLL) & 1;
            if (poll) CK(cudaMemsetAsync(h->d_nactive + slot, 0, 4, h->stream));
            if ((rc = launch_phase(h, MPCB200_PHASE_EVAL, B, 0, 0, poll ? h->d_nactive + slot : nullptr, timed(MPCB200_PHASE_EVAL)))) return rc;
            if (poll)
            {
                CK(cudaMemcpyAsync(h->h_nactive + slot, h->d_nactive + slot, 4, cudaMemcpyDeviceToHost, h->stream));
                CK(cudaEventRecord(h->poll_ev[slot], h->stream));
                if (pending >= 0)
                {
                    CK(cudaEventSynchronize(h->poll_ev[pending]));
                    if (h->h_nactive[pending] == 0) done = true;
                }
                pending = slot;
            }
            if (it == h->cfg.max_iter || done) break;
            if ((rc = launch_phase(h, MPCB200_PHASE_KKT, B, 0, 0, nullptr, timed(MPCB200_PHASE_KKT)))) return rc;
            if ((rc = launch_phase(h, MPCB200_PHASE_LINESEARCH, B, 0, 0, nullptr, timed(MPCB200_PHASE_LINESEARCH)))) return rc;
        }
    }
    gather_outputs_kernel<<<grid_for(B, WARPS_PER_CTA), WARPS_PER_CTA * 32, 0, h->stream>>>(h->L, h->ws, B, h->batch.out());
    h->stats.launches_total += 1;
    CK(cudaGetLastError());
    return 0;
}

// fold the cycle counters of the fused kernel into the per-phase statistics: average time a CTA spent in each phase.  The raw
// counters hold the launches since the last fold, all of the grid h->fused_grid (a blocking solve folds its own launch); the
// device-memory solves have folded theirs on the device already.
static int collect_fused_counters(mpcb200_handle* h)
{
    unsigned long long cnt[2 * CNT_WORDS];
    static_assert(sizeof(cnt) == CNT_BYTES, "raw counters + folded counters");
    CK(cudaMemcpy(cnt, h->d_counters, sizeof(cnt), cudaMemcpyDeviceToHost));
    double fold[CNT_WORDS];
    memcpy(fold, cnt + CNT_WORDS, sizeof(fold));
    const double per_cta = h->fused_grid > 0 ? 1.0 / ((double)h->fused_grid * (double)h->clock_khz) : 0.0;  // cycles -> ms per CTA
    const double to_ms = 1.0 / (double)h->clock_khz;
    for (int p = 0; p < MPCB200_NUM_PHASES; ++p) h->stats.ms[p] += (double)cnt[CNT_CYC + p] * per_cta + fold[CNT_CYC + p] * to_ms;
    h->stats.gate_ms += (double)cnt[CNT_GATE] * per_cta + fold[CNT_GATE] * to_ms;
    h->stats.kkt_instances += (long long)cnt[CNT_KKT_INST] + (long long)fold[CNT_KKT_INST];
    h->stats.kkt_sweeps += (long long)cnt[CNT_KKT_SWEEPS] + (long long)fold[CNT_KKT_SWEEPS];
    h->stats.launches[MPCB200_PHASE_KKT] += (long long)cnt[CNT_KKT_INST] + (long long)fold[CNT_KKT_INST];
    CK(cudaMemsetAsync(h->d_counters, 0, sizeof(cnt), h->stream));
    return 0;
}

// the phased mode queues the iterations from the host: its launches do not share the solve kernel's clock
static int check_budget_mode(mpcb200_handle* h)
{
    if (h->budget_ns && h->solve_mode == 1)
        return set_err(h, MPCB200_E_UNSUPPORTED, "max_cpu_time (a time budget) needs the fused solve kernel: MPCB200_OPT_SOLVE_MODE 1 "
                                                 "(one launch per phase) has no budget; set the option to 0 or max_cpu_time to -1");
    return 0;
}

// With per-robot limits, geometry or weights set, a solve of `robots` robots needs a record of each kind set for each, and the
// persistent kernel (the phased mode has no per-robot form).  Checked before anything is enqueued.
static int check_robot_limits(mpcb200_handle* h, int robots)
{
    if (h->robot_limits_n == 0 && h->robot_geometry_n == 0 && h->robot_weights_n == 0 && h->robot_model_n == 0) return 0;
    if (h->solve_mode == 1)
        return set_err(h, MPCB200_E_UNSUPPORTED, std::string(h->robot_limits_n > 0 ? "per-robot limits need" :
                                                             h->robot_geometry_n > 0 ? "per-robot geometry needs" :
                                                             h->robot_weights_n > 0 ? "per-robot weights need" : "per-robot models need") +
                                                 " the fused solve kernel (MPCB200_OPT_SOLVE_MODE 0)");
    if (h->robot_limits_n > 0 && robots > h->robot_limits_n)
        return set_err(h, MPCB200_E_INVALID, "per-robot limits: " + std::to_string(robots) + " robots, " + std::to_string(h->robot_limits_n) +
                                             " records (mpcb200_set_robot_limits)");
    if (h->robot_geometry_n > 0 && robots > h->robot_geometry_n)
        return set_err(h, MPCB200_E_INVALID, "per-robot geometry: " + std::to_string(robots) + " robots, " + std::to_string(h->robot_geometry_n) +
                                             " records (mpcb200_set_robot_geometry)");
    if (h->robot_weights_n > 0 && robots > h->robot_weights_n)
        return set_err(h, MPCB200_E_INVALID, "per-robot weights: " + std::to_string(robots) + " robots, " + std::to_string(h->robot_weights_n) +
                                             " records (mpcb200_set_robot_weights)");
    if (h->robot_model_n > 0 && robots > h->robot_model_n)
        return set_err(h, MPCB200_E_INVALID, "per-robot models: " + std::to_string(robots) + " robots, " + std::to_string(h->robot_model_n) +
                                             " records (mpcb200_set_robot_model)");
    return 0;
}

// The solve of a batch on the device arrays: one launch of the persistent kernel.  Without a host synchronise behind it (the
// device-memory calls), its counters are folded on the device with the launch's own grid.
static int launch_solve_async(mpcb200_handle* h, const IoBuffers& io, int total)
{
    if (int rc = launch_fused(h, io, total, 0, 0)) return rc;
    fold_counters_kernel<<<1, CNT_WORDS, 0, h->stream>>>(h->d_counters, h->fused_grid);
    h->stats.launches_total += 1;
    CK(cudaGetLastError());
    return 0;
}

// the K candidates per robot of a multistart solve (mpcb200_step_batch_multistart)
struct Multistart { int B, K; double hysteresis; };

// One solve between the events t0 and t1: the batch (fused or phased, by the solve mode), a multistart batch (fused, then the
// selection) or the queue job (always fused).  Reports the device time of the solve and folds the counters of the fused kernel
// into the statistics.
static int timed_launch(mpcb200_handle* h, const IoBuffers& io, int total, int queue_mode, int force_cold, double* solve_time_s,
                        const Multistart* multi = nullptr)
{
    CK(cudaEventRecord(h->t0, h->stream));
    const int rc = (h->solve_mode == 1 && !queue_mode) ? solve_phased(h, total, force_cold)
                                                       : launch_fused(h, io, total, queue_mode, force_cold, multi ? multi->B : 0);
    if (rc) return rc;
    if (multi)
    {
        const int long_list = io.in.obst_count && io.in.obst_max > h->L.M;
        multistart_select_kernel<<<grid_for(multi->B, WARPS_PER_CTA), WARPS_PER_CTA * 32, 0, h->stream>>>(h->L, h->ws, multi->B, multi->K, multi->hysteresis,
                                                                                                      long_list, io.out(), h->d_winner);
        h->stats.launches_total += 1;
        CK(cudaGetLastError());
    }
    CK(cudaEventRecord(h->t1, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, h->t0, h->t1));
    if (solve_time_s) *solve_time_s = ms * 1e-3;
    ev_collect(h);
    return collect_fused_counters(h);
}

// results of `B` instances from `io` to the host, then a synchronise (Mem::Host), or into device arrays in stream order
// (Mem::Device; d2h_bytes counts the host copies only).  A null destination is skipped.
static int fetch_outputs(mpcb200_handle* h, const IoBuffers& io, int B, double* u_seq, double* x_seq, double* dt_out, int* status, double* kkt_err, int* iters,
                         Mem mem = Mem::Host)
{
    const size_t n = (size_t)B, N = (size_t)h->cfg.n;
    const cudaMemcpyKind kind = mem == Mem::Host ? cudaMemcpyDeviceToHost : cudaMemcpyDeviceToDevice;
    const long long counted = mem == Mem::Host ? 1 : 0;
    if (u_seq) { CK(cudaMemcpyAsync(u_seq, io.useq, n * N * 16, kind, h->stream)); h->stats.d2h_bytes += counted * (long long)(n * N * 16); }
    if (x_seq) { CK(cudaMemcpyAsync(x_seq, io.xseq, n * N * 24, kind, h->stream)); h->stats.d2h_bytes += counted * (long long)(n * N * 24); }
    if (dt_out) { CK(cudaMemcpyAsync(dt_out, io.dt, n * 8, kind, h->stream)); h->stats.d2h_bytes += counted * (long long)(n * 8); }
    if (status) { CK(cudaMemcpyAsync(status, io.status, n * 4, kind, h->stream)); h->stats.d2h_bytes += counted * (long long)(n * 4); }
    if (kkt_err) { CK(cudaMemcpyAsync(kkt_err, io.kkt, n * 8, kind, h->stream)); h->stats.d2h_bytes += counted * (long long)(n * 8); }
    if (iters) { CK(cudaMemcpyAsync(iters, io.iters, n * 4, kind, h->stream)); h->stats.d2h_bytes += counted * (long long)(n * 4); }
    if (mem == Mem::Host) CK(cudaStreamSynchronize(h->stream));
    return 0;
}

// ---- queue solve: `total` cold instances through the persistent kernel (continuous batching) ----------------------
extern "C" int mpcb200_solve_stream(mpcb200_handle* h, int total, const double* x0, const double* xf, const double* u_prev, double u_prev_dt,
                                    const mpcb200_obstacles* obst, const mpcb200_viapoints* vp, double* u_seq, double* x_seq, double* dt_out,
                                    int* status, double* kkt_err, int* iters, double* solve_time_s)
{
    if (!h) return MPCB200_E_INVALID;
    if (total < 1 || !x0 || !xf) return set_err(h, MPCB200_E_INVALID, "total >= 1, x0 and xf are required");
    if (h->robot_limits_n > 0) return set_err(h, MPCB200_E_UNSUPPORTED, "solve_stream with per-robot limits: queue entries are not robots");
    if (h->robot_geometry_n > 0) return set_err(h, MPCB200_E_UNSUPPORTED, "solve_stream with per-robot geometry: queue entries are not robots");
    if (h->robot_weights_n > 0) return set_err(h, MPCB200_E_UNSUPPORTED, "solve_stream with per-robot weights: queue entries are not robots");
    if (h->robot_model_n > 0) return set_err(h, MPCB200_E_UNSUPPORTED, "solve_stream with per-robot models: queue entries are not robots");
    CK(cudaSetDevice(h->device));
    int rc;
    if ((rc = io_reserve(h, h->queue, (size_t)total, 0))) return rc;
    if ((rc = load_inputs(h, h->queue, total, x0, xf, u_prev, u_prev_dt, obst, vp, nullptr, nullptr))) return rc;
    if ((rc = timed_launch(h, h->queue, total, 1, 1, solve_time_s))) return rc;
    return fetch_outputs(h, h->queue, total, u_seq, x_seq, dt_out, status, kkt_err, iters);
}

extern "C" int mpcb200_step_batch(mpcb200_handle* h, int B, const double* x0, const double* xf, const double* u_prev, double u_prev_dt,
                                  const mpcb200_obstacles* obst, const mpcb200_viapoints* vp, const double* x_init,
                                  const unsigned char* reinit, double* u_seq, double* x_seq, double* dt_out, int* status,
                                  double* kkt_err, int* iters, double* solve_time_s)
{
    int rc = check_batch(h, B);
    if (rc) return rc;
    if ((rc = check_budget_mode(h))) return rc;
    if ((rc = check_robot_limits(h, B))) return rc;
    CK(cudaSetDevice(h->device));
    if ((rc = load_inputs(h, h->batch, B, x0, xf, u_prev, u_prev_dt, obst, vp, x_init, reinit))) return rc;
    // the phased mode works on the instance blocks; the fused kernel reads the compact arrays itself
    if (h->solve_mode == 1 && (rc = scatter_to_blocks(h, B))) return rc;
    h->B = B;
    if ((rc = timed_launch(h, h->batch, B, 0, 0, solve_time_s))) return rc;
    return fetch_outputs(h, h->batch, B, u_seq, x_seq, dt_out, status, kkt_err, iters);
}

extern "C" int mpcb200_step_batch_multistart(mpcb200_handle* h, int B, int K, double hysteresis, const double* x0, const double* xf,
                                             const double* u_prev, double u_prev_dt, const mpcb200_obstacles* obst, const mpcb200_viapoints* vp,
                                             const double* x_init, const unsigned char* reinit, double* u_seq, double* x_seq, double* dt_out,
                                             int* status, double* kkt_err, int* iters, int* winner, double* solve_time_s)
{
    int rc = check_batch(h, B);
    if (rc) return rc;
    if (K < 1 || (long long)B * K > h->max_batch) return set_err(h, MPCB200_E_INVALID, "multistart: K >= 1 candidates per robot and B*K <= max_batch required");
    if (K - 1 > 2 * h->cfg.initial_guess_bumps)
        return set_err(h, MPCB200_E_INVALID, "multistart: K - 1 challengers need as many bumped lines besides the best (K - 1 <= 2 initial_guess_bumps)");
    if (!std::isfinite(hysteresis) || !(hysteresis > 0.0)) return set_err(h, MPCB200_E_INVALID, "multistart: hysteresis must be finite and > 0");
    if (K > 1 && h->cfg.reference_initial_guess)
        return set_err(h, MPCB200_E_UNSUPPORTED, "multistart: the challengers' bumped lines are solver-side preprocessing, off with reference_initial_guess");
    if (K > 1 && h->cfg.initial_guess_bumps > 31) return set_err(h, MPCB200_E_UNSUPPORTED, "multistart: initial_guess_bumps <= 31 with K > 1");
    if (h->solve_mode == 1) return set_err(h, MPCB200_E_UNSUPPORTED, "multistart needs the fused solve kernel (MPCB200_OPT_SOLVE_MODE 0)");
    if ((rc = check_robot_limits(h, B))) return rc;
    CK(cudaSetDevice(h->device));
    if ((rc = load_inputs(h, h->batch, B, x0, xf, u_prev, u_prev_dt, obst, vp, x_init, reinit))) return rc;
    h->B = B;
    const Multistart ms{B, K, hysteresis};
    if ((rc = timed_launch(h, h->batch, B * K, 0, 0, solve_time_s, &ms))) return rc;
    if (winner) { CK(cudaMemcpyAsync(winner, h->d_winner, (size_t)B * 4, cudaMemcpyDeviceToHost, h->stream)); h->stats.d2h_bytes += (long long)B * 4; }
    return fetch_outputs(h, h->batch, B, u_seq, x_seq, dt_out, status, kkt_err, iters);
}

extern "C" int mpcb200_upload_inputs(mpcb200_handle* h, int B, const double* x0, const double* xf, const double* u_prev, double u_prev_dt,
                                     const mpcb200_obstacles* obst, const mpcb200_viapoints* vp, const double* x_init)
{
    int rc = check_batch(h, B);
    if (rc) return rc;
    CK(cudaSetDevice(h->device));
    if ((rc = load_inputs(h, h->batch, B, x0, xf, u_prev, u_prev_dt, obst, vp, x_init, nullptr))) return rc;
    if ((rc = scatter_to_blocks(h, B))) return rc;
    h->B = B;
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}

extern "C" int mpcb200_solve_resident(mpcb200_handle* h, int cold, double* solve_time_s)
{
    if (!h || h->B < 1) return set_err(h, MPCB200_E_INVALID, "no resident inputs: call mpcb200_upload_inputs first");
    if (int rc = check_budget_mode(h)) return rc;
    if (int rc = check_robot_limits(h, h->B)) return rc;
    CK(cudaSetDevice(h->device));
    return timed_launch(h, h->batch, h->B, 0, cold ? 1 : 0, solve_time_s);
}

extern "C" int mpcb200_fetch_results(mpcb200_handle* h, double* u_seq, double* x_seq, double* dt_out, int* status, double* kkt_err, int* iters)
{
    if (!h || h->B < 1) return set_err(h, MPCB200_E_INVALID, "nothing to fetch");
    CK(cudaSetDevice(h->device));
    return fetch_outputs(h, h->batch, h->B, u_seq, x_seq, dt_out, status, kkt_err, iters);
}

extern "C" int mpcb200_device_controls(mpcb200_handle* h, void** dev_ptr, long long* n_doubles)
{
    if (!h || h->B < 1) return set_err(h, MPCB200_E_INVALID, "no batch solved yet");
    if (dev_ptr) *dev_ptr = h->batch.upacked;
    if (n_doubles) *n_doubles = (long long)h->B * (h->cfg.n - 1) * 2;
    return 0;
}

extern "C" int mpcb200_reset(mpcb200_handle* h, const unsigned char* which, int B)
{
    if (!h) return MPCB200_E_INVALID;
    CK(cudaSetDevice(h->device));
    const int n = which ? B : h->max_batch;
    if (n < 1 || n > h->max_batch) return set_err(h, MPCB200_E_INVALID, "batch size out of range");
    if (which) CK(cudaMemcpyAsync(h->batch.reinit, which, (size_t)n, cudaMemcpyHostToDevice, h->stream));
    reset_kernel<<<(n + 127) / 128, 128, 0, h->stream>>>(h->L, h->ws, n, which ? h->batch.reinit : nullptr);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}

extern "C" int mpcb200_resample(mpcb200_handle* h, int n_new)
{
    if (!h) return MPCB200_E_INVALID;
    if (n_new < 3 || n_new > h->n_cap) return set_err(h, MPCB200_E_INVALID, "resample: horizon must be in [3, n the handle was created with]");
    if (n_new == h->cfg.n) return MPCB200_OK;
    CK(cudaSetDevice(h->device));
    const int B = h->max_batch, n_old = h->cfg.n;
    const int rec_words = MPCB200_SCAL_WORDS + 5 * h->n_cap;
    if (!h->d_resample) CK(cudaMalloc(&h->d_resample, (size_t)B * rec_words * sizeof(double)));
    resample_pack_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(h->L, h->ws, h->d_resample, rec_words, B);
    CK(cudaGetLastError());
    h->cfg.n = n_new;
    make_layout(&h->cfg, h->L.M, h->L.V, h->L);
    resample_unpack_kernel<<<(B + 127) / 128, 128, 0, h->stream>>>(h->L, h->ws, h->d_resample, rec_words, n_old, B);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(h->stream));
    return MPCB200_OK;
}

extern "C" int mpcb200_get_horizon(const mpcb200_handle* h, int* n, int* n_capacity)
{
    if (!h) return MPCB200_E_INVALID;
    if (n) *n = h->cfg.n;
    if (n_capacity) *n_capacity = h->n_cap;
    return MPCB200_OK;
}

// ---- per-robot limits: records into d_limits; the solves launch solve_fused_robot_kernel while robot_limits_n > 0 ----
extern "C" int mpcb200_set_robot_limits(mpcb200_handle* h, int n, const double* limits)
{
    if (!h) return MPCB200_E_INVALID;
    if (n < 0 || n > h->max_batch) return set_err(h, MPCB200_E_INVALID, "set_robot_limits: n must be in [0, max_batch]");
    if (n > 0 && !limits) return set_err(h, MPCB200_E_INVALID, "set_robot_limits: limits are required for n > 0");
    for (int b = 0; b < n; ++b)
        if (!robot_limits_valid(h->cfg, limits + (size_t)b * MPCB200_LIMIT_WORDS))
            return set_err(h, MPCB200_E_INVALID, "set_robot_limits: record " + std::to_string(b) + " is not valid (NaN, u_ub <= u_lb, a bound "
                                                 "finite where the configuration's is not or the reverse, or a clearance not in [0, inf))");
    CK(cudaSetDevice(h->device));
    if (n > 0)
    {
        CK(cudaMemcpyAsync(h->d_limits, limits, (size_t)n * MPCB200_LIMIT_WORDS * 8, cudaMemcpyHostToDevice, h->stream));
        h->stats.h2d_bytes += (long long)n * MPCB200_LIMIT_WORDS * 8;
        CK(cudaStreamSynchronize(h->stream));
    }
    h->robot_limits_n = n;
    return MPCB200_OK;
}

extern "C" int mpcb200_set_robot_limits_async(mpcb200_handle* h, int n, const double* limits)
{
    if (!h) return MPCB200_E_INVALID;
    if (n < 0 || n > h->max_batch) return set_err(h, MPCB200_E_INVALID, "set_robot_limits_async: n must be in [0, max_batch]");
    if (n > 0 && !limits) return set_err(h, MPCB200_E_INVALID, "set_robot_limits_async: limits are required for n > 0");
    CK(cudaSetDevice(h->device));
    if (n > 0)
    {
        if (int rc = check_device_arrays(h, "set_robot_limits_async", {limits})) return rc;
        CK(cudaMemcpyAsync(h->d_limits, limits, (size_t)n * MPCB200_LIMIT_WORDS * 8, cudaMemcpyDeviceToDevice, h->stream));
    }
    h->robot_limits_n = n;
    return MPCB200_OK;
}

// With model records set, the pairs of model and geometry records the blocking setters would leave (model_n records at `model`,
// geo_n at `geo`): each robot's geometry (its record, else the configuration's values) valid for its types (its model record,
// else the handle's).  The first robot whose pair is not valid, or -1.
static int first_invalid_pair(const Cfg& c, int model_n, const double* model, int geo_n, const double* geo)
{
    const int n = model_n > geo_n ? model_n : geo_n;
    for (int b = 0; b < n; ++b)
    {
        const double* g = b < geo_n ? geo + (size_t)b * MPCB200_GEOMETRY_WORDS : nullptr;
        if (b < model_n ? !robot_model_valid(c, model + (size_t)b * MPCB200_MODEL_WORDS, g) : !robot_geometry_valid(c, g)) return b;
    }
    return -1;
}

// ---- per-robot geometry: records into d_geometry; the solves launch solve_fused_fleet_kernel while robot_geometry_n > 0 ----
extern "C" int mpcb200_set_robot_geometry(mpcb200_handle* h, int n, const double* geometry)
{
    if (!h) return MPCB200_E_INVALID;
    if (n < 0 || n > h->max_batch) return set_err(h, MPCB200_E_INVALID, "set_robot_geometry: n must be in [0, max_batch]");
    if (n > 0 && !geometry) return set_err(h, MPCB200_E_INVALID, "set_robot_geometry: geometry is required for n > 0");
    if (h->robot_model_n == 0)
    {
        if (n > 0 && !reads_geometry(h->cfg))
            return set_err(h, MPCB200_E_INVALID, "set_robot_geometry: a unicycle with a point footprint has no geometry to vary");
        for (int b = 0; b < n; ++b)
            if (!robot_geometry_valid(h->cfg, geometry + (size_t)b * MPCB200_GEOMETRY_WORDS))
                return set_err(h, MPCB200_E_INVALID, "set_robot_geometry: record " + std::to_string(b) + " is not valid (a wheelbase or length_rear "
                                                     "not finite and > 0, a length_front or radius not finite and >= 0, an offset, line end or vertex "
                                                     "not finite, or n_poly not an integer in [1, 16])");
    }
    else if (h->model_host)   // each record for its robot's types, and the robots without one keep a valid configuration geometry
    {
        const int b = first_invalid_pair(h->cfg, h->robot_model_n, h->h_model.data(), n, geometry);
        if (b >= 0)
            return set_err(h, MPCB200_E_INVALID, "set_robot_geometry: robot " + std::to_string(b) + " would have a geometry that is not valid "
                                                 "for the types of its model record (mpcb200_set_robot_model)");
    }
    CK(cudaSetDevice(h->device));
    if (n > 0)
    {
        CK(cudaMemcpyAsync(h->d_geometry, geometry, (size_t)n * MPCB200_GEOMETRY_WORDS * 8, cudaMemcpyHostToDevice, h->stream));
        h->stats.h2d_bytes += (long long)n * MPCB200_GEOMETRY_WORDS * 8;
        CK(cudaStreamSynchronize(h->stream));
    }
    h->robot_geometry_n = n;
    h->h_geometry.assign(geometry, geometry + (size_t)n * MPCB200_GEOMETRY_WORDS);
    h->geometry_host = true;
    return MPCB200_OK;
}

extern "C" int mpcb200_set_robot_geometry_async(mpcb200_handle* h, int n, const double* geometry)
{
    if (!h) return MPCB200_E_INVALID;
    if (n < 0 || n > h->max_batch) return set_err(h, MPCB200_E_INVALID, "set_robot_geometry_async: n must be in [0, max_batch]");
    if (n > 0 && !geometry) return set_err(h, MPCB200_E_INVALID, "set_robot_geometry_async: geometry is required for n > 0");
    if (n > 0 && h->robot_model_n == 0 && !reads_geometry(h->cfg))
        return set_err(h, MPCB200_E_INVALID, "set_robot_geometry_async: a unicycle with a point footprint has no geometry to vary");
    CK(cudaSetDevice(h->device));
    if (n > 0)
    {
        if (int rc = check_device_arrays(h, "set_robot_geometry_async", {geometry})) return rc;
        CK(cudaMemcpyAsync(h->d_geometry, geometry, (size_t)n * MPCB200_GEOMETRY_WORDS * 8, cudaMemcpyDeviceToDevice, h->stream));
    }
    h->robot_geometry_n = n;
    h->h_geometry.clear();
    h->geometry_host = n == 0;
    return MPCB200_OK;
}

// ---- per-robot weights: records into d_weights; the solves launch solve_fused_weights_kernel while robot_weights_n > 0 ----
extern "C" int mpcb200_set_robot_weights(mpcb200_handle* h, int n, const double* weights)
{
    if (!h) return MPCB200_E_INVALID;
    if (n < 0 || n > h->max_batch) return set_err(h, MPCB200_E_INVALID, "set_robot_weights: n must be in [0, max_batch]");
    if (n > 0 && !weights) return set_err(h, MPCB200_E_INVALID, "set_robot_weights: weights are required for n > 0");
    if (n > 0 && !reads_weights(h->cfg))
        return set_err(h, MPCB200_E_INVALID, "set_robot_weights: a minimum-time objective without terminal cost has no weights to vary");
    for (int b = 0; b < n; ++b)
        if (!robot_weights_valid(h->cfg, weights + (size_t)b * MPCB200_WEIGHT_WORDS))
            return set_err(h, MPCB200_E_INVALID, "set_robot_weights: record " + std::to_string(b) + " is not valid (a weight that is read "
                                                 "not finite, or Q and R switching the hybrid minimum-time term against the configuration)");
    CK(cudaSetDevice(h->device));
    if (n > 0)
    {
        CK(cudaMemcpyAsync(h->d_weights, weights, (size_t)n * MPCB200_WEIGHT_WORDS * 8, cudaMemcpyHostToDevice, h->stream));
        h->stats.h2d_bytes += (long long)n * MPCB200_WEIGHT_WORDS * 8;
        CK(cudaStreamSynchronize(h->stream));
    }
    h->robot_weights_n = n;
    return MPCB200_OK;
}

extern "C" int mpcb200_set_robot_weights_async(mpcb200_handle* h, int n, const double* weights)
{
    if (!h) return MPCB200_E_INVALID;
    if (n < 0 || n > h->max_batch) return set_err(h, MPCB200_E_INVALID, "set_robot_weights_async: n must be in [0, max_batch]");
    if (n > 0 && !weights) return set_err(h, MPCB200_E_INVALID, "set_robot_weights_async: weights are required for n > 0");
    if (n > 0 && !reads_weights(h->cfg))
        return set_err(h, MPCB200_E_INVALID, "set_robot_weights_async: a minimum-time objective without terminal cost has no weights to vary");
    CK(cudaSetDevice(h->device));
    if (n > 0)
    {
        if (int rc = check_device_arrays(h, "set_robot_weights_async", {weights})) return rc;
        CK(cudaMemcpyAsync(h->d_weights, weights, (size_t)n * MPCB200_WEIGHT_WORDS * 8, cudaMemcpyDeviceToDevice, h->stream));
    }
    h->robot_weights_n = n;
    return MPCB200_OK;
}

// ---- per-robot models: records into d_model; the solves launch solve_fused_models_kernel while robot_model_n > 0 ----
extern "C" int mpcb200_set_robot_model(mpcb200_handle* h, int n, const double* model)
{
    if (!h) return MPCB200_E_INVALID;
    if (n < 0 || n > h->max_batch) return set_err(h, MPCB200_E_INVALID, "set_robot_model: n must be in [0, max_batch]");
    if (n > 0 && !model) return set_err(h, MPCB200_E_INVALID, "set_robot_model: model is required for n > 0");
    for (int b = 0; b < n; ++b)
    {
        const double* m = model + (size_t)b * MPCB200_MODEL_WORDS;
        if (!model_word_valid(m[MPCB200_MOD_ROBOT_TYPE], MPCB200_ROBOT_KIN_BICYCLE) || !model_word_valid(m[MPCB200_MOD_FOOTPRINT_TYPE], MPCB200_FOOTPRINT_POLYGON))
            return set_err(h, MPCB200_E_INVALID, "set_robot_model: record " + std::to_string(b) + " is not valid (robot_type not an integer in "
                                                 "[0, 3] or footprint_type not an integer in [0, 4])");
    }
    // the geometry records of the blocking setter (or none) against the new types; geometry records of the async setter are the solve's to check
    if (h->geometry_host)
    {
        if (n == 0 && h->robot_geometry_n > 0 && !reads_geometry(h->cfg))
            return set_err(h, MPCB200_E_INVALID, "set_robot_model: clearing the model records would leave geometry records on a unicycle with a "
                                                 "point footprint (clear the geometry records first)");
        const int b = first_invalid_pair(h->cfg, n, model, h->robot_geometry_n, h->h_geometry.data());
        if (b >= 0)
            return set_err(h, MPCB200_E_INVALID, "set_robot_model: robot " + std::to_string(b) + " would have a geometry (its geometry record, or "
                                                 "the configuration's) that is not valid for its types");
    }
    CK(cudaSetDevice(h->device));
    if (n > 0)
    {
        CK(cudaMemcpyAsync(h->d_model, model, (size_t)n * MPCB200_MODEL_WORDS * 8, cudaMemcpyHostToDevice, h->stream));
        h->stats.h2d_bytes += (long long)n * MPCB200_MODEL_WORDS * 8;
        CK(cudaStreamSynchronize(h->stream));
    }
    h->robot_model_n = n;
    h->h_model.assign(model, model + (size_t)n * MPCB200_MODEL_WORDS);
    h->model_host = true;
    return MPCB200_OK;
}

extern "C" int mpcb200_set_robot_model_async(mpcb200_handle* h, int n, const double* model)
{
    if (!h) return MPCB200_E_INVALID;
    if (n < 0 || n > h->max_batch) return set_err(h, MPCB200_E_INVALID, "set_robot_model_async: n must be in [0, max_batch]");
    if (n > 0 && !model) return set_err(h, MPCB200_E_INVALID, "set_robot_model_async: model is required for n > 0");
    CK(cudaSetDevice(h->device));
    if (n > 0)
    {
        if (int rc = check_device_arrays(h, "set_robot_model_async", {model})) return rc;
        CK(cudaMemcpyAsync(h->d_model, model, (size_t)n * MPCB200_MODEL_WORDS * 8, cudaMemcpyDeviceToDevice, h->stream));
    }
    h->robot_model_n = n;
    h->h_model.clear();
    h->model_host = n == 0;
    return MPCB200_OK;
}

// ---- kernel-level access ------------------------------------------------------------------------------------
static int field_info(const mpcb200_handle* h, int field, int* off, int* cnt)
{
    const WsLayout& L = h->L;
    switch (field)
    {
        case MPCB200_F_X: *off = L.oX; *cnt = 3; return 0;
        case MPCB200_F_U: *off = L.oU; *cnt = 2; return 0;
        case MPCB200_F_NU: *off = L.oNU; *cnt = 3; return 0;
        case MPCB200_F_S: *off = L.oS; *cnt = L.RS; return 0;
        case MPCB200_F_LAM: *off = L.oLAM; *cnt = L.RS; return 0;
        case MPCB200_F_KKT: *off = L.oKKT; *cnt = KW; return 0;
        case MPCB200_F_STEP: *off = L.oSTEP; *cnt = 8; return 0;
        case MPCB200_F_SCAL: *off = L.oSCAL; *cnt = MPCB200_SCAL_WORDS; return 0;
        case MPCB200_F_OBSIDX: *off = L.oOBS; *cnt = L.K > 0 ? L.K : 1; return 0;
        case MPCB200_F_OBSGIDX: *off = L.oOGIDX; *cnt = L.M; return 0;
    }
    return -1;
}

extern "C" int mpcb200_ws_count(const mpcb200_handle* h, int field)
{
    int off, cnt;
    if (!h || field_info(h, field, &off, &cnt)) return MPCB200_E_INVALID;
    return cnt;
}

extern "C" int mpcb200_ws_read(mpcb200_handle* h, int field, int B, double* dst)
{
    int off, cnt, rc = check_batch(h, B);
    if (rc) return rc;
    if (!dst || field_info(h, field, &off, &cnt)) return set_err(h, MPCB200_E_INVALID, "bad field");
    CK(cudaSetDevice(h->device));
    const int N = h->L.N;
    if (field == MPCB200_F_KKT)
    {   // device layout: stage records [k][RSTR] inside the instance block; the API presents [B][42][N]
        std::vector<double> tmp((size_t)B * N * RSTR);
        CK(cudaMemcpy2DAsync(tmp.data(), (size_t)N * RSTR * 8, h->ws + off, (size_t)h->L.stride * 8, (size_t)N * RSTR * 8, (size_t)B, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        for (int b = 0; b < B; ++b)
            for (int k = 0; k < N; ++k)
                for (int f = 0; f < KW; ++f) dst[((size_t)b * KW + f) * N + k] = tmp[((size_t)b * N + k) * RSTR + f];
        return 0;
    }
    if (field == MPCB200_F_OBSIDX)
    {   // device layout: one signed byte per (slot, stage); the API presents doubles [B][K][N]
        const size_t nb = (size_t)cnt * N;
        std::vector<signed char> tmp((size_t)B * nb);
        CK(cudaMemcpy2DAsync(tmp.data(), nb, h->ws + off, (size_t)h->L.stride * 8, nb, (size_t)B, cudaMemcpyDeviceToHost, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        for (size_t i = 0; i < tmp.size(); ++i) dst[i] = (double)tmp[i];
        return 0;
    }
    const size_t words = (field == MPCB200_F_SCAL || field == MPCB200_F_OBSGIDX) ? (size_t)cnt : (size_t)cnt * N;
    CK(cudaMemcpy2DAsync(dst, words * 8, h->ws + off, (size_t)h->L.stride * 8, words * 8, (size_t)B, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}

extern "C" int mpcb200_ws_write(mpcb200_handle* h, int field, int B, const double* src)
{
    int off, cnt, rc = check_batch(h, B);
    if (rc) return rc;
    if (!src || field_info(h, field, &off, &cnt)) return set_err(h, MPCB200_E_INVALID, "bad field");
    CK(cudaSetDevice(h->device));
    const int N = h->L.N;
    if (field == MPCB200_F_KKT)
    {
        std::vector<double> tmp((size_t)B * N * RSTR, 0.0);
        for (int b = 0; b < B; ++b)
            for (int k = 0; k < N; ++k)
                for (int f = 0; f < KW; ++f) tmp[((size_t)b * N + k) * RSTR + f] = src[((size_t)b * KW + f) * N + k];
        CK(cudaMemcpy2DAsync(h->ws + off, (size_t)h->L.stride * 8, tmp.data(), (size_t)N * RSTR * 8, (size_t)N * RSTR * 8, (size_t)B, cudaMemcpyHostToDevice, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        return 0;
    }
    if (field == MPCB200_F_OBSIDX)
    {
        const size_t nb = (size_t)cnt * N;
        std::vector<signed char> tmp((size_t)B * nb);
        for (size_t i = 0; i < tmp.size(); ++i) tmp[i] = (signed char)src[i];
        CK(cudaMemcpy2DAsync(h->ws + off, (size_t)h->L.stride * 8, tmp.data(), nb, nb, (size_t)B, cudaMemcpyHostToDevice, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        return 0;
    }
    const size_t words = (field == MPCB200_F_SCAL || field == MPCB200_F_OBSGIDX) ? (size_t)cnt : (size_t)cnt * N;
    CK(cudaMemcpy2DAsync(h->ws + off, (size_t)h->L.stride * 8, src, words * 8, words * 8, (size_t)B, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}

extern "C" int mpcb200_run_phase(mpcb200_handle* h, int phase, int B)
{
    int rc = check_batch(h, B);
    if (rc) return rc;
    if (h->robot_limits_n > 0) return set_err(h, MPCB200_E_UNSUPPORTED, "the phase kernels have no per-robot limits (mpcb200_set_robot_limits)");
    if (h->robot_geometry_n > 0) return set_err(h, MPCB200_E_UNSUPPORTED, "the phase kernels have no per-robot geometry (mpcb200_set_robot_geometry)");
    if (h->robot_weights_n > 0) return set_err(h, MPCB200_E_UNSUPPORTED, "the phase kernels have no per-robot weights (mpcb200_set_robot_weights)");
    if (h->robot_model_n > 0) return set_err(h, MPCB200_E_UNSUPPORTED, "the phase kernels have no per-robot models (mpcb200_set_robot_model)");
    CK(cudaSetDevice(h->device));
    if ((rc = launch_phase(h, phase, B, 0, 1, nullptr, true))) return rc;
    CK(cudaStreamSynchronize(h->stream));
    ev_collect(h);
    return 0;
}

extern "C" int mpcb200_set_stream(mpcb200_handle* h, void* cuda_stream)
{
    if (!h) return MPCB200_E_INVALID;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    h->stream = cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream;
    return 0;
}

extern "C" int mpcb200_set_option(mpcb200_handle* h, int option, int value)
{
    if (!h) return MPCB200_E_INVALID;
    if (option == MPCB200_OPT_SOLVE_MODE && value >= 0 && value <= 1) { h->solve_mode = value; return 0; }
    if (option == MPCB200_OPT_CTAS_PER_SM && value >= 0 && value <= 32) { h->max_ctas_per_sm = value; return 0; }
    if (option == MPCB200_OPT_ORDER_BY_HISTORY && value >= 0 && value <= 1) { h->order_by_history = value; return 0; }
    if (option == MPCB200_OPT_SM_PHASE_SYNC && value >= -1 && value <= 2) { h->sm_phase_sync = value; return 0; }
    if (option == MPCB200_OPT_FORCE_GENERIC_MODEL && value >= 0 && value <= 1) { h->force_generic_model = value; return 0; }
    if (option == MPCB200_OPT_CRITICAL_PLACEMENT && value >= 0 && value <= 1) { h->critical_placement = value; return 0; }
    return set_err(h, MPCB200_E_INVALID, "unknown option or value");
}

extern "C" int mpcb200_kernel_model(const mpcb200_handle* h) { return h ? model_key_of(h->last_model) : MPCB200_E_INVALID; }
extern "C" int mpcb200_kernel_problem(const mpcb200_handle* h) { return h ? problem_key_of(h->last_model) : MPCB200_E_INVALID; }

extern "C" int mpcb200_set_timing(mpcb200_handle* h, unsigned phase_mask)
{
    if (!h) return MPCB200_E_INVALID;
    h->timing_mask = phase_mask;
    return 0;
}

extern "C" int mpcb200_time_phase(mpcb200_handle* h, int phase, int B, int reps, int flush_l2, double* ms_per_launch)
{
    int rc = check_batch(h, B);
    if (rc) return rc;
    if (h->robot_limits_n > 0) return set_err(h, MPCB200_E_UNSUPPORTED, "the phase kernels have no per-robot limits (mpcb200_set_robot_limits)");
    if (h->robot_geometry_n > 0) return set_err(h, MPCB200_E_UNSUPPORTED, "the phase kernels have no per-robot geometry (mpcb200_set_robot_geometry)");
    if (h->robot_weights_n > 0) return set_err(h, MPCB200_E_UNSUPPORTED, "the phase kernels have no per-robot weights (mpcb200_set_robot_weights)");
    if (h->robot_model_n > 0) return set_err(h, MPCB200_E_UNSUPPORTED, "the phase kernels have no per-robot models (mpcb200_set_robot_model)");
    if (reps < 1) reps = 1;
    CK(cudaSetDevice(h->device));
    double total = 0.0;
    for (int r = 0; r < reps; ++r)
    {
        if (flush_l2) { flush_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->d_flush, h->flush_n); CK(cudaGetLastError()); }
        CK(cudaEventRecord(h->t0, h->stream));
        if ((rc = launch_phase(h, phase, B, 0, 1, nullptr, false))) return rc;
        CK(cudaEventRecord(h->t1, h->stream));
        CK(cudaStreamSynchronize(h->stream));
        float ms = 0.f;
        CK(cudaEventElapsedTime(&ms, h->t0, h->t1));
        total += ms;
    }
    if (ms_per_launch) *ms_per_launch = total / reps;
    return 0;
}

extern "C" int mpcb200_stats_get(const mpcb200_handle* hc, mpcb200_stats* out)
{
    mpcb200_handle* h = const_cast<mpcb200_handle*>(hc);
    if (!h || !out) return MPCB200_E_INVALID;
    CK(cudaSetDevice(h->device));
    CK(cudaStreamSynchronize(h->stream));
    int rc = collect_fused_counters(h);   // also picks up the counters of phase-wise KKT launches
    if (rc) return rc;
    CK(cudaStreamSynchronize(h->stream));
    *out = h->stats;
    return 0;
}
extern "C" int mpcb200_stats_reset(mpcb200_handle* h)
{
    if (!h) return MPCB200_E_INVALID;
    memset(&h->stats, 0, sizeof(h->stats));
    CK(cudaSetDevice(h->device));
    CK(cudaMemsetAsync(h->d_counters, 0, CNT_BYTES, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}
extern "C" int mpcb200_export_controls(mpcb200_handle* h, void* dst_dev)
{
    if (!h || h->B < 1 || !dst_dev) return set_err(h, MPCB200_E_INVALID, "nothing to export");
    CK(cudaSetDevice(h->device));
    CK(cudaMemcpyAsync(dst_dev, h->batch.upacked, (size_t)h->B * (h->cfg.n - 1) * 16, cudaMemcpyDeviceToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}
// costmap -> point obstacles on the device.  Poses come from the host (host_pose) or are already on the device (dev_pose: the x0 array
// of a step); lists go to d_count / d_type / d_params ([B], [B][M], [B][M][7]; nullptr: scratch of this call).  Host maps
// (Mem::Host) are copied into the scratch and the kernels are bracketed by the events c0 / c1; device maps are read in place,
// with no events.
struct CostmapOut { int* count; int* found; int* type; double* params; };
static int costmap_run(mpcb200_handle* h, int B, const mpcb200_costmaps* maps, const double* host_pose, const double* dev_pose, double behind_robot_dist,
                       int max_per_instance, int* d_count, int* d_type, double* d_params, CostmapOut* out, Mem mem = Mem::Host)
{
    if (B < 1 || !maps || !maps->cost || !maps->origin || max_per_instance < 1)
        return set_err(h, MPCB200_E_INVALID, "costmap_obstacles: B >= 1, maps, poses and output arrays are required");
    if (maps->size_x < 2 || maps->size_y < 2 || !(maps->resolution > 0)) return set_err(h, MPCB200_E_INVALID, "costmap_obstacles: maps of at least 2 x 2 cells with a positive resolution");
    const size_t W = (size_t)maps->size_x, H = (size_t)maps->size_y, M = (size_t)max_per_instance;
    const int nrb = (int)((H - 1 + 31) / 32);            // 32-row blocks of the rows the reference visits
    const int ncg = (int)((W + MARK_COLS - 1) / MARK_COLS); // 16-column groups per row
    const int Wp = ncg * MARK_COLS;                      // mask row pitch: sixteen columns per marking thread
    const size_t mask_words = (size_t)B * nrb * Wp;
    const size_t map_bytes = mem == Mem::Host ? (size_t)B * W * H : 0;
    const size_t need = map_bytes + 16 + (size_t)B * 5 * 8 + 2 * (size_t)B * 4 + (size_t)B * M * (MPCB200_OBST_STRIDE * 8 + 4) +
                        mask_words * 4 + 512;
    if (need > h->cm_cap)
    {
        if (int rc = check_growth_allowed(h, "the costmap scratch")) return rc;
        CK(cudaStreamSynchronize(h->stream));
        if (h->d_cm) cudaFree(h->d_cm);
        h->d_cm = nullptr; h->cm_cap = 0;
        CK(cudaMalloc(&h->d_cm, need));
        h->cm_cap = need;
    }
    // carve the scratch: 16-byte aligned pieces first (mask rows are stored as uint4), then ints, then the maps
    char* p = (char*)h->d_cm;
    unsigned* d_mask = (unsigned*)p; p += mask_words * 4;
    double* s_params = (double*)p; p += (size_t)B * M * MPCB200_OBST_STRIDE * 8;
    double* d_origin = (double*)p; p += (size_t)B * 2 * 8;
    double* d_pose = (double*)p; p += (size_t)B * 3 * 8;
    int* s_count = (int*)p; p += (size_t)B * 4;
    int* d_found = (int*)p; p += (size_t)B * 4;
    int* s_type = (int*)p; p += (size_t)B * M * 4;
    p = (char*)(((uintptr_t)p + 15) & ~(uintptr_t)15);
    if (!d_count) d_count = s_count;
    if (!d_type) d_type = s_type;
    if (!d_params) d_params = s_params;
    const unsigned char* cost = maps->cost;
    const double* origin = maps->origin;
    if (mem == Mem::Host)
    {
        unsigned char* d_cost = (unsigned char*)p;        // 16-byte aligned
        CK(cudaMemcpyAsync(d_cost, maps->cost, (size_t)B * W * H, cudaMemcpyHostToDevice, h->stream));
        CK(cudaMemcpyAsync(d_origin, maps->origin, (size_t)B * 16, cudaMemcpyHostToDevice, h->stream));
        if (host_pose) CK(cudaMemcpyAsync(d_pose, host_pose, (size_t)B * 24, cudaMemcpyHostToDevice, h->stream));
        h->stats.h2d_bytes += (long long)((size_t)B * W * H + (size_t)B * (host_pose ? 40 : 16));
        cost = d_cost; origin = d_origin;
    }
    CostmapArgs a{maps->size_x, maps->size_y, maps->resolution, behind_robot_dist, cost, origin, host_pose ? d_pose : dev_pose};
    const dim3 grid_mark((unsigned)(((size_t)B * ncg * nrb + 255) / 256));
    // slots behind count[b] are padding: zeroed, so that what goes back to the caller (and on into step_batch) is defined
    CK(cudaMemsetAsync(d_type, 0, (size_t)B * M * 4, h->stream));
    CK(cudaMemsetAsync(d_params, 0, (size_t)B * M * MPCB200_OBST_STRIDE * 8, h->stream));
    if (mem == Mem::Host) CK(cudaEventRecord(h->c0, h->stream));
    // Load width: every row of every map must start VB-aligned, i.e. size_x and the base address are multiples of VB.  The
    // scratch copy is 16-byte aligned; a caller's map may start anywhere.  No load reaches past the B size_y size_x bytes: tiles
    // beyond the last map are not run (b < B), rows from size_y - 1 on are not loaded, and inside a row the 16-byte load covers
    // columns c0..c0+15 < size_x (size_x % 16 == 0), the 4- and 1-byte loads test every word or byte against size_x.
    const uintptr_t base = (uintptr_t)cost;
    if (W % 16 == 0 && base % 16 == 0) costmap_mark_kernel<16><<<grid_mark, 256, 0, h->stream>>>(a, B, nrb, ncg, Wp, d_mask);
    else if (W % 4 == 0 && base % 4 == 0) costmap_mark_kernel<4><<<grid_mark, 256, 0, h->stream>>>(a, B, nrb, ncg, Wp, d_mask);
    else costmap_mark_kernel<1><<<grid_mark, 256, 0, h->stream>>>(a, B, nrb, ncg, Wp, d_mask);
    costmap_emit_kernel<<<B, 256, 0, h->stream>>>(a, B, nrb, Wp, d_mask, max_per_instance, d_count, d_found, d_params, d_type);
    CK(cudaGetLastError());
    if (mem == Mem::Host) CK(cudaEventRecord(h->c1, h->stream));
    h->stats.launches_total += 2;
    out->count = d_count; out->found = d_found; out->type = d_type; out->params = d_params;
    return 0;
}

extern "C" int mpcb200_costmap_obstacles(mpcb200_handle* h, int B, const mpcb200_costmaps* maps, const double* robot_pose, double behind_robot_dist,
                                         int max_per_instance, int* count, int* found, int* type, double* params)
{
    if (!h) return MPCB200_E_INVALID;
    if (!robot_pose || !count || !type || !params) return set_err(h, MPCB200_E_INVALID, "costmap_obstacles: B >= 1, maps, poses and output arrays are required");
    CK(cudaSetDevice(h->device));
    CostmapOut o;
    int rc = costmap_run(h, B, maps, robot_pose, nullptr, behind_robot_dist, max_per_instance, nullptr, nullptr, nullptr, &o);
    if (rc) return rc;
    const size_t M = (size_t)max_per_instance;
    CK(cudaMemcpyAsync(count, o.count, (size_t)B * 4, cudaMemcpyDeviceToHost, h->stream));
    if (found) CK(cudaMemcpyAsync(found, o.found, (size_t)B * 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(type, o.type, (size_t)B * M * 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaMemcpyAsync(params, o.params, (size_t)B * M * MPCB200_OBST_STRIDE * 8, cudaMemcpyDeviceToHost, h->stream));
    h->stats.d2h_bytes += (long long)((size_t)B * 8 + (size_t)B * M * (4 + MPCB200_OBST_STRIDE * 8));
    CK(cudaStreamSynchronize(h->stream));
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, h->c0, h->c1));
    h->costmap_ms = ms;
    return MPCB200_OK;
}

// One planning cycle from the costmaps: MpcLocalPlannerROS::computeVelocityCommands' updateObstacleContainerWithCostmap
// (mpc_local_planner_ros.cpp:474-499) followed by Controller::step, for B robots, without the obstacle lists leaving the device:
// maps H2D -> mark / emit into the batch's obstacle arrays (robot pose = x0) -> association over the lists -> solve.
extern "C" int mpcb200_step_batch_costmap(mpcb200_handle* h, int B, const double* x0, const double* xf, const double* u_prev, double u_prev_dt,
                                          const mpcb200_costmaps* maps, double behind_robot_dist, int max_per_instance, const mpcb200_viapoints* vp,
                                          const double* x_init, const unsigned char* reinit, double* u_seq, double* x_seq, double* dt_out, int* status,
                                          double* kkt_err, int* iters, int* obst_found, double* solve_time_s)
{
    int rc = check_batch(h, B);
    if (rc) return rc;
    if (max_per_instance < 1 || max_per_instance > MAX_OBST_LIST) return set_err(h, MPCB200_E_UNSUPPORTED, "step_batch_costmap: 1..2048 obstacles per instance");
    if ((rc = check_budget_mode(h))) return rc;
    if ((rc = check_robot_limits(h, B))) return rc;
    CK(cudaSetDevice(h->device));
    IoBuffers& io = h->batch;
    // room for the lists in the batch's obstacle arrays
    if ((rc = io_reserve(h, io, io.rows, max_per_instance))) return rc;
    if ((rc = load_inputs(h, io, B, x0, xf, u_prev, u_prev_dt, nullptr, vp, x_init, reinit))) return rc;
    CostmapOut o;
    if ((rc = costmap_run(h, B, maps, nullptr, io.x0, behind_robot_dist, max_per_instance, io.obst_count, io.obst_type, io.obst, &o))) return rc;
    io.in.obst_count = io.obst_count; io.in.obst_max = max_per_instance;   // point obstacles only: no line-obstacle kernel variant needed
    h->B = B;
    if (h->solve_mode == 1 && (rc = scatter_to_blocks(h, B))) return rc;
    if ((rc = timed_launch(h, io, B, 0, 0, solve_time_s))) return rc;
    if (obst_found) CK(cudaMemcpyAsync(obst_found, o.found, (size_t)B * 4, cudaMemcpyDeviceToHost, h->stream));
    rc = fetch_outputs(h, io, B, u_seq, x_seq, dt_out, status, kkt_err, iters);
    float ms = 0.f;
    if (!rc && cudaEventElapsedTime(&ms, h->c0, h->c1) == cudaSuccess) h->costmap_ms = ms;
    return rc;
}

// the arguments of a feasibility check; *n = poses per trajectory
static int check_feasible_args(mpcb200_handle* h, int B, const mpcb200_costmaps* maps, const double* x_seq, int n_poses, const double* footprint_xy,
                               int n_footprint, double inscribed_radius, double min_resolution_angular, const unsigned char* feasible, int* n)
{
    if (!h) return MPCB200_E_INVALID;
    if (B < 1 || !maps || !maps->cost || !maps->origin || !feasible || n_footprint < 0 || (n_footprint > 0 && !footprint_xy))
        return set_err(h, MPCB200_E_INVALID, "check_feasible: B >= 1, maps, footprint and the output array are required");
    if (maps->size_x < 1 || maps->size_y < 1 || !(maps->resolution > 0)) return set_err(h, MPCB200_E_INVALID, "check_feasible: bad map geometry");
    if (!(inscribed_radius > 0) || !(min_resolution_angular > 0)) return set_err(h, MPCB200_E_INVALID, "check_feasible: inscribed_radius and min_resolution_angular must be > 0");
    *n = x_seq ? n_poses : h->cfg.n;
    if (*n < 1) return set_err(h, MPCB200_E_INVALID, "check_feasible: n_poses >= 1 required");
    if (!x_seq && (h->B < B)) return set_err(h, MPCB200_E_INVALID, "check_feasible: no solved batch of this size on the device (pass x_seq)");
    return 0;
}

extern "C" int mpcb200_check_feasible(mpcb200_handle* h, int B, const mpcb200_costmaps* maps, const double* x_seq, int n_poses, const double* footprint_xy,
                                      int n_footprint, double inscribed_radius, double circumscribed_radius, double min_resolution_angular,
                                      int look_ahead_idx, unsigned char* feasible)
{
    (void)circumscribed_radius;   // CostmapModel::footprintCost does not use it either
    int n = 0;
    if (int rc = check_feasible_args(h, B, maps, x_seq, n_poses, footprint_xy, n_footprint, inscribed_radius, min_resolution_angular, feasible, &n)) return rc;
    CK(cudaSetDevice(h->device));
    const size_t W = (size_t)maps->size_x, H = (size_t)maps->size_y;
    const size_t need = (size_t)B * n * 24 + (size_t)B * 16 + (size_t)(n_footprint > 0 ? n_footprint : 1) * 16 + (size_t)B * W * H + (size_t)B + 256;
    if (need > h->fz_cap)
    {
        if (h->d_fz) cudaFree(h->d_fz);
        h->d_fz = nullptr; h->fz_cap = 0;
        CK(cudaMalloc(&h->d_fz, need));
        h->fz_cap = need;
    }
    char* p = (char*)h->d_fz;
    double* d_x = (double*)p; p += (size_t)B * n * 24;
    double* d_origin = (double*)p; p += (size_t)B * 16;
    double* d_fp = (double*)p; p += (size_t)(n_footprint > 0 ? n_footprint : 1) * 16;
    unsigned char* d_cost = (unsigned char*)p; p += (size_t)B * W * H;
    unsigned char* d_ok = (unsigned char*)p;
    CK(cudaMemcpyAsync(d_cost, maps->cost, (size_t)B * W * H, cudaMemcpyHostToDevice, h->stream));
    CK(cudaMemcpyAsync(d_origin, maps->origin, (size_t)B * 16, cudaMemcpyHostToDevice, h->stream));
    if (n_footprint > 0) CK(cudaMemcpyAsync(d_fp, footprint_xy, (size_t)n_footprint * 16, cudaMemcpyHostToDevice, h->stream));
    if (x_seq) CK(cudaMemcpyAsync(d_x, x_seq, (size_t)B * n * 24, cudaMemcpyHostToDevice, h->stream));
    h->stats.h2d_bytes += (long long)((size_t)B * W * H + (size_t)B * 16 + (size_t)n_footprint * 16 + (x_seq ? (size_t)B * n * 24 : 0));
    FeasArgs a{maps->size_x, maps->size_y, maps->resolution, d_cost, d_origin, x_seq ? d_x : h->batch.xseq, n, d_fp, n_footprint,
               inscribed_radius, min_resolution_angular, look_ahead_idx};
    feasible_kernel<<<grid_for(B, WARPS_PER_CTA), WARPS_PER_CTA * 32, 0, h->stream>>>(a, B, d_ok);
    h->stats.launches_total += 1;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(feasible, d_ok, (size_t)B, cudaMemcpyDeviceToHost, h->stream));
    h->stats.d2h_bytes += B;
    CK(cudaStreamSynchronize(h->stream));
    return MPCB200_OK;
}

extern "C" double mpcb200_costmap_last_ms(const mpcb200_handle* h) { return h ? h->costmap_ms : 0.0; }

// ---- device-memory entry points: the paths above with device arrays, stream-ordered, no host synchronise ----------------------
// the phased mode polls from the host, so only the persistent solve kernel serves them
static int check_async(mpcb200_handle* h, unsigned flags, unsigned known)
{
    if (h->solve_mode == 1)
        return set_err(h, MPCB200_E_UNSUPPORTED, "the _async entry points need the fused solve kernel: MPCB200_OPT_SOLVE_MODE 1 polls from the host");
    if (flags & ~known) return set_err(h, MPCB200_E_INVALID, "unknown flags");
    return 0;
}

extern "C" int mpcb200_step_batch_async(mpcb200_handle* h, int B, const double* x0, const double* xf, const double* u_prev, double u_prev_dt,
                                        const mpcb200_obstacles* obst, const mpcb200_viapoints* vp, const double* x_init,
                                        const unsigned char* reinit, unsigned flags,
                                        double* u_seq, double* x_seq, double* dt_out, int* status, double* kkt_err, int* iters)
{
    int rc = check_batch(h, B);
    if (rc) return rc;
    if ((rc = check_async(h, flags, MPCB200_ASYNC_LINE_OBSTACLES))) return rc;
    if ((rc = check_robot_limits(h, B))) return rc;
    CK(cudaSetDevice(h->device));
    if ((rc = check_device_arrays(h, "step_batch_async", {x0, xf, u_prev, obst ? obst->count : nullptr, obst ? obst->type : nullptr,
                                                          obst ? obst->params : nullptr, vp ? vp->count : nullptr, vp ? vp->poses : nullptr,
                                                          x_init, reinit, u_seq, x_seq, dt_out, status, kkt_err, iters})))
        return rc;
    if ((rc = load_inputs(h, h->batch, B, x0, xf, u_prev, u_prev_dt, obst, vp, x_init, reinit, Mem::Device, flags))) return rc;
    h->B = B;
    if ((rc = launch_solve_async(h, h->batch, B))) return rc;
    return fetch_outputs(h, h->batch, B, u_seq, x_seq, dt_out, status, kkt_err, iters, Mem::Device);
}

extern "C" int mpcb200_step_batch_costmap_async(mpcb200_handle* h, int B, const double* x0, const double* xf, const double* u_prev,
                                                double u_prev_dt, const mpcb200_costmaps* maps, double behind_robot_dist, int max_per_instance,
                                                const mpcb200_viapoints* vp, const double* x_init, const unsigned char* reinit,
                                                double* u_seq, double* x_seq, double* dt_out, int* status, double* kkt_err, int* iters,
                                                int* obst_found)
{
    int rc = check_batch(h, B);
    if (rc) return rc;
    if (max_per_instance < 1 || max_per_instance > MAX_OBST_LIST) return set_err(h, MPCB200_E_UNSUPPORTED, "step_batch_costmap: 1..2048 obstacles per instance");
    if ((rc = check_async(h, 0u, 0u))) return rc;
    if ((rc = check_robot_limits(h, B))) return rc;
    if (!maps) return set_err(h, MPCB200_E_INVALID, "costmap_obstacles: B >= 1, maps, poses and output arrays are required");
    CK(cudaSetDevice(h->device));
    if ((rc = check_device_arrays(h, "step_batch_costmap_async", {maps->cost, maps->origin, x0, xf, u_prev, vp ? vp->count : nullptr,
                                                                  vp ? vp->poses : nullptr, x_init, reinit, u_seq, x_seq, dt_out, status,
                                                                  kkt_err, iters, obst_found})))
        return rc;
    IoBuffers& io = h->batch;
    if ((rc = io_reserve(h, io, io.rows, max_per_instance))) return rc;
    if ((rc = load_inputs(h, io, B, x0, xf, u_prev, u_prev_dt, nullptr, vp, x_init, reinit, Mem::Device))) return rc;
    CostmapOut o;
    if ((rc = costmap_run(h, B, maps, nullptr, io.x0, behind_robot_dist, max_per_instance, io.obst_count, io.obst_type, io.obst, &o, Mem::Device))) return rc;
    io.in.obst_count = io.obst_count; io.in.obst_max = max_per_instance;   // point obstacles only: no line-obstacle kernel variant needed
    h->B = B;
    if ((rc = launch_solve_async(h, io, B))) return rc;
    if (obst_found) CK(cudaMemcpyAsync(obst_found, o.found, (size_t)B * 4, cudaMemcpyDeviceToDevice, h->stream));
    return fetch_outputs(h, io, B, u_seq, x_seq, dt_out, status, kkt_err, iters, Mem::Device);
}

extern "C" int mpcb200_check_feasible_async(mpcb200_handle* h, int B, const mpcb200_costmaps* maps, const double* x_seq, int n_poses,
                                            const double* footprint_xy, int n_footprint, double inscribed_radius, double circumscribed_radius,
                                            double min_resolution_angular, int look_ahead_idx, unsigned char* feasible)
{
    (void)circumscribed_radius;
    int n = 0;
    if (int rc = check_feasible_args(h, B, maps, x_seq, n_poses, footprint_xy, n_footprint, inscribed_radius, min_resolution_angular, feasible, &n)) return rc;
    CK(cudaSetDevice(h->device));
    if (int rc = check_device_arrays(h, "check_feasible_async", {maps->cost, maps->origin, x_seq, n_footprint > 0 ? footprint_xy : nullptr, feasible}))
        return rc;
    // maps, footprint and trajectories are read in place; x_seq = NULL: the trajectories of the last solve
    FeasArgs a{maps->size_x, maps->size_y, maps->resolution, maps->cost, maps->origin, x_seq ? x_seq : h->batch.xseq, n, footprint_xy, n_footprint,
               inscribed_radius, min_resolution_angular, look_ahead_idx};
    feasible_kernel<<<grid_for(B, WARPS_PER_CTA), WARPS_PER_CTA * 32, 0, h->stream>>>(a, B, feasible);
    h->stats.launches_total += 1;
    CK(cudaGetLastError());
    return MPCB200_OK;
}

extern "C" int mpcb200_flush_l2(mpcb200_handle* h)
{
    if (!h) return MPCB200_E_INVALID;
    CK(cudaSetDevice(h->device));
    flush_kernel<<<h->num_sms * 8, 256, 0, h->stream>>>(h->d_flush, h->flush_n);
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(h->stream));
    return 0;
}

// =================================================================================================================
// several devices of one node behind one handle (SURVEY 8e): instances are independent, so the batch is cut into contiguous
// blocks, one per device; every device solves its block with its own handle on its own stream (one host thread each), and ONE
// NCCL all-gather over NVLink leaves the packed optimal controls of the whole batch on every device.  No other collective.
// NCCL is loaded at run time (dlopen) when a multi-device handle is created: the single-device library has no NCCL dependency.
// =================================================================================================================
#include <dlfcn.h>
#include <thread>

struct NcclApi
{
    void* lib = nullptr;
    int (*CommInitAll)(void**, int, const int*) = nullptr;
    int (*CommDestroy)(void*) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
};
#define MPC_NCCL_FLOAT64 8   /* ncclFloat64 / ncclDouble (nccl.h) */

struct mpcb200_multi
{
    int n_dev = 0, max_per = 0, n = 0;
    std::vector<int> devices;
    std::vector<mpcb200_handle*> h;
    std::vector<void*> comm;
    std::vector<double*> d_all;      // per device: gathered packed controls [n_dev][max_per][N-1][2]
    NcclApi nccl;
    std::string err;
};
static std::string g_multi_err = "";
static int multi_err(mpcb200_multi* m, int code, const std::string& msg) { if (m) m->err = msg; else g_multi_err = msg; return code; }

static bool load_nccl(NcclApi& a, std::string& why)
{
    const char* names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char* nm : names) { a.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); if (a.lib) break; }
    if (!a.lib) { why = std::string("NCCL not found (dlopen libnccl.so.2): ") + (dlerror() ? dlerror() : ""); return false; }
#define NSYM(field, name) a.field = (decltype(a.field))dlsym(a.lib, name); if (!a.field) { why = std::string("NCCL symbol missing: ") + name; return false; }
    NSYM(CommInitAll, "ncclCommInitAll") NSYM(CommDestroy, "ncclCommDestroy") NSYM(AllGather, "ncclAllGather")
    NSYM(GroupStart, "ncclGroupStart") NSYM(GroupEnd, "ncclGroupEnd") NSYM(GetErrorString, "ncclGetErrorString")
#undef NSYM
    return true;
}

extern "C" void mpcb200_destroy_multi(mpcb200_multi* m)
{
    if (!m) return;
    for (size_t r = 0; r < m->comm.size(); ++r) if (m->comm[r] && m->nccl.CommDestroy) m->nccl.CommDestroy(m->comm[r]);
    for (size_t r = 0; r < m->d_all.size(); ++r) if (m->d_all[r]) { cudaSetDevice(m->devices[r]); cudaFree(m->d_all[r]); }
    for (auto* h : m->h) if (h) mpcb200_destroy(h);
    delete m;
}

extern "C" int mpcb200_create_multi(const mpcb200_config* cfg, int max_batch_total, const int* devices, int n_devices, mpcb200_multi** out)
{
    if (!cfg || !out || max_batch_total < 1 || !devices || n_devices < 1) return multi_err(nullptr, MPCB200_E_INVALID, "bad arguments");
    mpcb200_multi* m = new mpcb200_multi();
    m->n_dev = n_devices; m->n = cfg->n;
    m->max_per = (max_batch_total + n_devices - 1) / n_devices;
    m->devices.assign(devices, devices + n_devices);
    m->h.assign(n_devices, nullptr); m->comm.assign(n_devices, nullptr); m->d_all.assign(n_devices, nullptr);
    for (int r = 0; r < n_devices; ++r)
    {
        const int rc = mpcb200_create(cfg, m->max_per, devices[r], &m->h[r]);
        if (rc) { const std::string e = mpcb200_last_error(nullptr); mpcb200_destroy_multi(m); return multi_err(nullptr, rc, e); }
    }
    if (n_devices > 1)
    {
        std::string why;
        if (!load_nccl(m->nccl, why)) { mpcb200_destroy_multi(m); return multi_err(nullptr, MPCB200_E_UNSUPPORTED, why); }
        const int nrc = m->nccl.CommInitAll(m->comm.data(), n_devices, devices);
        if (nrc != 0) { const std::string e = std::string("ncclCommInitAll: ") + m->nccl.GetErrorString(nrc); mpcb200_destroy_multi(m); return multi_err(nullptr, MPCB200_E_CUDA, e); }
    }
    const size_t words = (size_t)n_devices * m->max_per * (cfg->n - 1) * 2;
    for (int r = 0; r < n_devices; ++r)
    {
        if (cudaSetDevice(devices[r]) != cudaSuccess || cudaMalloc(&m->d_all[r], words * 8) != cudaSuccess)
        { mpcb200_destroy_multi(m); return multi_err(nullptr, MPCB200_E_CUDA, "cudaMalloc of the gathered controls failed"); }
    }
    *out = m;
    return MPCB200_OK;
}

extern "C" const char* mpcb200_multi_last_error(const mpcb200_multi* m) { return m ? m->err.c_str() : g_multi_err.c_str(); }
extern "C" mpcb200_handle* mpcb200_multi_handle(mpcb200_multi* m, int rank) { return (m && rank >= 0 && rank < m->n_dev) ? m->h[rank] : nullptr; }
extern "C" int mpcb200_multi_device_controls(mpcb200_multi* m, int rank, void** dev_ptr, long long* n_doubles)
{
    if (!m || rank < 0 || rank >= m->n_dev) return MPCB200_E_INVALID;
    if (dev_ptr) *dev_ptr = m->d_all[rank];
    if (n_doubles) *n_doubles = (long long)m->n_dev * m->max_per * (m->n - 1) * 2;
    return MPCB200_OK;
}

extern "C" int mpcb200_multi_fetch_controls(mpcb200_multi* m, int rank, double* host)
{
    if (!m || rank < 0 || rank >= m->n_dev || !host) return MPCB200_E_INVALID;
    if (cudaSetDevice(m->devices[rank]) != cudaSuccess ||
        cudaMemcpy(host, m->d_all[rank], (size_t)m->n_dev * m->max_per * (m->n - 1) * 16, cudaMemcpyDeviceToHost) != cudaSuccess)
        return multi_err(m, MPCB200_E_CUDA, "copy of the gathered controls failed");
    return MPCB200_OK;
}

extern "C" int mpcb200_step_batch_multi(mpcb200_multi* m, int B, const double* x0, const double* xf, const double* u_prev, double u_prev_dt,
                                        const mpcb200_obstacles* obst, const mpcb200_viapoints* vp, const double* x_init, const unsigned char* reinit,
                                        double* u_seq, double* x_seq, double* dt_out, int* status, double* kkt_err, int* iters, double* solve_time_s)
{
    if (!m) return MPCB200_E_INVALID;
    if (B < 1 || B > m->n_dev * m->max_per) return multi_err(m, MPCB200_E_INVALID, "batch size out of range");
    const int G = m->n_dev, N = m->n;
    const int per = (B + G - 1) / G;   // contiguous blocks: device r gets instances [r per, min((r+1) per, B))
    std::vector<int> rcs(G, 0);
    std::vector<double> secs(G, 0.0);
    std::vector<std::thread> th;
    for (int r = 0; r < G; ++r)
    {
        const int b0 = r * per, nb = std::max(0, std::min(per, B - b0));
        if (nb == 0) continue;
        th.emplace_back([=, &rcs, &secs]() {
            mpcb200_obstacles ob; mpcb200_viapoints vv;
            const mpcb200_obstacles* pob = nullptr; const mpcb200_viapoints* pvp = nullptr;
            if (obst && obst->count && obst->max_per_instance > 0)
            {
                const size_t M = (size_t)obst->max_per_instance;
                ob.max_per_instance = obst->max_per_instance; ob.count = obst->count + b0; ob.type = obst->type + (size_t)b0 * M;
                ob.params = obst->params + (size_t)b0 * M * MPCB200_OBST_STRIDE;
                pob = &ob;
            }
            if (vp && vp->count && vp->max_per_instance > 0)
            {
                vv.max_per_instance = vp->max_per_instance; vv.count = vp->count + b0; vv.poses = vp->poses + (size_t)b0 * vp->max_per_instance * 3;
                pvp = &vv;
            }
            rcs[r] = mpcb200_step_batch(m->h[r], nb, x0 + (size_t)b0 * 3, xf + (size_t)b0 * 3, u_prev ? u_prev + (size_t)b0 * 2 : nullptr, u_prev_dt, pob, pvp,
                                        x_init ? x_init + (size_t)b0 * N * 3 : nullptr, reinit ? reinit + b0 : nullptr,
                                        u_seq ? u_seq + (size_t)b0 * N * 2 : nullptr, x_seq ? x_seq + (size_t)b0 * N * 3 : nullptr, dt_out ? dt_out + b0 : nullptr,
                                        status ? status + b0 : nullptr, kkt_err ? kkt_err + b0 : nullptr, iters ? iters + b0 : nullptr, &secs[r]);
        });
    }
    for (auto& t : th) t.join();
    for (int r = 0; r < G; ++r)
        if (rcs[r]) return multi_err(m, rcs[r], std::string("device ") + std::to_string(m->devices[r]) + ": " + mpcb200_last_error(m->h[r]));
    // ---- all-gather of the packed optimal controls: every device ends up with u* of every instance ----
    const size_t count = (size_t)per * (N - 1) * 2;
    if (G > 1)
    {
        int nrc = m->nccl.GroupStart();
        for (int r = 0; r < G && nrc == 0; ++r)
        {
            cudaSetDevice(m->devices[r]);
            nrc = m->nccl.AllGather(m->h[r]->batch.upacked, m->d_all[r], count, MPC_NCCL_FLOAT64, m->comm[r], m->h[r]->stream);
        }
        const int erc = m->nccl.GroupEnd();
        if (nrc == 0) nrc = erc;
        if (nrc != 0) return multi_err(m, MPCB200_E_CUDA, std::string("ncclAllGather: ") + m->nccl.GetErrorString(nrc));
        for (int r = 0; r < G; ++r)
        {
            cudaSetDevice(m->devices[r]);
            if (cudaStreamSynchronize(m->h[r]->stream) != cudaSuccess) return multi_err(m, MPCB200_E_CUDA, "stream synchronisation after the all-gather failed");
        }
    }
    else
    {
        cudaSetDevice(m->devices[0]);
        if (cudaMemcpyAsync(m->d_all[0], m->h[0]->batch.upacked, count * 8, cudaMemcpyDeviceToDevice, m->h[0]->stream) != cudaSuccess ||
            cudaStreamSynchronize(m->h[0]->stream) != cudaSuccess)
            return multi_err(m, MPCB200_E_CUDA, "copy of the controls failed");
    }
    if (solve_time_s) { double mx = 0.0; for (double s_ : secs) mx = s_ > mx ? s_ : mx; *solve_time_s = mx; }
    return MPCB200_OK;
}
#endif  // MPCB200_ENTRY_UNIT
