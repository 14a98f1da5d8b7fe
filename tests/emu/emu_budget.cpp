// emu_budget.cpp -- the CPU warp emulator (emu.cpp, TEST INFRASTRUCTURE) with the time budget of a solve (mpcb200_config.max_cpu_time).
//
// The emulator has no clock: the budget is made to run out just before the evaluation of a chosen iteration, and from then on every
// evaluation sees it expired -- the decision thread 0 of solve_fused_kernel takes from %globaltimer.  Compiled as one unit with emu.cpp,
// so that the solve without a budget (emu_solve) and the one with it run the same code.
#include "emu.cpp"

extern "C" {

// emu_eval with the budget state of the solve passed in (eval_finish tests it after the iteration cap)
static int eval_budget(const Cfg* cp, double* W, double uprev_dt, bool expired)
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
    const double mu = eval_finish(c, L, W, a[0], true, &fin, expired);
    if (fin) return 1;
    for (int k = 0; k < N; ++k) eval_finalize_stage(L, W, k, mu);
    return 0;
}

// emu_solve with a budget that runs out just before the evaluation of iteration `expire_at` (iterations counted over all outer
// iterations of the solve): the control flow of solve_fused_kernel under max_cpu_time, where an instance the budget stopped runs no
// further outer iteration
int emu_solve_expiring(const Cfg* cp, double* W, double uprev_dt, int force_cold, int expire_at)
{
    const Cfg& c = *cp;
    WsLayout L;
    make_layout(cp, MAX_OBST, MAX_VP, L);
    emu_init(cp, W, force_cold);
    const int outer = c.outer_iterations > 0 ? c.outer_iterations : 1;
    int done = 0;   // iterations of this solve so far
    for (int oi = 0; oi < outer; ++oi)
    {
        emu_associate(cp, W, uprev_dt, oi == 0);
        for (int it = 0; it <= c.max_iter; ++it)
        {
            if (eval_budget(cp, W, uprev_dt, done >= expire_at)) break;
            if (it == c.max_iter) break;
            if (emu_kkt(cp, W)) break;
            emu_linesearch(cp, W, uprev_dt);
            ++done;
        }
        if (ASC(MPCB200_SC_STATUS) == (double)MPCB200_STATUS_MAX_TIME) break;
    }
    const double st = ASC(MPCB200_SC_STATUS);
    return st < 0 ? MPCB200_STATUS_MAX_ITER : (int)st;
}

}  // extern "C"
