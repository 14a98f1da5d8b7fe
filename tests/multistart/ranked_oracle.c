/* ranked_oracle.c -- the oracle's cold initial guess from the bumped line of rank `rank`, the initial guess of multistart challenger
 * k = rank (TEST INFRASTRUCTURE).  The oracle itself (mpc_oracle.c) is compiled into this library with the flags of
 * oracle/Makefile; on top of it the lines are ordered by repeated selection with orc_init_cold's rule (strictly better beyond
 * rounding noise, lower m first), the lines of the lower ranks left out.  Rank 0 is orc_init_cold. */
#include "../../oracle/mpc_oracle.c"

void orc_init_cold_rank(const orc_problem* p, int rank, orc_ws* ws)
{
    orc_problem line = *p;
    line.n_obst = 0;
    orc_init_cold(&line, NULL, ws);   /* the straight line start -> goal, zero controls, dt = dt_ref */
    const int N = ws->N;
    const int nb = p->cfg->reference_initial_guess ? 0 : p->cfg->initial_guess_bumps;
    if (nb <= 0 || p->n_obst <= 0 || (rank > 0 && 2 * nb + 1 > 64)) return;
    double nx = -(p->xf[1] - p->x0[1]), ny = p->xf[0] - p->x0[0];
    const double nn = sqrt(nx * nx + ny * ny);
    if (!(nn > 1e-9)) return;
    nx /= nn; ny /= nn;
    double best_a = 0.0;
    unsigned long long taken = 0ull;
    for (int r = 0; r <= rank; ++r)
    {
        double best = 1e300;
        int best_i = -1;
        for (int m = -nb; m <= nb; ++m)
        {
            if (r > 0 && ((taken >> (m + nb)) & 1ull)) continue;
            const double A = ORC_BUMP_STEP * (double)m;
            const double score = bump_score(p, ws, A, nx, ny);
            if (score < best - 1e-9 * (1.0 + best)) { best = score; best_a = A; best_i = m + nb; }
        }
        if (best_i < 0 || r == rank) break;
        taken |= 1ull << best_i;
    }
    for (int k = 1; k <= N - 2; ++k)
    {
        const double o = best_a * sin(M_PI * (double)k / (double)(N - 1));
        ws->X[IX(0, k)] += o * nx;
        ws->X[IX(1, k)] += o * ny;
    }
    if (best_a != 0.0 && p->cfg->robot_type != MPCB200_ROBOT_UNICYCLE)
        for (int k = 1; k <= N - 2; ++k)
            ws->X[IX(2, k)] = atan2(ws->X[IX(1, k + 1)] - ws->X[IX(1, k - 1)], ws->X[IX(0, k + 1)] - ws->X[IX(0, k - 1)]);
}
