// ranked_emu.cpp -- the emulator's cold initial guess from the bumped line of rank `rank` (TEST INFRASTRUCTURE): the emulator
// (emu/emu.cpp, compiled into this library with the flags of emu/Makefile) and the serial ranking of the device headers
// (bump_select_serial -> bump_ranked_amplitude, mpc_stage.h), the cold branch of emu_init with a rank.
#include "../emu/emu.cpp"

extern "C" void emu_init_cold_rank(const Cfg* cp, double* W, int rank)
{
    const Cfg& c = *cp;
    WsLayout L;
    make_layout(cp, MAX_OBST, MAX_VP, L);
    for (int k = 0; k < L.N; ++k) init_cold_stage(c, L, W, k, W + L.oXINIT);
    bump_select_serial(c, L, W, rank);
    ASC(MPCB200_SC_DT) = c.dt_ref;
    ASC(MPCB200_SC_COLD) = 2.0;
}
