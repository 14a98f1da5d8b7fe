// robot_limits_emu.cpp -- the per-robot-limits functions of the device headers on the CPU (TEST INFRASTRUCTURE): the emulator
// (emu/emu.cpp, compiled into this library with the flags of emu/Makefile) and the validity check and configuration patch that
// the solve kernel and the blocking setter call (robot_limits_valid / apply_robot_limits, mpc_core.h).
#include "../emu/emu.cpp"

extern "C" int emu_robot_limits_valid(const Cfg* c, const double* rec) { return robot_limits_valid(*c, rec) ? 1 : 0; }
extern "C" void emu_apply_robot_limits(Cfg* c, const double* rec) { apply_robot_limits(*c, rec); }
