// robot_weights_emu.cpp -- the per-robot-weights functions of the device headers on the CPU (TEST INFRASTRUCTURE): the emulator
// (emu/emu.cpp, compiled into this library with the flags of emu/Makefile) and the validity check and configuration patch that
// the solve kernel and the blocking setter call (robot_weights_valid / apply_robot_weights, mpc_core.h).
#include "../emu/emu.cpp"

extern "C" int emu_robot_weights_valid(const Cfg* c, const double* rec) { return robot_weights_valid(*c, rec) ? 1 : 0; }
extern "C" void emu_apply_robot_weights(Cfg* c, const double* rec) { apply_robot_weights(*c, rec); }
