// robot_geometry_emu.cpp -- the per-robot-geometry functions of the device headers on the CPU (TEST INFRASTRUCTURE): the emulator
// (emu/emu.cpp, compiled into this library with the flags of emu/Makefile) and the validity check and configuration patch that
// the solve kernel and the blocking setter call (robot_geometry_valid / apply_robot_geometry, mpc_core.h).
#include "../emu/emu.cpp"

extern "C" int emu_robot_geometry_valid(const Cfg* c, const double* rec) { return robot_geometry_valid(*c, rec) ? 1 : 0; }
extern "C" void emu_apply_robot_geometry(Cfg* c, const double* rec) { apply_robot_geometry(*c, rec); }
