// robot_model_emu.cpp -- the per-robot-model functions of the device headers on the CPU (TEST INFRASTRUCTURE): the emulator
// (emu/emu.cpp, compiled into this library with the flags of emu/Makefile) and the validity check and configuration patch that
// the solve kernel and the blocking setters call (robot_model_valid / apply_robot_model, mpc_core.h).
#include "../emu/emu.cpp"

extern "C" int emu_robot_model_valid(const Cfg* c, const double* model, const double* geo) { return robot_model_valid(*c, model, geo) ? 1 : 0; }
extern "C" void emu_apply_robot_model(Cfg* c, const double* model) { apply_robot_model(*c, model); }
