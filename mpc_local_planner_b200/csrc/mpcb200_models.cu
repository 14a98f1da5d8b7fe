// mpcb200_models.cu -- the per-robot-model entries of the solve kernel (solve_fused_models_kernel, mpcb200.cu: the MODEL_GENERIC
// variants, 16 instantiations) in a translation unit of their own.  The build compiles it beside mpcb200.cu and mpcb200_weights.cu,
// so the table adds no time to the library's build, and the compiles of the other two units hold the same kernels as before.
#define MPCB200_ENTRY_UNIT
#include "mpcb200.cu"

// every key maps to the MODEL_GENERIC entry: the types are read from the CTA's configuration at run time
struct ModelsEntry
{
    template <bool LINES, bool EXT, int WARPS, int MODEL, bool MULTI> static constexpr auto get() { return solve_fused_models_kernel<LINES, EXT, WARPS, MODEL_GENERIC, MULTI>; }
};

const void* models_kernel_variant(bool lines, bool ext, bool small, bool multi)
{
    return reinterpret_cast<const void*>(fused_variant<ModelsEntry>(lines, ext, small, MODEL_GENERIC, multi));
}
