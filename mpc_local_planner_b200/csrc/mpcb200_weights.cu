// mpcb200_weights.cu -- the per-robot-weights entries of the solve kernel (solve_fused_weights_kernel, mpcb200.cu: the full
// variant table, 28 instantiations) in a translation unit of their own.  The build compiles it beside mpcb200.cu, so the table
// adds no time to the library's build, and the compile of mpcb200.cu holds the same kernels as before the table existed.
#define MPCB200_ENTRY_UNIT
#include "mpcb200.cu"

struct WeightsEntry
{
    template <bool LINES, bool EXT, int WARPS, int MODEL, bool MULTI> static constexpr auto get() { return solve_fused_weights_kernel<LINES, EXT, WARPS, MODEL, MULTI>; }
};

const void* weights_kernel_variant(bool lines, bool ext, bool small, int model, bool multi)
{
    return reinterpret_cast<const void*>(fused_variant<WeightsEntry>(lines, ext, small, model, multi));
}
