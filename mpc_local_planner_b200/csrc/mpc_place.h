// mpc_place.h -- which instance a CTA of the solve kernel takes when the critical placement is on (MPCB200_OPT_CRITICAL_PLACEMENT).
//
// A batch ordered longest first by history ends with its slowest instance, and an instance runs its iterations faster on an SM
// it shares with fewer CTAs.  So the H leading instances of the order (the heavy part, H <= the SM count, planned by
// order_by_history_kernel) go one per SM, to SMs that keep at most `cotenants` other CTAs:
//   - admission, once per CTA at its first take: one add on its SM's word gives the CTA its arrival rank on the SM.  The
//     first CTA of an SM claims the next heavy instance (a shared claim counter) and publishes in the same word whether the SM
//     became heavy; the later CTAs wait for that (the first CTA is resident and has only its claim left to do).  On a heavy SM
//     the CTAs of rank > cotenants exit without taking anything;
//   - takes: the light part order[H..total) through the queue counter, which starts at H, then whatever heavy instance no CTA
//     has claimed (a heavy part larger than the SMs that got a CTA).
// Every instance is taken exactly once (each one through exactly one counter), and the first CTA of every SM takes instances
// until both parts are drained, so the launch terminates.  Order of execution only: results are bit-identical.
//
// Written once for the device (CUDA atomics) and for the CPU test of tests/emu/place_stress.cpp (std::atomic), through an
// atomic policy A as in mpc_gate.h: A::Word, add on a Word and on an int (both return the old value), load of a Word, pause.
#pragma once

#ifdef __CUDACC__
#define PLACE_HD __host__ __device__ __forceinline__
#else
#define PLACE_HD inline
#endif

namespace place
{
typedef unsigned long long u64;
constexpr u64 RANK_MASK = 0xFFFFFFFFull, DECIDED = 1ull << 32, HEAVY = 1ull << 33;   // the SM word: arrivals | decided | heavy
constexpr int TAKE = -1;    // admission: take from the queue
constexpr int LEAVE = -2;   // admission: exit without an instance
constexpr int ADMIT = -3;   // before the first take of a CTA: admission first

// heavy[0] = H, heavy[1] = heavy instances claimed so far.  Returns a heavy instance, TAKE or LEAVE.
template <class A> PLACE_HD int admit(typename A::Word* sm, int* heavy, const int* order, unsigned cotenants)
{
    const u64 old = A::add(sm, 1ull);
    const unsigned rank = (unsigned)(old & RANK_MASK);
    if (rank == 0u)
    {
        const int h = A::add(heavy + 1, 1);
        A::add(sm, h < heavy[0] ? DECIDED | HEAVY : DECIDED);
        return h < heavy[0] ? order[h] : TAKE;
    }
    u64 w = old;
    while (!(w & DECIDED)) { A::pause(); w = A::load(sm); }
    return (w & HEAVY) && rank > cotenants ? LEAVE : TAKE;
}

// Returns the next instance, or `total` once both parts are drained.
template <class A> PLACE_HD int take(int* queue, int* heavy, const int* order, int total)
{
    const int q = A::add(queue, 1);
    if (q < total) return order[q];
    const int h = A::add(heavy + 1, 1);
    return h < heavy[0] ? order[h] : total;
}
}  // namespace place
