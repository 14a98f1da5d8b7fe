// mpc_gate.h -- the phase gates of the solve kernel: one barrier per SM whose membership changes while the CTAs iterate.
//
// The barrier is one 64-bit word, generation (bits 32..63) | arrived (16..31) | members (0..15).  A CTA is a member while it
// iterates on an instance (join after the association, leave after the last iteration).  The generation counts the barriers that
// opened; generation mod nph is the phase the barrier opens (eval, KKT, line search with three gates; KKT, line search with two),
// and a CTA that arrives out of step keeps arriving until the generation matches its phase.
//
// An arrival is one atomic add; its return value tells the CTA whether it is the last to arrive.  The last one opens the barrier
// with one more add (generation + 1, arrived count back to 0).  Between those two adds every member has arrived and waits, so no
// one arrives; join waits for the release so that it never counts itself into a barrier that is opening, and a member that
// leaves has not arrived, so it never sees that state.  A CTA that leaves opens the barrier if the others waited for it only.
//
// The protocol is written once for the device (CUDA atomics) and for the CPU test of tests/emu/gate_stress.cpp (std::atomic),
// through an atomic policy A: A::Word, add (returns the old value), cas (returns the old value), load and pause.  The word
// orders nothing but itself (no data crosses CTAs), so relaxed atomics and loads are enough.
#pragma once

#ifdef __CUDACC__
#define GATE_HD __host__ __device__ __forceinline__
#else
#define GATE_HD inline
#endif

namespace gate
{
typedef unsigned long long u64;
constexpr u64 ARRIVE_ONE = 1ull << 16, GEN_ONE = 1ull << 32;
GATE_HD unsigned members(u64 w) { return (unsigned)(w & 0xFFFFull); }
GATE_HD unsigned arrived(u64 w) { return (unsigned)((w >> 16) & 0xFFFFull); }
GATE_HD unsigned generation(u64 w) { return (unsigned)(w >> 32); }

template <class A> GATE_HD void join(typename A::Word* st)
{
    u64 old = A::load(st);
    for (;;)
    {
        if (arrived(old) > 0u && arrived(old) >= members(old)) { A::pause(); old = A::load(st); continue; }   // being released
        const u64 seen = A::cas(st, old, old + 1ull);
        if (seen == old) return;
        old = seen;
    }
}

template <class A> GATE_HD void leave(typename A::Word* st)
{
    u64 old = A::load(st);
    for (;;)
    {
        const unsigned m = members(old) - 1u, ar = arrived(old);
        const u64 next = ar > 0u && ar >= m ? ((u64)(generation(old) + 1u) << 32) | m : old - 1ull;   // the others waited for this CTA only
        const u64 seen = A::cas(st, old, next);
        if (seen == old) return;
        old = seen;
    }
}

// Returns once a barrier of phase `phase` has opened; the value is the member count the CTA saw at that arrival.
template <class A> GATE_HD unsigned arrive(typename A::Word* st, unsigned phase, unsigned nph)
{
    for (;;)
    {
        const u64 old = A::add(st, ARRIVE_ONE);
        const unsigned g = generation(old), ar = arrived(old) + 1u;
        if (ar >= members(old)) A::add(st, GEN_ONE - (u64)ar * ARRIVE_ONE);
        else
            while (generation(A::load(st)) == g) A::pause();
        if (g % nph == phase) return members(old);
    }
}
}  // namespace gate
