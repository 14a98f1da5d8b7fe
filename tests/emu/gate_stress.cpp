// gate_stress.cpp -- the phase-gate protocol of the solve kernel (mpc_gate.h) on the CPU, TEST INFRASTRUCTURE.
//
// Threads play the CTAs of one SM: they take instances from a shared queue, join, run the gate sequence of solve_fused_kernel
// (gate, eval, [done], gate, KKT, [given up], gate, line search, ...) for a random number of iterations with random work in
// between, leave, and take the next instance.  Like the kernel, a thread that arrives after the queue is drained -- alone on
// the SM, or in any case with <tail> = 1 (the kernel's longest-first order) -- leaves and runs its remaining iterations
// without gates.  Checked:
//   - a barrier opens only when all its members have arrived: while a member works between two gates (or between its join and
//     its first arrival) the generation does not change;
//   - an arrival returns at a barrier of its own phase;
//   - at the end the word is back to no members and no arrivals;
//   - no deadlock: every thread finishes within the time limit (otherwise the program exits with status 2).
// usage: gate_stress <threads> <gates 2|3> <instances> <seed> <tail 0|1>; exit status 0 when every check holds.
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <thread>
#include <vector>

#include "../../mpc_local_planner_b200/csrc/mpc_gate.h"

struct HostAtomics
{
    typedef std::atomic<unsigned long long> Word;
    static unsigned long long add(Word* w, unsigned long long v) { return w->fetch_add(v); }
    static unsigned long long cas(Word* w, unsigned long long expected, unsigned long long desired)
    {
        w->compare_exchange_strong(expected, desired);
        return expected;   // the value seen: equal to the argument exactly when the exchange happened
    }
    static unsigned long long load(Word* w) { return w->load(std::memory_order_acquire); }
    static void pause() { std::this_thread::yield(); }
};

static std::atomic<unsigned long long> word{0};
static std::atomic<int> queue{0}, errors{0}, finished{0};
static std::atomic<long long> barriers_passed{0};

static void fail(const char* what, int t)
{
    if (errors.fetch_add(1) < 10) std::fprintf(stderr, "thread %d: %s\n", t, what);
}

// random work of a member: the generation must stay what it was when the work began
static void work(std::mt19937& rng, unsigned gen, int t)
{
    const int spin = (int)(rng() % 200u);
    for (volatile int i = 0; i < spin; ++i) {}
    if (rng() % 8u == 0u) std::this_thread::yield();
    if (gate::generation(HostAtomics::load(&word)) != gen) fail("a barrier opened while a member was working", t);
}

static void cta(int t, unsigned nph, int total, unsigned seed, bool tail)
{
    std::mt19937 rng(seed * 7919u + (unsigned)t);
    bool gated = true;   // false: left after the queue drained, no more gates in this launch
    auto gate_at = [&](unsigned phase)
    {
        if (!gated) return;
        const bool drained = queue.load() >= total;
        const unsigned m = gate::arrive<HostAtomics>(&word, phase, nph);
        const unsigned g = gate::generation(HostAtomics::load(&word));
        if ((g - 1u) % nph != phase) fail("an arrival returned at a barrier of another phase", t);
        barriers_passed.fetch_add(1);
        if ((m == 1u || tail) && drained) { gate::leave<HostAtomics>(&word); gated = false; return; }
        work(rng, g, t);
    };
    for (;;)
    {
        const int q = queue.fetch_add(1);
        if (q >= total) break;
        const int outer = 1 + (int)(rng() % 2u);
        for (int oi = 0; oi < outer; ++oi)
        {
            if (rng() % 4u == 0u) std::this_thread::yield();   // set-up / association of the instance: not a member
            if (gated)
            {
                gate::join<HostAtomics>(&word);
                work(rng, gate::generation(HostAtomics::load(&word)), t);
            }
            const int iters = 1 + (int)(rng() % 12u);
            for (int it = 0;; ++it)
            {
                if (nph == 3u) gate_at(0u);
                if (it == iters) break;   // converged at this evaluation
                gate_at(nph - 2u);
                if (rng() % 64u == 0u) break;   // inertia correction failed: given up
                gate_at(nph - 1u);
                if (rng() % 64u == 0u) break;   // line search jammed: given up
            }
            if (gated) gate::leave<HostAtomics>(&word);
        }
    }
    finished.fetch_add(1);
}

int main(int argc, char** argv)
{
    if (argc != 6) { std::fprintf(stderr, "usage: gate_stress <threads> <gates 2|3> <instances> <seed> <tail 0|1>\n"); return 1; }
    const int nt = std::atoi(argv[1]), total = std::atoi(argv[3]);
    const unsigned nph = (unsigned)std::atoi(argv[2]), seed = (unsigned)std::atoi(argv[4]);
    const bool tail = std::atoi(argv[5]) != 0;
    std::vector<std::thread> th;
    for (int t = 0; t < nt; ++t) th.emplace_back(cta, t, nph, total, seed, tail);
    const auto t0 = std::chrono::steady_clock::now();
    while (finished.load() < nt)
    {
        std::this_thread::sleep_for(std::chrono::milliseconds(5));
        if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(20))
        {
            const unsigned long long w = word.load();
            std::fprintf(stderr, "deadlock: %d of %d threads finished, generation %u arrived %u members %u\n", finished.load(), nt,
                         gate::generation(w), gate::arrived(w), gate::members(w));
            std::fflush(stderr);
            std::_Exit(2);
        }
    }
    for (auto& x : th) x.join();
    const unsigned long long w = word.load();
    if (gate::members(w) != 0u || gate::arrived(w) != 0u) fail("the word does not return to no members and no arrivals", -1);
    std::printf("threads %d gates %u instances %d: %lld barriers passed, %u opened, %d errors\n", nt, nph, total,
                barriers_passed.load(), gate::generation(w), errors.load());
    return errors.load() ? 1 : 0;
}
