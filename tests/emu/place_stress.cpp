// place_stress.cpp -- the critical placement of the solve kernel (mpc_place.h) on the CPU, TEST INFRASTRUCTURE.
//
// Threads play the CTAs of a launch: <sms> SMs with <per_sm> CTAs each, the last <absent> of them without an admission word (PTX
// does not promise %smid < the SM count), started in a random order with random delays.  Each CTA runs the kernel's take step:
// admission on its SM's word, then takes until it gets `total`, with random work per instance.  Checked:
//   - every instance of the order is taken exactly once;
//   - an SM whose first CTA took a heavy instance runs at most 1 + <cotenants> CTAs; the others exit without an instance;
//   - admission hands out heavy instances only, at most one per SM, and the heavy part is drained in every run;
//   - the launch terminates: every thread finishes within the time limit (otherwise the program exits with status 2).
// usage: place_stress <sms> <per_sm> <absent> <total> <H> <cotenants> <seed>; exit status 0 when every check holds.
#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <thread>
#include <vector>

#include "../../mpc_local_planner_b200/csrc/mpc_place.h"

struct HostAtomics
{
    typedef std::atomic<unsigned long long> Word;
    static unsigned long long add(Word* w, unsigned long long v) { return w->fetch_add(v); }
    static int add(int* w, int v) { return __atomic_fetch_add(w, v, __ATOMIC_RELAXED); }
    static unsigned long long load(Word* w) { return w->load(std::memory_order_relaxed); }
    static void pause() { std::this_thread::yield(); }
};

static std::atomic<int> errors{0}, finished{0};

static void fail(const char* what, int t)
{
    if (errors.fetch_add(1) < 10) std::fprintf(stderr, "CTA %d: %s\n", t, what);
}

int main(int argc, char** argv)
{
    if (argc != 8) { std::fprintf(stderr, "usage: place_stress <sms> <per_sm> <absent> <total> <H> <cotenants> <seed>\n"); return 1; }
    const int sms = std::atoi(argv[1]), per_sm = std::atoi(argv[2]), absent = std::atoi(argv[3]), total = std::atoi(argv[4]);
    const int H = std::atoi(argv[5]);
    const unsigned cotenants = (unsigned)std::atoi(argv[6]), seed = (unsigned)std::atoi(argv[7]);
    const int words = sms - absent, ctas = sms * per_sm;
    std::mt19937 rng(seed);
    std::vector<int> order(total);
    for (int i = 0; i < total; ++i) order[i] = i;
    std::shuffle(order.begin(), order.end(), rng);
    std::vector<HostAtomics::Word> sm_word(words);
    for (auto& w : sm_word) w.store(0ull);
    int heavy[2] = {H, 0};   // [0] H, [1] claims
    int queue = H;           // the light part starts at H
    std::vector<std::atomic<int>> taken(total);
    for (auto& x : taken) x.store(0);
    std::vector<std::atomic<int>> running(sms), heavy_at_admission(sms);
    for (int s = 0; s < sms; ++s) { running[s].store(0); heavy_at_admission[s].store(0); }
    std::vector<int> start(ctas);   // CTA t -> SM; the threads start in a random order
    for (int t = 0; t < ctas; ++t) start[t] = t % sms;
    std::shuffle(start.begin(), start.end(), rng);

    auto cta = [&](int t)
    {
        std::mt19937 r(seed * 7919u + (unsigned)t);
        const int sm = start[t];
        for (volatile int i = 0, n = (int)(r() % 2000u); i < n; ++i) {}
        int next = place::TAKE;
        if (sm < words)
        {
            next = place::admit<HostAtomics>(&sm_word[sm], heavy, order.data(), cotenants);
            if (next >= 0)
            {
                heavy_at_admission[sm].fetch_add(1);
                bool is_heavy = false;
                for (int h = 0; h < H; ++h) is_heavy = is_heavy || order[h] == next;
                if (!is_heavy) fail("an instance of the light part taken at admission", t);
            }
        }
        if (next == place::LEAVE) { finished.fetch_add(1); return; }
        running[sm].fetch_add(1);
        for (;;)
        {
            const int inst = next >= 0 ? next : place::take<HostAtomics>(&queue, heavy, order.data(), total);
            next = place::TAKE;
            if (inst == total) break;
            if (inst < 0 || inst > total) { fail("an instance out of range", t); break; }
            if (taken[inst].fetch_add(1) != 0) fail("an instance taken twice", t);
            for (volatile int i = 0, n = (int)(r() % 500u); i < n; ++i) {}
            if (r() % 8u == 0u) std::this_thread::yield();
        }
        finished.fetch_add(1);
    };
    std::vector<std::thread> th;
    for (int t = 0; t < ctas; ++t) th.emplace_back(cta, t);
    const auto t0 = std::chrono::steady_clock::now();
    while (finished.load() < ctas)
    {
        if (std::chrono::steady_clock::now() - t0 > std::chrono::seconds(30)) { std::printf("deadlock: %d of %d CTAs finished\n", finished.load(), ctas); std::fflush(stdout); std::_Exit(2); }
        std::this_thread::sleep_for(std::chrono::milliseconds(1));
    }
    for (auto& x : th) x.join();
    int heavy_sms = 0;
    for (int i = 0; i < total; ++i)
        if (taken[i].load() != 1) { fail("an instance not taken exactly once", -1); break; }
    for (int s = 0; s < sms; ++s)
    {
        if (heavy_at_admission[s].load() > 1) fail("two heavy instances admitted on one SM", -1);
        if (heavy_at_admission[s].load() == 1)
        {
            ++heavy_sms;
            if (running[s].load() > 1 + (int)cotenants) fail("a heavy SM runs more CTAs than the cap", -1);
        }
        else if (s < words && running[s].load() != per_sm) fail("a light SM lost a CTA", -1);
    }
    if (heavy[1] < H) fail("the heavy part was not drained", -1);
    if (heavy_sms > H || heavy_sms > words) fail("more heavy SMs than heavy instances or SMs with a word", -1);
    std::printf("%d CTAs, %d heavy SMs, %d errors\n", ctas, heavy_sms, errors.load());
    return errors.load() ? 1 : 0;
}
