// TEST-ONLY host emulation of whmec_heuristic_batch: the host plan (heuristic_batch.cpp) and the sweep of heuristic_device.h,
// run by a host executor in place of heuristic.cu.  Every phase visits its rows (or elements) in a seeded random order, so a
// phase whose result depended on the order in which the CTA's threads run would not equal whmec_heuristic (the tests compare bit
// for bit); the tables of a group run in a random order too.  The work region starts filled with 0xFF bytes (NaN floats, huge
// indices), so a read of a row, record or scratch word that the sweep never wrote shows.
#include <algorithm>
#include <cstring>
#include <numeric>
#include <random>
#include <string>
#include <vector>

#include "../../whatshap_b200/csrc/heuristic_batch.h"

using namespace whmec;

namespace {

struct HostExec {
    std::mt19937_64 &rng;
    std::vector<uint32_t> perm;
    template <class F>
    void rows(uint32_t n, F f) {
        perm.resize(n);
        std::iota(perm.begin(), perm.end(), 0u);
        std::shuffle(perm.begin(), perm.end(), rng);
        for (uint32_t k = 0; k < n; ++k) f(perm[k]);
    }
    template <class F>
    void single(F f) {
        f();
    }
    void sync() {}
    int32_t atomic_cas(int32_t *p, int32_t cmp, int32_t v) {
        const int32_t old = *p;
        if (old == cmp) *p = v;
        return old;
    }
    template <class T>
    void atomic_min(T *p, T v) {
        if (v < *p) *p = v;
    }
    void atomic_add(uint32_t *p, uint32_t v) { *p += v; }
    void store(uint32_t *p, uint32_t v) { *p = v; }
    uint32_t scan(uint32_t *a, uint32_t n) {
        uint32_t sum = 0;
        for (uint32_t i = 0; i < n; ++i) {
            const uint32_t v = a[i];
            a[i] = sum;
            sum += v;
        }
        return sum;
    }
};

uint64_t g_budget = ~0ull, g_seed = 0;
std::vector<int32_t> g_group_of;  // per table of the last call: its group, -1 for none
uint32_t g_groups = 0, g_fallbacks = 0;

}  // namespace

namespace whmec {

uint64_t heur_budget(int, std::string &) { return g_budget; }

int heur_run_group(int, const std::vector<HeurLayout> &layouts, const HeurGroup &g, std::vector<uint8_t> &in, std::vector<uint8_t> &out, float *ms,
                   std::string &) {
    std::mt19937_64 rng(g_seed + 7919 * g_groups);
    std::vector<uint8_t> work(g.work_bytes, 0xFF);
    out.assign(g.out_bytes, 0xFF);
    std::vector<uint32_t> order(g.members.size());
    std::iota(order.begin(), order.end(), 0u);
    std::shuffle(order.begin(), order.end(), rng);
    for (uint32_t j : order) {
        const HeurLayout &L = layouts[g.members[j]];
        const HeurDevTable d = heur_bind(L, in.data(), work.data(), out.data());
        HostExec x{rng, {}};
        HeurShared sh;
        std::memset(&sh, 0xFF, sizeof(sh));
        heur_sweep(x, sh, d);
        if (L.table < g_group_of.size()) g_group_of[L.table] = (int32_t)g_groups;
        if (*d.status != HEUR_OK) ++g_fallbacks;
    }
    ++g_groups;
    *ms = 0;
    return WHMEC_OK;
}

}  // namespace whmec

extern "C" int whemul_heuristic_batch(const whmec_problem *const *problems, whmec_heuristic_solution *const *solutions, const uint32_t *row_limits,
                                      const int *allow_mutations, uint32_t n_tables, uint64_t budget, uint64_t seed, int *status, char *errs,
                                      size_t errlen, int32_t *group_of, uint32_t *info /* [2]: groups, tables handed back */) {
    g_budget = budget ? budget : ~0ull;
    g_seed = seed;
    g_groups = g_fallbacks = 0;
    g_group_of.assign(n_tables, -1);
    const int rc = whmec_heuristic_batch(problems, solutions, row_limits, allow_mutations, n_tables, 0, status, errs, errlen, nullptr, nullptr);
    std::copy(g_group_of.begin(), g_group_of.end(), group_of);
    info[0] = g_groups;
    info[1] = g_fallbacks;
    return rc;
}
