// TEST-ONLY: whmec_merge_reads (validation, partners, chunk cuts, removal loop and output of merge_plan.cpp) with the runners of
// merge.cu executed on the host, using the per-thread code of merge.h: the bit packing of every word, the pairs of a chunk one
// after another (hooked in pair order), the roots, and per accumulation chunk the keys, a serial stable sort and the sum of each
// run.  The budget is WHMEC_MERGE_ARENA_BUDGET (no limit without it).
#include <algorithm>
#include <cstdlib>
#include <numeric>
#include <string>
#include <vector>

#include "../../whatshap_b200/csrc/merge_plan.h"

namespace whmec {

namespace {

struct EmulSet {
    std::vector<uint64_t> words;
    std::vector<uint32_t> parent;
};

}  // namespace

uint64_t mg_budget(int, std::string &) {
    const char *h = std::getenv("WHMEC_MERGE_ARENA_BUDGET");
    return h ? std::strtoull(h, nullptr, 10) : ~0ull;
}

int mg_open_set(int, MgCall &call, std::string &) {
    if (!call.dev) call.dev = new EmulSet();
    EmulSet &E = *(EmulSet *)call.dev;
    const uint64_t nw = call.woff[call.n_reads];
    E.words.assign(nw + 1, 0);
    for (uint64_t w = 0; w < nw; ++w) E.words[w] = mg_pack_word(w, call.woff.data(), call.roff.data(), call.allele, call.n_reads);
    E.parent.resize(call.n_reads);
    std::iota(E.parent.begin(), E.parent.end(), 0u);
    call.st.kernel_launches += 2;
    return WHMEC_OK;
}

int mg_run_pairs(int, MgCall &call, std::string &) {
    EmulSet &E = *(EmulSet *)call.dev;
    const uint64_t np = call.p1 - call.p0;
    if (call.host_edges) call.flag.resize(np), call.diff.resize(np);
    for (uint64_t t = 0; t < np; ++t) {
        uint32_t j, i;
        mg_pair(call.p0 + t, call.pstart.data(), call.n_reads, j, i);
        int64_t d;
        const uint8_t f = mg_eval(j, i, call.begin.data(), call.roff.data(), call.woff.data(), E.words.data(), call.thr_diff,
                                  call.thr_neg_diff, call.max_error_rate, d);
        if (call.host_edges) {
            call.flag[t] = f, call.diff[t] = d;
        } else if (f & MG_BLUE) {
            mg_hook(E.parent.data(), j, i);
            ++call.blue;
        }
    }
    ++call.st.kernel_launches;
    return WHMEC_OK;
}

int mg_roots(int, MgCall &call, std::string &) {
    EmulSet &E = *(EmulSet *)call.dev;
    for (uint32_t x = 0; x < call.n_reads; ++x) E.parent[x] = mg_find(E.parent.data(), x);
    call.parent = E.parent;
    ++call.st.kernel_launches;
    return WHMEC_OK;
}

int mg_run_accumulate(int, MgCall &call, std::string &) {
    const uint32_t ne = (uint32_t)call.entries.size();
    std::vector<uint64_t> keys(ne);
    std::vector<uint32_t> order(ne);
    for (uint32_t k = 0; k < ne; ++k) keys[k] = mg_key(call.entries[k], call.pmin, call.pos_bits), order[k] = k;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return keys[a] < keys[b]; });
    call.runs.clear();
    for (uint32_t a = 0; a < ne;) {
        uint32_t b = a + 1;
        while (b < ne && keys[order[b]] == keys[order[a]]) ++b;
        call.runs.push_back(mg_sum_run(call.entries.data(), order.data(), a, b));
        a = b;
    }
    call.st.kernel_launches += 6;
    return WHMEC_OK;
}

void mg_close(MgCall &call) {
    delete (EmulSet *)call.dev;
    call.dev = nullptr;
}

}  // namespace whmec
