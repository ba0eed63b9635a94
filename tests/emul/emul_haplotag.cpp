// TEST-ONLY: whmec_haplotag (group walk, block ranks, chunk cut and entry gather of haplotag_plan.cpp) with the chunk runner of
// haplotag.cu executed on the host, using the per-entry visit and the per-group choice of haplotag.h: the counts and their
// exclusive sum, the keys of each entry at its offset, a serial stable sort of (key, ordinal) and the choice of each group.  The
// chunk budget is WHMEC_HAPLOTAG_ARENA_BUDGET (no limit without it).
#include <algorithm>
#include <cstdlib>
#include <string>
#include <utility>
#include <vector>

#include "../../whatshap_b200/csrc/haplotag_plan.h"

namespace whmec {

uint64_t ht_budget(int, std::string &) {
    const char *h = std::getenv("WHMEC_HAPLOTAG_ARENA_BUDGET");
    return h ? std::strtoull(h, nullptr, 10) : ~0ull;
}

void ht_close(HtCall &) {}

int ht_run_chunk(int, HtCall &call, std::string &) {
    HtTable t = call.host;
    t.rank = call.rank.data();
    const uint32_t ne = (uint32_t)call.entries.size(), ng = (uint32_t)call.gstart.size() - 1;
    std::vector<uint32_t> koff(ne + 1, 0);
    uint64_t error = ~0ull;
    for (uint32_t i = 0; i < ne; ++i) {
        uint32_t c = 0;
        const uint32_t kind = ht_visit(call.entries[i], t, call.ploidy, [&](uint32_t, uint32_t) { ++c; });
        koff[i + 1] = koff[i] + c;
        if (kind != HT_OK) error = std::min(error, ht_error_code(2 * (call.e0 + i), kind));
    }
    call.st.kernel_launches += 2;
    call.error = error;
    if (error != ~0ull && call.ploidy >= 2) return WHMEC_OK;
    const uint32_t nk = koff[ne];
    call.st.keys += nk;
    std::vector<std::pair<uint64_t, uint32_t>> kv(nk);
    for (uint32_t i = 0; i < ne; ++i) {
        const HtEntry &e = call.entries[i];
        const uint64_t g = (uint64_t)e.group << (call.hap_bits + call.rank_bits);
        uint32_t k = koff[i];
        ht_visit(e, t, call.ploidy, [&](uint32_t rank, uint32_t h) { kv[k++] = {g | (uint64_t)rank << call.hap_bits | h, i}; });
    }
    std::stable_sort(kv.begin(), kv.end(), [](const auto &a, const auto &b) { return a.first < b.first; });
    std::vector<uint64_t> keys(nk);
    std::vector<uint32_t> ords(nk);
    for (uint32_t k = 0; k < nk; ++k) keys[k] = kv[k].first, ords[k] = kv[k].second;
    call.choice.resize(ng);
    for (uint32_t g = 0; g < ng; ++g) {
        const HtChoice c = ht_choose(keys.data(), ords.data(), koff[call.gstart[g]], koff[call.gstart[g + 1]], call.entries.data(), call.ploidy,
                                     call.hap_bits, call.rank_bits);
        call.choice[g] = c;
        call.st.runs += c.runs;
        if (c.n_blocks && call.ploidy < 2) call.error = std::min(call.error, ht_error_code(2 * (call.e0 + call.gstart[g + 1]) - 1, HT_INDEX));
    }
    call.st.kernel_launches += 3;
    return WHMEC_OK;
}

}  // namespace whmec
