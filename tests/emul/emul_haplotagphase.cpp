// TEST-ONLY: whmec_haplotagphase (phase-set ranks, entry binning, chunk cut and entry gather of haplotagphase_plan.cpp) with the
// chunk runners of haplotagphase.cu executed on the host, using the per-entry lookup, the per-position walk and the choice of
// haplotagphase.h: the keys of every entry, a serial stable sort of (key, chunk index), the walk of each position, and serial
// stable sorts of the positions and records by first entry.  The chunk budget is WHMEC_HAPLOTAGPHASE_ARENA_BUDGET (no limit
// without it).
#include <algorithm>
#include <cstdlib>
#include <numeric>
#include <string>
#include <utility>
#include <vector>

#include "../../whatshap_b200/csrc/haplotagphase_plan.h"

namespace whmec {

uint64_t hp_budget(int, std::string &) {
    const char *h = std::getenv("WHMEC_HAPLOTAGPHASE_ARENA_BUDGET");
    return h ? std::strtoull(h, nullptr, 10) : ~0ull;
}

void hp_close(HpCall &) {}

static uint32_t bits_for(uint64_t max_value) {
    uint32_t b = 0;
    while (b < 64 && (max_value >> b)) ++b;
    return b;
}

template <class K>
static void sort_pairs(std::vector<K> &keys, std::vector<uint32_t> &vals, int end_bit) {
    const K mask = end_bit >= (int)(8 * sizeof(K)) ? ~(K)0 : (((K)1 << end_bit) - 1);
    std::vector<uint32_t> idx(keys.size());
    std::iota(idx.begin(), idx.end(), 0);
    std::stable_sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return (keys[a] & mask) < (keys[b] & mask); });
    std::vector<K> k2(keys.size());
    std::vector<uint32_t> v2(vals.size());
    for (size_t j = 0; j < idx.size(); ++j) k2[j] = keys[idx[j]], v2[j] = vals[idx[j]];
    keys.swap(k2), vals.swap(v2);
}

int hp_run_votes(int, HpCall &call, std::string &) {
    const uint32_t ne = call.n_entries, np = call.n_cpos;
    const uint32_t ib = bits_for(ne), pos_bits = bits_for(np - 1);
    std::vector<uint64_t> keys(ne), rkey(ne);
    std::vector<uint32_t> vals(ne), rval(ne), pkey(np), pval(np);
    std::vector<HpRecord> rec(ne);
    uint64_t error = ~0ull;
    for (uint32_t i = 0; i < ne; ++i) {
        const HpEntry &e = call.entries[i];
        uint32_t x = 0;
        const uint32_t kind = hp_lookup(e, call.host, call.p0 + e.pos, x);
        if (kind != HP_OK) error = std::min(error, hp_error_code(e.ordinal, kind));
        keys[i] = (uint64_t)e.pos << (call.ps_bits + 1) | (uint64_t)e.ps << 1 | x;
        vals[i] = i;
    }
    sort_pairs(keys, vals, (int)(pos_bits + call.ps_bits + 1));
    call.choice.resize(np);
    for (uint32_t c = 0; c < np; ++c) {
        HpPick k;
        HpChoice ch = hp_walk(keys.data(), vals.data(), call.pstart[c], call.pstart[c + 1], call.entries, call.ps_bits, ib, rec.data(),
                              rkey.data(), rval.data(), k);
        if (ch.voted) hp_finish(k, call.host, call.p0 + c, call.gap, call.only_indels, ch);
        call.choice[c] = ch;
        pkey[c] = ch.voted ? ch.first : UINT32_MAX;
        pval[c] = c;
    }
    sort_pairs(rkey, rval, (int)(2 * ib));
    sort_pairs(pkey, pval, (int)ib);
    call.st.kernel_launches += 6;
    call.error = error;
    uint64_t nr = 0, nv = 0;
    for (const HpChoice &c : call.choice) nr += c.n_ps, nv += c.voted;
    call.order.assign(pval.begin(), pval.begin() + nv);
    call.records.resize(nr);
    for (uint64_t j = 0; j < nr; ++j) call.records[j] = rec[rval[j]];
    return WHMEC_OK;
}

int hp_run_runs(int, HpCall &call, std::string &) {
    const uint32_t np = call.n_cpos;
    call.choice.resize(np);
    for (uint32_t c = 0; c < np; ++c) {
        HpPick k;
        hp_pick_runs(call.run_ps, call.run_h, call.run_score, call.roff[c], call.roff[c + 1], k);
        HpChoice ch{};
        ch.voted = 1;
        hp_finish(k, call.host, call.tpos[c], call.gap, call.only_indels, ch);
        call.choice[c] = ch;
    }
    ++call.st.kernel_launches;
    return WHMEC_OK;
}

}  // namespace whmec
