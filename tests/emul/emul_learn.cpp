// TEST-ONLY: whmec_learn (host walk, floors, variant windows and chunk cut of learn_plan.cpp) with the chunk runner of learn.cu
// executed on the host, using the per-read emit and reference k-mer of learn.h: entries of at most LN_SHORT bytes in a loop,
// longer ones as 32 lanes that each count their share of the bytes, take the exclusive sum of the lanes before them and write
// (the kernel's warp scan); then a serial sort, run-length encoding and the row filter.  The chunk budget is
// WHMEC_LEARN_ARENA_BUDGET (no limit without it).  Also exports the interval form of the variant windows.
#include <algorithm>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../whatshap_b200/csrc/learn_plan.h"

namespace whmec {

uint64_t ln_budget(int, std::string &) {
    const char *h = std::getenv("WHMEC_LEARN_ARENA_BUDGET");
    return h ? std::strtoull(h, nullptr, 10) : ~0ull;
}

void ln_close(LnCall &) {}

namespace {

// false when an entry's keys disagree with the plan's count (the kernels' check)
template <class K>
bool run(LnCall &call, const LnChunk &c) {
    const LnRange g{c.lo, c.hi, call.k};
    std::vector<K> keys(c.n_keys);
    for (uint32_t e = c.e0; e < c.e1; ++e) {
        const LnEntry &en = call.entries[e];
        const LnRead &r = call.reads[en.read];
        const LnOp *ops = call.ops + r.op0;
        const uint8_t *q = call.query + r.q;
        if (en.b1 - en.b0 <= LN_SHORT) {
            if (ln_emit<K>(r, ops, q, en.b0, en.b1, g, keys.data() + en.key_off, en.n_keys) != en.n_keys) return false;
            continue;
        }
        uint64_t before = 0;
        for (uint32_t lane = 0; lane < 32; ++lane) {
            uint32_t i0, i1;
            ln_lane_span(en.b0, en.b1, lane, i0, i1);
            const uint64_t n = ln_emit<K>(r, ops, q, i0, i1, g, (K *)nullptr, 0);
            ln_emit<K>(r, ops, q, i0, i1, g, keys.data() + en.key_off + before, en.n_keys > before ? en.n_keys - before : 0);
            before += n;
        }
        if (before != en.n_keys) return false;
    }
    std::sort(keys.begin(), keys.end());
    const LnRef f{call.code.data(), call.base.data(), call.mask.data(), call.b0};
    for (size_t i = 0; i < keys.size();) {
        size_t j = i;
        while (j < keys.size() && keys[j] == keys[i]) ++j;
        ++call.st.distinct;
        const int64_t col = c.lo + (int64_t)(keys[i] >> (2 * call.k));
        if (ln_output(call.iv.data(), (uint32_t)(call.iv.size() / 2), col)) {
            const int32_t row[4] = {(int32_t)col, (int32_t)ln_ref_kmer(f, col, call.k), (int32_t)(keys[i] & ((1u << (2 * call.k)) - 1)),
                                    (int32_t)(j - i)};
            call.rows.insert(call.rows.end(), row, row + 4);
        }
        i = j;
    }
    return true;
}

}  // namespace

int ln_run_chunk(int, LnCall &call, const LnChunk &c, std::string &msg) {
    call.st.kernel_launches += 5;
    if (c.wide ? run<uint64_t>(call, c) : run<uint32_t>(call, c)) return WHMEC_OK;
    msg = "whmec_learn: a read's keys disagree with the plan's count (internal error)";
    return WHMEC_ERR_CUDA;
}

}  // namespace whmec

// ln_intervals over columns lo..hi: writes at most cap interval bounds to iv, returns their count (or the count needed), and the
// offset after hi in *off
extern "C" uint64_t whemul_learn_intervals(const int32_t *pos, const int32_t *len, uint32_t n, uint32_t *off, int64_t lo, int64_t hi,
                                           int64_t window, int64_t k, int64_t *iv, uint64_t cap) {
    std::vector<int64_t> v;
    *off = whmec::ln_intervals(pos, len, n, *off, lo, hi, window, k, v);
    std::copy(v.begin(), v.begin() + std::min<uint64_t>(cap, v.size()), iv);
    return v.size();
}
