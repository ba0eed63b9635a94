// Read assignment of `whatshap haplotag` (whmec_haplotag, DESIGN §4.15): the per-entry visit and the per-group choice, shared by
// the kernels of haplotag.cu and the host emulation tests/emul/emul_haplotag.cpp.
//
// An entry is one (position, allele, quality) of a group member, in the group's visit order.  Its visit checks the allele,
// finds the position in its sample's phase table and calls emit(block rank, h) for every phase-tuple index h whose allele is
// the entry's.  Each match becomes the key group << (rank_bits + hap_bits) | rank << hap_bits | h with the entry's chunk ordinal
// as its value; after a stable sort a group's keys are contiguous and ascend by block, then haplotype, each run in visit order.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define HT_HD __host__ __device__ __forceinline__
#else
#define HT_HD inline
#endif

namespace whmec {

enum HtError : uint32_t { HT_OK = 0, HT_ASSERT = 1, HT_KEY = 2, HT_INDEX = 3 };

// An error's code: the visit key, 2 o for an entry error at call-wide ordinal o and 2 end - 1 for a group's choice (after its
// entries', before the next group's), above the kind.  The least code is the first error the reference raises.
HT_HD uint64_t ht_error_code(uint64_t visit, uint32_t kind) { return visit << 2 | kind; }

struct HtEntry {
    int64_t pos;
    int32_t allele;
    int32_t quality;
    uint32_t group;   // chunk-local
    uint32_t sample;
};

struct HtTable {              // every sample's phase table
    const uint64_t *soff;     // [n_samples + 1] into pos / rank / aoff
    const int64_t *pos;       // ascending within a sample
    const uint32_t *rank;     // dense block rank (over all samples)
    const uint64_t *aoff;     // into allele
    const int32_t *allele;
};

struct HtChoice {             // one group's outcome
    int64_t quality;          // best - second best score of the chosen block
    uint32_t n_blocks;
    uint32_t rank;            // the chosen block
    int32_t hap;              // its best haplotype
    uint32_t runs;            // distinct (block, haplotype) of the group
};

// Visits entry e: HT_ASSERT, HT_KEY or HT_INDEX as the reference raises them (the allele before the lookup before the index);
// emit(rank, h) for each match before that.
template <class Emit>
HT_HD uint32_t ht_visit(const HtEntry &e, const HtTable &t, int64_t ploidy, Emit &&emit) {
    if (e.allele != 0 && e.allele != 1) return HT_ASSERT;
    uint64_t lo = t.soff[e.sample], hi = t.soff[e.sample + 1];
    const uint64_t end = hi;
    while (lo < hi) {
        const uint64_t mid = lo + (hi - lo) / 2;
        if (t.pos[mid] < e.pos) lo = mid + 1;
        else hi = mid;
    }
    if (lo == end || t.pos[lo] != e.pos) return HT_KEY;
    const uint64_t a0 = t.aoff[lo], a1 = t.aoff[lo + 1];
    for (uint64_t a = a0; a < a1; ++a) {
        if (t.allele[a] != e.allele) continue;
        const int64_t h = (int64_t)(a - a0);
        if (h >= ploidy) return HT_INDEX;
        emit(t.rank[lo], (uint32_t)h);
    }
    return HT_OK;
}

// The top two of a multiset of scores, and the lowest index holding the top.
struct HtTop {
    int64_t t1, t2;
    int64_t idx;
    HT_HD void reset() { t1 = t2 = INT64_MIN, idx = -1; }
    HT_HD void add(int64_t v, int64_t h) {  // h ascending over the calls
        if (v > t1) t2 = t1, t1 = v, idx = h;
        else if (v > t2) t2 = v;
    }
};

// The choice of one group from its sorted keys [k0, k1) and their chunk ordinals.  ploidy >= 2 (smaller ploidies are refused
// before, for a group with a block).  A block's first ordinal is the least of its keys' (the first key of each run after the
// stable sort), and ties of the top score go to the block with the least.
HT_HD HtChoice ht_choose(const uint64_t *keys, const uint32_t *ords, uint32_t k0, uint32_t k1, const HtEntry *en, int64_t ploidy,
                         uint32_t hap_bits, uint32_t rank_bits) {
    int64_t best_top = INT64_MIN, best_q = 0, best_hap = -1;
    uint32_t best_ord = UINT32_MAX, n_blocks = 0, runs = 0;
    uint64_t best_block = 0;
    const uint64_t hmask = ((uint64_t)1 << hap_bits) - 1;
    for (uint32_t i = k0; i < k1;) {
        const uint64_t block = keys[i] >> hap_bits;  // (with the group, which is the same throughout)
        HtTop top;
        top.reset();
        int64_t present = 0, gap = -1, expect = 0;
        uint32_t first = UINT32_MAX;
        while (i < k1 && keys[i] >> hap_bits == block) {
            const uint64_t key = keys[i];
            const int64_t h = (int64_t)(key & hmask);
            int64_t s = 0;
            for (; i < k1 && keys[i] == key; ++i) {
                s += en[ords[i]].quality;
                first = ords[i] < first ? ords[i] : first;
            }
            if (gap < 0 && h > expect) gap = expect;
            expect = h + 1;
            top.add(s, h);
            ++present;
        }
        runs += (uint32_t)present;
        if (gap < 0) gap = expect;
        // the haplotypes no allele matched score 0: the lowest of them is gap, and ploidy - present of them exist
        const int64_t absent = ploidy - present;
        int64_t hap = top.idx;
        if (absent >= 1) {
            if (0 > top.t1 || (0 == top.t1 && gap < hap)) hap = gap;
            top.add(0, gap);
            if (absent >= 2) top.add(0, gap);
        }
        ++n_blocks;
        if (top.t1 > best_top || (top.t1 == best_top && first < best_ord)) {
            best_top = top.t1, best_ord = first, best_block = block, best_hap = hap;
            best_q = ploidy >= 2 ? top.t1 - top.t2 : 0;
        }
    }
    HtChoice c;
    c.quality = best_q;
    c.n_blocks = n_blocks;
    c.rank = (uint32_t)(best_block & (((uint64_t)1 << rank_bits) - 1));
    c.hap = (int32_t)best_hap;
    c.runs = runs;
    return c;
}

}  // namespace whmec
