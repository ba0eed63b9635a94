// Read merging of `whatshap phase --merge-reads` (whmec_merge_reads, DESIGN §4.17): the per-thread code of merge.cu, shared with
// the host emulation (tests/emul/emul_merge.cpp).  A set's alleles are packed as bits, each read from a 64-bit word boundary;
// pair p of a chunk is (j, i) with pstart[j] <= p < pstart[j + 1] and i = j + 1 + p - pstart[j].
#pragma once
#include <cstdint>

#ifdef __CUDACC__
#define MG_HD __host__ __device__ __forceinline__
#else
#define MG_HD inline
#endif

namespace whmec {

constexpr uint8_t MG_BLUE = 1, MG_NOTBLUE = 2;

// One entry of a merged read, gathered for the accumulation: its component within the chunk (by representative), position,
// allele and quality.
struct MgEntry {
    uint32_t comp;
    int32_t pos;
    int32_t quality;
    uint32_t allele;
};

// One (component, position) of the accumulation: the summed read.
struct MgRun {
    uint32_t comp;
    int32_t pos;
    int64_t quality;
    uint32_t allele;
    uint32_t pad;
};

// Word w of a set's packed alleles: bit b is the allele of entry (w - woff[r]) * 64 + b of read r, zero past the read's end.
MG_HD uint64_t mg_pack_word(uint64_t w, const uint64_t *woff, const uint64_t *roff, const uint8_t *allele, uint32_t n_reads) {
    uint32_t lo = 0, hi = n_reads;  // the read r with woff[r] <= w < woff[r + 1]
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (woff[mid] <= w) lo = mid;
        else hi = mid;
    }
    const uint64_t e0 = roff[lo] + (w - woff[lo]) * 64, e1 = roff[lo + 1];
    uint64_t bits = 0;
    for (uint32_t b = 0; b < 64 && e0 + b < e1; ++b) bits |= (uint64_t)(allele[e0 + b] & 1) << b;
    return bits;
}

// 64 alleles of a packed read from bit s on (the word after the last is readable: the packed array has one padding word).
MG_HD uint64_t mg_bits(const uint64_t *words, uint64_t s) {
    const uint64_t q = s >> 6;
    const uint32_t sh = (uint32_t)(s & 63);
    return sh ? (words[q] >> sh) | (words[q + 1] << (64 - sh)) : words[q];
}

MG_HD uint32_t mg_popcount(uint64_t x) {
#ifdef __CUDA_ARCH__
    return (uint32_t)__popcll(x);
#else
    return (uint32_t)__builtin_popcountll(x);
#endif
}

// The pair (j, i) of global pair index p: j the last read with pstart[j] <= p.
MG_HD void mg_pair(uint64_t p, const uint64_t *pstart, uint32_t n_reads, uint32_t &j, uint32_t &i) {
    uint32_t lo = 0, hi = n_reads;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) / 2;
        if (pstart[mid] <= p) lo = mid;
        else hi = mid;
    }
    j = lo;
    i = (uint32_t)(lo + 1 + (p - pstart[lo]));
}

// eval_overlap of (j, i) and the edge rule: the flags (MG_BLUE, MG_NOTBLUE) and m - mm.  The slice alleles_j[hang:] starts at
// hang (hang >= 0) or at max(len_j + hang, 0) (hang < 0); the queue rule keeps hang below len_j, so the overlap is not empty.
MG_HD uint8_t mg_eval(uint32_t j, uint32_t i, const int64_t *begin, const uint64_t *roff, const uint64_t *woff, const uint64_t *words,
                      int64_t thr_diff, int64_t thr_neg_diff, double max_error_rate, int64_t &diff) {
    const int64_t len_j = (int64_t)(roff[j + 1] - roff[j]), len_i = (int64_t)(roff[i + 1] - roff[i]);
    const int64_t hang = begin[i] - begin[j];
    const int64_t start = hang >= 0 ? hang : (len_j + hang > 0 ? len_j + hang : 0);
    const int64_t ovl = len_j - start < len_i ? len_j - start : len_i;
    const uint64_t *wj = words + woff[j], *wi = words + woff[i];
    int64_t mm = 0;
    for (int64_t k = 0; k < ovl; k += 64) {
        uint64_t x = mg_bits(wj, (uint64_t)(start + k)) ^ wi[k >> 6];
        if (ovl - k < 64) x &= (1ull << (ovl - k)) - 1;
        mm += mg_popcount(x);
    }
    const int64_t m = ovl - mm;
    diff = m - mm;
    const int64_t lo = m < mm ? m : mm;
    uint8_t f = 0;
    if (ovl >= thr_neg_diff && (double)lo / (double)ovl <= max_error_rate && m - mm >= thr_diff) {
        f = MG_BLUE;
        if (mm - m >= thr_neg_diff) f |= MG_NOTBLUE;
    }
    return f;
}

// Union by least root: parents only decrease and stay inside a component, so every component ends rooted at its least read
// whatever the order of the hooks.
MG_HD uint32_t mg_find(uint32_t *parent, uint32_t x) {
    uint32_t p = parent[x];
    while (p != x) {
        x = p;
        p = parent[x];
    }
    return x;
}

MG_HD uint32_t mg_cas(uint32_t *a, uint32_t expect, uint32_t desired) {
#ifdef __CUDA_ARCH__
    return atomicCAS(a, expect, desired);
#else
    const uint32_t old = *a;
    if (old == expect) *a = desired;
    return old;
#endif
}

MG_HD void mg_hook(uint32_t *parent, uint32_t u, uint32_t v) {
    uint32_t a = mg_find(parent, u), b = mg_find(parent, v);
    while (a != b) {
        if (a > b) {
            const uint32_t t = a;
            a = b, b = t;
        }
        const uint32_t old = mg_cas(&parent[b], b, a);  // b is a root: hang it under a
        if (old == b) break;
        b = mg_find(parent, old);
        a = mg_find(parent, a);
    }
}

// The accumulation key of a gathered entry: component, then position above the chunk's least position.
MG_HD uint64_t mg_key(const MgEntry &e, int32_t pmin, uint32_t pos_bits) {
    return (uint64_t)e.comp << pos_bits | (uint64_t)((int64_t)e.pos - pmin);
}

// One run of equal keys in sorted order: z0 and z1 summed, allele 0 when z0 >= z1, quality |z1 - z0|.
MG_HD MgRun mg_sum_run(const MgEntry *en, const uint32_t *order, uint32_t a, uint32_t b) {
    int64_t z0 = 0, z1 = 0;
    for (uint32_t k = a; k < b; ++k) {
        const MgEntry &e = en[order[k]];
        if (e.allele & 1) z1 += e.quality;
        else z0 += e.quality;
    }
    const MgEntry &e = en[order[a]];
    MgRun r{};
    r.comp = e.comp, r.pos = e.pos;
    r.allele = z0 >= z1 ? 0 : 1;
    r.quality = z1 >= z0 ? z1 - z0 : z0 - z1;
    return r;
}

}  // namespace whmec
