// K-mer pair counts of `whatshap learn` (whmec_learn, DESIGN §4.13): the per-read emit and the per-row reference k-mer, shared by
// the kernels of learn.cu and the host emulation tests/emul/emul_learn.cpp.
//
// A read is its query bytes and the query-consuming runs of its CIGAR (LnOp, built by learn_plan.cpp).  Byte i of a run emits
// the k-mer (h, column) when at least k bytes were read since the last S operation (caller.cpp's `consecutive >= k`), where h is
// the last k ACGT bytes of query[0..i] (zero-filled; other bytes leave it unchanged) and the column is the run's first column,
// plus i - q0 for M, = and X.  A kept k-mer (column above the read's floor and inside the chunk) becomes the key
// (column - chunk start) << 2k | h, twice for a read with a single k-mer.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define LN_HD __host__ __device__ __forceinline__
#else
#define LN_HD inline
#endif

namespace whmec {

constexpr uint32_t LN_SHORT = 512;  // an entry with more query bytes than this takes a warp

struct LnOp {        // one query-consuming run of a CIGAR operation (M, I, =, X)
    uint32_t q0;     // query index of its first byte
    uint32_t len;    // bytes (> 0)
    uint32_t reset;  // query index where `consecutive` last restarted (the first byte after the last S before the run, or 0)
    int32_t col0;    // column (1-based reference position + 1 of caller.cpp's pos) of its first byte's k-mer
    uint32_t adv;    // 1: M, = or X (the column advances per byte); 0: I
};

struct LnRead {
    uint64_t q;      // offset of the query in the call's query bytes
    uint64_t op0;    // first run in the call's run list
    uint32_t n_ops;
    uint32_t weight; // 2 for a read with a single k-mer (add_read and advance_to both count it), else 1
    int32_t floor;   // T_r: its k-mers at columns <= floor were popped before it was added and are dropped
    uint32_t pad;
};

struct LnEntry {     // one read's part of one chunk: query bytes [b0, b1) hold its n_keys kept keys, written from key_off
    uint32_t read, b0, b1, n_keys;
    uint64_t key_off;
};

struct LnRange {
    int64_t lo, hi;  // the chunk's columns
    uint32_t k;
};

LN_HD uint32_t ln_code(uint8_t c) { return c == 'A' ? 0u : c == 'C' ? 1u : c == 'G' ? 2u : c == 'T' ? 3u : 4u; }

// h after query[0..i): its last k ACGT bytes, the latest in the low bits, zero-filled
LN_HD uint32_t ln_seed(const uint8_t *q, uint32_t i, uint32_t k) {
    uint32_t h = 0, n = 0;
    for (uint32_t j = i; j > 0 && n < k; --j) {
        const uint32_t c = ln_code(q[j - 1]);
        if (c < 4) h |= c << (2 * n++);
    }
    return h;
}

// The column of byte i of run o.
LN_HD int64_t ln_col(const LnOp &o, uint32_t i) { return (int64_t)o.col0 + (o.adv ? (int64_t)(i - o.q0) : 0); }

// The keys of read r's kept k-mers at query bytes [i0, i1) inside chunk g, written to out[0 .. cap) (when out is not null; a key
// beyond cap is not written); returns how many there are.  A caller whose plan gave cap keys checks that the return equals it.
template <class K>
LN_HD uint64_t ln_emit(const LnRead &r, const LnOp *ops, const uint8_t *q, uint32_t i0, uint32_t i1, const LnRange &g, K *out, uint64_t cap) {
    if (i0 >= i1) return 0;
    const uint32_t k = g.k, mask = (1u << (2 * k)) - 1;
    uint32_t lo = 0, hi = r.n_ops - 1;  // the run holding byte i0: the last with q0 <= i0
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) / 2;
        if (ops[mid].q0 <= i0) lo = mid;
        else hi = mid - 1;
    }
    uint32_t j = lo;
    LnOp o = ops[j];
    uint32_t h = out ? ln_seed(q, i0, k) : 0;
    uint64_t n = 0;
    for (uint32_t i = i0; i < i1; ++i) {
        while (i >= o.q0 + o.len) o = ops[++j];
        if (out) {
            const uint32_t c = ln_code(q[i]);
            if (c < 4) h = ((h << 2) | c) & mask;
        }
        if (i + 1 < o.reset + k) continue;
        const int64_t col = ln_col(o, i);
        if (col <= r.floor || col < g.lo || col > g.hi) continue;
        if (out) {
            const K key = ((K)(col - g.lo) << (2 * k)) | (K)h;
            if (n < cap) out[n] = key;
            if (r.weight == 2 && n + 1 < cap) out[n + 1] = key;
        }
        n += r.weight;
    }
    return n;
}

// Lane `lane` of the warp that takes an entry: its share of the bytes [b0, b1).
LN_HD void ln_lane_span(uint32_t b0, uint32_t b1, uint32_t lane, uint32_t &i0, uint32_t &i1) {
    const uint64_t n = b1 - b0, span = (n + 31) / 32, s0 = span * lane, s1 = span * (lane + 1);
    i0 = b0 + (uint32_t)(s0 < n ? s0 : n);
    i1 = b0 + (uint32_t)(s1 < n ? s1 : n);
}

// The reference bytes [b0, hi - 1] of a call's columns [b0 + 1, hi] as codes of their ACGT bytes, after k seed codes (the last
// k ACGT bytes before b0, zero-filled), and per 32 bytes a prefix count and an ACGT mask: column c's k-mer is the k codes before
// prefix(c - b0) = base[x / 32] + popcount of the mask bits below x % 32.
struct LnRef {
    const uint8_t *code;
    const uint32_t *base;
    const uint32_t *mask;
    int64_t b0;
};

LN_HD uint32_t ln_popc(uint32_t v) {
#ifdef __CUDA_ARCH__
    return (uint32_t)__popc(v);
#else
    return (uint32_t)__builtin_popcount(v);
#endif
}

LN_HD uint32_t ln_ref_kmer(const LnRef &f, int64_t col, uint32_t k) {
    const uint64_t x = (uint64_t)(col - f.b0);
    const uint32_t p = f.base[x / 32] + ln_popc(f.mask[x / 32] & ((1u << (x % 32)) - 1u));
    uint32_t h = 0;
    for (uint32_t j = p - k; j < p; ++j) h = (h << 2) | f.code[j];
    return h;
}

// Whether column c lies in one of the n sorted, disjoint output intervals iv[2i] .. iv[2i + 1].
LN_HD bool ln_output(const int64_t *iv, uint32_t n, int64_t c) {
    uint32_t lo = 0, hi = n;  // the first interval whose end is >= c
    while (lo < hi) {
        const uint32_t mid = (lo + hi) / 2;
        if (iv[2 * mid + 1] < c) lo = mid + 1;
        else hi = mid;
    }
    return lo < n && iv[2 * lo] <= c;
}

}  // namespace whmec
