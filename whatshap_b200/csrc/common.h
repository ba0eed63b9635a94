// Shared host/device definitions of the packed (column-major) form of one DP instance.
//
// The reference walks a ReadSet column by column through ColumnIterator / ColumnIndexingScheme
// objects (src/columniterator.cpp:91-139, src/columnindexingscheme.cpp:7-34,62-85).  Here that
// structure is computed once on the host (pack.cpp) into flat per-column records that live in
// HBM for the duration of a plan.
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define WHMEC_HD __host__ __device__ __forceinline__
#else
#define WHMEC_HD inline
#endif

namespace whmec {

constexpr uint32_t UMAX = 0xFFFFFFFFu;  // +infinity of the reference's unsigned arithmetic
constexpr uint32_t MAX_ACTIVE = 32;     // the reference's limit (graycodes.cpp:12, columnindexingscheme.cpp:42-44): a cell index is 32 bits
constexpr uint32_t MAX_T = 256;         // 4 trios: every path but the wide column sweep (DESIGN §4.7)
constexpr uint32_t WIDE_T = 1024;       // 5 trios: the wide column sweep only
constexpr uint64_t WIDE_FN_BYTES_MAX = 16ull << 30;  // host and device bytes of the cost functions a five-trio table may use
constexpr uint32_t FN_STRIDE = 32;      // deltas per cost function

// One variant column.  Bit j of a bipartition index <-> j-th active read (ascending read index).
struct ColMeta {
    uint32_t a;          // active reads (ColumnIndexingScheme::read_ids.size())
    uint32_t bw;         // backward_projection_width: reads shared with column k-1 = bits [0,bw)
    uint32_t keep;       // forward projection mask as a bit set: bit j kept in column k+1
    uint32_t f;          // popcount(keep): log2 of the forward projection size actually used
    uint32_t d;          // a - f dropped reads
    uint32_t rc;         // recombcost[k]
    uint32_t first;      // 1 for column 0: previous cost is 0 for every j (pedigreedptable.cpp:275-278)
    uint32_t bp_width;   // bits per packed back-pointer entry: 0,1,2,4,8,16,32
    uint64_t bp_off;     // offset of this column's back-pointers in the arena, in 32-bit words
    uint32_t fn_off;     // first cost function of this column in the function arrays
    uint32_t grp_off;    // index into fn_group[]: T+1 offsets (relative to fn_off) per transmission value
    uint8_t dpos[32];    // positions of the dropped bits, ascending
};

// Affine cost function of one (transmission value, allele assignment) pair:
//   cost_F(x) = c0 + sum_j bit_j(x) * delta[j]      (mod 2^32, as the reference's unsigned sums)
// derived from PedigreeColumnCostComputer (src/pedigreecolumncostcomputer.cpp:14-114): with the
// assignment fixed, the cost separates over reads.

WHMEC_HD uint32_t popc32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __popc(x);
#else
    return (uint32_t)__builtin_popcount(x);
#endif
}

WHMEC_HD uint32_t ctz32(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return __ffs(x) - 1;
#else
    return (uint32_t)__builtin_ctz(x);
#endif
}

WHMEC_HD uint32_t low_mask(uint32_t bits) { return bits >= 32 ? 0xFFFFFFFFu : ((1u << bits) - 1u); }

// pdep(v, mask): scatter the low bits of v to the set positions of mask (no hardware pdep on GPUs).  Masks that are one
// contiguous run of bits -- the usual case: reads are ordered by their start, the reads that end are the lowest bits and the
// long-lived ones the highest -- take one shift instead of a loop over the bits (the backtrace walks through these per column).
WHMEC_HD bool mask_is_one_run(uint32_t mask, uint32_t *shift) {
    if (mask == 0) return false;
    const uint32_t s = ctz32(mask), m = mask >> s;
    *shift = s;
    return (m & (m + 1u)) == 0;
}

WHMEC_HD uint32_t pdep32(uint32_t v, uint32_t mask) {
    uint32_t shift;
    if (mask_is_one_run(mask, &shift)) return (v << shift) & mask;
    uint32_t out = 0;
    while (mask) {
        uint32_t low = mask & (0u - mask);
        if (v & 1u) out |= low;
        v >>= 1;
        mask ^= low;
    }
    return out;
}

WHMEC_HD uint32_t pext32(uint32_t v, uint32_t mask) {
    uint32_t shift;
    if (mask_is_one_run(mask, &shift)) return (v & mask) >> shift;
    uint32_t out = 0, o = 0;
    while (mask) {
        uint32_t low = mask & (0u - mask);
        if (v & low) out |= 1u << o;
        ++o;
        mask ^= low;
    }
    return out;
}

// Rank-order enumeration of the candidates of one forward-projection entry.
//
// The reference visits the 2^a indices of a column in Gray-code order and updates the
// projection with strict '<' (pedigreedptable.cpp:239-327), so among equal values the
// candidate with the smallest Gray rank inv_gray(x) wins.  Restricted to the 2^d candidates
// x = kept | pdep(delta, drop) of one output, Gray rank order is
//     delta_r = gray(r) ^ gray(c),   r = 0 .. 2^d-1,   gray(v) = v ^ (v >> 1),
// where bit i of c is the parity of the KEPT bits above the i-th dropped position.
WHMEC_HD uint32_t rank_offset(const ColMeta &m, uint32_t kept_bits) {
    uint32_t c = 0;
    for (uint32_t i = 0; i < m.d; ++i) {
        uint32_t p = m.dpos[i];
        uint32_t above = (p >= 31) ? 0u : (kept_bits >> (p + 1));
        c |= (popc32(above) & 1u) << i;
    }
    return c ^ (c >> 1);
}

WHMEC_HD uint32_t candidate_index(const ColMeta &m, uint32_t out_index, uint32_t r) {
    uint32_t drop = ~m.keep & low_mask(m.a);
    uint32_t kept = pdep32(out_index, m.keep);
    uint32_t delta = (r ^ (r >> 1)) ^ rank_offset(m, kept);
    return kept | pdep32(delta, drop);
}

inline uint32_t round_bp_width(uint32_t bits) {
    if (bits == 0) return 0;
    uint32_t w = 1;
    while (w < bits) w <<= 1;
    return w;
}

}  // namespace whmec
