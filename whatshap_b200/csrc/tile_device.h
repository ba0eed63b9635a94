// Per-thread pieces of the tile kernel (host/device; see dp_device.h for why).
//
// Inside a tile the bipartition index is LOCAL: bit q <-> q-th local read (same relative order
// as the reference's canonical index, columnindexingscheme.cpp:62-85); the tile id supplies the
// bits of the global reads.  With one individual and trusted or distrusted genotypes the
// column cost of the reference (pedigreecolumncostcomputer.cpp:101-114) collapses to
//     cost(x) = min(K0, K2 + E(x), K1 - E(x)),   E(x) = sum_j bit_j(x) * (+-phred_j)
// (derivation in DESIGN.md); E is looked up as TL[x & 127] + TH[x >> 7].
#pragma once
#include "common.h"
#include "dp_device.h"
#include "tile_plan.h"

namespace whmec {

constexpr uint32_t TILE_TL_BITS = TILE_MMAX < 7 ? 2 : 7;
constexpr uint32_t TILE_TL_SIZE = 1u << TILE_TL_BITS;              // 128
constexpr uint32_t TILE_TH_SIZE = 1u << (TILE_MMAX - TILE_TL_BITS);  // 256

// Tile-major hand-offs (Panel::in_layout == 1) whose chunks are at least 128 bytes travel as one bulk copy per producer tile;
// smaller chunks are gathered element by element (tile.cu).  The planner's tests count the panels of either kind with this rule.
constexpr uint32_t BULK_MAX_GA = 6;     // bulk-copy hand-off: at most 2^6 chunks ...
constexpr uint32_t BULK_MIN_J = 5;      // ... of at least 2^5 entries (128 bytes)
WHMEC_HD bool bulk_handoff(uint32_t gA, uint32_t jb) { return gA <= BULK_MAX_GA && jb >= BULK_MIN_J; }

struct TileCtx {
    const TileCol *tc;
    uint32_t tile;
    const int32_t *TL;    // [128]  sum over local bits 0..6
    const int32_t *TH;    // [256]  K2 + E(global bits of this tile) + sum over local bits 7..14
    uint32_t cg;          // bit i: parity of the global reads above dropped bit i that are set in this tile
    const uint32_t *Sin;  // [2^l_in] previous projection values of this tile
};

WHMEC_HD int32_t tile_tl_entry(const TileCol &tc, uint32_t idx) {
    int32_t s = 0;
    for (uint32_t q = 0; q < TILE_TL_BITS; ++q)
        if ((idx >> q) & 1u) s += tc.w_local[q];
    return s;
}

WHMEC_HD int32_t tile_th_entry(const TileCol &tc, uint32_t tile, uint32_t idx) {
    int32_t s = tc.K2;
    for (uint32_t b = 0; b < tc.g; ++b)
        if ((tile >> b) & 1u) s += tc.w_global[b];
    for (uint32_t q = TILE_TL_BITS; q < TILE_MMAX; ++q)
        if ((idx >> (q - TILE_TL_BITS)) & 1u) s += tc.w_local[q];
    return s;
}

WHMEC_HD uint32_t tile_cg(const TileCol &tc, uint32_t tile) {
    uint32_t c = 0;
    const uint32_t nd = tc.d < 16 ? tc.d : 16;
    for (uint32_t i = 0; i < nd; ++i) c |= (popc32(tile & tc.gabove[i]) & 1u) << i;
    return c;
}

WHMEC_HD uint32_t tile_cell_cost(const TileCtx &c, uint32_t x) {
    const uint32_t u = (uint32_t)(c.TL[x & (TILE_TL_SIZE - 1)] + c.TH[x >> TILE_TL_BITS]);
    const uint32_t v = c.tc->K12 - u;
    uint32_t m = u < v ? u : v;
    return m < c.tc->K0 ? m : c.tc->K0;
}

// Mirrored panels (Panel::half).  With one individual cost(x) == cost(~x) (~ = all reads of the column change sides), so
// every projection is symmetric, S(f) == S(~f), and the tile that fixes the global reads to ~t is the mirror image of
// tile t: only tiles with top tile-id bit 0 are computed.  The VALUES of the mirror tile are the same numbers; its
// back-pointers are not, because the reference breaks ties by visiting order.  For output f the candidate with dropped-bit
// pattern delta has rank r = inv_gray(delta ^ gray(c)), c_i = parity of the kept bits above the i-th dropped bit
// (common.h: rank_offset).  The mirror output ~f has candidates ~x with patterns ~delta and parities c_i ^ NKA_i
// (NKA_i = number of kept bits above the i-th dropped bit, mod 2), hence rank r' = r ^ km with the per-column constant
//     km = inv_gray(ones_d) ^ NKA          (TileCol::km, planner).
// The winner of ~f is therefore the candidate minimising (value, r ^ km): one more key per candidate.  km == 0: both
// outputs store the same number.  Chain end: rank = inv_gray(canonical index), km = inv_gray(ones_a).

// Regular column: best (value << 32 | r) over candidates r in [r0, r1) of local output entry o,
// visited in the reference's Gray-rank order (common.h: rank_offset).  `mirror` (optional): best (value << 32 | r ^ km),
// the key of the mirror output.
WHMEC_HD uint64_t tile_eval(const TileCtx &c, uint32_t o, uint32_t r0, uint32_t r1, uint64_t *mirror = nullptr) {
    const TileCol &tc = *c.tc;
    const uint32_t m = tc.l_in + tc.n_new;
    const uint32_t keepmask = ~tc.dropmask & low_mask(m);
    const uint32_t kept = pdep32(o, keepmask);
    uint32_t cpar = c.cg;
    for (uint32_t i = 0; i < tc.d; ++i) cpar ^= (popc32(kept >> (tc.dpos[i] + 1)) & 1u) << i;
    const uint32_t cgray = cpar ^ (cpar >> 1);
    uint32_t x = kept | pdep32((r0 ^ (r0 >> 1)) ^ cgray, tc.dropmask);
    const uint32_t inmask = low_mask(tc.l_in);
    uint64_t best = KEY_INF, best2 = KEY_INF;
    const uint32_t km = tc.km;
    for (uint32_t r = r0; r < r1; ++r) {
        const uint32_t val = tile_cell_cost(c, x) + c.Sin[x & inmask];
        const uint64_t key = ((uint64_t)val << 32) | r;
        if (key < best) best = key;
        const uint64_t key2 = ((uint64_t)val << 32) | (r ^ km);
        if (key2 < best2) best2 = key2;
        if (r + 1 < r1) x ^= 1u << tc.dpos[ctz32(r + 1)];
    }
    if (mirror) *mirror = best2;
    return best;
}

// Chain end (every read ends, pedigreedptable.cpp:306-315): best (value << 32 | Gray rank of the
// canonical index) over local cells [x0, x1); gpart = canonical bits contributed by the tile id.
WHMEC_HD uint64_t tile_eval_end(const TileCtx &c, uint32_t gpart, uint32_t x0, uint32_t x1) {
    const TileCol &tc = *c.tc;
    const uint32_t inmask = low_mask(tc.l_in);
    uint64_t best = KEY_INF;
    for (uint32_t x = x0; x < x1; ++x) {
        const uint32_t val = tile_cell_cost(c, x) + c.Sin[x & inmask];
        uint32_t g = pdep32(x, tc.lmask_col) | gpart;
        g ^= g >> 1; g ^= g >> 2; g ^= g >> 4; g ^= g >> 8; g ^= g >> 16;  // inverse Gray code = visiting rank
        const uint64_t key = ((uint64_t)val << 32) | g;
        if (key < best) best = key;
        if (tc.half) {  // the same cell of the mirror tile: same value, visiting rank g ^ inv_gray(ones_a)
            const uint64_t key2 = ((uint64_t)val << 32) | (g ^ tc.km);
            if (key2 < best) best = key2;
        }
    }
    return best;
}

// Bits per thread of a fast column (the width of one element of the thread-packed layout).
WHMEC_HD uint32_t tile_fast_bits_per_thread(const TileCol &tc) { return (1u << tc.pad1) << (tc.pad0 == 2 ? 1 : 0); }

// Thread-packed layout: index of the back-pointer bit of local output `lo` inside the tile's slice of the arena
// (output o = warp * 2^LG * 32 + it * 32 + lane, + nout / 2 for the twin; element = thread; a thread shifts its bits in
// in the order (it = 0, twin of 0, it = 1, ...), so the j-th one sits at bit N - 1 - j of the element).
WHMEC_HD uint32_t tile_packed_bit_index(const TileCol &tc, uint32_t lo) {
    const uint32_t lg = tc.pad1, it_count = 1u << lg;
    const uint32_t half = 1u << (tc.l_out - 1);
    uint32_t twin = 0;
    if (tc.pad0 == 2 && lo >= half) {
        twin = 1;
        lo -= half;
    }
    const uint32_t warp = lo >> (lg + 5), it = (lo >> 5) & (it_count - 1), lane = lo & 31u;
    const uint32_t n = tile_fast_bits_per_thread(tc);
    const uint32_t j = tc.pad0 == 2 ? 2 * it + twin : it;
    return (warp * 32 + lane) * n + (n - 1 - j);
}


// One backtrace step (pedigreedptable.cpp:155-160): from the cell x of column k (whose backward width is `bw`) to the cell of
// column k - 1 (records pm / pt) through the tile-layout back-pointers.
// The back-pointer read by that step (the rank of the winning candidate of the entry x projects to), apart from the step itself:
// the warp backtrace of tile.cu reads the back-pointers of several columns ahead speculatively.
WHMEC_HD uint32_t tile_backtrace_bp(uint32_t bw, const ColMeta &pm, const TileCol &pt, const uint32_t *arena, uint32_t x) {
    const uint32_t o = x & low_mask(bw);   // canonical forward-projection entry of column k-1
    const uint32_t fmask = low_mask(pm.f);
    uint32_t tile = pext32(o, pt.gmask_out);
    uint32_t lo = pext32(o, ~pt.gmask_out & fmask);
    uint64_t section = 0;
    if (pt.half && ((tile >> (pt.g - 1)) & 1u)) {  // output of an uncomputed tile: stored by its mirror image
        tile = ~tile & low_mask(pt.g);
        lo = ~lo & low_mask(pt.l_out);
        if (pt.km != 0) section = pt.bp_tile_words;
    }
    uint32_t at = lo;
    if (pt.pad2 & 1u) at = tile_packed_bit_index(pt, lo);  // thread-packed bits
    return bp_load(arena, pt.bp_off + (uint64_t)tile * pt.bp_tile_stride + section, pt.bp_width, at);
}

WHMEC_HD uint32_t tile_backtrace_step(uint32_t bw, const ColMeta &pm, const TileCol &pt, const uint32_t *arena, uint32_t x) {
    const uint32_t o = x & low_mask(bw);   // canonical forward-projection entry of column k-1
    const uint32_t fmask = low_mask(pm.f);
    uint32_t tile = pext32(o, pt.gmask_out);
    uint32_t lo = pext32(o, ~pt.gmask_out & fmask);
    uint64_t section = 0;
    if (pt.half && ((tile >> (pt.g - 1)) & 1u)) {  // output of an uncomputed tile: stored by its mirror image
        tile = ~tile & low_mask(pt.g);
        lo = ~lo & low_mask(pt.l_out);
        if (pt.km != 0) section = pt.bp_tile_words;
    }
    uint32_t at = lo;
    if (pt.pad2 & 1u) at = tile_packed_bit_index(pt, lo);  // thread-packed bits
    const uint32_t bp = bp_load(arena, pt.bp_off + (uint64_t)tile * pt.bp_tile_stride + section, pt.bp_width, at);
    return candidate_index(pm, o, bp);
}

// Backtrace of one chain through the tile-layout back-pointers (pedigreedptable.cpp:144-160).
WHMEC_HD void tile_backtrace_chain(const ColMeta *cols, const TileCol *tcols, const uint32_t *arena, uint32_t k_first,
                                   uint32_t k_last, uint64_t end_key, uint32_t *path_index) {
    uint32_t r = (uint32_t)end_key;
    uint32_t x = r ^ (r >> 1);  // Gray code of the winning rank = canonical index in the last column
    path_index[k_last] = x;
    for (uint32_t k = k_last; k > k_first; --k) {
        x = tile_backtrace_step(cols[k].bw, cols[k - 1], tcols[k - 1], arena, x);
        path_index[k - 1] = x;
    }
}

}  // namespace whmec
