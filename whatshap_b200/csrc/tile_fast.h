// Steady-state column of the tile kernel (see tile.cu: fast_kind), as host/device code: the CUDA kernel emits the
// back-pointer bits as warp ballots, the test-only emulation (tests/emul) records them lane by lane.
#pragma once
#include "tile_device.h"

namespace whmec {

#if defined(__CUDACC__)
using TilePair = uint2;
#define WHMEC_UMIN(a, b) min(a, b)
#define WHMEC_POPC(x) popc32(x)
#else
struct alignas(8) TilePair {
    uint32_t x, y;
};
#define WHMEC_UMIN(a, b) ((a) < (b) ? (a) : (b))
#define WHMEC_POPC(x) popc32(x)
#endif

// The two 32-entry tables of a fast column: per warp  K2 + E(global reads of this tile) + output bits 5+LG .. 9+LG,
// per lane the weights of output bits 0..4  (output bit q <-> local bit q + 1: local bit 0 is the read that ends).
WHMEC_HD int32_t tile_fast_warp_entry(const TileCol &tc, uint32_t tile, uint32_t warp) {
    const uint32_t lg = tc.pad1;
    int32_t s = tc.K2;
    for (uint32_t b = 0; b < tc.g; ++b)
        if ((tile >> b) & 1u) s += tc.w_global[b];
#pragma unroll
    for (uint32_t q = 0; q < 5; ++q)
        if ((warp >> q) & 1u) s += tc.w_local[6 + lg + q];
    return s;
}

WHMEC_HD int32_t tile_fast_lane_entry(const TileCol &tc, uint32_t lane) {
    int32_t s = 0;
#pragma unroll
    for (uint32_t q = 0; q < 5; ++q)
        if ((lane >> q) & 1u) s += tc.w_local[q + 1];
    return s;
}

// (bits << 1) | (t >> 31): one SHF.L.W on the device
WHMEC_HD uint32_t tile_shift_in_sign(uint32_t bits, uint32_t t) {
#if defined(__CUDA_ARCH__)
    return __funnelshift_l(t, bits, 1);
#else
    return (bits << 1) | (t >> 31);
#endif
}

// plain expressions (no recursion, no calls) so that they fold to constants once the loops are unrolled
#define cx_ctz(x) (((x) & 1) ? 0 : ((x) & 2) ? 1 : ((x) & 4) ? 2 : ((x) & 8) ? 3 : 4)
#define cx_parity(x) ((((x) >> 0) ^ ((x) >> 1) ^ ((x) >> 2) ^ ((x) >> 3) ^ ((x) >> 4)) & 1)

// Fast path of column_drop1 for dropped bit 0 (see fast_kind).  Warp w owns 32 * 2^LG consecutive
// outputs; every shared-memory address inside the loop is a per-thread base plus a compile-time
// offset, the E() of the 2^LG outputs of a thread are subset sums built with one add each, the two
// candidate cells of an output share one 64-bit load (and with SHARE the two outputs that differ
// only in the newly started read share it too), back-pointers leave as warp ballots.
// `emit(word, bit)`: this thread's bit of back-pointer word `word` of its warp (words are numbered from the warp's first).
// PACKED (TileCol::pad2 == 1, the default layout since round 2): the thread keeps the bits of its own 2^LG (x 2 with SHARE) outputs in a
// register and hands them to `emit.store(bits)` once per column.  No predicate is formed: with all values below 2^28
// (the tile path's precondition) "candidate 1 wins" is the sign of v1 - v0 - par, and one funnel shift moves that sign
// bit into the register — IADD3 + SHF per output instead of IADD + ISETP + VOTE + STG.  The outputs arrive in the order
// (it = 0, twin of 0, it = 1, ...), so the first one ends up in the highest of the thread's bits (tile_packed_bit_index).
// MIRROR (column of a mirrored panel with TileCol::km == 1, see tile_device.h): the back-pointer of the mirror output ~o,
// which no tile computes, is the same comparison with the opposite tie-break parity: sign(v1 - v0 - !par) ^ !par.  It goes to
// `emit.mirror(word, bit)` / `emit.store_mirror(bits)` (the second section of the tile's slice).
// The part of a fast column that does not touch the previous projection: the thread's addresses, the column's constants and
// the subset sums E() of its outputs.  The kernel's steady-state loop computes it for column j + 1 between ARRIVING at the
// column barrier and WAITING on it (split barrier), so that this work fills the time in which the warps of the block drift apart.
template <int LG>
struct FastPrep {
    const TilePair *sin2;
    uint32_t *so;
    uint32_t half, wp, wn, K0, K12, par0;
    uint32_t ue[1 << LG];
};

template <int LG, bool SHARE>
WHMEC_HD void column_fast_prep(FastPrep<LG> &pr, const TileCol &tc, const int32_t *__restrict__ TW, const int32_t *__restrict__ T5,
                               uint32_t cg, const uint32_t *__restrict__ Sin, uint32_t *__restrict__ Sout, uint32_t tid) {
    constexpr int IT = 1 << LG;
    const uint32_t lane = tid & 31u, warp = tid >> 5;
    const uint32_t obase = warp * (IT * 32u) + lane;      // o = obase + 32*it  (+ nout/2 for the shared twin)
    const uint32_t pmask = (1u << (tc.l_in - 1)) - 1u;    // candidate pairs of the previous projection
    pr.sin2 = reinterpret_cast<const TilePair *>(Sin) + (obase & pmask);
    pr.so = Sout + obase;
    pr.half = 1u << (tc.l_out - 1);
    pr.wp = (uint32_t)tc.w_local[0];
    pr.wn = SHARE ? (uint32_t)tc.w_local[tc.l_out] : 0u;  // the read that starts in this column
    pr.K0 = tc.K0;
    pr.K12 = tc.K12;
    pr.par0 = (WHMEC_POPC(obase) + (cg & 1u)) & 1u;  // parity of the bits above the dropped one
    pr.ue[0] = (uint32_t)(TW[warp] + T5[lane]);
#pragma unroll
    for (int it = 1; it < IT; ++it) pr.ue[it] = pr.ue[it & (it - 1)] + (uint32_t)tc.w_local[6 + cx_ctz(it)];
}

template <int LG, bool HASK0, bool SHARE, bool PACKED, bool MIRROR, class Emit>
WHMEC_HD void column_fast_body(const FastPrep<LG> &pr, Emit emit) {
    constexpr int IT = 1 << LG;
    const TilePair *sin2 = pr.sin2;
    uint32_t *so = pr.so;
    const uint32_t half = pr.half, wp = pr.wp, wn = pr.wn, K0 = pr.K0, K12 = pr.K12, par0 = pr.par0;
    uint32_t bits = 0, mbits = 0;
#pragma unroll
    for (int it = 0; it < IT; ++it) {
        const TilePair s = sin2[it * 32];
        const uint32_t par = par0 ^ (uint32_t)cx_parity(it);
        {
            const uint32_t u0 = pr.ue[it], u1 = u0 + wp;
            uint32_t c0 = WHMEC_UMIN(u0, K12 - u0), c1 = WHMEC_UMIN(u1, K12 - u1);
            if (HASK0) { c0 = WHMEC_UMIN(c0, K0); c1 = WHMEC_UMIN(c1, K0); }
            const uint32_t v0 = c0 + s.x, v1 = c1 + s.y;
            const bool pick1 = v1 < v0 + par;  // par == 0: candidate 0 is visited first and keeps ties
            so[it * 32] = WHMEC_UMIN(v0, v1);
            if (PACKED) bits = tile_shift_in_sign(bits, v1 - v0 - par);  // sign set <=> pick1
            else emit((uint32_t)it, pick1 != (par != 0));
            if (MIRROR) {
                const uint32_t q = par ^ 1u;
                if (PACKED) mbits = tile_shift_in_sign(mbits, v1 - v0 - q);
                else emit.mirror((uint32_t)it, (v1 < v0 + q) != (q != 0));
            }
        }
        if (SHARE) {  // twin output: the new read on side 1 (one more bit above the dropped one)
            const uint32_t u0 = pr.ue[it] + wn, u1 = u0 + wp;
            uint32_t c0 = WHMEC_UMIN(u0, K12 - u0), c1 = WHMEC_UMIN(u1, K12 - u1);
            if (HASK0) { c0 = WHMEC_UMIN(c0, K0); c1 = WHMEC_UMIN(c1, K0); }
            const uint32_t v0 = c0 + s.x, v1 = c1 + s.y;
            const uint32_t parb = par ^ 1u;
            const bool pick1 = v1 < v0 + parb;
            so[half + it * 32] = WHMEC_UMIN(v0, v1);
            if (PACKED) bits = tile_shift_in_sign(bits, v1 - v0 - parb);
            else emit((half >> 5) + (uint32_t)it, pick1 != (parb != 0));
            if (MIRROR) {
                const uint32_t q = parb ^ 1u;
                if (PACKED) mbits = tile_shift_in_sign(mbits, v1 - v0 - q);
                else emit.mirror((half >> 5) + (uint32_t)it, (v1 < v0 + q) != (q != 0));
            }
        }
    }
    if (PACKED) {
        // stored bit = pick1 ^ par, par = par0 ^ parity(it) ^ twin: fold the compile-time part and the thread's par0 in at once
        constexpr uint32_t N = SHARE ? 2 * IT : IT;
        uint32_t cm = 0;
#pragma unroll
        for (int it = 0; it < IT; ++it) {
            if (SHARE) cm |= ((uint32_t)cx_parity(it) << (N - 1 - 2 * it)) | (((uint32_t)cx_parity(it) ^ 1u) << (N - 2 - 2 * it));
            else cm |= (uint32_t)cx_parity(it) << (N - 1 - it);
        }
        const uint32_t all = N >= 32 ? 0xFFFFFFFFu : ((1u << N) - 1u);
        emit.store((bits ^ cm ^ (par0 ? all : 0u)) & all);
        if (MIRROR) emit.store_mirror((mbits ^ cm ^ all ^ (par0 ? all : 0u)) & all);  // q = !par throughout
    }
}

// Steady-state panels (every column the twin fast column of one tile size): what column_fast_prep reads from the 288-byte
// TileCol, as one 32-byte record per column (two 128-bit loads), built once per (tile, panel) next to the warp / lane tables.
struct alignas(16) SteadyCol {
    int32_t wp, wn;   // w_local[0] (the read that ends), w_local[l_out] (the read that starts)
    int32_t w[3];     // w_local[6 .. 8]: output bits 5 .. 7, the bits a thread's 2^LG outputs differ in
    uint32_t K12, cg, pad;
};

WHMEC_HD SteadyCol steady_col(const TileCol &tc, uint32_t cg) {
    SteadyCol sc;
    sc.wp = tc.w_local[0];
    sc.wn = tc.w_local[tc.l_out];
    sc.w[0] = tc.w_local[6];
    sc.w[1] = tc.w_local[7];
    sc.w[2] = tc.w_local[8];
    sc.K12 = tc.K12;
    sc.cg = cg;
    sc.pad = 0;
    return sc;
}

// column_fast_prep<LG, true> of a steady-state column from its SteadyCol and the constants of the panel:
// pair_off = obase & pmask, half = 2^(l_out - 1) and popc(obase) do not change inside a panel (l_in and l_out are the same for
// all its columns).  K0 is not used (steady columns have no homozygous term).
template <int LG>
WHMEC_HD void steady_prep(FastPrep<LG> &pr, const SteadyCol &sc, int32_t tw, int32_t t5, const uint32_t *__restrict__ Sin,
                          uint32_t *__restrict__ Sout, uint32_t obase, uint32_t pair_off, uint32_t half, uint32_t pop_obase) {
    constexpr int IT = 1 << LG;
    static_assert(LG <= 3, "SteadyCol holds the weights of three output bits");
    pr.sin2 = reinterpret_cast<const TilePair *>(Sin) + pair_off;
    pr.so = Sout + obase;
    pr.half = half;
    pr.wp = (uint32_t)sc.wp;
    pr.wn = (uint32_t)sc.wn;
    pr.K0 = 0;
    pr.K12 = sc.K12;
    pr.par0 = (pop_obase + (sc.cg & 1u)) & 1u;
    pr.ue[0] = (uint32_t)(tw + t5);
#pragma unroll
    for (int it = 1; it < IT; ++it) pr.ue[it] = pr.ue[it & (it - 1)] + (uint32_t)sc.w[cx_ctz(it)];
}

// ---- narrow steady-state columns (Panel::narrow, DESIGN §4.1) ---------------------------------------------------------------
// A narrow panel keeps its projection as 16-bit halfwords h = 2 (v - base) (one base per tile and panel), two per 32-bit word,
// and a word is worked on as a pair of halves: Hopper's DPX instructions add and compare both halves at once
// (VIADDMNMX.U16x2, VIMNMX.U16x2).  Every half stays inside [0, 2^16) (the planner's bound), so a plain 32-bit add of two
// such pairs, read as lo + 65536 * hi with signed halves, is exact in both halves as well.
//
// Keys.  Candidate c of an output gets the key 2 (v_c + cost_c) + (c == the candidate the reference visits second): the
// minimum of the two keys is 2 * the output's value plus the output's back-pointer bit (pick1 ^ par, the bit the u32 path
// stores); the keys never tie (their low bits differ).
//
// Thread mapping (2^14 outputs, 1024 threads, 16 outputs each).  A word holds outputs o and o + 1 (the halves of the same
// words in the next column are again its candidates: the layout of the halfword array does not change from column to
// column).  Thread (warp w, lane L) owns the words of the outputs  w * 256 + iq * 64 + 2 L + {0, 1}  (iq = 0..3) and their
// twins (+ 2^13): the halfwords 4 (w * 128 + iq * 32 + L) .. + 3 of the input are the candidates of both words of a
// quad, one 64-bit load.  The back-pointer element of thread-packed lane l (16 bits, tile_packed_bit_index) holds outputs
// with lane bits l, so lane L produces half of the elements of lanes 2 (L & 15) and 2 (L & 15) + 1, lane L ^ 16 the other
// half: one shuffle joins them, and the lanes L < 16 store both elements as one 32-bit word.
constexpr uint32_t NARROW_TWIN_WORDS = 1u << 12;  // words between an output pair and its twins (2^13 outputs)

WHMEC_HD uint32_t narrow_vmin2(uint32_t a, uint32_t b) {  // per-half unsigned min: VIMNMX.U16x2
#if defined(__CUDA_ARCH__)
    return __vminu2(a, b);
#else
    const uint32_t lo = (a & 0xFFFFu) < (b & 0xFFFFu) ? (a & 0xFFFFu) : (b & 0xFFFFu);
    const uint32_t hi = (a >> 16) < (b >> 16) ? (a >> 16) : (b >> 16);
    return lo | (hi << 16);
#endif
}

WHMEC_HD uint32_t narrow_viaddmin2(uint32_t a, uint32_t b, uint32_t c) {  // per half min(a + b mod 2^16, c): VIADDMNMX.U16x2
#if defined(__CUDA_ARCH__)
    return __viaddmin_u16x2(a, b, c);
#else
    return narrow_vmin2(((a + b) & 0xFFFFu) | (((a >> 16) + (b >> 16)) << 16), c);
#endif
}

WHMEC_HD uint32_t narrow_prmt(uint32_t a, uint32_t b, uint32_t sel) {  // PRMT: byte i of the result = byte sel_i of (b:a)
#if defined(__CUDA_ARCH__)
    return __byte_perm(a, b, sel);
#else
    const uint64_t ab = ((uint64_t)b << 32) | a;
    uint32_t r = 0;
    for (uint32_t i = 0; i < 4; ++i) r |= (uint32_t)((ab >> (8 * ((sel >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
    return r;
#endif
}

// The constants of one narrow column for the threads whose output bits have parity p (with the column's cg: the tie-break
// parity par of their first output), built once per (tile, column, p) next to the steady-state tables.
// Candidate roles: the VIADDMNMX below adds 4 |wp| (wp = weight of the read that ends) to the cost pair of one candidate,
// which must not wrap; with wp < 0 the roles of the two candidates swap (the "first" candidate is candidate 1: its U is
// U + wp, its parity 1 - par, and the PRMT selectors exchange the candidates' values).  Below, U and par are those of the
// first candidate.
// Word (iq, twin) of a thread starts from  a = 2 U + par  per half (par of the high half = 1 - par of the low one);
// a[0] = u * 131074 + a0c with u the thread's U of output 2L, a[i] = a[0] + d[i].  With f = parity(iq) ^ twin,
// kp[f] - a = 2 (K12 - U) + par per half, and  min(2 U' + 1 - par, 2 (K12 - U') + 1 - par)  of the other candidate
// (U' = U + |wp|) = viaddmin(a, w4, kp[f] - a) + dy[f].
struct alignas(16) NarrowCol {
    uint32_t a0c;
    uint32_t d[7];
    uint32_t kp[2], dy[2];
    uint32_t w4, selx, sely, pad;
};

WHMEC_HD NarrowCol narrow_col(const TileCol &tc, uint32_t cg, uint32_t p) {
    NarrowCol nc;
    const bool neg = tc.w_local[0] < 0;
    const uint32_t awp = (uint32_t)(neg ? -tc.w_local[0] : tc.w_local[0]);
    const uint32_t q = (p ^ cg ^ (neg ? 1u : 0u)) & 1u;  // par of the first candidate of the low half of word 0
    const uint32_t G = q ? 65535u : (uint32_t)-65535;    // a(f = 1) - a(f = 0) at equal U
    const uint32_t d6 = (uint32_t)tc.w_local[7] * 131074u, d7 = (uint32_t)tc.w_local[8] * 131074u;
    const uint32_t dn = (uint32_t)tc.w_local[tc.l_out] * 131074u;
    nc.a0c = ((uint32_t)tc.w_local[1] << 17) + (q ? 1u : 65536u);
    nc.d[0] = dn + G;            // (iq 0, twin)
    nc.d[1] = d6 + G;            // (iq 1)
    nc.d[2] = d6 + dn;           // (iq 1, twin)
    nc.d[3] = d7 + G;            // (iq 2)
    nc.d[4] = d7 + dn;           // (iq 2, twin)
    nc.d[5] = d6 + d7;           // (iq 3)
    nc.d[6] = d6 + d7 + dn + G;  // (iq 3, twin)
    nc.kp[0] = tc.K12 * 131074u + (q ? 2u : 131072u);
    nc.kp[1] = nc.kp[0] + 2u * G;
    nc.dy[0] = G - awp * 131074u;
    nc.dy[1] = (0u - G) - awp * 131074u;
    nc.w4 = awp * 262148u;
    nc.selx = neg ? 0x7632u : 0x5410u;  // halves 0 / 1 of the two words of a quad: candidate 0 / 1
    nc.sely = neg ? 0x5410u : 0x7632u;
    nc.pad = 0;
    return nc;
}

// Narrow lane table: U of output 2L of lane L (output bits 1..5; the warp table adds K2, the global reads and bits 8..12),
// plus wp when candidate 1 is the first one.
WHMEC_HD int32_t narrow_lane_entry(const TileCol &tc, uint32_t lane) {
    int32_t s = tile_fast_lane_entry(tc, (2u * lane) & 31u);
    if (lane >> 4) s += tc.w_local[6];
    if (tc.w_local[0] < 0) s += tc.w_local[0];
    return s;
}

// What a thread carries of one narrow column across the column barrier (like FastPrep, but small: the record is read by the
// body, so that the thread's registers are not tied up while it waits).
struct NarrowPrep {
    const TilePair *sin;    // this thread's first candidate quad
    uint32_t *so;           // this thread's first output word
    const NarrowCol *nc;    // the column's record for the parity of the thread's outputs
    uint32_t a0;
};

WHMEC_HD void narrow_prep(NarrowPrep &pr, const NarrowCol *nc, uint32_t u, const uint32_t *__restrict__ Hin, uint32_t *__restrict__ Hout,
                          uint32_t word0) {
    pr.sin = reinterpret_cast<const TilePair *>(Hin) + word0;
    pr.so = Hout + word0;
    pr.nc = nc;
    pr.a0 = u * 131074u + nc->a0c;
}

// One narrow column of one thread: stores its 8 output words, returns its 16 back-pointer bits (bits of outputs 2L + 0 in the
// low half, 2L + 1 in the high half, at the element positions of lane group L & 16 == 0; narrow_bp_word places them).
WHMEC_HD uint32_t narrow_column_body(const NarrowPrep &pr) {
    const NarrowCol nc = *pr.nc;
    uint32_t bits = 0;
#pragma unroll
    for (int iq = 0; iq < 4; ++iq) {
        const TilePair s = pr.sin[iq * 32];
        const uint32_t x = narrow_prmt(s.x, s.y, nc.selx);  // first candidate of outputs 2L, 2L + 1
        const uint32_t y = narrow_prmt(s.x, s.y, nc.sely);  // the other candidate
#pragma unroll
        for (int tw = 0; tw < 2; ++tw) {
            const int f = (int)(cx_parity(iq) ^ tw);
            const uint32_t a = (iq == 0 && tw == 0) ? pr.a0 : pr.a0 + nc.d[2 * iq + tw - 1];
            const uint32_t c0 = narrow_vmin2(a, nc.kp[f] - a);
            const uint32_t c1 = narrow_viaddmin2(a, nc.w4, nc.kp[f] - a);
            const uint32_t m = narrow_vmin2(x + c0, y + c1 + nc.dy[f]);
            pr.so[iq * 32 + tw * NARROW_TWIN_WORDS] = m & 0xFFFEFFFEu;
            // element bit 15 - 4 iq - tw (lane group 0); the shifts between consecutive outputs are 1 and 3
            bits = (iq == 0 && tw == 0) ? (m & 0x10001u) : (bits << (tw ? 1 : 3)) + (m & 0x10001u);
        }
    }
    return bits;
}

// The 32-bit word that lane L (< 16) of a warp stores: its bits and those of lane L + 16 (bits of the lane group 1, two
// element positions lower).
WHMEC_HD uint32_t narrow_bp_word(uint32_t bits_lo_group, uint32_t bits_hi_group) { return (bits_lo_group << 2) | bits_hi_group; }

template <int LG, bool HASK0, bool SHARE, bool PACKED = false, bool MIRROR = false, class Emit>
WHMEC_HD void column_fast(const TileCol &tc, const int32_t *__restrict__ TW, const int32_t *__restrict__ T5,
                          uint32_t cg, const uint32_t *__restrict__ Sin, uint32_t *__restrict__ Sout, Emit emit, uint32_t tid) {
    FastPrep<LG> pr;
    column_fast_prep<LG, SHARE>(pr, tc, TW, T5, cg, Sin, Sout, tid);
    column_fast_body<LG, HASK0, SHARE, PACKED, MIRROR>(pr, emit);
}

}  // namespace whmec
