// Fused pedigree sweep for one trio (T == 4 transmission values), host/device per-item code.
//
// One thread block owns one DP-independent chain and walks all its columns with the projection in shared memory
// (ped_fused_kernel, whmec.cu); the test-only emulation (tests/emul) runs the same functions item by item on the CPU.
// Reference: the T-dimension of PedigreeDPTable::compute_column (src/pedigreedptable.cpp:239-327).
//
// What makes this fast where the general column code (dp_device.h) is not:
//  * a work item evaluates ALL FOUR transmission values of one projection entry: the index arithmetic of a candidate
//    cell (scatter of the output index, Gray-rank offset, walk over the dropped reads) is done once, the four previous
//    values arrive as one 128-bit shared-memory load;
//  * the cost functions of a column live in 16 fixed register slots (4 per transmission value, unused slots hold +inf),
//    so that "min over the allowed allele assignments" is three VIMNMX per transmission value with no run-time group
//    boundaries; a Gray step to the next candidate adds one signed delta per slot (four 128-bit broadcast loads);
//  * +inf is 2^30 (every real value stays below 2^28, Packed::safe31), sums never wrap and no addition is guarded;
//  * the transition minima min_j(value_j + popcount(i ^ j) * rc) for the next column are formed from registers by the
//    thread that owns the four values.
// Columns outside this shape (more than 4 allowed assignments per transmission value, more than 16 active reads, more
// than 2^12 projection entries, T != 4) keep the general batched sweep.
#pragma once
#include "common.h"
#include "dp_device.h"

namespace whmec {

constexpr uint32_t PF_T = 4;            // transmission values (one trio)
constexpr uint32_t PF_GS = 4;           // cost-function slots per transmission value
constexpr uint32_t PF_SLOTS = PF_T * PF_GS;
constexpr uint32_t PF_INF = 1u << 30;   // +infinity of this path (UMAX at the boundaries)
constexpr uint32_t PF_MAX_A = 16;       // active reads per column (two byte tables)
constexpr uint32_t PF_MAX_F = 12;       // log2 projection entries per transmission value
constexpr uint32_t PF_THREADS = 1024;
constexpr uint32_t PF_MAX_CLUSTER = 8;  // CTAs per chain of ped_fused_cluster_kernel (whmec.cu), at most

constexpr uint32_t PF_ROW = 20;         // words per row of a byte table: 16 slots + 4 words of skew (rows 0..7 start in 8 different
                                        // groups of four banks, so the 128-bit loads of a quarter warp spread over all banks)

struct PedFusedCol {                    // one column, staged in shared memory
    ColMeta m;
    uint32_t drop;                      // dropped positions as a bit set
    uint32_t rc_next;                   // recombination cost of the next column of the chain (0 at the chain's end)
    alignas(16) uint32_t c0[PF_SLOTS];
    alignas(16) int32_t sd[PF_MAX_A][2][PF_SLOTS];  // signed step of slot s when bit `pos` becomes 1 / 0:  +delta / -delta
    uint32_t pd_lo[TAB_SIZE], pd_hi[TAB_SIZE];
    uint32_t pd_drop[32];               // scatter of a d-bit pattern into the dropped positions (d <= 5; else computed)
    uint32_t above[8];                  // per dropped position i (i < 8): the OUTPUT-index bits whose kept position lies above it
    alignas(16) int32_t tab[2][TAB_SIZE][PF_ROW];   // [half][byte value][slot]: sum of the slot's deltas over cell bits 0..7 / 8..15
};

struct PedQuad {
    uint32_t val[PF_T], r[PF_T], b[PF_T];  // per transmission value: best value, rank of its candidate, that candidate's index into M
};

// Row b of the previous column's transition minima sits at row pf_swz(b): within a warp the candidates of neighbouring outputs
// share their low index bits (the reads that end are the oldest = lowest bits), the swizzle moves the bits that do differ into
// the bank-selecting position (128-bit row loads: 8 rows per wavefront).
// The low bits in question are gray(r) ^ cg(o), and cg(o) flips bit 2 with the parity of o (three reads end at the three lowest
// positions: the steady state of a trio) -- so the XOR term is (o0, o1, o0 ^ o1), which together with that parity flip is a
// bijection of the 8 neighbours (o0, o1, o2); a plain (o0, o1, o2) term would collide pairwise.
WHMEC_HD uint32_t pf_swz(uint32_t b) {
    const uint32_t h = b >> 3;
    return b ^ ((h & 3u) | (((h ^ (h >> 1)) & 1u) << 2));
}

// Is the fused sweep applicable to column `m` with the given function groups?
WHMEC_HD bool pf_column_ok(const ColMeta &m, const uint32_t *group /* [T + 1] */) {
    if (m.a > PF_MAX_A || m.f > PF_MAX_F) return false;
    for (uint32_t t = 0; t < PF_T; ++t)
        if (group[t + 1] - group[t] > PF_GS) return false;
    return true;
}

// Slot s = t * PF_GS + q holds the q-th function of transmission value t (or +inf).  One call fills slot `s`.
// (the staging functions read the column's ColMeta `m` and the function arrays from global memory, so that one barrier
// separates "stage column k" from "sweep column k")
WHMEC_HD void pf_stage_slot(PedFusedCol &C, const ColMeta &m, uint32_t s, const uint32_t *fn_c0, const int32_t *fn_delta, const uint32_t *group) {
    const uint32_t t = s / PF_GS, q = s % PF_GS;
    const uint32_t g0 = group[t], g1 = group[t + 1];
    const bool used = g0 + q < g1;
    const uint32_t F = m.fn_off + g0 + q;
    C.c0[s] = used ? fn_c0[F] : PF_INF;
    for (uint32_t pos = 0; pos < PF_MAX_A; ++pos) {
        const int32_t d = (used && pos < m.a) ? fn_delta[(size_t)F * FN_STRIDE + pos] : 0;
        C.sd[pos][1][s] = d;
        C.sd[pos][0][s] = (int32_t)(0u - (uint32_t)d);
    }
}

// 16 consecutive entries of one byte table of slot s (subset sums, one add per entry): run = (hi4 * 2 + half) * 16 + s
// (neighbouring lanes fill neighbouring slots of the same rows: conflict-free stores).
WHMEC_HD void pf_stage_table_run(PedFusedCol &C, const ColMeta &m, uint32_t run, const int32_t *fn_delta, const uint32_t *group) {
    const uint32_t s = run & 15u, half = (run >> 4) & 1u, hi4 = run >> 5;
    const uint32_t t = s / PF_GS, q = s % PF_GS;
    const bool used = group[t] + q < group[t + 1];
    const int32_t *dl = fn_delta + (size_t)(m.fn_off + group[t] + q) * FN_STRIDE + half * TAB_BITS;
    uint32_t d[TAB_BITS];
    for (uint32_t j = 0; j < TAB_BITS; ++j) d[j] = (used && half * TAB_BITS + j < m.a) ? (uint32_t)dl[j] : 0u;
    uint32_t base = 0;  // sums wrap like the reference's unsigned costs
    for (uint32_t b = 0; b < 4; ++b)
        if ((hi4 >> b) & 1u) base += d[4 + b];
    uint32_t sub[16];
    sub[0] = base;
    for (uint32_t i = 1; i < 16; ++i) sub[i] = sub[i & (i - 1)] + d[ctz32(i)];
    for (uint32_t i = 0; i < 16; ++i) {
        const uint32_t idx = 16 * hi4 + i;
        C.tab[half][half ? idx : pf_swz(idx)][s] = (int32_t)sub[i];  // low table: rows swizzled like the rows of M (same index bits)
    }
}

WHMEC_HD void pf_stage_pdep(PedFusedCol &C, const ColMeta &m, uint32_t v /* < 2 * TAB_SIZE */) {
    const uint32_t keep_lo = lowest_set_bits(m.keep, TAB_BITS), keep_hi = lowest_set_bits(m.keep & ~keep_lo, TAB_BITS);
    if (v < TAB_SIZE) C.pd_lo[v] = pdep32(v, keep_lo);
    else C.pd_hi[v - TAB_SIZE] = pdep32(v - TAB_SIZE, keep_hi);
    const uint32_t drop = ~m.keep & low_mask(m.a);
    if (v < 32) C.pd_drop[v] = pdep32(v, drop);
    else if (v < 40) {
        const uint32_t i = v - 32;
        C.above[i] = i < m.d ? pext32(m.keep & ~low_mask(m.dpos[i] + 1u), m.keep) : 0u;  // kept positions above dropped position i, as output bits
    }
}

// scatter of a candidate's dropped-bit pattern
WHMEC_HD uint32_t pf_scatter_drop(const PedFusedCol &C, uint32_t pattern) {
    return C.m.d <= 5 ? C.pd_drop[pattern] : pdep32(pattern, C.drop);
}

// Gray-rank offset of output o (common.h: rank_offset): bit i = parity of the kept bits above the i-th dropped position
WHMEC_HD uint32_t pf_rank_offset(const PedFusedCol &C, uint32_t o, uint32_t kept) {
    if (C.m.d > 8) return rank_offset(C.m, kept);
    uint32_t c = 0;
    for (uint32_t i = 0; i < C.m.d; ++i) c |= (popc32(o & C.above[i]) & 1u) << i;
    return c ^ (c >> 1);
}

// Candidates r in [r0, r1) of projection entry `o`, all four transmission values: per value the smallest
// (value, rank) -- strict '<' in the reference's visiting order.  M: transition minima of the previous column,
// [2^bw][4] (for the chain's first column the single row derived from the chain's input vector).
WHMEC_HD void pf_walk(const PedFusedCol &C, const uint32_t *__restrict__ M, uint32_t o, uint32_t r0, uint32_t r1, PedQuad &out) {
    const ColMeta &m = C.m;
    const uint32_t kept = C.pd_lo[o & (TAB_SIZE - 1)] | C.pd_hi[(o >> TAB_BITS) & (TAB_SIZE - 1)];
    const uint32_t cg = pf_rank_offset(C, o, kept);
    uint32_t x = kept | pf_scatter_drop(C, (r0 ^ (r0 >> 1)) ^ cg);
    uint32_t cost[PF_SLOTS];
    {
        const int32_t *lo = C.tab[0][pf_swz(x & (TAB_SIZE - 1))], *hi = C.tab[1][(x >> TAB_BITS) & (TAB_SIZE - 1)];
#pragma unroll
        for (uint32_t s = 0; s < PF_SLOTS; ++s) cost[s] = C.c0[s] + (uint32_t)(lo[s] + hi[s]);
    }
    const uint32_t bmask = low_mask(m.bw);
    uint32_t best[PF_T], br[PF_T];
#pragma unroll
    for (uint32_t t = 0; t < PF_T; ++t) {
        best[t] = UMAX;
        br[t] = r0;
    }
    for (uint32_t r = r0; r < r1; ++r) {
        const uint32_t *mrow = M + (size_t)pf_swz(x & bmask) * PF_T;
#pragma unroll
        for (uint32_t t = 0; t < PF_T; ++t) {
            uint32_t cur = cost[t * PF_GS];
#pragma unroll
            for (uint32_t q = 1; q < PF_GS; ++q) cur = cost[t * PF_GS + q] < cur ? cost[t * PF_GS + q] : cur;
            const uint32_t v = cur + mrow[t];
            if (v < best[t]) {
                best[t] = v;
                br[t] = r;
            }
        }
        if (r + 1 < r1) {
            const uint32_t pos = m.dpos[ctz32(r + 1)];
            x ^= 1u << pos;
            const int32_t *step = C.sd[pos][(x >> pos) & 1u];
#pragma unroll
            for (uint32_t s = 0; s < PF_SLOTS; ++s) cost[s] += (uint32_t)step[s];
        }
    }
#pragma unroll
    for (uint32_t t = 0; t < PF_T; ++t) {
        out.val[t] = best[t] < PF_INF ? best[t] : PF_INF;
        out.r[t] = br[t];
        out.b[t] = (kept | pf_scatter_drop(C, (br[t] ^ (br[t] >> 1)) ^ cg)) & bmask;  // index of the winner into M / A
    }
}

// Back-pointer of entry (o, t) from its winner: (r << tb) | argmin j of the transition the winner was reached through
// (A: argmins belonging to M, same swizzled rows); b = the winner's index into M (PedQuad::b).
WHMEC_HD uint32_t pf_backpointer(const uint8_t *__restrict__ A, uint32_t t, uint32_t val, uint32_t r, uint32_t b) {
    const uint32_t j = val < PF_INF ? A[(size_t)pf_swz(b) * PF_T + t] : 0u;
    return (r << 2) | j;
}

// the same from a merged key (small columns): the winner's index is rebuilt from its rank
WHMEC_HD uint32_t pf_backpointer_of_key(const PedFusedCol &C, const uint8_t *__restrict__ A, uint32_t o, uint32_t t, uint32_t val, uint32_t r) {
    const uint32_t b = val < PF_INF ? (candidate_index(C.m, o, r) & low_mask(C.m.bw)) : 0u;
    return pf_backpointer(A, t, val, r, b);
}

// min_j(row[j] + popcount(i ^ j) * rc) with the smallest minimising j (transition_min of dp_device.h on this path's +inf).
WHMEC_HD uint32_t pf_transition(const uint32_t *row, uint32_t i, uint32_t rc, uint32_t *arg) {
    uint32_t mn = PF_INF, mj = 0;
#pragma unroll
    for (uint32_t j = 0; j < PF_T; ++j) {
        if (row[j] >= PF_INF) continue;
        const uint32_t v = row[j] + popc32(i ^ j) * rc;
        if (v < mn) {
            mn = v;
            mj = j;
        }
    }
    *arg = mj;
    return mn < PF_INF ? mn : PF_INF;
}

// The row the chain's first column reads: from the chain's input vector (UMAX = +inf), or, for the very first column of the
// table, from "previous cost 0 for every j" (pedigreedptable.cpp:275-278).
WHMEC_HD void pf_first_row(const ColMeta &m, const uint32_t *invec /* [4], UMAX = inf */, uint32_t *M0, uint8_t *A0) {
    uint32_t row[PF_T];
    for (uint32_t j = 0; j < PF_T; ++j) row[j] = m.first ? 0u : (invec[j] == UMAX ? PF_INF : invec[j]);
    for (uint32_t i = 0; i < PF_T; ++i) {
        uint32_t arg;
        M0[i] = pf_transition(row, i, m.rc, &arg);
        A0[i] = (uint8_t)arg;
    }
}

// lanes per projection entry: columns with fewer than PF_THREADS entries spread an entry's 2^d candidates over 2^lc items
// Pass 1 -> pass 2 for ONE table that starts at chain 0 of `rows` (several tables in one sweep: one thread per table, each on
// its own chains).  Chain c's transfer matrix is Mat[u][i] = rows[c][i ^ u]; the table's first chain ignores its input (its
// row IS its output, its input vector is written as zeros); every later chain's true input is the min-plus fold of the
// chains in front of it -- of THIS table only: the fold restarts where a table starts.
WHMEC_HD void pf_fold_table(const uint32_t *rows, uint32_t n_chains, uint32_t *in_vecs) {
    uint32_t in[PF_T], out[PF_T];
    for (uint32_t i = 0; i < PF_T; ++i) {
        in[i] = rows[i];
        in_vecs[i] = 0;
    }
    for (uint32_t c = 1; c < n_chains; ++c) {
        for (uint32_t i = 0; i < PF_T; ++i) {
            in_vecs[(size_t)c * PF_T + i] = in[i];
            out[i] = UMAX;
        }
        const uint32_t *row = rows + (size_t)c * PF_T;
        for (uint32_t u = 0; u < PF_T; ++u) {
            if (in[u] == UMAX) continue;
            for (uint32_t i = 0; i < PF_T; ++i) {
                const uint32_t mv = row[i ^ u];
                if (mv != UMAX && in[u] + mv < out[i]) out[i] = in[u] + mv;
            }
        }
        for (uint32_t i = 0; i < PF_T; ++i) in[i] = out[i];
    }
}

WHMEC_HD uint32_t pf_lane_bits(uint32_t f, uint32_t d) {
    uint32_t lc = 0;
    while (((1u << f) << lc) < PF_THREADS && lc < d) ++lc;
    return lc;
}

// ---- symmetry of the transfer matrices.  Swapping the two haplotypes of a FOUNDER q (= complementing the bits of q's
// reads) together with flipping, in every trio where q is a parent, the transmission bit that selects q's haplotype maps
// the DP onto itself: cost_{t ^ mask_q}(x ^ reads_q) == cost_t(x), and popcount(i ^ j) is invariant.  Hence a chain's
// transfer matrix satisfies Mat[u ^ m][i ^ m] == Mat[u][i] for every m in the group generated by the founders' masks, and
// only one row per coset of that group has to be swept.  For a trio (both parents founders) the group is everything:
// one unit sweep gives the whole matrix, Mat[u][i] = Mat[0][i ^ u].
inline uint32_t pf_symmetry_group(uint32_t n_ind, uint32_t n_trios, const uint32_t *trios /* father, mother, child */, uint32_t *masks /* [T] out */) {
    const uint32_t T = 1u << (2 * n_trios);
    uint32_t gens[64], ng = 0;
    for (uint32_t q = 0; q < n_ind; ++q) {
        bool child = false;
        uint32_t mask = 0;
        for (uint32_t r = 0; r < n_trios; ++r) {
            if (trios[3 * r + 2] == q) child = true;
            if (trios[3 * r] == q) mask |= 1u << (2 * r);
            if (trios[3 * r + 1] == q) mask |= 1u << (2 * r + 1);
        }
        if (!child && mask && ng < 64) gens[ng++] = mask;
    }
    uint32_t count = 0;
    masks[count++] = 0;
    for (uint32_t g = 0; g < ng; ++g) {
        bool have = false;
        for (uint32_t i = 0; i < count; ++i) have |= masks[i] == gens[g];
        if (have) continue;
        const uint32_t old = count;
        for (uint32_t i = 0; i < old && count < T; ++i) masks[count++] = masks[i] ^ gens[g];
    }
    return count;
}

}  // namespace whmec
