// Per-thread pieces of the column kernel, written host/device so that the exact same code can be
// single-stepped on the CPU by the test-only emulation harness (tests/emul) before it is run
// on a GPU.  The product only ever calls these from __global__ kernels (whmec.cu).
#pragma once
#include "common.h"

namespace whmec {

// Value/back-pointer key of one projection entry:
//   bits 63..32  DP value (UMAX = +inf)
//   bits 31..tb  r  = rank-order index of the winning candidate among the 2^d of this output
//   bits tb-1..0 j  = argmin transmission value of the previous column (smallest j on ties)
// min() over keys reproduces the reference's strict-'<' updates in Gray-code visiting order
// (pedigreedptable.cpp:293-296,320-324).
constexpr uint64_t KEY_INF = 0xFFFFFFFFFFFFFFFFull;

constexpr int NF_REG = 16;  // most cost functions kept incrementally in registers per thread

// Optional per-column lookup tables (built once per thread block in shared memory) that replace the
// bit loops of the initialisation: scatter of the output index into the kept positions, and the
// value of every cost function on the low / high byte of a cell index.
constexpr uint32_t TAB_BITS = 8, TAB_SIZE = 1u << TAB_BITS;

struct ColTables {
    const uint32_t *pd_lo, *pd_hi;   // pdep(v, lowest 8 kept bits), pdep(v, next 8 kept bits)
    uint32_t keep_rest;              // kept bits beyond the first 16
    const int32_t *lo, *hi;          // [function][256]: sum of deltas over cell bits 0..7 / 8..15
};

struct ColView {
    const ColMeta *m;
    uint32_t T, tb;
    const uint32_t *fn_c0;     // functions of this column's transmission group i
    const int32_t *fn_delta;   // [nf][FN_STRIDE]
    uint32_t nf;
    const uint32_t *prev;      // [2^bw][T] values of the previous projection (ignored if m->first)
    const ColTables *tab;      // nullptr: use the bit loops
    uint32_t tab_fn0;          // index of this group's first function inside the tables
    // Optional pre-transformed previous projection: prevm[b*T+i] = min_j(prev[b][j] + popcount(i^j)*rc)
    // with prevarg the smallest minimising j (transition_min below).  Exact whenever no 32-bit sum
    // wraps (the batched pedigree path requires that); nullptr: raw values in `prev`.
    const uint32_t *prevm;
    union {
        const uint8_t *prevarg;     // T <= 256
        const uint16_t *prevarg16;  // T = 1024 (eval_candidates<true>, the wide column sweep)
    };
};

// min over the previous transmission value for target value i (pedigreedptable.cpp:270-297 without the
// column's own cost): smallest j wins ties, all-infinite rows give (UMAX, 0).
WHMEC_HD uint32_t transition_min(const uint32_t *row /* [T] */, uint32_t T, uint32_t i, uint32_t rc, uint32_t *arg) {
    uint32_t mn = UMAX, mj = 0;
    for (uint32_t j = 0; j < T; ++j) {
        if (row[j] == UMAX) continue;
        const uint32_t val = row[j] + popc32(i ^ j) * rc;
        if (val < mn) {
            mn = val;
            mj = j;
        }
    }
    *arg = mj;
    return mn;
}

WHMEC_HD uint32_t lowest_set_bits(uint32_t mask, uint32_t count) {
    uint32_t out = 0;
    for (uint32_t i = 0; i < count && mask; ++i) {
        uint32_t low = mask & (0u - mask);
        out |= low;
        mask ^= low;
    }
    return out;
}

// One run of 16 consecutive table entries of cost function F: entries [16*hi4, 16*hi4+16) of the
// byte table `half` (0: cell bits 0..7, 1: bits 8..15).  Subset sums with one add per entry.
WHMEC_HD void build_cost_table_run(const int32_t *delta /* [FN_STRIDE] of F */, uint32_t half, uint32_t hi4, int32_t *out16) {
    const int32_t *d = delta + half * TAB_BITS;
    uint32_t base = 0;  // sums wrap like the reference's unsigned costs (no signed overflow)
    for (uint32_t q = 0; q < 4; ++q)
        if ((hi4 >> q) & 1u) base += (uint32_t)d[4 + q];
    out16[0] = (int32_t)base;
    for (uint32_t i = 1; i < 16; ++i) out16[i] = (int32_t)((uint32_t)out16[i & (i - 1)] + (uint32_t)d[ctz32(i)]);
}

// Best key over candidates r in [r0, r1) of forward-projection entry `o` for transmission value i.
// Reference: one iteration of the Gray-code loop body (pedigreedptable.cpp:239-327), restricted
// to the candidates projecting onto `o` and visited in the same relative order.
template <int NFR, bool EXACT = false, bool WIDE = false>
WHMEC_HD uint64_t eval_candidates_t(const ColView &v, uint32_t o, uint32_t i, uint32_t r0, uint32_t r1) {
    const ColMeta &m = *v.m;
    const uint32_t drop = ~m.keep & low_mask(m.a);
    uint32_t kept;
    if (v.tab) {
        kept = v.tab->pd_lo[o & (TAB_SIZE - 1)] | v.tab->pd_hi[(o >> TAB_BITS) & (TAB_SIZE - 1)];
        if (v.tab->keep_rest) kept |= pdep32(o >> (2 * TAB_BITS), v.tab->keep_rest);
    } else {
        kept = pdep32(o, m.keep);
    }
    const uint32_t cg = rank_offset(m, kept);
    uint32_t x = kept | pdep32((r0 ^ (r0 >> 1)) ^ cg, drop);
    const uint32_t bmask = low_mask(m.bw);
    const bool incremental = EXACT || v.nf <= (uint32_t)NFR;

    uint32_t cost[NFR];
    if (incremental) {
#pragma unroll
        for (int F = 0; F < NFR; ++F) {
            if (EXACT || (uint32_t)F < v.nf) {
                uint32_t c = v.fn_c0[F];
                uint32_t j0 = 0;
                if (v.tab) {  // bits 0..15 from the byte tables, the rest (a > 16) bit by bit
                    const size_t t = (size_t)(v.tab_fn0 + F) * TAB_SIZE;
                    c += (uint32_t)(v.tab->lo[t + (x & (TAB_SIZE - 1))] + v.tab->hi[t + ((x >> TAB_BITS) & (TAB_SIZE - 1))]);
                    j0 = 2 * TAB_BITS;
                }
                for (uint32_t j = j0; j < m.a; ++j)
                    if ((x >> j) & 1u) c += (uint32_t)v.fn_delta[F * FN_STRIDE + j];
                cost[F] = c;
            } else {
                cost[F] = UMAX;
            }
        }
    }

    uint64_t best = KEY_INF;
    uint32_t best_b = 0;
    for (uint32_t r = r0; r < r1; ++r) {
        // get_cost(): min over allowed assignments (pedigreecolumncostcomputer.cpp:101-114)
        uint32_t cur = UMAX;
        if (incremental) {
#pragma unroll
            for (int F = 0; F < NFR; ++F)
                if ((EXACT || (uint32_t)F < v.nf) && cost[F] < cur) cur = cost[F];
        } else {
            for (uint32_t F = 0; F < v.nf; ++F) {
                uint32_t c = v.fn_c0[F];
                for (uint32_t j = 0; j < m.a; ++j)
                    if ((x >> j) & 1u) c += (uint32_t)v.fn_delta[F * FN_STRIDE + j];
                if (c < cur) cur = c;
            }
        }
        // min over previous transmission values (pedigreedptable.cpp:270-297), first j wins
        const uint32_t b = x & bmask;
        uint32_t mn = UMAX, mj = 0;
        if (v.prevm && !m.first) {
            const uint32_t pm = v.prevm[(size_t)b * v.T + i];
            if (cur < UMAX && pm < UMAX) mn = cur + pm;
        } else {
            for (uint32_t j = 0; j < v.T; ++j) {
                uint32_t prev = m.first ? 0u : v.prev[(size_t)b * v.T + j];
                uint32_t val = (cur < UMAX && prev < UMAX) ? cur + prev : UMAX;
                if (val < UMAX) val += popc32(i ^ j) * m.rc;
                if (val < mn) {
                    mn = val;
                    mj = j;
                }
            }
        }
        uint64_t key = ((uint64_t)mn << 32) | ((uint64_t)r << v.tb) | mj;
        if (key < best) {
            best = key;
            best_b = b;
        }
        // step to the next candidate in Gray-rank order: exactly one dropped bit flips
        if (r + 1 < r1) {
            const uint32_t pos = m.dpos[ctz32(r + 1)];
            x ^= 1u << pos;
            if (incremental) {
                const bool set = (x >> pos) & 1u;
#pragma unroll
                for (int F = 0; F < NFR; ++F)
                    if (EXACT || (uint32_t)F < v.nf) {
                        uint32_t dlt = (uint32_t)v.fn_delta[F * FN_STRIDE + pos];
                        cost[F] += set ? dlt : (0u - dlt);
                    }
            }
        }
    }
    // the argmin j of the winner is looked up once (it never decides between candidates: r is unique)
    if (v.prevm && !m.first && (uint32_t)(best >> 32) != UMAX) {
        if constexpr (WIDE) best |= v.prevarg16[(size_t)best_b * v.T + i];
        else best |= v.prevarg[(size_t)best_b * v.T + i];
    }
    return best;
}

// Values-only evaluation for several input vectors at once (pass 1 of the batched pedigree sweep):
// the column costs of a cell are shared by all T right-hand sides, only the previous values differ.
// No tie-breaking is needed here — pass 2 recomputes the winners with the true inputs.
//   planes:       previous projection of right-hand side u at planes + u * plane_stride
//   first_chain:  the chain's first column: right-hand side u is the unit vector e_u, i.e. the
//                 transition minimum is popcount(i ^ u) * rc without touching memory
//   transformed:  planes hold transition minima (see ColView::prevm), else raw values
constexpr uint32_t MULTI_MAX = 8;

WHMEC_HD void eval_values_multi(const ColView &v, uint32_t o, uint32_t i, uint32_t r0, uint32_t r1, const uint32_t *planes,
                                uint64_t plane_stride, bool first_chain, bool transformed, uint32_t *mn /* [T] */) {
    const ColMeta &m = *v.m;
    const uint32_t drop = ~m.keep & low_mask(m.a);
    uint32_t kept;
    if (v.tab) {
        kept = v.tab->pd_lo[o & (TAB_SIZE - 1)] | v.tab->pd_hi[(o >> TAB_BITS) & (TAB_SIZE - 1)];
        if (v.tab->keep_rest) kept |= pdep32(o >> (2 * TAB_BITS), v.tab->keep_rest);
    } else {
        kept = pdep32(o, m.keep);
    }
    uint32_t x = kept | pdep32(r0 ^ (r0 >> 1), drop);
    const uint32_t bmask = low_mask(m.bw);
    for (uint32_t u = 0; u < v.T; ++u) mn[u] = UMAX;
    for (uint32_t r = r0; r < r1; ++r) {
        uint32_t cur = UMAX;
        for (uint32_t F = 0; F < v.nf; ++F) {
            uint32_t c = v.fn_c0[F];
            uint32_t j0 = 0;
            if (v.tab) {
                const size_t t = (size_t)(v.tab_fn0 + F) * TAB_SIZE;
                c += (uint32_t)(v.tab->lo[t + (x & (TAB_SIZE - 1))] + v.tab->hi[t + ((x >> TAB_BITS) & (TAB_SIZE - 1))]);
                j0 = 2 * TAB_BITS;
            }
            for (uint32_t j = j0; j < m.a; ++j)
                if ((x >> j) & 1u) c += (uint32_t)v.fn_delta[F * FN_STRIDE + j];
            if (c < cur) cur = c;
        }
        if (cur != UMAX) {
            const size_t b = (size_t)(x & bmask) * v.T;
            for (uint32_t u = 0; u < v.T; ++u) {
                uint32_t pm;
                if (first_chain) {
                    // the very first column of the table ignores its input: min_j popcount(i^j)*rc = 0
                    pm = m.first ? 0u : popc32(i ^ u) * m.rc;
                } else if (transformed) {
                    pm = planes[u * plane_stride + b + i];
                } else {
                    uint32_t arg;
                    pm = transition_min(planes + u * plane_stride + b, v.T, i, m.rc, &arg);
                }
                if (pm != UMAX && cur + pm < mn[u]) mn[u] = cur + pm;
            }
        }
        if (r + 1 < r1) x ^= 1u << m.dpos[ctz32(r + 1)];
    }
}

// Dispatch on the number of cost functions of the transmission group: the common small groups get a
// small code path (the whole kernel otherwise thrashes the instruction cache).  WIDE: the argmins of
// the transformed projection are 16-bit (T = 1024).
template <bool WIDE = false>
WHMEC_HD uint64_t eval_candidates(const ColView &v, uint32_t o, uint32_t i, uint32_t r0, uint32_t r1) {
    switch (v.nf) {  // exact small counts: no per-function predicates in the candidate loop
        case 1: return eval_candidates_t<1, true, WIDE>(v, o, i, r0, r1);
        case 2: return eval_candidates_t<2, true, WIDE>(v, o, i, r0, r1);
        case 3: return eval_candidates_t<3, true, WIDE>(v, o, i, r0, r1);
        case 4: return eval_candidates_t<4, true, WIDE>(v, o, i, r0, r1);
        default: break;
    }
    return eval_candidates_t<NF_REG, false, WIDE>(v, o, i, r0, r1);
}

// One backtrace step (pedigreedptable.cpp:155-160): given the back-pointer word of entry
// (b, tv) of column k-1's projection, recover that column's bipartition index.
WHMEC_HD uint32_t backpointer_to_index(const ColMeta &m, uint32_t tb, uint32_t out_index, uint32_t bp, uint32_t *argmin_j) {
    *argmin_j = bp & low_mask(tb);
    return candidate_index(m, out_index, bp >> tb);
}

// Read entry e of a packed back-pointer array (width in {0,1,2,4,8,16,32} bits).
WHMEC_HD uint32_t bp_load(const uint32_t *arena, uint64_t off_words, uint32_t width, uint64_t e) {
    if (width == 0) return 0;
    uint64_t bit = e * width;
    uint32_t word = arena[off_words + (bit >> 5)];
    return (width == 32) ? word : ((word >> (bit & 31)) & ((1u << width) - 1u));
}

// Packed back-pointer store used by the host-side emulation and by single-thread writers.
WHMEC_HD void bp_store_serial(uint32_t *arena, uint64_t off_words, uint32_t width, uint64_t e, uint32_t value) {
    if (width == 0) return;
    uint64_t bit = e * width;
    uint32_t *w = &arena[off_words + (bit >> 5)];
    if (width == 32) {
        *w = value;
    } else {
        uint32_t mask = ((1u << width) - 1u) << (bit & 31);
        *w = (*w & ~mask) | ((value << (bit & 31)) & mask);
    }
}

struct BtView {
    const ColMeta *cols;
    const uint32_t *arena;
    uint32_t T, tb;
};

// Backtrace from column k_last down to k_first (pedigreedptable.cpp:144-160).  (x, tv) is the
// cell chosen in k_last and prev_tv the argmin transmission value it was reached from.  Returns the
// transmission value the walk hands to column k_first - 1; with path_index == nullptr nothing is
// written (the walk only determines that value).
WHMEC_HD uint32_t backtrace_range(const BtView &v, uint32_t k_last, uint32_t k_first, uint32_t x, uint32_t tv,
                                  uint32_t prev_tv, uint32_t *path_index, uint32_t *path_tv) {
    if (path_index) {
        path_index[k_last] = x;
        path_tv[k_last] = tv;
    }
    for (uint32_t k = k_last; k > k_first; --k) {
        const uint32_t b = x & low_mask(v.cols[k].bw);
        const ColMeta &pm = v.cols[k - 1];
        const uint32_t bp = bp_load(v.arena, pm.bp_off, pm.bp_width, (uint64_t)b * v.T + prev_tv);
        uint32_t j;
        x = backpointer_to_index(pm, v.tb, b, bp, &j);
        tv = prev_tv;
        prev_tv = j;
        if (path_index) {
            path_index[k - 1] = x;
            path_tv[k - 1] = tv;
        }
    }
    return prev_tv;
}

// A chain (maximal run of columns connected by reads) is entered from its successor through the single
// projection index 0 of its last column: the successor's first column has bw == 0, so the step of
// backtrace_range that crosses the boundary reads entry (0, prev_tv).  `u` is that prev_tv.
WHMEC_HD void chain_entry(const BtView &v, uint32_t k_last, uint32_t u, uint32_t *x, uint32_t *prev_tv) {
    const ColMeta &m = v.cols[k_last];
    const uint32_t bp = bp_load(v.arena, m.bp_off, m.bp_width, u);
    *x = backpointer_to_index(m, v.tb, 0, bp, prev_tv);
}

// Min-plus fold of per-chain T x T transfer matrices over chains [c_first, n_chains): in <- in (x) M_c.
// Matrix row u of chain c is the T-vector `row(c, u)`; `each(c, in)` sees the input of chain c.
template <class Row, class Each>
WHMEC_HD void fold_chains(uint32_t T, uint32_t c_first, uint32_t n_chains, uint32_t *in, Row row, Each each) {
    uint32_t outv[MAX_T];
    for (uint32_t c = c_first; c < n_chains; ++c) {
        each(c, in);
        for (uint32_t i = 0; i < T; ++i) outv[i] = UMAX;
        for (uint32_t u = 0; u < T; ++u) {
            if (in[u] == UMAX) continue;
            const uint32_t *M = row(c, u);
            for (uint32_t i = 0; i < T; ++i) {
                if (M[i] == UMAX) continue;
                const uint32_t s = in[u] + M[i];
                if (s < outv[i]) outv[i] = s;
            }
        }
        for (uint32_t i = 0; i < T; ++i) in[i] = outv[i];
    }
}

// Pick the optimum of the last column (pedigreedptable.cpp:306-315): smallest (value, Gray rank, i).
WHMEC_HD void pick_optimum(const ColMeta &last, const uint32_t *vals, const uint32_t *arena, uint32_t T, uint32_t tb,
                           uint32_t *cost, uint32_t *x, uint32_t *tv, uint32_t *prev_tv) {
    uint32_t best_val = UMAX, best_r = UMAX, best_i = 0, best_j = 0;
    bool have = false;
    for (uint32_t i = 0; i < T; ++i) {
        uint32_t bp = bp_load(arena, last.bp_off, last.bp_width, i);
        uint32_t r = bp >> tb, val = vals[i];
        if (val == UMAX) continue;
        if (!have || val < best_val || (val == best_val && r < best_r)) {
            have = true;
            best_val = val;
            best_r = r;
            best_i = i;
            best_j = bp & low_mask(tb);
        }
    }
    *cost = best_val;
    *x = candidate_index(last, 0, have ? best_r : 0);
    *tv = best_i;
    *prev_tv = best_j;
}

}  // namespace whmec
