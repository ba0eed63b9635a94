// The row-limited heuristic on the device (whmec_heuristic_batch, DESIGN §4.10): one CTA sweeps one table's columns.
//
// heur_sweep() below is the whole sweep of one table, written once against an executor `X` that supplies the CTA-wide
// primitives: X::rows(n, f) runs f(i) for every row i < n in any order (the threads of the CTA on the device; a shuffled order
// in the host emulation, tests/emul/emul_heuristic_batch.cpp), X::single(f) runs f once, X::sync() is a barrier,
// X::scan(a, n) turns a[0..n) into its exclusive prefix sums and returns the total, and the atomics are those of the device.
// Every phase writes the rows in the order heuristic.cpp produces them (the merges, ties and the final argmin depend on it),
// and every float expression keeps heuristic.cpp's operand order (the .cu is compiled with -fmad=false), so the bipartition,
// transmission vector and hence every output equal whmec_heuristic's bit for bit.
//
// Rows live in two buffers (ping-pong), structure of arrays with row stride `cap`: a phase that reorders rows (merge, prune)
// writes the other buffer, a phase that appends rows (placement twins, transmission variants) writes behind the current ones.
// A phase that would need more than `cap` rows, and a column whose totals are not numbers or whose rows all vanish, stop the
// table with status HEUR_FALLBACK: the host then runs whmec_heuristic on it.
#pragma once
#include <stdint.h>
#include <math.h>
#include <string.h>

#include "common.h"

#if defined(__CUDACC__)
#define HEUR_FN __device__
#else
#define HEUR_FN inline
#endif

namespace whmec {

constexpr uint32_t HEUR_MAX_S = 16;        // samples a device table may have (best_phasing keeps its per-sample state in registers)
constexpr uint32_t HEUR_MAX_CAP = 65535;   // rows per buffer: back-pointers are 16 bits, as in heuristic.cpp
constexpr int32_t HEUR_OK = 0, HEUR_FALLBACK = 1;

struct HeurRows {       // one row buffer; element (e, r) at [e * cap + r]
    float *votes;       // [2S * Wmax]: haplotype h, window column x at e = h * Wmax + x
    uint8_t *side;      // [Amax]: sides of the active reads (kept reads first)
    uint8_t *placed;    // [NNmax]: sides given to the reads that start in the current column
    uint32_t *tv;
    float *score, *mut;
    uint32_t *from;     // row of the previous column this row continues
};

struct HeurDevTable {
    // inputs (heuristic_batch.cpp: heur_pack)
    const float *rc, *mc;                // [n]
    const float *ev;                     // [nnz] vote of every entry: q * a - q * (1 - a)
    const uint32_t *read_off;            // [m + 1] entry offsets of the table
    const uint32_t *ent_col;             // [nnz]
    const uint32_t *last, *sample;       // [m] last column and sample index of every read
    const uint32_t *start;               // [n + 1]
    const int8_t *gt;                    // [S][n]
    const uint32_t *trios;               // [3 * n_trios] sample indices
    const uint8_t *seen;                 // [S] initial `seen`
    // work
    HeurRows rows[2];
    int32_t *ht;                         // [ht_mask + 1] merge hash table
    uint32_t *a0, *a1, *a2, *a3;         // [cap] per-row scratch
    unsigned long long *best;            // [cap] per-group winner
    float *f0, *f1;                      // [cap]
    float *add;                          // [NNmax][Wmax] votes of the new reads
    int32_t *equal_to;                   // [NNmax]
    uint32_t *active, *kept;             // [Amax]
    // records: per column and row (at most rcap rows per column)
    uint16_t *back;                      // [n][rcap]
    uint32_t *rtv;                       // [n][rcap]
    uint8_t *rplaced;                    // [rcap * m]: column k's at rcap * start[k], row r's n_new sides at r * n_new
    // outputs
    uint8_t *part;                       // [m]
    uint32_t *tv_out;                    // [n]
    int32_t *status;
    uint32_t n, m, S, n_trios, row_limit, cap, rcap, Wmax, Amax, NNmax, ht_mask, distrust;
};

struct HeurShared {     // the CTA's shared scalars
    uint32_t count, W, W_prev, nk, n_active, right, fail, radix_prefix, radix_k, min_key;
    uint32_t hist[256];
    uint32_t warp_sums[33];
    uint8_t seen[HEUR_MAX_S];
};

WHMEC_HD float heur_min(float a, float b) { return (b < a) ? b : a; }  // std::min
WHMEC_HD float heur_max(float a, float b) { return (a < b) ? b : a; }  // std::max
WHMEC_HD float heur_abs(float a) { return fabsf(a); }                 // std::abs

// a monotone key of a float (canonical +0), for radix selection and argmin
WHMEC_HD uint32_t heur_key(float f) {
    f = f + 0.0f;
    uint32_t u;
    memcpy(&u, &f, 4);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
WHMEC_HD float heur_float(uint32_t u) {
    float f;
    memcpy(&f, &u, 4);
    return f;
}
WHMEC_HD float heur_unkey(uint32_t k) { return heur_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k); }
WHMEC_HD float heur_inf() { return heur_float(0x7F800000u); }

// The votes of one row, optionally with a read's votes `add` added to haplotype `hmod` (a placement before it is written).
struct HeurVotes {
    const float *v;
    uint32_t cap, Wmax, r;
    int32_t hmod;
    const float *add;
    WHMEC_HD float operator()(uint32_t h, uint32_t x) const {
        const float b = v[((size_t)h * Wmax + x) * cap + r];
        return (int32_t)h == hmod ? b + add[x] : b;
    }
};

// votes against the transmission `t` between parents and children over window columns 0 .. ahead (heuristic.cpp: mutation_cost)
WHMEC_HD float heur_mutation_cost(const HeurVotes &q, const uint32_t *trios, uint32_t n_trios, uint32_t W, float mc, uint32_t t, bool flips,
                                  uint32_t ahead) {
    float cost = 0.0;
    const uint32_t lastw = ahead < W - 1 ? ahead : W - 1;
    for (uint32_t i = 0; i <= lastw; ++i)
        for (uint32_t k = 0; k < n_trios; ++k) {
            const uint32_t a = trios[3 * k], b = trios[3 * k + 1], c = trios[3 * k + 2];
            const uint32_t sel_a = (t >> (2 * k)) & 1, sel_b = (t >> (2 * k + 1)) & 1;
            const float ca = q(2 * c, i), cb = q(2 * c + 1, i);
            const float pa = q(2 * a + sel_a, i), pb = q(2 * b + sel_b, i);
            if (flips) {
                if (ca * pa < 0) cost += heur_min(mc, heur_min(heur_abs(ca), heur_abs(pa)));
                if (cb * pb < 0) cost += heur_min(mc, heur_min(heur_abs(cb), heur_abs(pb)));
            } else {
                cost += (ca * pa < 0) * mc;
                cost += (cb * pb < 0) * mc;
            }
        }
    return cost;
}

// the score a placement of votes `add` on haplotype `row` (other: its sibling) costs (heuristic.cpp: add_votes, without the add)
WHMEC_HD float heur_add_votes(const HeurVotes &q, uint32_t row, uint32_t other, const float *add, const int8_t *target, uint32_t W,
                              bool distrust) {
    float penalty = 0;
    for (uint32_t i = 0; i < W; ++i) {
        const float basis = q(row, i), co = q(other, i);
        if (distrust) {
            if (basis * add[i] < 0) penalty += heur_min(heur_abs(basis), heur_abs(add[i]));
        } else if (target[i] == 1) {
            if (add[i] <= 0) penalty += heur_min(-add[i], heur_max(basis - co, (float)0));
            else penalty += heur_min(add[i], heur_max(co - basis, (float)0));
        } else {
            penalty += heur_abs(add[i]) * (add[i] * (target[i] - 1) < 0);
        }
    }
    return penalty;
}

// whether a new read is branched on (heuristic.cpp: `useful`)
WHMEC_HD bool heur_useful(const HeurVotes &q, uint32_t s, const float *b, const int8_t *target, uint32_t W, bool distrust) {
    bool useful = false;
    if (distrust) {
        for (uint32_t j = 0; j < W && !useful; ++j) {
            const float s0 = q(2 * s, j), s1 = q(2 * s + 1, j);
            useful |= (b[j] != 0 && s0 * s1 < 0) || ((b[j] + s0) * s0 <= 0 && (b[j] + s1) * s1 <= 0);
        }
    } else {
        for (uint32_t j = 0; j < W && !useful; ++j) useful |= (target[j] == 1 && b[j] != 0);
    }
    return useful;
}

// cost of the best joint phasing of column `col` under the first window column of the row's votes (heuristic.cpp: best_phasing)
WHMEC_HD float heur_best_phasing(const HeurVotes &q, const HeurDevTable &d, uint32_t t, uint32_t col) {
    const uint32_t S = d.S;
    const float mc = d.mc[col];
    float pc[HEUR_MAX_S * 5];
    uint8_t ph[HEUR_MAX_S][4], nph[HEUR_MAX_S], ctr[HEUR_MAX_S];
    for (uint32_t s = 0; s < S; ++s) {
        const float a0 = q(2 * s, 0), a1 = q(2 * s + 1, 0);
        float *c = &pc[s * 5];
        c[0] = (a0 * (a0 > 0) + a1 * (a1 > 0));
        c[1] = (-a0 * (a0 < 0) + a1 * (a1 > 0));
        c[2] = (a0 * (a0 > 0) - a1 * (a1 < 0));
        c[3] = (-a0 * (a0 < 0) - a1 * (a1 < 0));
        float largest = c[0];
        for (int i = 1; i < 4; ++i)
            if (largest < c[i]) largest = c[i];
        c[4] = largest;
    }
    for (uint32_t s = 0; s < S; ++s) {
        nph[s] = 0;
        ctr[s] = 0;
        if (d.distrust) {
            for (int i = 0; i < 4; ++i)
                if (pc[s * 5 + i] < pc[s * 5 + 4] + 2 * mc) ph[s][nph[s]++] = (uint8_t)i;
        } else {
            const int g = d.gt[(size_t)s * d.n + col];
            if (g == 0) ph[s][nph[s]++] = 0;
            else if (g == 2) ph[s][nph[s]++] = 3;
            else {
                ph[s][nph[s]++] = 1;
                ph[s][nph[s]++] = 2;
            }
        }
    }
    float best = heur_inf();
    for (uint32_t s = 0; s < S; ++s)
        if (nph[s] == 0) return best;
    while (ctr[S - 1] < nph[S - 1]) {
        float cost = 0.0;
        for (uint32_t k = 0; k < d.n_trios; ++k) {
            const uint32_t a = d.trios[3 * k], b = d.trios[3 * k + 1], c = d.trios[3 * k + 2];
            const uint32_t sel_a = (t >> (2 * k)) & 1, sel_b = (t >> (2 * k + 1)) & 1;
            const int child = ph[c][ctr[c]];
            const int8_t ca = child & 1, cb = (child & 2) >> 1;
            const int8_t pa = (ph[a][ctr[a]] & (1 + sel_a)) >> sel_a;
            const int8_t pb = (ph[b][ctr[b]] & (1 + sel_b)) >> sel_b;
            cost += (pa != ca) * mc;
            cost += (pb != cb) * mc;
        }
        for (uint32_t s = 0; s < S; ++s) cost += pc[s * 5 + ph[s][ctr[s]]];
        if (cost < best) best = cost;
        ++ctr[0];
        for (uint32_t j = 0; j + 1 < S; ++j)
            if (ctr[j] >= nph[j]) {
                ctr[j] = 0;
                ++ctr[j + 1];
            }
    }
    return best;
}

WHMEC_HD HeurVotes heur_votes(const HeurRows &b, const HeurDevTable &d, uint32_t r, int32_t hmod = -1, const float *add = nullptr) {
    return HeurVotes{b.votes, d.cap, d.Wmax, r, hmod, add};
}

// Copies the fields of row `src` of `a` to row `dst` of `b`: scalars, the first n_side sides, the first n_placed placements and
// the votes of window columns < W (element-parallel over `rows` copies: dst_of(j) / src_of(j) for j < rows).
template <class X, class Src, class Dst>
HEUR_FN void heur_copy_rows(X &x, const HeurDevTable &d, const HeurRows &a, const HeurRows &b, uint32_t rows, Src src_of, Dst dst_of,
                            uint32_t n_side, uint32_t n_placed, uint32_t W) {
    const size_t cap = d.cap;
    x.rows(rows, [&](uint32_t j) {
        const uint32_t s = src_of(j), t = dst_of(j);
        b.tv[t] = a.tv[s];
        b.score[t] = a.score[s];
        b.mut[t] = a.mut[s];
        b.from[t] = a.from[s];
        for (uint32_t i = 0; i < n_side; ++i) b.side[i * cap + t] = a.side[i * cap + s];
        for (uint32_t i = 0; i < n_placed; ++i) b.placed[i * cap + t] = a.placed[i * cap + s];
    });
    const uint32_t per_row = 2 * d.S * W;
    x.rows(rows * per_row, [&](uint32_t idx) {
        const uint32_t j = idx % rows, e = idx / rows;
        const size_t el = (size_t)(e / W) * d.Wmax + e % W;
        b.votes[el * cap + dst_of(j)] = a.votes[el * cap + src_of(j)];
    });
}

// Keeps the rows below the (row_limit + 1)-th smallest total and all rows at the minimum, in order (heuristic.cpp: prune).
// The threshold is found by a radix select on the totals' keys.  cur / count are updated.
template <class X>
HEUR_FN void heur_prune(X &x, HeurShared &sh, const HeurDevTable &d, int &cur, uint32_t n_side, uint32_t n_placed) {
    const HeurRows &a = d.rows[cur], &b = d.rows[cur ^ 1];
    const uint32_t count = sh.count;
    x.single([&] {
        sh.radix_prefix = 0;
        sh.radix_k = d.row_limit;
        sh.min_key = 0xFFFFFFFFu;
    });
    x.sync();
    x.rows(count, [&](uint32_t r) {
        const float tot = a.score[r] + a.mut[r];
        if (tot != tot) x.store(&sh.fail, 1u);
        d.a0[r] = heur_key(tot);
        x.atomic_min(&sh.min_key, d.a0[r]);
    });
    for (int shift = 24; shift >= 0; shift -= 8) {
        x.rows(256, [&](uint32_t i) { sh.hist[i] = 0; });
        x.sync();
        const uint32_t mask = shift == 24 ? 0u : (0xFFFFFFFFu << (shift + 8));
        const uint32_t prefix = sh.radix_prefix;
        x.rows(count, [&](uint32_t r) {
            const uint32_t k = d.a0[r];
            if ((k & mask) == prefix) x.atomic_add(&sh.hist[(k >> shift) & 255u], 1u);
        });
        x.sync();
        x.single([&] {
            uint32_t k = sh.radix_k, digit = 0;
            while (sh.hist[digit] <= k) k -= sh.hist[digit++];
            sh.radix_k = k;
            sh.radix_prefix = prefix | (digit << shift);
        });
        x.sync();
    }
    const float too_high = heur_unkey(sh.radix_prefix), mn = heur_unkey(sh.min_key);
    x.rows(count, [&](uint32_t r) {
        const float tot = a.score[r] + a.mut[r];
        d.a1[r] = (tot < too_high || tot == mn) ? 1u : 0u;
        d.a2[r] = d.a1[r];
    });
    x.sync();
    const uint32_t total = x.scan(d.a1, count);
    const uint32_t kept = total < HEUR_MAX_CAP ? total : HEUR_MAX_CAP;  // (heuristic.cpp: at most MAX_ROWS)
    x.rows(count, [&](uint32_t r) {
        if (d.a2[r] && d.a1[r] < kept) d.a3[d.a1[r]] = r;
    });
    x.sync();
    heur_copy_rows(x, d, a, b, kept, [&](uint32_t j) { return d.a3[j]; }, [](uint32_t j) { return j; }, n_side, n_placed, sh.W);
    x.sync();
    cur ^= 1;
    x.single([&] { sh.count = kept; });
    x.sync();
}

// First row holding the smallest score below +inf (heuristic.cpp: `q.score > old.score` from +inf, and the final argmin): the
// key orders by score, then row; ~0 when no score is below +inf.
WHMEC_HD unsigned long long heur_argmin_key(float score, uint32_t r) {
    return score < heur_inf() ? ((unsigned long long)heur_key(score) << 32) | r : ~0ull;
}

// The sweep of one table (heuristic.cpp: Solver::run from `solve` to the backtrace); d.status says whether it completed.
template <class X>
HEUR_FN void heur_sweep(X &x, HeurShared &sh, const HeurDevTable &d) {
    const size_t cap = d.cap;
    const uint32_t S = d.S, n = d.n;
    int cur = 0;
    x.single([&] {
        sh.count = 1;
        sh.W = 1;
        sh.n_active = 0;
        sh.right = 0;
        sh.fail = 0;
        for (uint32_t s = 0; s < S; ++s) sh.seen[s] = d.seen[s];
        const HeurRows &a = d.rows[0];
        a.tv[0] = 0;
        a.score[0] = 0;
        a.mut[0] = 0;
        a.from[0] = 0;
        for (uint32_t h = 0; h < 2 * S; ++h) a.votes[(size_t)h * d.Wmax * cap] = 0.0f;
    });
    x.sync();
    for (uint32_t col = 0; col < n; ++col) {
        const uint32_t s0 = d.start[col], n_new = d.start[col + 1] - s0;
        // ---- 1. reads that are still active, window of this column
        x.single([&] {
            uint32_t nk = 0;
            for (uint32_t i = 0; i < sh.n_active; ++i)
                if (d.last[d.active[i]] >= col) {
                    d.active[nk] = d.active[i];
                    d.kept[nk++] = i;
                }
            sh.nk = nk;
            sh.W_prev = sh.W;
            uint32_t right = sh.right > col ? sh.right : col;
            for (uint32_t r = s0; r < s0 + n_new; ++r) right = right > d.last[r] ? right : d.last[r];
            sh.right = right;
            sh.W = right + 1 - col;
        });
        x.rows(d.ht_mask + 1, [&](uint32_t i) { d.ht[i] = -1; });
        x.sync();
        // ---- merge: rows equal in tv and the kept sides form a group (first occurrence first), which continues its first
        // row of lowest score
        {
            const HeurRows &a = d.rows[cur], &b = d.rows[cur ^ 1];
            const uint32_t count = sh.count, nk = sh.nk, W = sh.W, W_prev = sh.W_prev;
            x.rows(count, [&](uint32_t r) {
                uint64_t h = 1469598103934665603ull ^ a.tv[r];
                for (uint32_t k = 0; k < nk; ++k) h = (h ^ a.side[(size_t)d.kept[k] * cap + r]) * 1099511628211ull;
                h ^= h >> 29;
                uint32_t slot = (uint32_t)(h * 0x9E3779B97F4A7C15ull >> 32) & d.ht_mask;
                for (;;) {
                    const int32_t old = x.atomic_cas(&d.ht[slot], -1, (int32_t)r);
                    if (old < 0) break;
                    bool same = a.tv[old] == a.tv[r];
                    for (uint32_t k = 0; k < nk && same; ++k) same = a.side[(size_t)d.kept[k] * cap + old] == a.side[(size_t)d.kept[k] * cap + r];
                    if (same) {
                        x.atomic_min(&d.ht[slot], (int32_t)r);
                        break;
                    }
                    slot = (slot + 1) & d.ht_mask;
                }
                d.a0[r] = slot;
            });
            x.sync();
            x.rows(count, [&](uint32_t r) {
                d.a1[r] = d.ht[d.a0[r]] == (int32_t)r ? 1u : 0u;
                d.best[r] = ~0ull;
            });
            x.sync();
            const uint32_t groups = x.scan(d.a1, count);  // a1[leader] = its group
            x.rows(count, [&](uint32_t r) {
                const uint32_t lead = (uint32_t)d.ht[d.a0[r]];
                const uint32_t g = d.a1[lead];
                if (lead == r) d.a2[g] = r;
                x.atomic_min(&d.best[g], heur_argmin_key(a.score[r], r));
            });
            x.sync();
            x.rows(groups, [&](uint32_t g) {
                const uint32_t lead = d.a2[g];
                const unsigned long long w = d.best[g];
                b.tv[g] = a.tv[lead];
                b.mut[g] = 0;
                if (w != ~0ull) {
                    b.score[g] = a.score[(uint32_t)w];
                    b.from[g] = (uint32_t)w;
                } else {
                    b.score[g] = heur_inf();
                    b.from[g] = 0;
                }
                d.a3[g] = w != ~0ull ? (uint32_t)w : 0xFFFFFFFFu;
                for (uint32_t k = 0; k < nk; ++k) b.side[k * cap + g] = a.side[(size_t)d.kept[k] * cap + lead];
            });
            x.sync();
            // the window moves on by one column and widens to W
            x.rows(groups * 2 * S * W, [&](uint32_t idx) {
                const uint32_t g = idx % groups, e = idx / groups, h = e / W, xw = e % W;
                const uint32_t w = d.a3[g];
                b.votes[((size_t)h * d.Wmax + xw) * cap + g] =
                    (w != 0xFFFFFFFFu && xw + 1 < W_prev) ? a.votes[((size_t)h * d.Wmax + xw + 1) * cap + w] : 0.0f;
            });
            x.single([&] { sh.count = groups; });
            cur ^= 1;
            x.sync();
        }
        // ---- 2. votes of the new reads; a read that agrees in sign and support with an earlier new read of its sample merges
        x.single([&] {
            const uint32_t W = sh.W;
            for (uint32_t i = 0; i < n_new; ++i) {
                const uint32_t r = s0 + i;
                d.active[sh.nk + i] = r;
                float *b = d.add + (size_t)i * d.Wmax;
                for (uint32_t xw = 0; xw < W; ++xw) b[xw] = 0.0f;
                for (uint32_t e = d.read_off[r]; e < d.read_off[r + 1]; ++e) b[d.ent_col[e] - col] += d.ev[e];
                d.equal_to[i] = -1;
                for (uint32_t j = 0; j < i; ++j) {
                    if (d.equal_to[j] != -1 || d.sample[s0 + j] != d.sample[r]) continue;
                    const float *aj = d.add + (size_t)j * d.Wmax;
                    bool same = true;
                    for (uint32_t xw = 0; xw < W; ++xw)
                        if (aj[xw] * b[xw] < 0 || (aj[xw] != 0.0) != (b[xw] != 0.0)) {
                            same = false;
                            break;
                        }
                    if (same) {
                        d.equal_to[i] = (int32_t)j;
                        float *aw = d.add + (size_t)j * d.Wmax;
                        for (uint32_t xw = 0; xw < W; ++xw) aw[xw] += b[xw];
                        break;
                    }
                }
            }
            sh.n_active = sh.nk + n_new;
        });
        x.sync();
        const uint32_t nk = sh.nk, W = sh.W;
        // ---- 3. placement of every new read: each row takes side 0; where the sample was seen, a twin takes side 1
        for (uint32_t i = 0; i < n_new; ++i) {
            const uint32_t s = d.sample[s0 + i];
            const int8_t *target = d.gt + (size_t)s * n + col;
            const float *bv = d.add + (size_t)i * d.Wmax;
            const HeurRows &a = d.rows[cur];
            const uint32_t count = sh.count;
            const int32_t eq = d.equal_to[i];
            if (eq >= 0) {
                x.rows(count, [&](uint32_t r) { a.placed[i * cap + r] = a.placed[(size_t)eq * cap + r]; });
            } else {
                const bool seen = sh.seen[s] != 0;
                x.rows(count, [&](uint32_t r) {
                    const HeurVotes v = heur_votes(a, d, r);
                    const bool useful = heur_useful(v, s, bv, target, W, d.distrust);
                    uint32_t code = 0;  // bit 0: a twin is appended, bit 1: the row becomes its twin
                    if (seen) {
                        const float ts = a.score[r] + heur_add_votes(v, 2 * s + 1, 2 * s, bv, target, W, d.distrust);
                        const float tm = heur_mutation_cost(heur_votes(a, d, r, 2 * s + 1, bv), d.trios, d.n_trios, W, d.mc[col], a.tv[r], true, 5);
                        d.f0[r] = ts;
                        d.f1[r] = tm;
                        code = useful ? 1u : 0u;
                    }
                    const float qs = a.score[r] + heur_add_votes(v, 2 * s, 2 * s + 1, bv, target, W, d.distrust);
                    const float qm = heur_mutation_cost(heur_votes(a, d, r, 2 * s, bv), d.trios, d.n_trios, W, d.mc[col], a.tv[r], true, 5);
                    if (seen && !useful && qs + qm > d.f0[r] + d.f1[r]) code = 2;
                    d.a1[r] = code & 1u;
                    d.a2[r] = code;
                    if (code == 2) {
                        a.score[r] = d.f0[r];
                        a.mut[r] = d.f1[r];
                        a.placed[i * cap + r] = 1;
                    } else {
                        a.score[r] = qs;
                        a.mut[r] = qm;
                        a.placed[i * cap + r] = 0;
                    }
                });
                x.sync();
                const uint32_t twins = x.scan(d.a1, count);
                if (count + twins > cap) {
                    x.single([&] { sh.fail = 1; });
                    x.sync();
                    break;
                }
                x.rows(count, [&](uint32_t r) {
                    if (!(d.a2[r] & 1u)) return;
                    const uint32_t t = count + d.a1[r];
                    a.tv[t] = a.tv[r];
                    a.score[t] = d.f0[r];
                    a.mut[t] = d.f1[r];
                    a.from[t] = a.from[r];
                    for (uint32_t k = 0; k < nk; ++k) a.side[k * cap + t] = a.side[k * cap + r];
                    for (uint32_t k = 0; k < i; ++k) a.placed[k * cap + t] = a.placed[k * cap + r];
                    a.placed[i * cap + t] = 1;
                });
                // votes: the twin is the row before its placement, with the read on haplotype 2s + 1
                x.rows(count * 2 * S * W, [&](uint32_t idx) {
                    const uint32_t r = idx % count, e = idx / count, h = e / W, xw = e % W;
                    const size_t el = ((size_t)h * d.Wmax + xw) * cap;
                    const uint32_t code = d.a2[r];
                    const float v = a.votes[el + r];
                    if (code & 1u) a.votes[el + count + d.a1[r]] = h == 2 * s + 1 ? v + bv[xw] : v;
                    if ((code == 2 && h == 2 * s + 1) || (code != 2 && h == 2 * s)) a.votes[el + r] = v + bv[xw];
                });
                x.single([&] { sh.count = count + twins; });
                x.sync();
            }
            x.single([&] { sh.seen[s] = 1; });
            x.sync();
            if (sh.count > d.row_limit) heur_prune(x, sh, d, cur, nk, i + 1);
            if (sh.fail) break;
        }
        if (sh.fail) break;
        // ---- 5. other transmission values for rows that pay for mutations here, in row order and ascending t
        {
            const HeurRows &a = d.rows[cur];
            const uint32_t count = sh.count, T = 1u << (2 * d.n_trios);
            x.rows(count, [&](uint32_t r) {
                const HeurVotes v = heur_votes(a, d, r);
                const float m0 = heur_mutation_cost(v, d.trios, d.n_trios, W, d.mc[col], a.tv[r], false, 0);
                a.mut[r] = m0;
                uint32_t k = 0;
                if (m0 > 0)
                    for (uint32_t t = 0; t < T; ++t) {
                        if (t == a.tv[r]) continue;
                        const float cost = d.rc[col] * (float)popc32(a.tv[r] ^ t);
                        if (cost >= m0) continue;
                        const float other = heur_mutation_cost(v, d.trios, d.n_trios, W, d.mc[col], t, false, 0);
                        if (other + cost >= m0) continue;
                        ++k;
                    }
                d.a1[r] = k;
                d.a2[r] = k;
            });
            x.sync();
            const uint32_t added = x.scan(d.a1, count);
            if (count + added > cap) {
                x.single([&] { sh.fail = 1; });
                x.sync();
                break;
            }
            if (added) {
                x.rows(count, [&](uint32_t r) {
                    if (!d.a2[r]) return;
                    const HeurVotes v = heur_votes(a, d, r);
                    const float m0 = a.mut[r];
                    uint32_t slot = count + d.a1[r];
                    for (uint32_t t = 0; t < T; ++t) {
                        if (t == a.tv[r]) continue;
                        const float cost = d.rc[col] * (float)popc32(a.tv[r] ^ t);
                        if (cost >= m0) continue;
                        const float other = heur_mutation_cost(v, d.trios, d.n_trios, W, d.mc[col], t, false, 0);
                        if (other + cost >= m0) continue;
                        a.tv[slot] = t;
                        a.score[slot] = a.score[r] + cost;
                        a.mut[slot] = other;
                        a.from[slot] = a.from[r];
                        d.a3[slot - count] = r;
                        ++slot;
                    }
                });
                x.sync();
                x.rows(added, [&](uint32_t j) {
                    const uint32_t r = d.a3[j], t = count + j;
                    for (uint32_t k = 0; k < nk; ++k) a.side[k * cap + t] = a.side[k * cap + r];
                    for (uint32_t k = 0; k < n_new; ++k) a.placed[k * cap + t] = a.placed[k * cap + r];
                });
                x.rows(added * 2 * S * W, [&](uint32_t idx) {
                    const uint32_t j = idx % added, e = idx / added;
                    const size_t el = ((size_t)(e / W) * d.Wmax + e % W) * cap;
                    a.votes[el + count + j] = a.votes[el + d.a3[j]];
                });
                x.single([&] { sh.count = count + added; });
            }
            x.sync();
            if (sh.count > d.row_limit) heur_prune(x, sh, d, cur, nk, n_new);
            if (sh.fail) break;
        }
        // ---- 6. the column is settled: cost of its best joint phasing; 7. records
        {
            const HeurRows &a = d.rows[cur];
            const uint32_t count = sh.count;
            if (count == 0 || count > d.rcap) {  // (no rows: heuristic.cpp's "kept no solution")
                x.single([&] { sh.fail = 1; });
                x.sync();
                break;
            }
            x.rows(count, [&](uint32_t r) {
                a.score[r] = a.score[r] + heur_best_phasing(heur_votes(a, d, r), d, a.tv[r], col);
                d.back[(size_t)col * d.rcap + r] = (uint16_t)a.from[r];
                d.rtv[(size_t)col * d.rcap + r] = a.tv[r];
                uint8_t *rec = d.rplaced + (size_t)d.rcap * s0 + (size_t)r * n_new;
                for (uint32_t k = 0; k < n_new; ++k) {
                    rec[k] = a.placed[k * cap + r];
                    a.side[(nk + k) * cap + r] = a.placed[k * cap + r];
                }
            });
            x.sync();
        }
    }
    // ---- best row of the last column (first minimum), walk back
    x.single([&] {
        if (sh.fail) {
            *d.status = HEUR_FALLBACK;
            return;
        }
        const HeurRows &a = d.rows[cur];
        unsigned long long best = ~0ull;
        for (uint32_t r = 0; r < sh.count; ++r) {
            const unsigned long long k = heur_argmin_key(a.score[r], r);
            if (k < best) best = k;
        }
        uint32_t row = best == ~0ull ? 0u : (uint32_t)best;
        const uint32_t tv_mask = d.n_trios ? (uint32_t)((1ull << (2 * d.n_trios)) - 1) : 0u;
        for (uint32_t col = n; col-- > 0;) {
            const uint32_t s0 = d.start[col], n_new = d.start[col + 1] - s0;
            for (uint32_t i = 0; i < n_new; ++i) d.part[s0 + i] = d.rplaced[(size_t)d.rcap * s0 + (size_t)n_new * row + i];
            d.tv_out[col] = d.rtv[(size_t)col * d.rcap + row] & tv_mask;
            row = d.back[(size_t)col * d.rcap + row];
        }
        *d.status = HEUR_OK;
    });
    x.sync();
}

}  // namespace whmec
