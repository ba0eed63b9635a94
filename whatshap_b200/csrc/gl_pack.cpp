// Host packing of the genotyping DP (gl_pack.h).  Restates, once per problem:
//   phred -> error probability          src/genotypecolumncostcomputer.cpp:24-45
//   transmission transition matrix      src/transitionprobabilitycomputer.cpp:18-44
//   allele-assignment priors            src/transitionprobabilitycomputer.cpp:46-89
// in the reference's long double arithmetic, rounded to double for the device.
#include "gl_pack.h"

#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>

#include "bounded.h"

namespace whmec {

namespace {

long double phred_probability(uint32_t phred) {  // genotypecolumncostcomputer.cpp:24-45
    if (phred == 0) return 0.9999L;
    return powl(10.0L, -(long double)(int)phred / 10.0L);
}

}  // namespace

namespace {

int pack_impl(const whmec_problem *p, bool continues, bool continued, Packed &pk, GlPacked &g, std::string &err);

}  // namespace

int gl_pack(const whmec_problem *p, Packed &pk, GlPacked &g, std::string &err) { return pack_impl(p, false, false, pk, g, err); }

int gl_pack_segment(const whmec_problem *p, bool continues, bool continued, Packed &pk, GlPacked &g, std::string &err) {
    int rc = pack_impl(p, continues, continued, pk, g, err);
    if (rc == WHMEC_OK && pk.T == 1) {
        err = "genotyping segments: a single individual's chains are independent tables already (shard them with whmec_genotype)";
        return WHMEC_ERR_UNSUPPORTED;
    }
    return rc;
}

namespace {

int pack_impl(const whmec_problem *p, bool continues, bool continued, Packed &pk, GlPacked &g, std::string &err) {
    g = GlPacked();
    if (p->n_cols > 0 && !p->gl) {
        // assert(gls != nullptr), transitionprobabilitycomputer.cpp:66
        err = "genotyping needs genotype likelihoods (priors) for every individual and column";
        return WHMEC_ERR_INPUT;
    }
    if (p->n_trios > 4 && p->n_trios < p->n_ind) {  // (before packing: with every assignment allowed, T = 1024 packs 2^20 functions per column)
        err = "unsupported: genotyping supports at most 4 trio relationships (T = 4^trios <= 256)";
        return WHMEC_ERR_UNSUPPORTED;
    }
    whmec_problem q = *p;
    q.distrust = 1;  // the column structure does not depend on genotypes; no genotype constraint applies here
    int rc = pack_problem(&q, pk, err, false);
    if (rc != WHMEC_OK) return rc;
    for (uint32_t r = 0; r < pk.n_reads; ++r)
        if (pk.read_first[r] == pk.read_last[r]) {
            // the reference asserts first column < last column (backwardcolumniterator.cpp:41) and aborts
            err = "genotyping: a read covers a single variant (reads need at least two)";
            return WHMEC_ERR_INPUT;
        }
    const uint32_t n = pk.n, T = pk.T, P = pk.P, nA = 1u << P, n_ind = pk.n_ind;
    if (n_ind > GL_MAX_IND || P > GL_MAX_P) {
        err = "unsupported pedigree size for genotyping";
        return WHMEC_ERR_UNSUPPORTED;
    }
    g.cols.resize(n);
    g.eps.resize(pk.act_phred.size());
    for (size_t e = 0; e < pk.act_phred.size(); ++e) g.eps[e] = (double)phred_probability(pk.act_phred[e]);
    g.trans.resize((size_t)n * T * T);
    g.q.resize((size_t)n * T * nA);
    const uint32_t trio_bits = pk.tb;
    for (uint32_t k = 0; k < n; ++k) {
        const ColMeta &m = pk.cols[k];
        GlCol &c = g.cols[k];
        c.a = m.a;
        c.bw = m.bw;
        c.keep = m.keep;
        c.f = m.f;
        // Without transmission values (T == 1) a chain boundary hands over a single number, which cancels in the
        // per-column normalisation: every DP-independent chain is then a table of its own (and they can be
        // processed group by group when the backward tables of all columns do not fit the device).
        c.first = (k == 0 && !continues) || (k > 0 && T == 1 && pk.cols[k - 1].f == 0);
        c.last = (k + 1 == n && !continued) || (T == 1 && m.f == 0);
        c.act_off = pk.act_off[k];
        c.beta_off = g.beta_doubles;
        const uint64_t proj = ((uint64_t)1 << m.f) * T;
        if (!c.last) g.beta_doubles += proj;
        g.max_proj = std::max(g.max_proj, proj);
        c.trans_off = (uint64_t)k * T * T;
        c.q_off = (uint64_t)k * T * nA;
        // transmission transitions
        const long double r = powl(10.0L, -(long double)p->recombcost[k] / 10.0L);
        std::vector<long double> bern(trio_bits + 1);
        for (uint32_t i = 0; i <= trio_bits; ++i) bern[i] = powl(r, (long double)i) * powl(1.0L - r, (long double)(trio_bits - i));
        for (uint32_t i = 0; i < T; ++i) {
            long double norm = 0.0L;
            for (uint32_t j = 0; j < T; ++j) norm += bern[popc32(i ^ j)];
            for (uint32_t j = 0; j < T; ++j) g.trans[c.trans_off + (size_t)i * T + j] = (double)(bern[popc32(i ^ j)] / norm);
        }
        // allele-assignment priors
        for (uint32_t i = 0; i < T; ++i) {
            const int8_t *h = &pk.h2p[(size_t)i * n_ind * 2];
            std::map<std::vector<uint8_t>, size_t> count;
            std::vector<std::vector<uint8_t>> geno(nA);
            std::vector<long double> prob(nA);
            for (uint32_t A = 0; A < nA; ++A) {
                long double pr = 1.0L;
                std::vector<uint8_t> gv(n_ind);
                for (uint32_t ind = 0; ind < n_ind; ++ind) {
                    const uint32_t gi = ((A >> h[2 * ind]) & 1u) + ((A >> h[2 * ind + 1]) & 1u);
                    pr *= p->gl[((size_t)ind * n + k) * 3 + gi];
                    gv[ind] = (uint8_t)gi;
                }
                count[gv] += 1;
                prob[A] = pr;
                geno[A] = gv;
            }
            long double norm = 0.0L;
            for (uint32_t A = 0; A < nA; ++A) {
                prob[A] /= count[geno[A]];
                norm += prob[A];
            }
            for (uint32_t A = 0; A < nA; ++A) g.q[c.q_off + (size_t)i * nA + A] = (double)(prob[A] / norm);
        }
    }
    return WHMEC_OK;
}

// doubles of B_k: none for a table's last column; a continued segment's last column owns T (beta_in)
uint64_t own_beta(const GlPacked &g, uint32_t T, uint32_t k) { return g.cols[k].last ? 0 : ((uint64_t)1 << g.cols[k].f) * T; }

}  // namespace

void gl_schedule(const GlPacked &g, uint32_t T, uint32_t lo, uint32_t hi, GlSchedule &out) {
    out = GlSchedule();
    out.beta_base = g.cols[lo].beta_off;
    // the group ends a table: its last column owns no entries, unless the table is continued in another segment
    out.beta_doubles = g.cols[hi - 1].beta_off + own_beta(g, T, hi - 1) - out.beta_base;
    struct Table {
        uint32_t begin, end;  // columns [begin, end)
        uint64_t f_off, f_size;
    };
    std::vector<Table> tables;
    uint32_t longest = 0;
    for (uint32_t k = lo, begin = lo; k < hi; ++k)
        if (g.cols[k].last || k + 1 == hi) {
            uint64_t size = g.cols[begin].first ? 1 : T;  // a continuing segment: F_{lo-1} = alpha_in, T entries
            for (uint32_t q = begin; q <= k; ++q)
                if (!g.cols[q].last) size = std::max(size, ((uint64_t)1 << g.cols[q].f) * T);
            tables.push_back(Table{begin, k + 1, out.f_pool_doubles, size});
            out.f_pool_doubles += 2 * size;
            longest = std::max(longest, k + 1 - begin);
            begin = k + 1;
        }
    // backward: step s handles the s-th column from the right of every table that still has a column to its left
    for (uint32_t s = 0; s + 1 < longest; ++s) {
        out.bwd_begin.push_back((uint32_t)out.steps.size());
        for (const Table &t : tables) {
            if (t.end - t.begin < s + 2) continue;
            const uint32_t k = t.end - 1 - s;
            GlStep st{};
            st.k = k;
            st.cells_log2 = g.cols[k].a;
            st.cur_off = g.cols[k - 1].beta_off - out.beta_base;
            st.n_scale = ((uint64_t)1 << g.cols[k - 1].f) * T;
            out.steps.push_back(st);
        }
    }
    out.bwd_begin.push_back((uint32_t)out.steps.size());
    for (uint32_t s = 0; s < longest; ++s) {
        out.fwd_begin.push_back((uint32_t)out.steps.size());
        for (const Table &t : tables) {
            if (t.end - t.begin <= s) continue;
            const uint32_t k = t.begin + s;
            GlStep st{};
            st.k = k;
            st.cells_log2 = g.cols[k].a;
            st.cur_off = t.f_off + (uint64_t)(s & 1) * t.f_size;
            st.prev_off = t.f_off + (uint64_t)((s + 1) & 1) * t.f_size;
            st.n_scale = g.cols[k].last ? 0 : ((uint64_t)1 << g.cols[k].f) * T;
            st.n_clear = t.f_size;
            out.steps.push_back(st);
        }
    }
    out.fwd_begin.push_back((uint32_t)out.steps.size());
}

void gl_groups_split(const GlPacked &g, uint32_t T, uint64_t budget, std::vector<uint32_t> &begin, std::vector<uint8_t> &alone) {
    begin.assign(1, 0);
    alone.clear();
    const uint32_t n = (uint32_t)g.cols.size();
    uint64_t run = 0, table = 0, widest = (n && !g.cols[0].first) ? T : 1;  // a continuing segment: alpha_in in the F pool
    uint32_t table_begin = 0;
    for (uint32_t k = 0; k < n; ++k) {
        if (!g.cols[k].last) {
            const uint64_t proj = ((uint64_t)1 << g.cols[k].f) * T;
            table += proj;
            widest = std::max(widest, proj);
            if (k + 1 < n) continue;  // a continued segment's table ends at its last column all the same
        }
        const uint64_t cost = table + 2 * widest;  // a table ends here: its backward tables and its two projection buffers
        if (cost > budget) {  // a group of its own: close the open group (if any) before it and start a new one after it
            if (table_begin > begin.back()) {
                begin.push_back(table_begin);
                alone.push_back(0);
            }
            begin.push_back(k + 1);
            alone.push_back(1);
            run = 0;
        } else {
            if (run + cost > budget) {  // close the group before this table
                begin.push_back(table_begin);
                alone.push_back(0);
                run = 0;
            }
            run += cost;
        }
        table_begin = k + 1;
        table = 0;
        widest = 1;
    }
    if (begin.back() < n) {
        begin.push_back(n);
        alone.push_back(0);
    }
}

bool gl_groups(const GlPacked &g, uint32_t T, uint64_t budget, std::vector<uint32_t> &begin) {
    std::vector<uint8_t> alone;
    gl_groups_split(g, T, budget, begin, alone);
    return std::find(alone.begin(), alone.end(), 1) == alone.end();
}

bool gl_bounded(const GlPacked &g, uint32_t T, uint32_t lo, uint32_t hi, uint64_t budget, GlBounded &out) {
    out = GlBounded();
    const uint32_t m = hi - lo;
    auto own = [&](uint32_t k) { return own_beta(g, T, k); };  // doubles of B_k
    uint64_t f_size = g.cols[lo].first ? 1 : T;  // a continuing segment: F_{lo-1} = alpha_in, T entries
    for (uint32_t k = lo; k < hi; ++k) f_size = std::max(f_size, own(k));
    out.f_pool_doubles = 2 * f_size;
    const uint64_t tail = own(hi - 1);  // a continued segment: beta_in, the checkpoint of the last segment
    if (budget <= out.f_pool_doubles + tail) return false;
    // mirrored order: column j is column hi - 1 - j.  A mirrored segment that starts at j + 1 is a segment that ends at column
    // hi - 2 - j; its checkpoint is B_{hi - 2 - j}.
    std::vector<uint64_t> off(m + 1, 0), ck(m, 0);
    for (uint32_t j = 0; j < m; ++j) {
        off[j + 1] = off[j] + own(hi - 1 - j);
        if (j + 1 < m) ck[j] = own(hi - 2 - j);
    }
    std::vector<uint32_t> mcuts;
    if (!cut_column_segments(off, ck, budget - out.f_pool_doubles - tail, mcuts, out.arena_doubles, out.ckpt_doubles)) return false;
    out.ckpt_doubles += tail;
    for (size_t c = mcuts.size(); c-- > 0;) out.cuts.push_back(hi - mcuts[c]);
    const uint32_t S = (uint32_t)out.cuts.size() - 1;
    const std::vector<uint32_t> &c = out.cuts;
    const uint64_t A = out.arena_doubles;
    std::vector<uint64_t> ckpt(S, 0);  // store offset of segment s's checkpoint (s < S - 1; s = S - 1 only with a tail)
    uint64_t at = 0;
    for (uint32_t s = 0; s + 1 < S || (tail && s < S); ++s) {
        ckpt[s] = A + at;
        at += own(c[s + 1] - 1);
    }
    if (tail) out.tail_off = ckpt[S - 1];
    auto beta_off = [&](uint32_t k) { return g.cols[k].beta_off; };
    auto backward = [&](uint32_t k, uint64_t dst) {  // column k reads B_k, adds into B_{k-1} at dst
        GlStep st{};
        st.k = k;
        st.cells_log2 = g.cols[k].a;
        st.cur_off = dst;
        st.n_scale = own(k - 1);
        out.steps.push_back(st);
    };
    // the backward tables of segment s: zero its window but the last column's, put the checkpoint there and sweep
    auto resweep = [&](uint32_t s, GlSweep &sw, bool clear) {
        const uint64_t base = beta_off(c[s]);
        sw.beta_base = base;
        sw.clear = clear ? beta_off(c[s + 1] - 1) - base : 0;
        if (s + 1 < S || tail) {
            sw.copy_dst = beta_off(c[s + 1] - 1) - base;
            sw.copy_src = ckpt[s];
            sw.copy_n = own(c[s + 1] - 1);
        }
        sw.bwd_begin = (uint32_t)out.steps.size();
        for (uint32_t k = c[s + 1] - 1; k > c[s]; --k) backward(k, beta_off(k - 1) - base);
    };
    for (uint32_t s = S; s-- > 0;) {  // pass A (the store starts zeroed)
        GlSweep sw{};
        resweep(s, sw, s + 1 < S);
        if (s > 0) backward(c[s], ckpt[s - 1]);
        sw.bwd_end = sw.fwd_begin = sw.fwd_end = (uint32_t)out.steps.size();
        out.sweeps.push_back(sw);
    }
    for (uint32_t s = 0; s < S; ++s) {  // pass B
        GlSweep sw{};
        if (s > 0) resweep(s, sw, true);
        else {
            sw.beta_base = beta_off(c[0]);
            sw.bwd_begin = (uint32_t)out.steps.size();
        }
        sw.bwd_end = sw.fwd_begin = (uint32_t)out.steps.size();
        for (uint32_t k = c[s]; k < c[s + 1]; ++k) {  // as gl_schedule's forward steps of a one-table group
            const uint32_t i = k - lo;
            GlStep st{};
            st.k = k;
            st.cells_log2 = g.cols[k].a;
            st.cur_off = (uint64_t)(i & 1) * f_size;
            st.prev_off = (uint64_t)((i + 1) & 1) * f_size;
            st.n_scale = own(k);
            st.n_clear = f_size;
            out.steps.push_back(st);
        }
        sw.fwd_end = (uint32_t)out.steps.size();
        out.sweeps.push_back(sw);
    }
    return true;
}

int gl_plan(const GlPacked &g, uint32_t T, uint64_t budget, std::vector<GlUnit> &units, std::string &err) {
    std::vector<uint32_t> begin;
    std::vector<uint8_t> alone;
    gl_groups_split(g, T, budget, begin, alone);
    units.assign(alone.size(), GlUnit());
    uint64_t need = 0;  // > 0: the least budget that the refused tables fit
    for (size_t q = 0; q < units.size(); ++q) {
        GlUnit &u = units[q];
        u.bounded = alone[q];
        const uint32_t hi = begin[q + 1];
        if (!u.bounded) {
            gl_schedule(g, T, begin[q], hi, u.sc);
            u.work_doubles = u.sc.beta_doubles + 1 + u.sc.f_pool_doubles;
            u.alpha_at = u.sc.beta_doubles + 1 + u.sc.steps[u.sc.fwd_begin[0]].prev_off;
            u.beta_at = g.cols[hi - 1].beta_off - u.sc.beta_base;
        } else if (gl_bounded(g, T, begin[q], hi, budget, u.bd)) {
            const uint64_t store = u.bd.arena_doubles + u.bd.ckpt_doubles;
            u.work_doubles = store + u.bd.f_pool_doubles;
            u.alpha_at = store + u.bd.steps[u.bd.sweeps[u.bd.cuts.size() - 1].fwd_begin].prev_off;  // pass B's first step
            u.beta_at = u.bd.tail_off;
        } else {  // the least budget with a cut that fits (bisection), at most the table's resident cost.  A continued segment keeps
                  // beta_in twice there: in its last column's backward table (beta_doubles) and as the last segment's checkpoint
            GlSchedule whole;
            gl_schedule(g, T, begin[q], hi, whole);
            uint64_t no = budget, yes = whole.beta_doubles + whole.f_pool_doubles + own_beta(g, T, hi - 1);
            GlBounded probe;
            while (yes - no > 1) {
                const uint64_t mid = no + (yes - no) / 2;
                (gl_bounded(g, T, begin[q], hi, mid, probe) ? yes : no) = mid;
            }
            need = std::max(need, yes);
        }
    }
    if (need) {
        err = "genotyping: " + std::to_string(budget * 8) + " bytes for backward tables and projection buffers hold no segment of a table; it needs at least " +
              std::to_string(need * 8) + " bytes";
        return WHMEC_ERR_UNSUPPORTED;
    }
    return WHMEC_OK;
}

void gl_transfer_plan(const GlPacked &g, uint32_t T, bool continues, GlTransfer &out) {
    out = GlTransfer();
    const uint32_t n = (uint32_t)g.cols.size();
    out.n_in = continues ? std::min(T, GL_T_LOCAL) : 1;
    out.n_batches = continues ? T / out.n_in : 1;
    uint64_t f_size = T;  // the inputs: [u][T]
    for (uint32_t k = 0; k < n; ++k) f_size = std::max(f_size, ((uint64_t)1 << g.cols[k].f) * T);
    const uint64_t half = f_size * out.n_in;
    out.f_pool_doubles = 2 * half;
    for (uint32_t k = 0; k < n; ++k) {
        GlStep st{};
        st.k = k;
        st.cells_log2 = g.cols[k].a;
        st.cur_off = (uint64_t)(k & 1) * half;
        st.prev_off = (uint64_t)((k + 1) & 1) * half;
        st.n_scale = ((uint64_t)1 << g.cols[k].f) * T * out.n_in;
        st.n_clear = half;
        out.steps.push_back(st);
    }
    out.in_off = half;                       // steps[0].prev_off
    out.out_off = n ? out.steps[n - 1].cur_off : 0;
}

void gl_transfer_combine(const GlTransfer &tp, uint32_t T, const std::vector<double> &rows, const std::vector<double> &col_max, double *m) {
    if (tp.n_in * tp.n_batches < T) {  // a segment that starts the table: every row is the one row it computed
        for (uint32_t u = 0; u < T; ++u) std::copy(rows.begin(), rows.begin() + T, m + (size_t)u * T);
        return;
    }
    const size_t n = tp.steps.size(), B = tp.n_batches;
    std::vector<long double> mant(B, 1.0L);  // batch b's product of scales = mant[b] * 2^ex[b], mant in [0.5, 1)
    std::vector<int64_t> ex(B, 0);
    for (size_t b = 0; B > 1 && b < B; ++b)
        for (size_t k = 0; k < n; ++k) {
            const double mx = col_max[b * n + k];
            if (!(mx > 0.0)) continue;  // an all-zero column is not divided (its rows stay 0)
            int e = 0;
            mant[b] = frexpl(mant[b] * (long double)mx, &e);
            ex[b] += e;
        }
    size_t top = 0;
    for (size_t b = 1; b < B; ++b)
        if (ex[b] > ex[top] || (ex[b] == ex[top] && mant[b] > mant[top])) top = b;
    for (size_t b = 0; b < B; ++b) {
        const int64_t d = std::max<int64_t>(ex[b] - ex[top], -100000);  // far below the smallest double: 0
        const double f = B > 1 ? (double)ldexpl(mant[b] / mant[top], (int)d) : 1.0;
        for (size_t e = b * tp.n_in * T; e < (b + 1) * tp.n_in * T; ++e) m[e] = rows[e] * f;
    }
}

void gl_scale_host(double *v, uint64_t n) {
    double mx = 0.0;
    for (uint64_t i = 0; i < n; ++i) mx = v[i] > mx ? v[i] : mx;
    if (!(mx > 0.0)) return;
    const double inv = 1.0 / mx;
    for (uint64_t i = 0; i < n; ++i) v[i] *= inv;
}

void gl_normalise(const double *acc, uint32_t n, uint32_t n_ind, double *likelihoods) {
    for (uint32_t k = 0; k < n; ++k) {
        const double *a0 = acc + (size_t)k * n_ind * 3;
        const double total = a0[0] + a0[1] + a0[2];  // every (x, i, A) lands in exactly one genotype of each individual
        for (uint32_t ind = 0; ind < n_ind; ++ind)
            for (uint32_t gi = 0; gi < 3; ++gi) likelihoods[((size_t)ind * n + k) * 3 + gi] = a0[ind * 3 + gi] / total;
    }
}

}  // namespace whmec

// compute_genotypes (src/genotyper.cpp:12-54): columns are independent; within a column the factors are applied in
// the order of the column iterator (ascending read index) so that every double equals the reference's.
extern "C" int whmec_compute_genotypes(const whmec_problem *p, double *gl, int8_t *gt, char *err, size_t errlen) {
    using namespace whmec;
    std::string msg;
    int rc = WHMEC_OK;
    try {
        if (!p || !gl || !gt) {
            msg = "null argument";
            rc = WHMEC_ERR_INPUT;
        } else {
            whmec_problem q = *p;
            q.n_ind = 1;  // one sample's reads; no pedigree, no genotype constraint
            q.n_trios = 0;
            q.trios = nullptr;
            q.distrust = 0;
            std::vector<uint8_t> het(p->n_cols, 1);
            std::vector<uint32_t> zero_ind(p->n_reads, 0), no_cost(p->n_cols, 0);
            q.gt = het.data();
            q.gl = nullptr;
            q.read_ind = zero_ind.data();
            if (!q.recombcost) q.recombcost = no_cost.data();
            Packed pk;
            rc = pack_problem(&q, pk, msg, false);
            if (rc == WHMEC_OK) {
                const uint32_t n = pk.n;
                const uint32_t n_tasks = n / 2048 + 1, step = (n + n_tasks - 1) / n_tasks;
                parallel_tasks(n_tasks, host_threads(16), [&](uint32_t task) {
                    for (uint32_t k = task * step; k < std::min(n, (task + 1) * step); ++k) {
                        double d[3] = {1.0 / 3.0, 1.0 / 3.0, 1.0 / 3.0};
                        const uint64_t e0 = pk.act_off[k];
                        for (uint32_t j = 0; j < pk.cols[k].a; ++j) {
                            const uint8_t al = pk.act_allele[e0 + j];
                            if (al > 1) continue;
                            const double p_wrong = std::max(0.05, std::pow(10.0, -((double)pk.act_phred[e0 + j]) / 10.0));
                            const double f_same = 2.0 / 3.0 - 1.0 / 3.0 * p_wrong, f_het = 1.0 / 3.0, f_other = 1.0 / 3.0 * p_wrong;
                            const double f[3] = {al == 0 ? f_same : f_other, f_het, al == 0 ? f_other : f_same};
                            double sum = 0.0;  // operator* (genotypedistribution.cpp:56-66)
                            for (int i = 0; i < 3; ++i) {
                                d[i] *= f[i];
                                sum += d[i];
                            }
                            for (int i = 0; i < 3; ++i) d[i] /= sum;
                        }
                        double p_sum = 0.0;  // normalize (:24-36)
                        for (int i = 0; i < 3; ++i) p_sum += d[i];
                        if (p_sum <= 0.0) d[0] = d[1] = d[2] = 1.0 / 3.0;
                        else
                            for (int i = 0; i < 3; ++i) d[i] /= p_sum;
                        int best_index = 0;  // likeliestGenotype / errorProbability (:12-22,37-55)
                        double best = 0.0;
                        for (int i = 0; i < 3; ++i)
                            if (d[i] > best) {
                                best = d[i];
                                best_index = i;
                            }
                        double p_err = 0.0;
                        for (int i = 0; i < 3; ++i)
                            if (i != best_index) p_err += d[i];
                        gt[k] = p_err < 0.1 ? (int8_t)best_index : (int8_t)-1;
                        for (int i = 0; i < 3; ++i) gl[(size_t)k * 3 + i] = d[i];
                    }
                });
            }
        }
    } catch (const std::exception &e) {
        msg = e.what();
        rc = WHMEC_ERR_INPUT;
    }
    if (rc != WHMEC_OK && err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = 0;
    }
    return rc;
}
