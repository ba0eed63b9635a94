// Host plan of whmec_genotype_batch (gl_batch.h): group cuts and the one step list of a group.
#include "gl_batch.h"

#include <algorithm>

namespace whmec {

namespace {

struct SubTable {     // a single individual's chain, or a whole pedigree table: columns [begin, end) of member m
    uint32_t m, begin, end;
    uint64_t f_off, f_size;
};

// The sub-tables of a table: runs of columns that end at a `last` column (gl_pack: a chain end when T == 1, else the table end).
template <class F>
void for_sub_tables(const GlPacked &g, uint32_t T, F &&fn) {
    const uint32_t n = (uint32_t)g.cols.size();
    for (uint32_t k = 0, begin = 0; k < n; ++k)
        if (g.cols[k].last || k + 1 == n) {
            uint64_t size = 1;  // F_{-1} of a table's first column: one entry
            for (uint32_t q = begin; q <= k; ++q)
                if (!g.cols[q].last) size = std::max(size, ((uint64_t)1 << g.cols[q].f) * T);
            fn(begin, k + 1, size);
            begin = k + 1;
        }
}

uint64_t input_bytes(const Packed &pk, const GlPacked &g) {
    return (uint64_t)pk.n * sizeof(GlCol) + g.eps.size() * 10 + pk.h2p.size() + (g.trans.size() + g.q.size()) * 8 + (uint64_t)pk.n * pk.n_ind * 3 * 8 +
           (uint64_t)pk.n * 2 * (sizeof(GlStep) + 4) + sizeof(GlBatchTable);
}

template <class V, class S>
uint64_t append(V &dst, const S &src) {
    const uint64_t at = dst.size();
    dst.insert(dst.end(), src.data(), src.data() + src.size());
    return at;
}

}  // namespace

uint64_t gl_batch_cost(const Packed &pk, const GlPacked &g) {
    uint64_t pool = 0;
    for_sub_tables(g, pk.T, [&](uint32_t, uint32_t, uint64_t size) { pool += 2 * size; });
    return g.beta_doubles + pool + (input_bytes(pk, g) + 7) / 8;
}

void gl_batch_groups(const std::vector<uint64_t> &cost, uint64_t budget, std::vector<std::vector<uint32_t>> &groups, std::vector<uint32_t> &alone) {
    groups.clear();
    alone.clear();
    const uint64_t room = budget > 0 ? budget - 1 : 0;  // one spare double per group's store
    uint64_t run = 0;
    for (uint32_t t = 0; t < cost.size(); ++t) {
        if (cost[t] == 0) continue;
        if (cost[t] > room) {
            alone.push_back(t);
            continue;
        }
        if (groups.empty() || run + cost[t] > room) {
            groups.emplace_back();
            run = 0;
        }
        groups.back().push_back(t);
        run += cost[t];
    }
}

void gl_batch_plan(const std::vector<Packed> &pks, const std::vector<GlPacked> &gs, const std::vector<uint32_t> &members, GlBatchGroup &out) {
    out = GlBatchGroup();
    out.members = members;
    std::vector<SubTable> subs;
    uint32_t longest = 0;
    for (uint32_t m = 0; m < members.size(); ++m) {
        const Packed &pk = pks[members[m]];
        const GlPacked &g = gs[members[m]];
        GlBatchTable d{};
        d.cols = append(out.cols, g.cols);
        d.act = append(out.eps, g.eps);
        append(out.allele, pk.act_allele);
        append(out.ind, pk.act_ind);
        d.h2p = append(out.h2p, pk.h2p);
        d.trans = append(out.trans, g.trans);
        d.q = append(out.q, g.q);
        d.beta_base = out.store_doubles;
        d.acc_base = out.acc_doubles;
        d.T = pk.T;
        d.P = pk.P;
        d.n_ind = pk.n_ind;
        d.n_cols = pk.n;
        out.tables.push_back(d);
        out.store_doubles += g.beta_doubles;
        out.acc_doubles += (uint64_t)pk.n * pk.n_ind * 3;
        for_sub_tables(g, pk.T, [&](uint32_t begin, uint32_t end, uint64_t size) {
            subs.push_back(SubTable{m, begin, end, out.f_pool_doubles, size});
            out.f_pool_doubles += 2 * size;
            longest = std::max(longest, end - begin);
        });
    }
    out.store_doubles += 1;  // a table's last column points one past its backward tables (never read)
    auto close_launch = [&](std::vector<uint32_t> &begin) {
        const uint32_t n = (uint32_t)out.steps.size() - begin.back();
        out.launches += 2 * ((n + GL_MAX_GRID_Y - 1) / GL_MAX_GRID_Y);
    };
    // backward: step s handles the s-th column from the right of every sub-table that still has a column to its left
    for (uint32_t s = 0; s + 1 < longest; ++s) {
        out.bwd_begin.push_back((uint32_t)out.steps.size());
        for (const SubTable &t : subs) {
            if (t.end - t.begin < s + 2) continue;
            const GlBatchTable &d = out.tables[t.m];
            const GlPacked &g = gs[members[t.m]];
            const uint32_t k = t.end - 1 - s;
            GlStep st{};
            st.k = k;
            st.cells_log2 = g.cols[k].a;
            st.cur_off = d.beta_base + g.cols[k - 1].beta_off;
            st.n_scale = ((uint64_t)1 << g.cols[k - 1].f) * d.T;
            out.steps.push_back(st);
            out.step_table.push_back(t.m);
        }
        close_launch(out.bwd_begin);
    }
    out.bwd_begin.push_back((uint32_t)out.steps.size());
    for (uint32_t s = 0; s < longest; ++s) {
        out.fwd_begin.push_back((uint32_t)out.steps.size());
        for (const SubTable &t : subs) {
            if (t.end - t.begin <= s) continue;
            const GlBatchTable &d = out.tables[t.m];
            const GlPacked &g = gs[members[t.m]];
            const uint32_t k = t.begin + s;
            GlStep st{};
            st.k = k;
            st.cells_log2 = g.cols[k].a;
            st.cur_off = t.f_off + (uint64_t)(s & 1) * t.f_size;
            st.prev_off = t.f_off + (uint64_t)((s + 1) & 1) * t.f_size;
            st.n_scale = g.cols[k].last ? 0 : ((uint64_t)1 << g.cols[k].f) * d.T;
            st.n_clear = t.f_size;
            out.steps.push_back(st);
            out.step_table.push_back(t.m);
        }
        close_launch(out.fwd_begin);
    }
    out.fwd_begin.push_back((uint32_t)out.steps.size());
}

}  // namespace whmec
