// TEST-ONLY host emulation of a tile group of whmec_solve_batch: the host code that forms the union of several tables'
// schedules (tile_plan.cpp: merge_tile_tables, cut_table_groups) is the product's; the union is then swept by the emulated
// schedule of emul_sched.cpp (work items in a seeded random order that respects only the completion counters), every chain
// is backtraced and every table's cost is the sum of its chains' optima, as tile_table_cost_kernel forms it.
#include "emul_sched.cpp"

namespace {

// the invariants of whemul_sched_check on a union, plus the numbering of tables: returns 0 or the first one broken
//   8  chains / columns of table t are exactly [table_chain[t], table_chain[t+1]) / [table_col[t], table_col[t+1])
//   9  state buffers and back-pointer words of different tables do not overlap
int check_union(const TileUnion &un, const std::vector<const Packed *> &pks, const std::vector<const TileSchedule *> &tss) {
    const TileSchedule &ts = un.ts;
    const Packed &pk = un.pk;
    const uint32_t np = (uint32_t)ts.panels.size();
    std::vector<uint32_t> round_of(np);
    for (uint32_t r = 0; r + 1 < ts.round_begin.size(); ++r)
        for (uint32_t q = ts.round_begin[r]; q < ts.round_begin[r + 1]; ++q) round_of[q] = r;
    uint64_t item = 0;
    for (uint32_t q = 0; q < np; ++q) {
        const Panel &P = ts.panels[q];
        if (P.tile_begin != item) return 1;
        item += panel_tiles(P);
        if (P.fresh) {
            if (P.producer != TILE_NO_PANEL || P.producer_tiles != 0 || P.col_begin != pk.chain_begin[P.chain]) return 2;
            continue;
        }
        if (P.producer >= q) return 3;
        const Panel &A = ts.panels[P.producer];
        if (A.chain != P.chain || A.col_end != P.col_begin || A.ends_chain) return 3;
        if ((uint64_t)A.tile_begin + panel_tiles(A) > P.tile_begin) return 4;
        if (P.producer_tiles != panel_tiles(A)) return 5;
        if (P.in_off != A.out_off || (!P.ends_chain && P.out_off == P.in_off) || A.in_off == A.out_off) return 6;
        if (round_of[P.producer] + 1 != round_of[q]) return 7;
    }
    uint64_t state_at = 0, bp_at = 0;
    for (size_t t = 0; t < pks.size(); ++t) {
        if (un.table_chain[t + 1] - un.table_chain[t] != pks[t]->chain_begin.size() - 1 || un.table_col[t + 1] - un.table_col[t] != pks[t]->n) return 8;
        for (uint32_t c = un.table_chain[t]; c < un.table_chain[t + 1]; ++c)
            if (pk.chain_begin[c] < un.table_col[t] || pk.chain_begin[c + 1] > un.table_col[t + 1]) return 8;
        for (uint32_t k = un.table_col[t]; k < un.table_col[t + 1]; ++k) {
            const TileCol &tc = ts.cols[k];
            const uint64_t words = (uint64_t)tc.bp_tile_stride << (tc.g - tc.half);
            if (words && (tc.bp_off < bp_at || tc.bp_off + words > bp_at + tss[t]->bp_words)) return 9;
        }
        for (const Panel &P : ts.panels)
            if (P.chain >= un.table_chain[t] && P.chain < un.table_chain[t + 1] && !P.ends_chain &&
                (P.out_off < state_at || P.out_off + ((uint64_t)1 << (P.s_out + P.g)) > state_at + tss[t]->state_words))
                return 9;
        state_at += tss[t]->state_words;
        bp_at += tss[t]->bp_words;
    }
    return 0;
}

}  // namespace

// status[t]: WHMEC_OK, the packer's error code, or 100 (no columns / the tile planner declines: not part of the group).
// info4: tables in the group, chains, panels, work items of the union.  Returns the first broken invariant of the union, or 0.
extern "C" int whemul_batch_solve(const whmec_problem *const *problems, whmec_solution *const *sols, uint32_t n_tables, uint64_t seed, int *status,
                                  uint64_t *info4) {
    std::vector<Packed> packed(n_tables);
    std::vector<TileSchedule> sched(n_tables);
    std::vector<uint32_t> members;
    std::vector<const Packed *> pks;
    std::vector<const TileSchedule *> tss;
    for (uint32_t t = 0; t < n_tables; ++t) {
        std::string msg;
        status[t] = pack_problem(problems[t], packed[t], msg, false);
        if (status[t] != WHMEC_OK) continue;
        if (packed[t].n) plan_tiles(packed[t], sched[t]);
        if (!sched[t].eligible) {
            status[t] = 100;
            continue;
        }
        members.push_back(t);
        pks.push_back(&packed[t]);
        tss.push_back(&sched[t]);
    }
    TileUnion un;
    merge_tile_tables(pks, tss, un);
    const int broken = check_union(un, pks, tss);
    if (broken) return broken;
    const TileSchedule &ts = un.ts;
    std::mt19937_64 rng(seed);
    std::vector<uint32_t> state(ts.state_words + 1, POISON), arena(ts.bp_words + 1, 0);
    const uint32_t n_chains = un.table_chain[members.size()];
    std::vector<uint64_t> chain_key(n_chains, KEY_INF);
    SchedInfo info;
    run_segment(un.pk, ts, 0, (uint32_t)ts.panels.size(), rng, state, arena, chain_key, info);
    std::vector<uint32_t> pidx(un.pk.n);
    for (uint32_t c = 0; c < n_chains; ++c)
        tile_backtrace_chain(un.pk.cols.data(), ts.cols.data(), arena.data(), un.pk.chain_begin[c], un.pk.chain_begin[c + 1] - 1, chain_key[c], pidx.data());
    for (size_t i = 0; i < members.size(); ++i) {
        const uint32_t t = members[i];
        uint32_t cost = 0;
        for (uint32_t c = un.table_chain[i]; c < un.table_chain[i + 1]; ++c) cost += (uint32_t)(chain_key[c] >> 32);
        sols[t]->cost = cost;
        const std::vector<uint32_t> ptv(packed[t].n, 0);
        std::string msg;
        status[t] = build_outputs(packed[t], pidx.data() + un.table_col[i], ptv.data(), sols[t], msg);
    }
    if (info4) {
        info4[0] = members.size();
        info4[1] = n_chains;
        info4[2] = ts.panels.size();
        info4[3] = info.items;
    }
    return 0;
}

// cut_table_groups as the product calls it: groups as (first, last) pairs in out_groups (returns their number), tables that
// take the single-table path in out_alone (*n_alone)
extern "C" uint32_t whemul_cut_groups(const uint64_t *bytes, const uint64_t *items, uint32_t n, uint64_t budget, uint32_t *out_groups, uint32_t *out_alone,
                                      uint32_t *n_alone) {
    std::vector<std::pair<uint32_t, uint32_t>> groups;
    std::vector<uint32_t> alone;
    cut_table_groups(std::vector<uint64_t>(bytes, bytes + n), std::vector<uint64_t>(items, items + n), budget, groups, alone);
    for (size_t g = 0; g < groups.size(); ++g) {
        out_groups[2 * g] = groups[g].first;
        out_groups[2 * g + 1] = groups[g].second;
    }
    std::copy(alone.begin(), alone.end(), out_alone);
    *n_alone = (uint32_t)alone.size();
    return (uint32_t)groups.size();
}

// device bytes and work items the product counts for one table (0, 0: not a tile table)
extern "C" int whemul_table_bytes(const whmec_problem *p, uint64_t *out2) {
    Packed pk;
    std::string msg;
    out2[0] = out2[1] = 0;
    const int rc = pack_problem(p, pk, msg, false);
    if (rc != WHMEC_OK || pk.n == 0) return rc;
    TileSchedule ts;
    plan_tiles(pk, ts);
    if (!ts.eligible) return 100;
    out2[0] = tile_table_bytes(pk, ts);
    out2[1] = tile_table_items(ts);
    return 0;
}
