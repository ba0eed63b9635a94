// TEST-ONLY host emulation of a fused-trio group of whmec_solve_batch: the union of the tables' packed forms is the product's
// (csrc/batch.h: merge_column_tables), every chain of the union is swept by the host mirror of ped_fused_kernel (emul.cpp:
// fused_chain), the fold between the passes is the per-thread code of ped_fused_tables_prefix_kernel (ped_fused.h:
// pf_fold_table, one call per table), and every table is backtraced from the optimum of its own last chain.
#include "emul.cpp"

#include "../../whatshap_b200/csrc/batch.h"

// status[t]: WHMEC_OK, the packer's error code, or 100 (outside the fused shape: not part of the group).
// info2: tables in the group, chains of the union.
extern "C" int whemul_fused_batch_solve(const whmec_problem *const *problems, whmec_solution *const *sols, uint32_t n_tables, int *status,
                                        uint64_t *info2) {
    std::vector<Packed> packed(n_tables);
    std::vector<uint32_t> members;
    std::vector<const Packed *> pks;
    for (uint32_t t = 0; t < n_tables; ++t) {
        std::string msg;
        Packed &pk = packed[t];
        status[t] = pack_problem(problems[t], pk, msg);
        if (status[t] != WHMEC_OK) continue;
        bool ok = pk.n > 0 && pk.T == PF_T && pk.safe31;
        for (uint32_t k = 0; k < pk.n && ok; ++k) ok = pf_column_ok(pk.cols[k], pk.fn_group.data() + pk.cols[k].grp_off);
        if (!ok) {
            status[t] = 100;
            continue;
        }
        members.push_back(t);
        pks.push_back(&pk);
    }
    PackedUnion un;
    merge_column_tables(pks, un);
    const Packed &pk = un.pk;
    const uint32_t B = (uint32_t)members.size(), C = un.table_chain[B], T = PF_T;
    std::vector<uint32_t> arena(pk.bp_words + 1, 0), rows((size_t)C * T), in_vecs((size_t)C * T, 0xDEADBEEF), out_vecs((size_t)C * T);
    for (uint32_t c = 0; c < C; ++c) fused_chain(pk, c, nullptr, true, arena, &rows[(size_t)c * T]);
    for (uint32_t t = 0; t < B; ++t)  // ped_fused_tables_prefix_kernel, thread t
        pf_fold_table(&rows[(size_t)un.table_chain[t] * T], un.table_chain[t + 1] - un.table_chain[t], &in_vecs[(size_t)un.table_chain[t] * T]);
    for (uint32_t c = 0; c < C; ++c) fused_chain(pk, c, &in_vecs[(size_t)c * T], false, arena, &out_vecs[(size_t)c * T]);
    std::vector<uint32_t> pidx(pk.n), ptv(pk.n);
    BtView bv{pk.cols.data(), arena.data(), T, pk.tb};
    for (uint32_t i = 0; i < B; ++i) {
        const uint32_t k0 = un.table_col[i], k1 = un.table_col[i + 1], c_last = un.table_chain[i + 1] - 1;
        if (un.table_end[c_last] != i + 1) return 1;
        uint32_t cost, x, tv, ptvv;
        pick_optimum(pk.cols[k1 - 1], &out_vecs[(size_t)c_last * T], arena.data(), T, pk.tb, &cost, &x, &tv, &ptvv);
        backtrace_range(bv, k1 - 1, k0, x, tv, ptvv, pidx.data(), ptv.data());
        sols[members[i]]->cost = cost;
        std::string msg;
        status[members[i]] = build_outputs(*pks[i], pidx.data() + k0, ptv.data() + k0, sols[members[i]], msg);
    }
    if (info2) {
        info2[0] = B;
        info2[1] = C;
    }
    return 0;
}

// The fold of ped_fused_tables_prefix_kernel over given rows: thread t folds the chains [table_chain[t], table_chain[t + 1]).
extern "C" void whemul_fold_tables(const uint32_t *rows, const uint32_t *table_chain, uint32_t n_tables, uint32_t *in_vecs) {
    for (uint32_t t = 0; t < n_tables; ++t)
        if (table_chain[t + 1] > table_chain[t])
            pf_fold_table(rows + (size_t)table_chain[t] * PF_T, table_chain[t + 1] - table_chain[t], in_vecs + (size_t)table_chain[t] * PF_T);
}
