// Several pedigree tables in one sweep of the column-kernel paths (whmec_solve_batch, fused-trio group).
//
// Pedigree chains are coupled only through the fold of their transfer matrices, and a table's first column ignores its input
// (pedigreedptable.cpp:275-278), so the fold can restart at a table boundary: the packed forms of several tables concatenate
// into one (columns, cost functions, back-pointer words and chains renumbered globally) that the fused sweep takes as it
// takes one table, as long as the fold, the backtrace's entries and the optimum are formed per table.  Plain C++ (used by
// whmec.cu and by the test-only emulation).
#pragma once
#include <algorithm>
#include <cstring>
#include <vector>

#include "pack.h"

namespace whmec {

struct PackedUnion {
    Packed pk;                          // what the sweep and the backtrace read: cols, cost functions, chain_begin, T, tb, bp_words
    std::vector<uint32_t> table_chain;  // [tables + 1] first chain of every table
    std::vector<uint32_t> table_col;    // [tables + 1] first column of every table
    std::vector<uint32_t> table_end;    // [chains] t + 1 when the chain is the last one of table t, else 0
};

// Device bytes one pedigree table adds to a union, and its cost functions (their offsets are 32-bit).
inline uint64_t column_table_bytes(const Packed &pk) {
    return pk.bp_words * 4 + (pk.fn_delta.size() + pk.fn_c0.size() + pk.fn_group.size()) * 4 + (uint64_t)pk.n * (sizeof(ColMeta) + 8) +
           pk.chain_begin.size() * 64;
}
inline uint64_t column_table_functions(const Packed &pk) { return pk.fn_c0.size() + pk.fn_group.size(); }

// All tables have the same T (the caller groups by pedigree shape).
inline void merge_column_tables(const std::vector<const Packed *> &pks, PackedUnion &out) {
    const size_t B = pks.size();
    out = PackedUnion();
    Packed &pk = out.pk;
    out.table_chain.assign(B + 1, 0);
    out.table_col.assign(B + 1, 0);
    std::vector<uint64_t> fn_base(B + 1, 0), grp_base(B + 1, 0), bp_base(B + 1, 0);
    pk.safe31 = pk.nowrap = true;
    for (size_t t = 0; t < B; ++t) {
        const Packed &q = *pks[t];
        out.table_chain[t + 1] = out.table_chain[t] + (uint32_t)q.chain_begin.size() - 1;
        out.table_col[t + 1] = out.table_col[t] + q.n;
        fn_base[t + 1] = fn_base[t] + q.fn_c0.size();
        grp_base[t + 1] = grp_base[t] + q.fn_group.size();
        bp_base[t + 1] = bp_base[t] + q.bp_words;
        pk.safe31 = pk.safe31 && q.safe31;
        pk.nowrap = pk.nowrap && q.nowrap;
        pk.max_d = std::max(pk.max_d, q.max_d);
        pk.n_reads += q.n_reads;
    }
    if (B) {
        pk.n_ind = pks[0]->n_ind;
        pk.n_trios = pks[0]->n_trios;
        pk.T = pks[0]->T;
        pk.tb = pks[0]->tb;
        pk.P = pks[0]->P;
    }
    pk.n = out.table_col[B];
    pk.bp_words = bp_base[B];
    pk.cols.resize(pk.n);
    pk.fn_c0.resize(fn_base[B]);
    pk.fn_delta.resize(fn_base[B] * FN_STRIDE);
    pk.fn_group.resize(grp_base[B]);
    pk.chain_begin.resize((size_t)out.table_chain[B] + 1);
    out.table_end.assign(out.table_chain[B], 0);
    for (size_t t = 0; t < B; ++t) {
        const Packed &q = *pks[t];
        const uint32_t k0 = out.table_col[t];
        for (uint32_t k = 0; k < q.n; ++k) {
            ColMeta &m = pk.cols[k0 + k];
            m = q.cols[k];
            m.bp_off += bp_base[t];
            m.fn_off += (uint32_t)fn_base[t];
            m.grp_off += (uint32_t)grp_base[t];
        }
        if (!q.fn_c0.empty()) std::memcpy(&pk.fn_c0[fn_base[t]], q.fn_c0.data(), q.fn_c0.size() * 4);
        if (!q.fn_delta.empty()) std::memcpy(&pk.fn_delta[fn_base[t] * FN_STRIDE], q.fn_delta.data(), q.fn_delta.size() * 4);
        if (!q.fn_group.empty()) std::memcpy(&pk.fn_group[grp_base[t]], q.fn_group.data(), q.fn_group.size() * 4);
        for (uint32_t c = out.table_chain[t]; c < out.table_chain[t + 1]; ++c) pk.chain_begin[c] = k0 + q.chain_begin[c - out.table_chain[t]];
        if (out.table_chain[t + 1] > out.table_chain[t]) out.table_end[out.table_chain[t + 1] - 1] = (uint32_t)t + 1;
    }
    pk.chain_begin[out.table_chain[B]] = pk.n;
}

}  // namespace whmec
