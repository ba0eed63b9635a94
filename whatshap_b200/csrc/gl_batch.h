// Many genotyping tables in one call (whmec_genotype_batch, DESIGN §4.9): the host plan of a GROUP of tables whose sub-tables
// (a single individual's chains, or a whole pedigree table) all advance by one column per launch, whatever their shapes.
// Plain C++ (used by genotype.cu and by the test-only emulation, tests/emul/emul_gl_batch.cpp).
#pragma once
#include <vector>

#include "gl_pack.h"

namespace whmec {

constexpr uint32_t GL_MAX_GRID_Y = 65535;  // steps one launch can carry (grid.y); a longer step is split into several launches

// One table of a group, as gl_batch_backward_kernel / gl_batch_forward_kernel see it: its GlView as offsets into the group's
// concatenated inputs, where its backward tables start in the group's store, and where its posterior accumulators start.
// The GlCol records keep the table's own act_off / beta_off / trans_off / q_off: they are relative to these offsets.
struct GlBatchTable {
    uint64_t cols;       // GlCol records
    uint64_t act;        // entries of eps / allele / ind
    uint64_t h2p;        // entries of h2p
    uint64_t trans, q;   // doubles
    uint64_t beta_base;  // doubles: B_k of column k sits at store + beta_base + cols[k].beta_off
    uint64_t acc_base;   // doubles: the posterior accumulators, [n_cols][n_ind * 3] from here
    uint32_t T, P, n_ind, n_cols;
};

struct GlBatchInputs {  // the group's concatenated inputs: device pointers in the kernels, host pointers in the emulation
    const GlCol *cols;
    const double *eps;
    const uint8_t *allele;
    const uint8_t *ind;
    const int8_t *h2p;
    const double *trans;
    const double *q;
};

WHMEC_HD GlView gl_batch_view(const GlBatchInputs &in, const GlBatchTable &t) {
    return GlView{in.cols + t.cols, in.eps + t.act, in.allele + t.act, in.ind + t.act, in.h2p + t.h2p, in.trans + t.trans, in.q + t.q, t.T, t.P, t.n_ind};
}

// The plan of one group.  One step list for all tables: backward launch s holds the s-th column from the right of every
// sub-table that still has a column to its left, forward launch s the s-th column from the left of every sub-table that has
// one.  Backward steps write into the store (cur_off absolute), forward steps into the F pool (cur_off / prev_off absolute);
// gl_scale_kernel reads the same GlStep records.  step_table[e] is the position in `tables` of step e's table.
struct GlBatchGroup {
    std::vector<uint32_t> members;     // the tables, as positions in the caller's list
    std::vector<GlBatchTable> tables;  // one per member
    std::vector<GlCol> cols;           // the concatenated inputs, uploaded once
    std::vector<double> eps, trans, q;
    std::vector<uint8_t> allele, ind;
    std::vector<int8_t> h2p;
    std::vector<GlStep> steps;
    std::vector<uint32_t> step_table;
    std::vector<uint32_t> bwd_begin, fwd_begin;  // launch s covers steps [begin[s], begin[s + 1])
    uint64_t store_doubles = 0;   // every member's backward tables (+ 1 spare)
    uint64_t f_pool_doubles = 0;  // two projection buffers per sub-table
    uint64_t acc_doubles = 0;     // every member's posterior accumulators
    uint32_t launches = 0;        // two per launch of the step list (the step kernel and gl_scale_kernel), splits at GL_MAX_GRID_Y included
};

// Doubles a table takes in a group: backward tables, two projection buffers per sub-table, and its inputs, accumulators, steps
// and descriptor (rounded up to doubles).  The group budget covers the sum over its members.
uint64_t gl_batch_cost(const Packed &pk, const GlPacked &g);

// Cuts the tables with cost[t] > 0 (in list order; cost 0: not in the batch) into consecutive groups whose costs add up to at
// most `budget` doubles.  A table whose cost alone exceeds the budget joins no group; it is listed in `alone`.
void gl_batch_groups(const std::vector<uint64_t> &cost, uint64_t budget, std::vector<std::vector<uint32_t>> &groups, std::vector<uint32_t> &alone);

// The plan of the group of tables `members` (positions in pks / gs; every one packed, with at least one column).
void gl_batch_plan(const std::vector<Packed> &pks, const std::vector<GlPacked> &gs, const std::vector<uint32_t> &members, GlBatchGroup &out);

}  // namespace whmec
