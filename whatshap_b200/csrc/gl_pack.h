// Host packing of the forward-backward genotyping DP (see gl_device.h): per-column records, error
// probabilities, transition and allele-assignment probabilities.  Plain C++ (used by genotype.cu and by the
// test-only emulation).
#pragma once
#include <string>
#include <vector>

#include "gl_device.h"
#include "pack.h"

namespace whmec {

struct GlPacked {
    std::vector<GlCol> cols;
    std::vector<double> eps;          // aligned with Packed::act_allele / act_ind
    std::vector<double> trans, q;
    uint64_t beta_doubles = 0;        // sum over columns but the last of 2^f * T
    uint64_t max_proj = 1;            // largest projection column (doubles)
    GlView view(const Packed &pk) const {
        return GlView{cols.data(), eps.data(), pk.act_allele.data(), pk.act_ind.data(), pk.h2p.data(), trans.data(), q.data(), pk.T, pk.P, pk.n_ind};
    }
};

// Launch schedule of a group of tables (columns [lo, hi), whole tables): one launch advances EVERY table of the group
// by one column, so the launch count is 4 x (longest table) instead of 4 x (columns).  Shared by genotype.cu and the
// test-only emulation, which executes the same steps with the same buffer offsets.
struct GlStep {           // one column of one table inside a launch (grid.y)
    uint32_t k;           // column
    uint32_t cells_log2;  // a_k
    uint64_t cur_off;     // forward: F_k in the F pool; backward: B_{k-1} in the group's backward store (doubles)
    uint64_t prev_off;    // forward: F_{k-1} in the F pool (cleared after the step); backward: unused
    uint64_t n_scale;     // entries of the finished column at cur_off to rescale (0: none)
    uint64_t n_clear;     // forward: entries at prev_off to clear for the next column
};
struct GlSchedule {
    std::vector<GlStep> steps;
    std::vector<uint32_t> bwd_begin, fwd_begin;  // launch s covers steps [begin[s], begin[s + 1])
    uint64_t beta_base = 0, beta_doubles = 0;    // the group's slice of the backward tables
    uint64_t f_pool_doubles = 0;                 // two projection buffers per table
};
void gl_schedule(const GlPacked &g, uint32_t T, uint32_t lo, uint32_t hi, GlSchedule &out);

// Cuts the columns into groups of whole tables whose backward tables + two projection buffers per table stay within
// `budget` doubles: group q = columns [begin[q], begin[q + 1]).  False if a single table exceeds the budget.
bool gl_groups(const GlPacked &g, uint32_t T, uint64_t budget, std::vector<uint32_t> &begin);

// The same groups, except that a table which alone exceeds the budget becomes a group of its own with alone[q] = 1
// (alone[q] = 0 for the other groups).  Without such a table the groups are those of gl_groups.
void gl_groups_split(const GlPacked &g, uint32_t T, uint64_t budget, std::vector<uint32_t> &begin, std::vector<uint8_t> &alone);

// Memory-bounded forward-backward of one table, columns [lo, hi), whose backward tables do not fit (DESIGN §4.5).
// Segment s = columns [cuts[s], cuts[s + 1]).  All segments share an arena at the start of the backward store; behind it
// sit the checkpoints, one per segment but the last: the scaled backward table of the segment's last column.
// Pass A runs the backward steps of the whole table right to left, segment by segment; the step of a segment's first
// column writes into the checkpoint of the segment to its left.  Pass B runs left to right: every segment but the first
// (whose backward tables pass A left in the arena) first sweeps its backward steps again from its checkpoint (the last
// segment from B = 1), then runs its forward steps.  One launch per step; the projection buffers carry across segments.
// A continued segment of a table (gl_pack_segment) keeps beta_in as one more checkpoint, the last segment's, in place of B = 1.
struct GlSweep {             // one segment's part of pass A or pass B, in this order:
    uint64_t beta_base;      //   B_k of the segment's columns sits at store + cols[k].beta_off - beta_base
    uint64_t clear;          //   zero store[0, clear) (the backward steps accumulate)
    uint64_t copy_dst, copy_src, copy_n;  // copy store[copy_src, +copy_n) to store[copy_dst] (copy_n = 0: none)
    uint32_t bwd_begin, bwd_end;          // backward steps [bwd_begin, bwd_end), then
    uint32_t fwd_begin, fwd_end;          // forward steps [fwd_begin, fwd_end)
};
struct GlBounded {
    std::vector<GlStep> steps;           // offsets: backward into the store, forward into the F pool
    std::vector<GlSweep> sweeps;         // pass A, then pass B
    std::vector<uint32_t> cuts;          // cuts[0] = lo, cuts.back() = hi
    uint64_t arena_doubles = 0, ckpt_doubles = 0;  // the store: arena, then the checkpoints
    uint64_t f_pool_doubles = 0;         // the table's two projection buffers
    uint64_t tail_off = 0;               // a continued segment: the store offset of beta_in (its last checkpoint)
};
// Cuts with bounded.h's cut_column_segments applied to the mirrored column order, so that the first segment, the one
// swept backward only once, is as large as fits.  The store + F pool stay within `budget` doubles; false when no cut fits.
bool gl_bounded(const GlPacked &g, uint32_t T, uint32_t lo, uint32_t hi, uint64_t budget, GlBounded &out);

// Everything one genotyping call runs under `budget` doubles for backward tables, checkpoints and projection buffers:
// groups of whole tables (gl_groups_split; gl_schedule) and, for a table that alone exceeds the budget, its bounded plan.
struct GlUnit {
    bool bounded;
    GlSchedule sc;         // !bounded
    GlBounded bd;          // bounded
    uint64_t work_doubles; // store + F pool: backward tables (+ 1 spare) or arena + checkpoints, and projection buffers
    // A segment of a table (gl_pack_segment) takes its inputs here, in the unit's work buffer (store, then F pool), after the
    // buffer is cleared: alpha_in (T doubles) where the first forward step reads F_{lo-1}; beta_in (T doubles) where the
    // backward tables of the unit's last column are read from (a continued segment's last column is not `last`).
    uint64_t alpha_at, beta_at;
};
// WHMEC_ERR_UNSUPPORTED when a table has no cut that fits; `err` then states a budget that fits ("needs at least N bytes").
int gl_plan(const GlPacked &g, uint32_t T, uint64_t budget, std::vector<GlUnit> &units, std::string &err);

// Packs `p` (whose gl holds the genotype priors; gt and distrust are ignored) for the genotyping DP.
int gl_pack(const whmec_problem *p, Packed &pk, GlPacked &g, std::string &err);

// A SEGMENT of a pedigree table (DESIGN §4.5, whmec_genotype_segment_*): a run of whole chains packed as a problem of its own.
// `continues`: the segment does not start the table, so its column 0 is not `first` (it reads F_{-1} = alpha_in through its
// real transmission matrix).  `continued`: it does not end the table, so its last column is not `last` and owns a T-entry
// backward table, which holds beta_in.  WHMEC_ERR_UNSUPPORTED for T == 1 (chains are independent tables already).
int gl_pack_segment(const whmec_problem *p, bool continues, bool continued, Packed &pk, GlPacked &g, std::string &err);

// The transfer pass of a segment: one forward-only sweep of its columns for a batch of n_in input vectors at once
// (gl_transfer_cell), the rows of a batch sharing one scale per column.  F pool: two buffers of f_size * n_in doubles,
// laid out [u][2^f * T] (stride 2^f_k * T in column k).  A continued or continuing segment with T > GL_T_LOCAL runs T / n_in
// batches, each from its own inputs, and records every column's scale so that the rows of all batches can be put on one scale
// afterwards.  A segment that starts the table ignores its input: one batch of one row.
struct GlTransfer {
    std::vector<GlStep> steps;  // one per column, left to right; cur_off / prev_off into the F pool, n_scale = 2^f_k * T * n_in
    uint32_t n_in = 1, n_batches = 1;
    uint64_t f_pool_doubles = 0;
    uint64_t in_off = 0;        // where batch b's inputs go before its sweep: rows [u][T], e_{b * n_in + u} (continues only)
    uint64_t out_off = 0;       // where the sweep leaves the batch's rows of the matrix: [u][T] at the last column
};
void gl_transfer_plan(const GlPacked &g, uint32_t T, bool continues, GlTransfer &out);

// Rows of the transfer matrix from the batches of gl_transfer_plan: m[u * T + i] (u < n_in * n_batches, or all T rows equal
// to the one row of a segment that starts the table).  With several batches, col_max[b * n_cols + k] is the scale batch b's
// column k was divided by (its largest entry; 0: none).  The rows of batch b are multiplied by prod_k col_max[b][k] / (the largest
// such product), which gives every row one scale.  The products are kept as a long double mantissa and a binary exponent, so
// neither overflows and thousands of columns add no more than ~1e-15 relative error.
void gl_transfer_combine(const GlTransfer &tp, uint32_t T, const std::vector<double> &rows, const std::vector<double> &col_max, double *m);

// Divides a finished projection column by its largest entry (no-op for an all-zero column).
void gl_scale_host(double *v, uint64_t n);

// likelihoods[(ind * n + k) * 3 + g] = acc[(k * n_ind + ind) * 3 + g] / (total of column k)   (genotypedptable.cpp:438-442)
void gl_normalise(const double *acc, uint32_t n, uint32_t n_ind, double *likelihoods);

}  // namespace whmec
