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
};
// WHMEC_ERR_UNSUPPORTED when a table has no cut that fits; `err` then states a budget that fits ("needs at least N bytes").
int gl_plan(const GlPacked &g, uint32_t T, uint64_t budget, std::vector<GlUnit> &units, std::string &err);

// Packs `p` (whose gl holds the genotype priors; gt and distrust are ignored) for the genotyping DP.
int gl_pack(const whmec_problem *p, Packed &pk, GlPacked &g, std::string &err);

// Divides a finished projection column by its largest entry (no-op for an all-zero column).
void gl_scale_host(double *v, uint64_t n);

// likelihoods[(ind * n + k) * 3 + g] = acc[(k * n_ind + ind) * 3 + g] / (total of column k)   (genotypedptable.cpp:438-442)
void gl_normalise(const double *acc, uint32_t n, uint32_t n_ind, double *likelihoods);

}  // namespace whmec
