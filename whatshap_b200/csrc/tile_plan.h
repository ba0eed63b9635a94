// Host planner of the tile path (single individual, T == 1).
//
// Idea.  The projection column of the reference (projection_column_table[k],
// src/pedigreedptable.h:40-41) is an array over all bipartitions of the reads shared by two
// neighbouring columns.  A read that stays active for the next s columns is a bit that no
// reduction touches during those columns; so the array can be cut along such "global" bits into
// 2^g independent tiles of 2^s entries, each tile small enough to live in the shared memory of
// one SM, and a whole PANEL of consecutive columns can be swept tile-locally without touching
// HBM: only when a global read is about to end is the state written back (in the canonical
// layout of the reference's forward-projection index) and re-cut along a new set of bits.
// This is the same blocking that makes FFTs and bit-sliced scans cache-efficient.
//
// Everything here is plain C++ (used by tile.cu and by the test-only emulation).
#pragma once
#include <stdint.h>
#include <string>
#include <utility>
#include <vector>

#include "pack.h"

namespace whmec {

#ifndef WHMEC_TILE_SMAX   // overridden (small) only by the test-only emulation build to stress the planner
#define WHMEC_TILE_SMAX 14
#endif
constexpr uint32_t TILE_SMAX = WHMEC_TILE_SMAX;      // log2 entries of a tile's state buffer (2 x 64 KB of shared memory)
constexpr uint32_t TILE_MMAX = WHMEC_TILE_SMAX + 1;  // log2 cells a tile evaluates per column
constexpr uint32_t TILE_GMAX = 18;   // log2 tiles per panel (32 active reads = 14 local + 18 global)
constexpr uint32_t TILE_KINF = 1u << 30;
constexpr uint64_t TILE_SAFE_BOUND = 1ull << 28;  // every real cost must stay below this
constexpr uint32_t TILE_NARROW_LIMIT = 1u << 15;  // narrow panels: every value minus the tile's base, plus a cost, stays below this

struct TileCol {            // one column as seen by a tile (device + host)
    uint8_t l_in, n_new, d, l_out;
    uint8_t kind;           // 0 regular, 1 chain end (all reads end: global min with full Gray rank)
    uint8_t g;
    uint8_t pad0, pad1;
    uint32_t dropmask;      // over m = l_in + n_new local bits
    uint32_t K0, K12;       // min over homozygous assignments; K1 + K2 (mod 2^32)
    int32_t K2;
    uint32_t bp_width;      // 0,1,2,4,8,16 bits per entry
    uint64_t bp_off;        // 32-bit words into the arena; tile t owns words [bp_off + t*bp_tile_words, +bp_tile_words)
    uint32_t bp_tile_words; // ceil(2^l_out * bp_width / 32)
    uint32_t pad2;          // fast columns: bit 0 = back-pointer bits packed per thread (tile_packed_bit_index), else warp-ballot order
    uint32_t half;          // 1: column of a mirrored panel (only the tiles whose top tile-id bit is 0 are computed, see Panel::half)
    uint32_t km;            // mirrored panels: rank of the mirror candidate = rank ^ km (d bits; chain end: a bits), see tile_device.h
    uint32_t bp_tile_stride;  // words between the slices of consecutive tiles: bp_tile_words, or twice that when the mirror
                            // outputs' back-pointers differ from the tile's own (half && km != 0): [own | mirror]
    uint32_t gmask_out;     // canonical mask (over f_k bits) of the global reads after this column
    uint32_t lmask_col;     // canonical mask (over a_k bits) of the local reads of this column
    int32_t w_local[16];    // signed weight of local bit q:  +phred if allele 0, -phred if allele 1
    int32_t w_global[TILE_GMAX];  // same for the read behind tile-id bit b
    uint32_t gabove[16];    // per dropped local bit i: tile-id bits of global reads canonically above it
    uint8_t dpos[16];       // local positions of the dropped bits, ascending
};

struct Panel {
    uint32_t chain;
    uint32_t col_begin, col_end;   // [begin, end) global column indices
    uint32_t g, s_in, s_out;       // log2 tiles, log2 tile entries in / out
    uint32_t lmask_in, gmask_in;   // canonical masks over the input state's bits
    uint32_t lmask_out, gmask_out; // canonical masks over the output state's bits (unused if ends_chain)
    uint32_t ends_chain;           // last column is the chain end: no state is written
    uint32_t fresh;                // first panel of its chain: the input state is the single value 0
    uint32_t tile_begin;           // first work item (one tile of one panel) of this panel in the sweep's item order
    // State hand-off layout between consecutive panels of a chain.  0 = canonical (the reference's
    // forward-projection index).  1 = tile-major: the producer tile t writes its 2^s_out entries
    // contiguously at (t << s_out); possible when the consumer's local reads are the producer's
    // global reads plus the LOW j local bits of the producer (the steady state), so that every
    // consumer tile gathers one contiguous 2^j chunk from each producer tile.
    uint32_t in_layout, out_layout;
    uint32_t in_gA, in_j, in_sA;   // tile-major input: producer's global bits, chunk bits, producer's s_out
    uint32_t in_gold;              // number of consumer tile-id bits that come from the old state
    // Complement symmetry (single individual): cost(x) = cost(~x) in every column, hence S(f) = S(~f) for every projection:
    // tile t of a panel with g >= 1 global reads holds exactly the mirror image of tile ~t.  `half` = 1: only the 2^(g-1)
    // tiles whose top tile-id bit (the youngest global read) is 0 are computed; a consumer that needs an entry of an
    // uncomputed tile reads the complemented index of the mirror tile, the back-pointers of the mirror outputs are
    // derived in the same pass (tile_device.h).
    uint32_t half;
    uint32_t in_half;              // the producer of the input state was a mirrored panel
    uint32_t in_top;               // canonical layout: bit (over the input state's index) of the producer's top global read
    // Steady-state panel (the bulk of a coverage-capped ReadSet): at most 16 columns, in every one exactly one read ends
    // (local bit 0) and one starts, the tile keeps 2^13 or 2^14 entries, no homozygous assignment, thread-packed
    // back-pointers, one mirror mode.  The kernel sweeps such a panel with all per-column tables built once, in
    // parallel, and no per-column dispatch.  steady = 1 + LG (2^LG twin pairs per thread), 0 otherwise.
    uint32_t steady;
    // Narrow steady-state panel (2^14-entry tiles, not mirrored with km != 0): the kernel sweeps it on 16-bit halfword pairs
    // (tile_fast.h), values relative to base = (the tile's first input entry) - narrow_spread.  narrow_spread bounds how far
    // apart any two input entries of one tile are; with it, every value of the panel minus base stays below TILE_NARROW_LIMIT
    // (the planner's proof: DESIGN §4.1).
    uint32_t narrow, narrow_spread;
    // The previous panel of the chain (index into TileSchedule::panels; TILE_NO_PANEL for a fresh panel), whose output is this
    // panel's input, and its number of computed tiles: the kernel starts a tile of this panel once that many tiles of the
    // producer have signalled their write-back.
    uint32_t producer, producer_tiles;
    uint64_t in_off, out_off;      // 32-bit word offsets of the chain's state buffers
};
constexpr uint32_t TILE_NO_PANEL = 0xFFFFFFFFu;

// Narrow panels: largest value minus the tile's base after the first `ncol` columns (DESIGN §4.1): twice the input spread
// (base = first input entry - spread) plus, per column, the largest cell cost min(K2 + E, K1 - E) <= K12 / 2.
inline uint64_t narrow_panel_bound(uint32_t spread, const TileCol *cols, uint32_t ncol) {
    uint64_t b = 2ull * spread;
    for (uint32_t j = 0; j < ncol; ++j) b += cols[j].K12 / 2;
    return b;
}
inline uint32_t panel_tiles(const Panel &P) { return 1u << (P.g - P.half); }  // computed tiles (mirrored panel: half of 2^g)

struct TileSchedule {
    bool eligible = false;
    std::string why;                      // reason when not eligible
    StagedVec<TileCol> cols;              // [n] indexed by global column (uploaded as it is)
    // Round r = the r-th panel of every chain that has one.  panels[] is grouped round by round (chains ascending inside a
    // round) and its work items are numbered in that order, so a panel's producer always comes earlier; segments of a
    // memory-bounded sweep are cut at round boundaries.
    StagedVec<Panel> panels;              // (uploaded as it is)
    std::vector<uint32_t> round_begin;    // panels of round r: [round_begin[r], round_begin[r+1])
    std::vector<uint32_t> round_tiles;    // work items of round r
    uint64_t state_words = 0;             // total size of the per-chain state double buffers
    uint64_t bp_words = 0;
    uint64_t state_traffic_bytes = 0;     // bytes of state written + read through global memory
};

// Builds the schedule; `eligible == false` (with `why`) means the column kernel must be used.
void plan_tiles(const Packed &pk, TileSchedule &out);

// ---- several tables in one sweep (whmec_solve_batch) -------------------------------------------------------------------
// Chains of different single-individual tables are as independent as the chains of one table, so the schedules of several
// tables concatenate into one: chains, columns, panels, work items, state buffers and back-pointer words are renumbered
// globally.  Round r of the union is round r of every table that has one (tables in input order), so a panel's producer
// still comes earlier in the item order and segments can still be cut at round boundaries.
struct TileUnion {
    Packed pk;                          // what the sweep and the backtrace read of a packed problem: n, cols, chain_begin
    TileSchedule ts;
    std::vector<uint32_t> table_chain;  // [tables + 1] first chain of every table
    std::vector<uint32_t> table_col;    // [tables + 1] first column of every table
};
void merge_tile_tables(const std::vector<const Packed *> &pks, const std::vector<const TileSchedule *> &tss, TileUnion &out);

// Device bytes one table adds to a union (records, state buffers, back-pointers, path) and its work items.
uint64_t tile_table_bytes(const Packed &pk, const TileSchedule &ts);
uint64_t tile_table_items(const TileSchedule &ts);

// Cuts tables 0 .. n-1 into consecutive groups [first, last) whose bytes fit `budget` together (and whose `items` -- work items of a
// tile union, cost functions of a pedigree union: both are numbered in 32 bits -- stay below 2^31); a table that does not fit alone is listed in `alone` instead (it takes the single-table path,
// which knows the memory-bounded sweep).  One budget for all groups: groups are resident one after the other.
void cut_table_groups(const std::vector<uint64_t> &bytes, const std::vector<uint64_t> &items, uint64_t budget,
                      std::vector<std::pair<uint32_t, uint32_t>> &groups, std::vector<uint32_t> &alone);

}  // namespace whmec
