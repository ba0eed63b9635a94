// Host planner of the column-kernel paths (whmec.cu, DESIGN §4.2): which sweep runs (column, batched or fused pedigree sweep),
// whether the back-pointers take the memory-bounded sweep and where its segments are cut, and the batched sweep's step lists.
// Plain C++ (used by whmec.cu and by the test-only emulation, which checks the plans on the CPU); whmec.cu allocates, uploads
// and launches what the plan lists.
#pragma once
#include <stdint.h>
#include <string>
#include <vector>

#include "common.h"
#include "pack.h"

namespace whmec {

// lanes per projection entry (log2): one thread per entry when the column has enough entries to fill
// the GPU, otherwise the 2^d candidates of an entry are spread over up to 32 lanes
#if defined(__CUDACC__)
__host__ __device__
#endif
inline uint32_t col_lane_bits(uint32_t log_entries, uint32_t d) {
    if (log_entries >= 14) return 0;
    const uint32_t want = 14 - log_entries;
    const uint32_t lc = d < want ? d : want;
    return lc < 5 ? lc : 5;
}

// One column step of one (chain, input) instance of the batched pedigree sweep (col_batched_kernel, col_multi_kernel).
struct PedStep {
    ColMeta cm;
    uint32_t nf;
    uint32_t slot;   // state slot of the instance (two value buffers per slot)
    uint32_t flags;  // bit 0: write back-pointers; bit 1: write transition minima for the next column;
                     // bit 2: the previous projection holds transition minima
    uint32_t rc_next;
};

// What the plan depends on besides the packed problem: the device and the environment switches (DESIGN §10).
struct ColPlanInput {
    uint64_t free_bytes = 0;     // free device memory (device_available_bytes)
    uint64_t hook = 0;           // WHMEC_COLUMN_ARENA_BUDGET in bytes, 0 = none
    bool fused = true;           // the fused trio sweep is allowed (WHMEC_PED_FUSED not 0)
    bool sequential = false;     // WHMEC_PED_SEQUENTIAL=1: no two-pass sweep for whole tables
    int segment = 0;             // 0 = whole table, 1 = first segment of a shared table, 2 = a continuing segment
    bool bounded_t1 = false;     // a single individual beyond the free HBM takes the memory-bounded sweep instead of a refusal
    uint32_t sms = 132;          // multiprocessors of the device
    uint32_t cluster = 0;        // WHMEC_PED_CLUSTER: 1, 2, 4 or 8 forces the fused sweep's cluster size; anything else: automatic
};

enum class ColPath { column, batched, fused, wide };  // wide: the column sweep of T = 1024 (DESIGN §4.7)

struct ColPlan {
    ColPath path = ColPath::column;  // batched and fused are the two-pass sweeps, wide sweeps column by column as `column`
    uint64_t max_ent = 1;            // largest column (entries): the size of each value buffer
    uint64_t slots = 0;              // batched sweep: value-buffer slots, (chain, unit vector) instances + one per chain
    uint64_t fixed_bytes = 0;        // device memory of the plan besides the back-pointers and the batch buffers
    bool ped_multi = false;          // batched sweep: pass 1 runs the multi-RHS kernel
    // memory-bounded sweep (back-pointers beyond the budget): segments share one arena, ColMeta::bp_off is rebased to the
    // segment's first column; the sweep leaves the last segment's back-pointers there, the backtrace sweeps the others
    bool bounded = false;
    bool over_hbm = false;           // refused: the back-pointers exceed the free HBM and the bounded sweep is not for this plan
    uint64_t budget_bytes = 0;       // bounded: the budget the segments were cut under
    std::vector<uint32_t> seg_col;   // column sweep: column cuts, segment s = columns [seg_col[s], seg_col[s + 1])
    std::vector<uint64_t> seg_ckpt;  // column sweep: word offset in the checkpoints of the values column seg_col[s] - 1 hands on (s >= 1)
    std::vector<uint32_t> seg_chain; // two-pass sweeps: chain cuts, segment s = chains [seg_chain[s], seg_chain[s + 1])
    uint64_t arena_words = 0, ckpt_words = 0;
    // batched sweep: steps[begin[st], begin[st + 1]) run in launch st of a pass, on grid[st] blocks
    std::vector<PedStep> steps;
    std::vector<uint32_t> clen;      // columns per chain
    std::vector<uint32_t> ped_begin[3], ped_grid[3];  // [0] pass 1 (per-input instances), [1] pass 2, [2] pass 1 multi-RHS
    std::vector<std::vector<uint32_t>> seg_begin, seg_grid;  // bounded: pass 2 of every segment (instead of ped_begin[1])
    uint32_t cluster = 1;            // fused sweep: CTAs per chain
    bool two_pass() const { return path == ColPath::batched || path == ColPath::fused; }
};

// Plans the column-kernel sweep of `pk` (packed with deltas) and rebases pk.cols[k].bp_off when the plan is bounded.
// WHMEC_ERR_UNSUPPORTED with a message when the plan cannot run: the table exceeds the free HBM (over_hbm), no segment fits
// ("needs at least N bytes"), or a table segment cannot run the two-pass sweep.
int col_plan(Packed &pk, const ColPlanInput &in, ColPlan &plan, std::string &msg);

}  // namespace whmec
