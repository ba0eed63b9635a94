// K-mer pair counts of `whatshap learn` (whmec_learn, DESIGN §4.13): the host plan.  learn_plan.cpp walks the CIGARs into runs,
// sets the floors, turns the variant windows into output intervals and cuts the columns into chunks; learn.cu (and the test-only
// emulation tests/emul/emul_learn.cpp) runs a chunk.
#pragma once
#include <string>
#include <vector>

#include "../../include/whmec.h"
#include "hostpool.h"
#include "learn.h"

namespace whmec {

// pop_column over the columns lo..hi in order, from variant offset `off`: appends the columns it outputs to iv as sorted,
// disjoint intervals [iv[2i], iv[2i + 1]] and returns the offset after hi.  The windows are those of caller.cpp in 64-bit
// arithmetic; with one variant left there is no next one.
uint32_t ln_intervals(const int32_t *pos, const int32_t *len, uint32_t n, uint32_t off, int64_t lo, int64_t hi, int64_t window,
                      int64_t k, std::vector<int64_t> &iv);

// One chunk: columns [lo, hi], the reads' parts entries [e0, e1) of the call's entry list, n_keys keys (32-bit when wide is false).
struct LnChunk {
    int64_t lo = 0, hi = 0;
    uint32_t e0 = 0, e1 = 0;
    uint64_t n_keys = 0;
    bool wide = false;
};

// Bytes of device memory one key of a chunk takes at most: both sort buffers, the runs, the counts, the flagged and the selected
// rows (64), and its share of the chunk's entries and warp list (28 bytes per entry; an entry has at least one key).
constexpr uint64_t LN_KEY_BYTES = 96;

// What one call hands to the chunk runner.
struct LnCall {
    uint32_t k = 0;
    const uint8_t *query = nullptr;   // the caller's query bytes
    uint64_t query_bytes = 0;
    const LnRead *reads = nullptr;
    uint32_t n_reads = 0;
    const LnOp *ops = nullptr;
    uint64_t n_ops = 0;
    std::vector<uint8_t> code;        // LnRef of the call's columns
    std::vector<uint32_t> base, mask;
    int64_t b0 = 0;
    std::vector<int64_t> iv;          // output intervals
    std::vector<LnEntry> entries;     // every chunk's entries, chunk by chunk
    std::vector<int32_t> rows;        // [n][4], appended chunk by chunk
    void *dev = nullptr;              // the runner's per-call state
    whmec_learn_stats st{};
};

// Columns [lo, hi] cut into chunks of at most cap keys each (a chunk has at least one column), with the entries of each; reads
// are the call's reads with their runs.
std::vector<LnChunk> ln_chunks(LnCall &call, int64_t lo, int64_t hi, uint64_t cap);

// Implemented by learn.cu and by the emulation: the device bytes a call may take (0 with msg on failure), one chunk's run (its
// rows appended to call.rows), and the release of the per-call state.
uint64_t ln_budget(int device, std::string &msg);
int ln_run_chunk(int device, LnCall &call, const LnChunk &c, std::string &msg);
void ln_close(LnCall &call);

}  // namespace whmec
