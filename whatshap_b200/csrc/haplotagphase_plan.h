// Votes of `whatshap haplotagphase` (whmec_haplotagphase, DESIGN §4.16): the host plan.  haplotagphase_plan.cpp ranks each
// sample's phase sets, bins the entries of the counted reads by position, cuts whole positions of one sample into chunks and
// gathers each chunk's entries in read order; haplotagphase.cu (and the test-only emulation tests/emul/emul_haplotagphase.cpp)
// runs a chunk.
#pragma once
#include <string>
#include <vector>

#include "../../include/whmec.h"
#include "haplotagphase.h"

namespace whmec {

// Device bytes a chunk takes at most per entry (the entry, two key and two value buffers of each of the two sorts, the record,
// its gathered copy and a share of the sorts' scratch), per position (its key start, choice and two sort buffers) and per run.
constexpr uint64_t HP_ENTRY_BYTES = sizeof(HpEntry) + 2 * 8 + 2 * 4 + 2 * sizeof(HpRecord) + 2 * 8 + 2 * 4 + 16;
constexpr uint64_t HP_POS_BYTES = 4 + sizeof(HpChoice) + 2 * 4 + 2 * 4 + 8;
constexpr uint64_t HP_RUN_BYTES = 3 * 8;

// What one call hands to the chunk runner: the position tables, then per chunk its entries (vote form) or runs (runs form).
struct HpCall {
    HpTable host{};                  // the caller's tables
    uint64_t n_pos = 0;
    double gap = 0;
    int only_indels = 0;
    // the current chunk: table positions p0 .. p0 + n_cpos (vote form), or runs-form positions with their table index
    uint64_t p0 = 0;
    uint32_t n_cpos = 0;
    uint32_t ps_bits = 0;
    const HpEntry *entries = nullptr; // vote form, in read order
    uint32_t n_entries = 0;
    std::vector<uint32_t> pstart;     // vote form: [n_cpos + 1] into the sorted keys
    std::vector<uint64_t> tpos;       // runs form: [n_cpos] table index of each position
    std::vector<uint64_t> roff;       // runs form: [n_cpos + 1] into run_ps / run_h / run_score
    const int64_t *run_ps = nullptr, *run_h = nullptr, *run_score = nullptr;
    // its results
    std::vector<HpChoice> choice;     // [n_cpos]
    std::vector<uint32_t> order;      // vote form: the voted chunk positions by first entry
    std::vector<HpRecord> records;    // vote form: every position's phase sets, positions in order, each's sets by first entry
    uint64_t error = ~0ull;           // vote form: the least (entry ordinal << 2 | kind) the chunk found, ~0 for none
    void *dev = nullptr;              // the runner's per-call state
    whmec_haplotagphase_stats st{};
};

// Implemented by haplotagphase.cu and by the emulation: the device bytes a call may take (0 with msg on failure), one chunk's
// run in either form, and the release of the per-call state.
uint64_t hp_budget(int device, std::string &msg);
int hp_run_votes(int device, HpCall &call, std::string &msg);
int hp_run_runs(int device, HpCall &call, std::string &msg);
void hp_close(HpCall &call);

}  // namespace whmec
