// Read assignment of `whatshap haplotag` (whmec_haplotag, DESIGN §4.15): the host plan.  haplotag_plan.cpp walks each sample's
// reads into groups, ranks the blocks, cuts the groups into chunks and gathers each chunk's entries in visit order; haplotag.cu
// (and the test-only emulation tests/emul/emul_haplotag.cpp) runs a chunk.
#pragma once
#include <string>
#include <vector>

#include "../../include/whmec.h"
#include "haplotag.h"

namespace whmec {

// Device bytes a chunk takes at most per entry (the entry, its count and offset) and per possible match (two key buffers, two
// ordinal buffers and a share of the sort's scratch), and per group (its entry start and its choice).
constexpr uint64_t HT_ENTRY_BYTES = sizeof(HtEntry) + 8;
constexpr uint64_t HT_MATCH_BYTES = 2 * 8 + 2 * 4 + 8;
constexpr uint64_t HT_GROUP_BYTES = 4 + sizeof(HtChoice);

// What one call hands to the chunk runner: the phase tables, then per chunk its entries and group starts.
struct HtCall {
    HtTable host{};                  // the tables in host memory (soff, pos, aoff, allele are the caller's)
    uint32_t n_samples = 0;
    uint64_t n_pos = 0, n_alleles = 0;
    std::vector<uint32_t> rank;      // [n_pos]
    int64_t ploidy = 0;
    uint32_t hap_bits = 0, rank_bits = 0;
    // the current chunk
    uint64_t e0 = 0;                 // the call-wide ordinal of its first entry
    std::vector<HtEntry> entries;    // in visit order
    std::vector<uint32_t> gstart;    // [groups + 1] into entries
    // its results
    std::vector<HtChoice> choice;    // [groups]
    uint64_t error = ~0ull;          // the least (visit key << 2 | kind) the chunk found, ~0 for none
    void *dev = nullptr;             // the runner's per-call state
    whmec_haplotag_stats st{};
};

// Implemented by haplotag.cu and by the emulation: the device bytes a call may take (0 with msg on failure), one chunk's run
// (choice and error filled), and the release of the per-call state.
uint64_t ht_budget(int device, std::string &msg);
int ht_run_chunk(int device, HtCall &call, std::string &msg);
void ht_close(HtCall &call);

}  // namespace whmec
