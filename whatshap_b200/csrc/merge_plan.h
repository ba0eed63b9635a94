// Read merging of `whatshap phase --merge-reads` (whmec_merge_reads, DESIGN §4.17): the host plan.  merge_plan.cpp validates
// a set, finds each read's last partner and the pair prefix sums, cuts the pairs and the merged reads into chunks, runs the
// removal loop when not-blue edges can exist and lays out the output; merge.cu (and the test-only emulation
// tests/emul/emul_merge.cpp) runs the set's device work.
#pragma once
#include <string>
#include <vector>

#include "../../include/whmec.h"
#include "merge.h"

namespace whmec {

// Device bytes per read while its set is resident (begin, read and word offsets, pair start, parent), per packed word, per pair
// of a chunk (its flags and m - mm) and per entry of an accumulation chunk (the entry, two key and two value buffers, the run
// head, its scan, the run start, the run and a share of the sort's scratch).
constexpr uint64_t MG_READ_BYTES = 8 + 8 + 8 + 8 + 4;
constexpr uint64_t MG_WORD_BYTES = 8;
constexpr uint64_t MG_PAIR_BYTES = 1 + 8;
constexpr uint64_t MG_ENTRY_BYTES = sizeof(MgEntry) + 2 * 8 + 2 * 4 + 4 + 4 + 4 + sizeof(MgRun) + 16;

// What the plan hands to the runner: one set's resident arrays, then per chunk its pairs or its gathered entries.
struct MgCall {
    uint32_t n_reads = 0;
    uint64_t n_entries = 0;
    std::vector<uint64_t> roff;    // [n_reads + 1] set-local entry offsets
    std::vector<int64_t> begin;    // [n_reads]
    std::vector<uint64_t> woff;    // [n_reads + 1] packed words
    std::vector<uint64_t> pstart;  // [n_reads + 1] pair prefix sums
    const uint8_t *allele = nullptr;  // the set's alleles
    int64_t thr_diff = 0, thr_neg_diff = 0;
    double max_error_rate = 0;
    bool host_edges = false;       // not-blue edges can exist: the pairs' flags come back, no hooking on the device
    // the current pair chunk [p0, p1) and, with host_edges, its flags and m - mm
    uint64_t p0 = 0, p1 = 0;
    std::vector<uint8_t> flag;
    std::vector<int64_t> diff;
    uint64_t blue = 0;             // blue edges the device hooked (without host_edges)
    std::vector<uint32_t> parent;  // [n_reads] the roots, after mg_roots
    // the current accumulation chunk: entries of whole components, and its runs
    std::vector<MgEntry> entries;
    uint32_t n_comp = 0;
    int32_t pmin = 0;
    uint32_t pos_bits = 0;
    std::vector<MgRun> runs;
    void *dev = nullptr;           // the runner's per-call state
    whmec_merge_stats st{};
};

// Implemented by merge.cu and by the emulation: the device bytes a call may take (0 with msg on failure); the set's upload, bit
// packing and parent initialisation; one pair chunk; the roots of the hooked parents; one accumulation chunk; the release of
// the per-call state.
uint64_t mg_budget(int device, std::string &msg);
int mg_open_set(int device, MgCall &call, std::string &msg);
int mg_run_pairs(int device, MgCall &call, std::string &msg);
int mg_roots(int device, MgCall &call, std::string &msg);
int mg_run_accumulate(int device, MgCall &call, std::string &msg);
void mg_close(MgCall &call);

}  // namespace whmec
