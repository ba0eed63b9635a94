// Allele detection from the CIGAR alone (whmec_detect_alleles_cigar, DESIGN §4.14): the host preparation.
// cigar_alleles_plan.cpp normalizes the variants, applies the conflict filter, builds the allele targets, checks every alignment and
// cuts the alignments into chunks; cigar_alleles.cu (and the test-only emulation tests/emul/emul_cigar_alleles.cpp) runs a chunk.
#pragma once
#include <string>
#include <vector>

#include "../../include/whmec.h"
#include "cigar_alleles.h"
#include "hostpool.h"

namespace whmec {

// What one call hands to the chunk runner.
struct CaPlan {
    StagedVec<CaAln> alns;            // [n_alignments]
    std::vector<CaVar> vars;          // conflict-free variants and a sentinel
    std::vector<CaAllele> alleles;
    uint32_t first_bad = UMAX;        // the first alignment whose op loop reaches an unknown operation or has no CIGAR (UMAX: none)
    std::string bad_msg;              // what the reference raises there
    std::string err;                  // a refusal of the whole call (empty when none)
};

// Normalization (BiallelicVcfVariant / MultiallelicVcfVariant.normalized), detect_non_overlapping_variants, build_var_progress and
// the per-alignment checks (WHMEC_HOST_THREADS workers).
void ca_prepare(const whmec_realign_input &in, const whmec_query_qualities *q, CaPlan &plan);

struct CaChunk {
    uint32_t a0 = 0, a1 = 0;        // alignments [a0, a1)
    uint64_t op_lo = 0, op_hi = 0;  // their CIGAR operations
    uint64_t q_lo = 0, q_hi = 0;    // query bytes
    uint64_t qual_lo = 0, qual_hi = 0;
    uint64_t bytes = 0;             // device bytes of the chunk without its items
};

// Device bytes per item in a window: the item, its outcome, the compacted outcome and the compaction's scratch.
constexpr uint64_t CA_ITEM_BYTES = sizeof(CaItem) + 2 * sizeof(CaCall) + 1;
// Device bytes of a chunk's alignments, operations, bytes, counts and scan.
uint64_t ca_chunk_bytes(const CaChunk &c);
// Alignments cut, in order, into chunks whose ca_chunk_bytes stay within half the budget (a chunk has at least one alignment).
std::vector<CaChunk> ca_chunks(const CaPlan &plan, const whmec_realign_input &in, const whmec_query_qualities *q, uint64_t budget);
// Items per window of a chunk under `budget` (at least one).
uint64_t ca_window(const CaChunk &c, uint64_t budget);

// What the runner returns: the calls in order, the first alignment on which a handler raises (UMAX: none), the counters.
struct CaRun {
    std::vector<CaCall> calls;
    uint32_t raised = UMAX;
    const CaPlan *plan = nullptr;
    const whmec_realign_input *in = nullptr;
    const whmec_query_qualities *q = nullptr;
    uint64_t budget = 0;
    void *dev = nullptr;  // the runner's per-call state
    whmec_realign_stats st{};
};

// Implemented by cigar_alleles.cu and by the emulation: the device bytes a call may take (0 with msg on failure), one chunk's
// run (its items in windows of ca_window), and the release of the per-call state.
uint64_t ca_budget(int device, std::string &msg);
int ca_run_chunk(int device, CaRun &run, const CaChunk &c, std::string &msg);
void ca_close(CaRun &run);

}  // namespace whmec
