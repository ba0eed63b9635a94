// Allele detection by re-alignment (whmec_realign, DESIGN §4.11; k-mer mode whmec_realign_kmerald, §4.12): the host plan.
// realign_plan.cpp walks the CIGARs into items and jobs and cuts them into chunks; realign.cu (and the test-only emulation
// tests/emul/emul_realign.cpp) runs a chunk.
#pragma once
#include <string>
#include <vector>

#include "../../include/whmec.h"
#include "hostpool.h"
#include "kmerald.h"
#include "realign.h"

namespace whmec {

// The items of every alignment in alignment order (each alignment's items in the order the reference yields them), and their
// jobs.  err: the reference's failure on the first failing alignment (empty when none).
struct RaPlan {
    StagedVec<RaItem> items;
    StagedVec<RaJob> jobs;
    std::vector<uint64_t> item_off;  // [n_alignments + 1]
    uint64_t cells = 0;
    std::string err;
};

// The walk of one alignment (_iterate_cigar + realign's window and allele steps) appended to `items` and `jobs` (jobs' item
// fields count from items.size() on entry).  Returns false with the reference's failure in `err`.  With `km` (k-mer mode) the
// window is km->window instead of the overhang, the jobs are allele 0 and the variant's alternative_allele (allele 1, always;
// the restricted genotypes are ignored), and a variant without alternative_allele fails.
bool ra_walk_alignment(const whmec_realign_input &in, uint32_t a, std::vector<RaItem> &items, std::vector<RaJob> &jobs, std::string &err,
                       const whmec_kmerald_params *km = nullptr);
// All alignments on the host workers.
void ra_plan(const whmec_realign_input &in, RaPlan &plan, const whmec_kmerald_params *km = nullptr);

// A job's scratch field as the walk leaves it: RA_NO_SCRATCH for a one-thread job, else the bytes of its warp's work area
// (unit cost: one byte per text column for the hand-over between 32-word groups; affine: three float rows over the query).
uint64_t ra_job_need(uint64_t q_len, uint64_t target_len, int affine);
// The same for a k-mer job: RA_NO_SCRATCH when both strings have at most KA_SHORT bytes, else ka_scratch_bytes.
uint64_t ka_job_need(uint64_t q_len, uint64_t target_len);

struct RaChunk {
    uint32_t item0 = 0, item1 = 0;  // items [item0, item1) and their jobs [job0, job1)
    uint32_t job0 = 0, job1 = 0;
    uint64_t q_lo = 0, q_hi = 0;    // query bytes the items read
    int64_t r_lo = 0, r_hi = 0;     // reference bytes
    uint64_t scratch = 0;           // bytes of the warp jobs' work areas
    uint64_t bytes = 0;             // device bytes of the chunk
};

// Device bytes a chunk takes: descriptors, outputs, query and reference slices and scratch.
uint64_t ra_chunk_bytes(const RaChunk &c);
// Items cut, in order, into chunks of at most `budget` bytes (a chunk has at least one item).  Replaces the warp jobs' needs
// (ra_job_need) by their scratch offsets relative to their chunk.
std::vector<RaChunk> ra_chunks(const RaItem *items, uint32_t n_items, RaJob *jobs, uint64_t budget);

// What one call hands to the chunk runner.
struct RaCall {
    RaBufs host;                    // the caller's bytes (q0 = r0 = 0)
    uint64_t n_alleles = 0;         // allele slots (al_off has n_alleles + 1 entries)
    uint32_t n_variants = 0;
    uint64_t ref_len = 0;
    RaParams params{};
    bool decide = true;             // false: distances only (whmec_edit_distance_batch, whmec_kmer_align_batch)
    bool kmerald = false;           // k-mer mode: kparams, float distances in kdist
    KaParams kparams{};             // the caller's costs table (host pointers)
    float *kdist = nullptr;         // [jobs], k-mer mode without decide
    const RaItem *items = nullptr;
    const RaJob *jobs = nullptr;
    int64_t *dist = nullptr;        // [jobs], unit and affine mode without decide
    uint8_t *status = nullptr;      // [jobs]: 1 = distance beyond int64
    int32_t *call = nullptr;        // [items]: position of the called allele among the item's jobs, -1: none
    int64_t *quality = nullptr;     // [items]
    void *dev = nullptr;            // the runner's per-call state
    whmec_realign_stats st{};
};

// Implemented by realign.cu and by the emulation: the device bytes a chunk may take (0 with msg on failure), one chunk's run,
// and the release of the per-call state.
uint64_t ra_budget(int device, std::string &msg);
void install_pinned_staging();  // whmec.cu
int ra_run_chunk(int device, RaCall &call, const RaChunk &c, std::string &msg);
void ra_close(RaCall &call);

}  // namespace whmec
