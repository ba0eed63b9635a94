/*
 * whmec.h — C ABI of the CUDA (sm_90a) weighted-MEC / PedMEC dynamic program.
 *
 * This is the drop-in boundary for ONE hot path of WhatsHap: the PedigreeDPTable
 * column sweep.  The reference exposes that path as a C++ class bound through
 * Cython; there is no C ABI in the reference, so every entry point below names
 * the reference interface it replaces (paths relative to the whatshap source
 * tree):
 *
 *   whmec_solve            <- PedigreeDPTable::PedigreeDPTable  src/pedigreedptable.cpp:15-37
 *                             (ctor runs compute_table :84-174) + get_super_reads :344-388
 *                             + get_optimal_partitioning :391-406 + get_optimal_score :338-341,
 *                             bound at whatshap/cpp.pxd:86-90 / whatshap/core.pyx:364-416
 *   whmec_plan_*           <- same path, split into upload / forward sweep / backtrace so that
 *                             a caller (bench.py) can keep the packed ReadSet resident in HBM
 *   whmec_read_sort_key    <- ReadSet::read_comparator_t tie-break hash  src/readset.h:39-81
 *   whmec_compute_genotypes <- compute_genotypes  src/genotyper.cpp:12-54 (priors for the genotyping DP)
 *   whmec_genotype         <- GenotypeDPTable::GenotypeDPTable  src/genotypedptable.cpp:17-48 (ctor runs the
 *                             backward and the forward pass :118-215) + get_genotype_likelihoods :445-451,
 *                             bound at whatshap/core.pyx:581-600  (sibling DP, SURVEY.md 8(f) rank 4)
 *
 * Plain pointers and sizes only.  All input pointers are caller-owned host
 * memory, read-only, and need to stay valid only for the duration of the call.
 * Output arrays are caller-allocated.  No global mutable state; calls are
 * re-entrant; CUDA work is issued on a stream private to the call/plan.
 */
#ifndef WHMEC_H
#define WHMEC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define WHMEC_ABI_VERSION 2

/* return codes */
#define WHMEC_OK 0
#define WHMEC_ERR_MENDELIAN 1   /* "Error: Mendelian conflict"   (pedigreedptable.cpp:301-303) */
#define WHMEC_ERR_INPUT 2       /* unsorted reads / malformed arrays (columniterator.cpp:29,32) */
#define WHMEC_ERR_CUDA 3        /* CUDA runtime failure, message in err */
#define WHMEC_ERR_UNSUPPORTED 4 /* > 32 active reads (graycodes.cpp:12), cost range, HBM budget */

/* allele codes in ent_allele (src/entry.h:8) */
#define WHMEC_ALLELE_REF 0
#define WHMEC_ALLELE_ALT 1
#define WHMEC_ALLELE_BLANK 2
#define WHMEC_ALLELE_EQUAL_SCORES 3 /* only ever produced, in sr_allele */

/* genotype code meaning "no diploid biallelic genotype" (never matches an assignment) */
#define WHMEC_GT_OTHER 255

/*
 * One DP instance = one (chromosome x family) call of the reference constructor.
 *
 * Reads are given in final ReadSet order (sorted by first position); that order
 * defines the bit position of a read inside a column's bipartition index
 * (src/columniterator.cpp:91-139).  Entries are CSR over reads; ent_col is the
 * COLUMN INDEX (0..n_cols-1) of the entry's position and must be strictly
 * increasing inside a read.  A read is active in columns [first, last]; columns in
 * that span without an entry are BLANK (columniterator.cpp:131).
 */
typedef struct whmec_problem {
    uint32_t n_cols;
    const uint32_t *positions;   /* [n_cols] genomic positions (only echoed into results) */
    uint32_t n_reads;
    const uint64_t *read_off;    /* [n_reads+1] */
    const uint32_t *ent_col;     /* [nnz] */
    const uint8_t *ent_allele;   /* [nnz] 0/1/2 */
    const uint32_t *ent_phred;   /* [nnz] */
    const uint32_t *read_ind;    /* [n_reads] pedigree INDEX of the read's sample */
    const uint32_t *recombcost;  /* [n_cols] */
    uint32_t n_ind;
    uint32_t n_trios;
    const uint32_t *trios;       /* [3*n_trios] (father, mother, child) indices; trio r owns tv bits 2r,2r+1 */
    uint32_t distrust;           /* distrust_genotypes */
    const uint8_t *gt;           /* [n_ind*n_cols] canonical genotype index 0/1/2 or WHMEC_GT_OTHER */
    const double *gl;            /* [n_ind*n_cols*3] phred GLs (0/0,0/1,1/1); required iff distrust */
} whmec_problem;

typedef struct whmec_solution {
    uint32_t cost;               /* get_optimal_score() */
    uint32_t *path_index;        /* [n_cols] optimal bipartition index per column (index_path[k].index) */
    uint32_t *path_tv;           /* [n_cols] transmission value per column (index_path[k].inheritance_value) */
    uint8_t *partition;          /* [n_reads] get_optimal_partitioning() AFTER core.pyx:414 mapping (0/1) */
    uint8_t *sr_allele;          /* [n_ind][2][n_cols] super-read alleles in {0,1,3} */
    uint32_t *sr_quality;        /* [n_ind][n_cols] super-read quality */
} whmec_solution;

/* Work/traffic accounting of one solve; all byte counts follow SURVEY.md §8(d). */
typedef struct whmec_stats {
    uint64_t cells;              /* sum_k 2^{a_k} * T */
    uint64_t algorithmic_bytes;  /* sum_k T*(4*2^{bw_k} + (8 + 4*[T>1])*2^{f_k}) */
    uint64_t backptr_bytes;      /* bytes of packed back-pointers actually stored in HBM */
    uint64_t state_bytes;        /* bytes of projection state written+read to global memory */
    uint32_t kernel_launches;    /* CUDA kernels launched by the last forward sweep */
    uint32_t n_chains;           /* DP-independent column chains found (T==1) */
    uint32_t max_active;         /* max_k a_k */
    uint32_t transmissions;      /* T */
    float sweep_ms;              /* device time of the last forward sweep (CUDA events) */
    float h2d_ms, d2h_ms;        /* device-timed copies of the last solve */
    uint64_t h2d_bytes, d2h_bytes;
    uint32_t path_kind;          /* 1 = tile kernel, 2 = column kernel, 3 = batched pedigree sweep, 4 = genotyping (forward-backward) */
    uint32_t reserved;
} whmec_stats;

typedef struct whmec_plan whmec_plan;

/* Library / device introspection (no GPU needed for the first two). */
int whmec_abi_version(void);
const char *whmec_build_info(void);
int whmec_device_count(void);

/* Pack the problem on the host, upload it to `device`, allocate state and back-pointer
 * storage.  Host-detectable errors (Mendelian conflict, unsorted input) are reported here. */
int whmec_plan_create(const whmec_problem *p, int device, whmec_plan **out, char *err, size_t errlen);
/* Enqueue the forward sweep on the plan's stream and wait for it; may be called repeatedly
 * (each call recomputes everything from the resident inputs). */
int whmec_plan_sweep(whmec_plan *plan, char *err, size_t errlen);
/* Download back-pointers / optimum, run the backtrace and the super-read pass. */
int whmec_plan_finish(whmec_plan *plan, whmec_solution *s, char *err, size_t errlen);
int whmec_plan_stats(const whmec_plan *plan, whmec_stats *st);
void whmec_plan_destroy(whmec_plan *plan);

/* One-shot: create + sweep + finish + destroy, host buffers in, host buffers out. */
int whmec_solve(const whmec_problem *p, whmec_solution *s, int device, whmec_stats *st_or_null,
                char *err, size_t errlen);

/* ---- Genotype likelihoods by the forward-backward algorithm (the reference's GenotypeDPTable) ----------
 * Same inputs as whmec_solve, read differently where the reference does: p->gl holds, per individual and
 * column, the PRIOR probabilities of the genotypes 0/0, 0/1, 1/1 (required; the reference asserts on missing
 * ones, src/transitionprobabilitycomputer.cpp:66), recombcost[k] is the phred-scaled recombination
 * probability between columns k-1 and k, phred scores are error probabilities 10^(-q/10) (0 -> 0.9999,
 * src/genotypecolumncostcomputer.cpp:26-33); p->gt and p->distrust are ignored.  Every read must cover at
 * least two columns (the reference asserts, src/backwardcolumniterator.cpp:41): WHMEC_ERR_INPUT otherwise.
 * likelihoods (caller-allocated, [n_ind][n_cols][3] doubles) receives get_genotype_likelihoods(individual, column)
 * for every individual (pedigree index order) and column.  Floating point: the reference computes in 80-bit long
 * double with running-sum scaling, the device in double with max scaling; the normalised likelihoods agree to
 * ~1e-13 (the reference's own tests compare with 1e-9, whatshap/testhelpers.py:11-15).  st->backptr_bytes reports
 * the bytes of backward tables kept in HBM, st->sweep_ms the device time of both passes. */
int whmec_genotype(const whmec_problem *p, double *likelihoods, int device, whmec_stats *st_or_null, char *err, size_t errlen);

/* Per-column genotype priors of one sample's reads, the step `whatshap genotype` runs before the DP above
 * (compute_genotypes, src/genotyper.cpp:12-54, bound at whatshap/core.pyx:602-617): every read entry multiplies a
 * (hom-ref, het, hom-alt) distribution by the likelihood of its allele with error max(0.05, 10^(-phred/10)), renormalising
 * after every factor (src/genotypedistribution.cpp:56-66).  Host only, bit-identical doubles (same operation order).
 * Uses positions / reads of `p` (pedigree fields ignored).  gl: [n_cols][3]; gt: [n_cols], the likeliest genotype index
 * if the probability of the others is < 0.1, else -1 (the reference's empty Genotype). */
int whmec_compute_genotypes(const whmec_problem *p, double *gl, int8_t *gt, char *err, size_t errlen);

/* ---- A pedigree table (T = 4^trios > 1) shared by several GPUs --------------------------------
 * The reference sweeps a family's table on one thread (src/pedigreedptable.cpp:84-174).  Columns that no
 * read spans cut it into chains that exchange only the T projection values of the cut
 * (pedigreedptable.cpp:272-297), and a chain is min-plus linear in them.  A SEGMENT is a run of whole
 * chains given as a problem of its own (its columns, its reads, recombcost of exactly these columns);
 * one process per GPU holds one segment, and the caller (whatshap_b200/multigpu.py) moves T x T u32
 * matrices and T-vectors between the processes:
 *   1. whmec_segment_create   pack + upload; `continues` != 0 unless the segment starts the table
 *   2. whmec_segment_transfer matrix[u*T + i] = value at transmission value i behind the segment when the
 *                             vector handed to it is 0 at u and +inf (0xFFFFFFFF) elsewhere; the first
 *                             segment ignores its input (pedigreedptable.cpp:275-278): all rows equal
 *   3. (caller) all-gather the matrices, fold them left to right -> every segment's true input vector
 *   4. whmec_segment_sweep    sweep with the true input (NULL for the first segment), writing the same
 *                             back-pointers the single sweep would; out_vec = the T values behind it
 *   5. whmec_segment_exits    exits[u] = transmission value the backtrace hands to the preceding segment
 *                             when it enters this one with u; is_last: entered at the optimum of the
 *                             table's last column instead (all T answers equal)
 *   6. (caller) all-gather, follow the realised entries right to left
 *   7. whmec_segment_finish   backtrace from `entry` (< 0: this segment ends the table) + outputs for the
 *                             segment's columns and reads; s->cost is the table's optimum iff entry < 0
 * Results are bit-identical to whmec_solve on the whole table.  WHMEC_ERR_UNSUPPORTED: single-individual
 * problems (their chains are independent, shard them with whmec_solve), costs beyond 2^28. */
int whmec_segment_create(const whmec_problem *p, int device, int continues, whmec_plan **out, char *err, size_t errlen);
int whmec_segment_transfer(whmec_plan *plan, uint32_t *matrix /* [T*T] */, char *err, size_t errlen);
int whmec_segment_sweep(whmec_plan *plan, const uint32_t *in_vec /* [T] or NULL */, uint32_t *out_vec /* [T] */,
                        char *err, size_t errlen);
int whmec_segment_exits(whmec_plan *plan, int is_last, uint32_t *exits /* [T] */, char *err, size_t errlen);
int whmec_segment_finish(whmec_plan *plan, int entry, whmec_solution *s, char *err, size_t errlen);

/* ---- Coverage-capping read selection (host only; the step before the DP) -------------------------
 * whatshap/readselect.pyx:240-272 picks reads greedily by score until every variant is covered or max_cov
 * is reached.  Which read wins a tie is decided by the sift rules of the reference's positional max-heap
 * (whatshap/priorityqueue.pyx; scores are int triples compared lexicographically), by the iteration order
 * of a std::unordered_set<int> of freshly covered positions (readselect.pyx:117,135) and by the iteration
 * order of CPython sets of read indices.  The first two are reproduced here (the second by using the very
 * same container); the sets stay in Python (whatshap_b200/readselect.py), which hands their iteration
 * orders in as arrays.  Reads are CSR over entries in ReadSet order; the arrays given to _create must
 * outlive the selector.  Output arrays must hold n_reads (resp. the longest read's) elements. */
typedef struct whmec_selector whmec_selector;
whmec_selector *whmec_selector_create(uint32_t n_reads, uint32_t n_variants, const uint64_t *read_off, const int32_t *ent_pos,
                                      const uint32_t *ent_rank /* rank of ent_pos among `positions` */,
                                      const int32_t *positions /* sorted, distinct */, uint32_t max_cov);
void whmec_selector_destroy(whmec_selector *sel);
/* A slice (readselect.pyx:108-166) starts: queue items[0..n) in this order with scores[3*item .. 3*item+2]. */
void whmec_selector_begin_slice(whmec_selector *sel, const uint32_t *items, const int32_t *scores, uint32_t n);
/* Pop until a read is taken (returns 1: *read, the variant ranks it covers first in fresh_ranks[0..*n_fresh), in the
 * order the caller must process them) or the queue is empty (returns 0).  Reads popped on the way whose span is
 * already at max_cov are appended to over[0..*n_over). */
int whmec_selector_next(whmec_selector *sel, uint32_t *read, uint32_t *fresh_ranks, uint32_t *n_fresh, uint32_t *over,
                        uint32_t *n_over);
/* Score update after a read was taken (readselect.pyx:38-52,160-164) for items[0..n) in this order: if still queued,
 * the first component drops by the number of the item's variants that are not among the last fresh ones. */
void whmec_selector_rescore(whmec_selector *sel, const uint32_t *items, uint32_t n);
/* Bridging pass after a slice (readselect.pyx:199-228): queue items in order; a popped read whose span is full is
 * removed (taken 0), one that connects two blocks of the reads taken so far is taken (taken 1), others stay.
 * slice_reads: the reads the slice took.  Returns the number of removed[] / taken[] entries. */
uint32_t whmec_selector_bridge(whmec_selector *sel, const uint32_t *items, const int32_t *scores, uint32_t n,
                               const uint32_t *slice_reads, uint32_t n_slice, uint32_t *removed, uint8_t *taken);

/* Sort key of ReadSet::sort() ties: std::hash<std::string>(name) ^ std::hash<int>(source_id)
 * as computed by libstdc++ (64-bit murmur, seed 0xc70f6907); src/readset.h:68-72. */
uint64_t whmec_read_sort_key(const char *name, size_t len, int32_t source_id);

/* ---- PedMecHeuristic: the reference's row-limited heuristic PedMEC solver (`whatshap phase --algorithm=heuristic`) -------------
 * Replaces cpp.PedMecHeuristic(readset, recombcost, pedigree, distrust_genotypes, positions, row_limit, allow_mutations, verbosity)
 * + solve() + getOptBipartition / getOptTransmission / getOptHaplotypes / getMutations / getOptScore
 * (whatshap/cpp.pxd:261-272, whatshap/core.pyx:674-734, src/pedmecheuristic.cpp:9-81,121-409).
 * HOST code: the heuristic is a sequential beam search over float scores (at most row_limit partial solutions per column, each
 * extended read by read), not the exact DP of this library's CUDA path; it is built for completeness of the operator surface.
 * `p->read_ind` carries the reads' SAMPLE ids, which the reference requires to be the zero-based pedigree indices
 * (src/pedmecheuristic.h:66); p->gt must hold a diploid biallelic genotype (0, 1, 2) for every sample and column. */
typedef struct whmec_heuristic_solution {
    float score;            /* out: getOptScore() -- the reference never assigns its optScore, so this is 0 */
    uint32_t n_samples;     /* out: distinct sample ids among the reads and the trio members */
    uint8_t *partition;     /* [n_reads]  getOptBipartition(): 1 = true (core.pyx:719 reports 0 for true, 1 for false) */
    uint32_t *transmission; /* [n_cols]   getOptTransmission() */
    int8_t *haplotypes;     /* [n_ind][2][n_cols] getOptHaplotypes(), rows of samples >= n_samples untouched */
    uint8_t *mutated;       /* [n_ind][2][n_cols] 1 = getMutations() lists (haplotype, column) for the sample */
} whmec_heuristic_solution;
int whmec_heuristic(const whmec_problem *p, uint32_t row_limit, int allow_mutations, whmec_heuristic_solution *s, char *err,
                    size_t errlen);

#ifdef __cplusplus
}
#endif
#endif /* WHMEC_H */
