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
 *   whmec_realign          <- ReadSetReader.detect_alleles_by_alignment  whatshap/variants.py:599-912 (allele detection
 *                             by re-alignment, the step that builds the ReadSet)
 *   whmec_realign_kmerald  <- the same with use_kmerald=True  whatshap/variants.py:731-794, align.pyx:199-271
 *   whmec_detect_alleles_cigar <- _detect_alleles (allele detection without a reference)  whatshap/_variants.pyx:84-298,
 *                             whatshap/variants.py:409-597
 *   whmec_learn            <- Caller (the k-mer pair counts of `whatshap learn`)  src/caller.cpp, whatshap/core.pyx:651-671
 *   whmec_haplotag         <- prepare_haplotag_information (read assignment of `whatshap haplotag`)  whatshap/cli/haplotag.py:322-427
 *   whmec_haplotagphase    <- compute_votes + best_candidate + consensus (`whatshap haplotagphase`)  whatshap/cli/haplotagphase.py:203-395
 *   whmec_merge_reads      <- ReadMerger.merge (`whatshap phase --merge-reads`)  whatshap/merge.py:40-207
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
#define WHMEC_ERR_UNSUPPORTED 4 /* > 32 active reads (graycodes.cpp:12), more than 5 trios (T > 1024), cost range, a column beyond the HBM
                                   budget; five-trio tables: cost functions beyond 16 GiB, genotyping and table segments */

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
    uint32_t path_kind;          /* 1 = tile kernel, 2 = column kernel, 3 = batched pedigree sweep, 4 = genotyping (forward-backward),
                                    5 = wide column sweep (five trios, T = 1024), 6 = heuristic swept on the device */
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

/* ---- Several tables in one call --------------------------------------------------------------------------
 * `whatshap phase` builds one PedigreeDPTable per (chromosome x family); one such table rarely fills a GPU.  This entry point
 * takes n_tables independent problems and gives every one of them the solution whmec_solve gives it alone, bit for bit
 * (cost, path, partition, super-reads, ties included).
 *   - Single-individual tables that the tile kernel covers are swept TOGETHER: their chains are as independent as the chains
 *     of one table, so one persistent launch sweeps the panels of all of them, one launch backtraces all chains, and the
 *     per-table costs are reduced on the device.  Tables are grouped (consecutively) so that a group's device memory fits
 *     under one reading of the free memory; a table that does not fit alone takes the single-table path.
 *   - Trio tables (T = 4) whose columns all have the fused kernel's shape are swept TOGETHER as well: pass 1 and pass 2 of the
 *     fused sweep take the union of their chains, the fold between the passes restarts at every table, and the backtrace
 *     enters every table's last chain at that table's optimum.  Groups are cut under WHMEC_COLUMN_ARENA_BUDGET likewise.
 *   - Every other table (larger pedigrees, distrusted genotypes outside the fused shape, tables the tile planner declines,
 *     tables without columns) is solved inside the call by the single-table path, one after the other.
 * Errors are per table: status[t] and the message at errs + t * errlen (errs may be NULL) are what whmec_solve would have
 * returned for table t -- a Mendelian conflict or unsorted input in one table leaves the others solved.  The return value is
 * WHMEC_OK unless the call itself failed: WHMEC_ERR_INPUT for null arguments, WHMEC_ERR_CUDA for a CUDA failure (then every
 * status[] holds the code and every message the reason; running out of host memory fails the call the same way, with
 * WHMEC_ERR_UNSUPPORTED).  n_tables == 0 does nothing.  Every table of the list is packed on the host before the first sweep:
 * hand long lists over in slices.
 * stats (optional, [n_tables]): cells, algorithmic bytes, chains, max_active, T, path_kind, back-pointer and state bytes of
 * every table; times are 0 (tables share their sweeps).  total (optional): sums over the call; sweep_ms is the device time of
 * all sweeps, kernel_launches counts the sweep launches of the whole call, path_kind is 0 when the tables took different paths. */
int whmec_solve_batch(const whmec_problem *const *problems, whmec_solution *const *solutions, uint32_t n_tables, int device,
                      int *status /* [n_tables] */, char *errs /* [n_tables][errlen] or NULL */, size_t errlen,
                      whmec_stats *stats_or_null /* [n_tables] */, whmec_stats *total_or_null);

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
 * ~1e-13 (the reference's own tests compare with 1e-9, whatshap/testhelpers.py:11-15).  A table whose backward
 * tables do not fit the free HBM is cut into segments that share one arena and is swept backward again from
 * checkpoints (same likelihoods, more launches).  Besides pedigrees beyond GL_MAX_*, WHMEC_ERR_UNSUPPORTED only when
 * the fixed per-column arrays do not fit, or when not even one column per segment does; the message then says "needs at least N bytes" (for backward
 * tables, checkpoints and projection buffers).  st->backptr_bytes reports the bytes of backward tables kept in HBM (with
 * a table cut into segments: the largest store allocated, arena + checkpoints), st->sweep_ms the device time of both
 * passes, st->kernel_launches includes the repeated backward sweeps. */
int whmec_genotype(const whmec_problem *p, double *likelihoods, int device, whmec_stats *st_or_null, char *err, size_t errlen);

/* Many genotyping tables in one call (`whatshap genotype` builds one GenotypeDPTable per chromosome x family; with a
 * multi-sample VCF and no pedigree, every sample is a family of its own).  likelihoods[t] receives what whmec_genotype writes
 * for problems[t] ([n_ind][n_cols][3] doubles).  Tables are cut, in list order, into groups whose backward tables, projection
 * buffers and inputs fit the budget whmec_genotype uses (the free HBM, or WHMEC_GENOTYPE_ARENA_BUDGET); one group is one
 * upload and one step list: launch s advances the s-th column of every chain of a single individual and of every pedigree
 * table of the group, whatever its T, so a group costs 2 x (backward + forward steps of its longest chain or pedigree table)
 * launches.  A table that does not fit a group alone runs inside the call through whmec_genotype's own path (memory-bounded
 * mode included).  Errors are per table: status[t] and the message at errs + t * errlen (errs may be NULL) are what
 * whmec_genotype returns for table t.  The return value is WHMEC_ERR_INPUT for null arguments, WHMEC_ERR_CUDA for a device
 * failure (then every status holds it and every message the reason; running out of host memory while grouping or uploading
 * fails the call the same way, with WHMEC_ERR_UNSUPPORTED, as in whmec_solve_batch), WHMEC_OK otherwise; n_tables == 0 does
 * nothing.  stats (optional, [n_tables]): cells,
 * T, path_kind 4 and back-pointer bytes (backward tables) of every table, times 0; total (optional): sweep time and kernel
 * launches of the whole call. */
int whmec_genotype_batch(const whmec_problem *const *problems, double *const *likelihoods /* [n_tables] -> [n_ind][n_cols][3] */,
                         uint32_t n_tables, int device, int *status /* [n_tables] */, char *errs /* [n_tables][errlen] or NULL */,
                         size_t errlen, whmec_stats *stats_or_null /* [n_tables] */, whmec_stats *total_or_null);

/* Per-column genotype priors of one sample's reads, the step `whatshap genotype` runs before the DP above
 * (compute_genotypes, src/genotyper.cpp:12-54, bound at whatshap/core.pyx:602-617): every read entry multiplies a
 * (hom-ref, het, hom-alt) distribution by the likelihood of its allele with error max(0.05, 10^(-phred/10)), renormalising
 * after every factor (src/genotypedistribution.cpp:56-66).  Host only, bit-identical doubles (same operation order).
 * Uses positions / reads of `p` (pedigree fields ignored).  gl: [n_cols][3]; gt: [n_cols], the likeliest genotype index
 * if the probability of the others is < 0.1, else -1 (the reference's empty Genotype). */
int whmec_compute_genotypes(const whmec_problem *p, double *gl, int8_t *gt, char *err, size_t errlen);

/* ---- A pedigree table (1 < T = 4^trios <= 256) shared by several GPUs --------------------------------
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
 * problems (their chains are independent, shard them with whmec_solve), costs beyond 2^28, five-trio tables (T = 1024). */
int whmec_segment_create(const whmec_problem *p, int device, int continues, whmec_plan **out, char *err, size_t errlen);
int whmec_segment_transfer(whmec_plan *plan, uint32_t *matrix /* [T*T] */, char *err, size_t errlen);
int whmec_segment_sweep(whmec_plan *plan, const uint32_t *in_vec /* [T] or NULL */, uint32_t *out_vec /* [T] */,
                        char *err, size_t errlen);
int whmec_segment_exits(whmec_plan *plan, int is_last, uint32_t *exits /* [T] */, char *err, size_t errlen);
int whmec_segment_finish(whmec_plan *plan, int entry, whmec_solution *s, char *err, size_t errlen);

/* ---- A pedigree table (T = 4^trios > 1) genotyped by several GPUs -----------------------------
 * whmec_genotype sweeps a family's forward-backward table column by column on one device.  A SEGMENT is a run of whole chains
 * given as a problem of its own (as for whmec_segment_*: its columns, its reads, its priors, recombcost of exactly these
 * columns).  Only the T values of the cut cross between segments, and both recursions are linear in them: a segment's
 * forward output is alpha . M for a T x T transfer matrix M.  The caller (whatshap_b200/multigpu.py) moves T x T double
 * matrices and T-vectors between the processes:
 *   1. whmec_genotype_segment_create   pack + upload; `continues` != 0 unless the segment starts the table, `continued` != 0
 *                                      unless it ends the table
 *   2. whmec_genotype_segment_transfer matrix[u*T + i] = forward value at transmission value i of the segment's last column when
 *                                      the vector handed to it is e_u (the table's last segment: the total mass at i); the
 *                                      first segment ignores its input: all rows equal.  One positive factor on the whole
 *                                      matrix is left open (it cancels in the normalisation)
 *   3. (caller) all-gather the matrices and fold them: alpha_1 = M_0[0], alpha_{s+1} = alpha_s . M_s (left to right),
 *      beta_{S-2} = M_{S-1} . 1, beta_s = M_{s+1} . beta_{s+1} (right to left), each divided by its largest entry
 *   4. whmec_genotype_segment_run      the backward and forward passes of the segment from its true inputs: alpha_in (iff
 *                                      continues) is the forward vector in front of it, beta_in (iff continued) the backward
 *                                      vector behind it; likelihoods [n_ind][segment columns][3] as whmec_genotype's
 * The likelihoods agree with whmec_genotype on the whole table to ~1e-14.  A segment whose backward tables do not fit runs in
 * memory-bounded mode, like a table of whmec_genotype.  st (optional) receives the pass's device time and launches.
 * WHMEC_ERR_UNSUPPORTED: single-individual problems (their chains are independent tables; shard them with whmec_genotype);
 * WHMEC_ERR_INPUT: a missing alpha_in / beta_in. */
typedef struct whmec_gl_segment whmec_gl_segment;
int whmec_genotype_segment_create(const whmec_problem *p, int device, int continues, int continued, whmec_gl_segment **out, char *err,
                                  size_t errlen);
int whmec_genotype_segment_transfer(whmec_gl_segment *s, double *matrix /* [T*T] */, whmec_stats *st_or_null, char *err, size_t errlen);
int whmec_genotype_segment_run(whmec_gl_segment *s, const double *alpha_in /* [T] iff continues */, const double *beta_in /* [T] iff continued */,
                               double *likelihoods /* [n_ind][n_cols][3] */, whmec_stats *st_or_null, char *err, size_t errlen);
void whmec_genotype_segment_destroy(whmec_gl_segment *s);

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

/* Many heuristic tables in one call (`whatshap phase --algorithm=heuristic` builds one PedMecHeuristic per chromosome x family;
 * with a multi-sample VCF every sample is a table of its own).  solutions[t] receives, bit for bit, what
 * whmec_heuristic(problems[t], row_limits[t], allow_mutations[t], ...) writes.  On the GPU one CTA sweeps one table, its partial
 * solutions spread over the CTA's threads; tables are cut, longest first (columns x row_limit), into groups whose device memory
 * fits the free HBM (or WHMEC_HEURISTIC_ARENA_BUDGET), one launch per group.  whmec_heuristic runs inside the call, with the
 * same result, for: allow_mutations == 0, tables without reads, columns or samples, more than 16 samples, input errors, tables
 * that fit no group alone, and tables whose partial solutions outgrow their device row buffers (ties at the optimum can keep
 * any number of them).  Errors are per table: status[t] and the message at errs + t * errlen (errs may be NULL) are what
 * whmec_heuristic returns for table t.  The return value is WHMEC_ERR_INPUT for null arguments, WHMEC_ERR_CUDA for a device
 * failure (then every status holds it and every message the reason; running out of host memory fails the call the same way,
 * with WHMEC_ERR_UNSUPPORTED), WHMEC_OK otherwise; n_tables == 0 does nothing.  stats (optional, [n_tables]): path_kind 6 for
 * a table swept on the device (0: whmec_heuristic), cells = columns x row_limit, max_active, transmissions; total (optional):
 * device time and launches of the call, bytes copied to and from the device. */
int whmec_heuristic_batch(const whmec_problem *const *problems, whmec_heuristic_solution *const *solutions, const uint32_t *row_limits /* [n_tables] */,
                          const int *allow_mutations /* [n_tables] */, uint32_t n_tables, int device, int *status /* [n_tables] */,
                          char *errs /* [n_tables][errlen] or NULL */, size_t errlen, whmec_stats *stats_or_null /* [n_tables] */,
                          whmec_stats *total_or_null);

/* ---- Allele detection by re-alignment: ReadSetReader.detect_alleles_by_alignment(variants, restricted_genotypes, 0, alignment,
 * reference, overhang, use_affine, gap_start, gap_extend, default_mismatch) for many alignments in one call
 * (whatshap/variants.py:599-912, whatshap/_variants.pyx:10-81, whatshap/align.pyx:16-196).  kmer alignment: whmec_realign_kmerald.
 * The host walks every CIGAR against the variant list (WHMEC_HOST_THREADS workers) and lists the (alignment, variant) items and
 * their alleles; the device builds each padded allele from the reference, strips common prefix and suffix, computes every
 * allele's distance and makes the call.  Work goes in chunks of items under the free HBM (or WHMEC_REALIGN_ARENA_BUDGET bytes). */
typedef struct whmec_realign_input {
    uint32_t n_alignments;
    const int32_t *reference_start;  /* [n_alignments] */
    const uint64_t *cigar_off;       /* [n_alignments + 1] into cigar_op / cigar_len; an empty CIGAR yields nothing */
    const uint8_t *cigar_op;         /* pysam codes MIDNSHP=X = 0..8; others raise when the walk reaches them */
    const int32_t *cigar_len;
    const uint64_t *query_off;       /* [n_alignments + 1] into query */
    const uint8_t *query;            /* query_sequence bytes, compared case-sensitively */
    uint32_t n_variants;
    const int32_t *position;         /* [n_variants] */
    const uint32_t *allele_first;    /* [n_variants + 1]: variant v's alleles are slots allele_first[v] .. allele_first[v+1]-1, reference allele first */
    const uint64_t *allele_off;      /* [allele_first[n_variants] + 1] into allele_bytes */
    const uint8_t *allele_bytes;
    const uint64_t *restrict_off;    /* NULL: no restricted genotypes; else [n_variants + 1] into restrict_allele */
    const int32_t *restrict_allele;  /* per variant: the allele indices of its genotype (Genotype.as_vector()) */
    const uint8_t *reference;
    uint64_t reference_len;
    int32_t overhang;                /* >= 0 */
    int32_t affine;                  /* 0: edit_distance (quality 30); 1: edit_distance_affine_gap (quality d_best - d_second) */
    int32_t gap_start, gap_extend;
    double mismatch;                 /* default_mismatch, used as a float32 */
} whmec_realign_input;

typedef struct whmec_realign_output { /* filled by the library; release with whmec_realign_release */
    uint64_t *call_off;              /* [n_alignments + 1] into the three arrays below */
    uint32_t *variant;               /* index into the variant list */
    int32_t *allele;
    int64_t *quality;
} whmec_realign_output;

typedef struct whmec_realign_stats {
    uint64_t items;                  /* (alignment, variant) pairs aligned */
    uint64_t jobs;                   /* allele alignments */
    uint64_t short_jobs, long_jobs;  /* one thread per job / one warp per job */
    uint64_t long_items;             /* items with at least one warp job */
    uint64_t cells;                  /* sum of untrimmed query x target lengths */
    uint64_t h2d_bytes, d2h_bytes;
    uint32_t chunks, kernel_launches;
    float device_ms;                 /* device time of the launches (CUDA events) */
    float plan_ms;                   /* host walk */
} whmec_realign_stats;

/* Returns WHMEC_OK, WHMEC_ERR_INPUT for malformed arguments and for every input on which the reference raises (an unknown CIGAR
 * operation, a failed window assert, an empty allele list after the restriction, a distance beyond int64): err then names the
 * first such alignment (and variant); WHMEC_ERR_CUDA for a device failure.  out is only filled on WHMEC_OK.  stats may be NULL. */
int whmec_realign(const whmec_realign_input *in, int device, whmec_realign_output *out, whmec_realign_stats *stats, char *err,
                  size_t errlen);
void whmec_realign_release(whmec_realign_output *out);

/* edit_distance(query[i], target[i]) and edit_distance_affine_gap(query[i], target[i], [mismatch] * len(query[i]), gap_start,
 * gap_extend) for n pairs (align.pyx:16-196); either output may be NULL.  Return codes as whmec_realign. */
int whmec_edit_distance_batch(uint32_t n, const uint64_t *query_off, const uint8_t *query, const uint64_t *target_off,
                              const uint8_t *target, double mismatch, int32_t gap_start, int32_t gap_extend, int64_t *unit_out,
                              int64_t *affine_out, int device, whmec_realign_stats *stats, char *err, size_t errlen);

/* ---- Allele detection by k-mer re-alignment: detect_alleles_by_alignment(..., use_kmerald=True, kmerald_costs, kmer_size,
 * kmerald_gappenalty, kmerald_window) (whatshap/variants.py:731-794, whatshap/align.pyx:199-271), `whatshap genotype
 * --use-kmerald`.  Each covered, non-symbolic variant's query window (kmerald_window for the overhang) is cut into k-mers
 * (enumerate_all_kmers) and aligned (kmer_align) against the k-mers of allele 0 and of the variant's alternative_allele; the
 * smaller distance is called with quality 30, a tie or NaN gives no call.  The restricted genotypes, overhang, affine and the
 * affine costs of whmec_realign_input are ignored. */
typedef struct whmec_kmer_costs {
    uint64_t n;                      /* < 2^32 */
    const uint64_t *key;             /* [n], strictly ascending: (uint64_t)ref_kmer << 32 | read_kmer; read k-mer 0 stands for the
                                        reference's -5 (the ref k-mer's default cost; a real k-mer is never 0) */
    const float *cost;               /* [n]: float(value) as a float32 */
} whmec_kmer_costs;

typedef struct whmec_kmerald_params {
    int32_t kmer_size;               /* 1..15 */
    float gap_penalty;
    int32_t window;                  /* int(kmerald_window), >= 0 */
    const whmec_kmer_costs *costs;
    const uint64_t *alt_off;         /* [n_variants + 1] into alt_bytes: each variant's alternative_allele (NULL in the batch) */
    const uint8_t *alt_bytes;
    const uint8_t *has_alt;          /* [n_variants]: 0 for a variant without alternative_allele (the reference raises on it) */
} whmec_kmerald_params;

/* Return codes, output, release (whmec_realign_release) and errors as whmec_realign; a covered, non-symbolic variant without
 * alternative_allele is one more input on which the reference raises.  stats->short_jobs / long_jobs: one thread / one warp
 * per allele alignment. */
int whmec_realign_kmerald(const whmec_realign_input *in, const whmec_kmerald_params *params, int device, whmec_realign_output *out,
                          whmec_realign_stats *stats, char *err, size_t errlen);

/* kmer_align(enumerate_all_kmers(s1[i], k), enumerate_all_kmers(s2[i], k), costs, gap_penalty) for n pairs, as float32
 * (params' alt fields are not used).  Return codes as whmec_realign. */
int whmec_kmer_align_batch(uint32_t n, const uint64_t *s1_off, const uint8_t *s1, const uint64_t *s2_off, const uint8_t *s2,
                           const whmec_kmerald_params *params, float *out, int device, whmec_realign_stats *stats, char *err,
                           size_t errlen);

/* ---- Allele detection from the CIGAR alone (`whatshap phase --no-reference`, `whatshap haplotag --no-reference`): per alignment a,
 * _detect_alleles(normalized, var_progress, 0, a) of ReadSetReader._alignments_to_reads (whatshap/variants.py:409-597,
 * whatshap/_variants.pyx:84-298), for many alignments in one call.  For alignments in non-decreasing reference_start order (as
 * _usable_alignments yields them) the reference's running index gives the same answer as first = 0.  The library normalizes the
 * variants (strip common suffixes, then common prefixes), drops those detect_non_overlapping_variants drops and builds each allele's
 * match, insert and delete targets; the device walks every CIGAR into enqueued (alignment, variant) items and resolves each item.
 * The reference, restricted genotypes, overhang and affine fields of whmec_realign_input are ignored; query holds query_sequence. */
typedef struct whmec_query_qualities {
    const uint64_t *qual_off;        /* [n_alignments + 1] into qual; an empty range: no (or empty) query_qualities, 30 per base */
    const uint8_t *qual;             /* query_qualities */
    const uint8_t *missing;          /* NULL or [n_alignments]: bit 0, query_sequence is None (reading a base raises TypeError);
                                        bit 1, cigartuples is None (iterating it raises TypeError) */
} whmec_query_qualities;

/* q may be NULL (30 per base, every sequence and CIGAR present).  Output, release (whmec_realign_release), return codes and the
 * chunk budget (WHMEC_REALIGN_ARENA_BUDGET) as whmec_realign.  WHMEC_ERR_INPUT for malformed arguments, for positions, lengths and
 * spans that would leave the reference's C ints, for a variant without alternative alleles that the conflict filter reaches (its
 * max() raises ValueError), and for every alignment on which the reference raises (an operation outside 0..8: ValueError; a base
 * or quality index past the end of query_sequence or query_qualities: IndexError; a missing sequence or CIGAR: TypeError); err
 * then names the first such alignment and the exception.  stats: items = enqueued variants, jobs = short_jobs = their alleles (one
 * thread per item), long_jobs = long_items = 0, cells = calls, chunks = item windows run. */
int whmec_detect_alleles_cigar(const whmec_realign_input *in, const whmec_query_qualities *q, int device, whmec_realign_output *out,
                               whmec_realign_stats *stats, char *err, size_t errlen);

/* ---- K-mer pair counts of `whatshap learn`: the rows the reference's Caller (src/caller.cpp, whatshap/core.pyx:651-671) writes
 * for the reads run_learn hands it (whatshap/cli/learn.py), for many reads in one call.  A read's k-mer at column c is counted iff
 * c > its floor T_r = max(k - 1, pos_m + k - 1 over every read m before it); a read with a single k-mer counts it twice.  The
 * popped columns (k .. L with `final`, else k .. max(k - 1, max pos_r + k - 1), or the given range) pass the variant windows in
 * order (pop_column); each remaining column that has counts gives one row per read k-mer, rows ascending by column, then by
 * read k-mer (the reference's order within a column is its unordered_map's).  The host walks every CIGAR (WHMEC_HOST_THREADS
 * workers) and cuts the columns into chunks under the free HBM less 512 MB (or WHMEC_LEARN_ARENA_BUDGET bytes); the device emits
 * one key per kept k-mer, sorts and run-length encodes the keys and attaches the reference k-mers. */
typedef struct whmec_learn_input {
    const uint8_t *reference;        /* the chromosome's bytes (only A, C, G and T count; N and lower case leave the k-mer as it is) */
    uint64_t reference_len;          /* L, k <= L < 2^31 */
    uint32_t n_alignments;           /* in the order of the add_read calls */
    const int32_t *reference_start;  /* [n_alignments]: alignment.pos */
    const uint64_t *cigar_off;       /* [n_alignments + 1] into cigar_op / cigar_len */
    const uint8_t *cigar_op;         /* pysam codes MIDNSHP=X = 0..8 */
    const int32_t *cigar_len;        /* >= 0 */
    const uint64_t *query_off;       /* [n_alignments + 1] into query */
    const uint8_t *query;            /* query_alignment_sequence bytes */
    uint32_t n_variants;             /* > 0: the whole list all_variants was given, in its order */
    const int32_t *variant_pos;      /* [n_variants]: VCF position (1-based) */
    const int32_t *variant_len;      /* [n_variants]: len(REF) */
    uint32_t first_variant;          /* the variant list's state before the first popped column (its front), < n_variants */
    int32_t k;                       /* 1..15 */
    int32_t window;
    int32_t final;                   /* 1: pop columns k..L (final_pop); 0: k..max(k - 1, max target) (a Caller that is abandoned) */
    int64_t col_lo, col_hi;          /* col_lo > 0: pop exactly the columns col_lo..col_hi instead (k <= col_lo, col_hi <= L) */
    const int32_t *floor;            /* NULL: the floors as above; else [n_alignments]: each read's T_r (>= k - 1) */
} whmec_learn_input;

typedef struct whmec_learn_output {  /* filled by the library (rows) or by the caller (for whmec_learn_write) */
    uint64_t n_rows;
    int32_t *rows;                   /* [n_rows][4]: column, reference k-mer, read k-mer, count */
    uint32_t next_variant;           /* the variant list's front after the last popped column */
} whmec_learn_output;

typedef struct whmec_learn_stats {
    uint64_t alignments;
    uint64_t kmers;                  /* k-mers the reads enumerate */
    uint64_t kept;                   /* keys counted (above the floor, in the popped columns; a single k-mer twice) */
    uint64_t distinct;               /* distinct (column, read k-mer) keys */
    uint64_t rows;                   /* those in output columns */
    uint64_t h2d_bytes, d2h_bytes;
    uint32_t chunks, kernel_launches;
    float device_ms;                 /* device time of the chunks' launches (CUDA events) */
    float plan_ms;                   /* host walk, floors, variant windows and chunk cut */
} whmec_learn_stats;

/* Returns WHMEC_OK, WHMEC_ERR_INPUT for malformed arguments and for every input on which the reference aborts or reads out of
 * bounds (k outside 1..15, L < k, an empty variant list, a read without a k-mer, P, B or an unknown operation of non-zero length
 * or a CIGAR that ends while query bytes remain, pos + k - 1 > L or a k-mer column beyond L, positions outside int32): err then
 * names the first such alignment; WHMEC_ERR_CUDA for a device failure.  out is only filled on WHMEC_OK.  stats may be NULL. */
int whmec_learn(const whmec_learn_input *in, int device, whmec_learn_output *out, whmec_learn_stats *stats, char *err, size_t errlen);
void whmec_learn_release(whmec_learn_output *out);
/* Writes out's rows as the reference does ("%d\t%d\t%d\t%d\n"), appending (append != 0) or truncating.  WHMEC_ERR_INPUT when
 * the file cannot be written. */
int whmec_learn_write(const char *path, const whmec_learn_output *out, int append, char *err, size_t errlen);

/* ---- Read assignment of `whatshap haplotag`: the sums of prepare_haplotag_information (whatshap/cli/haplotag.py), for the
 * reads of many samples in one call.  Per sample, in read order, a read whose representation is already processed is skipped;
 * otherwise it opens a group with the unprocessed reads of its BX id within linked_read_cutoff of its reference_start (in read
 * order), and every member's representation becomes processed.  The group's entries (opening read first, then the linked
 * reads, each in its own order) add their quality to (block, h) for every phase-tuple index h whose allele equals theirs.  The
 * group takes the block with the highest maximum score (ties: the block matched first), in it the haplotype with the highest
 * score (ties: the lowest index; haplotypes no allele matched score 0), and quality = best - second best of the ploidy scores.
 * The host walks the groups and cuts them into chunks under the free HBM less 512 MB (or WHMEC_HAPLOTAG_ARENA_BUDGET bytes); the
 * device emits one (group, block, haplotype) key per match, radix-sorts the keys and reduces each group's runs. */
typedef struct whmec_haplotag_input {
    uint32_t n_samples;
    const uint64_t *phase_off;       /* [n_samples + 1] into phase_pos / phase_block / allele_off */
    const int64_t *phase_pos;        /* per sample ascending, distinct: the positions with a phase and a block id */
    const int64_t *phase_block;      /* int(block_id) */
    const uint64_t *allele_off;      /* [phase_off[n_samples] + 1] into allele */
    const int32_t *allele;           /* the phase tuples (an allele outside int32 or None as -1) */
    uint32_t n_reads;                /* every sample's reads, samples in ascending order, each sample's in ReadSet order */
    const uint64_t *read_off;        /* [n_reads + 1] into the entries */
    const int64_t *entry_pos;
    const int32_t *entry_allele;     /* an allele outside int32 as -1 */
    const int32_t *entry_quality;
    const uint32_t *read_sample;     /* [n_reads] < n_samples, non-decreasing */
    const int64_t *read_repr;        /* [n_reads] interned representation, >= 0 */
    const int64_t *read_bx;          /* [n_reads] interned BX tag, -1 for none (or when linked reads are ignored) */
    const int64_t *reference_start;  /* [n_reads] */
    int64_t ploidy;
    int64_t linked_read_cutoff;
} whmec_haplotag_input;

typedef struct whmec_haplotag_output {  /* caller-allocated [n_reads] arrays */
    int64_t *group;                  /* the group's opening read, -1 for a skipped read */
    int32_t *n_blocks;               /* at an opening read: blocks its group matched (0 elsewhere) */
    int64_t *block;                  /* at an opening read: the chosen block id */
    int32_t *haplotype;              /* at an opening read: the haplotype, -1 when not tagged (no block, or quality 0) */
    int64_t *quality;                /* at an opening read: best - second best score */
    int32_t error_kind;              /* the first error in visit order: 0 none, 1 AssertionError (allele not 0 or 1), 2 KeyError
                                        (position without phase), 3 IndexError (a match at h >= ploidy, or ploidy < 2 at a choice) */
    int64_t error_read;              /* the read it happened at (the opening read for a choice) */
    int64_t error_entry;             /* the entry of that read, -1 for a choice */
} whmec_haplotag_output;

typedef struct whmec_haplotag_stats {
    uint64_t entries;                /* entries of the groups */
    uint64_t groups;
    uint64_t keys;                   /* matches (one key each) */
    uint64_t runs;                   /* distinct (group, block, haplotype) */
    uint64_t h2d_bytes, d2h_bytes;
    uint32_t chunks, kernel_launches;
    float device_ms;                 /* device time of the chunks' launches (CUDA events) */
    float plan_ms;                   /* host group walk and chunk cut */
} whmec_haplotag_stats;

/* Returns WHMEC_OK (also when error_kind is set: then only the error fields are meaningful), WHMEC_ERR_INPUT for malformed
 * arguments, WHMEC_ERR_UNSUPPORTED when one group's keys cannot be sorted in one call (more than 2^30 matches, or more than 64
 * key bits), WHMEC_ERR_CUDA for a device failure.  stats may be NULL. */
int whmec_haplotag(const whmec_haplotag_input *in, int device, whmec_haplotag_output *out, whmec_haplotag_stats *stats, char *err,
                   size_t errlen);

/* ---- Votes of `whatshap haplotagphase`: compute_votes, best_candidate and consensus (whatshap/cli/haplotagphase.py) for many
 * samples in one call.  Per sample, a read with HP_tag < 1 or PS_tag < 1 is skipped, one with HP_tag > 2 is skipped and counted;
 * every entry of the others at a heterozygous position adds its quality to the key (PS_tag - 1, (HP_tag - 1) ^ allele_to_id
 * [allele]) of its position, the first read to reach (position, phase set) inserting (ps, 0) and (ps, 1).  A position takes the
 * key with the highest score (ties: the key inserted first), q = score / total as a double; an unphased position is dropped when
 * 100 q < gap_threshold or (only_indels and it is an SNV).  Positions come out in the order the reads first reached them.
 * The runs form (n_runs_pos > 0 in place of reads) hands over votes a caller holds: per position its (ps, h, score) in key
 * order, chosen by the same rule.  The host bins the entries by position and cuts whole positions of one sample into chunks under
 * the free HBM less 512 MB (or WHMEC_HAPLOTAGPHASE_ARENA_BUDGET bytes); the device emits one key per entry, radix-sorts the keys,
 * walks each position's runs in one thread and orders positions and keys by first entry. */
typedef struct whmec_haplotagphase_input {
    uint32_t n_samples;
    const uint64_t *pos_off;         /* [n_samples + 1] into the position arrays */
    const int64_t *pos;              /* per sample ascending, distinct */
    const uint8_t *pos_flags;        /* 1 homozygous, 2 phased (phase is not None), 4 SNV */
    const uint64_t *a2i_off;         /* [pos_off[n_samples] + 1]: allele -> id pairs, merged as the reference merges records */
    const int64_t *a2i_allele;
    const int64_t *a2i_id;
    const uint64_t *i2a_off;         /* [pos_off[n_samples] + 1]: id -> allele pairs */
    const int64_t *i2a_id;
    const int64_t *i2a_allele;
    uint64_t n_reads;                /* the vote form: every sample's reads, samples ascending */
    const uint32_t *read_sample;     /* [n_reads], non-decreasing */
    const int64_t *read_hp;          /* HP_tag */
    const int64_t *read_ps;          /* PS_tag */
    const uint64_t *read_off;        /* [n_reads + 1] into the entries */
    const int64_t *entry_pos;
    const int64_t *entry_allele;
    const int32_t *entry_quality;
    uint64_t n_runs_pos;             /* the runs form: voted positions, each a position of its sample's table, in vote order */
    const uint32_t *runs_sample;     /* [n_runs_pos], non-decreasing */
    const int64_t *runs_pos;
    const uint64_t *run_off;         /* [n_runs_pos + 1] into the runs */
    const int64_t *run_ps;
    const int64_t *run_h;
    const int64_t *run_score;
    double gap_threshold;
    int32_t only_indels;
} whmec_haplotagphase_input;

typedef struct whmec_haplotagphase_output {
    uint64_t *voted_off;             /* caller-allocated [n_samples + 1]: sample s's voted positions in [voted_off[s], voted_off[s+1]) */
    uint64_t *skipped;               /* caller-allocated [n_samples]: reads with HP_tag > 2 */
    int32_t *entry_error;            /* caller-allocated [n_samples]: the sample's first vote error, 0 none, 1 KeyError (position
                                        missing), 2 KeyError (allele missing from allele_to_id), 3 KeyError (ht ^ id not 0 or 1) */
    uint64_t *entry_error_at;        /* caller-allocated [n_samples]: its entry (an index into entry_pos) */
    /* library-allocated, [n_voted] per position in vote order, freed by whmec_haplotagphase_release */
    uint64_t n_voted;
    int64_t *voted_pos;
    int64_t *phase_set;              /* the best key's ps (PS_tag - 1, or run_ps) */
    int64_t *haplotype;              /* the best key's h */
    int64_t *score;
    int64_t *total;
    int64_t *allele;                 /* [n_voted][2]: id_to_allele[h], id_to_allele[1 - h] of a kept position */
    uint8_t *kept;
    int32_t *error;                  /* 0, 1 ZeroDivisionError (total 0), 2 KeyError (id_to_allele of a kept position), 3 ValueError
                                        (|score| or |total| reaches 2^53), 4 IndexError (a runs-form position without runs) */
    /* the vote form: every position's keys in insertion order, (ps, 0) and (ps, 1) per phase set */
    uint64_t *key_off;               /* [n_voted + 1] into the keys */
    int64_t *key_ps;
    int64_t *key_score;              /* h alternates 0, 1 */
} whmec_haplotagphase_output;

typedef struct whmec_haplotagphase_stats {
    uint64_t entries;                /* entries that voted */
    uint64_t positions;              /* voted positions */
    uint64_t records;                /* distinct (position, phase set) */
    uint64_t h2d_bytes, d2h_bytes;
    uint32_t chunks, kernel_launches;
    float device_ms;                 /* device time of the chunks' launches (CUDA events) */
    float plan_ms;                   /* host binning, chunk cut and gather */
} whmec_haplotagphase_stats;

/* Returns WHMEC_OK (errors of the reference are reported in entry_error and error), WHMEC_ERR_INPUT for malformed arguments,
 * WHMEC_ERR_UNSUPPORTED when one position has 2^31 entries or more, WHMEC_ERR_CUDA for a device failure.  stats may be NULL. */
int whmec_haplotagphase(const whmec_haplotagphase_input *in, int device, whmec_haplotagphase_output *out, whmec_haplotagphase_stats *stats,
                        char *err, size_t errlen);
void whmec_haplotagphase_release(whmec_haplotagphase_output *out);

/* ---- Read merging of `whatshap phase --merge-reads`: ReadMerger.merge (whatshap/merge.py) for many readsets in one call.  Per
 * set, read i has begin = its first position and end = begin + its number of entries; read j < i is compared with i iff
 * end_j > begin_k for every k in (j, i].  The pair counts match m and mismatch mm over alleles_j[begin_i - begin_j:] (Python slice
 * semantics) against alleles_i; the edge is blue when m + mm >= thr_neg_diff, min(m, mm) / (m + mm) <= max_error_rate and
 * m - mm >= thr_diff, and also not-blue when in addition mm - m >= thr_neg_diff.  For every not-blue edge inside one blue
 * component the blue edge of least m - mm on a bidirectional BFS path is removed until its ends part.  A blue component of two
 * reads or more becomes one read at its least member: per position the qualities of each allele summed (z0, z1), allele
 * z0 < z1, quality |z1 - z0|, positions ascending.  The host finds the pairs and cuts them into chunks under the free HBM less
 * 512 MB (or WHMEC_MERGE_ARENA_BUDGET bytes); the device packs alleles as bits, evaluates one pair per thread, hooks blue
 * edges into a parent array when no not-blue edge can exist (thr_diff + thr_neg_diff > 0; else the edges come back to the host
 * for the removal loop), and sums the merged reads' entries by (representative, position) with a radix sort. */
typedef struct whmec_merge_input {
    uint32_t n_sets;
    const uint64_t *set_off;         /* [n_sets + 1] into the reads */
    const uint64_t *read_off;        /* [set_off[n_sets] + 1] into the entries */
    const int32_t *position;
    const uint8_t *allele;
    const int32_t *quality;
    int64_t thr_diff;
    int64_t thr_neg_diff;
    double max_error_rate;
} whmec_merge_input;

typedef struct whmec_merge_output {
    int32_t *error_kind;             /* caller-allocated [n_sets]: 0 none, 1 IndexError (an empty read), 2 AssertionError (an allele
                                        other than 0 or 1); a set with an error has no output reads */
    uint64_t *error_read;            /* caller-allocated [n_sets]: the first offending read, an index within its set */
    int64_t *representative;         /* caller-allocated [set_off[n_sets]]: every read's least component member, within its set */
    uint64_t *out_off;               /* caller-allocated [n_sets + 1] into the output reads */
    /* library-allocated, freed by whmec_merge_reads_release */
    uint64_t n_out;
    uint64_t *out_read;              /* [n_out]: the input read (a singleton or a representative), an index within its set */
    uint64_t *out_entry_off;         /* [n_out + 1] into the output entries */
    int32_t *out_position;
    uint8_t *out_allele;
    int64_t *out_quality;
} whmec_merge_output;

typedef struct whmec_merge_stats {
    uint64_t reads, entries, pairs;
    uint64_t blue_edges, notblue_edges, removed_edges;
    uint64_t merged_components;      /* blue components of two reads or more */
    uint64_t output_reads;
    uint64_t h2d_bytes, d2h_bytes;
    uint32_t chunks, kernel_launches;
    float device_ms;                 /* device time of the launches (CUDA events) */
    float plan_ms;                   /* host validation, pair counts, chunk cut, removal loop and output layout */
} whmec_merge_stats;

/* Returns WHMEC_OK (also when error_kind is set), WHMEC_ERR_INPUT for malformed arguments, WHMEC_ERR_UNSUPPORTED when a set has
 * 2^32 reads or more, WHMEC_ERR_CUDA for a device failure.  stats may be NULL. */
int whmec_merge_reads(const whmec_merge_input *in, int device, whmec_merge_output *out, whmec_merge_stats *stats, char *err,
                      size_t errlen);
void whmec_merge_reads_release(whmec_merge_output *out);

#ifdef __cplusplus
}
#endif
#endif /* WHMEC_H */
