// Host packer: ReadSet/Pedigree (flat CSR form) -> per-column records + affine cost functions,
// and the inverse step from the optimal path to the reference's outputs.
//
// Restates, on the host and once per problem, what the reference recomputes per column:
//   ColumnIterator::get_next               src/columniterator.cpp:91-139
//   ColumnIndexingScheme ctor/set_next     src/columnindexingscheme.cpp:7-34,62-85
//   PedigreePartitions                     src/pedigreepartitions.cpp:7-42
//   PedigreeColumnCostComputer ctor        src/pedigreecolumncostcomputer.cpp:14-50
//   get_alleles / get_super_reads          src/pedigreecolumncostcomputer.cpp:117-175, src/pedigreedptable.cpp:344-406
#include "pack.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <functional>
#include <thread>

namespace whmec {

namespace {

constexpr uint32_t MAX_IND = 16;
constexpr uint32_t MAX_P = 10;

// src/pedigreepartitions.cpp:7-42
bool build_h2p(const whmec_problem *p, uint32_t tv, int8_t *h2p /* [n_ind][2] */) {
    std::vector<int> triple_of(p->n_ind, -1);
    for (uint32_t r = 0; r < p->n_trios; ++r) triple_of[p->trios[3 * r + 2]] = (int)r;
    for (uint32_t i = 0; i < p->n_ind; ++i) h2p[2 * i] = h2p[2 * i + 1] = -1;
    int q = 0;
    for (uint32_t i = 0; i < p->n_ind; ++i)
        if (triple_of[i] < 0) {
            h2p[2 * i] = (int8_t)q;
            h2p[2 * i + 1] = (int8_t)(q + 1);
            q += 2;
        }
    // resolve children; at most n_ind rounds, otherwise the pedigree is cyclic
    for (uint32_t round = 0; round <= p->n_ind; ++round) {
        bool pending = false;
        for (uint32_t i = 0; i < p->n_ind; ++i) {
            if (h2p[2 * i] != -1) continue;
            int r = triple_of[i];
            uint32_t f = p->trios[3 * r], m = p->trios[3 * r + 1];
            if (h2p[2 * f] == -1 || h2p[2 * m] == -1) {
                pending = true;
                continue;
            }
            h2p[2 * i] = h2p[2 * f + (((tv >> (2 * r)) & 1) ? 0 : 1)];
            h2p[2 * i + 1] = h2p[2 * m + (((tv >> (2 * r + 1)) & 1) ? 0 : 1)];
        }
        if (!pending) return true;
    }
    return false;
}

}  // namespace

int pack_problem(const whmec_problem *p, Packed &pk, std::string &err, bool want_deltas) {
    const bool timing = std::getenv("WHMEC_TIMING") != nullptr;
    auto tnow = [] { return std::chrono::steady_clock::now(); };
    auto tms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    const auto t_start = tnow();
    const uint32_t n = p->n_cols;
    pk = Packed();
    pk.has_deltas = want_deltas;
    pk.n = n;
    pk.n_reads = p->n_reads;
    pk.n_ind = p->n_ind;
    pk.n_trios = p->n_trios;
    if (n > 0 && (!p->recombcost || (!p->distrust && !p->gt))) {
        err = "recombcost and genotypes must be given for every column";
        return WHMEC_ERR_INPUT;
    }
    if (p->n_reads > 0 && (!p->read_off || !p->ent_col || !p->ent_allele || !p->ent_phred || !p->read_ind)) {
        err = "read arrays must not be null";
        return WHMEC_ERR_INPUT;
    }
    if (p->n_trios > 0 && !p->trios) {
        err = "trios must not be null";
        return WHMEC_ERR_INPUT;
    }
    if (p->n_ind == 0 || p->n_ind > MAX_IND) {
        err = "pedigree must have between 1 and 16 individuals";
        return WHMEC_ERR_UNSUPPORTED;
    }
    if (p->n_trios >= p->n_ind || p->n_trios > 5) {
        err = "unsupported pedigree: at most 5 trio relationships (T = 4^trios <= 1024)";
        return p->n_trios > 5 ? WHMEC_ERR_UNSUPPORTED : WHMEC_ERR_INPUT;
    }
    pk.P = 2 * (p->n_ind - p->n_trios);
    if (pk.P > MAX_P) {
        err = "unsupported pedigree: more than 10 founder haplotypes";
        return WHMEC_ERR_UNSUPPORTED;
    }
    pk.tb = 2 * p->n_trios;
    pk.T = 1u << pk.tb;
    const uint32_t T = pk.T, P = pk.P;
    {
        std::vector<int> child_count(p->n_ind, 0);
        for (uint32_t r = 0; r < p->n_trios; ++r) {
            for (int q = 0; q < 3; ++q)
                if (p->trios[3 * r + q] >= p->n_ind) {
                    err = "trio refers to an individual outside the pedigree";
                    return WHMEC_ERR_INPUT;
                }
            if (++child_count[p->trios[3 * r + 2]] > 1) {
                err = "individual is the child of two trios";
                return WHMEC_ERR_INPUT;
            }
        }
    }
    pk.h2p.assign((size_t)T * p->n_ind * 2, -1);
    for (uint32_t t = 0; t < T; ++t)
        if (!build_h2p(p, t, &pk.h2p[(size_t)t * p->n_ind * 2])) {
            err = "cyclic pedigree";
            return WHMEC_ERR_INPUT;
        }
    if (p->distrust && !p->gl && n > 0) {
        err = "distrust_genotypes requires genotype likelihoods for every individual and column";
        return WHMEC_ERR_INPUT;
    }

    // ---- read spans and the checks of the ColumnIterator constructor (columniterator.cpp:25-33); ranges of
    //      reads are checked by independent host threads, the reference's error is that of the first failing read
    std::vector<uint32_t> first(p->n_reads), last(p->n_reads);
    uint64_t phred_total = 0;
    {
        constexpr uint32_t READS_PER_TASK = 4096;
        const uint32_t n_tasks = (p->n_reads + READS_PER_TASK - 1) / READS_PER_TASK;
        struct Range {
            const char *err = nullptr;
            int rc = WHMEC_OK;
            uint64_t phred = 0;
        };
        std::vector<Range> ranges(n_tasks);
        parallel_tasks(n_tasks, host_threads(32), [&](uint32_t task) {
            Range &rg = ranges[task];
            const uint32_t r_begin = task * READS_PER_TASK, r_end = std::min(p->n_reads, r_begin + READS_PER_TASK);
            uint64_t phred = 0;
            auto fail = [&](const char *msg) {
                rg.err = msg;
                rg.rc = WHMEC_ERR_INPUT;
            };
            for (uint32_t r = r_begin; r < r_end; ++r) {
                const uint64_t b = p->read_off[r], e = p->read_off[r + 1];
                if (e <= b) return fail("No variants present");
                for (uint64_t q = b; q < e; ++q) {
                    if (q > b && p->ent_col[q] <= p->ent_col[q - 1]) return fail("ColumnIterator: encountered read with unsorted variants.");
                    if (p->ent_allele[q] > 2) return fail("allele of a read entry must be 0 (REF), 1 (ALT) or 2 (BLANK)");
                    phred += p->ent_phred[q];
                }
                first[r] = p->ent_col[b];
                last[r] = p->ent_col[e - 1];
                if (last[r] >= n) return fail("read entry refers to a column outside positions");
                // the preceding read (an empty one fails in its own right, before this read is looked at)
                const uint32_t prev_first = (r > 0 && p->read_off[r] > p->read_off[r - 1]) ? p->ent_col[p->read_off[r - 1]] : 0;
                if (first[r] < prev_first) return fail("ColumnIterator: reads in ReadSet are not sorted.");
                if (p->read_ind[r] >= p->n_ind) return fail("read refers to an individual outside the pedigree");
            }
            rg.phred = phred;
        });
        for (const Range &rg : ranges) {
            if (rg.rc != WHMEC_OK) {
                err = rg.err;
                return rg.rc;
            }
            phred_total += rg.phred;
        }
    }

    pk.read_first = first;
    pk.read_last = last;
    if (n > 0 && p->n_reads > 0 && first[p->n_reads - 1] >= n) {
        err = "read starts at a column that is not in positions";
        return WHMEC_ERR_INPUT;
    }

    const auto t_valid = tnow();
    // ---- split the columns at DP-independent chain boundaries (no read spans the cut) into chunks
    //      that are packed by independent host threads
    std::vector<int32_t> span(n + 2, 0);  // span[k] > 0: some read is active in both k-1 and k
    for (uint32_t r = 0; r < p->n_reads; ++r)
        if (last[r] > first[r]) {
            span[first[r] + 1] += 1;
            span[last[r] + 1] -= 1;
        }
    std::vector<uint32_t> cut;  // chunk starts (columns)
    {
        const uint32_t hw = host_threads(32);
        const uint32_t target = std::max<uint32_t>(256, n / (4 * hw) + 1);
        int32_t run = 0;
        uint32_t last_cut = 0;
        cut.push_back(0);
        for (uint32_t k = 1; k < n; ++k) {
            run += span[k];
            if (run == 0 && k - last_cut >= target) {
                cut.push_back(k);
                last_cut = k;
            }
        }
        cut.push_back(n);
    }
    const uint32_t n_chunks = n ? (uint32_t)cut.size() - 1 : 0;
    struct Chunk {
        size_t act_base = 0, act_count = 0;  // this chunk's slice of the (column, active read) arrays
        uint32_t max_a = 0, max_d = 0;
        uint64_t base_total = 0, rc_total = 0;
        uint64_t words = 0, cells = 0, alg_bytes = 0;  // back-pointer words (column-kernel layout), DP cells, algorithmic bytes of the chunk
        std::vector<uint32_t> chain_starts;            // columns of this chunk that begin a DP-independent chain
        int rc = WHMEC_OK;
        uint32_t err_col = 0;
        std::string err;
    };
    std::vector<Chunk> chunks(n_chunks);
    std::vector<uint32_t> chunk_first_read(n_chunks + 1, p->n_reads);
    {
        uint32_t r = 0;
        for (uint32_t c = 0; c < n_chunks; ++c) {
            while (r < p->n_reads && first[r] < cut[c]) ++r;
            chunk_first_read[c] = r;
        }
    }
    pk.cols.resize(n);
    pk.act_off.resize(n + 1);
    pk.fn_group.resize((size_t)n * (T + 1));
    // a read is active in every column of its span: the (column, active read) arrays have exactly
    // sum(last - first + 1) entries, and a chunk's slice starts after the reads that precede it
    {
        size_t total = 0;
        uint32_t ci = 0;
        for (uint32_t r = 0; r < p->n_reads; ++r) {
            while (ci < n_chunks && chunk_first_read[ci] == r) chunks[ci++].act_base = total;
            total += (size_t)last[r] - first[r] + 1;
        }
        while (ci < n_chunks) chunks[ci++].act_base = total;
        pk.act_read.resize(total);
        pk.act_allele.resize(total);
        pk.act_phred.resize(total);
        pk.act_ind.resize(total);
    }

    // ---- pass 1: the allowed allele assignments of every (column, transmission value) depend on the genotypes only
    //      (pedigreecolumncostcomputer.cpp:14-50); counting them first gives every column its slice of the function
    //      arrays, so that the chunk workers write their results in place (no per-chunk buffers, no merge copy)
    const uint32_t n_asg = 1u << P;
    const uint32_t pack_threads = host_threads(32);
    std::vector<uint32_t> fn_off_of(n + 1, 0);
    // allow[t][i][g]: bit set over the assignments A under which individual i has genotype index g (columns only select)
    const uint32_t W = (n_asg + 63) / 64;
    std::vector<uint64_t> allow((size_t)T * p->n_ind * 3 * W, 0);
    for (uint32_t t = 0; t < T; ++t) {
        const int8_t *h2p = &pk.h2p[(size_t)t * p->n_ind * 2];
        for (uint32_t i = 0; i < p->n_ind; ++i)
            for (uint32_t A = 0; A < n_asg; ++A) {
                const uint32_t g = ((A >> h2p[2 * i]) & 1) + ((A >> h2p[2 * i + 1]) & 1);
                allow[(((size_t)t * p->n_ind + i) * 3 + g) * W + A / 64] |= 1ull << (A % 64);
            }
    }
    // allowed assignments of (column k, transmission value t) as a bit set in `out` (W words); returns their number
    auto allowed = [&](uint32_t k, uint32_t t, uint64_t *out) -> uint32_t {
        for (uint32_t w = 0; w < W; ++w) out[w] = ~0ull;
        if (n_asg < 64) out[0] = (1ull << n_asg) - 1;
        if (!p->distrust)
            for (uint32_t i = 0; i < p->n_ind; ++i) {
                const uint8_t g = p->gt[(size_t)i * n + k];
                for (uint32_t w = 0; w < W; ++w) out[w] &= g <= 2 ? allow[(((size_t)t * p->n_ind + i) * 3 + g) * W + w] : 0ull;
            }
        uint32_t count = 0;
        for (uint32_t w = 0; w < W; ++w) count += (uint32_t)__builtin_popcountll(out[w]);
        return count;
    };
    {
        const uint32_t n_tasks = n / 1024 + 1, step = (n + n_tasks - 1) / n_tasks;
        parallel_tasks(n_tasks, pack_threads, [&](uint32_t task) {
            uint64_t set[16];
            for (uint32_t k = task * step; k < std::min(n, (task + 1) * step); ++k) {
                uint32_t count = 0;
                for (uint32_t t = 0; t < T; ++t) {
                    pk.fn_group[(size_t)k * (T + 1) + t] = count;
                    count += allowed(k, t, set);
                }
                pk.fn_group[(size_t)k * (T + 1) + T] = count;
                fn_off_of[k + 1] = count;  // 0: Mendelian conflict, reported by the chunk worker in column order
            }
        });
        // one function per (transmission value, allowed assignment): with T = 1024 and distrusted genotypes a column can hold 2^20
        // of them (147 MB), so five-trio inputs are refused before the arrays are allocated
        uint64_t fn_count = 0;
        for (uint32_t k = 0; k < n; ++k) fn_count += fn_off_of[k + 1];
        const uint64_t fn_bytes = fn_count * (3 * 4 + (want_deltas ? FN_STRIDE * 4 : 0));
        if (T > MAX_T && fn_bytes > WIDE_FN_BYTES_MAX) {
            err = "unsupported: the cost functions of this five-trio pedigree need " + std::to_string(fn_bytes) + " bytes (at most " +
                  std::to_string(WIDE_FN_BYTES_MAX) + ")";
            return WHMEC_ERR_UNSUPPORTED;
        }
        for (uint32_t k = 0; k < n; ++k) fn_off_of[k + 1] += fn_off_of[k];
        const size_t fn_total = fn_off_of[n];
        pk.fn_c0.resize(fn_total);
        pk.fn_asg.resize(fn_total);
        pk.fn_base.resize(fn_total);
        pk.fn_delta.resize(want_deltas ? fn_total * FN_STRIDE : 0);
    }

    auto build_chunk = [&](uint32_t ci) {
        Chunk &ch = chunks[ci];
        const uint32_t kb = cut[ci], ke = cut[ci + 1];
        // active reads of the current column (ascending read index = bit order) and their entry cursors
        uint32_t active[MAX_ACTIVE];
        uint64_t cursor[MAX_ACTIVE];
        uint32_t na = 0;
        uint32_t next_read = chunk_first_read[ci];
        const uint32_t read_end = chunk_first_read[ci + 1];
        for (uint32_t k = kb; k < ke; ++k) {
            // reads that ended before k leave; the survivors are the reads shared with column k-1, which are
            // therefore the lowest bits (backward projection width, columnindexingscheme.cpp:62-85)
            uint32_t w = 0;
            for (uint32_t j = 0; j < na; ++j)
                if (last[active[j]] >= k) {
                    active[w] = active[j];
                    cursor[w] = cursor[j];
                    ++w;
                }
            na = w;
            while (next_read < read_end && first[next_read] == k) {
                if (na == MAX_ACTIVE) {
                    ch.rc = WHMEC_ERR_UNSUPPORTED;
                    ch.err_col = k;
                    ch.err = "more than 32 reads are active in one column (coverage too high)";
                    return;
                }
                active[na] = next_read;
                cursor[na] = p->read_off[next_read];
                ++na;
                ++next_read;
            }
            ColMeta &m = pk.cols[k];
            std::memset(&m, 0, sizeof m);
            m.a = na;
            ch.max_a = std::max(ch.max_a, m.a);
            m.rc = p->recombcost[k];
            m.first = (k == 0);
            m.bw = (k == 0) ? 0 : w;
            const size_t e0 = ch.act_base + ch.act_count;
            pk.act_off[k] = e0;
            uint32_t *a_read = pk.act_read.data() + e0, *a_phred = pk.act_phred.data() + e0;
            uint8_t *a_allele = pk.act_allele.data() + e0, *a_ind = pk.act_ind.data() + e0;
            uint32_t keep = 0;
            for (uint32_t j = 0; j < na; ++j) {
                const uint32_t r = active[j];
                uint64_t cur = cursor[j];
                while (p->ent_col[cur] < k) ++cur;
                cursor[j] = cur;
                a_read[j] = r;
                a_ind[j] = (uint8_t)p->read_ind[r];
                if (p->ent_col[cur] == k) {
                    a_allele[j] = p->ent_allele[cur];
                    a_phred[j] = p->ent_phred[cur];
                } else {  // gap inside the read's span: BLANK entry, phred 0 (columniterator.cpp:131)
                    a_allele[j] = 2;
                    a_phred[j] = 0;
                }
                if (k + 1 < n && last[r] >= k + 1) keep |= 1u << j;
            }
            ch.act_count += na;
            m.keep = keep;
            m.f = popc32(keep);
            m.d = m.a - m.f;
            ch.max_d = std::max(ch.max_d, m.d);
            {
                uint32_t di = 0;
                for (uint32_t drop = ~keep & low_mask(na); drop; drop &= drop - 1) m.dpos[di++] = (uint8_t)ctz32(drop);
            }

            // cost functions per (transmission value, allowed assignment), written to this column's slice
            m.fn_off = fn_off_of[k];
            m.grp_off = k * (T + 1);
            if (fn_off_of[k + 1] == fn_off_of[k]) {  // no transmission value admits any assignment: pedigreedptable.cpp:301-303
                ch.rc = WHMEC_ERR_MENDELIAN;
                ch.err_col = k;
                ch.err = "Error: Mendelian conflict";
                return;
            }
            uint32_t F = m.fn_off;
            uint32_t max_base = 0;
            for (uint32_t t = 0; t < T; ++t) {
                const int8_t *h2p = &pk.h2p[(size_t)t * p->n_ind * 2];
                // A read on haplotype 0 of its individual sits in partition h2p[ind][0] and costs its phred when
                // the allele assigned to that partition differs from the read's (cost computer :59-67): at x = 0
                // the cost of an assignment is a sum over partitions of S[partition][allele that differs].
                uint32_t S[MAX_P][2];
                for (uint32_t q = 0; q < P; ++q) S[q][0] = S[q][1] = 0;
                for (uint32_t j = 0; j < na; ++j)
                    if (a_allele[j] <= 1) S[h2p[2 * a_ind[j]]][a_allele[j] ^ 1] += a_phred[j];
                uint64_t set[16];
                allowed(k, t, set);
                for (uint32_t A = 0; A < n_asg; ++A) {
                    if (!((set[A / 64] >> (A % 64)) & 1)) continue;
                    unsigned int base = 0;
                    if (p->distrust)
                        for (uint32_t i = 0; i < p->n_ind; ++i) {
                            const uint32_t a0 = (A >> h2p[2 * i]) & 1, a1 = (A >> h2p[2 * i + 1]) & 1;
                            // pedigreecolumncostcomputer.cpp:37  `unsigned += double`
                            const double g = p->gl[((size_t)i * n + k) * 3 + (a0 + a1)];
                            base = (unsigned int)((double)base + g);
                        }
                    max_base = std::max(max_base, base);
                    uint32_t c0 = base;
                    for (uint32_t q = 0; q < P; ++q) c0 += S[q][(A >> q) & 1];
                    if (want_deltas) {
                        // moving read j to haplotype 1 changes the cost by (cost on partition h2p[ind][1]) - (cost on h2p[ind][0])
                        int32_t *delta = &pk.fn_delta[(size_t)F * FN_STRIDE];
                        std::memset(delta, 0, sizeof(int32_t) * FN_STRIDE);
                        for (uint32_t j = 0; j < na; ++j) {
                            const uint8_t al = a_allele[j];
                            if (al > 1) continue;  // BLANK contributes nothing
                            const uint32_t w2 = a_phred[j];
                            const uint32_t ind = a_ind[j];
                            const uint32_t cost0 = (((A >> h2p[2 * ind]) & 1) != al) ? w2 : 0;
                            const uint32_t cost1 = (((A >> h2p[2 * ind + 1]) & 1) != al) ? w2 : 0;
                            delta[j] = (int32_t)(cost1 - cost0);
                        }
                    }
                    pk.fn_c0[F] = c0;
                    pk.fn_asg[F] = A;
                    pk.fn_base[F] = base;
                    ++F;
                }
            }
            ch.base_total += max_base;
            ch.rc_total += (uint64_t)m.rc * pk.tb;
            // chains, back-pointer layout (chunk-relative until the chunks' sizes are known), accounting (SURVEY.md 8(d)).
            // A chunk starts at a chain boundary, so "the previous column forwards nothing" is decided inside the chunk.
            if (k == kb || pk.cols[k - 1].f == 0) ch.chain_starts.push_back(k);
            // the last column stores its winner too (f == 0); columns that drop many reads have few entries and
            // keep one word per entry (a thread block owns one entry there and writes its word alone)
            m.bp_width = m.d >= 8 ? 32 : round_bp_width(m.d + pk.tb);
            m.bp_off = ch.words;
            const uint64_t entries = ((uint64_t)1 << m.f) * T;
            ch.words += (entries * m.bp_width + 31) / 32;
            ch.cells += ((uint64_t)1 << m.a) * T;
            uint64_t bytes = (uint64_t)4 * T * ((uint64_t)1 << m.bw);
            if (k + 1 != n) bytes += (uint64_t)(8 + (T > 1 ? 4 : 0)) * T * ((uint64_t)1 << m.f);
            ch.alg_bytes += bytes;
        }
    };
    parallel_tasks(n_chunks, pack_threads, build_chunk);
    const auto t_chunks = tnow();
    // the reference reports the first failing column (columns are visited in order)
    for (uint32_t ci = 0; ci < n_chunks; ++ci)
        if (chunks[ci].rc != WHMEC_OK) {
            err = chunks[ci].err;
            return chunks[ci].rc;
        }
    uint32_t max_a = 0;
    uint64_t base_total = 0, rc_total = 0;
    for (uint32_t ci = 0; ci < n_chunks; ++ci) {
        max_a = std::max(max_a, chunks[ci].max_a);
        pk.max_d = std::max(pk.max_d, chunks[ci].max_d);
        base_total += chunks[ci].base_total;
        rc_total += chunks[ci].rc_total;
    }
    pk.act_off[n] = pk.act_read.size();
    pk.safe31 = (phred_total + base_total + rc_total) < (1ull << 28);
    pk.nowrap = (phred_total + base_total + rc_total) < UMAX;
    const auto t_merge = tnow();
    if (timing)
        std::fprintf(stderr, "[whmec] pack: validate %.2f ms, count + chunks(%u) %.2f ms, totals %.2f ms\n", tms(t_start, t_valid), n_chunks,
                     tms(t_valid, t_chunks), tms(t_chunks, t_merge));

    // ---- chains, back-pointer layout, accounting: per-chunk results, made absolute here
    uint64_t words = 0;
    whmec_stats &st = pk.stats;
    std::vector<uint64_t> word_base(n_chunks, 0);
    for (uint32_t ci = 0; ci < n_chunks; ++ci) {
        const Chunk &ch = chunks[ci];
        word_base[ci] = words;
        words += ch.words;
        st.cells += ch.cells;
        st.algorithmic_bytes += ch.alg_bytes;
        pk.chain_begin.insert(pk.chain_begin.end(), ch.chain_starts.begin(), ch.chain_starts.end());
    }
    const bool flush = stage_flush_enabled();
    parallel_tasks(n_chunks, pack_threads, [&](uint32_t ci) {
        if (word_base[ci])
            for (uint32_t k = cut[ci]; k < cut[ci + 1]; ++k) pk.cols[k].bp_off += word_base[ci];
        if (flush) stage_flush(&pk.cols[cut[ci]], (size_t)(cut[ci + 1] - cut[ci]) * sizeof(ColMeta));  // (hostpool.h: stage_flush)
    });
    pk.chain_begin.push_back(n);
    pk.bp_words = words;
    st.backptr_bytes = words * 4;
    st.n_chains = n ? (uint32_t)pk.chain_begin.size() - 1 : 0;
    st.max_active = max_a;
    st.transmissions = T;
    return WHMEC_OK;
}

int build_outputs(const Packed &pk, const uint32_t *path_index, const uint32_t *path_tv,
                  whmec_solution *s, std::string &err) {
    const uint32_t n = pk.n, P = pk.P;
    if (s->path_index && path_index != s->path_index) std::memcpy(s->path_index, path_index, sizeof(uint32_t) * n);
    if (s->path_tv && path_tv != s->path_tv) std::memcpy(s->path_tv, path_tv, sizeof(uint32_t) * n);
    // get_optimal_partitioning (pedigreedptable.cpp:391-406) + core.pyx:414: a read is reported in
    // partition 0 iff its bit is 0 in some column it is active in.
    // Column ranges are handled by independent host threads; a read that spans two ranges may be cleared by both
    // (same value, relaxed atomic byte stores).
    if (s->partition) std::memset(s->partition, 1, pk.n_reads);
    const bool want_superreads = s->sr_allele || s->sr_quality;
    if (!s->partition && !want_superreads) return WHMEC_OK;
    // get_super_reads -> get_alleles (pedigreecolumncostcomputer.cpp:117-175)
    std::atomic<int> failed{0};
    auto do_range = [&](uint32_t kb, uint32_t ke) {
    for (uint32_t k = kb; k < ke; ++k) {
        const ColMeta &m = pk.cols[k];
        const uint32_t t = path_tv[k], x = path_index[k];
        if (s->partition) {
            const uint32_t *reads = pk.act_read.data() + pk.act_off[k];
            for (uint32_t zero = ~x & low_mask(m.a); zero; zero &= zero - 1)
                __atomic_store_n(&s->partition[reads[ctz32(zero)]], (uint8_t)0, __ATOMIC_RELAXED);
        }
        if (!want_superreads) continue;
        const int8_t *h2p = &pk.h2p[(size_t)t * pk.n_ind * 2];
        uint32_t cp[MAX_P][2];
        for (uint32_t q = 0; q < P; ++q) cp[q][0] = cp[q][1] = 0;
        const uint64_t e0 = pk.act_off[k];
        for (uint32_t j = 0; j < m.a; ++j) {
            uint8_t al = pk.act_allele[e0 + j];
            if (al > 1) continue;
            int part = h2p[2 * pk.act_ind[e0 + j] + ((x >> j) & 1)];
            cp[part][al == 0 ? 1 : 0] += pk.act_phred[e0 + j];
        }
        uint32_t best = UMAX;
        uint32_t call[MAX_IND][2];
        uint32_t bfa[MAX_IND][2][2];
        for (uint32_t i = 0; i < pk.n_ind; ++i) {
            call[i][0] = call[i][1] = 2;
            bfa[i][0][0] = bfa[i][0][1] = bfa[i][1][0] = bfa[i][1][1] = UMAX;
        }
        const uint32_t g0 = m.fn_off + pk.fn_group[m.grp_off + t], g1 = m.fn_off + pk.fn_group[m.grp_off + t + 1];
        for (uint32_t F = g0; F < g1; ++F) {
            const uint32_t A = pk.fn_asg[F];
            uint32_t cost = pk.fn_base[F];
            for (uint32_t q = 0; q < P; ++q) cost += cp[q][(A >> q) & 1];
            bool new_best = false;
            if (cost <= best) {  // '<=': the LAST best assignment is reported (:131)
                best = cost;
                new_best = true;
            }
            for (uint32_t i = 0; i < pk.n_ind; ++i) {
                uint32_t a0 = (A >> h2p[2 * i]) & 1, a1 = (A >> h2p[2 * i + 1]) & 1;
                if (new_best) {
                    call[i][0] = a0;
                    call[i][1] = a1;
                }
                if (cost < bfa[i][0][a0]) bfa[i][0][a0] = cost;
                if (cost < bfa[i][1][a1]) bfa[i][1][a1] = cost;
            }
        }
        if (best == UMAX) {
            failed.store(1);
            return;
        }
        for (uint32_t i = 0; i < pk.n_ind; ++i) {
            uint32_t quality = 0;
            for (uint32_t h = 0; h < 2; ++h) {
                // (:162) abs((int)c0 - (int)c1): int casts (UMAX -> -1), two's-complement difference, magnitude
                const int32_t diff = (int32_t)(bfa[i][h][0] - bfa[i][h][1]);
                quality = diff < 0 ? 0u - (uint32_t)diff : (uint32_t)diff;
                if (quality == 0) call[i][h] = WHMEC_ALLELE_EQUAL_SCORES;
            }
            if (s->sr_allele) {
                s->sr_allele[((size_t)i * 2 + 0) * n + k] = (uint8_t)call[i][0];
                s->sr_allele[((size_t)i * 2 + 1) * n + k] = (uint8_t)call[i][1];
            }
            if (s->sr_quality) s->sr_quality[(size_t)i * n + k] = quality;
        }
    }
    };
    {
        const uint32_t n_ranges = std::min<uint32_t>(n / 1024 + 1, 64);
        const uint32_t step = (n + n_ranges - 1) / n_ranges;
        parallel_tasks(n_ranges, host_threads(16), [&](uint32_t t) { do_range(std::min(n, t * step), std::min(n, (t + 1) * step)); });
    }
    if (failed.load()) {
        err = "Error: Mendelian conflict";
        return WHMEC_ERR_MENDELIAN;
    }
    return WHMEC_OK;
}

}  // namespace whmec

extern "C" uint64_t whmec_read_sort_key(const char *name, size_t len, int32_t source_id) {
    // ReadSet::name_and_source_id_hasher_t (src/readset.h:68-72): libstdc++'s std::hash on both parts.
    return (uint64_t)(std::hash<std::string>()(std::string(name, len)) ^ std::hash<int>()((int)source_id));
}
