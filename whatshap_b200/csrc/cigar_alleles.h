// Allele detection from the CIGAR alone (whmec_detect_alleles_cigar, `--no-reference`, DESIGN §4.14): the per-thread code shared by
// the kernels of cigar_alleles.cu and the host emulation (tests/emul/emul_cigar_alleles.cpp), and the records the host plan of
// cigar_alleles_plan.cpp builds.
//
// The reference is whatshap/_variants.pyx:84-298 (_detect_alleles and its three handlers).  Its op loop enqueues a conflict-free
// variant when the variant starts within an operation's reference span; every enqueued variant then runs the handler of each later
// M, I, D, = and X operation until none of its alleles is pending.  Per allele, "resolved" (progress == length) and "failed" (-1)
// are absorbing under all three handlers, so an allele's outcome depends only on its variant's enqueue point and the operations
// after it; the queue only fixes the output order, which is the enqueue order filtered by the final state.  Hence:
//   ca_walk     one alignment's op loop and enqueue rules: the items (alignment, variant, operation, query positions), in enqueue order;
//   ca_resolve  one item: the three handlers over each allele from the item's operation on, then the call (or none).
#pragma once
#include <stdint.h>

#include "common.h"

namespace whmec {

constexpr int32_t CA_NO_QUAL = 30;  // the quality of a base without query_qualities, of an inserted or deleted base, of an empty allele

// One alignment as the kernels see it.
struct CaAln {
    uint64_t op0;        // first CIGAR operation in the call's cigar arrays
    uint64_t q0, qual0;  // first query byte, first quality byte
    uint32_t n_ops;      // operations the op loop reaches before the reference raises: up to the first unknown operation, else all
    uint32_t q_len;      // len(query_sequence)
    uint32_t qual_len;   // len(query_qualities); 0: quality 30 per base
    int32_t ref_start;
    uint32_t j0;         // the first conflict-free variant the skip loop stops at (with `first` = 0)
    uint32_t missing;    // 1: query_sequence is None (reading a base raises TypeError)
};

// A conflict-free variant, in list order; entry n_vars is a sentinel whose `first` ends the last variant's alleles.
struct CaVar {
    int32_t pos;      // normalized position
    int32_t ref_len;  // len(normalized reference allele)
    uint32_t id;      // index into the caller's variant list
    uint32_t first;   // its alleles are CaAllele slots first .. next.first - 1, reference allele first
};

// One allele of a conflict-free variant (build_var_progress): its normalized bytes and its three targets.
struct CaAllele {
    uint64_t off;  // first byte in the call's allele bytes
    int32_t match, ins, del;
    int32_t pad;
};

// One enqueued variant (the reference's var_progress[j].reset(query_start); vqueue.append(...)).
struct CaItem {
    uint32_t aln;    // index into the chunk's alignments
    uint32_t var;    // index into the conflict-free variants
    uint32_t op;     // the operation at which it was enqueued
    int32_t qpos;    // query_pos at that operation
    int32_t qstart;  // query_start
};

// An item's outcome: allele -1 for no call.
struct CaCall {
    uint32_t alignment;  // index into the call's alignments
    uint32_t variant;    // index into the caller's variant list
    int32_t allele;
    int32_t pad;
    int64_t quality;
};

// Where a chunk's slices live: CIGAR operation op0 of an alignment is op[op0 - op_lo], its query bytes q[q0 - q_lo ..], its
// qualities qual[qual0 - qual_lo ..].
struct CaBufs {
    const uint8_t *op;
    const int32_t *len;
    uint64_t op_lo;
    const uint8_t *q;
    uint64_t q_lo;
    const uint8_t *qual;
    uint64_t qual_lo;
    const CaAln *alns;
    const CaVar *vars;
    uint32_t n_vars;
    const CaAllele *alleles;
    const uint8_t *ab;
};

// The op loop of _detect_alleles (_variants.pyx:109-166) for alignment `a`: emit(item) for every enqueued variant, in order.
template <class Emit>
WHMEC_HD void ca_walk(const CaBufs &b, uint32_t a, Emit &emit) {
    const CaAln A = b.alns[a];
    const uint8_t *ops = b.op + (A.op0 - b.op_lo);
    const int32_t *lens = b.len + (A.op0 - b.op_lo);
    int64_t ref_pos = A.ref_start, qp = 0;
    uint32_t j = A.j0;
    for (uint32_t i = 0; i < A.n_ops; ++i) {
        const int op = ops[i];
        const int64_t len = lens[i];
        while (j < b.n_vars && b.vars[j].pos < ref_pos) ++j;  // the skip loop runs first at every operation
        if (op == 3) {
            ref_pos += len;
            continue;
        }
        if (op == 4) {
            qp += len;
            continue;
        }
        if (op == 5 || op == 6) continue;
        const int64_t ref_end = ref_pos + len;
        for (; j < b.n_vars && b.vars[j].pos < ref_end; ++j) {
            const CaVar v = b.vars[j];
            if (op == 1 && v.ref_len > 0) break;     // an insertion in front of a non-insertion variant
            if (op == 2 && v.ref_len == 0) continue;  // a deletion skips an insertion variant for good
            emit(CaItem{a, j, i, (int32_t)qp, (int32_t)(op != 2 ? qp + v.pos - ref_pos : qp)});
        }
        if (op != 2) qp += len;       // M, =, X, I
        if (op != 1) ref_pos += len;  // M, =, X, D
    }
}

// Python's s[i] on a sequence of length n (missing: s is None): false where it raises.
WHMEC_HD bool ca_index(int64_t i, int64_t n, bool missing, int64_t &x) {
    if (missing || i < -n || i >= n) return false;
    x = i < 0 ? i + n : i;
    return true;
}

// One item (_variants.pyx:168-222, 224-298): returns false where the reference raises (a base or quality index out of range, or a
// missing query sequence) at one of the item's operations; else allele is the call (-1: none) with its quality.  n_alleles: the
// variant's allele count.
WHMEC_HD bool ca_resolve(const CaBufs &b, const CaItem &it, int32_t &allele, int64_t &quality, uint32_t &n_alleles) {
    const CaAln A = b.alns[it.aln];
    const uint8_t *ops = b.op + (A.op0 - b.op_lo);
    const int32_t *lens = b.len + (A.op0 - b.op_lo);
    const uint8_t *q = b.q + (A.q0 - b.q_lo), *ql = b.qual + (A.qual0 - b.qual_lo);
    const int64_t n = A.q_len, nq = A.qual_len;
    const uint32_t k0 = b.vars[it.var].first, k1 = b.vars[it.var + 1].first;
    n_alleles = k1 - k0;
    allele = -1;
    quality = 0;
    int64_t best_len = -1;
    bool pending = false;
    for (uint32_t k = k0; k < k1; ++k) {
        const CaAllele al = b.alleles[k];
        const uint8_t *s = b.ab + al.off;
        const int64_t L = (int64_t)al.match + al.ins + al.del;
        int64_t progress = 0, matched = 0, inserted = 0, deleted = 0, qsum = 0, qp = it.qpos;
        for (uint32_t i = it.op; progress >= 0 && progress < L && i < A.n_ops; ++i) {
            const int op = ops[i];
            const int64_t len = lens[i];
            if (op == 0 || op == 7 || op == 8) {  // _detect_alleles_match: every step reads the same query base
                int64_t consumed = it.qstart - qp > 0 ? it.qstart - qp : 0, x, y;
                const int64_t base = it.qstart + matched + inserted;
                while (matched < al.match && consumed < len) {
                    if (!ca_index(base, n, A.missing, x)) return false;
                    if (q[x] != s[matched + inserted]) break;
                    ++consumed;
                    if (nq) {
                        if (!ca_index(base, nq, false, y)) return false;
                        qsum += ql[y];
                    } else {
                        qsum += CA_NO_QUAL;
                    }
                    ++matched, ++progress;
                }
                if (consumed < len && progress < L) progress = -1;
                qp += len;
            } else if (op == 1) {  // _detect_alleles_insertion
                int64_t consumed = 0, x;
                while (inserted < al.ins && consumed < len) {
                    ++consumed;
                    if (!ca_index(it.qstart + matched + inserted, n, A.missing, x)) return false;
                    if (q[x] != s[matched + inserted]) break;
                    ++inserted, ++progress;
                    qsum += CA_NO_QUAL;
                }
                if (consumed < len && 0 < progress && progress < L) progress = -1;
                qp += len;
            } else if (op == 2) {  // _detect_alleles_deletion
                const int64_t consumed = len > 0 ? (al.del - deleted < len ? al.del - deleted : len) : 0;
                deleted += consumed, progress += consumed;
                qsum += CA_NO_QUAL * consumed;
                if (consumed < len && progress < L) progress = -1;
            } else if (op == 4) {
                qp += len;
            }
        }
        if (progress >= 0 && progress < L) {
            pending = true;
        } else if (progress == L && L > best_len) {  // the first longest resolved allele
            best_len = L;
            allele = (int32_t)(k - k0);
            quality = L > 0 ? qsum / L : CA_NO_QUAL;
        }
    }
    if (pending) allele = -1;
    return true;
}

// Walk visitors: count an alignment's items; write those with index in [lo, hi) of the chunk (k: the alignment's first index).
struct CaCount {
    uint32_t n = 0;
    WHMEC_HD void operator()(const CaItem &) { ++n; }
};
struct CaEmit {
    CaItem *out;
    uint64_t k, lo, hi;
    WHMEC_HD void operator()(const CaItem &it) {
        if (k >= lo && k < hi) out[k - lo] = it;
        ++k;
    }
};

}  // namespace whmec
