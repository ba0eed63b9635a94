// Allele detection from the CIGAR alone (whmec_detect_alleles_cigar, DESIGN §4.14): the host preparation, the chunk plan and the C
// entry point.  The preparation restates VcfVariant.normalized (whatshap/vcf.py:147-165, 226-242), detect_non_overlapping_variants and
// build_var_progress (whatshap/variants.py:550-597) once per call, and checks each alignment's operations; no base is read here.  The
// device work of a chunk is ca_run_chunk (cigar_alleles.cu).
#include "cigar_alleles_plan.h"

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <new>
#include <unordered_set>

namespace whmec {

namespace {

void put_err(char *err, size_t errlen, const std::string &msg) {
    if (err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = '\0';
    }
}

constexpr uint64_t CA_ALIGN = 256;
constexpr uint64_t CA_SCRATCH = 64 << 10;  // the count scan's scratch and the compaction's fixed scratch
constexpr int64_t I32_MIN = -(1ll << 31), I32_END = 1ll << 31;
uint64_t up(uint64_t b) { return (b + CA_ALIGN - 1) / CA_ALIGN * CA_ALIGN; }

bool in_i32(int64_t x) { return x >= I32_MIN && x < I32_END; }

}  // namespace

void ca_prepare(const whmec_realign_input &in, const whmec_query_qualities *q, CaPlan &plan) {
    const uint32_t nv = in.n_variants;
    const uint32_t threads = host_threads(32);
    // normalized(): `suf` bytes stripped from the end of every allele, then `pre` from the front, the position advanced by `pre`
    std::vector<uint64_t> pre(nv), suf(nv);
    auto len_of = [&](uint32_t slot) { return in.allele_off[slot + 1] - in.allele_off[slot]; };
    auto byte_of = [&](uint32_t slot, uint64_t i) { return in.allele_bytes[in.allele_off[slot] + i]; };
    const uint32_t n_tasks = std::max(1u, std::min(nv, threads * 8));
    parallel_tasks(n_tasks, threads, [&](uint32_t t) {
        for (uint32_t v = (uint32_t)((uint64_t)nv * t / n_tasks); v < (uint32_t)((uint64_t)nv * (t + 1) / n_tasks); ++v) {
            const uint32_t f0 = in.allele_first[v], f1 = in.allele_first[v + 1];
            const uint64_t rl = len_of(f0);
            uint64_t s = 0, p = 0;
            for (;; ++s) {  // while ref and all(alts) and all(ref[-1] == alt[-1] for alt in alts)
                bool go = s < rl;
                for (uint32_t k = f0 + 1; go && k < f1; ++k) go = len_of(k) > s && byte_of(k, len_of(k) - 1 - s) == byte_of(f0, rl - 1 - s);
                if (!go) break;
            }
            for (;; ++p) {  // while ref and all(alts) and all(ref[0] == alt[0] for alt in alts)
                bool go = p < rl - s;
                for (uint32_t k = f0 + 1; go && k < f1; ++k) go = len_of(k) - s > p && byte_of(k, p) == byte_of(f0, p);
                if (!go) break;
            }
            pre[v] = p, suf[v] = s;
        }
    });
    auto npos = [&](uint32_t v) { return (int64_t)in.position[v] + (int64_t)pre[v]; };
    auto nlen = [&](uint32_t slot, uint32_t v) { return (int64_t)(len_of(slot) - pre[v] - suf[v]); };
    // detect_non_overlapping_variants: the first of equal positions only; a deletion drops itself and the consecutive entries after it
    // that start inside it
    std::vector<uint8_t> conflicting(nv, 0);
    std::unordered_set<int64_t> seen;
    seen.reserve(nv);
    for (uint32_t j = 0; j < nv; ++j) {
        if (!seen.insert(npos(j)).second) {
            conflicting[j] = 1;
            continue;
        }
        const uint32_t f0 = in.allele_first[j], f1 = in.allele_first[j + 1];
        if (f1 == f0 + 1) {
            plan.err = "variant " + std::to_string(j) + " has no alternative allele (detect_non_overlapping_variants: max() of an empty "
                       "sequence raises ValueError)";
            return;
        }
        const int64_t ref = nlen(f0, j);
        int64_t max_del = INT64_MIN;
        for (uint32_t k = f0 + 1; k < f1; ++k) max_del = std::max(max_del, ref - nlen(k, j));
        if (max_del > 0) {
            const int64_t end = npos(j) + ref;
            if (j + 1 < nv && npos(j + 1) < end) {
                conflicting[j] = 1;
                while (j + 1 < nv && npos(j + 1) < end) conflicting[++j] = 1;
            }
        }
    }
    // build_var_progress over the conflict-free variants, in list order
    for (uint32_t v = 0; v < nv; ++v) {
        if (conflicting[v]) continue;
        if (!in_i32(npos(v))) {
            plan.err = "variant " + std::to_string(v) + ": the normalized position leaves the 32-bit range of the reference's C ints";
            return;
        }
        const uint32_t f0 = in.allele_first[v], f1 = in.allele_first[v + 1];
        const int64_t rl = nlen(f0, v);
        if (rl >= I32_END) {
            plan.err = "variant " + std::to_string(v) + ": the reference allele is longer than 2^31 - 1";
            return;
        }
        plan.vars.push_back(CaVar{(int32_t)npos(v), (int32_t)rl, v, (uint32_t)plan.alleles.size()});
        plan.alleles.push_back(CaAllele{in.allele_off[f0] + pre[v], (int32_t)rl, 0, 0, 0});
        for (uint32_t k = f0 + 1; k < f1; ++k) {
            const int64_t al = nlen(k, v);
            if (al >= I32_END) {
                plan.err = "variant " + std::to_string(v) + ": an alternative allele is longer than 2^31 - 1";
                return;
            }
            plan.alleles.push_back(CaAllele{in.allele_off[k] + pre[v], (int32_t)std::min(rl, al), (int32_t)std::max<int64_t>(0, al - rl),
                                            (int32_t)std::max<int64_t>(0, rl - al), 0});
        }
        if (plan.alleles.size() >= UMAX) {
            plan.err = "more than 2^32 - 1 alleles of conflict-free variants in one call";
            return;
        }
    }
    const uint32_t n_vars = (uint32_t)plan.vars.size();
    plan.vars.push_back(CaVar{0, 0, UMAX, (uint32_t)plan.alleles.size()});
    // the skip loop from j = 0 stops at the first variant at or after reference_start: a search over the prefix maxima
    std::vector<int32_t> pmax(n_vars);
    int32_t vmin = 0;
    for (uint32_t j = 0; j < n_vars; ++j) {
        pmax[j] = j ? std::max(pmax[j - 1], plan.vars[j].pos) : plan.vars[j].pos;
        vmin = j ? std::min(vmin, plan.vars[j].pos) : plan.vars[j].pos;
    }
    // the alignments: operations up to the first unknown one, C int ranges, first variant
    const uint32_t na = in.n_alignments;
    plan.alns.resize(na);
    const uint32_t a_tasks = std::max(1u, std::min(na, threads * 8));
    std::vector<uint32_t> bad(a_tasks, UMAX), refused(a_tasks, UMAX);
    std::vector<std::string> bad_msg(a_tasks), refused_msg(a_tasks);
    parallel_tasks(a_tasks, threads, [&](uint32_t t) {
        for (uint32_t a = (uint32_t)((uint64_t)na * t / a_tasks); a < (uint32_t)((uint64_t)na * (t + 1) / a_tasks); ++a) {
            const uint8_t missing = q && q->missing ? q->missing[a] : 0;
            const uint64_t c0 = in.cigar_off[a], c1 = missing & 2 ? c0 : in.cigar_off[a + 1];
            uint64_t n_ops = c1 - c0;
            if (missing & 2) {
                if (bad[t] == UMAX) bad[t] = a, bad_msg[t] = "TypeError ('NoneType' object is not iterable: cigartuples is None)";
            }
            for (uint64_t i = 0; i < c1 - c0; ++i)
                if (in.cigar_op[c0 + i] > 8) {
                    n_ops = i;
                    if (bad[t] == UMAX) bad[t] = a, bad_msg[t] = "ValueError (Unsupported CIGAR operation: " + std::to_string(in.cigar_op[c0 + i]) + ")";
                    break;
                }
            const uint64_t q_len = in.query_off[a + 1] - in.query_off[a];
            const uint64_t qual_len = q ? q->qual_off[a + 1] - q->qual_off[a] : 0;
            // the reference's ref_pos, ref_end, query_pos and query_start are C ints
            int64_t r = in.reference_start[a], qp = 0, rmin = r, rmax = r, qmin = 0, qmax = 0;
            bool ok = n_ops < UMAX && q_len < (uint64_t)I32_END && qual_len < (uint64_t)I32_END;
            for (uint64_t i = 0; ok && i < n_ops; ++i) {
                const int op = in.cigar_op[c0 + i];
                const int64_t len = in.cigar_len[c0 + i];
                if (op != 4 && op != 5 && op != 6) rmin = std::min(rmin, r + len), rmax = std::max(rmax, r + len);
                if (op == 0 || op == 7 || op == 8 || op == 1 || op == 4) qp += len;
                if (op == 0 || op == 7 || op == 8 || op == 2 || op == 3) r += len;
                rmin = std::min(rmin, r), rmax = std::max(rmax, r), qmin = std::min(qmin, qp), qmax = std::max(qmax, qp);
                ok = in_i32(r) && in_i32(qp) && in_i32(rmin) && in_i32(rmax);
            }
            ok = ok && in_i32(qmax + (rmax - rmin)) && (n_vars == 0 || in_i32(qmin + (int64_t)vmin - rmax));
            if (!ok && refused[t] == UMAX) {
                refused[t] = a;
                refused_msg[t] = "alignment " + std::to_string(a) + ": positions, lengths or spans leave the 32-bit range of the reference's C ints";
            }
            const uint32_t j0 = (uint32_t)(std::lower_bound(pmax.begin(), pmax.end(), in.reference_start[a]) - pmax.begin());
            plan.alns[a] = CaAln{c0, in.query_off[a], q ? q->qual_off[a] : 0, (uint32_t)n_ops, (uint32_t)q_len, (uint32_t)qual_len,
                                 in.reference_start[a], j0, (uint32_t)(missing & 1)};
        }
    });
    for (uint32_t t = 0; t < a_tasks; ++t)
        if (refused[t] != UMAX) {
            plan.err = refused_msg[t];
            return;
        }
    for (uint32_t t = 0; t < a_tasks; ++t)
        if (bad[t] != UMAX) {
            plan.first_bad = bad[t];
            plan.bad_msg = bad_msg[t];
            break;
        }
}

uint64_t ca_chunk_bytes(const CaChunk &c) {
    const uint64_t na = c.a1 - c.a0, nops = c.op_hi - c.op_lo;
    return up(na * sizeof(CaAln)) + 2 * up((na + 1) * 8) + up(nops) + up(nops * 4) + up(c.q_hi - c.q_lo) + up(c.qual_hi - c.qual_lo) + CA_SCRATCH;
}

std::vector<CaChunk> ca_chunks(const CaPlan &plan, const whmec_realign_input &in, const whmec_query_qualities *q, uint64_t budget) {
    std::vector<CaChunk> out;
    const uint32_t na = in.n_alignments;
    CaChunk c;
    for (uint32_t a = 0; a < na; ++a) {
        const CaAln &A = plan.alns[a];
        const uint64_t q1 = A.q0 + A.q_len, qual1 = A.qual0 + A.qual_len, op1 = A.op0 + A.n_ops;
        CaChunk g = c;
        g.a1 = a + 1;
        g.op_lo = std::min(g.op_lo, A.op0), g.op_hi = std::max(g.op_hi, op1);
        g.q_lo = std::min(g.q_lo, A.q0), g.q_hi = std::max(g.q_hi, q1);
        g.qual_lo = std::min(g.qual_lo, A.qual0), g.qual_hi = std::max(g.qual_hi, qual1);
        if (c.a1 == c.a0 || ca_chunk_bytes(g) > budget / 2) {
            if (c.a1 > c.a0) out.push_back(c);
            g = CaChunk{a, a + 1, A.op0, op1, A.q0, q1, A.qual0, qual1, 0};
        }
        g.bytes = ca_chunk_bytes(g);
        c = g;
    }
    if (c.a1 > c.a0) out.push_back(c);
    return out;
}

uint64_t ca_window(const CaChunk &c, uint64_t budget) { return budget > c.bytes ? std::max<uint64_t>(1, (budget - c.bytes) / CA_ITEM_BYTES) : 1; }

}  // namespace whmec

using namespace whmec;

extern "C" int whmec_detect_alleles_cigar(const whmec_realign_input *in, const whmec_query_qualities *q, int device, whmec_realign_output *out,
                                          whmec_realign_stats *stats, char *err, size_t errlen) {
    if (!in || !out || (in->n_alignments && (!in->reference_start || !in->cigar_off || !in->query_off)) ||
        (in->n_alignments && in->cigar_off[in->n_alignments] && (!in->cigar_op || !in->cigar_len)) ||
        (in->n_variants && (!in->position || !in->allele_first || !in->allele_off)) || (q && in->n_alignments && !q->qual_off)) {
        put_err(err, errlen, "whmec_detect_alleles_cigar: null or malformed arguments");
        return WHMEC_ERR_INPUT;
    }
    std::memset(out, 0, sizeof(*out));
    for (uint32_t v = 0; v < in->n_variants; ++v)
        if (in->allele_first[v + 1] <= in->allele_first[v]) {
            put_err(err, errlen, "whmec_detect_alleles_cigar: variant " + std::to_string(v) + " has no reference allele");
            return WHMEC_ERR_INPUT;
        }
    std::string msg;
    uint64_t budget = ca_budget(device, msg);  // (first: selects the device and the page-locked staging memory)
    if (!msg.empty()) {
        put_err(err, errlen, msg);
        return WHMEC_ERR_CUDA;
    }
    try {
        const auto t0 = std::chrono::steady_clock::now();
        CaPlan plan;
        ca_prepare(*in, q, plan);
        if (!plan.err.empty()) {
            put_err(err, errlen, plan.err);
            return WHMEC_ERR_INPUT;
        }
        CaRun run;
        run.plan = &plan, run.in = in, run.q = q;
        const uint64_t n_bytes = in->n_variants ? in->allele_off[in->allele_first[in->n_variants]] : 0;
        const uint64_t fixed = up(plan.vars.size() * sizeof(CaVar)) + up(plan.alleles.size() * sizeof(CaAllele)) + up(n_bytes) + 2 * CA_ALIGN;
        run.budget = budget > fixed ? budget - fixed : 0;
        const std::vector<CaChunk> chunks = ca_chunks(plan, *in, q, run.budget);
        run.st.plan_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
        int rc = WHMEC_OK;
        for (const CaChunk &c : chunks) {
            if (std::min(plan.first_bad, run.raised) < c.a0) break;  // the first raising alignment is known
            if ((rc = ca_run_chunk(device, run, c, msg)) != WHMEC_OK) break;
        }
        ca_close(run);
        if (rc != WHMEC_OK) {
            put_err(err, errlen, msg);
            return rc;
        }
        const uint32_t first = std::min(plan.first_bad, run.raised);
        if (first != UMAX) {
            std::string why = plan.bad_msg;
            if (run.raised <= plan.first_bad)  // a handler raised before the op loop reached the unknown operation
                why = plan.alns[first].missing ? "TypeError ('NoneType' object is not subscriptable: query_sequence is None)"
                                               : "IndexError (a base or quality index past the end of query_sequence or query_qualities)";
            put_err(err, errlen, "alignment " + std::to_string(first) + ": the reference raises " + why);
            return WHMEC_ERR_INPUT;
        }
        const uint64_t n_calls = run.calls.size();
        out->call_off = (uint64_t *)std::malloc((in->n_alignments + 1) * sizeof(uint64_t));
        out->variant = (uint32_t *)std::malloc(std::max<uint64_t>(n_calls, 1) * sizeof(uint32_t));
        out->allele = (int32_t *)std::malloc(std::max<uint64_t>(n_calls, 1) * sizeof(int32_t));
        out->quality = (int64_t *)std::malloc(std::max<uint64_t>(n_calls, 1) * sizeof(int64_t));
        if (!out->call_off || !out->variant || !out->allele || !out->quality) throw std::bad_alloc();
        uint64_t w = 0;
        out->call_off[0] = 0;
        for (uint32_t a = 0; a < in->n_alignments; ++a) {
            for (; w < n_calls && run.calls[w].alignment == a; ++w) {
                out->variant[w] = run.calls[w].variant;
                out->allele[w] = run.calls[w].allele;
                out->quality[w] = run.calls[w].quality;
            }
            out->call_off[a + 1] = w;
        }
        run.st.cells = n_calls;
        run.st.short_jobs = run.st.jobs;
        if (stats) *stats = run.st;
        return WHMEC_OK;
    } catch (const std::bad_alloc &) {
        whmec_realign_release(out);
        put_err(err, errlen, "whmec_detect_alleles_cigar: out of host memory");
        return WHMEC_ERR_UNSUPPORTED;
    }
}
