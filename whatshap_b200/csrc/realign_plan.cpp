// Allele detection by re-alignment (whmec_realign, DESIGN §4.11; k-mer mode, §4.12): the host walk, the chunk plan and the C
// entry points.  The walk restates whatshap/_variants.pyx:10-81 (_iterate_cigar) and the window steps of ReadSetReader.realign
// (whatshap/variants.py:599-682, 724-831) for one alignment; the device work of a chunk is ra_run_chunk (realign.cu).
#include "realign_plan.h"

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <new>

namespace whmec {

namespace {

void put_err(char *err, size_t errlen, const std::string &msg) {
    if (err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = '\0';
    }
}

// Python's s[lo:hi] on a sequence of length n: first byte and length
void py_slice(int64_t lo, int64_t hi, int64_t n, int64_t &first, int64_t &len) {
    auto norm = [n](int64_t x) {
        if (x < 0) x = std::max<int64_t>(x + n, 0);
        return std::min(x, n);
    };
    first = norm(lo);
    len = std::max<int64_t>(norm(hi) - first, 0);
}

struct CigarView {
    const uint8_t *op;
    const int32_t *len;
    uint32_t n;
};

// ReadSetReader.cigar_prefix_length over split_cigar_left (left) or split_cigar_right (!left) at (i, consumed).
bool prefix_length(const CigarView &cg, bool left, uint32_t i, int64_t consumed, int64_t want, int64_t &ref_bases, int64_t &query_bases,
                   std::string &why) {
    const bool mid = left ? consumed > 0 : consumed < cg.len[i];
    const uint32_t count = (uint32_t)mid + (left ? i : cg.n - i - 1);
    int64_t rp = 0, qp = 0;
    for (uint32_t k = 0; k < count; ++k) {
        int op;
        int64_t length;
        if (k == 0 && mid) {
            op = cg.op[i];
            length = left ? consumed : cg.len[i] - consumed;
        } else {
            const uint32_t e = left ? i - 1 - (k - mid) : i + 1 + (k - mid);
            op = cg.op[e];
            length = cg.len[e];
        }
        if (op == 0 || op == 7 || op == 8) {
            rp += length;
            qp += length;
            if (rp >= want) {
                ref_bases = want, query_bases = qp + want - rp;
                return true;
            }
        } else if (op == 2) {
            rp += length;
            if (rp >= want) {
                ref_bases = want, query_bases = qp;
                return true;
            }
        } else if (op == 1) {
            qp += length;
        } else if (op == 4 || op == 5) {
        } else if (op == 3) {
            ref_bases = want, query_bases = qp;
            return true;
        } else {
            why = "unknown CIGAR operator " + std::to_string(op) + " in the window (cigar_prefix_length)";
            return false;
        }
    }
    if (!(rp < want)) {
        why = "the window's CIGAR covers no reference base (cigar_prefix_length: assert ref_pos < reference_bases)";
        return false;
    }
    ref_bases = rp, query_bases = qp;
    return true;
}

uint64_t allele_len(const whmec_realign_input &in, uint32_t v, uint32_t a) {
    const uint32_t slot = in.allele_first[v] + a;
    return in.allele_off[slot + 1] - in.allele_off[slot];
}

constexpr uint64_t RA_ALIGN = 256;
uint64_t up(uint64_t b) { return (b + RA_ALIGN - 1) / RA_ALIGN * RA_ALIGN; }

}  // namespace

uint64_t ra_job_need(uint64_t q_len, uint64_t target_len, int affine) {
    if (affine) return q_len <= RA_SHORT ? RA_NO_SCRATCH : (3 * (q_len + 1) * sizeof(float) + 15) / 16 * 16;
    return std::min(q_len, target_len) <= RA_SHORT ? RA_NO_SCRATCH : (std::max(q_len, target_len) + 15) / 16 * 16;
}

uint64_t ka_job_need(uint64_t q_len, uint64_t target_len) {
    return q_len <= KA_SHORT && target_len <= KA_SHORT ? RA_NO_SCRATCH : ka_scratch_bytes(q_len, target_len);
}

bool ra_walk_alignment(const whmec_realign_input &in, uint32_t a, std::vector<RaItem> &items, std::vector<RaJob> &jobs, std::string &err,
                       const whmec_kmerald_params *km) {
    const uint64_t c0 = in.cigar_off[a], c1 = in.cigar_off[a + 1];
    if (c1 == c0) return true;  // `if not cigartuples: return`
    const CigarView cg{in.cigar_op + c0, in.cigar_len + c0, (uint32_t)(c1 - c0)};
    const int64_t qlen = (int64_t)(in.query_off[a + 1] - in.query_off[a]);
    const uint32_t n = in.n_variants;
    auto fail = [&](int64_t var, const std::string &why) {
        err = "alignment " + std::to_string(a) + (var >= 0 ? ", variant " + std::to_string(var) : std::string()) + ": " + why;
        return false;
    };
    // realign() for variant `index`, split at (i, consumed), query position qpos
    auto emit = [&](uint32_t index, uint32_t i, int64_t consumed, int64_t qpos) {
        const uint32_t n_alleles = in.allele_first[index + 1] - in.allele_first[index];
        for (uint32_t k = 1; k < n_alleles; ++k)
            if (allele_len(in, index, k) > 0 && in.allele_bytes[in.allele_off[in.allele_first[index] + k]] == '<') return true;  // symbolic
        const int64_t ref_len = (int64_t)allele_len(in, index, 0);
        int64_t lr, lq, rr, rq;
        std::string why;
        const int64_t window = km ? km->window : in.overhang;
        if (!prefix_length(cg, true, i, consumed, window, lr, lq, why)) return fail(index, why);
        if (!prefix_length(cg, false, i, consumed, ref_len + window, rr, rq, why)) return fail(index, why);
        const int64_t pos = in.position[index];
        if (!(pos - lr >= 0)) return fail(index, "the window starts before the reference (assert variant.position - left_ref_bases >= 0)");
        if (!(pos + rr <= (int64_t)in.reference_len))
            return fail(index, "the window ends after the reference (assert variant.position + right_ref_bases <= len(reference))");
        if (km && !km->has_alt[index]) return fail(index, "the variant has no alternative_allele (a multiallelic variant: the reference raises AttributeError)");
        RaItem it{};
        int64_t qfirst, qn;
        py_slice(qpos - lq, qpos + rq, qlen, qfirst, qn);
        it.q = in.query_off[a] + (uint64_t)qfirst;
        it.q_len = (uint32_t)qn;
        it.r = pos - lr;
        it.left = (uint32_t)lr;
        it.right = (uint32_t)rr;
        it.ref_len = (uint32_t)ref_len;
        it.variant = index;
        it.alignment = a;
        it.job0 = (uint32_t)jobs.size();
        const uint32_t item = (uint32_t)items.size();
        if (km) {  // allele 0 and alternative_allele, which the k-mer call reads as slot 2 * index + 1 (whmec_realign_kmerald)
            const uint64_t alt_len = km->alt_off[index + 1] - km->alt_off[index];
            jobs.push_back(RaJob{item, 0, ka_job_need(it.q_len, lr + rr)});
            jobs.push_back(RaJob{item, 1, ka_job_need(it.q_len, lr + alt_len + (uint64_t)std::max<int64_t>(rr - ref_len, 0))});
        }
        for (uint32_t k = 0; k < n_alleles && !km; ++k) {
            if (in.restrict_off) {
                const int32_t *g0 = in.restrict_allele + in.restrict_off[index], *g1 = in.restrict_allele + in.restrict_off[index + 1];
                if (std::find(g0, g1, (int32_t)k) == g1) continue;
            }
            const uint64_t tl = k == 0 ? lr + rr : lr + allele_len(in, index, k) + (uint64_t)std::max<int64_t>(rr - ref_len, 0);
            jobs.push_back(RaJob{item, k, ra_job_need(it.q_len, tl, in.affine)});
        }
        it.n_jobs = (uint32_t)jobs.size() - it.job0;
        if (it.n_jobs == 0) return fail(index, "no allele is left after the restricted genotype (the reference's distance list is empty)");
        items.push_back(it);
        return true;
    };
    int64_t ref_pos = in.reference_start[a], query_pos = 0, v = 0;
    uint32_t j = 0;
    while (j < n && in.position[j] < ref_pos) ++j;
    for (uint32_t i = 0; i < cg.n; ++i) {
        const int op = cg.op[i];
        const int64_t length = cg.len[i];
        if (j < n) v = in.position[j];
        if (op == 0 || op == 7 || op == 8 || op == 2) {
            while (j < n && v < ref_pos + length) {
                if (!(v >= ref_pos)) return fail(j, "variants out of order (assert v_position >= ref_pos)");
                if (!emit(j, i, v - ref_pos, op == 2 ? query_pos : query_pos + v - ref_pos)) return false;
                if (++j < n) v = in.position[j];
            }
            if (op != 2) query_pos += length;
            ref_pos += length;
        } else if (op == 1) {
            if (j < n && v == ref_pos) {
                if (!emit(j, i, 0, query_pos)) return false;
                if (++j < n) v = in.position[j];
            }
            query_pos += length;
        } else if (op == 3) {
            while (j < n && v < ref_pos + length) {
                if (!(v >= ref_pos)) return fail(j, "variants out of order (assert v_position >= ref_pos)");
                if (++j < n) v = in.position[j];
            }
            ref_pos += length;
        } else if (op == 4) {
            query_pos += length;
        } else if (op == 5 || op == 6) {
        } else {
            return fail(-1, "Unsupported CIGAR operation: " + std::to_string(op));
        }
    }
    return true;
}

void ra_plan(const whmec_realign_input &in, RaPlan &plan, const whmec_kmerald_params *km) {
    const uint32_t n = in.n_alignments;
    const uint32_t threads = host_threads(32);
    const uint32_t n_tasks = std::max(1u, std::min(n, threads * 8));
    std::vector<std::vector<RaItem>> items(n_tasks);
    std::vector<std::vector<RaJob>> jobs(n_tasks);
    std::vector<std::string> errs(n_tasks);
    std::vector<std::vector<uint64_t>> counts(n_tasks);
    parallel_tasks(n_tasks, threads, [&](uint32_t t) {
        const uint32_t a0 = (uint32_t)((uint64_t)n * t / n_tasks), a1 = (uint32_t)((uint64_t)n * (t + 1) / n_tasks);
        for (uint32_t a = a0; a < a1; ++a) {
            if (!ra_walk_alignment(in, a, items[t], jobs[t], errs[t], km)) return;
            counts[t].push_back(items[t].size());
        }
    });
    for (uint32_t t = 0; t < n_tasks; ++t)
        if (!errs[t].empty()) {  // the first failing alignment, as the reference meets it
            plan.err = errs[t];
            return;
        }
    std::vector<uint64_t> ibase(n_tasks + 1, 0), jbase(n_tasks + 1, 0);
    for (uint32_t t = 0; t < n_tasks; ++t) ibase[t + 1] = ibase[t] + items[t].size(), jbase[t + 1] = jbase[t] + jobs[t].size();
    if (ibase[n_tasks] >= (1ull << 32) || jbase[n_tasks] >= (1ull << 32)) {
        plan.err = "more than 2^32 - 1 items or allele alignments in one call: hand the alignments over in slices";
        return;
    }
    plan.items.resize(ibase[n_tasks]);
    plan.jobs.resize(jbase[n_tasks]);
    plan.item_off.assign(n + 1, 0);
    std::vector<uint64_t> cells(n_tasks, 0);
    parallel_tasks(n_tasks, threads, [&](uint32_t t) {
        const uint32_t a0 = (uint32_t)((uint64_t)n * t / n_tasks);
        for (size_t k = 0; k < counts[t].size(); ++k) plan.item_off[a0 + k + 1] = ibase[t] + counts[t][k];
        for (size_t k = 0; k < items[t].size(); ++k) {
            RaItem it = items[t][k];
            it.job0 += (uint32_t)jbase[t];
            plan.items[ibase[t] + k] = it;
        }
        for (size_t k = 0; k < jobs[t].size(); ++k) {
            RaJob jb = jobs[t][k];
            const RaItem &it = items[t][jb.item];
            jb.item += (uint32_t)ibase[t];
            plan.jobs[jbase[t] + k] = jb;
            cells[t] += (uint64_t)it.q_len * (it.left + it.right);
        }
    });
    for (uint64_t c : cells) plan.cells += c;
}

uint64_t ra_chunk_bytes(const RaChunk &c) {
    const uint64_t ni = c.item1 - c.item0, nj = c.job1 - c.job0;
    return up(ni * sizeof(RaItem)) + up(nj * sizeof(RaJob)) + up(nj * 4) /* warp job list */ + up(nj * 8) + up(nj) + up(ni * 4) + up(ni * 8) +
           up(c.q_hi - c.q_lo) + up((uint64_t)(c.r_hi - c.r_lo)) + up(c.scratch);
}

std::vector<RaChunk> ra_chunks(const RaItem *items, uint32_t n_items, RaJob *jobs, uint64_t budget) {
    std::vector<RaChunk> out;
    RaChunk c;
    bool open = false;
    for (uint32_t i = 0; i < n_items; ++i) {
        const RaItem &it = items[i];
        uint64_t need = 0;
        for (uint32_t k = it.job0; k < it.job0 + it.n_jobs; ++k)
            if (jobs[k].scratch != RA_NO_SCRATCH) need += jobs[k].scratch;
        RaChunk g = c;
        if (open) {
            g.item1 = i + 1;
            g.job1 = it.job0 + it.n_jobs;
            g.q_lo = std::min(g.q_lo, it.q), g.q_hi = std::max(g.q_hi, it.q + it.q_len);
            g.r_lo = std::min(g.r_lo, it.r), g.r_hi = std::max(g.r_hi, it.r + (int64_t)(it.left + it.right));
            g.scratch += need;
        }
        if (!open || ra_chunk_bytes(g) > budget) {
            if (open) {
                c.bytes = ra_chunk_bytes(c);
                out.push_back(c);
            }
            g = RaChunk{i, i + 1, it.job0, it.job0 + it.n_jobs, it.q, it.q + it.q_len, it.r, it.r + (int64_t)(it.left + it.right), need, 0};
            open = true;
        }
        uint64_t off = g.scratch - need;
        for (uint32_t k = it.job0; k < it.job0 + it.n_jobs; ++k)
            if (jobs[k].scratch != RA_NO_SCRATCH) {
                const uint64_t b = jobs[k].scratch;
                jobs[k].scratch = off;
                off += b;
            }
        c = g;
    }
    if (open) {
        c.bytes = ra_chunk_bytes(c);
        out.push_back(c);
    }
    return out;
}

namespace {

// Runs every chunk of `call`'s items and jobs; `fixed`: device bytes the call holds besides its chunks.
int run_chunks(int device, RaCall &call, uint32_t n_items, RaJob *jobs, uint64_t budget, uint64_t fixed, std::string &msg) {
    budget = budget > fixed ? budget - fixed : 0;
    const std::vector<RaChunk> chunks = ra_chunks(call.items, n_items, jobs, budget);
    call.st.chunks = (uint32_t)chunks.size();
    int rc = WHMEC_OK;
    for (const RaChunk &c : chunks)
        if ((rc = ra_run_chunk(device, call, c, msg)) != WHMEC_OK) break;
    ra_close(call);
    return rc;
}

void count_jobs(RaCall &call, uint32_t n_items, const RaJob *jobs) {
    for (uint32_t i = 0; i < n_items; ++i) {
        const RaItem &it = call.items[i];
        bool any = false;
        for (uint32_t k = it.job0; k < it.job0 + it.n_jobs; ++k) {
            const bool lng = jobs[k].scratch != RA_NO_SCRATCH;
            any |= lng;
            ++(lng ? call.st.long_jobs : call.st.short_jobs);
        }
        call.st.long_items += any;
        call.st.jobs += it.n_jobs;
    }
    call.st.items = n_items;
}

}  // namespace

}  // namespace whmec

using namespace whmec;

namespace {

// The checks of a k-mer mode's parameters (name: the entry point), empty when they pass.
std::string ka_check(const whmec_kmerald_params *km, uint32_t n_variants, bool alts, const char *name) {
    if (!km || !km->costs || km->kmer_size < 1 || km->kmer_size > 15 || km->window < 0 ||
        (alts && n_variants && (!km->alt_off || !km->has_alt)))
        return std::string(name) + ": null or malformed k-mer parameters (kmer_size 1..15, window >= 0)";
    const whmec_kmer_costs &c = *km->costs;
    if (c.n >= (1ull << 32) || (c.n && (!c.key || !c.cost))) return std::string(name) + ": null or oversized costs table (n < 2^32)";
    for (uint64_t i = 1; i < c.n; ++i)
        if (c.key[i] <= c.key[i - 1]) return std::string(name) + ": the costs' keys are not strictly ascending at entry " + std::to_string(i);
    return std::string();
}

KaParams ka_params(const whmec_kmerald_params &km) {
    return KaParams{(uint32_t)km.kmer_size, km.gap_penalty, km.costs->key, km.costs->cost, (uint32_t)km.costs->n};
}

// whmec_realign (km == NULL) and whmec_realign_kmerald, after their argument checks
int realign_call(const whmec_realign_input *in, const whmec_kmerald_params *km, int device, whmec_realign_output *out,
                 whmec_realign_stats *stats, char *err, size_t errlen) {
    std::memset(out, 0, sizeof(*out));
    for (uint32_t v = 0; v < in->n_variants; ++v)
        if (in->allele_first[v + 1] <= in->allele_first[v]) {
            put_err(err, errlen, "whmec_realign: variant " + std::to_string(v) + " has no reference allele");
            return WHMEC_ERR_INPUT;
        }
    std::string msg;
    const uint64_t budget = ra_budget(device, msg);  // (first: selects the device and the page-locked staging memory)
    if (!msg.empty()) {
        put_err(err, errlen, msg);
        return WHMEC_ERR_CUDA;
    }
    try {
        const auto t0 = std::chrono::steady_clock::now();
        RaPlan plan;
        ra_plan(*in, plan, km);
        if (!plan.err.empty()) {
            put_err(err, errlen, plan.err);
            return WHMEC_ERR_INPUT;
        }
        const uint32_t ni = (uint32_t)plan.items.size(), nj = (uint32_t)plan.jobs.size();
        RaCall call;
        call.host = RaBufs{in->query, 0, in->reference, 0, in->allele_bytes, in->allele_off, in->allele_first};
        call.n_alleles = in->n_variants ? in->allele_first[in->n_variants] : 0;
        call.n_variants = in->n_variants;
        call.ref_len = in->reference_len;
        call.params = RaParams{in->affine, (float)in->mismatch, in->gap_start, in->gap_extend};
        call.items = plan.items.data();
        call.jobs = plan.jobs.data();
        // k-mer mode: the device's allele slots are, per variant v, an empty slot 2v and alternative_allele as slot 2v + 1, so
        // that ra_target reads allele 1 of variant v as alternative_allele
        std::vector<uint64_t> slot_off;
        std::vector<uint32_t> slot_first;
        if (km) {
            const uint32_t nv = in->n_variants;
            slot_off.resize(2 * (uint64_t)nv + 1);
            slot_first.resize((uint64_t)nv + 1);
            slot_off[0] = 0;
            for (uint32_t v = 0; v < nv; ++v) {
                slot_first[v] = 2 * v;
                slot_off[2 * v + 1] = km->alt_off[v];
                slot_off[2 * v + 2] = km->alt_off[v + 1];
            }
            slot_first[nv] = 2 * nv;
            if (nv) slot_off[0] = km->alt_off[0];
            call.host = RaBufs{in->query, 0, in->reference, 0, km->alt_bytes, slot_off.data(), slot_first.data()};
            call.n_alleles = 2 * (uint64_t)nv;
            call.kmerald = true;
            call.kparams = ka_params(*km);
        }
        RawVec<int64_t> dist(nj), quality(ni);
        RawVec<int32_t> called(ni);
        std::vector<uint8_t> status(nj, 0);
        call.dist = dist.data(), call.status = status.data(), call.call = called.data(), call.quality = quality.data();
        count_jobs(call, ni, plan.jobs.data());
        call.st.cells = plan.cells;
        call.st.plan_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
        const uint64_t fixed = 3 * RA_ALIGN + (call.n_alleles + 1) * 8 + (uint64_t)(in->n_variants + 1) * 4 +
                               (call.n_alleles ? call.host.al_off[call.n_alleles] : 0) +
                               (km ? 2 * RA_ALIGN + (uint64_t)call.kparams.n * 12 : 0);
        int rc = ni ? run_chunks(device, call, ni, plan.jobs.data(), budget, fixed, msg) : WHMEC_OK;
        if (rc != WHMEC_OK) {
            put_err(err, errlen, msg);
            return rc;
        }
        for (uint32_t k = 0; k < nj; ++k)
            if (status[k]) {
                const RaItem &it = plan.items[plan.jobs[k].item];
                put_err(err, errlen, "alignment " + std::to_string(it.alignment) + ", variant " + std::to_string(it.variant) +
                                         ": the affine distance is not finite or beyond int64 (int() of the reference raises)");
                return WHMEC_ERR_INPUT;
            }
        uint64_t n_calls = 0;
        for (uint32_t i = 0; i < ni; ++i) n_calls += called[i] >= 0;
        out->call_off = (uint64_t *)std::malloc((in->n_alignments + 1) * sizeof(uint64_t));
        out->variant = (uint32_t *)std::malloc(std::max<uint64_t>(n_calls, 1) * sizeof(uint32_t));
        out->allele = (int32_t *)std::malloc(std::max<uint64_t>(n_calls, 1) * sizeof(int32_t));
        out->quality = (int64_t *)std::malloc(std::max<uint64_t>(n_calls, 1) * sizeof(int64_t));
        if (!out->call_off || !out->variant || !out->allele || !out->quality) throw std::bad_alloc();
        uint64_t w = 0;
        out->call_off[0] = 0;
        for (uint32_t a = 0; a < in->n_alignments; ++a) {
            for (uint64_t i = plan.item_off[a]; i < plan.item_off[a + 1]; ++i)
                if (called[i] >= 0) {
                    const RaItem &it = plan.items[i];
                    out->variant[w] = it.variant;
                    out->allele[w] = (int32_t)plan.jobs[it.job0 + called[i]].allele;
                    out->quality[w] = quality[i];
                    ++w;
                }
            out->call_off[a + 1] = w;
        }
        if (stats) *stats = call.st;
        return WHMEC_OK;
    } catch (const std::bad_alloc &) {
        whmec_realign_release(out);
        put_err(err, errlen, "whmec_realign: out of host memory");
        return WHMEC_ERR_UNSUPPORTED;
    }
}

}  // namespace

extern "C" int whmec_realign(const whmec_realign_input *in, int device, whmec_realign_output *out, whmec_realign_stats *stats, char *err,
                             size_t errlen) {
    if (!in || !out || (in->n_alignments && (!in->reference_start || !in->cigar_off || !in->query_off)) ||
        (in->n_variants && (!in->position || !in->allele_first || !in->allele_off)) || in->overhang < 0 ||
        (in->affine != 0 && in->affine != 1)) {
        put_err(err, errlen, "whmec_realign: null or malformed arguments");
        return WHMEC_ERR_INPUT;
    }
    return realign_call(in, nullptr, device, out, stats, err, errlen);
}

extern "C" int whmec_realign_kmerald(const whmec_realign_input *in, const whmec_kmerald_params *params, int device, whmec_realign_output *out,
                                     whmec_realign_stats *stats, char *err, size_t errlen) {
    if (!in || !out || (in->n_alignments && (!in->reference_start || !in->cigar_off || !in->query_off)) ||
        (in->n_variants && (!in->position || !in->allele_first || !in->allele_off))) {
        put_err(err, errlen, "whmec_realign_kmerald: null or malformed arguments");
        return WHMEC_ERR_INPUT;
    }
    const std::string bad = ka_check(params, in->n_variants, true, "whmec_realign_kmerald");
    if (!bad.empty()) {
        put_err(err, errlen, bad);
        return WHMEC_ERR_INPUT;
    }
    return realign_call(in, params, device, out, stats, err, errlen);
}

extern "C" void whmec_realign_release(whmec_realign_output *out) {
    if (!out) return;
    std::free(out->call_off);
    std::free(out->variant);
    std::free(out->allele);
    std::free(out->quality);
    std::memset(out, 0, sizeof(*out));
}

extern "C" int whmec_edit_distance_batch(uint32_t n, const uint64_t *query_off, const uint8_t *query, const uint64_t *target_off,
                                         const uint8_t *target, double mismatch, int32_t gap_start, int32_t gap_extend, int64_t *unit_out,
                                         int64_t *affine_out, int device, whmec_realign_stats *stats, char *err, size_t errlen) {
    if (n && (!query_off || !target_off)) {
        put_err(err, errlen, "whmec_edit_distance_batch: null arguments");
        return WHMEC_ERR_INPUT;
    }
    std::string msg;
    const uint64_t budget = ra_budget(device, msg);
    if (!msg.empty()) {
        put_err(err, errlen, msg);
        return WHMEC_ERR_CUDA;
    }
    try {
        whmec_realign_stats total{};
        for (int affine = 0; affine < 2; ++affine) {
            int64_t *dst = affine ? affine_out : unit_out;
            if (!dst || !n) continue;
            StagedVec<RaItem> items(n);
            StagedVec<RaJob> jobs(n);
            uint64_t cells = 0;
            for (uint32_t i = 0; i < n; ++i) {
                // a pair is an item whose "reference" window is the target and whose only allele is allele 0
                const uint64_t ql = query_off[i + 1] - query_off[i], tl = target_off[i + 1] - target_off[i];
                if (ql >= (1ull << 31) || tl >= (1ull << 31)) {
                    put_err(err, errlen, "whmec_edit_distance_batch: pair " + std::to_string(i) + " is longer than 2^31 - 1");
                    return WHMEC_ERR_INPUT;
                }
                items[i] = RaItem{query_off[i], (int64_t)target_off[i], (uint32_t)ql, (uint32_t)tl, 0, 0, 0, i, 1, i};
                jobs[i] = RaJob{i, 0, ra_job_need(ql, tl, affine)};
                cells += ql * tl;
            }
            RaCall call;
            call.host = RaBufs{query, 0, target, 0, nullptr, nullptr, nullptr};
            call.params = RaParams{affine, (float)mismatch, gap_start, gap_extend};
            call.decide = false;
            call.items = items.data();
            call.jobs = jobs.data();
            std::vector<uint8_t> status(n, 0);
            call.dist = dst, call.status = status.data();
            count_jobs(call, n, jobs.data());
            call.st.cells = cells;
            const int rc = run_chunks(device, call, n, jobs.data(), budget, 0, msg);
            if (rc != WHMEC_OK) {
                put_err(err, errlen, msg);
                return rc;
            }
            for (uint32_t i = 0; i < n; ++i)
                if (status[i]) {
                    put_err(err, errlen, "pair " + std::to_string(i) + ": the affine distance is not finite or beyond int64");
                    return WHMEC_ERR_INPUT;
                }
            total.items += call.st.items, total.jobs += call.st.jobs, total.short_jobs += call.st.short_jobs;
            total.long_jobs += call.st.long_jobs, total.long_items += call.st.long_items, total.cells += call.st.cells;
            total.h2d_bytes += call.st.h2d_bytes, total.d2h_bytes += call.st.d2h_bytes, total.chunks += call.st.chunks;
            total.kernel_launches += call.st.kernel_launches, total.device_ms += call.st.device_ms;
        }
        if (stats) *stats = total;
        return WHMEC_OK;
    } catch (const std::bad_alloc &) {
        put_err(err, errlen, "whmec_edit_distance_batch: out of host memory");
        return WHMEC_ERR_UNSUPPORTED;
    }
}

extern "C" int whmec_kmer_align_batch(uint32_t n, const uint64_t *s1_off, const uint8_t *s1, const uint64_t *s2_off, const uint8_t *s2,
                                      const whmec_kmerald_params *params, float *out, int device, whmec_realign_stats *stats, char *err,
                                      size_t errlen) {
    if (n && (!s1_off || !s2_off || !out)) {
        put_err(err, errlen, "whmec_kmer_align_batch: null arguments");
        return WHMEC_ERR_INPUT;
    }
    const std::string bad = ka_check(params, 0, false, "whmec_kmer_align_batch");
    if (!bad.empty()) {
        put_err(err, errlen, bad);
        return WHMEC_ERR_INPUT;
    }
    std::string msg;
    const uint64_t budget = ra_budget(device, msg);
    if (!msg.empty()) {
        put_err(err, errlen, msg);
        return WHMEC_ERR_CUDA;
    }
    try {
        StagedVec<RaItem> items(n);
        StagedVec<RaJob> jobs(n);
        uint64_t cells = 0;
        for (uint32_t i = 0; i < n; ++i) {
            // a pair is an item whose query is s2 (the columns) and whose allele 0 ("reference" window) is s1 (the rows)
            const uint64_t l1 = s1_off[i + 1] - s1_off[i], l2 = s2_off[i + 1] - s2_off[i];
            if (l1 >= (1ull << 31) || l2 >= (1ull << 31)) {
                put_err(err, errlen, "whmec_kmer_align_batch: pair " + std::to_string(i) + " is longer than 2^31 - 1");
                return WHMEC_ERR_INPUT;
            }
            items[i] = RaItem{s2_off[i], (int64_t)s1_off[i], (uint32_t)l2, (uint32_t)l1, 0, 0, 0, i, 1, i};
            jobs[i] = RaJob{i, 0, ka_job_need(l2, l1)};
            cells += l1 * l2;
        }
        RaCall call;
        call.host = RaBufs{s2, 0, s1, 0, nullptr, nullptr, nullptr};
        call.decide = false;
        call.kmerald = true;
        call.kparams = ka_params(*params);
        call.items = items.data();
        call.jobs = jobs.data();
        std::vector<uint8_t> status(n, 0);
        call.kdist = out, call.status = status.data();
        count_jobs(call, n, jobs.data());
        call.st.cells = cells;
        const int rc = n ? run_chunks(device, call, n, jobs.data(), budget, 2 * RA_ALIGN + (uint64_t)call.kparams.n * 12, msg) : WHMEC_OK;
        if (rc != WHMEC_OK) {
            put_err(err, errlen, msg);
            return rc;
        }
        if (stats) *stats = call.st;
        return WHMEC_OK;
    } catch (const std::bad_alloc &) {
        put_err(err, errlen, "whmec_kmer_align_batch: out of host memory");
        return WHMEC_ERR_UNSUPPORTED;
    }
}
