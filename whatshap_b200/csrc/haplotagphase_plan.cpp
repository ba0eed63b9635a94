// Votes of `whatshap haplotagphase` (whmec_haplotagphase, DESIGN §4.16): phase-set ranks, entry binning, chunk cut and entry
// gather on the host, and the C entry point.  The binning restates the read loop of compute_votes (whatshap/cli/
// haplotagphase.py) once per entry; the sums, the choice and the order are hp_run_votes' (haplotagphase.cu).
#include "haplotagphase_plan.h"

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

uint32_t bits_for(uint64_t max_value) {  // bits that hold 0 .. max_value
    uint32_t b = 0;
    while (b < 64 && (max_value >> b)) ++b;
    return b;
}

std::string check_csr(const uint64_t *off, uint64_t n, const void *a, const void *b) {
    if (!n) return std::string();
    if (!off) return "null offsets";
    if (off[0] != 0) return "offsets must start at 0";
    for (uint64_t i = 0; i < n; ++i)
        if (off[i + 1] < off[i]) return "offsets must not decrease";
    if (off[n] && (!a || !b)) return "null pair arrays";
    return std::string();
}

std::string check(const whmec_haplotagphase_input *in, const whmec_haplotagphase_output *out) {
    if (!in || !out || !in->pos_off || !out->voted_off || (in->n_samples && (!out->skipped || !out->entry_error || !out->entry_error_at)))
        return "null arguments";
    const uint32_t ns = in->n_samples;
    const uint64_t np = in->pos_off[ns];
    if (in->pos_off[0] != 0) return "pos_off must start at 0";
    if (np && (!in->pos || !in->pos_flags)) return "null positions";
    for (uint32_t s = 0; s < ns; ++s) {
        if (in->pos_off[s + 1] < in->pos_off[s]) return "pos_off must not decrease";
        for (uint64_t p = in->pos_off[s] + 1; p < in->pos_off[s + 1]; ++p)
            if (in->pos[p] <= in->pos[p - 1]) return "a sample's positions must ascend";
    }
    std::string bad = check_csr(in->a2i_off, np, in->a2i_allele, in->a2i_id);
    if (bad.empty()) bad = check_csr(in->i2a_off, np, in->i2a_id, in->i2a_allele);
    if (!bad.empty()) return "allele tables: " + bad;
    if (np && (!in->a2i_off || !in->i2a_off)) return "null allele tables";
    if (in->run_off) {
        if (in->n_reads) return "reads and runs in one call";
        const uint64_t nv = in->n_runs_pos;
        if (nv && (!in->runs_sample || !in->runs_pos)) return "null runs positions";
        bad = check_csr(in->run_off, nv, in->run_ps, in->run_h);
        if (!bad.empty()) return "runs: " + bad;
        if (nv && in->run_off[nv] && !in->run_score) return "null run scores";
        for (uint64_t v = 0; v < nv; ++v)
            if (in->runs_sample[v] >= ns || (v && in->runs_sample[v] < in->runs_sample[v - 1]))
                return "runs_sample must lie below n_samples and not decrease";
        return std::string();
    }
    const uint64_t nr = in->n_reads;
    if (nr && (!in->read_sample || !in->read_hp || !in->read_ps || !in->read_off)) return "null read arrays";
    if (nr && in->read_off[0] != 0) return "read_off must start at 0";
    for (uint64_t r = 0; r < nr; ++r) {
        if (in->read_off[r + 1] < in->read_off[r]) return "read_off must not decrease";
        if (in->read_sample[r] >= ns || (r && in->read_sample[r] < in->read_sample[r - 1]))
            return "read_sample must lie below n_samples and not decrease";
    }
    if (nr && in->read_off[nr] && (!in->entry_pos || !in->entry_allele || !in->entry_quality)) return "null entries";
    return std::string();
}

struct PosOut {                   // one voted position of a sample, before the samples' outputs are laid out
    uint64_t first;               // the ordinal of its first entry (vote form), its input index (runs form)
    uint64_t table;               // its table index
    HpChoice c;
    uint64_t rec0;                // its records in Sample::records
};

struct Sample {
    std::vector<PosOut> pos;
    std::vector<HpRecord> records;
    std::vector<int64_t> rank_id;  // phase-set rank -> PS_tag - 1
};

template <class T>
T *alloc(uint64_t n) {
    T *p = (T *)std::malloc(std::max<uint64_t>(n, 1) * sizeof(T));
    if (!p) throw std::bad_alloc();
    return p;
}

// The call's outputs from every sample's voted positions (and, in the vote form, their records).
void lay_out(std::vector<Sample> &samples, bool vote_form, whmec_haplotagphase_output *out) {
    uint64_t nv = 0, nk = 0;
    out->voted_off[0] = 0;
    for (size_t s = 0; s < samples.size(); ++s) {
        nv += samples[s].pos.size();
        nk += 2 * samples[s].records.size();
        out->voted_off[s + 1] = nv;
    }
    out->n_voted = nv;
    out->voted_pos = alloc<int64_t>(nv), out->phase_set = alloc<int64_t>(nv), out->haplotype = alloc<int64_t>(nv);
    out->score = alloc<int64_t>(nv), out->total = alloc<int64_t>(nv), out->allele = alloc<int64_t>(2 * nv);
    out->kept = alloc<uint8_t>(nv), out->error = alloc<int32_t>(nv);
    out->key_off = alloc<uint64_t>(nv + 1), out->key_ps = alloc<int64_t>(nk), out->key_score = alloc<int64_t>(nk);
    uint64_t v = 0, k = 0;
    out->key_off[0] = 0;
    for (Sample &S : samples) {
        for (const PosOut &p : S.pos) {
            const HpChoice &c = p.c;
            out->phase_set[v] = vote_form ? S.rank_id[c.ps] : c.ps;
            out->haplotype[v] = c.h, out->score[v] = c.score, out->total[v] = c.total;
            out->allele[2 * v] = c.allele0, out->allele[2 * v + 1] = c.allele1;
            out->kept[v] = c.kept, out->error[v] = c.error;
            for (uint64_t j = 0; vote_form && j < c.n_ps; ++j) {
                const HpRecord &r = S.records[p.rec0 + j];
                out->key_ps[k] = out->key_ps[k + 1] = S.rank_id[r.ps];
                out->key_score[k] = r.s0, out->key_score[k + 1] = r.s1;
                k += 2;
            }
            out->key_off[++v] = k;
        }
    }
}

int run_votes(const whmec_haplotagphase_input *in, int device, uint64_t cap, HpCall &call, std::vector<Sample> &samples,
              whmec_haplotagphase_output *out, std::string &msg) {
    const uint32_t ns = in->n_samples;
    std::vector<HpEntry> buf;
    std::vector<uint32_t> epos, count, chunk_of;
    std::vector<uint64_t> cstart;
    std::vector<int64_t> ids;
    uint64_t r0 = 0;
    for (uint32_t s = 0; s < ns; ++s) {
        const auto t0 = std::chrono::steady_clock::now();
        Sample &S = samples[s];
        uint64_t r1 = r0;
        while (r1 < in->n_reads && in->read_sample[r1] == s) ++r1;
        const uint64_t P0 = in->pos_off[s], P1 = in->pos_off[s + 1], np = P1 - P0;
        const uint64_t x0 = r0 < in->n_reads ? in->read_off[r0] : 0, x1 = r1 > r0 ? in->read_off[r1] : x0;
        // the counted reads (HP and PS at least 1, HP at most 2) and their phase sets' ranks
        uint64_t skipped = 0;
        ids.clear();
        for (uint64_t r = r0; r < r1; ++r) {
            const int64_t ht = in->read_hp[r] - 1, ps = in->read_ps[r] - 1;
            if (ht < 0 || ps < 0) continue;
            if (ht > 1) {
                ++skipped;
                continue;
            }
            ids.push_back(ps);
        }
        std::sort(ids.begin(), ids.end());
        ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
        S.rank_id = ids;
        out->skipped[s] = skipped;
        // bin the entries of counted reads at heterozygous positions; a position missing from the table is a KeyError
        uint64_t error = ~0ull;
        epos.assign(x1 - x0, UINT32_MAX);
        count.assign(np, 0);
        for (uint64_t r = r0; r < r1; ++r) {
            const int64_t ht = in->read_hp[r] - 1, ps = in->read_ps[r] - 1;
            if (ht < 0 || ps < 0 || ht > 1) continue;
            for (uint64_t x = in->read_off[r]; x < in->read_off[r + 1]; ++x) {
                const int64_t *it = std::lower_bound(in->pos + P0, in->pos + P1, in->entry_pos[x]);
                if (it == in->pos + P1 || *it != in->entry_pos[x]) {
                    error = std::min(error, hp_error_code(x, HP_KEY_POSITION));
                    continue;
                }
                const uint64_t p = (uint64_t)(it - in->pos);
                if (in->pos_flags[p] & HP_HOMOZYGOUS) continue;
                epos[x - x0] = (uint32_t)(p - P0);
                if (++count[p - P0] >= (1u << 31)) {
                    msg = "whmec_haplotagphase: a position has 2^31 entries or more";
                    return WHMEC_ERR_UNSUPPORTED;
                }
            }
        }
        const uint32_t ps_bits = bits_for(ids.empty() ? 0 : ids.size() - 1);
        // chunks of whole positions under the budget, fewer than 2^31 entries and 2^31 positions each
        chunk_of.assign(np, 0);
        cstart.assign(1, 0);
        uint64_t n_chunks = 0;
        for (uint64_t c0 = 0; c0 < np;) {
            uint64_t c1 = c0, ne = 0, bytes = 0;
            while (c1 < np) {
                const uint64_t b = count[c1] * HP_ENTRY_BYTES + HP_POS_BYTES;
                if (c1 > c0 && (bytes + b > cap || ne + count[c1] >= (1u << 31) || c1 - c0 >= (1u << 31) - 1)) break;
                bytes += b, ne += count[c1], chunk_of[c1] = (uint32_t)n_chunks, ++c1;
            }
            cstart.push_back(c1);
            ++n_chunks;
            c0 = c1;
        }
        // gather: the entries of each chunk in read order, chunk after chunk
        std::vector<uint64_t> eoff(n_chunks + 1, 0);
        for (uint64_t p = 0; p < np; ++p) eoff[chunk_of[p] + 1] += count[p];
        for (uint64_t c = 0; c < n_chunks; ++c) eoff[c + 1] += eoff[c];
        buf.resize(eoff[n_chunks]);
        {
            std::vector<uint64_t> fill(eoff.begin(), eoff.end() - 1);
            for (uint64_t r = r0; r < r1; ++r) {
                const int64_t ht = in->read_hp[r] - 1;
                if (ht < 0 || ht > 1 || in->read_ps[r] < 1) continue;
                const uint32_t rank = (uint32_t)(std::lower_bound(ids.begin(), ids.end(), in->read_ps[r] - 1) - ids.begin());
                for (uint64_t x = in->read_off[r]; x < in->read_off[r + 1]; ++x) {
                    const uint32_t lp = epos[x - x0];
                    if (lp == UINT32_MAX) continue;
                    const uint64_t c = chunk_of[lp];
                    buf[fill[c]++] = HpEntry{in->entry_allele[x], x, (uint32_t)(lp - cstart[c]), rank, in->entry_quality[x], (uint32_t)ht};
                }
            }
        }
        call.st.entries += buf.size();
        call.st.plan_ms += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
        for (uint64_t c = 0; c < n_chunks; ++c) {
            const auto t1 = std::chrono::steady_clock::now();
            call.p0 = P0 + cstart[c];
            call.n_cpos = (uint32_t)(cstart[c + 1] - cstart[c]);
            call.ps_bits = ps_bits;
            call.entries = buf.data() + eoff[c];
            call.n_entries = (uint32_t)(eoff[c + 1] - eoff[c]);
            call.pstart.assign(1, 0);
            for (uint64_t p = cstart[c]; p < cstart[c + 1]; ++p) call.pstart.push_back(call.pstart.back() + count[p]);
            call.st.plan_ms += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t1).count();
            if (!call.n_entries) continue;  // no position of the chunk voted
            ++call.st.chunks;
            int rc = hp_run_votes(device, call, msg);
            if (rc != WHMEC_OK) return rc;
            error = std::min(error, call.error);
            uint64_t rec = 0;
            for (uint32_t cp : call.order) {
                const HpChoice &ch = call.choice[cp];
                S.pos.push_back(PosOut{call.entries[ch.first].ordinal, call.p0 + cp, ch, S.records.size() + rec});
                rec += ch.n_ps;
            }
            S.records.insert(S.records.end(), call.records.begin(), call.records.end());
        }
        // chunks are cut by table position: their voted positions merge by first entry
        std::stable_sort(S.pos.begin(), S.pos.end(), [](const PosOut &a, const PosOut &b) { return a.first < b.first; });
        out->entry_error[s] = error == ~0ull ? 0 : (int32_t)(error & 3);
        out->entry_error_at[s] = error == ~0ull ? 0 : error >> 2;
        call.st.positions += S.pos.size();
        call.st.records += S.records.size();
        r0 = r1;
    }
    return WHMEC_OK;
}

int run_runs(const whmec_haplotagphase_input *in, int device, uint64_t cap, HpCall &call, std::vector<Sample> &samples,
             whmec_haplotagphase_output *out, std::string &msg) {
    const uint64_t nv = in->n_runs_pos;
    const auto t0 = std::chrono::steady_clock::now();
    std::vector<uint64_t> table(nv);
    for (uint64_t v = 0; v < nv; ++v) {
        const uint32_t s = in->runs_sample[v];
        const int64_t *a = in->pos + in->pos_off[s], *b = in->pos + in->pos_off[s + 1];
        const int64_t *it = std::lower_bound(a, b, in->runs_pos[v]);
        if (it == b || *it != in->runs_pos[v]) {
            msg = "whmec_haplotagphase: a runs position is missing from its sample's positions";
            return WHMEC_ERR_INPUT;
        }
        table[v] = (uint64_t)(it - in->pos);
    }
    for (uint32_t s = 0; s < in->n_samples; ++s) out->skipped[s] = 0, out->entry_error[s] = 0, out->entry_error_at[s] = 0;
    call.st.plan_ms += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
    call.run_ps = in->run_ps, call.run_h = in->run_h, call.run_score = in->run_score;
    for (uint64_t v0 = 0; v0 < nv;) {
        uint64_t v1 = v0, bytes = 0;
        while (v1 < nv) {
            const uint64_t b = (in->run_off[v1 + 1] - in->run_off[v1]) * HP_RUN_BYTES + HP_POS_BYTES;
            if (v1 > v0 && (bytes + b > cap || v1 - v0 >= (1u << 31) - 1)) break;
            bytes += b, ++v1;
        }
        call.n_cpos = (uint32_t)(v1 - v0);
        call.tpos.assign(table.begin() + v0, table.begin() + v1);
        call.roff.assign(in->run_off + v0, in->run_off + v1 + 1);
        ++call.st.chunks;
        int rc = hp_run_runs(device, call, msg);
        if (rc != WHMEC_OK) return rc;
        for (uint64_t v = v0; v < v1; ++v)
            samples[in->runs_sample[v]].pos.push_back(PosOut{v, table[v], call.choice[v - v0], 0});
        v0 = v1;
    }
    call.st.positions = nv;
    return WHMEC_OK;
}

}  // namespace

}  // namespace whmec

using namespace whmec;

extern "C" void whmec_haplotagphase_release(whmec_haplotagphase_output *out) {
    if (!out) return;
    for (void *p : {(void *)out->voted_pos, (void *)out->phase_set, (void *)out->haplotype, (void *)out->score, (void *)out->total,
                    (void *)out->allele, (void *)out->kept, (void *)out->error, (void *)out->key_off, (void *)out->key_ps,
                    (void *)out->key_score})
        std::free(p);
    out->voted_pos = out->phase_set = out->haplotype = out->score = out->total = out->allele = out->key_ps = out->key_score = nullptr;
    out->kept = nullptr, out->error = nullptr, out->key_off = nullptr, out->n_voted = 0;
}

extern "C" int whmec_haplotagphase(const whmec_haplotagphase_input *in, int device, whmec_haplotagphase_output *out,
                                   whmec_haplotagphase_stats *stats, char *err, size_t errlen) {
    const std::string bad = check(in, out);
    if (!bad.empty()) {
        put_err(err, errlen, "whmec_haplotagphase: " + bad);
        return WHMEC_ERR_INPUT;
    }
    out->n_voted = 0;
    out->voted_pos = out->phase_set = out->haplotype = out->score = out->total = out->allele = out->key_ps = out->key_score = nullptr;
    out->kept = nullptr, out->error = nullptr, out->key_off = nullptr;
    std::string msg;
    const uint64_t budget = hp_budget(device, msg);
    if (!msg.empty()) {
        put_err(err, errlen, msg);
        return WHMEC_ERR_CUDA;
    }
    HpCall call;
    try {
        const uint64_t np = in->pos_off[in->n_samples];
        call.n_pos = np;
        call.host = HpTable{in->pos_flags, in->a2i_off, in->a2i_allele, in->a2i_id, in->i2a_off, in->i2a_id, in->i2a_allele};
        call.gap = in->gap_threshold;
        call.only_indels = in->only_indels;
        const uint64_t n_a2i = np ? in->a2i_off[np] : 0, n_i2a = np ? in->i2a_off[np] : 0;
        // the position tables stay resident; chunks get the rest
        const uint64_t fixed = np * (1 + 2 * 8) + (n_a2i + n_i2a) * 16 + 64 * 256 + (1 << 20);
        const uint64_t cap = budget > fixed ? budget - fixed : 0;
        std::vector<Sample> samples(in->n_samples);
        const bool vote_form = in->run_off == nullptr;
        int rc = vote_form ? run_votes(in, device, cap, call, samples, out, msg) : run_runs(in, device, cap, call, samples, out, msg);
        hp_close(call);
        if (rc != WHMEC_OK) {
            put_err(err, errlen, msg);
            return rc;
        }
        lay_out(samples, vote_form, out);
        for (uint64_t v = 0, s = 0; s < samples.size(); ++s)
            for (const PosOut &p : samples[s].pos) out->voted_pos[v++] = in->pos[p.table];
        if (stats) *stats = call.st;
        return WHMEC_OK;
    } catch (const std::bad_alloc &) {
        hp_close(call);
        whmec_haplotagphase_release(out);
        put_err(err, errlen, "whmec_haplotagphase: out of host memory");
        return WHMEC_ERR_UNSUPPORTED;
    } catch (const std::exception &e) {  // nothing may cross the C boundary
        hp_close(call);
        whmec_haplotagphase_release(out);
        put_err(err, errlen, std::string("whmec_haplotagphase: ") + e.what());
        return WHMEC_ERR_UNSUPPORTED;
    }
}
