// Read assignment of `whatshap haplotag` (whmec_haplotag, DESIGN §4.15): the group walk, block ranks, chunk cut and entry gather
// on the host, and the C entry point.  The walk restates the grouping loop of prepare_haplotag_information (whatshap/cli/
// haplotag.py) once per read; the per-entry sums are ht_run_chunk's (haplotag.cu).
#include "haplotag_plan.h"

#include <algorithm>
#include <chrono>
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

std::string check(const whmec_haplotag_input *in, const whmec_haplotag_output *out) {
    if (!in || !out || !in->phase_off) return "null arguments";
    const uint32_t ns = in->n_samples, nr = in->n_reads;
    const uint64_t np = in->phase_off[ns];
    if (np && (!in->phase_pos || !in->phase_block || !in->allele_off)) return "null phase table";
    if (in->allele_off && in->allele_off[np] && !in->allele) return "null phase alleles";
    if (nr && (!in->read_off || !in->read_sample || !in->read_repr || !in->read_bx || !in->reference_start || !out->group ||
               !out->n_blocks || !out->block || !out->haplotype || !out->quality))
        return "null read arrays";
    if (nr && in->read_off[nr] && (!in->entry_pos || !in->entry_allele || !in->entry_quality)) return "null entries";
    if (nr >= (1u << 31)) return "more than 2^31 - 1 reads";
    if (in->phase_off[0] != 0) return "phase_off must start at 0";
    for (uint32_t s = 0; s < ns; ++s) {
        if (in->phase_off[s + 1] < in->phase_off[s]) return "phase_off must not decrease";
        for (uint64_t p = in->phase_off[s] + 1; p < in->phase_off[s + 1]; ++p)
            if (in->phase_pos[p] <= in->phase_pos[p - 1]) return "a sample's phase positions must ascend";
    }
    if (np && in->allele_off[0] != 0) return "allele_off must start at 0";
    for (uint64_t p = 0; p < np; ++p)
        if (in->allele_off[p + 1] < in->allele_off[p]) return "allele_off must not decrease";
    if (nr && in->read_off[0] != 0) return "read_off must start at 0";
    for (uint32_t r = 0; r < nr; ++r) {
        if (in->read_off[r + 1] < in->read_off[r]) return "read_off must not decrease";
        if (in->read_sample[r] >= ns || (r && in->read_sample[r] < in->read_sample[r - 1]))
            return "read_sample must lie below n_samples and not decrease";
        if (in->read_repr[r] < 0 || in->read_bx[r] < -1) return "negative representation or BX id";
    }
    return std::string();
}

struct Groups {
    std::vector<uint32_t> opener;     // per group
    std::vector<uint64_t> moff;       // [groups + 1] into members
    std::vector<uint32_t> members;    // the groups' reads in visit order
    std::vector<uint64_t> mstart;     // [members + 1]: call-wide ordinal of each member's first entry
};

// The reference's grouping loop, sample by sample: out->group of every read, and the groups with their members in visit order.
void walk(const whmec_haplotag_input &in, int64_t *group, Groups &g) {
    const uint32_t nr = in.n_reads;
    int64_t max_repr = -1, max_bx = -1;
    for (uint32_t r = 0; r < nr; ++r) max_repr = std::max(max_repr, in.read_repr[r]), max_bx = std::max(max_bx, in.read_bx[r]);
    std::vector<uint32_t> processed((size_t)(max_repr + 1), 0);  // the stamp (sample + 1) that processed a representation
    std::vector<uint32_t> bx_first((size_t)(max_bx + 1), 0), bx_stamp((size_t)(max_bx + 1), 0), bx_next(nr, UINT32_MAX);
    std::vector<uint32_t> bx_last((size_t)(max_bx + 1), 0);
    std::vector<uint32_t> members;
    g.moff.push_back(0);
    g.mstart.push_back(0);
    uint64_t ordinal = 0;
    for (uint32_t r0 = 0; r0 < nr;) {
        uint32_t r1 = r0;
        while (r1 < nr && in.read_sample[r1] == in.read_sample[r0]) ++r1;
        const uint32_t stamp = in.read_sample[r0] + 1;
        for (uint32_t r = r0; r < r1; ++r) {  // this sample's reads of each BX id, in read order
            const int64_t b = in.read_bx[r];
            if (b < 0) continue;
            if (bx_stamp[b] != stamp) bx_stamp[b] = stamp, bx_first[b] = r;
            else bx_next[bx_last[b]] = r;
            bx_last[b] = r;
        }
        for (uint32_t r = r0; r < r1; ++r) group[r] = -1;
        for (uint32_t r = r0; r < r1; ++r) {
            if (processed[in.read_repr[r]] == stamp) continue;
            processed[in.read_repr[r]] = stamp;
            members.assign(1, r);
            const int64_t b = in.read_bx[r];
            if (b >= 0) {
                const int64_t s = in.reference_start[r];
                for (uint32_t m = bx_first[b]; m != UINT32_MAX; m = bx_next[m]) {
                    const int64_t t = in.reference_start[m];
                    const uint64_t d = s >= t ? (uint64_t)s - (uint64_t)t : (uint64_t)t - (uint64_t)s;
                    if (processed[in.read_repr[m]] != stamp && in.linked_read_cutoff >= 0 && d <= (uint64_t)in.linked_read_cutoff)
                        members.push_back(m);
                }
            }
            for (uint32_t m : members) {
                processed[in.read_repr[m]] = stamp;
                group[m] = r;
                g.members.push_back(m);
                ordinal += in.read_off[m + 1] - in.read_off[m];
                g.mstart.push_back(ordinal);
            }
            g.opener.push_back(r);
            g.moff.push_back(g.members.size());
        }
        for (uint32_t r = r0; r < r1; ++r) bx_next[r] = UINT32_MAX;
        r0 = r1;
    }
}

}  // namespace

}  // namespace whmec

using namespace whmec;

extern "C" int whmec_haplotag(const whmec_haplotag_input *in, int device, whmec_haplotag_output *out, whmec_haplotag_stats *stats,
                              char *err, size_t errlen) {
    const std::string bad = check(in, out);
    if (!bad.empty()) {
        put_err(err, errlen, "whmec_haplotag: " + bad);
        return WHMEC_ERR_INPUT;
    }
    out->error_kind = 0;
    out->error_read = out->error_entry = -1;
    std::string msg;
    const uint64_t budget = ht_budget(device, msg);
    if (!msg.empty()) {
        put_err(err, errlen, msg);
        return WHMEC_ERR_CUDA;
    }
    HtCall call;
    try {
        const auto t0 = std::chrono::steady_clock::now();
        const uint32_t ns = in->n_samples, nr = in->n_reads;
        const uint64_t np = in->phase_off[ns];
        call.n_samples = ns;
        call.n_pos = np;
        call.n_alleles = np ? in->allele_off[np] : 0;
        call.host = HtTable{in->phase_off, in->phase_pos, nullptr, in->allele_off, in->allele};
        call.ploidy = in->ploidy;
        // dense block ranks, sample by sample (their order does not matter: ties between blocks go by visit order)
        call.rank.resize(np);
        uint64_t n_ranks = 0, longest = 0;
        std::vector<int64_t> ids;
        for (uint32_t s = 0; s < ns; ++s) {
            const uint64_t p0 = in->phase_off[s], p1 = in->phase_off[s + 1];
            ids.assign(in->phase_block + p0, in->phase_block + p1);
            std::sort(ids.begin(), ids.end());
            ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
            for (uint64_t p = p0; p < p1; ++p) {
                call.rank[p] = (uint32_t)(n_ranks + (std::lower_bound(ids.begin(), ids.end(), in->phase_block[p]) - ids.begin()));
                longest = std::max<uint64_t>(longest, in->allele_off[p + 1] - in->allele_off[p]);
            }
            n_ranks += ids.size();
        }
        std::vector<int64_t> rank_id(n_ranks);
        for (uint64_t p = 0; p < np; ++p) rank_id[call.rank[p]] = in->phase_block[p];
        // a match needs h < ploidy and h < the tuple's length
        const uint64_t hmax = std::max<uint64_t>(1, std::min<uint64_t>(longest, in->ploidy > 0 ? (uint64_t)in->ploidy : 1));
        call.hap_bits = bits_for(hmax - 1);
        call.rank_bits = bits_for(n_ranks ? n_ranks - 1 : 0);
        if (n_ranks >= (1ull << 32) || call.hap_bits + call.rank_bits >= 64) {
            put_err(err, errlen, "whmec_haplotag: blocks and haplotypes need more than 63 key bits");
            return WHMEC_ERR_UNSUPPORTED;
        }
        const uint32_t group_bits_max = std::min<uint32_t>(31, 64 - call.hap_bits - call.rank_bits);

        Groups g;
        walk(*in, out->group, g);
        const uint64_t ng = g.opener.size();
        for (uint32_t r = 0; r < nr; ++r) out->n_blocks[r] = 0, out->block[r] = 0, out->haplotype[r] = -1, out->quality[r] = 0;
        call.st.groups = ng;
        call.st.entries = g.mstart.back();

        // chunks of whole groups under the budget, less the phase tables that stay resident
        const uint64_t fixed = (ns + 1) * 8 + np * (8 + 4 + 8) + 8 + call.n_alleles * 4 + 64 * 256 + (1 << 20);
        const uint64_t cap = budget > fixed ? budget - fixed : 0;
        const uint64_t per_entry = HT_ENTRY_BYTES + hmax * HT_MATCH_BYTES;
        call.st.plan_ms = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
        int rc = WHMEC_OK;
        for (uint64_t c0 = 0; c0 < ng && rc == WHMEC_OK;) {
            const auto t1 = std::chrono::steady_clock::now();
            uint64_t c1 = c0, ne = 0, bytes = 0;
            while (c1 < ng && c1 - c0 < (1ull << group_bits_max)) {
                const uint64_t e = g.mstart[g.moff[c1 + 1]] - g.mstart[g.moff[c1]];
                const uint64_t b = e * per_entry + HT_GROUP_BYTES;
                if (c1 > c0 && (bytes + b > cap || (ne + e) * hmax > (1ull << 30))) break;
                if ((ne + e) * hmax > (1ull << 30)) {
                    put_err(err, errlen, "whmec_haplotag: a group has more than 2^30 possible matches");
                    ht_close(call);
                    return WHMEC_ERR_UNSUPPORTED;
                }
                bytes += b, ne += e, ++c1;
            }
            // the chunk's entries in visit order
            call.e0 = g.mstart[g.moff[c0]];
            call.entries.resize(ne);
            call.gstart.assign(1, 0);
            HtEntry *dst = call.entries.data();
            for (uint64_t k = c0; k < c1; ++k) {
                for (uint64_t j = g.moff[k]; j < g.moff[k + 1]; ++j) {
                    const uint32_t m = g.members[j];
                    for (uint64_t x = in->read_off[m]; x < in->read_off[m + 1]; ++x)
                        *dst++ = HtEntry{in->entry_pos[x], in->entry_allele[x], in->entry_quality[x], (uint32_t)(k - c0), in->read_sample[m]};
                }
                call.gstart.push_back((uint32_t)(dst - call.entries.data()));
            }
            call.st.plan_ms += std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t1).count();
            ++call.st.chunks;
            if ((rc = ht_run_chunk(device, call, msg)) != WHMEC_OK) break;
            if (call.error != ~0ull) {  // the first error in visit order: no later chunk can hold an earlier one
                const uint64_t visit = call.error >> 2;
                out->error_kind = (int32_t)(call.error & 3);
                if (visit % 2 == 0) {
                    const uint64_t o = visit / 2;
                    const size_t j = std::upper_bound(g.mstart.begin(), g.mstart.end(), o) - g.mstart.begin() - 1;
                    out->error_read = g.members[j];
                    out->error_entry = (int64_t)(o - g.mstart[j]);
                } else {
                    const uint64_t end = (visit + 1) / 2;
                    for (uint64_t k = c0; k < c1; ++k)
                        if (g.mstart[g.moff[k + 1]] == end) {
                            out->error_read = g.opener[k];
                            break;
                        }
                    out->error_entry = -1;
                }
                break;
            }
            for (uint64_t k = c0; k < c1; ++k) {
                const HtChoice &ch = call.choice[k - c0];
                const uint32_t r = g.opener[k];
                out->n_blocks[r] = (int32_t)ch.n_blocks;
                if (!ch.n_blocks) continue;
                out->block[r] = rank_id[ch.rank];
                out->quality[r] = ch.quality;
                out->haplotype[r] = ch.quality != 0 ? ch.hap : -1;
            }
            c0 = c1;
        }
        ht_close(call);
        if (rc != WHMEC_OK) {
            put_err(err, errlen, msg);
            return rc;
        }
        if (stats) *stats = call.st;
        return WHMEC_OK;
    } catch (const std::bad_alloc &) {
        ht_close(call);
        put_err(err, errlen, "whmec_haplotag: out of host memory");
        return WHMEC_ERR_UNSUPPORTED;
    } catch (const std::exception &e) {  // nothing may cross the C boundary
        ht_close(call);
        put_err(err, errlen, std::string("whmec_haplotag: ") + e.what());
        return WHMEC_ERR_UNSUPPORTED;
    }
}
