// TEST-ONLY: whmec_realign_kmerald and whmec_kmer_align_batch (host walk and chunk plan of realign_plan.cpp) with the k-mer chunk
// runner of realign.cu (ka_short_kernel, ka_long_kernel, ka_decide_kernel) executed on the host, using the per-job code of
// kmerald.h: one-thread jobs in a loop, each warp job as 32 lanes stepped in lock-step, every lane reading what its upper
// neighbour produced one step earlier (the kernel's __shfl_up_sync).  Unit-cost and affine calls are refused (their emulation
// is emul_realign.cpp).  The chunk budget is WHMEC_REALIGN_ARENA_BUDGET (no limit without it).  Also exports
// enumerate_all_kmers.
#include <cstdlib>
#include <string>
#include <vector>

#include "../../whatshap_b200/csrc/realign_plan.h"

namespace whmec {

uint64_t ra_budget(int, std::string &) {
    const char *h = std::getenv("WHMEC_REALIGN_ARENA_BUDGET");
    return h ? std::strtoull(h, nullptr, 10) : ~0ull;
}

void ra_close(RaCall &) {}

namespace {

float long_job(const RaBufs &b, const RaItem &it, uint32_t allele, const KaParams &p) {
    const RaSeq q = ra_query(b, it), t = ra_target(b, it, allele);
    std::vector<uint8_t> area(ka_scratch_bytes(q.len, t.len));
    const KaScratch s(area.data(), q.len, t.len);
    uint32_t m = ka_kmers(t, p.k, s.a), n = ka_kmers(q, p.k, s.b), x = 0;
    if (!ka_trim(s.a, s.b, m, n, x)) return 0.0f;
    if (m == 0) return p.gap * (float)n;
    const uint32_t *a = s.a + x, *bq = s.b + x;
    KaLane ln[32];
    float out[32] = {}, prev[32];
    for (uint32_t l = 0; l < 32; ++l) ln[l].init(m, l, 32, a, s.row, s.S, p);
    for (uint32_t st = 0; st < n + 31; ++st) {
        for (uint32_t l = 0; l < 32; ++l) prev[l] = out[l];
        for (uint32_t l = 0; l < 32; ++l) {
            const int64_t j = (int64_t)st - l + 1;
            if (!ln[l].active() || j < 1 || j > n) continue;
            out[l] = ln[l].step(a, s.row, s.S, l ? prev[l - 1] : p.gap * (float)j, bq[j - 1], p);
        }
    }
    return s.S[m];
}

}  // namespace

int ra_run_chunk(int, RaCall &call, const RaChunk &c, std::string &msg) {
    if (!call.kmerald) {
        msg = "the k-mer emulation runs k-mer calls only";
        return WHMEC_ERR_UNSUPPORTED;
    }
    // the chunk's slices only, as on the device
    const std::vector<uint8_t> qs(call.host.q + c.q_lo, call.host.q + c.q_hi), rs(call.host.ref + c.r_lo, call.host.ref + c.r_hi);
    const RaBufs b{qs.data(), c.q_lo, rs.data(), c.r_lo, call.host.al, call.host.al_off, call.host.al_first};
    std::vector<float> dist(c.job1 - c.job0);
    for (uint32_t k = c.job0; k < c.job1; ++k) {
        const RaJob &jb = call.jobs[k];
        const RaItem &it = call.items[jb.item];
        dist[k - c.job0] = jb.scratch == RA_NO_SCRATCH ? ka_short_job(b, it, jb.allele, call.kparams) : long_job(b, it, jb.allele, call.kparams);
        if (!call.decide) call.kdist[k] = dist[k - c.job0];
    }
    if (call.decide)
        for (uint32_t i = c.item0; i < c.item1; ++i) {
            const RaItem &it = call.items[i];
            call.call[i] = ka_decide(dist[it.job0 - c.job0], dist[it.job0 - c.job0 + 1]);
            call.quality[i] = 30;
        }
    call.st.kernel_launches += 2 + call.decide;
    return WHMEC_OK;
}

}  // namespace whmec

// enumerate_all_kmers(s[0..len), k) into out (at most len entries); returns the count
extern "C" uint32_t whemul_enumerate_kmers(const uint8_t *s, uint32_t len, uint32_t k, uint32_t *out) {
    const whmec::RaSeq seq{s, nullptr, nullptr, len, 0, 0, 0, len};
    return whmec::ka_kmers(seq, k, out);
}
