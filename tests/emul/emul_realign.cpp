// TEST-ONLY: whmec_realign and whmec_edit_distance_batch (host walk and chunk plan of realign_plan.cpp) with the chunk runner
// of realign.cu executed on the host: the per-job code of realign.h, one-thread jobs in a loop and each warp job as 32 lanes
// stepped in lock-step, every lane reading what its upper neighbour produced one step earlier (the kernel's __shfl_up_sync).
// The chunk budget is WHMEC_REALIGN_ARENA_BUDGET (no limit without it).
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

int64_t unit_warp(const RaSeq &p, const RaSeq &x, std::vector<int8_t> &hrow) {
    const uint32_t words = (p.len + 63) / 64, groups = (words + 31) / 32;
    int64_t d = 0;
    for (uint32_t g = 0; g < groups; ++g) {
        RaUnitLane ln[32];
        int out[32] = {0}, prev[32];
        for (uint32_t l = 0; l < 32; ++l) ln[l].init(p, 32 * g + l);
        for (uint32_t s = 0; s < x.len + 31; ++s) {
            for (uint32_t l = 0; l < 32; ++l) prev[l] = out[l];
            for (uint32_t l = 0; l < 32; ++l) {
                const int64_t j = (int64_t)s - l;
                if (!ln[l].active || j < 0 || j >= x.len) continue;
                const int hin = l ? prev[l - 1] : g ? hrow[j] : 1;
                out[l] = ln[l].step(p, x.at((uint32_t)j), hin);
                if (l == 31 && g + 1 < groups) hrow[j] = (int8_t)out[l];
            }
        }
        if (g + 1 == groups) d = ln[(words - 1) % 32].score;
    }
    return d;
}

bool affine_warp(const RaSeq &q, const RaSeq &t, const RaParams &pr, int64_t &d) {
    const uint32_t m = q.len;
    std::vector<float> A(m + 1), B(m + 1), C(m + 1);
    RaAffLane ln[32];
    RaCell out[32] = {}, prev[32];
    for (uint32_t l = 0; l < 32; ++l) ln[l].init(m, l, 32, A.data(), B.data(), C.data(), pr);
    for (uint32_t s = 0; s < t.len + 31; ++s) {
        for (uint32_t l = 0; l < 32; ++l) prev[l] = out[l];
        for (uint32_t l = 0; l < 32; ++l) {
            const int64_t j = (int64_t)s - l + 1;
            if (!ln[l].active() || j < 1 || j > t.len) continue;
            out[l] = ln[l].step(A.data(), B.data(), C.data(), l ? prev[l - 1] : ra_affine_top((uint32_t)j, pr), q, t.at((uint32_t)(j - 1)), pr);
        }
    }
    return ra_trunc(ra_min3(A[m], B[m], C[m]), d);
}

}  // namespace

int ra_run_chunk(int, RaCall &call, const RaChunk &c, std::string &) {
    // the chunk's slices only, as on the device
    const std::vector<uint8_t> qs(call.host.q + c.q_lo, call.host.q + c.q_hi), rs(call.host.ref + c.r_lo, call.host.ref + c.r_hi);
    const RaBufs b{qs.data(), c.q_lo, rs.data(), c.r_lo, call.host.al, call.host.al_off, call.host.al_first};
    std::vector<int64_t> dist(c.job1 - c.job0);
    std::vector<int8_t> scratch(c.scratch + 1);
    for (uint32_t k = c.job0; k < c.job1; ++k) {
        const RaJob &jb = call.jobs[k];
        const RaItem &it = call.items[jb.item];
        int64_t d = 0;
        bool ok = true;
        if (jb.scratch == RA_NO_SCRATCH) {
            ok = ra_short_job(b, it, jb.allele, call.params, d);
        } else {
            RaSeq q = ra_query(b, it), t = ra_target(b, it, jb.allele);
            ra_trim(q, t);
            if (!call.params.affine) {
                const RaSeq &p = q.len <= t.len ? q : t, &x = q.len <= t.len ? t : q;
                std::vector<int8_t> hrow(x.len + 1);
                d = p.len <= RA_SHORT ? ra_unit_short(q, t) : unit_warp(p, x, hrow);
            } else if (q.len <= RA_SHORT) {
                ok = ra_trunc(ra_affine_short(q, t, call.params), d);
            } else {
                ok = affine_warp(q, t, call.params, d);
            }
        }
        dist[k - c.job0] = d;
        call.status[k] = !ok;
        if (!call.decide) call.dist[k] = d;
    }
    if (call.decide)
        for (uint32_t i = c.item0; i < c.item1; ++i) {
            const RaItem &it = call.items[i];
            call.call[i] = ra_decide(dist.data() + (it.job0 - c.job0), it.n_jobs, call.params.affine, call.quality[i]);
        }
    call.st.kernel_launches += 2 + call.decide;
    return WHMEC_OK;
}

}  // namespace whmec
