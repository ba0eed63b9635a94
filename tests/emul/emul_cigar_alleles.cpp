// TEST-ONLY: whmec_detect_alleles_cigar (host preparation and chunk plan of cigar_alleles_plan.cpp) with the chunk runner of
// cigar_alleles.cu executed on the host: the per-thread code of cigar_alleles.h over the chunk's slices only, the count walk, the
// scan, and per window the emit walk, one resolve per item and the selection of the calls.  The chunk budget is
// WHMEC_REALIGN_ARENA_BUDGET (no limit without it).
#include <algorithm>
#include <cstdlib>
#include <string>
#include <vector>

#include "../../whatshap_b200/csrc/cigar_alleles_plan.h"

namespace whmec {

uint64_t ca_budget(int, std::string &) {
    const char *h = std::getenv("WHMEC_REALIGN_ARENA_BUDGET");
    return h ? std::strtoull(h, nullptr, 10) : ~0ull;
}

void ca_close(CaRun &) {}

int ca_run_chunk(int, CaRun &run, const CaChunk &c, std::string &) {
    const whmec_realign_input &in = *run.in;
    const CaPlan &P = *run.plan;
    const uint32_t na = c.a1 - c.a0;
    const std::vector<CaAln> alns(P.alns.begin() + c.a0, P.alns.begin() + c.a1);
    const std::vector<uint8_t> op(in.cigar_op + c.op_lo, in.cigar_op + c.op_hi), q(in.query + c.q_lo, in.query + c.q_hi);
    const std::vector<int32_t> len(in.cigar_len + c.op_lo, in.cigar_len + c.op_hi);
    const std::vector<uint8_t> qual = run.q ? std::vector<uint8_t>(run.q->qual + c.qual_lo, run.q->qual + c.qual_hi) : std::vector<uint8_t>();
    const CaBufs b{op.data(), len.data(), c.op_lo, q.data(), c.q_lo, qual.data(), c.qual_lo, alns.data(), P.vars.data(),
                   (uint32_t)(P.vars.size() - 1), P.alleles.data(), in.allele_bytes};
    std::vector<uint64_t> first(na + 1, 0);
    for (uint32_t a = 0; a < na; ++a) {
        CaCount n;
        ca_walk(b, a, n);
        first[a + 1] = first[a] + n.n;
    }
    run.st.kernel_launches += 2;
    const uint64_t items = first[na];
    run.st.items += items;
    const uint64_t window = std::min<uint64_t>({ca_window(c, run.budget), std::max<uint64_t>(items, 1), 1ull << 30});
    std::vector<CaItem> win(window);
    for (uint64_t lo = 0; lo < items; lo += window) {
        const uint64_t hi = std::min(items, lo + window);
        for (uint32_t a = 0; a < na; ++a) {
            if (first[a + 1] <= lo || first[a] >= hi) continue;
            CaEmit e{win.data(), first[a], lo, hi};
            ca_walk(b, a, e);
        }
        uint32_t raised = UMAX;
        for (uint64_t k = 0; k < hi - lo; ++k) {
            CaCall call{c.a0 + win[k].aln, P.vars[win[k].var].id, -1, 0, 0};
            uint32_t n_alleles = 0;
            if (!ca_resolve(b, win[k], call.allele, call.quality, n_alleles)) raised = std::min(raised, call.alignment), call.allele = -1;
            run.st.jobs += n_alleles;
            if (call.allele >= 0) run.calls.push_back(call);
        }
        run.st.kernel_launches += 3;
        ++run.st.chunks;
        run.raised = std::min(run.raised, raised);
        if (raised != UMAX) break;
    }
    return WHMEC_OK;
}

}  // namespace whmec
