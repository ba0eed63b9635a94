// TEST-ONLY census of the tile planner's schedule for one problem (pack_problem + plan_tiles, as the library runs them):
// which hand-off feeds every panel, which panels are steady or mirrored, and the largest number of global reads.  The
// bulk / small-chunk split is the kernel's own rule (bulk_handoff, tile_device.h).  test_high_coverage_golden.py uses it to
// check that the stored high-coverage instances reach the kernel paths they are meant to hold to the reference.
#include <algorithm>
#include <cstring>
#include <string>

#include "../../whatshap_b200/csrc/pack.h"
#include "../../whatshap_b200/csrc/tile_device.h"
#include "../../whatshap_b200/csrc/tile_plan.h"

using namespace whmec;

// out[CENSUS_N]:
//   [0, 24)  panels by [hand-off 4][steady 2][mirror 3]
//            hand-off: 0 fresh, 1 canonical, 2 tile-major bulk copies, 3 tile-major small chunks (per-element gather)
//            steady:   Panel::steady != 0
//            mirror:   0 not mirrored, 1 mirrored with km == 0 in every column, 2 mirrored with km != 0 in some column
//   24, 25   mirrored columns with km == 0, with km != 0
//   26       largest g of a panel
//   27       chains
//   28       bulk hand-offs with in_gA == BULK_MAX_GA (the largest that still travels as bulk copies)
//   29       panels
// Returns 0, 100 when the planner declines the problem, or minus the packing error.
constexpr uint32_t CENSUS_N = 30;

extern "C" uint32_t whemul_census_size() { return CENSUS_N; }

extern "C" int whemul_census(const whmec_problem *p, uint64_t *out) {
    Packed pk;
    std::string msg;
    const int rc = pack_problem(p, pk, msg);
    if (rc != WHMEC_OK) return -rc;
    std::memset(out, 0, CENSUS_N * sizeof(uint64_t));
    if (pk.n == 0) return 100;
    TileSchedule ts;
    plan_tiles(pk, ts);
    if (!ts.eligible) return 100;
    for (const Panel &P : ts.panels) {
        uint32_t handoff = 0;
        if (!P.fresh) handoff = P.in_layout == 0 ? 1 : bulk_handoff(P.in_gA, P.in_j) ? 2 : 3;
        uint32_t mirror = 0;
        if (P.half) {
            mirror = 1;
            for (uint32_t k = P.col_begin; k < P.col_end; ++k)
                if (ts.cols[k].half && ts.cols[k].km != 0) mirror = 2;
        }
        ++out[(handoff * 2 + (P.steady ? 1 : 0)) * 3 + mirror];
        for (uint32_t k = P.col_begin; k < P.col_end; ++k)
            if (ts.cols[k].half) ++out[ts.cols[k].km == 0 ? 24 : 25];
        out[26] = std::max<uint64_t>(out[26], P.g);
        if (handoff == 2 && P.in_gA == BULK_MAX_GA) ++out[28];
    }
    out[27] = pk.chain_begin.size() - 1;
    out[29] = ts.panels.size();
    return 0;
}
