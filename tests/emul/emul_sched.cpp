// TEST-ONLY host emulation of the tile kernel's SCHEDULE (tile.cu: one launch per segment, work items claimed out of round
// order, per-panel completion counters): the work items of a segment run in a seeded random order, an item only once the
// counter of its producer panel -- as the kernel derives it from the Panel fields -- is complete.  Per tile, the generic
// per-output code of tile_device.h (the steady-state column code is held to it by test_emulation.py).
#include <algorithm>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "../../whatshap_b200/csrc/pack.h"
#include "../../whatshap_b200/csrc/tile_device.h"
#include "../../whatshap_b200/csrc/tile_plan.h"

using namespace whmec;

namespace {

constexpr uint32_t POISON = 0xDEADBEEFu;

// one work item: tile t of panel P, state buffers and arena as the kernel leaves them
void run_item(const Packed &pk, const TileSchedule &ts, const Panel &P, uint32_t t, std::vector<uint32_t> &state, std::vector<uint32_t> &arena,
              std::vector<uint64_t> &chain_key) {
    std::vector<uint32_t> bufA(1u << TILE_SMAX), bufB(1u << TILE_SMAX);
    std::vector<int32_t> TL(TILE_TL_SIZE), TH(TILE_TH_SIZE);
    uint32_t *Sin = bufA.data(), *Sout = bufB.data();
    if (P.fresh) Sin[0] = 0;
    else if (P.in_layout == 1) {
        const uint32_t told = t & low_mask(P.in_gold);
        for (uint32_t i = 0; i < (1u << P.s_in); ++i) {
            uint32_t tA = i & low_mask(P.in_gA), at = (told << P.in_j) + (i >> P.in_gA);
            if (P.in_half && ((tA >> (P.in_gA - 1)) & 1u)) {
                tA = ~tA & low_mask(P.in_gA);
                at = ~at & low_mask(P.in_sA);
            }
            Sin[i] = state[P.in_off + ((uint64_t)tA << P.in_sA) + at];
        }
    } else {
        const uint32_t gpart = pdep32(t, P.gmask_in), fmask_in = P.lmask_in | P.gmask_in;
        for (uint32_t l = 0; l < (1u << P.s_in); ++l) {
            uint32_t e = pdep32(l, P.lmask_in) | gpart;
            if (P.in_half && (e & P.in_top)) e = ~e & fmask_in;
            Sin[l] = state[P.in_off + e];
        }
    }
    for (uint32_t k = P.col_begin; k < P.col_end; ++k) {
        const TileCol &tc = ts.cols[k];
        for (uint32_t i = 0; i < TILE_TL_SIZE; ++i) TL[i] = tile_tl_entry(tc, i);
        for (uint32_t i = 0; i < TILE_TH_SIZE; ++i) TH[i] = tile_th_entry(tc, t, i);
        TileCtx c{&tc, t, TL.data(), TH.data(), tile_cg(tc, t), Sin};
        const uint32_t m = tc.l_in + tc.n_new;
        if (tc.kind == 1) {
            const uint64_t key = tile_eval_end(c, pdep32(t, ~tc.lmask_col & low_mask(pk.cols[k].a)), 0, 1u << m);
            chain_key[P.chain] = std::min(chain_key[P.chain], key);
            continue;
        }
        const uint64_t slice = tc.bp_off + (uint64_t)t * tc.bp_tile_stride;
        for (uint32_t o = 0; o < (1u << tc.l_out); ++o) {
            uint64_t mkey;
            const uint64_t key = tile_eval(c, o, 0, 1u << tc.d, &mkey);
            Sout[o] = (uint32_t)(key >> 32);
            const uint32_t at = (tc.pad0 && (tc.pad2 & 1u)) ? tile_packed_bit_index(tc, o) : o;  // the fast columns' bit order
            bp_store_serial(arena.data(), slice, tc.bp_width, at, (uint32_t)key);
            if (tc.half && tc.km != 0) bp_store_serial(arena.data(), slice + tc.bp_tile_words, tc.bp_width, at, (uint32_t)mkey);
        }
        std::swap(Sin, Sout);
    }
    if (!P.ends_chain && P.out_layout == 1) {
        for (uint32_t l = 0; l < (1u << P.s_out); ++l) state[P.out_off + ((uint64_t)t << P.s_out) + l] = Sin[l];
    } else if (!P.ends_chain) {
        const uint32_t gpart = pdep32(t, P.gmask_out);
        for (uint32_t l = 0; l < (1u << P.s_out); ++l) state[P.out_off + (pdep32(l, P.lmask_out) | gpart)] = Sin[l];
    }
}

struct SchedInfo {
    uint64_t items = 0, max_ready = 0, out_of_order = 0, canonical = 0, tile_major = 0, mirrored = 0;
};

// One launch: the work items of panels [p0, p1) in a random order that respects the completion counters only.
void run_segment(const Packed &pk, const TileSchedule &ts, uint32_t p0, uint32_t p1, std::mt19937_64 &rng, std::vector<uint32_t> &state,
                 std::vector<uint32_t> &arena, std::vector<uint64_t> &chain_key, SchedInfo &info) {
    std::vector<uint32_t> done(p1 - p0, 0);                   // the launch's counters, zeroed in front of it
    std::vector<std::vector<uint32_t>> consumers(p1 - p0);  // panels of the segment waiting for panel q
    std::vector<std::pair<uint32_t, uint32_t>> ready;      // (panel, tile)
    auto release = [&](uint32_t q) {
        for (uint32_t t = 0; t < panel_tiles(ts.panels[q]); ++t) ready.push_back({q, t});
    };
    for (uint32_t q = p0; q < p1; ++q) {
        const Panel &P = ts.panels[q];
        if (!P.fresh && P.producer >= p0) consumers[P.producer - p0].push_back(q);  // the kernel's wait condition
        else release(q);
    }
    uint64_t last_item = 0;
    bool first = true;
    while (!ready.empty()) {
        info.max_ready = std::max<uint64_t>(info.max_ready, ready.size());
        const size_t pick = rng() % ready.size();
        const auto [q, t] = ready[pick];
        ready[pick] = ready.back();
        ready.pop_back();
        const Panel &P = ts.panels[q];
        const uint64_t item = (uint64_t)P.tile_begin + t;
        if (!first && item < last_item) ++info.out_of_order;
        first = false;
        last_item = item;
        run_item(pk, ts, P, t, state, arena, chain_key);
        ++info.items;
        if (P.ends_chain) continue;
        ++done[q - p0];  // the item's signal; a consumer starts once the count reaches ITS target
        auto &cs = consumers[q - p0];
        for (size_t i = 0; i < cs.size();)
            if (done[q - p0] >= ts.panels[cs[i]].producer_tiles) {
                release(cs[i]);
                cs[i] = cs.back();
                cs.pop_back();
            } else {
                ++i;
            }
    }
}

}  // namespace

// Solve through the emulated schedule.  n_segments > 1: the rounds are cut into that many segments (a memory-bounded
// sweep): the forward sweep keeps a checkpoint of the state in front of every segment, the back-pointers of every segment
// but the last are then overwritten, and every such segment is swept again from its checkpoint before the backtrace.
// info6: work items run, largest number of items ready at once, items run before a lower-numbered one, panels with the
// canonical / tile-major hand-off, mirrored panels.  Returns 100 when the planner declines the problem.
extern "C" int whemul_sched_solve(const whmec_problem *p, whmec_solution *s, uint64_t seed, uint32_t n_segments, uint64_t *info6, char *err,
                                  size_t errlen) {
    Packed pk;
    std::string msg;
    auto fail = [&](int code) {
        if (err && errlen) {
            std::strncpy(err, msg.c_str(), errlen - 1);
            err[errlen - 1] = 0;
        }
        return code;
    };
    int rc = pack_problem(p, pk, msg);
    if (rc != WHMEC_OK) return fail(rc);
    const uint32_t n = pk.n;
    if (n == 0) {
        s->cost = 0;
        if (s->partition) std::memset(s->partition, 1, p->n_reads);
        return WHMEC_OK;
    }
    TileSchedule ts;
    plan_tiles(pk, ts);
    if (!ts.eligible) {
        msg = ts.why;
        return fail(100);
    }
    SchedInfo info;
    for (const Panel &P : ts.panels) {
        if (!P.fresh) ++(P.in_layout == 1 ? info.tile_major : info.canonical);
        info.mirrored += P.half;
    }
    const uint32_t n_rounds = (uint32_t)ts.round_begin.size() - 1, K = std::max(1u, std::min(n_segments, n_rounds));
    std::vector<uint32_t> cut(K + 1);
    for (uint32_t i = 0; i <= K; ++i) cut[i] = (uint32_t)((uint64_t)n_rounds * i / K);
    std::mt19937_64 rng(seed);
    std::vector<uint32_t> state(ts.state_words + 1, POISON), arena(ts.bp_words + 1, 0);
    std::vector<std::vector<uint32_t>> ckpt(K);
    const uint32_t n_chains = (uint32_t)pk.chain_begin.size() - 1;
    std::vector<uint64_t> chain_key(n_chains, KEY_INF);
    for (uint32_t sg = 0; sg < K; ++sg) {
        ckpt[sg] = state;
        run_segment(pk, ts, ts.round_begin[cut[sg]], ts.round_begin[cut[sg + 1]], rng, state, arena, chain_key, info);
    }
    for (uint32_t sg = K - 1; sg-- > 0;) {  // the backtrace's re-sweeps, last segment first
        for (uint32_t q = ts.round_begin[cut[sg]]; q < ts.round_begin[cut[sg + 1]]; ++q)
            for (uint32_t k = ts.panels[q].col_begin; k < ts.panels[q].col_end; ++k) {
                const TileCol &tc = ts.cols[k];
                std::fill_n(arena.begin() + tc.bp_off, (uint64_t)tc.bp_tile_stride << (tc.g - tc.half), POISON);
            }
        state = ckpt[sg];  // (the checkpoint of segment 0 is the poisoned state the sweep started from)
        run_segment(pk, ts, ts.round_begin[cut[sg]], ts.round_begin[cut[sg + 1]], rng, state, arena, chain_key, info);
    }
    std::vector<uint32_t> pidx(n), ptv(n, 0);
    uint64_t total = 0;
    for (uint32_t c = 0; c < n_chains; ++c) {
        total += chain_key[c] >> 32;
        tile_backtrace_chain(pk.cols.data(), ts.cols.data(), arena.data(), pk.chain_begin[c], pk.chain_begin[c + 1] - 1, chain_key[c], pidx.data());
    }
    s->cost = (uint32_t)total;
    if (info6) {
        const uint64_t v[6] = {info.items, info.max_ready, info.out_of_order, info.canonical, info.tile_major, info.mirrored};
        std::memcpy(info6, v, sizeof v);
    }
    rc = build_outputs(pk, pidx.data(), ptv.data(), s, msg);
    return rc == WHMEC_OK ? WHMEC_OK : fail(rc);
}

// Invariants of the planner's schedule that the kernel's counters rely on.  Returns 0, or the number of the first one broken:
//   1  items are numbered panel after panel without gaps
//   2  a fresh panel starts its chain and has no producer
//   3  a producer is the previous panel of the same chain, earlier in the panel array
//   4  ... and all its items come before the consumer's
//   5  the counter target is the producer's number of computed tiles
//   6  the consumer reads the buffer the producer wrote, and writes the other one: a panel's output is never its input
//   7  the producer is the round before the consumer's (segments are cut at round boundaries)
// out2: panels, panels with a producer.
extern "C" int whemul_sched_check(const whmec_problem *p, uint64_t *out2) {
    Packed pk;
    std::string msg;
    int rc = pack_problem(p, pk, msg);
    if (rc != WHMEC_OK) return -rc;
    TileSchedule ts;
    plan_tiles(pk, ts);
    if (!ts.eligible) return 100;
    const uint32_t np = (uint32_t)ts.panels.size();
    std::vector<uint32_t> round_of(np);
    for (uint32_t r = 0; r + 1 < ts.round_begin.size(); ++r)
        for (uint32_t q = ts.round_begin[r]; q < ts.round_begin[r + 1]; ++q) round_of[q] = r;
    out2[0] = np;
    out2[1] = 0;
    uint64_t item = 0;
    for (uint32_t q = 0; q < np; ++q) {
        const Panel &P = ts.panels[q];
        if (P.tile_begin != item) return 1;
        item += panel_tiles(P);
        if (P.fresh) {
            if (P.producer != TILE_NO_PANEL || P.producer_tiles != 0 || P.col_begin != pk.chain_begin[P.chain]) return 2;
            continue;
        }
        ++out2[1];
        if (P.producer >= q) return 3;
        const Panel &A = ts.panels[P.producer];
        if (A.chain != P.chain || A.col_end != P.col_begin || A.ends_chain) return 3;
        if ((uint64_t)A.tile_begin + panel_tiles(A) > P.tile_begin) return 4;
        if (P.producer_tiles != panel_tiles(A)) return 5;
        if (P.in_off != A.out_off || (!P.ends_chain && P.out_off == P.in_off) || A.in_off == A.out_off) return 6;
        if (round_of[P.producer] + 1 != round_of[q]) return 7;
    }
    return 0;
}
