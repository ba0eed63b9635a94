// TEST-ONLY host emulation of the tile kernel's narrow steady-state panels (Panel::narrow, tile_fast.h: narrow_column_body).
// Builds on the tile emulation of emul_tile.cpp, which is included so that its per-column helpers are visible here:
// whemul_narrow_solve is whemul_tile_solve with one more dispatch -- a narrow panel runs the kernel's narrow code thread by
// thread and every one of its columns is checked against the 32-bit steady column on the same input.
// whemul_narrow_census counts the planner's steady and narrow panels.
#include "emul_tile.cpp"

#include <algorithm>
#include <climits>

namespace {

// Narrow steady-state panel (Panel::narrow) of tile t: the kernel's narrow code (tile.cu: steady_columns_narrow) thread by
// thread, warp by warp for the back-pointer words, with every column checked against the 32-bit steady column run on the
// same input: same values, same back-pointer words, values inside the planner's bound.  The narrow results go on.
struct NarrowStats {
    uint64_t columns = 0, value_mismatches = 0, bp_mismatches = 0, bound_violations = 0, max_spread = 0;
    int64_t min_slack = INT64_MAX;  // smallest (bound - (largest value - base)) over the checked columns
};
NarrowStats g_narrow;

void narrow_panel(const TileSchedule &ts, const Panel &P, uint32_t t, uint32_t *Sin, uint32_t *arena) {
    constexpr uint32_t N = 1u << TILE_SMAX;
    std::vector<uint32_t> ref(Sin, Sin + N), ref2(N), bp_ref, H0(N / 2), H1(N / 2);
    uint32_t *Hin = H0.data(), *Hout = H1.data();
    const uint32_t base = Sin[0] - P.narrow_spread;
    for (uint32_t x = 0; x < N; ++x) {
        if (Sin[x] - base > 2u * P.narrow_spread) ++g_narrow.bound_violations;  // (also catches Sin[x] < base: wraps)
        Hin[x >> 1] |= ((Sin[x] - base) << 1) << (16 * (x & 1u));
    }
    for (uint32_t k = P.col_begin; k < P.col_end; ++k) {
        const TileCol &tc = ts.cols[k];
        uint32_t *slice = arena + tc.bp_off + (uint64_t)t * tc.bp_tile_stride;
        run_fast_column(tc, t, ref.data(), ref2.data(), slice);
        std::swap(ref, ref2);
        bp_ref.assign(slice, slice + tc.bp_tile_words);
        std::memset(slice, 0, tc.bp_tile_words * sizeof(uint32_t));
        int32_t TW[32], T5[32];
        for (uint32_t i = 0; i < 32; ++i) {
            TW[i] = tile_fast_warp_entry(tc, t, i);
            T5[i] = narrow_lane_entry(tc, i);
        }
        const uint32_t cg = tile_cg(tc, t);
        const NarrowCol nc[2] = {narrow_col(tc, cg, 0), narrow_col(tc, cg, 1)};
        for (uint32_t w = 0; w < 32; ++w) {
            uint32_t bits[32];
            for (uint32_t lane = 0; lane < 32; ++lane) {
                NarrowPrep pr;
                narrow_prep(pr, &nc[(popc32(w) + popc32(lane)) & 1u], (uint32_t)(TW[w] + T5[lane]), Hin, Hout, w * 128u + lane);
                bits[lane] = narrow_column_body(pr);
            }
            for (uint32_t lane = 0; lane < 16; ++lane) slice[w * 16 + lane] = narrow_bp_word(bits[lane], bits[lane + 16]);
        }
        std::swap(Hin, Hout);
        for (uint32_t i = 0; i < tc.bp_tile_words; ++i) g_narrow.bp_mismatches += slice[i] != bp_ref[i];
        const uint64_t bound = narrow_panel_bound(P.narrow_spread, &ts.cols[P.col_begin], k + 1 - P.col_begin);
        uint32_t lo = 0xFFFFFFFFu, hi = 0;
        for (uint32_t x = 0; x < N; ++x) {
            const uint32_t h = (Hin[x >> 1] >> (16 * (x & 1u))) & 0xFFFFu;
            g_narrow.value_mismatches += (h & 1u) != 0 || base + (h >> 1) != ref[x];
            lo = std::min(lo, ref[x]);
            hi = std::max(hi, ref[x]);
        }
        const int64_t slack = (int64_t)bound - (int64_t)(hi - base);
        g_narrow.bound_violations += slack < 0;
        g_narrow.min_slack = std::min(g_narrow.min_slack, slack);
        g_narrow.max_spread = std::max<uint64_t>(g_narrow.max_spread, hi - lo);
        ++g_narrow.columns;
    }
    for (uint32_t x = 0; x < N; ++x) Sin[x] = base + (((Hin[x >> 1] >> (16 * (x & 1u))) & 0xFFFFu) >> 1);
}

}  // namespace

// whemul_tile_solve with narrow panels: the same sweep, where a narrow panel runs narrow_panel (returns 100 when the planner
// declares the problem not eligible for the tile path)
extern "C" int whemul_narrow_solve(const whmec_problem *p, whmec_solution *s, uint32_t chunk, uint32_t *n_panels,
                                 char *err, size_t errlen) {
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
    if (n_panels) *n_panels = (uint32_t)ts.panels.size();
    std::vector<uint32_t> state(ts.state_words + 1, 0xDEADBEEF), arena(ts.bp_words + 1, 0);
    const uint32_t n_chains = (uint32_t)pk.chain_begin.size() - 1;
    std::vector<uint64_t> chain_key(n_chains, KEY_INF);
    std::vector<uint32_t> bufA(1u << TILE_SMAX), bufB(1u << TILE_SMAX);
    std::vector<int32_t> TL(TILE_TL_SIZE), TH(TILE_TH_SIZE);
    const char *fast_env = std::getenv("WHEMUL_TILE_FAST");
    const bool use_fast = !(fast_env && fast_env[0] == '0');
    uint64_t fast_columns = 0, packed_columns = 0;
    g_narrow = NarrowStats();
    for (size_t r = 0; r + 1 < ts.round_begin.size(); ++r)
        for (uint32_t pi = ts.round_begin[r]; pi < ts.round_begin[r + 1]; ++pi) {
            const Panel &P = ts.panels[pi];
            for (uint32_t t = 0; t < (1u << (P.g - P.half)); ++t) {  // mirrored panel: tiles with top tile-id bit 0 only
                uint32_t *Sin = bufA.data(), *Sout = bufB.data();
                if (P.fresh) Sin[0] = 0;
                else if (P.in_layout == 1) {
                    const uint32_t told = t & low_mask(P.in_gold);
                    for (uint32_t i = 0; i < (1u << P.s_in); ++i) {
                        uint32_t tA = i & low_mask(P.in_gA), at = (told << P.in_j) + (i >> P.in_gA);  // producer tile, its local index
                        if (P.in_half && ((tA >> (P.in_gA - 1)) & 1u)) {  // not computed: complemented index of the mirror tile
                            tA = ~tA & low_mask(P.in_gA);
                            at = ~at & low_mask(P.in_sA);
                        }
                        Sin[i] = state[P.in_off + ((uint64_t)tA << P.in_sA) + at];
                    }
                } else {
                    const uint32_t gpart = pdep32(t, P.gmask_in);
                    const uint32_t fmask_in = P.lmask_in | P.gmask_in;
                    for (uint32_t l = 0; l < (1u << P.s_in); ++l) {
                        uint32_t e = pdep32(l, P.lmask_in) | gpart;
                        if (P.in_half && (e & P.in_top)) e = ~e & fmask_in;
                        Sin[l] = state[P.in_off + e];
                    }
                }
                if (P.narrow && use_fast) {  // (P.narrow: the whole panel is steady-state columns, never a chain end)
                    narrow_panel(ts, P, t, Sin, arena.data());
                    fast_columns += P.col_end - P.col_begin;
                    packed_columns += P.col_end - P.col_begin;
                }
                for (uint32_t k = (P.narrow && use_fast) ? P.col_end : P.col_begin; k < P.col_end; ++k) {
                    const TileCol &tc = ts.cols[k];
                    for (uint32_t i = 0; i < TILE_TL_SIZE; ++i) TL[i] = tile_tl_entry(tc, i);
                    for (uint32_t i = 0; i < TILE_TH_SIZE; ++i) TH[i] = tile_th_entry(tc, t, i);
                    TileCtx c{&tc, t, TL.data(), TH.data(), tile_cg(tc, t), Sin};
                    const uint32_t m = tc.l_in + tc.n_new;
                    if (tc.kind == 1) {
                        const uint32_t gpart = pdep32(t, ~tc.lmask_col & low_mask(pk.cols[k].a));
                        uint64_t best = KEY_INF;
                        uint32_t step = chunk ? chunk : (1u << m);
                        for (uint32_t x0 = 0; x0 < (1u << m); x0 += step) {
                            uint32_t x1 = x0 + step < (1u << m) ? x0 + step : (1u << m);
                            uint64_t key = tile_eval_end(c, gpart, x0, x1);
                            if (key < best) best = key;
                        }
                        if (best < chain_key[P.chain]) chain_key[P.chain] = best;
                    } else if (tc.pad0 && use_fast) {
                        run_fast_column(tc, t, Sin, Sout, arena.data() + tc.bp_off + (uint64_t)t * tc.bp_tile_stride);
                        ++fast_columns;
                        packed_columns += (tc.pad2 & 1u) != 0;
                        std::swap(Sin, Sout);
                    } else {
                        const uint32_t ncand = 1u << tc.d;
                        for (uint32_t o = 0; o < (1u << tc.l_out); ++o) {
                            uint64_t best = KEY_INF, mbest = KEY_INF;
                            uint32_t step = chunk ? chunk : ncand;
                            for (uint32_t r0 = 0; r0 < ncand; r0 += step) {
                                uint32_t r1 = r0 + step < ncand ? r0 + step : ncand;
                                uint64_t mkey;
                                uint64_t key = tile_eval(c, o, r0, r1, &mkey);
                                if (key < best) best = key;
                                if (mkey < mbest) mbest = mkey;
                            }
                            Sout[o] = (uint32_t)(best >> 32);
                            // WHEMUL_TILE_FAST=0 on a column the planner marked thread-packed: same bit positions as the fast code
                            const uint32_t at = (tc.pad0 && (tc.pad2 & 1u)) ? tile_packed_bit_index(tc, o) : o;
                            const uint64_t slice = tc.bp_off + (uint64_t)t * tc.bp_tile_stride;
                            bp_store_serial(arena.data(), slice, tc.bp_width, at, (uint32_t)best);
                            if (tc.half && tc.km != 0) bp_store_serial(arena.data(), slice + tc.bp_tile_words, tc.bp_width, at, (uint32_t)mbest);
                        }
                        std::swap(Sin, Sout);
                    }
                }
                if (!P.ends_chain && P.out_layout == 1) {
                    for (uint32_t l = 0; l < (1u << P.s_out); ++l) state[P.out_off + ((uint64_t)t << P.s_out) + l] = Sin[l];
                } else if (!P.ends_chain) {
                    const uint32_t gpart = pdep32(t, P.gmask_out);
                    for (uint32_t l = 0; l < (1u << P.s_out); ++l) state[P.out_off + (pdep32(l, P.lmask_out) | gpart)] = Sin[l];
                }
            }
        }
    std::vector<uint32_t> pidx(n), ptv(n, 0);
    uint64_t total = 0;
    for (uint32_t c = 0; c < n_chains; ++c) {
        total += chain_key[c] >> 32;
        tile_backtrace_chain(pk.cols.data(), ts.cols.data(), arena.data(), pk.chain_begin[c], pk.chain_begin[c + 1] - 1,
                             chain_key[c], pidx.data());
    }
    s->cost = (uint32_t)total;
    rc = build_outputs(pk, pidx.data(), ptv.data(), s, msg);
    if (rc != WHMEC_OK) return fail(rc);
    return WHMEC_OK;
}

// Narrow panels of the last whemul_narrow_solve (see narrow_panel): (tile, column) pairs, value and back-pointer word mismatches
// against the 32-bit columns, bound violations, largest max - min of a tile's column, smallest slack below the bound
// (out6[5] as int64; INT64_MAX when no narrow column ran).
extern "C" void whemul_last_narrow_stats(int64_t *out6) {
    out6[0] = (int64_t)g_narrow.columns;
    out6[1] = (int64_t)g_narrow.value_mismatches;
    out6[2] = (int64_t)g_narrow.bp_mismatches;
    out6[3] = (int64_t)g_narrow.bound_violations;
    out6[4] = (int64_t)g_narrow.max_spread;
    out6[5] = g_narrow.min_slack;
}

// Panels of the planner's schedule: out2[0] steady, out2[1] narrow (of those).  Returns 0, 100 when the planner declines the
// problem, or minus the packing error.
extern "C" int whemul_narrow_census(const whmec_problem *p, uint64_t *out2) {
    Packed pk;
    std::string msg;
    const int rc = pack_problem(p, pk, msg);
    if (rc != WHMEC_OK) return -rc;
    out2[0] = out2[1] = 0;
    if (pk.n == 0) return 100;
    TileSchedule ts;
    plan_tiles(pk, ts);
    if (!ts.eligible) return 100;
    for (const Panel &P : ts.panels) {
        out2[0] += P.steady != 0;
        out2[1] += P.narrow != 0;
    }
    return 0;
}
