// Host planner of the tile path: cuts every DP-independent chain into panels (see tile_plan.h).
#include "tile_plan.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace whmec {

namespace {

// reads of column k in canonical order
inline const uint32_t *col_reads(const Packed &pk, uint32_t k) { return pk.act_read.data() + pk.act_off[k]; }

}  // namespace

void plan_tiles(const Packed &pk, TileSchedule &ts) {
    ts = TileSchedule();
    if (pk.T != 1 || pk.n_ind != 1) {
        ts.why = "more than one individual (the tile kernel covers the single-individual cost form)";
        return;
    }
    if (!pk.safe31) {
        ts.why = "cost range exceeds the exact range of the tile arithmetic";
        return;
    }
    const bool timing = std::getenv("WHMEC_TIMING") != nullptr;
    const char *packed_env = std::getenv("WHMEC_TILE_PACKED_BP");
    const bool packed_bp = !(packed_env && packed_env[0] == '0');  // the default; "0" keeps the warp-ballot layout
    const char *mirror_env = std::getenv("WHMEC_TILE_MIRROR");
    const bool mirror_on = !(mirror_env && mirror_env[0] == '0');  // "0": every tile of every panel is computed (test hook)
    auto tnow = [] { return std::chrono::steady_clock::now(); };
    auto tms = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    const auto t0 = tnow();
    const uint32_t n = pk.n;
    ts.cols.resize(n);  // every column is written by exactly one committed panel
    const uint32_t n_chains = (uint32_t)pk.chain_begin.size() - 1;
    std::vector<std::vector<Panel>> per_chain(n_chains);
    struct Small {
        uint32_t v[32];
        uint32_t n = 0;
        void push(uint32_t x) { v[n++] = x; }
    };
    struct PanelSets { Small G, Lout, Lold, Gold; };  // fixed-size sets: no heap traffic per panel
    std::vector<std::vector<PanelSets>> per_chain_sets(n_chains);
    // per-chain results; offsets are chain-relative until all chains are planned (chains are planned by
    // independent host threads)
    std::vector<uint64_t> chain_state_words(n_chains, 0), chain_bp_words(n_chains, 0), chain_traffic(n_chains, 0);
    std::vector<std::string> chain_why(n_chains);

    // Sets of reads are small (at most 32 reads are active in a column) and are kept as ascending arrays;
    // "where does read r sit in the current column / in the tile's local order" are O(1) look-ups in
    // per-chain tables indexed by (read - first read of the chain) and validated by a stamp.
    auto plan_chain = [&](uint32_t c) -> bool {
        const uint32_t k0 = pk.chain_begin[c], k1 = pk.chain_begin[c + 1] - 1;
        uint32_t fmax = 0, rbase = 0xFFFFFFFFu, rtop = 0;
        for (uint32_t k = k0; k <= k1; ++k) {
            const ColMeta &m = pk.cols[k];
            fmax = std::max(fmax, m.f);
            if (m.a) {
                const uint32_t *reads = col_reads(pk, k);
                rbase = std::min(rbase, reads[0]);
                rtop = std::max(rtop, reads[m.a - 1]);
            }
        }
        const uint32_t nr = rbase == 0xFFFFFFFFu ? 0 : rtop - rbase + 1;
        // stamped tables: column position, position in the tile's local order, membership in L / G / Lold / Gold
        std::vector<uint32_t> col_stamp(nr, 0), cur_stamp(nr, 0), l_stamp(nr, 0), g_stamp(nr, 0), lold_stamp(nr, 0), gold_stamp(nr, 0);
        std::vector<uint8_t> col_pos(nr, 0), cur_pos(nr, 0);
        std::vector<uint8_t> sym_ok(k1 - k0 + 1, 0);
        uint32_t tick = 0;     // one per visited column
        uint32_t attempt = 0;  // one per tried tile size
        // at least 4 words so that every chain's buffers stay 16-byte aligned (vector stores of whole tiles)
        const uint64_t buf_words = std::max<uint64_t>(4, (uint64_t)1 << fmax);
        const uint64_t chain_state = 0;
        chain_state_words[c] = 2 * buf_words;
        uint64_t bp_words = 0;
        uint32_t pcount = 0;

        Small state;  // reads kept after column k-1, canonical (ascending) order
        uint32_t k = k0;
        while (k <= k1) {
            const ColMeta &m0 = pk.cols[k];
            const uint32_t fin = state.n;
            const uint32_t n_new0 = m0.a - m0.bw;
            if (fin != m0.bw && !(k == k0 && m0.bw == 0)) {
                chain_why[c] = "internal: state/backward width mismatch";
                return false;
            }
            // Candidates for the tile-local bits: the reads of the incoming state plus the reads
            // that start in this column (at a panel's first column new reads may become global, which
            // is how a chain that starts with more reads than one tile holds is cut).
            const uint32_t *reads0 = col_reads(pk, k);
            const uint32_t n_cand = state.n + n_new0;
            auto by_last = [&](uint32_t a, uint32_t b) { return pk.read_last[a] < pk.read_last[b]; };
            Small old_by_end = state, new_by_end;
            for (uint32_t q = m0.bw; q < m0.a; ++q) new_by_end.push(reads0[q]);
            std::stable_sort(old_by_end.v, old_by_end.v + old_by_end.n, by_last);
            std::stable_sort(new_by_end.v, new_by_end.v + new_by_end.n, by_last);
            // Local bits: the soonest-ending old reads (as many as the input buffer holds) and then the
            // soonest-ending new reads; everything else is global for this panel.
            int s_try = (int)std::min<uint32_t>(n_cand, TILE_MMAX);
            bool placed = false;
            uint32_t last_size = 0xFFFFFFFFu;
            for (; s_try >= 0 && !placed; --s_try) {
                const uint32_t l_old = std::min<uint32_t>({state.n, TILE_SMAX, (uint32_t)s_try});
                const uint32_t l_new = std::min<uint32_t>(n_new0, (uint32_t)s_try - l_old);
                const uint32_t s0 = l_old + l_new;
                if (s0 == last_size) continue;
                last_size = s0;
                if (n_cand - s0 > TILE_GMAX) break;
                ++attempt;
                Small Lold, Gold, G;
                for (uint32_t q = 0; q < l_old; ++q) Lold.push(old_by_end.v[q]);
                for (uint32_t q = l_old; q < old_by_end.n; ++q) Gold.push(old_by_end.v[q]);
                G = Gold;
                for (uint32_t q = l_new; q < new_by_end.n; ++q) G.push(new_by_end.v[q]);
                std::sort(G.v, G.v + G.n);
                std::sort(Lold.v, Lold.v + Lold.n);
                std::sort(Gold.v, Gold.v + Gold.n);
                for (uint32_t q = 0; q < Lold.n; ++q) l_stamp[Lold.v[q] - rbase] = attempt;
                for (uint32_t q = 0; q < l_new; ++q) l_stamp[new_by_end.v[q] - rbase] = attempt;
                for (uint32_t q = 0; q < G.n; ++q) g_stamp[G.v[q] - rbase] = attempt;
                const uint32_t n_new_local0 = l_new;
                Small Lcur = Lold;
                uint32_t n_accepted = 0;
                uint32_t j = k;
                bool ends_chain = false;
                for (; j <= k1; ++j) {
                    const ColMeta &m = pk.cols[j];
                    const uint32_t *reads = col_reads(pk, j);
                    const uint32_t n_new = (j == k) ? n_new_local0 : (m.a - m.bw);
                    const uint32_t l_in = Lcur.n;
                    const uint32_t mm = l_in + n_new;
                    if (mm > TILE_MMAX) break;
                    ++tick;
                    Small cur = Lcur;
                    for (uint32_t q = m.bw; q < m.a; ++q)  // new reads are the top bits (global ones excluded)
                        if (j != k || l_stamp[reads[q] - rbase] == attempt) cur.push(reads[q]);
                    for (uint32_t q = 0; q < cur.n; ++q) {
                        cur_stamp[cur.v[q] - rbase] = tick;
                        cur_pos[cur.v[q] - rbase] = (uint8_t)q;
                    }
                    for (uint32_t q = 0; q < m.a; ++q) {
                        col_stamp[reads[q] - rbase] = tick;
                        col_pos[reads[q] - rbase] = (uint8_t)q;
                    }
                    const bool chain_end = (m.f == 0);
                    uint32_t dropmask = 0, d = 0;
                    bool drops_global = false;
                    for (uint32_t drop = ~m.keep & low_mask(m.a); drop; drop &= drop - 1) {
                        const uint32_t r = reads[ctz32(drop)] - rbase;
                        if (cur_stamp[r] != tick) drops_global = true;
                        else {
                            dropmask |= 1u << cur_pos[r];
                            ++d;
                        }
                    }
                    if (!chain_end && drops_global) break;
                    const uint32_t l_out = mm - d;
                    if (!chain_end && l_out > TILE_SMAX) break;
                    TileCol &tc = ts.cols[j];  // a non-empty attempt is always committed, so this is final
                    std::memset(&tc, 0, sizeof tc);
                    tc.l_in = (uint8_t)l_in;
                    tc.n_new = (uint8_t)n_new;
                    tc.kind = chain_end ? 1 : 0;
                    tc.g = (uint8_t)G.n;
                    if (chain_end) {
                        tc.d = (uint8_t)mm;
                        tc.l_out = 0;
                        tc.dropmask = low_mask(mm);
                    } else {
                        tc.d = (uint8_t)d;
                        tc.l_out = (uint8_t)l_out;
                        tc.dropmask = dropmask;
                    }
                    // costs: K_A = cost of assignment A at x = 0 (pack.cpp), signed read weights
                    uint32_t K0 = TILE_KINF, K1 = TILE_KINF, K2 = TILE_KINF;
                    const uint32_t g0 = m.fn_off + pk.fn_group[m.grp_off], g1 = m.fn_off + pk.fn_group[m.grp_off + 1];
                    for (uint32_t F = g0; F < g1; ++F) {
                        const uint32_t A = pk.fn_asg[F], c0 = pk.fn_c0[F];
                        if (A == 0 || A == 3) K0 = std::min(K0, c0);
                        else if (A == 1) K1 = c0;
                        else K2 = c0;
                    }
                    tc.K0 = K0;
                    tc.K2 = (int32_t)K2;
                    tc.K12 = K1 + K2;
                    const uint8_t *alleles = pk.act_allele.data() + pk.act_off[j];
                    const uint32_t *phreds = pk.act_phred.data() + pk.act_off[j];
                    auto weight_of = [&](uint32_t read) -> int32_t {
                        const uint32_t r = read - rbase;
                        if (col_stamp[r] != tick) return 0;
                        const uint8_t al = alleles[col_pos[r]];
                        const int32_t w = (int32_t)phreds[col_pos[r]];
                        return al == 0 ? w : (al == 1 ? -w : 0);
                    };
                    uint32_t lmask_col = 0;
                    for (uint32_t q = 0; q < mm; ++q) {
                        tc.w_local[q] = weight_of(cur.v[q]);
                        if (col_stamp[cur.v[q] - rbase] == tick) lmask_col |= 1u << col_pos[cur.v[q] - rbase];
                    }
                    tc.lmask_col = lmask_col;
                    for (uint32_t b = 0; b < G.n; ++b) tc.w_global[b] = weight_of(G.v[b]);
                    uint32_t di = 0;
                    Small nextL;  // state after this column
                    for (uint32_t q = 0; q < mm; ++q) {
                        if (!((tc.dropmask >> q) & 1)) {
                            nextL.push(cur.v[q]);
                            continue;
                        }
                        if (di < 16) {
                            tc.dpos[di] = (uint8_t)q;
                            // tile-id bits of the global reads canonically above this read (G is ascending)
                            uint32_t below = 0;
                            while (below < G.n && G.v[below] <= cur.v[q]) ++below;
                            tc.gabove[di] = low_mask(G.n) & ~low_mask(below);
                        }
                        ++di;
                    }
                    // mirror rank constant (tile_device.h): rank of the complemented candidate among the candidates of the
                    // complemented output = rank ^ km,  km = inv_gray(ones_d) ^ NKA,  NKA bit i = parity of the KEPT bits
                    // (local and global) canonically above the i-th dropped bit;  chain end: km = inv_gray(ones_a)
                    {
                        uint32_t km = 0;
                        if (chain_end) {
                            for (uint32_t i = 0; i < m.a; ++i) km |= ((m.a - i) & 1u) << i;
                        } else {
                            for (uint32_t i = 0; i < d && i < 16; ++i) {
                                const uint32_t kept_above = (mm - 1 - tc.dpos[i]) - (d - 1 - i) + popc32(tc.gabove[i]);
                                km |= ((kept_above ^ (d - i)) & 1u) << i;
                            }
                        }
                        tc.km = km;
                        // symmetry of the column cost under complementing every read
                        int64_t etot = 0;
                        for (uint32_t q = 0; q < mm; ++q) etot += tc.w_local[q];
                        for (uint32_t b = 0; b < G.n; ++b) etot += tc.w_global[b];
                        const bool both_inf = K1 >= TILE_KINF && K2 >= TILE_KINF;
                        sym_ok[j - k0] = (both_inf || (K1 < TILE_KINF && K2 < TILE_KINF && (int64_t)K1 - (int64_t)K2 == etot)) ? 1 : 0;
                    }
                    if (!chain_end) {
                        uint32_t gm = 0, rank = 0;
                        for (uint32_t keep = m.keep; keep; keep &= keep - 1, ++rank)
                            if (g_stamp[reads[ctz32(keep)] - rbase] == attempt) gm |= 1u << rank;
                        tc.gmask_out = gm;
                    }
                    // kernel path hint (tile.cu: fast_kind): steady-state columns
                    if (tc.kind == 0 && tc.d == 1 && tc.dpos[0] == 0 && tc.l_out >= 10 && tc.l_in >= 1 && tc.l_in + 4 >= tc.l_out &&
                        TILE_SMAX == 14) {
                        if (tc.n_new == 1 && tc.l_out >= 11) {
                            tc.pad0 = 2;
                            tc.pad1 = (uint8_t)(tc.l_out - 11);
                        } else {
                            tc.pad0 = 1;
                            tc.pad1 = (uint8_t)(tc.l_out - 10);
                        }
                    }
                    // thread-packed back-pointer bits where a thread owns 8 or 16 outputs (default; WHMEC_TILE_PACKED_BP=0: warp ballots)
                    if (packed_bp && tc.pad0) {
                        const uint32_t per_thread = (1u << tc.pad1) << (tc.pad0 == 2 ? 1 : 0);
                        if (per_thread == 8 || per_thread == 16) tc.pad2 = 1;
                    }
                    ++n_accepted;
                    Lcur = nextL;
                    if (chain_end) {
                        ends_chain = true;
                        ++j;
                        break;
                    }
                }
                if (n_accepted == 0) continue;  // try a smaller tile
                // commit the panel [k, j)
                for (uint32_t q = 0; q < Lold.n; ++q) lold_stamp[Lold.v[q] - rbase] = attempt;
                for (uint32_t q = 0; q < Gold.n; ++q) gold_stamp[Gold.v[q] - rbase] = attempt;
                Panel P;
                std::memset(&P, 0, sizeof P);
                P.chain = c;
                P.col_begin = k;
                P.col_end = j;
                P.g = G.n;
                P.s_in = Lold.n;
                for (uint32_t q = 0; q < state.n; ++q) {
                    if (lold_stamp[state.v[q] - rbase] == attempt) P.lmask_in |= 1u << q;
                    if (gold_stamp[state.v[q] - rbase] == attempt) P.gmask_in |= 1u << q;
                }
                P.ends_chain = ends_chain ? 1 : 0;
                P.fresh = (k == k0) ? 1 : 0;
                P.in_off = chain_state + (uint64_t)(pcount & 1) * buf_words;
                P.out_off = chain_state + (uint64_t)((pcount + 1) & 1) * buf_words;
                Small kept;
                if (!ends_chain) {
                    const ColMeta &ml = pk.cols[j - 1];
                    const uint32_t *reads = col_reads(pk, j - 1);
                    for (uint32_t keep = ml.keep; keep; keep &= keep - 1) kept.push(reads[ctz32(keep)]);
                    P.s_out = Lcur.n;
                    // Lcur is the local order after column j-1, whose tick is still current
                    for (uint32_t q = 0; q < kept.n; ++q) {
                        bool in_lcur = false;
                        for (uint32_t z = 0; z < Lcur.n; ++z) in_lcur |= (Lcur.v[z] == kept.v[q]);
                        if (in_lcur) P.lmask_out |= 1u << q;
                        if (g_stamp[kept.v[q] - rbase] == attempt) P.gmask_out |= 1u << q;
                    }
                    chain_traffic[c] += 2ull * 4ull * ((uint64_t)1 << kept.n);
                }
                // Mirrored panel (Panel::half): needs cost(x) == cost(~x) in every column, i.e. K1 == K2 + (sum of all signed
                // weights) or no heterozygous assignment at all -- always true for the reference's cost form; checked anyway.
                bool half = mirror_on && G.n >= 1;
                for (uint32_t q = k; q < j && half; ++q) half = sym_ok[q - k0] != 0;
                P.half = half ? 1 : 0;
                for (uint32_t q = k; q < j; ++q) {
                    TileCol &tc = ts.cols[q];
                    tc.bp_width = tc.kind == 1 ? 0 : round_bp_width(tc.d);
                    tc.bp_off = bp_words;
                    // every tile's slice starts on a word boundary
                    uint64_t per_tile_words = ((((uint64_t)1 << tc.l_out) * tc.bp_width) + 31) / 32;
                    tc.bp_tile_words = (uint32_t)per_tile_words;
                    tc.half = half ? 1 : 0;
                    if (!half) tc.km = 0;  // (computed per column below; only meaningful for mirrored panels)
                    const uint32_t sections = (half && tc.km != 0 && tc.kind == 0) ? 2 : 1;
                    tc.bp_tile_stride = (uint32_t)(per_tile_words * sections);
                    bp_words += (per_tile_words * sections) << (tc.g - (half ? 1 : 0));
                }
                P.in_gold = Gold.n;
                {  // steady-state panel?
                    const TileCol &t0 = ts.cols[k];
                    bool steady = !ends_chain && j - k <= 16 && t0.pad0 == 2 && (t0.pad2 & 1u) && (t0.pad1 == 2 || t0.pad1 == 3);
                    for (uint32_t q = k; q < j && steady; ++q) {
                        const TileCol &tc = ts.cols[q];
                        steady = tc.kind == 0 && tc.pad0 == 2 && tc.pad1 == t0.pad1 && (tc.pad2 & 1u) && tc.K0 >= TILE_KINF &&
                                 tc.l_in == t0.l_in && tc.l_out == t0.l_out && (tc.half && tc.km != 0) == (t0.half && t0.km != 0);
                    }
                    P.steady = steady ? 1u + t0.pad1 : 0u;
                }
                per_chain[c].push_back(P);
                per_chain_sets[c].push_back(PanelSets{G, Lcur, Lold, Gold});
                ++pcount;
                state = kept;
                k = j;
                placed = true;
            }
            if (!placed) {
                chain_why[c] = "a column drops more reads at once than a tile can hold";
                return false;
            }
        }
        chain_bp_words[c] = bp_words;
        return true;
    };
    {
        const uint32_t nthreads = std::min(host_threads(32), std::max(1u, n_chains / 2));
        std::atomic<bool> failed{false};
        parallel_tasks(n_chains, nthreads, [&](uint32_t c) {
            if (!failed.load() && !plan_chain(c)) failed.store(true);
        });
        if (failed.load()) {
            for (uint32_t c = 0; c < n_chains; ++c)
                if (!chain_why[c].empty()) {
                    ts.why = chain_why[c];
                    break;
                }
            return;
        }
    }
    const auto t1 = tnow();
    // make the chain-relative offsets absolute: a prefix over the chains, then every chain on its own (host threads)
    std::vector<uint64_t> state_base(n_chains + 1, 0), bp_base(n_chains + 1, 0);
    size_t max_panels = 0;
    for (uint32_t c = 0; c < n_chains; ++c) {
        state_base[c + 1] = state_base[c] + chain_state_words[c];
        bp_base[c + 1] = bp_base[c] + chain_bp_words[c];
        ts.state_traffic_bytes += chain_traffic[c];
        max_panels = std::max(max_panels, per_chain[c].size());
    }
    const uint64_t state_words = state_base[n_chains], bp_words = bp_base[n_chains];
    const uint32_t asm_threads = std::min(host_threads(32), std::max(1u, n_chains / 2));
    parallel_tasks(n_chains, asm_threads, [&](uint32_t c) {
        for (Panel &P : per_chain[c]) {
            P.in_off += state_base[c];
            P.out_off += state_base[c];
        }
        if (bp_base[c])
            for (uint32_t k = pk.chain_begin[c]; k < pk.chain_begin[c + 1]; ++k) ts.cols[k].bp_off += bp_base[c];
        // the chain's records are final: out of this thread's cache, ready for the DMA engine (WHMEC_FLUSH_UPLOAD=1)
        if (stage_flush_enabled())
            stage_flush(&ts.cols[pk.chain_begin[c]], (size_t)(pk.chain_begin[c + 1] - pk.chain_begin[c]) * sizeof(TileCol));
        // hand-off layouts between consecutive panels of the chain (see Panel in tile_plan.h)
        for (size_t q = 0; q + 1 < per_chain[c].size(); ++q) {
            Panel &A = per_chain[c][q], &B = per_chain[c][q + 1];
            const PanelSets &sa = per_chain_sets[c][q], &sb = per_chain_sets[c][q + 1];
            if (A.ends_chain) continue;
            B.in_half = A.half;
            B.in_top = 0;
            for (uint32_t gmk = A.gmask_out; gmk; gmk &= gmk - 1) B.in_top = gmk & (0u - gmk);  // highest set bit = top global read
            if (sa.G.n && sa.Lout.n && sa.G.v[sa.G.n - 1] > sa.Lout.v[0]) continue;  // producer's global reads must be the oldest
            if (sb.Lold.n < sa.G.n) continue;
            const size_t j = sb.Lold.n - sa.G.n;
            if (j < 2 || j > sa.Lout.n) continue;  // chunks of at least 4 entries
            // the consumer's old local reads must be the producer's global reads followed by its first j local reads
            if (!std::equal(sa.G.v, sa.G.v + sa.G.n, sb.Lold.v) || !std::equal(sa.Lout.v, sa.Lout.v + j, sb.Lold.v + sa.G.n)) continue;
            A.out_layout = 1;
            B.in_layout = 1;
            B.in_gA = sa.G.n;
            B.in_j = (uint32_t)j;
            B.in_sA = A.s_out;
        }
    });

    // launch rounds: round r = r-th panel of every chain that has one; every round fills its own slice of the panel array
    ts.round_begin.assign(max_panels + 1, 0);
    for (uint32_t c = 0; c < n_chains; ++c)
        for (size_t r = 0; r < per_chain[c].size(); ++r) ++ts.round_begin[r + 1];
    for (size_t r = 0; r < max_panels; ++r) ts.round_begin[r + 1] += ts.round_begin[r];
    ts.panels.resize(ts.round_begin[max_panels]);
    ts.round_tiles.assign(max_panels, 0);
    ts.round_tile_log.assign(max_panels, -1);
    parallel_tasks((uint32_t)max_panels, asm_threads, [&](uint32_t r) {
        uint32_t tiles = 0, at = ts.round_begin[r];
        int32_t tlog = -1;
        bool uniform = true;
        for (uint32_t c = 0; c < n_chains; ++c)
            if (r < per_chain[c].size()) {
                Panel &P = ts.panels[at];
                P = per_chain[c][r];
                P.tile_begin = tiles;
                tiles += 1u << (P.g - P.half);
                const int32_t mine = (int32_t)(P.g - P.half);
                if (at == ts.round_begin[r]) tlog = mine;
                else if (tlog != mine) uniform = false;
                ++at;
            }
        ts.round_tiles[r] = tiles;
        ts.round_tile_log[r] = (uniform && tlog >= 0) ? tlog : -1;
    });
    ts.state_words = state_words;
    ts.bp_words = bp_words;
    ts.eligible = true;
    if (timing) std::fprintf(stderr, "[whmec] plan: chains %.2f ms, assemble %.2f ms\n", tms(t0, t1), tms(t1, tnow()));
}

}  // namespace whmec
