// Host planner of the column-kernel paths (col_plan.h).
#include "col_plan.h"

#include <algorithm>

#include "bounded.h"
#include "dp_device.h"
#include "ped_fused.h"

namespace whmec {

namespace {

constexpr uint64_t RESERVE = 512ull << 20;  // free HBM left to everything else on the device

// The launches of one pass of the batched sweep over chains [c_lo, c_hi), appended to plan.steps.
//   pass 0: chain 0 (true input) and, without the multi-RHS kernel, every (chain, unit vector);
//   pass 1: chains with their true inputs, back-pointers written; pass 2: one multi-RHS instance per chain >= 1.
// With the multi-RHS kernel pass 0 is empty: chain 0 (whose input is known: the first column of the table ignores it) runs in
// pass 1 like every other chain.
void add_steps(const Packed &pk, ColPlan &plan, int pass, uint32_t c_lo, uint32_t c_hi, std::vector<uint32_t> &begin,
               std::vector<uint32_t> &grid) {
    const uint32_t T = pk.T, C = (uint32_t)pk.chain_begin.size() - 1;
    const std::vector<uint32_t> &clen = plan.clen;
    auto blocks_for = [&](const ColMeta &m) -> uint32_t {
        const uint64_t nent = ((uint64_t)1 << m.f) * T;
        if (m.d > 7) return (uint32_t)nent;
        const uint64_t epb = 256u >> col_lane_bits(m.f + pk.tb, m.d);
        return (uint32_t)((nent + epb - 1) / epb);
    };
    uint32_t len = 0;
    for (uint32_t c = c_lo; c < c_hi; ++c) len = std::max(len, clen[c]);
    for (uint32_t st = 0; st < len; ++st) {
        begin.push_back((uint32_t)plan.steps.size());
        uint32_t gmax = 0;
        const uint32_t c_begin = (pass == 0 && !plan.ped_multi) ? c_lo : (pass == 0 ? c_hi : c_lo);
        for (uint32_t c = c_begin; c < c_hi; ++c) {
            if (clen[c] <= st) continue;
            const uint32_t kcol = pk.chain_begin[c] + st;
            const ColMeta &m = pk.cols[kcol];
            const uint32_t reps = pass == 0 ? T : 1;
            // a column hands transition minima to the next one of its chain when the T values of a
            // projection index are produced inside one thread block
            auto xform = [&](uint32_t k) {
                const ColMeta &q = pk.cols[k];
                return k + 1 < pk.chain_begin[c + 1] && q.d <= 7 && T <= (256u >> col_lane_bits(q.f + pk.tb, q.d));
            };
            for (uint32_t u = 0; u < reps; ++u) {
                PedStep ps;
                ps.cm = m;
                ps.nf = pk.fn_group[m.grp_off + T];
                ps.slot = pass == 1 ? (C * T + c) : (c * T + u);
                ps.flags = pass == 1 ? 1u : 0u;
                if (xform(kcol)) ps.flags |= 2u;
                if (st > 0 && xform(kcol - 1)) ps.flags |= 4u;
                if (pass == 2 && st == 0) ps.flags |= 8u;
                ps.rc_next = kcol + 1 < pk.n ? pk.cols[kcol + 1].rc : 0;
                plan.steps.push_back(ps);
            }
            gmax = std::max(gmax, blocks_for(m));
        }
        grid.push_back(gmax);
    }
    begin.push_back((uint32_t)plan.steps.size());
}

}  // namespace

int col_plan(Packed &pk, const ColPlanInput &in, ColPlan &plan, std::string &msg) {
    plan = ColPlan{};
    const uint32_t n = pk.n, T = pk.T, C = (uint32_t)pk.chain_begin.size() - 1;
    for (const ColMeta &m : pk.cols) plan.max_ent = std::max<uint64_t>(plan.max_ent, ((uint64_t)1 << m.f) * T);
    const uint64_t max_ent = plan.max_ent, free_b = in.free_bytes, hook = in.hook;
    const bool wide = T > MAX_T;  // five trios: only the wide column sweep, which also holds the transformed projection (4 + 2 bytes)
    const uint64_t need = pk.bp_words * 4 + max_ent * (4 * 2 + 8 + (wide ? 6 : 0)) + pk.fn_delta.size() * 4 + (uint64_t)n * sizeof(ColMeta);
    const uint64_t fixed = need - pk.bp_words * 4;  // everything but the back-pointers
    plan.fixed_bytes = fixed;
    const uint64_t hbm_budget = free_b > fixed + RESERVE ? free_b - fixed - RESERVE : 0;
    // the hook's budget is the arena's, checkpoints come on top (as with WHMEC_TILE_ARENA_BUDGET); the free HBM's covers both
    const bool over_hbm = need + RESERVE > free_b, over_hook = hook && pk.bp_words * 4 > hook;
    // single individuals: solve_impl first solves groups of chains one after another (grouped.h); the bounded sweep is for
    // what no group size fits (bounded_t1)
    plan.bounded = !in.segment && (over_hook || (over_hbm && (T > 1 || in.bounded_t1)));
    if (over_hbm && !plan.bounded) {
        plan.over_hbm = true;
        msg = "back-pointer storage exceeds the free HBM of this device";
        return WHMEC_ERR_UNSUPPORTED;
    }
    // which sweep: pedigrees with several chains take a two-pass sweep (fused trio kernel or batched), the rest the column sweep
    const bool two_pass_shape = !wide && (C >= 2 || in.segment) && pk.safe31 && !(in.sequential && !in.segment);
    // one trio, shapes of ped_fused.h: one block per chain with the projection in shared memory (3 launches)
    bool fused = in.fused && T == PF_T && two_pass_shape;
    for (uint32_t k = 0; k < n && fused; ++k) fused = pf_column_ok(pk.cols[k], pk.fn_group.data() + pk.cols[k].grp_off);
    // batched sweep: the batch buffers (values + argmins of every (chain, unit vector) instance) count against the free HBM as well
    plan.slots = (uint64_t)C * T + C;
    const uint64_t batch_bytes = plan.slots * 2 * max_ent * 5;
    auto batch_ok = [&](uint64_t arena_bytes) {
        return T > 1 && two_pass_shape && plan.slots * 2 * max_ent * 4 < (8ull << 30) && (uint64_t)C * T <= 65535 &&
               fixed + arena_bytes + batch_bytes + RESERVE <= free_b;
    };
    plan.arena_words = pk.bp_words;
    bool two_pass = true;  // (resident: whatever the conditions above allow)
    if (plan.bounded) {
        std::vector<uint64_t> off(n + 1);
        for (uint32_t k = 0; k < n; ++k) off[k] = pk.cols[k].bp_off;
        off[n] = pk.bp_words;
        // two-pass sweeps: segments of whole chains, after pass 1 every chain's input is known (no checkpoints)
        two_pass = false;
        if (fused || batch_ok(0)) {
            plan.budget_bytes = over_hook ? hook : fused ? hbm_budget : (hbm_budget > batch_bytes ? hbm_budget - batch_bytes : 0);
            two_pass = cut_chain_segments(pk.chain_begin, off, plan.budget_bytes / 4, plan.seg_chain, plan.arena_words) &&
                       (fused || batch_ok(plan.arena_words * 4));
        }
        std::vector<uint32_t> cuts;  // column cuts of the segments
        if (two_pass) {
            for (uint32_t c : plan.seg_chain) cuts.push_back(pk.chain_begin[c]);
        } else {  // a chain alone exceeds the budget, or no two-pass sweep: column sweep with checkpoints
            plan.seg_chain.clear();
            fused = false;
            std::vector<uint64_t> ck(n);
            uint64_t widest = 0, widest_ck = 0;
            for (uint32_t k = 0; k < n; ++k) {
                ck[k] = ((uint64_t)1 << pk.cols[k].f) * T;
                widest = std::max(widest, off[k + 1] - off[k]);
                widest_ck = std::max(widest_ck, ck[k]);
            }
            plan.budget_bytes = over_hook ? hook : hbm_budget;
            // (the hook's cut counts the arena alone against the free HBM)
            const bool fits = over_hook ? cut_column_segments(off, {}, hook / 4, plan.seg_col, plan.arena_words, plan.ckpt_words) &&
                                              fixed + 4 * plan.arena_words + RESERVE <= free_b
                                        : cut_column_segments(off, ck, hbm_budget / 4, plan.seg_col, plan.arena_words, plan.ckpt_words);
            if (!fits) {
                msg = over_hook ? "memory-bounded sweep: an arena of " + std::to_string(hook) + " bytes holds no segment; it needs at least " +
                                      std::to_string(4 * widest) + " bytes (the widest column's back-pointers), checkpoints on top"
                                : "memory-bounded sweep: " + std::to_string(hbm_budget) + " bytes of free HBM hold no segment; it needs at least " +
                                      std::to_string(4 * (widest + widest_ck)) + " bytes (the widest column's back-pointers and the largest checkpoint)";
                return WHMEC_ERR_UNSUPPORTED;
            }
            // segment s >= 1 starts from the values column seg_col[s] - 1 hands on
            plan.seg_ckpt.assign(plan.seg_col.size() - 1, 0);
            plan.ckpt_words = 0;
            for (size_t sg = 1; sg + 1 < plan.seg_col.size(); ++sg) {
                plan.seg_ckpt[sg] = plan.ckpt_words;
                plan.ckpt_words += ck[plan.seg_col[sg] - 1];
            }
            cuts = plan.seg_col;
        }
        for (size_t sg = 0; sg + 1 < cuts.size(); ++sg)
            for (uint32_t k = cuts[sg]; k < cuts[sg + 1]; ++k) pk.cols[k].bp_off -= off[cuts[sg]];
    }
    if (fused) {
        plan.path = ColPath::fused;
        // fewer chains than SMs: a cluster of 2 / 4 / 8 CTAs per chain (WHMEC_PED_CLUSTER=n forces n, 1 = off)
        uint32_t cs = 1;
        while (cs * 2 <= PF_MAX_CLUSTER && (uint64_t)C * cs * 2 <= (uint64_t)in.sms) cs *= 2;
        if (in.cluster == 1 || in.cluster == 2 || in.cluster == 4 || in.cluster == 8) cs = in.cluster;
        plan.cluster = cs;
    } else if (two_pass && batch_ok(plan.arena_words * 4)) {
        plan.path = ColPath::batched;
        plan.clen.resize(C);
        for (uint32_t c = 0; c < C; ++c) plan.clen[c] = pk.chain_begin[c + 1] - pk.chain_begin[c];
        plan.ped_multi = T <= MULTI_MAX;
        for (int pass = 0; pass < 3; ++pass) {
            if (pass == 2 && !plan.ped_multi) continue;
            if (pass == 1 && plan.bounded) continue;  // per segment, below
            add_steps(pk, plan, pass, 0, C, plan.ped_begin[pass], plan.ped_grid[pass]);
        }
        if (plan.bounded) {
            const size_t S = plan.seg_chain.size() - 1;
            plan.seg_begin.assign(S, {});
            plan.seg_grid.assign(S, {});
            for (size_t sg = 0; sg < S; ++sg) add_steps(pk, plan, 1, plan.seg_chain[sg], plan.seg_chain[sg + 1], plan.seg_begin[sg], plan.seg_grid[sg]);
        }
    }
    if (wide) plan.path = ColPath::wide;
    if (in.segment && !plan.two_pass()) {
        msg = "unsupported: this segment cannot run the two-pass pedigree sweep (costs beyond 2^28 or state beyond the budget)";
        return WHMEC_ERR_UNSUPPORTED;
    }
    return WHMEC_OK;
}

}  // namespace whmec
