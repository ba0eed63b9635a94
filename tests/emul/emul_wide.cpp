// TEST-ONLY host emulation of the wide column sweep (T = 1024, DESIGN §4.7): steps the per-thread code of wide_xform_kernel and
// wide_step_kernel (whatshap_b200/csrc/wide_device.h) round by round and chunk by chunk, finalizes keys as col_finalize_kernel
// does, walks the back-pointers with backtrace_range and builds the outputs with the product's build_outputs.  Also exposes the
// planner's route for five-trio tables.  Built into tests/emul/libwhemul_wide.so by tests/emul/wide.mk.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "../../whatshap_b200/csrc/col_plan.h"
#include "../../whatshap_b200/csrc/hostpool.h"
#include "../../whatshap_b200/csrc/wide_device.h"

using namespace whmec;

namespace {

int fail_with(const std::string &msg, char *err, size_t errlen, int code) {
    if (err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = 0;
    }
    return code;
}

// wide_xform_kernel on `rows` blocks: the same relaxation rounds, every lane reading the keys of the previous round
void xform_rows(const uint32_t *prev /* nullptr: zeros */, uint64_t rows, uint32_t rc, uint32_t *prevm, uint16_t *prevarg) {
    std::vector<uint64_t> key(WIDE_T), next(WIDE_T);
    for (uint64_t b = 0; b < rows; ++b) {
        for (uint32_t i = 0; i < WIDE_T; ++i) key[i] = wide_key(prev ? prev[b * WIDE_T + i] : 0u, i);
        for (uint32_t q = 0; q < WIDE_TB; ++q) {
            for (uint32_t i = 0; i < WIDE_T; ++i) next[i] = wide_relax(key[i], key[i ^ (1u << q)], rc);
            key.swap(next);
        }
        for (uint32_t i = 0; i < WIDE_T; ++i) {
            prevm[b * WIDE_T + i] = wide_key_value(key[i]);
            prevarg[b * WIDE_T + i] = wide_key_arg(key[i]);
        }
    }
}

}  // namespace

// The transform of `rows` rows of 1024 values next to transition_min on the same rows (first != 0: the rows are ignored, as for
// the table's first column).  vals/args: the transform; ref_vals/ref_args: transition_min.  [rows][1024] each.
extern "C" void whemul_wide_xform(const uint32_t *prev, uint64_t rows, uint32_t rc, int first, uint32_t *vals, uint16_t *args,
                                  uint32_t *ref_vals, uint32_t *ref_args) {
    xform_rows(first ? nullptr : prev, rows, rc, vals, args);
    std::vector<uint32_t> zero(WIDE_T, 0);
    for (uint64_t b = 0; b < rows; ++b)
        for (uint32_t i = 0; i < WIDE_T; ++i)
            ref_vals[b * WIDE_T + i] = transition_min(first ? zero.data() : prev + b * WIDE_T, WIDE_T, i, rc, &ref_args[b * WIDE_T + i]);
}

// The wide sweep of a five-trio table on the host.  transform: 1 transformed projection (exact when Packed::nowrap), 0 raw values
// through eval_candidates' O(T) loop, -1 as the device chooses (transform iff nowrap).  info[3]: nowrap, the columns that ran the
// transform, the largest chunk split (wide_chunk_bits).
extern "C" int whemul_wide_solve(const whmec_problem *p, int transform, whmec_solution *s, uint32_t *info, char *err, size_t errlen) {
    Packed pk;
    std::string msg;
    int rc = pack_problem(p, pk, msg, true);
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    if (pk.T != WIDE_T || pk.n == 0) return fail_with("the wide sweep is for five-trio tables with columns", err, errlen, WHMEC_ERR_INPUT);
    if (pk.max_d + pk.tb > 32) return fail_with("unsupported: dropped reads + transmission bits exceed 32", err, errlen, WHMEC_ERR_UNSUPPORTED);
    const uint32_t n = pk.n, T = pk.T, tb = pk.tb;
    const bool xform = transform < 0 ? pk.nowrap : transform != 0;
    uint64_t max_ent = 1;
    for (const ColMeta &m : pk.cols) max_ent = std::max<uint64_t>(max_ent, ((uint64_t)1 << m.f) * T);
    std::vector<uint32_t> arena(pk.bp_words + 1, 0), vals[2] = {std::vector<uint32_t>(max_ent), std::vector<uint32_t>(max_ent)};
    std::vector<uint32_t> prevm(max_ent);
    std::vector<uint16_t> prevarg(max_ent);
    std::vector<uint64_t> keys(max_ent);
    uint32_t n_xform = 0, max_L = 0;
    for (uint32_t k = 0; k < n; ++k) {
        const ColMeta &m = pk.cols[k];
        const uint32_t *prev = vals[(k & 1) ^ 1].data();
        uint32_t *out = vals[k & 1].data();
        ColMeta mk = m;
        if (xform) {
            xform_rows(m.first ? nullptr : prev, m.first ? 1 : (uint64_t)1 << m.bw, m.rc, prevm.data(), prevarg.data());
            mk.first = 0;
            ++n_xform;
        }
        const uint32_t L = wide_chunk_bits(m.f, m.d);
        max_L = std::max(max_L, L);
        const uint64_t nent = ((uint64_t)1 << m.f) * T;
        const uint32_t tasks = (uint32_t)std::min<uint64_t>(nent / 1024 + 1, 256);
        parallel_tasks(tasks, host_threads(32), [&](uint32_t t) {
            for (uint64_t e = nent * t / tasks; e < nent * (t + 1) / tasks; ++e) {
                const uint32_t o = (uint32_t)(e >> WIDE_TB), i = (uint32_t)e & (WIDE_T - 1);
                const uint32_t g0 = pk.fn_group[m.grp_off + i], g1 = pk.fn_group[m.grp_off + i + 1];
                ColView v;
                v.m = &mk;
                v.T = T;
                v.tb = tb;
                v.fn_c0 = pk.fn_c0.data() + m.fn_off + g0;
                v.fn_delta = pk.fn_delta.data() + (size_t)(m.fn_off + g0) * FN_STRIDE;
                v.nf = g1 - g0;
                v.prev = prev;
                v.tab = nullptr;
                v.tab_fn0 = 0;
                v.prevm = xform ? prevm.data() : nullptr;
                v.prevarg16 = prevarg.data();
                uint64_t key = KEY_INF;
                for (uint32_t c = 0; c < (1u << L); ++c) key = std::min(key, wide_entry_key(v, o, i, c, L));
                keys[e] = key;
            }
        });
        for (uint64_t e = 0; e < nent; ++e) {  // col_finalize_kernel
            out[e] = (uint32_t)(keys[e] >> 32);
            bp_store_serial(arena.data(), m.bp_off, m.bp_width, e, (uint32_t)keys[e] & low_mask(m.d + tb));
        }
    }
    std::vector<uint32_t> path_index(n), path_tv(n);
    uint32_t cost, x, tv, ptv;
    const BtView bv{pk.cols.data(), arena.data(), T, tb};
    pick_optimum(pk.cols[n - 1], vals[(n - 1) & 1].data(), arena.data(), T, tb, &cost, &x, &tv, &ptv);
    backtrace_range(bv, n - 1, 0, x, tv, ptv, path_index.data(), path_tv.data());
    s->cost = cost;
    info[0] = pk.nowrap;
    info[1] = n_xform;
    info[2] = max_L;
    rc = build_outputs(pk, path_index.data(), path_tv.data(), s, msg);
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    return WHMEC_OK;
}

// col_plan for the given free bytes and WHMEC_COLUMN_ARENA_BUDGET hook.  info[5]: path (0 column, 1 batched, 2 fused, 3 wide),
// bounded, arena words, checkpoint words, resident back-pointer words.  cuts: the column cuts of a bounded plan ([cap]).
extern "C" int whemul_wide_plan(const whmec_problem *p, uint64_t free_bytes, uint64_t hook, int segment, uint64_t *info, uint32_t *cuts,
                                uint32_t *n_cuts, uint32_t cap, char *err, size_t errlen) {
    Packed pk;
    std::string msg;
    int rc = pack_problem(p, pk, msg, true);
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    ColPlanInput in;
    in.free_bytes = free_bytes;
    in.hook = hook;
    in.segment = segment;
    ColPlan plan;
    const uint64_t bp_words = pk.bp_words;
    rc = col_plan(pk, in, plan, msg);
    const uint64_t out[5] = {(uint64_t)plan.path, plan.bounded, plan.arena_words, plan.ckpt_words, bp_words};
    std::copy(out, out + 5, info);
    const std::vector<uint32_t> &c = plan.seg_chain.empty() ? plan.seg_col : plan.seg_chain;
    *n_cuts = (uint32_t)std::min<size_t>(c.size(), cap);
    std::copy(c.begin(), c.begin() + *n_cuts, cuts);
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    return WHMEC_OK;
}
