// TEST-ONLY host emulation of the column kernel's driver loop.
//
// Runs pack.cpp and the __host__ __device__ per-thread functions of dp_device.h (the same code
// the CUDA kernels execute) serially on the CPU so that their logic can be checked against the
// oracle on a machine without a GPU.  It is built into tests/emul/libwhemul.so by
// tests/emul/Makefile, loaded only by tests/test_emulation.py, and is NOT a fallback: the product
// library (whatshap_b200/csrc) contains no CPU execution path.
#include <algorithm>
#include <atomic>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../whatshap_b200/csrc/hostpool.h"
#include "../../whatshap_b200/csrc/pack.h"
#include "../../whatshap_b200/csrc/dp_device.h"
#include "../../whatshap_b200/csrc/ped_fused.h"
#include <memory>

using namespace whmec;

namespace {

int fail_with(const std::string &msg, char *err, size_t errlen, int code) {
    if (err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = 0;
    }
    return code;
}

// Columns [k0, k1) swept one after the other, every thread's work done serially.  `prev` holds the
// projection handed to column k0 (ignored by a column with m.first) and ends as column k1-1's.
int sweep_columns(const Packed &pk, uint32_t k0, uint32_t k1, uint32_t chunk, std::vector<uint32_t> &prev,
                  std::vector<uint32_t> &arena, std::string &msg) {
    const uint32_t T = pk.T, tb = pk.tb;
    std::vector<uint32_t> cur, prevm;
    std::vector<uint8_t> prevarg;
    bool have_xform = false;
    for (uint32_t k = k0; k < k1; ++k) {
        const ColMeta &m = pk.cols[k];
        if (m.d + tb > 32) { msg = "d + tb > 32"; return WHMEC_ERR_UNSUPPORTED; }
        uint64_t nout = (uint64_t)1 << m.f, ncand = (uint64_t)1 << m.d;
        cur.assign(nout * T, UMAX);
        // per-column lookup tables, as a thread block builds them in shared memory
        const uint32_t nf_col = pk.fn_group[m.grp_off + T];
        std::vector<uint32_t> pd_lo(TAB_SIZE), pd_hi(TAB_SIZE);
        std::vector<int32_t> tlo((size_t)nf_col * TAB_SIZE), thi((size_t)nf_col * TAB_SIZE);
        const uint32_t keep_lo = lowest_set_bits(m.keep, TAB_BITS), keep_hi = lowest_set_bits(m.keep & ~keep_lo, TAB_BITS);
        for (uint32_t vv = 0; vv < TAB_SIZE; ++vv) {
            pd_lo[vv] = pdep32(vv, keep_lo);
            pd_hi[vv] = pdep32(vv, keep_hi);
        }
        for (uint32_t F = 0; F < nf_col; ++F)
            for (uint32_t half = 0; half < 2; ++half)
                for (uint32_t hi4 = 0; hi4 < 16; ++hi4)
                    build_cost_table_run(pk.fn_delta.data() + (size_t)(m.fn_off + F) * FN_STRIDE, half, hi4,
                                         (half ? thi.data() : tlo.data()) + (size_t)F * TAB_SIZE + 16 * hi4);
        ColTables tab{pd_lo.data(), pd_hi.data(), m.keep & ~keep_lo & ~keep_hi, tlo.data(), thi.data()};
        const bool use_tab = (k % 2) == 0;  // exercise both initialisation paths
        for (uint64_t o = 0; o < nout; ++o)
            for (uint32_t i = 0; i < T; ++i) {
                ColView v;
                v.m = &m; v.T = T; v.tb = tb;
                uint32_t g0 = pk.fn_group[m.grp_off + i], g1 = pk.fn_group[m.grp_off + i + 1];
                v.fn_c0 = pk.fn_c0.data() + m.fn_off + g0;
                v.fn_delta = pk.fn_delta.data() + (size_t)(m.fn_off + g0) * FN_STRIDE;
                v.nf = g1 - g0;
                v.prev = prev.data();
                v.tab = use_tab ? &tab : nullptr;
                v.tab_fn0 = g0;
                v.prevm = have_xform ? prevm.data() : nullptr;
                v.prevarg = have_xform ? prevarg.data() : nullptr;
                uint64_t best = KEY_INF;
                uint64_t step = chunk ? chunk : ncand;
                for (uint64_t r0 = 0; r0 < ncand; r0 += step) {  // chunked like the atomic kernel
                    uint64_t r1 = r0 + step < ncand ? r0 + step : ncand;
                    uint64_t key = eval_candidates(v, (uint32_t)o, i, (uint32_t)r0, (uint32_t)r1);
                    if (key < best) best = key;
                }
                cur[o * T + i] = (uint32_t)(best >> 32);
                bp_store_serial(arena.data(), m.bp_off, m.bp_width, o * T + i, (uint32_t)best & low_mask(m.d + tb));
            }
        prev.swap(cur);
        // every third hand-over keeps raw values, the others pre-apply the transition minimum of the next
        // column (as the batched pedigree kernels do in their epilogue)
        // (only when sums cannot wrap: the product uses transition minima on the batched path, which requires pk.safe31)
        have_xform = pk.safe31 && (k + 1 < k1) && (k % 3 != 2);
        if (have_xform) {
            prevm.assign(nout * T, UMAX);
            prevarg.assign(nout * T, 0);
            for (uint64_t o = 0; o < nout; ++o)
                for (uint32_t i = 0; i < T; ++i) {
                    uint32_t arg;
                    prevm[o * T + i] = transition_min(&prev[o * T], T, i, pk.cols[k + 1].rc, &arg);
                    prevarg[o * T + i] = (uint8_t)arg;
                }
        }
    }
    return WHMEC_OK;
}

}  // namespace

extern "C" int whemul_solve(const whmec_problem *p, whmec_solution *s, uint32_t chunk, char *err, size_t errlen) {
    Packed pk;
    std::string msg;
    int rc = pack_problem(p, pk, msg);
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    const uint32_t n = pk.n, T = pk.T, tb = pk.tb;
    if (n == 0) {
        s->cost = 0;
        if (s->partition) std::memset(s->partition, 1, p->n_reads);
        return WHMEC_OK;
    }
    std::vector<uint32_t> arena(pk.bp_words + 1, 0), prev;
    rc = sweep_columns(pk, 0, n, chunk, prev, arena, msg);
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    std::vector<uint32_t> pidx(n), ptv(n);
    BtView bv{pk.cols.data(), arena.data(), T, tb};
    uint32_t cost, x, tv, ptvv;
    pick_optimum(pk.cols[n - 1], prev.data(), arena.data(), T, tb, &cost, &x, &tv, &ptvv);
    backtrace_range(bv, n - 1, 0, x, tv, ptvv, pidx.data(), ptv.data());
    s->cost = cost;
    rc = build_outputs(pk, pidx.data(), ptv.data(), s, msg);
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    return WHMEC_OK;
}

// ---- segments of a pedigree table: same entry points and semantics as whmec_segment_* (include/whmec.h),
// ---- built from the same __host__ __device__ functions the CUDA kernels call
struct whemul_segment {
    Packed pk;
    bool continues = false;
    std::vector<uint32_t> arena, last_vals, exits;
    bool swept = false;
};

extern "C" int whemul_segment_create(const whmec_problem *p, int continues, whemul_segment **out, char *err, size_t errlen) {
    std::string msg;
    whemul_segment *sg = new whemul_segment();
    *out = nullptr;
    int rc = pack_problem(p, sg->pk, msg);
    if (rc == WHMEC_OK && (sg->pk.T == 1 || sg->pk.n == 0 || !sg->pk.safe31)) {
        msg = "unsupported segment";
        rc = WHMEC_ERR_UNSUPPORTED;
    }
    if (rc != WHMEC_OK) {
        delete sg;
        return fail_with(msg, err, errlen, rc);
    }
    sg->continues = continues != 0;
    if (sg->continues) sg->pk.cols[0].first = 0;
    sg->arena.assign(sg->pk.bp_words + 1, 0);
    *out = sg;
    return WHMEC_OK;
}

extern "C" void whemul_segment_destroy(whemul_segment *sg) { delete sg; }

extern "C" int whemul_segment_transfer(whemul_segment *sg, uint32_t *matrix, char *err, size_t errlen) {
    const Packed &pk = sg->pk;
    const uint32_t T = pk.T, C = (uint32_t)pk.chain_begin.size() - 1;
    std::string msg;
    // per-chain matrices from unit inputs (what pass 1 of the batched sweep leaves in its planes) ...
    std::vector<uint32_t> M((size_t)C * T * T);
    for (uint32_t c = 0; c < C; ++c)
        for (uint32_t u = 0; u < T; ++u) {
            std::vector<uint32_t> prev(T, UMAX);
            prev[u] = 0;
            int rc = sweep_columns(pk, pk.chain_begin[c], pk.chain_begin[c + 1], 0, prev, sg->arena, msg);
            if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
            std::memcpy(&M[((size_t)c * T + u) * T], prev.data(), (size_t)T * 4);
        }
    // ... folded like ped_prefix_kernel does with `matrix` given
    for (uint32_t u0 = 0; u0 < T; ++u0) {
        uint32_t in[MAX_T];
        uint32_t c_first = 0;
        if (sg->continues) {
            for (uint32_t i = 0; i < T; ++i) in[i] = i == u0 ? 0u : UMAX;
        } else {
            for (uint32_t i = 0; i < T; ++i) in[i] = M[(size_t)u0 * T + i];  // every plane of chain 0 holds its true output
            c_first = 1;
        }
        fold_chains(T, c_first, C, in, [&](uint32_t c, uint32_t u) { return &M[((size_t)c * T + u) * T]; },
                    [](uint32_t, const uint32_t *) {});
        std::memcpy(matrix + (size_t)u0 * T, in, (size_t)T * 4);
    }
    return WHMEC_OK;
}

extern "C" int whemul_segment_sweep(whemul_segment *sg, const uint32_t *in_vec, uint32_t *out_vec, char *err, size_t errlen) {
    const Packed &pk = sg->pk;
    std::string msg;
    if (sg->continues != (in_vec != nullptr)) return fail_with("input vector / continues mismatch", err, errlen, WHMEC_ERR_INPUT);
    std::vector<uint32_t> prev;
    if (in_vec) prev.assign(in_vec, in_vec + pk.T);
    int rc = sweep_columns(pk, 0, pk.n, 0, prev, sg->arena, msg);
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    sg->last_vals = prev;
    std::memcpy(out_vec, prev.data(), (size_t)pk.T * 4);
    sg->swept = true;
    return WHMEC_OK;
}

namespace {
// bt_chain_start of whmec.cu
void chain_start(const whemul_segment *sg, const BtView &bv, uint32_t c, uint32_t u, int entry, uint32_t *x, uint32_t *tv,
                 uint32_t *ptv, uint32_t *cost) {
    const Packed &pk = sg->pk;
    const uint32_t C = (uint32_t)pk.chain_begin.size() - 1, k_last = pk.chain_begin[c + 1] - 1;
    if (c + 1 == C && entry < 0) {
        pick_optimum(pk.cols[k_last], sg->last_vals.data(), sg->arena.data(), pk.T, pk.tb, cost, x, tv, ptv);
    } else {
        *tv = u;
        chain_entry(bv, k_last, u, x, ptv);
    }
}

void chain_exits(whemul_segment *sg, int entry) {
    const Packed &pk = sg->pk;
    const uint32_t T = pk.T, C = (uint32_t)pk.chain_begin.size() - 1;
    BtView bv{pk.cols.data(), sg->arena.data(), T, pk.tb};
    sg->exits.assign((size_t)C * T, 0);
    for (uint32_t c = 0; c < C; ++c)
        for (uint32_t u = 0; u < T; ++u) {
            uint32_t x, tv, ptv, cost;
            chain_start(sg, bv, c, u, entry, &x, &tv, &ptv, &cost);
            sg->exits[(size_t)c * T + u] = backtrace_range(bv, pk.chain_begin[c + 1] - 1, pk.chain_begin[c], x, tv, ptv, nullptr, nullptr);
        }
}
}  // namespace

extern "C" int whemul_segment_exits(whemul_segment *sg, int is_last, uint32_t *exits, char *err, size_t errlen) {
    const Packed &pk = sg->pk;
    const uint32_t T = pk.T, C = (uint32_t)pk.chain_begin.size() - 1;
    if (!sg->swept) return fail_with("exits before sweep", err, errlen, WHMEC_ERR_INPUT);
    chain_exits(sg, is_last ? -1 : 0);
    for (uint32_t t = 0; t < T; ++t) {
        uint32_t e = t;
        for (uint32_t c = C; c-- > 0;) e = sg->exits[(size_t)c * T + e];
        exits[t] = e;
    }
    return WHMEC_OK;
}

extern "C" int whemul_segment_finish(whemul_segment *sg, int entry, whmec_solution *s, char *err, size_t errlen) {
    const Packed &pk = sg->pk;
    const uint32_t T = pk.T, C = (uint32_t)pk.chain_begin.size() - 1, n = pk.n;
    std::string msg;
    if (!sg->swept) return fail_with("finish before sweep", err, errlen, WHMEC_ERR_INPUT);
    chain_exits(sg, entry);
    std::vector<uint32_t> entries(C), pidx(n), ptv(n);
    uint32_t e = entry < 0 ? 0u : (uint32_t)entry;
    for (uint32_t c = C; c-- > 0;) {
        entries[c] = e;
        e = sg->exits[(size_t)c * T + e];
    }
    BtView bv{pk.cols.data(), sg->arena.data(), T, pk.tb};
    uint32_t total = 0;
    for (uint32_t c = 0; c < C; ++c) {
        uint32_t x, tv, ptvv, cost = 0;
        chain_start(sg, bv, c, entries[c], entry, &x, &tv, &ptvv, &cost);
        backtrace_range(bv, pk.chain_begin[c + 1] - 1, pk.chain_begin[c], x, tv, ptvv, pidx.data(), ptv.data());
        if (c + 1 == C) total = cost;
    }
    s->cost = total;
    int rc = build_outputs(pk, pidx.data(), ptv.data(), s, msg);
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    return WHMEC_OK;
}

// ---- host mirror of ped_fused_kernel (csrc/whmec.cu): the same phases in the same order, every phase run item by item
// ---- with the per-item code of ped_fused.h; checks the scheme (slots, tables, lanes per entry, merge of partial keys,
// ---- buffers M / R / A, one unit row per chain + symmetry + prefix + true inputs), not the CUDA glue itself
namespace {

void fused_chain(const Packed &pk, uint32_t c, const uint32_t *in_vec, bool unit, std::vector<uint32_t> &arena, uint32_t *out_vec) {
    const uint32_t k0 = pk.chain_begin[c], k1 = pk.chain_begin[c + 1];
    const uint32_t max_ent = PF_T << PF_MAX_F;
    std::vector<uint32_t> M(max_ent, 0xDEADBEEF), R(max_ent, 0xDEADBEEF);
    std::vector<uint8_t> A(max_ent, 0xEE);
    std::vector<uint64_t> keys(max_ent);
    auto Cp = std::make_unique<PedFusedCol>();
    PedFusedCol &C = *Cp;
    for (uint32_t k = k0; k < k1; ++k) {
        C.m = pk.cols[k];
        const ColMeta &m = C.m;
        const uint32_t *group = pk.fn_group.data() + m.grp_off;
        for (uint32_t s = 0; s < PF_SLOTS; ++s) pf_stage_slot(C, m, s, pk.fn_c0.data(), pk.fn_delta.data(), group);
        C.drop = ~m.keep & low_mask(m.a);
        C.rc_next = k + 1 < k1 ? pk.cols[k + 1].rc : 0u;
        for (uint32_t v = 0; v < 2 * TAB_SIZE; ++v) pf_stage_pdep(C, m, v);
        if (k == k0) {
            uint32_t invec[PF_T];
            for (uint32_t j = 0; j < PF_T; ++j) invec[j] = unit ? (j == 0 ? 0u : UMAX) : in_vec[j];
            pf_first_row(m, invec, M.data(), A.data());
        }
        for (uint32_t run = 0; run < PF_SLOTS * 32; ++run) pf_stage_table_run(C, m, run, pk.fn_delta.data(), group);
        const uint32_t f = m.f, d = m.d, nout = 1u << f, nent = nout * PF_T;
        const uint32_t lc = pf_lane_bits(f, d), per = 1u << (d - lc), items = nout << lc;
        if (lc) std::fill(keys.begin(), keys.begin() + nent, KEY_INF);
        for (uint32_t item = 0; item < items; ++item) {
            const uint32_t o = item & (nout - 1u), chunk = item >> f;
            PedQuad q;
            pf_walk(C, M.data(), o, chunk * per, (chunk + 1) * per, q);
            for (uint32_t t = 0; t < PF_T; ++t) {
                if (lc) {
                    keys[o * PF_T + t] = std::min(keys[o * PF_T + t], ((uint64_t)q.val[t] << 32) | q.r[t]);
                } else {
                    R[o * PF_T + t] = q.val[t];
                    if (!unit) bp_store_serial(arena.data(), m.bp_off, m.bp_width, (uint64_t)o * PF_T + t,
                                               pf_backpointer(A.data(), t, q.val[t], q.r[t], q.b[t]) & low_mask(d + 2));
                }
            }
        }
        if (lc)
            for (uint32_t e = 0; e < nent; ++e) {
                R[e] = (uint32_t)(keys[e] >> 32);
                if (!unit) bp_store_serial(arena.data(), m.bp_off, m.bp_width, e,
                                           pf_backpointer_of_key(C, A.data(), e >> 2, e & 3u, R[e], (uint32_t)keys[e]) & low_mask(d + 2));
            }
        if (k + 1 < k1)
            for (uint32_t o = 0; o < nout; ++o) {
                uint32_t row[PF_T], mv[PF_T], arg[PF_T];
                for (uint32_t j = 0; j < PF_T; ++j) row[j] = R[o * PF_T + j];
                for (uint32_t i = 0; i < PF_T; ++i) mv[i] = pf_transition(row, i, C.rc_next, &arg[i]);
                for (uint32_t i = 0; i < PF_T; ++i) {
                    M[pf_swz(o) * PF_T + i] = mv[i];
                    A[pf_swz(o) * PF_T + i] = (uint8_t)arg[i];
                }
            }
    }
    for (uint32_t t = 0; t < PF_T; ++t) out_vec[t] = R[t] < PF_INF ? R[t] : UMAX;
}
}  // namespace

// returns 100 when the problem is outside the fused path's shape
extern "C" int whemul_ped_fused_solve(const whmec_problem *p, whmec_solution *s, char *err, size_t errlen) {
    Packed pk;
    std::string msg;
    int rc = pack_problem(p, pk, msg);
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    const uint32_t n = pk.n, T = pk.T;
    if (n == 0 || T != PF_T || !pk.safe31) return fail_with("not a problem for the fused pedigree sweep", err, errlen, 100);
    for (uint32_t k = 0; k < n; ++k)
        if (!pf_column_ok(pk.cols[k], pk.fn_group.data() + pk.cols[k].grp_off)) return fail_with("column outside the fused shape", err, errlen, 100);
    {   // the symmetry group of a trio is all of Z_2^2
        uint32_t masks[PF_T];
        if (pf_symmetry_group(p->n_ind, p->n_trios, p->trios, masks) != PF_T) return fail_with("unexpected symmetry group", err, errlen, 101);
    }
    const uint32_t C = (uint32_t)pk.chain_begin.size() - 1;
    std::vector<uint32_t> arena(pk.bp_words + 1, 0), rows((size_t)C * T), in_vecs((size_t)C * T, 0), out_vecs((size_t)C * T);
    for (uint32_t c = 0; c < C; ++c) fused_chain(pk, c, nullptr, true, arena, &rows[(size_t)c * T]);
    {   // ped_fused_prefix_kernel
        uint32_t in[PF_T], out[PF_T];
        for (uint32_t i = 0; i < T; ++i) in[i] = rows[i];
        for (uint32_t c = 1; c < C; ++c) {
            for (uint32_t i = 0; i < T; ++i) {
                in_vecs[(size_t)c * T + i] = in[i];
                out[i] = UMAX;
            }
            for (uint32_t u = 0; u < T; ++u) {
                if (in[u] == UMAX) continue;
                for (uint32_t i = 0; i < T; ++i) {
                    const uint32_t mv = rows[(size_t)c * T + (i ^ u)];
                    if (mv != UMAX && in[u] + mv < out[i]) out[i] = in[u] + mv;
                }
            }
            for (uint32_t i = 0; i < T; ++i) in[i] = out[i];
        }
    }
    for (uint32_t c = 0; c < C; ++c) fused_chain(pk, c, &in_vecs[(size_t)c * T], false, arena, &out_vecs[(size_t)c * T]);
    std::vector<uint32_t> pidx(n), ptv(n);
    BtView bv{pk.cols.data(), arena.data(), T, pk.tb};
    uint32_t cost, x, tv, ptvv;
    pick_optimum(pk.cols[n - 1], &out_vecs[(size_t)(C - 1) * T], arena.data(), T, pk.tb, &cost, &x, &tv, &ptvv);
    backtrace_range(bv, n - 1, 0, x, tv, ptvv, pidx.data(), ptv.data());
    s->cost = cost;
    rc = build_outputs(pk, pidx.data(), ptv.data(), s, msg);
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    return WHMEC_OK;
}

// A task that throws on a pool worker / on the caller: parallel_tasks must rethrow the first exception on the caller after
// every worker has let go of the job, and the pool must stay usable.  Returns 0 when all of that holds.
extern "C" int whemul_pool_throw_check(uint32_t n_threads) {
    using namespace whmec;
    for (int round = 0; round < 4; ++round) {
        std::atomic<uint32_t> ran{0};
        bool caught = false;
        try {
            parallel_tasks(256, n_threads, [&](uint32_t t) {
                ran.fetch_add(1);
                if (t == (uint32_t)(17 + 60 * round)) throw std::runtime_error("task failed");
            });
        } catch (const std::runtime_error &e) {
            caught = std::string(e.what()) == "task failed";
        }
        if (!caught || ran.load() == 0) return 1 + round;
        std::atomic<uint64_t> sum{0};
        parallel_tasks(1000, n_threads, [&](uint32_t t) { sum.fetch_add(t); });
        if (sum.load() != 999ull * 1000 / 2) return 10 + round;
    }
    return 0;
}
