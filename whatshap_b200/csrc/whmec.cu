// C ABI (include/whmec.h) + CUDA kernels of the weighted-MEC / PedMEC column sweep for sm_90a.
//
// Replaces, behind plain C entry points, the work of PedigreeDPTable's constructor
// (src/pedigreedptable.cpp:15-37 -> compute_table :84-174 -> compute_column :177-335) and of
// get_super_reads / get_optimal_partitioning / get_optimal_score (:338-406).
//
// There is deliberately NO CPU execution path in this library: if CUDA is unavailable every
// entry point that computes returns WHMEC_ERR_CUDA.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <malloc.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <new>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/whmec.h"
#include "common.h"
#include "dp_device.h"
#include "ped_fused.h"
#include "grouped.h"
#include "pack.h"
#include "tile.cuh"

using namespace whmec;

namespace {

#define CUDA_TRY(expr)                                                                              \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess) {                                                                    \
            msg = std::string(#expr) + ": " + cudaGetErrorString(_e);                               \
            return WHMEC_ERR_CUDA;                                                                  \
        }                                                                                           \
    } while (0)

void set_err(char *err, size_t errlen, const std::string &msg) {
    if (err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = 0;
    }
}

// ------------------------------------------------------------------------------------------
// Column kernel (general path: any pedigree, any read structure).  One launch per column.
// ------------------------------------------------------------------------------------------

// Pack `width`-bit back-pointers of 32 consecutive entries (one per lane) into 32-bit words.
__device__ __forceinline__ void bp_store_warp(uint32_t *arena, uint64_t off_words, uint32_t width, uint64_t e,
                                              uint32_t value, bool valid) {
    if (width == 0) return;  // uniform per launch
    const uint32_t per = 32u / width;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t sub = lane % per;
    uint32_t word = valid ? (width == 32 ? value : (value << (sub * width))) : 0u;
    for (uint32_t off = 1; off < per; off <<= 1) word |= __shfl_xor_sync(0xFFFFFFFFu, word, off);
    if (sub == 0 && valid) arena[off_words + e / per] = word;
}

// The cost functions of one column are read by every thread of the block many times: stage them in
// shared memory (up to FN_SMEM functions; beyond that the global arrays are used directly).
constexpr uint32_t FN_SMEM = 48;
constexpr uint32_t FN_TAB = 12;  // columns with at most this many cost functions get byte tables

struct ColShared {
    ColMeta m;
    uint32_t group[MAX_T + 1];
    uint32_t c0[FN_SMEM];
    int32_t delta[FN_SMEM * FN_STRIDE];
    uint32_t pd_lo[TAB_SIZE], pd_hi[TAB_SIZE];
    int32_t tlo[FN_TAB * TAB_SIZE], thi[FN_TAB * TAB_SIZE];
    ColTables tab;
    uint32_t staged, tabled;
};

// `cm` and `nf` arrive as kernel parameters (constant bank): no dependent global loads before the
// function arrays can be fetched.
__device__ __forceinline__ void stage_column(ColShared &S, const ColMeta &cm, uint32_t nf, uint32_t T,
                                             const uint32_t *fn_c0, const int32_t *fn_delta, const uint32_t *fn_group) {
    if (threadIdx.x < sizeof(ColMeta) / 4) ((uint32_t *)&S.m)[threadIdx.x] = ((const uint32_t *)&cm)[threadIdx.x];
    for (uint32_t i = threadIdx.x; i <= T; i += blockDim.x) S.group[i] = fn_group[cm.grp_off + i];
    if (threadIdx.x == 0) S.staged = nf <= FN_SMEM;
    if (nf <= FN_SMEM) {
        for (uint32_t i = threadIdx.x; i < nf; i += blockDim.x) S.c0[i] = fn_c0[cm.fn_off + i];
        // only the first `a` deltas of a function are ever read
        const uint32_t a = cm.a;
        for (uint32_t i = threadIdx.x; i < nf * a; i += blockDim.x) {
            const uint32_t F = i / a, j = i - F * a;
            S.delta[F * FN_STRIDE + j] = fn_delta[(size_t)(cm.fn_off + F) * FN_STRIDE + j];
        }
        // zero the unused deltas the byte tables may touch
        for (uint32_t i = threadIdx.x; i < nf * (2 * TAB_BITS); i += blockDim.x) {
            const uint32_t F = i / (2 * TAB_BITS), j = i - F * (2 * TAB_BITS);
            if (j >= a) S.delta[F * FN_STRIDE + j] = 0;
        }
    }
    const bool tabled = nf <= FN_TAB;
    const uint32_t keep_lo = lowest_set_bits(cm.keep, TAB_BITS), keep_hi = lowest_set_bits(cm.keep & ~keep_lo, TAB_BITS);
    if (tabled)
        for (uint32_t v = threadIdx.x; v < 2 * TAB_SIZE; v += blockDim.x) {
            if (v < TAB_SIZE) S.pd_lo[v] = pdep32(v, keep_lo);
            else S.pd_hi[v - TAB_SIZE] = pdep32(v - TAB_SIZE, keep_hi);
        }
    __syncthreads();
    if (tabled) {
        for (uint32_t run = threadIdx.x; run < nf * 32; run += blockDim.x) {
            const uint32_t F = run >> 5, half = (run >> 4) & 1u, hi4 = run & 15u;
            build_cost_table_run(S.delta + F * FN_STRIDE, half, hi4, (half ? S.thi : S.tlo) + F * TAB_SIZE + 16 * hi4);
        }
        if (threadIdx.x == 0) {
            S.tab.pd_lo = S.pd_lo;
            S.tab.pd_hi = S.pd_hi;
            S.tab.keep_rest = cm.keep & ~keep_lo & ~keep_hi;
            S.tab.lo = S.tlo;
            S.tab.hi = S.thi;
        }
    }
    if (threadIdx.x == 0) S.tabled = tabled;
    __syncthreads();
}

__device__ __forceinline__ ColView make_view(const ColShared &S, uint32_t T, uint32_t tb, const uint32_t *fn_c0,
                                             const int32_t *fn_delta, const uint32_t *prev, uint32_t i,
                                             const uint8_t *prevarg = nullptr) {
    ColView v;
    v.m = &S.m;
    v.T = T;
    v.tb = tb;
    const uint32_t g0 = S.group[i], g1 = S.group[i + 1];
    if (S.staged) {
        v.fn_c0 = S.c0 + g0;
        v.fn_delta = S.delta + (size_t)g0 * FN_STRIDE;
    } else {
        v.fn_c0 = fn_c0 + S.m.fn_off + g0;
        v.fn_delta = fn_delta + (size_t)(S.m.fn_off + g0) * FN_STRIDE;
    }
    v.nf = g1 - g0;
    v.prev = prev;
    v.tab = S.tabled ? &S.tab : nullptr;
    v.tab_fn0 = g0;
    v.prevm = prevarg ? prev : nullptr;  // `prev` holds transition minima when their argmins are given
    v.prevarg = prevarg;
    return v;
}

// lanes per projection entry (log2): one thread per entry when the column has enough entries to fill
// the GPU, otherwise the 2^d candidates of an entry are spread over up to 32 lanes
__host__ __device__ inline uint32_t col_lane_bits(uint32_t log_entries, uint32_t d) {
    if (log_entries >= 14) return 0;
    const uint32_t want = 14 - log_entries;
    const uint32_t lc = d < want ? d : want;
    return lc < 5 ? lc : 5;
}

// Body of the per-column kernels for d <= 7: thread (or lane group) per projection entry.
__device__ __forceinline__ void direct_body(ColShared &S, uint32_t *bpvals, uint32_t T, uint32_t tb,
                                            const uint32_t *fn_c0, const int32_t *fn_delta, const uint32_t *prev,
                                            uint32_t *out, uint32_t *arena, bool write_bp, const uint8_t *prevarg = nullptr,
                                            bool xform_out = false, uint32_t rc_next = 0, uint8_t *outarg = nullptr,
                                            uint32_t *svals = nullptr) {
    const ColMeta &sm = S.m;
    // 2^lc lanes share one projection entry (its 2^d candidates in parallel), so that even the small
    // columns of a pedigree expose enough threads to hide instruction latency
    const uint32_t lc = col_lane_bits(sm.f + tb, sm.d);
    const uint32_t per = 1u << (sm.d - lc);
    const uint64_t nent = ((uint64_t)1 << sm.f) * T;
    const uint32_t ent_per_block = blockDim.x >> lc;
    const uint32_t le = threadIdx.x >> lc;                 // entry within the block
    const uint64_t e = (uint64_t)blockIdx.x * ent_per_block + le;
    const uint32_t c = threadIdx.x & ((1u << lc) - 1u);   // candidate chunk of this lane
    unsigned long long key = KEY_INF;
    if (e < nent) {
        const uint32_t o = (uint32_t)(e >> tb), i = (uint32_t)e & (T - 1);
        ColView v = make_view(S, T, tb, fn_c0, fn_delta, prev, i, prevarg);
        key = eval_candidates(v, o, i, c * per, (c + 1) * per);
    }
    for (uint32_t off = 1; off < (1u << lc); off <<= 1) {
        const unsigned long long other = __shfl_xor_sync(0xFFFFFFFFu, key, off);
        key = other < key ? other : key;
    }
    if (c == 0) {
        if (xform_out) svals[le] = (uint32_t)(key >> 32);  // KEY_INF for entries beyond the column
        else if (e < nent) out[e] = (uint32_t)(key >> 32);
        bpvals[le] = e < nent ? ((uint32_t)key & low_mask(sm.d + tb)) : 0u;
    }
    __syncthreads();
    if (xform_out && threadIdx.x < ent_per_block) {
        // hand the NEXT column min_j(value_j + popcount(i^j) * rc_next) instead of the raw values: the T
        // values of one projection index sit next to each other in this block
        const uint64_t e2 = (uint64_t)blockIdx.x * ent_per_block + threadIdx.x;
        if (e2 < nent) {
            uint32_t arg;
            out[e2] = transition_min(&svals[threadIdx.x & ~(T - 1)], T, (uint32_t)e2 & (T - 1), rc_next, &arg);
            outarg[e2] = (uint8_t)arg;
        }
    }
    // pack this block's back-pointers: ent_per_block * width bits, a whole number of 32-bit words
    const uint32_t w = sm.bp_width;
    if (w && write_bp) {
        const uint32_t per_word = 32u / w;
        const uint32_t words = (ent_per_block * w) >> 5;
        const uint64_t first_word = ((uint64_t)blockIdx.x * ent_per_block * w) >> 5;
        if (threadIdx.x < words) {
            uint32_t word = 0;
            for (uint32_t q = 0; q < per_word; ++q) word |= (w == 32 ? bpvals[threadIdx.x] : (bpvals[threadIdx.x * per_word + q] << (q * w)));
            const uint64_t total_words = (nent * w + 31) >> 5;
            if (first_word + threadIdx.x < total_words) arena[sm.bp_off + first_word + threadIdx.x] = word;
        }
    }
}

// Thread e = o*T + i evaluates all 2^d candidates of its projection entry (d small).
__global__ void __launch_bounds__(256) col_direct_kernel(const __grid_constant__ ColMeta cm, uint32_t nf, uint32_t T,
                                                         uint32_t tb, const uint32_t *__restrict__ fn_c0,
                                                         const int32_t *__restrict__ fn_delta,
                                                         const uint32_t *__restrict__ fn_group,
                                                         const uint32_t *__restrict__ prev, uint32_t *__restrict__ out,
                                                         uint32_t *__restrict__ arena) {
    __shared__ ColShared S;
    __shared__ uint32_t bpvals[256];
    stage_column(S, cm, nf, T, fn_c0, fn_delta, fn_group);
    direct_body(S, bpvals, T, tb, fn_c0, fn_delta, prev, out, arena, true);
}

// ------------------------------------------------------------------------------------------
// Batched pedigree sweep.  Transmission vectors couple the DP-independent chains of a pedigree only
// through the T values handed from one chain to the next (pedigreedptable.cpp:272-297), and a chain
// is min-plus linear in that vector.  Pass 1 sweeps every chain once per unit input vector (values
// only) -> its T x T transfer matrix; a tiny prefix pass turns the matrices into every chain's true
// input vector; pass 2 re-sweeps every chain with its true input, writing the same back-pointers
// the sequential sweep would write (SURVEY.md section 8(e), verified there against the reference).
// All chains advance together: one launch = one column step of every (chain, input) instance.
// ------------------------------------------------------------------------------------------
struct PedStep {
    ColMeta cm;
    uint32_t nf;
    uint32_t slot;   // state slot of the instance (two value buffers per slot)
    uint32_t flags;  // bit 0: write back-pointers; bit 1: write transition minima for the next column;
                     // bit 2: the previous projection holds transition minima
    uint32_t rc_next;
};

__global__ void __launch_bounds__(256) col_batched_kernel(const PedStep *__restrict__ steps, uint32_t *__restrict__ vals,
                                                          uint64_t max_ent, uint32_t T, uint32_t tb,
                                                          const uint32_t *__restrict__ fn_c0, const int32_t *__restrict__ fn_delta,
                                                          const uint32_t *__restrict__ fn_group, uint32_t *__restrict__ arena,
                                                          uint32_t parity, uint8_t *__restrict__ args) {
    __shared__ ColShared S;
    __shared__ uint32_t bpvals[256];
    __shared__ uint32_t svals[256];
    __shared__ unsigned long long wkeys[8];
    const PedStep &st = steps[blockIdx.y];
    const uint64_t nent = ((uint64_t)1 << st.cm.f) * T;
    const uint32_t d = st.cm.d;
    uint64_t blocks_needed;
    if (d <= 7) {
        const uint32_t lc = col_lane_bits(st.cm.f + tb, d);
        const uint64_t epb = 256u >> lc;
        blocks_needed = (nent + epb - 1) / epb;
    } else {
        blocks_needed = nent;
    }
    if (blockIdx.x >= blocks_needed) return;
    const uint32_t *prev = vals + ((uint64_t)st.slot * 2 + (parity ^ 1u)) * max_ent;
    uint32_t *out = vals + ((uint64_t)st.slot * 2 + parity) * max_ent;
    const uint8_t *prevarg = (st.flags & 4u) ? args + ((uint64_t)st.slot * 2 + (parity ^ 1u)) * max_ent : nullptr;
    uint8_t *outarg = args + ((uint64_t)st.slot * 2 + parity) * max_ent;
    stage_column(S, st.cm, st.nf, T, fn_c0, fn_delta, fn_group);
    if (d <= 7) {
        direct_body(S, bpvals, T, tb, fn_c0, fn_delta, prev, out, arena, (st.flags & 1u) != 0, prevarg, (st.flags & 2u) != 0,
                    st.rc_next, outarg, svals);
        return;
    }
    // many reads end here (chain end): the block owns one entry and splits its 2^d candidates
    const uint64_t e = blockIdx.x;
    const uint32_t o = (uint32_t)(e >> tb), i = (uint32_t)e & (T - 1);
    const uint32_t per = 1u << (d - 8);
    ColView v = make_view(S, T, tb, fn_c0, fn_delta, prev, i, prevarg);
    unsigned long long key = eval_candidates(v, o, i, threadIdx.x * per, (threadIdx.x + 1) * per);
    for (int off = 16; off > 0; off >>= 1) {
        const unsigned long long other = __shfl_xor_sync(0xFFFFFFFFu, key, off);
        key = other < key ? other : key;
    }
    if ((threadIdx.x & 31) == 0) wkeys[threadIdx.x >> 5] = key;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) key = wkeys[w] < key ? wkeys[w] : key;
        out[e] = (uint32_t)(key >> 32);
        if (st.flags & 1u) arena[S.m.bp_off + e] = (uint32_t)key & low_mask(d + tb);  // bp_width == 32 for d >= 8
    }
}

// Pass 1 for the chains that need a transfer matrix: one instance per chain computes the values for all
// T unit input vectors at once (slots st.slot .. st.slot+T-1).  flags bit 3: first column of its chain.
__global__ void __launch_bounds__(256) col_multi_kernel(const PedStep *__restrict__ steps, uint32_t *__restrict__ vals,
                                                        uint64_t max_ent, uint32_t T, uint32_t tb,
                                                        const uint32_t *__restrict__ fn_c0, const int32_t *__restrict__ fn_delta,
                                                        const uint32_t *__restrict__ fn_group, uint32_t parity) {
    __shared__ ColShared S;
    __shared__ uint32_t svals[MULTI_MAX * 256];
    const PedStep &st = steps[blockIdx.y];
    const uint64_t nent = ((uint64_t)1 << st.cm.f) * T;
    const uint32_t d = st.cm.d;
    const uint32_t lc = d <= 7 ? col_lane_bits(st.cm.f + tb, d) : 0;
    const uint32_t ent_per_block = d <= 7 ? (256u >> lc) : 1u;
    if ((uint64_t)blockIdx.x * ent_per_block >= nent) return;
    const uint64_t plane_stride = 2 * max_ent;
    const uint32_t *planes = vals + ((uint64_t)st.slot * 2 + (parity ^ 1u)) * max_ent;
    uint32_t *out0 = vals + ((uint64_t)st.slot * 2 + parity) * max_ent;
    const bool first_chain = (st.flags & 8u) != 0, transformed = (st.flags & 4u) != 0, xform_out = (st.flags & 2u) != 0;
    stage_column(S, st.cm, st.nf, T, fn_c0, fn_delta, fn_group);
    uint32_t mn[MULTI_MAX];
    if (d <= 7) {
        const uint32_t per = 1u << (d - lc);
        const uint32_t le = threadIdx.x >> lc;
        const uint64_t e = (uint64_t)blockIdx.x * ent_per_block + le;
        const uint32_t c = threadIdx.x & ((1u << lc) - 1u);
        for (uint32_t u = 0; u < T; ++u) mn[u] = UMAX;
        if (e < nent) {
            const uint32_t o = (uint32_t)(e >> tb), i = (uint32_t)e & (T - 1);
            ColView v = make_view(S, T, tb, fn_c0, fn_delta, nullptr, i);
            eval_values_multi(v, o, i, c * per, (c + 1) * per, planes, plane_stride, first_chain, transformed, mn);
        }
        for (uint32_t u = 0; u < T; ++u) {
            uint32_t val = mn[u];
            for (uint32_t off = 1; off < (1u << lc); off <<= 1) {
                const uint32_t other = __shfl_xor_sync(0xFFFFFFFFu, val, off);
                val = other < val ? other : val;
            }
            if (c == 0) {
                if (xform_out) svals[u * 256 + le] = val;
                else if (e < nent) out0[u * plane_stride + e] = val;
            }
        }
        if (xform_out) {
            __syncthreads();
            if (threadIdx.x < ent_per_block) {
                const uint64_t e2 = (uint64_t)blockIdx.x * ent_per_block + threadIdx.x;
                if (e2 < nent)
                    for (uint32_t u = 0; u < T; ++u) {
                        uint32_t arg;
                        out0[u * plane_stride + e2] =
                            transition_min(&svals[u * 256 + (threadIdx.x & ~(T - 1))], T, (uint32_t)e2 & (T - 1), st.rc_next, &arg);
                    }
            }
        }
        return;
    }
    // chain end: the block owns one entry
    const uint64_t e = blockIdx.x;
    const uint32_t o = (uint32_t)(e >> tb), i = (uint32_t)e & (T - 1);
    const uint32_t per = 1u << (d - 8);
    ColView v = make_view(S, T, tb, fn_c0, fn_delta, nullptr, i);
    eval_values_multi(v, o, i, threadIdx.x * per, (threadIdx.x + 1) * per, planes, plane_stride, first_chain, transformed, mn);
    for (uint32_t u = 0; u < T; ++u) {
        uint32_t val = mn[u];
        for (int off = 16; off > 0; off >>= 1) {
            const uint32_t other = __shfl_xor_sync(0xFFFFFFFFu, val, off);
            val = other < val ? other : val;
        }
        if ((threadIdx.x & 31) == 0) svals[u * 8 + (threadIdx.x >> 5)] = val;
    }
    __syncthreads();
    if (threadIdx.x < T) {
        uint32_t val = UMAX;
        for (int w = 0; w < 8; ++w) val = svals[threadIdx.x * 8 + w] < val ? svals[threadIdx.x * 8 + w] : val;
        out0[threadIdx.x * plane_stride + e] = val;
    }
}

// ------------------------------------------------------------------------------------------
// Fused pedigree sweep for one trio (T == 4): one thread block per DP-independent chain walks ALL columns of its chain
// with the projection (transition minima M + argmins A of the previous column, raw values R of the current one) in
// shared memory; the per-item code is ped_fused.h.  Pass 1 sweeps every chain once with the unit input e_0 (values only)
// -- by the symmetry of ped_fused.h that single row determines the chain's whole transfer matrix, Mat[u][i] = row[i ^ u];
// a one-thread prefix folds the matrices into every chain's true input; pass 2 sweeps every chain with its true input and
// writes exactly the back-pointers of the column-by-column sweep.  Three launches for the whole table.
// ------------------------------------------------------------------------------------------
struct PedFusedArgs {
    const ColMeta *cols;
    const uint32_t *chain_begin, *fn_c0, *fn_group;
    const int32_t *fn_delta;
    uint32_t *arena;
    const uint32_t *in_vecs;  // [chains][4] true inputs (pass 2)
    uint32_t *out_vecs;       // [chains][4]: pass 1: row 0 of the chain's transfer matrix; pass 2: the chain's true output
    uint32_t unit;            // 1: pass 1 (input e_0, values only), 0: pass 2
};

constexpr uint32_t PF_MAX_ENT = PF_T << PF_MAX_F;
constexpr size_t PF_COL_BYTES = (sizeof(PedFusedCol) + 15) & ~(size_t)15;
constexpr size_t PF_SMEM = PF_COL_BYTES + (size_t)PF_MAX_ENT * (4 + 4 + 1);

// back-pointers of the four entries of projection index o (entry e = 4 o + t, `w` bits each)
__device__ __forceinline__ void pf_store_bp(uint32_t *arena, uint64_t bp_off, uint32_t w, uint32_t o, const uint32_t *v, bool valid) {
    if (w <= 8) {  // the four entries share one element of 4 w bits
        const uint32_t packed = valid ? (v[0] | (v[1] << w) | (v[2] << (2 * w)) | (v[3] << (3 * w))) : 0u;
        bp_store_warp(arena, bp_off, 4 * w, o, packed, valid);
    } else if (valid) {
        if (w == 16) {
            arena[bp_off + 2 * (uint64_t)o] = v[0] | (v[1] << 16);
            arena[bp_off + 2 * (uint64_t)o + 1] = v[2] | (v[3] << 16);
        } else {
            for (uint32_t t = 0; t < PF_T; ++t) arena[bp_off + 4 * (uint64_t)o + t] = v[t];
        }
    }
}

// stage column k of the chain (tables, slots, scatter tables; the chain's first column also gets the row it reads)
__device__ __forceinline__ void pf_stage_column(PedFusedCol &C, const PedFusedArgs &a, uint32_t c, uint32_t k, uint32_t k0, uint32_t k1,
                                                uint32_t *M, uint8_t *A, uint32_t tid) {
    const ColMeta &m = a.cols[k];  // global (L1 / L2): every staging thread reads what it needs itself
    const uint32_t *group = a.fn_group + m.grp_off;
    if (tid < PF_SLOTS * 32) pf_stage_table_run(C, m, tid, a.fn_delta, group);
    else if (tid < PF_SLOTS * 32 + PF_SLOTS) pf_stage_slot(C, m, tid - PF_SLOTS * 32, a.fn_c0, a.fn_delta, group);
    else if (tid >= 576 && tid < 576 + sizeof(ColMeta) / 4) ((uint32_t *)&C.m)[tid - 576] = ((const uint32_t *)&m)[tid - 576];
    else if (tid == 640) {
        C.drop = ~m.keep & low_mask(m.a);
        C.rc_next = k + 1 < k1 ? a.cols[k + 1].rc : 0u;
    } else if (tid == 641 && k == k0) {  // the row the chain's first column reads (row 0 is its own swizzle image)
        uint32_t invec[PF_T];
        for (uint32_t j = 0; j < PF_T; ++j) invec[j] = a.unit ? (j == 0 ? 0u : UMAX) : a.in_vecs[(size_t)c * PF_T + j];
        pf_first_row(m, invec, M, A);
    }
    if (tid >= 512) pf_stage_pdep(C, m, tid - 512);
}

__global__ void __launch_bounds__(PF_THREADS, 1) ped_fused_kernel(const PedFusedArgs a) {
    extern __shared__ __align__(16) unsigned char pf_raw[];
    PedFusedCol &C = *reinterpret_cast<PedFusedCol *>(pf_raw);
    uint32_t *M = reinterpret_cast<uint32_t *>(pf_raw + PF_COL_BYTES);  // transition minima of the previous column [2^bw][4], rows swizzled
    uint32_t *R = M + PF_MAX_ENT;                                       // raw values of the current column [2^f][4]
    uint8_t *A = reinterpret_cast<uint8_t *>(R + PF_MAX_ENT);           // argmins belonging to M
    unsigned long long *keys = reinterpret_cast<unsigned long long *>(R + PF_MAX_ENT / 2);  // small columns only (< 4096 entries)
    const uint32_t tid = threadIdx.x, c = blockIdx.x;
    const uint32_t k0 = a.chain_begin[c], k1 = a.chain_begin[c + 1];
    const bool write_bp = !a.unit;
    pf_stage_column(C, a, c, k0, k0, k1, M, A, tid);
    for (uint32_t k = k0; k < k1; ++k) {
        __syncthreads();  // column k staged; M / A hold the transition minima of column k - 1
        const uint32_t f = C.m.f, d = C.m.d, nout = 1u << f, nent = nout * PF_T;
        const uint32_t lc = pf_lane_bits(f, d), per = 1u << (d - lc), items = nout << lc;
        if (lc) {
            for (uint32_t e = tid; e < nent; e += PF_THREADS) keys[e] = KEY_INF;
            __syncthreads();
        }
        // ---- phase A: candidates
        for (uint32_t base = 0; base < items; base += PF_THREADS) {
            const uint32_t item = base + tid;
            const bool valid = item < items;
            PedQuad q;
            uint32_t o = 0;
            if (valid) {
                o = item & (nout - 1u);
                const uint32_t chunk = item >> f;
                pf_walk(C, M, o, chunk * per, (chunk + 1) * per, q);
            }
            if (lc) {
                if (valid)
                    for (uint32_t t = 0; t < PF_T; ++t) atomicMin(&keys[o * PF_T + t], ((unsigned long long)q.val[t] << 32) | q.r[t]);
            } else {
                if (valid) *reinterpret_cast<uint4 *>(R + (size_t)o * PF_T) = make_uint4(q.val[0], q.val[1], q.val[2], q.val[3]);
                if (write_bp) {
                    uint32_t v[PF_T] = {0, 0, 0, 0};
                    if (valid)
                        for (uint32_t t = 0; t < PF_T; ++t) v[t] = pf_backpointer(A, t, q.val[t], q.r[t], q.b[t]) & low_mask(d + 2);
                    pf_store_bp(a.arena, C.m.bp_off, C.m.bp_width, o, v, valid);
                }
            }
        }
        if (lc) {
            __syncthreads();
            for (uint32_t base = 0; base < nent; base += PF_THREADS) {
                const uint32_t e = base + tid;
                const bool valid = e < nent;
                const unsigned long long key = valid ? keys[e] : KEY_INF;
                const uint32_t val = (uint32_t)(key >> 32);
                uint32_t bp = 0;
                if (valid && write_bp) bp = pf_backpointer_of_key(C, A, e >> 2, e & 3u, val, (uint32_t)key) & low_mask(d + 2);
                if (write_bp) bp_store_warp(a.arena, C.m.bp_off, C.m.bp_width, e, bp, valid);
            }
            __syncthreads();  // every key consumed before R (which the key array overlaps) is written
            for (uint32_t e = tid; e < nent; e += PF_THREADS) R[e] = (uint32_t)(keys[e] >> 32);  // nent < 4096: R[0 .. nent) lies below the key array (R + 8192 words)
        }
        const uint32_t rc_next = C.rc_next;
        __syncthreads();  // R complete, C / M / A no longer read
        // ---- phase B: what the next column reads; and the next column's tables (disjoint memory)
        if (k + 1 < k1) {
            for (uint32_t o = tid; o < nout; o += PF_THREADS) {
                const uint4 r4 = *reinterpret_cast<const uint4 *>(R + (size_t)o * PF_T);
                const uint32_t row[PF_T] = {r4.x, r4.y, r4.z, r4.w};
                uint32_t mv[PF_T], arg[PF_T];
#pragma unroll
                for (uint32_t i = 0; i < PF_T; ++i) mv[i] = pf_transition(row, i, rc_next, &arg[i]);
                const uint32_t at = pf_swz(o);
                *reinterpret_cast<uint4 *>(M + (size_t)at * PF_T) = make_uint4(mv[0], mv[1], mv[2], mv[3]);
                *reinterpret_cast<uint32_t *>(A + (size_t)at * PF_T) = arg[0] | (arg[1] << 8) | (arg[2] << 16) | (arg[3] << 24);
            }
            pf_stage_column(C, a, c, k + 1, k0, k1, M, A, tid);
        }
    }
    __syncthreads();
    if (tid < PF_T) a.out_vecs[(size_t)c * PF_T + tid] = R[tid] < PF_INF ? R[tid] : UMAX;  // a chain ends with f == 0
}

// ---- the same sweep with a CLUSTER of CTAs per chain (fewer chains than SMs: cfg5 has 40 chains for 132 SMs, a table segment
// on one of 8 GPUs five).  Every CTA of the cluster holds the whole previous column (transition minima M + argmins A, double
// buffered) and the column's tables; a large column's outputs are split between the CTAs, and the thread that finishes an
// output forms its transition minima from registers and writes that row into the NEXT-column buffer of every CTA of the
// cluster through distributed shared memory.  One cluster barrier per column orders those writes against the next column's
// reads; columns with fewer than 32 outputs per CTA are computed by every CTA redundantly (no exchange).
constexpr size_t PF_CLUSTER_SMEM = PF_COL_BYTES + (size_t)PF_MAX_ENT * 2 * (4 + 1);
constexpr uint32_t PF_MAX_CLUSTER = 8;

__global__ void __launch_bounds__(PF_THREADS, 1) ped_fused_cluster_kernel(const PedFusedArgs a) {
    namespace cg = cooperative_groups;
    cg::cluster_group cluster = cg::this_cluster();
    const uint32_t cs = cluster.num_blocks(), cr = cluster.block_rank();
    extern __shared__ __align__(16) unsigned char pf_raw[];
    PedFusedCol &C = *reinterpret_cast<PedFusedCol *>(pf_raw);
    uint32_t *Mb = reinterpret_cast<uint32_t *>(pf_raw + PF_COL_BYTES);     // [2][PF_MAX_ENT]
    uint8_t *Ab = reinterpret_cast<uint8_t *>(Mb + 2 * PF_MAX_ENT);          // [2][PF_MAX_ENT]
    const uint32_t tid = threadIdx.x, c = blockIdx.x / cs;
    const uint32_t k0 = a.chain_begin[c], k1 = a.chain_begin[c + 1];
    const bool write_bp = !a.unit;
    pf_stage_column(C, a, c, k0, k0, k1, Mb, Ab, tid);
    const uint32_t *lastR = Mb;
    for (uint32_t k = k0; k < k1; ++k) {
        const uint32_t cur = (k - k0) & 1u;
        const uint32_t *M = Mb + cur * PF_MAX_ENT;
        const uint8_t *A = Ab + cur * PF_MAX_ENT;
        uint32_t *Mn = Mb + (cur ^ 1u) * PF_MAX_ENT;
        uint8_t *An = Ab + (cur ^ 1u) * PF_MAX_ENT;
        cluster.sync();  // column k staged here; every CTA's rows of column k - 1 have arrived; nobody reads the other buffer any more
        const uint32_t f = C.m.f, d = C.m.d, nout = 1u << f, nent = nout * PF_T;
        const uint32_t lc = pf_lane_bits(f, d), per = 1u << (d - lc), items = nout << lc;
        const uint32_t rc_next = C.rc_next;
        const bool more = k + 1 < k1;
        if (lc == 0 && nout >= 32u * cs) {
            // ---- large column: this CTA's share of the outputs
            const uint32_t share = ((nout / cs + 31u) / 32u) * 32u;
            const uint32_t lo = cr * share, hi = lo + share < nout ? lo + share : nout;
            for (uint32_t base = lo; base < hi; base += PF_THREADS) {
                const uint32_t o = base + tid;
                const bool valid = o < hi;
                PedQuad q;
                if (valid) pf_walk(C, M, o, 0, per, q);
                if (write_bp) {
                    uint32_t v[PF_T] = {0, 0, 0, 0};
                    if (valid)
                        for (uint32_t t = 0; t < PF_T; ++t) v[t] = pf_backpointer(A, t, q.val[t], q.r[t], q.b[t]) & low_mask(d + 2);
                    pf_store_bp(a.arena, C.m.bp_off, C.m.bp_width, o, v, valid);
                }
                if (valid && more) {
                    uint32_t mv[PF_T], arg[PF_T];
#pragma unroll
                    for (uint32_t i = 0; i < PF_T; ++i) mv[i] = pf_transition(q.val, i, rc_next, &arg[i]);
                    const uint32_t at = pf_swz(o);
                    const uint4 m4 = make_uint4(mv[0], mv[1], mv[2], mv[3]);
                    const uint32_t a4 = arg[0] | (arg[1] << 8) | (arg[2] << 16) | (arg[3] << 24);
                    uint32_t *mrow = Mn + (size_t)at * PF_T;
                    uint8_t *arow = An + (size_t)at * PF_T;
                    for (uint32_t r = 0; r < cs; ++r) {  // the same row in every CTA of the cluster (distributed shared memory)
                        *reinterpret_cast<uint4 *>(cluster.map_shared_rank(mrow, r)) = m4;
                        *reinterpret_cast<uint32_t *>(cluster.map_shared_rank(arow, r)) = a4;
                    }
                }
            }
        } else {
            // ---- small column (< 4096 entries): every CTA computes all of it; R and the merge keys live in the unused part of
            // the next-column buffer (rows of the next column: words [0, nent); R: [4096, 8192); keys: [8192, 16384))
            uint32_t *R = Mn + 4096;
            unsigned long long *keys = reinterpret_cast<unsigned long long *>(Mn + 8192);
            lastR = R;
            const bool bp_here = write_bp && cr == 0;
            if (lc) {
                for (uint32_t e = tid; e < nent; e += PF_THREADS) keys[e] = KEY_INF;
                __syncthreads();
            }
            for (uint32_t base = 0; base < items; base += PF_THREADS) {
                const uint32_t item = base + tid;
                const bool valid = item < items;
                PedQuad q;
                uint32_t o = 0;
                if (valid) {
                    o = item & (nout - 1u);
                    const uint32_t chunk = item >> f;
                    pf_walk(C, M, o, chunk * per, (chunk + 1) * per, q);
                }
                if (lc) {
                    if (valid)
                        for (uint32_t t = 0; t < PF_T; ++t) atomicMin(&keys[o * PF_T + t], ((unsigned long long)q.val[t] << 32) | q.r[t]);
                } else {
                    if (valid) *reinterpret_cast<uint4 *>(R + (size_t)o * PF_T) = make_uint4(q.val[0], q.val[1], q.val[2], q.val[3]);
                    if (bp_here) {
                        uint32_t v[PF_T] = {0, 0, 0, 0};
                        if (valid)
                            for (uint32_t t = 0; t < PF_T; ++t) v[t] = pf_backpointer(A, t, q.val[t], q.r[t], q.b[t]) & low_mask(d + 2);
                        pf_store_bp(a.arena, C.m.bp_off, C.m.bp_width, o, v, valid);
                    }
                }
            }
            if (lc) {
                __syncthreads();
                for (uint32_t base = 0; base < nent; base += PF_THREADS) {
                    const uint32_t e = base + tid;
                    const bool valid = e < nent;
                    const unsigned long long key = valid ? keys[e] : KEY_INF;
                    const uint32_t val = (uint32_t)(key >> 32);
                    uint32_t bp = 0;
                    if (valid && bp_here) bp = pf_backpointer_of_key(C, A, e >> 2, e & 3u, val, (uint32_t)key) & low_mask(d + 2);
                    if (bp_here) bp_store_warp(a.arena, C.m.bp_off, C.m.bp_width, e, bp, valid);
                    if (valid) R[e] = val;
                }
            }
            __syncthreads();  // R complete
            if (more)
                for (uint32_t o = tid; o < nout; o += PF_THREADS) {
                    const uint4 r4 = *reinterpret_cast<const uint4 *>(R + (size_t)o * PF_T);
                    const uint32_t row[PF_T] = {r4.x, r4.y, r4.z, r4.w};
                    uint32_t mv[PF_T], arg[PF_T];
#pragma unroll
                    for (uint32_t i = 0; i < PF_T; ++i) mv[i] = pf_transition(row, i, rc_next, &arg[i]);
                    const uint32_t at = pf_swz(o);
                    *reinterpret_cast<uint4 *>(Mn + (size_t)at * PF_T) = make_uint4(mv[0], mv[1], mv[2], mv[3]);
                    *reinterpret_cast<uint32_t *>(An + (size_t)at * PF_T) = arg[0] | (arg[1] << 8) | (arg[2] << 16) | (arg[3] << 24);
                }
        }
        __syncthreads();  // this CTA no longer reads C
        if (more) pf_stage_column(C, a, c, k + 1, k0, k1, Mb, Ab, tid);
    }
    __syncthreads();
    if (cr == 0 && tid < PF_T) a.out_vecs[(size_t)c * PF_T + tid] = lastR[tid] < PF_INF ? lastR[tid] : UMAX;  // a chain ends with f == 0
    cluster.sync();  // no CTA exits while a peer may still write into its shared memory
}

// Pass 1 -> pass 2.  Every chain's transfer matrix is Mat[u][i] = row[i ^ u] (ped_fused.h); a chain that starts the table
// ignores its input (its row IS its output).  Folded left to right in min-plus arithmetic:
//   matrix == nullptr (one thread): every chain's true input vector -> in_vecs; the first chain's input is `in_vec`
//     (a segment that continues a table, whmec_segment_sweep) or irrelevant (the table starts here);
//   matrix != nullptr (4 threads): thread u folds e_u through all chains -> row u of the segment's own transfer matrix
//     (whmec_segment_transfer); nothing else is written.
__global__ void ped_fused_prefix_kernel(const uint32_t *__restrict__ rows, uint32_t n_chains, const uint32_t *__restrict__ in_vec,
                                        uint32_t continues, uint32_t *__restrict__ in_vecs, uint32_t *__restrict__ matrix) {
    const uint32_t u0 = blockIdx.x * blockDim.x + threadIdx.x;
    if (u0 >= (matrix ? PF_T : 1u)) return;
    uint32_t in[PF_T], out[PF_T];
    uint32_t c_first = 0;
    if (continues) {
        for (uint32_t i = 0; i < PF_T; ++i) in[i] = matrix ? (i == u0 ? 0u : UMAX) : in_vec[i];
    } else {
        for (uint32_t i = 0; i < PF_T; ++i) in[i] = rows[i];  // the table starts here: chain 0's row is its true output
        if (!matrix)
            for (uint32_t i = 0; i < PF_T; ++i) in_vecs[i] = 0;  // (ignored by the table's first column)
        c_first = 1;
    }
    for (uint32_t c = c_first; c < n_chains; ++c) {
        for (uint32_t i = 0; i < PF_T; ++i) {
            if (!matrix) in_vecs[(size_t)c * PF_T + i] = in[i];
            out[i] = UMAX;
        }
        const uint32_t *row = rows + (size_t)c * PF_T;
        for (uint32_t u = 0; u < PF_T; ++u) {
            if (in[u] == UMAX) continue;
            for (uint32_t i = 0; i < PF_T; ++i) {
                const uint32_t mv = row[i ^ u];
                if (mv != UMAX && in[u] + mv < out[i]) out[i] = in[u] + mv;
            }
        }
        for (uint32_t i = 0; i < PF_T; ++i) in[i] = out[i];
    }
    if (matrix)
        for (uint32_t i = 0; i < PF_T; ++i) matrix[(size_t)u0 * PF_T + i] = in[i];
}

// pass 1 -> pass 2: the T x T transfer matrices of the chains, folded left to right in min-plus
// arithmetic (a few hundred operations per row).
//   pass-1 planes: chain c, unit vector u -> slot c*T + u;  pass-2 slot of chain c: n_chains*T + c.
//   in_vec == nullptr: the plan starts the DP table; chain 0's first column ignores its input
//     (pedigreedptable.cpp:275-278), every pass-1 plane of it holds the same, true, output.
//   in_vec != nullptr: the plan is a segment continuing a table and in_vec the T values handed over
//     by the columns before it (whmec_segment_sweep).
//   matrix == nullptr (one thread): store every chain's true input vector where its first column reads it.
//   matrix != nullptr (T threads): thread u folds the unit vector e_u through all chains -> row u of the
//     segment's own transfer matrix (whmec_segment_transfer); nothing else is written.
__global__ void ped_prefix_kernel(uint32_t *__restrict__ vals, uint64_t max_ent, uint32_t T, uint32_t n_chains,
                                  const uint32_t *__restrict__ chain_len, const uint32_t *__restrict__ in_vec,
                                  uint32_t continues, uint32_t *__restrict__ matrix) {
    const uint32_t u0 = blockIdx.x * blockDim.x + threadIdx.x;
    if (u0 >= (matrix ? T : 1u)) return;
    uint32_t in[MAX_T];
    uint32_t c_first = 0;
    if (matrix && continues) {
        for (uint32_t i = 0; i < T; ++i) in[i] = i == u0 ? 0u : UMAX;
    } else if (!matrix && in_vec) {
        for (uint32_t i = 0; i < T; ++i) in[i] = in_vec[i];
    } else {
        for (uint32_t i = 0; i < T; ++i) in[i] = vals[((uint64_t)0 * 2 + ((chain_len[0] - 1) & 1u)) * max_ent + i];
        c_first = 1;
    }
    fold_chains(
        T, c_first, n_chains, in,
        [&](uint32_t c, uint32_t u) { return vals + ((uint64_t)(c * T + u) * 2 + ((chain_len[c] - 1) & 1u)) * max_ent; },
        [&](uint32_t c, const uint32_t *cur) {
            if (matrix) return;
            uint32_t *dst = vals + ((uint64_t)(n_chains * T + c) * 2 + 1) * max_ent;  // read by the chain's first column (step 0)
            for (uint32_t i = 0; i < T; ++i) dst[i] = cur[i];
        });
    if (matrix)
        for (uint32_t i = 0; i < T; ++i) matrix[(uint64_t)u0 * T + i] = in[i];
}

// unit input vectors of pass 1: slot 1 + (c-1)*T + u gets 0 at u, +inf elsewhere
__global__ void ped_init_kernel(uint32_t *__restrict__ vals, uint64_t max_ent, uint32_t T, uint32_t n_slots) {
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n_slots * T) return;
    const uint32_t slot = idx / T, j = idx % T;
    const uint32_t u = slot % T;
    vals[((uint64_t)slot * 2 + 1) * max_ent + j] = (j == u) ? 0u : UMAX;
}

// Many dropped reads (chain ends): the 2^d candidates of an entry are split over 2^log_chunks
// threads; partial minima meet in a 64-bit atomicMin on the key.
__global__ void __launch_bounds__(256) col_chunk_kernel(const __grid_constant__ ColMeta cm, uint32_t nf, uint32_t T,
                                                        uint32_t tb, const uint32_t *__restrict__ fn_c0,
                                                        const int32_t *__restrict__ fn_delta,
                                                        const uint32_t *__restrict__ fn_group,
                                                        const uint32_t *__restrict__ prev, uint32_t log_chunks,
                                                        unsigned long long *__restrict__ keys) {
    __shared__ ColShared S;
    stage_column(S, cm, nf, T, fn_c0, fn_delta, fn_group);
    const ColMeta &sm = S.m;
    const uint64_t nent = ((uint64_t)1 << sm.f) * T;
    const uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t e = gid >> log_chunks;
    const uint32_t c = (uint32_t)(gid & ((1ull << log_chunks) - 1));
    unsigned long long key = KEY_INF;
    if (e < nent) {
        const uint32_t o = (uint32_t)(e >> tb), i = (uint32_t)e & (T - 1);
        const uint32_t per = 1u << (sm.d - log_chunks);
        ColView v = make_view(S, T, tb, fn_c0, fn_delta, prev, i);
        key = eval_candidates(v, o, i, c * per, (c + 1) * per);
    }
    if (log_chunks >= 5) {  // a whole warp works on the same entry: reduce before the atomic
        for (int off = 16; off > 0; off >>= 1) {
            unsigned long long other = __shfl_xor_sync(0xFFFFFFFFu, key, off);
            key = other < key ? other : key;
        }
        if ((threadIdx.x & 31) == 0 && e < nent) atomicMin(&keys[e], key);
    } else if (e < nent) {
        atomicMin(&keys[e], key);
    }
}

__global__ void __launch_bounds__(256) col_finalize_kernel(const ColMeta *__restrict__ cols, uint32_t k, uint32_t T,
                                                           uint32_t tb, const unsigned long long *__restrict__ keys,
                                                           uint32_t *__restrict__ out, uint32_t *__restrict__ arena) {
    const ColMeta &m = cols[k];
    const uint64_t nent = ((uint64_t)1 << m.f) * T;
    const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t bpv = 0;
    if (e < nent) {
        const unsigned long long key = keys[e];
        out[e] = (uint32_t)(key >> 32);
        bpv = (uint32_t)key & low_mask(m.d + tb);
    }
    bp_store_warp(arena, m.bp_off, m.bp_width, e, bpv, e < nent);
}

// Backtrace on the device: the packed back-pointers stay in HBM, only the path comes back.
// T == 1: DP-independent chains are traced by independent threads.
__global__ void backtrace_kernel(const ColMeta *__restrict__ cols, const uint32_t *__restrict__ arena,
                                 const uint32_t *__restrict__ chain_begin, uint32_t n_chains, uint32_t n,
                                 const uint32_t *__restrict__ last_vals, uint32_t *__restrict__ path_index,
                                 uint32_t *__restrict__ path_tv, uint32_t *__restrict__ result) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    BtView bv{cols, arena, 1, 0};
    if (c >= n_chains) return;
    const uint32_t k_first = chain_begin[c], k_last = chain_begin[c + 1] - 1;
    const ColMeta &m = cols[k_last];
    const uint32_t bp = bp_load(arena, m.bp_off, m.bp_width, 0);
    const uint32_t x = candidate_index(m, 0, bp);
    backtrace_range(bv, k_last, k_first, x, 0, 0, path_index, path_tv);
    if (k_last == n - 1) result[0] = last_vals[0];
}

// T > 1: transmission values couple the chains (pedigreedptable.cpp:272-297), but only through the one
// value `prev_tv` that the walk carries across a chain boundary (chain_entry).  Three small kernels
// instead of one thread walking the whole table:
//   exits:   thread (c, u) walks chain c as if entered with prev_tv = u and records the value it would
//            hand to chain c-1 (no path written).  The last chain of a plan that ends the table is entered
//            at the optimum of its last column instead (entry < 0), for every u alike.
//   entries: one thread follows the realised entry values right to left over the n_chains boundaries
//            (or, with seg_exits, thread u composes the exits of all chains: what the plan as a whole hands
//            to its predecessor when entered with u -- whmec_segment_exits).
//   paths:   thread c walks chain c again from its realised entry and writes the path.
struct BtArgs {
    const ColMeta *cols;
    const uint32_t *arena, *chain_begin, *last_vals;
    uint32_t T, tb, n_chains;
    int entry;  // prev_tv handed to the last chain by the columns after the plan; < 0: the plan ends the table
};

__device__ __forceinline__ void bt_chain_start(const BtArgs &a, const BtView &bv, uint32_t c, uint32_t u, uint32_t *x,
                                               uint32_t *tv, uint32_t *ptv, uint32_t *cost) {
    const uint32_t k_last = a.chain_begin[c + 1] - 1;
    if (c + 1 == a.n_chains && a.entry < 0) {
        pick_optimum(a.cols[k_last], a.last_vals, a.arena, a.T, a.tb, cost, x, tv, ptv);
    } else {
        *tv = u;
        chain_entry(bv, k_last, u, x, ptv);
    }
}

// backtrace_range (dp_device.h) by one warp: the walk is sequential, but the column records it reads are not -- the lanes stage
// them 16 columns at a time into shared memory, lane 0 walks them paying only for the dependent back-pointer loads.  Returns
// (on every lane) the transmission value handed to column k_first - 1.
constexpr uint32_t BTW_CHUNK = 16;
struct BtWarpSmem {
    ColMeta cols[BTW_CHUNK + 1];
    uint32_t x[BTW_CHUNK], tv[BTW_CHUNK];
};

__device__ __forceinline__ uint32_t backtrace_range_warp(const BtView &v, BtWarpSmem &S, uint32_t k_last, uint32_t k_first, uint32_t x,
                                                         uint32_t tv, uint32_t prev_tv, uint32_t *path_index, uint32_t *path_tv) {
    const uint32_t lane = threadIdx.x & 31u;
    if (path_index && lane == 0) {
        path_index[k_last] = x;
        path_tv[k_last] = tv;
    }
    for (uint32_t hi = k_last; hi > k_first;) {
        const uint32_t lo = hi - k_first > BTW_CHUNK ? hi - BTW_CHUNK : k_first, n = hi - lo;
        constexpr uint32_t CW = sizeof(ColMeta) / 4;
        for (uint32_t w = lane; w < (n + 1) * CW; w += 32) ((uint32_t *)S.cols)[w] = ((const uint32_t *)(v.cols + lo))[w];
        __syncwarp();
        if (lane == 0)
            for (uint32_t k = hi; k > lo; --k) {
                const uint32_t b = x & low_mask(S.cols[k - lo].bw);
                const ColMeta &pm = S.cols[k - 1 - lo];
                const uint32_t bp = bp_load(v.arena, pm.bp_off, pm.bp_width, (uint64_t)b * v.T + prev_tv);
                uint32_t j;
                x = backpointer_to_index(pm, v.tb, b, bp, &j);
                tv = prev_tv;
                prev_tv = j;
                S.x[k - 1 - lo] = x;
                S.tv[k - 1 - lo] = tv;
            }
        __syncwarp();
        if (path_index && lane < n) {
            path_index[lo + lane] = S.x[lane];
            path_tv[lo + lane] = S.tv[lane];
        }
        __syncwarp();
        hi = lo;
    }
    return __shfl_sync(0xFFFFFFFFu, prev_tv, 0);
}

// one warp per (chain, entry value)
__global__ void __launch_bounds__(32) bt_exits_kernel(const BtArgs a, uint32_t *__restrict__ exits) {
    __shared__ BtWarpSmem S;
    const uint32_t idx = blockIdx.x;
    if (idx >= a.n_chains * a.T) return;
    const uint32_t c = idx / a.T, u = idx % a.T;
    BtView bv{a.cols, a.arena, a.T, a.tb};
    uint32_t x, tv, ptv, cost;
    bt_chain_start(a, bv, c, u, &x, &tv, &ptv, &cost);
    const uint32_t out = backtrace_range_warp(bv, S, a.chain_begin[c + 1] - 1, a.chain_begin[c], x, tv, ptv, nullptr, nullptr);
    if (threadIdx.x == 0) exits[idx] = out;
}

__global__ void bt_entries_kernel(const BtArgs a, const uint32_t *__restrict__ exits, uint32_t *__restrict__ entries,
                                  uint32_t *__restrict__ seg_exits) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (seg_exits) {
        if (t >= a.T) return;
        uint32_t e = t;
        for (uint32_t c = a.n_chains; c-- > 0;) e = exits[c * a.T + e];
        seg_exits[t] = e;
        return;
    }
    if (t) return;
    uint32_t e = a.entry < 0 ? 0u : (uint32_t)a.entry;  // the optimum's exit is stored for every u alike
    for (uint32_t c = a.n_chains; c-- > 0;) {
        entries[c] = e;
        e = exits[c * a.T + e];
    }
}

// one warp per chain
__global__ void __launch_bounds__(32) bt_paths_kernel(const BtArgs a, const uint32_t *__restrict__ entries, uint32_t *__restrict__ path_index,
                                                      uint32_t *__restrict__ path_tv, uint32_t *__restrict__ result) {
    __shared__ BtWarpSmem S;
    const uint32_t c = blockIdx.x;
    if (c >= a.n_chains) return;
    BtView bv{a.cols, a.arena, a.T, a.tb};
    uint32_t x, tv, ptv, cost = 0;
    bt_chain_start(a, bv, c, entries[c], &x, &tv, &ptv, &cost);
    backtrace_range_warp(bv, S, a.chain_begin[c + 1] - 1, a.chain_begin[c], x, tv, ptv, path_index, path_tv);
    if (c + 1 == a.n_chains && threadIdx.x == 0) result[0] = cost;
}

// Device buffers come from the device's stream-ordered memory pool with an unlimited release
// threshold: a process that phases many chromosomes pays cudaMalloc for its largest problem once.
template <class Tp>
struct DevBuf {
    Tp *p = nullptr;
    size_t count = 0;
    cudaStream_t stream = nullptr;
    cudaError_t alloc(size_t n, cudaStream_t s) {
        count = n;
        stream = s;
        return cudaMallocAsync((void **)&p, std::max<size_t>(n, 1) * sizeof(Tp), s);
    }
    void release() {
        if (p) cudaFreeAsync(p, stream);
        p = nullptr;
    }
};

// ---- page-locked staging blocks: the memory behind StagedVec (hostpool.h) ------------------------------------------------
// The packer and the planner write the arrays that are uploaded as they are (per-column records, cost functions, panels)
// straight into page-locked blocks, so that an upload is one asynchronous DMA transfer per array: from pageable memory
// cudaMemcpyAsync goes through the driver's bounce buffer and blocks the calling thread for the whole copy.  Blocks are kept for the life of the process and reused
// (cudaHostAlloc costs milliseconds); small arrays stay on the heap.  WHMEC_PINNED_UPLOAD=0 switches the pool off (test hook).
struct PinnedPool {
    struct Block {
        void *p;
        size_t cap;
    };
    static constexpr size_t MIN_BYTES = 128u << 10;   // smaller arrays: heap (their upload is a latency-bound call either way)
    static constexpr size_t MAX_CACHED = 2ull << 30;  // free blocks kept for reuse
    static constexpr size_t MAX_BLOCK = 512ull << 20; // larger arrays (millions of columns) stay pageable: pinning gigabytes takes seconds
    std::mutex m;
    std::vector<Block> free_blocks;
    std::vector<Block> live;  // handed out (a handful per plan)
    size_t cached = 0;
    std::atomic<bool> enabled{true};  // re-read from the environment by every plan (test hook)

    // Block sizes come in classes (1 MiB, then eight steps per power of two), so that a request of the same size as an earlier
    // one always finds that earlier block again: repeated solves of same-sized problems never call cudaHostAlloc (which costs
    // milliseconds and, holding the address-space lock, stalls every other thread of the process that takes a page fault).
    static size_t size_class(size_t bytes) {
        size_t cap = (size_t)1 << 20;
        if (bytes <= cap) return cap;
        while (cap * 2 < bytes) cap *= 2;  // cap < bytes <= 2 * cap
        const size_t step = cap / 8;
        return cap + (bytes - cap + step - 1) / step * step;
    }

    void *alloc(size_t bytes) {
        if (bytes < MIN_BYTES || bytes > MAX_BLOCK || !enabled.load(std::memory_order_relaxed)) return nullptr;
        const size_t want = size_class(bytes);
        {
            std::lock_guard<std::mutex> lk(m);
            size_t best = SIZE_MAX;
            for (size_t i = 0; i < free_blocks.size(); ++i)
                if (free_blocks[i].cap >= bytes && free_blocks[i].cap <= 2 * want &&
                    (best == SIZE_MAX || free_blocks[i].cap < free_blocks[best].cap))
                    best = i;
            if (best != SIZE_MAX) {
                Block b = free_blocks[best];
                free_blocks.erase(free_blocks.begin() + (long)best);
                cached -= b.cap;
                live.push_back(b);
                return b.p;
            }
        }
        const size_t cap = want;
        void *p = nullptr;
        if (cudaHostAlloc(&p, cap, cudaHostAllocPortable) != cudaSuccess) {
            cudaGetLastError();  // clear the error of the failed allocation: the caller falls back to the heap
            return nullptr;
        }
        std::lock_guard<std::mutex> lk(m);
        live.push_back(Block{p, cap});
        return p;
    }
    bool release(void *p) {
        Block b{nullptr, 0};
        std::vector<Block> drop;
        {
            std::lock_guard<std::mutex> lk(m);
            for (size_t i = 0; i < live.size(); ++i)
                if (live[i].p == p) {
                    b = live[i];
                    live[i] = live.back();
                    live.pop_back();
                    break;
                }
            if (!b.p) return false;
            free_blocks.push_back(b);
            cached += b.cap;
            while (cached > MAX_CACHED && !free_blocks.empty()) {  // oldest first
                drop.push_back(free_blocks.front());
                cached -= free_blocks.front().cap;
                free_blocks.erase(free_blocks.begin());
            }
        }
        for (const Block &d : drop) cudaFreeHost(d.p);
        return true;
    }
};
// (heap singletons, never destroyed: a plan that outlives static destruction at process exit must still find them)
PinnedPool &g_pinned = *new PinnedPool();

void install_stage_hooks() {
    static std::once_flag once;
    std::call_once(once, [] {
        set_stage_hooks(StageHooks{[](size_t bytes) { return g_pinned.alloc(bytes); }, [](void *p) { return g_pinned.release(p); }});
    });
    const char *e = std::getenv("WHMEC_PINNED_UPLOAD");
    g_pinned.enabled.store(!(e && e[0] == '0'), std::memory_order_relaxed);
}

// ---- streams and events are reused across plans (creating them costs ~0.5 ms per solve) -----------------------------------
struct StreamSet {
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;    // sweep / backtrace
    cudaEvent_t evh0 = nullptr, evh1 = nullptr;  // uploads of plan_create (read after the first synchronisation that follows)
};
struct StreamCache {
    static constexpr int MAX_DEV = 64;
    static constexpr size_t KEEP = 8;
    std::mutex m;
    std::vector<StreamSet> idle[MAX_DEV];
    cudaError_t acquire(int device, StreamSet &out) {
        if (device >= 0 && device < MAX_DEV) {
            std::lock_guard<std::mutex> lk(m);
            if (!idle[device].empty()) {
                out = idle[device].back();
                idle[device].pop_back();
                return cudaSuccess;
            }
        }
        out = StreamSet{};
        cudaError_t e = cudaStreamCreateWithFlags(&out.stream, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaEventCreate(&out.ev0);
        if (e == cudaSuccess) e = cudaEventCreate(&out.ev1);
        if (e == cudaSuccess) e = cudaEventCreate(&out.evh0);
        if (e == cudaSuccess) e = cudaEventCreate(&out.evh1);
        if (e != cudaSuccess) destroy(out);
        return e;
    }
    static void destroy(StreamSet &s) {
        if (s.ev0) cudaEventDestroy(s.ev0);
        if (s.ev1) cudaEventDestroy(s.ev1);
        if (s.evh0) cudaEventDestroy(s.evh0);
        if (s.evh1) cudaEventDestroy(s.evh1);
        if (s.stream) cudaStreamDestroy(s.stream);
        s = StreamSet{};
    }
    // the stream must be idle (synchronised) and healthy
    void give_back(int device, StreamSet s) {
        if (!s.stream) return;
        if (device >= 0 && device < MAX_DEV) {
            std::lock_guard<std::mutex> lk(m);
            if (idle[device].size() < KEEP) {
                idle[device].push_back(s);
                return;
            }
        }
        destroy(s);
    }
};
StreamCache &g_streams = *new StreamCache();

// The device's default memory pool keeps what a solve frees (release threshold = unlimited): a process that phases many
// chromosomes pays cudaMalloc for its largest problem once.  The memory stays with this process until it exits; a host
// application that shares the GPU with other allocators opts out with WHMEC_KEEP_DEVICE_MEMORY=0 (the pool then trims at every
// synchronisation, the CUDA default).
void keep_pool_memory(int device) {
    static std::atomic<bool> done[64];  // zero-initialised; a second thread repeating the call is harmless
    if (device < 0 || device >= 64 || done[device].load()) return;
    const char *e = std::getenv("WHMEC_KEEP_DEVICE_MEMORY");
    if (e && e[0] == '0') {
        done[device].store(true);
        return;
    }
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
        uint64_t threshold = UINT64_MAX;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &threshold);
    }
    done[device].store(true);
}

}  // namespace

struct whmec_plan {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, evh0 = nullptr, evh1 = nullptr;
    bool h2d_pending = false;  // the uploads of plan_create are enqueued, their duration has not been read yet
    Packed pk;
    whmec_stats stats{};
    bool swept = false;
    bool sweep_pending = false;  // a sweep is enqueued but has not been waited for
    bool use_tiles = false;
    // column-kernel buffers
    DevBuf<ColMeta> d_cols;
    DevBuf<uint32_t> d_fn_c0, d_fn_group, d_val[2], d_arena, d_chain_begin, d_path_index, d_path_tv, d_result;
    DevBuf<int32_t> d_fn_delta;
    DevBuf<unsigned long long> d_keys;
    uint32_t last_buf = 0;
    // batched pedigree sweep (see col_batched_kernel)
    bool use_ped_batch = false;
    DevBuf<PedStep> d_ped_steps;
    DevBuf<uint32_t> d_ped_vals, d_chain_len;
    DevBuf<uint8_t> d_ped_args;
    std::vector<uint32_t> ped_begin[3], ped_grid[3];  // [0] pass 1 (per-input instances), [1] pass 2, [2] pass 1 multi-RHS
    bool ped_multi = false;
    uint64_t ped_max_ent = 0;
    uint32_t ped_slots = 0;
    const uint32_t *d_last_vals = nullptr;
    // segment of a pedigree table shared by several GPUs (whmec_segment_*): 0 = whole table,
    // 1 = first segment, 2 = segment continuing a table (its first column receives an input vector)
    int segment = 0;
    bool transferred = false;
    int exits_mode = 0;  // 0: not computed since the last sweep; 1: last chain entered at the optimum; 2: like any chain
    DevBuf<uint32_t> d_in_vec, d_matrix, d_bt_exits, d_bt_entries;
    // fused trio sweep (ped_fused_kernel / ped_fused_cluster_kernel, ped_fused.h)
    bool use_ped_fused = false;
    uint32_t ped_cluster = 1;  // CTAs per chain of the fused pedigree sweep
    DevBuf<uint32_t> d_chain_rows, d_chain_in, d_chain_out;
    uint32_t sweeps_done = 0;
    cudaGraphExec_t graph_exec = nullptr;
    // tile path
    TilePlan tiles;

    ~whmec_plan() {
        cudaSetDevice(device);
        // nothing of this plan may still be in flight when its buffers go back to their pools: the page-locked host blocks
        // behind pk / the tile schedule are the sources of asynchronous uploads
        const bool healthy = !stream || cudaStreamSynchronize(stream) == cudaSuccess;
        d_cols.release(); d_fn_c0.release(); d_fn_group.release(); d_val[0].release(); d_val[1].release();
        d_arena.release(); d_chain_begin.release(); d_path_index.release(); d_path_tv.release();
        d_result.release(); d_fn_delta.release(); d_keys.release();
        d_ped_steps.release(); d_ped_vals.release(); d_chain_len.release(); d_ped_args.release();
        d_in_vec.release(); d_matrix.release(); d_bt_exits.release(); d_bt_entries.release();
        d_chain_rows.release(); d_chain_in.release(); d_chain_out.release();
        tiles.release(stream);
        if (graph_exec) cudaGraphExecDestroy(graph_exec);
        StreamSet set{stream, ev0, ev1, evh0, evh1};
        if (stream && healthy) g_streams.give_back(device, set);  // (the frees above are stream-ordered: whoever takes the stream next queues behind them)
        else StreamCache::destroy(set);
    }
};

namespace {

// The packed problem and the tile schedule are tens of MB of freshly touched host memory per call;
// returning them to the OS on every free (glibc's default for large blocks) makes each call pay the
// page faults again.  Keep freed blocks in the process heap instead (opt out: WHMEC_KEEP_HOST_MEMORY=0).
void keep_host_memory() {
    static std::atomic<bool> done{false};
    if (done.exchange(true)) return;
    const char *e = std::getenv("WHMEC_KEEP_HOST_MEMORY");
    if (e && e[0] == '0') return;
    mallopt(M_MMAP_THRESHOLD, 1 << 30);
    mallopt(M_TRIM_THRESHOLD, 1 << 30);
}

int plan_create_impl(const whmec_problem *p, int device, whmec_plan *pl, std::string &msg, int segment = 0) {
    keep_host_memory();
    // the packer's upload arrays come from page-locked blocks, which belong to a CUDA context: select the device first
    // (a failure here is reported by the checked call below, after the input has been validated as before)
    if (cudaSetDevice(device) == cudaSuccess) install_stage_hooks();
    else cudaGetLastError();
    pl->device = device;
    pl->segment = segment;
    // single-individual problems normally run on the tile kernel, which needs no per-read cost deltas
    const char *force = std::getenv("WHMEC_FORCE_COLUMN_KERNEL");  // test hook: exercise the general path on T == 1
    const bool forced_column = force && force[0] == '1';
    const bool tile_candidate = p->n_ind == 1 && p->n_trios == 0 && !forced_column && !segment;
    using pclk = std::chrono::steady_clock;
    const bool timing = std::getenv("WHMEC_TIMING") != nullptr;
    auto pms = [](pclk::time_point a, pclk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    const auto tc0 = pclk::now();
    int rc = pack_problem(p, pl->pk, msg, !tile_candidate);
    if (rc != WHMEC_OK) return rc;
    Packed &pk = pl->pk;
    const auto tc1 = pclk::now();
    uint64_t h2d = 0;
    auto device_setup = [&]() -> int {  // device, stream + events (reused across plans), start of the upload window
        CUDA_TRY(cudaSetDevice(device));
        keep_pool_memory(device);
        StreamSet set;
        CUDA_TRY(g_streams.acquire(device, set));
        pl->stream = set.stream;
        pl->ev0 = set.ev0;
        pl->ev1 = set.ev1;
        pl->evh0 = set.evh0;
        pl->evh1 = set.evh1;
        CUDA_TRY(cudaEventRecord(pl->evh0, pl->stream));
        return WHMEC_OK;
    };
    if (tile_candidate && pk.n > 0) {
        // the per-column records of the packer (4 MB for 50k columns) travel while the host plans the tiles
        rc = device_setup();
        if (rc != WHMEC_OK) return rc;
        CUDA_TRY(pl->d_cols.alloc(pk.n, pl->stream));
        CUDA_TRY(cudaMemcpyAsync(pl->d_cols.p, pk.cols.data(), (size_t)pk.n * sizeof(ColMeta), cudaMemcpyHostToDevice, pl->stream));
        h2d += (uint64_t)pk.n * sizeof(ColMeta);
    }
    pl->use_tiles = tile_candidate && pk.n > 0 && pl->tiles.plan(pk);
    const auto tc2 = pclk::now();
    if (tile_candidate && !pl->use_tiles && pk.n > 0) {  // planner declined: the column kernel needs the deltas
        CUDA_TRY(cudaStreamSynchronize(pl->stream));  // the upload above reads the arrays that are packed again now
        h2d = 0;
        rc = pack_problem(p, pl->pk, msg, true);
        if (rc != WHMEC_OK) return rc;
    }
    pl->device = device;
    pl->stats = pk.stats;
    if (segment) {
        if (pk.T == 1 || pk.n == 0) {
            msg = "unsupported: table segments are for pedigrees (T > 1) and need at least one column; single-individual chains are independent problems";
            return WHMEC_ERR_UNSUPPORTED;
        }
        if (segment == 2) pk.cols[0].first = 0;  // column 0 reads the vector handed over by the preceding segment
    }
    if (pk.n == 0) return WHMEC_OK;
    if (pk.max_d + pk.tb > 32) {  // (most reads ending in one column: found by the packer's workers, not by another pass over the columns)
        msg = "unsupported: dropped reads + transmission bits exceed 32";
        return WHMEC_ERR_UNSUPPORTED;
    }
    if (!pl->stream) {
        rc = device_setup();
        if (rc != WHMEC_OK) return rc;
    }
    const uint32_t n = pk.n;

    CUDA_TRY(pl->d_path_index.alloc(n, pl->stream));
    CUDA_TRY(pl->d_path_tv.alloc(n, pl->stream));
    CUDA_TRY(pl->d_result.alloc(4, pl->stream));
    const auto tc3 = pclk::now();

    if (pl->use_tiles) {
        rc = pl->tiles.create(pk, pl->stream, h2d, msg, pl->d_cols.p);
        if (rc != WHMEC_OK) return rc;
        if (timing)
            std::fprintf(stderr, "[whmec] create: pack %.2f ms, plan %.2f ms, stream + events + result buffers %.2f ms, tiles.create (alloc + upload enqueue) %.2f ms\n",
                         pms(tc0, tc1), pms(tc1, tc2), pms(tc2, tc3), pms(tc3, pclk::now()));
        pl->stats.path_kind = 1;
        pl->stats.backptr_bytes = pl->tiles.backptr_bytes;
    } else {
        const size_t free_b = device_available_bytes();
        uint64_t max_ent = 1;
        for (const ColMeta &m : pk.cols) max_ent = std::max<uint64_t>(max_ent, ((uint64_t)1 << m.f) * pk.T);
        uint64_t need = pk.bp_words * 4 + max_ent * (4 * 2 + 8) + pk.fn_delta.size() * 4 + (uint64_t)n * sizeof(ColMeta);
        if (need + (512ull << 20) > free_b) {
            msg = "back-pointer storage exceeds the free HBM of this device";
            return WHMEC_ERR_UNSUPPORTED;
        }
        if (!pl->d_cols.p) CUDA_TRY(pl->d_cols.alloc(n, pl->stream));  // (already there when the tile planner declined the problem)
        CUDA_TRY(pl->d_fn_c0.alloc(pk.fn_c0.size(), pl->stream));
        CUDA_TRY(pl->d_fn_delta.alloc(pk.fn_delta.size(), pl->stream));
        CUDA_TRY(pl->d_fn_group.alloc(pk.fn_group.size(), pl->stream));
        CUDA_TRY(pl->d_chain_begin.alloc(pk.chain_begin.size(), pl->stream));
        CUDA_TRY(pl->d_val[0].alloc(max_ent, pl->stream));
        CUDA_TRY(pl->d_val[1].alloc(max_ent, pl->stream));
        CUDA_TRY(pl->d_keys.alloc(max_ent, pl->stream));
        CUDA_TRY(pl->d_arena.alloc(pk.bp_words + 1, pl->stream));
        auto up = [&](void *dst, const void *src, size_t bytes) {
            h2d += bytes;
            return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, pl->stream);
        };
        CUDA_TRY(up(pl->d_cols.p, pk.cols.data(), (size_t)n * sizeof(ColMeta)));
        CUDA_TRY(up(pl->d_fn_c0.p, pk.fn_c0.data(), pk.fn_c0.size() * 4));
        CUDA_TRY(up(pl->d_fn_delta.p, pk.fn_delta.data(), pk.fn_delta.size() * 4));
        CUDA_TRY(up(pl->d_fn_group.p, pk.fn_group.data(), pk.fn_group.size() * 4));
        CUDA_TRY(up(pl->d_chain_begin.p, pk.chain_begin.data(), pk.chain_begin.size() * 4));
        pl->stats.path_kind = 2;
        // pedigrees with several chains: batched two-pass sweep
        const char *seq = std::getenv("WHMEC_PED_SEQUENTIAL");
        const uint32_t C = (uint32_t)pk.chain_begin.size() - 1;
        // one trio, shapes of ped_fused.h: one block per chain with the projection in shared memory (3 launches)
        bool fused_ok = false;
        {
            const char *pf = std::getenv("WHMEC_PED_FUSED");
            fused_ok = !(pf && pf[0] == '0') && pk.T == PF_T && (C >= 2 || segment) && pk.safe31 && !(seq && seq[0] == '1' && !segment);
            for (uint32_t k = 0; k < n && fused_ok; ++k) fused_ok = pf_column_ok(pk.cols[k], pk.fn_group.data() + pk.cols[k].grp_off);
        }
        if (fused_ok) {
            CUDA_TRY(pl->d_chain_rows.alloc((size_t)C * PF_T, pl->stream));
            CUDA_TRY(pl->d_chain_in.alloc((size_t)C * PF_T, pl->stream));
            CUDA_TRY(pl->d_chain_out.alloc((size_t)C * PF_T, pl->stream));
            CUDA_TRY(cudaFuncSetAttribute(ped_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PF_SMEM));
            CUDA_TRY(cudaFuncSetAttribute(ped_fused_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PF_CLUSTER_SMEM));
            {   // fewer chains than SMs: a cluster of 2 / 4 / 8 CTAs per chain (WHMEC_PED_CLUSTER=n forces n, 1 = off)
                int dev = 0, sms = 132;
                CUDA_TRY(cudaGetDevice(&dev));
                CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
                uint32_t cs = 1;
                while (cs * 2 <= PF_MAX_CLUSTER && (uint64_t)C * cs * 2 <= (uint64_t)sms) cs *= 2;
                if (const char *e = std::getenv("WHMEC_PED_CLUSTER")) {
                    const int want = std::atoi(e);
                    if (want == 1 || want == 2 || want == 4 || want == 8) cs = (uint32_t)want;
                }
                pl->ped_cluster = cs;
            }
            pl->use_ped_fused = true;
            pl->use_ped_batch = true;  // two-pass sweep: the backtrace and the optimum read the chains' final values
            pl->d_last_vals = pl->d_chain_out.p + (size_t)(C - 1) * PF_T;
            pl->stats.path_kind = 3;
        } else if (pk.T > 1 && (C >= 2 || segment) && pk.safe31 && !(seq && seq[0] == '1' && !segment)) {
            const uint32_t T = pk.T;
            const uint32_t slots = C * T + C;
            // the batch buffers (values + argmins of every (chain, unit vector) instance) count against the free HBM as well
            if ((uint64_t)slots * 2 * max_ent * 4 < (8ull << 30) && (uint64_t)C * T <= 65535 &&
                need + (uint64_t)slots * 2 * max_ent * 5 + (512ull << 20) <= free_b) {
                std::vector<PedStep> steps;
                std::vector<uint32_t> clen(C);
                uint32_t maxlen = 0;
                for (uint32_t c = 0; c < C; ++c) {
                    clen[c] = pk.chain_begin[c + 1] - pk.chain_begin[c];
                    maxlen = std::max(maxlen, clen[c]);
                }
                auto blocks_for = [&](const ColMeta &m) -> uint32_t {
                    const uint64_t nent = ((uint64_t)1 << m.f) * T;
                    if (m.d > 7) return (uint32_t)nent;
                    const uint64_t epb = 256u >> col_lane_bits(m.f + pk.tb, m.d);
                    return (uint32_t)((nent + epb - 1) / epb);
                };
                pl->ped_multi = T <= MULTI_MAX;
                for (int pass = 0; pass < 3; ++pass) {
                    pl->ped_begin[pass].clear();
                    pl->ped_grid[pass].clear();
                    if (pass == 2 && !pl->ped_multi) continue;
                    for (uint32_t st = 0; st < maxlen; ++st) {
                        pl->ped_begin[pass].push_back((uint32_t)steps.size());
                        uint32_t gmax = 0;
                        // pass 0: chain 0 (true input) and, without the multi-RHS kernel, every (chain, unit vector);
                        // pass 1: chains >= 1 with their true inputs; pass 2: one multi-RHS instance per chain >= 1
                        // with the multi-RHS kernel pass 0 is empty: chain 0 (whose input is known: the first column
                        // of the table ignores it) runs in pass 1 like every other chain
                        const uint32_t c_begin = (pass == 0 && !pl->ped_multi) ? 0 : (pass == 0 ? C : 0);
                        const uint32_t c_end = C;
                        for (uint32_t c = c_begin; c < c_end; ++c) {
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
                                steps.push_back(ps);
                            }
                            gmax = std::max(gmax, blocks_for(m));
                        }
                        pl->ped_grid[pass].push_back(gmax);
                    }
                    pl->ped_begin[pass].push_back((uint32_t)steps.size());
                }
                CUDA_TRY(pl->d_ped_steps.alloc(steps.size(), pl->stream));
                CUDA_TRY(pl->d_ped_vals.alloc((uint64_t)slots * 2 * max_ent, pl->stream));
                CUDA_TRY(pl->d_ped_args.alloc((uint64_t)slots * 2 * max_ent, pl->stream));
                CUDA_TRY(pl->d_chain_len.alloc(C, pl->stream));
                CUDA_TRY(up(pl->d_ped_steps.p, steps.data(), steps.size() * sizeof(PedStep)));
                CUDA_TRY(up(pl->d_chain_len.p, clen.data(), C * 4));
                CUDA_TRY(cudaStreamSynchronize(pl->stream));  // `steps` and `clen` are stack-local
                pl->ped_max_ent = max_ent;
                pl->ped_slots = slots;
                pl->use_ped_batch = true;
                const uint32_t last_slot = C * T + (C - 1);
                pl->d_last_vals = pl->d_ped_vals.p + ((uint64_t)last_slot * 2 + ((clen[C - 1] - 1) & 1u)) * max_ent;
                pl->stats.path_kind = 3;
            }
        }
        if (segment && !pl->use_ped_batch) {
            msg = "unsupported: this segment cannot run the two-pass pedigree sweep (costs beyond 2^28 or state beyond the budget)";
            return WHMEC_ERR_UNSUPPORTED;
        }
        if (pk.T > 1) {
            CUDA_TRY(pl->d_bt_exits.alloc((size_t)C * pk.T, pl->stream));
            CUDA_TRY(pl->d_bt_entries.alloc(C, pl->stream));
        }
        if (segment) {
            CUDA_TRY(pl->d_in_vec.alloc(pk.T, pl->stream));
            CUDA_TRY(pl->d_matrix.alloc((size_t)pk.T * pk.T, pl->stream));
        }
    }
    // No synchronisation here: the uploads (asynchronous DMA from the page-locked arrays of `pk` / the tile schedule, which live
    // as long as the plan) overlap whatever the host does next; the sweep's first launch queues behind them on the same stream.
    CUDA_TRY(cudaEventRecord(pl->evh1, pl->stream));
    pl->h2d_pending = true;
    pl->stats.h2d_bytes = h2d;
    return WHMEC_OK;
}

// after a synchronisation of the plan's stream: the duration of the uploads of plan_create
void read_h2d_time(whmec_plan *pl) {
    if (!pl->h2d_pending) return;
    pl->h2d_pending = false;
    if (cudaEventElapsedTime(&pl->stats.h2d_ms, pl->evh0, pl->evh1) != cudaSuccess) {
        cudaGetLastError();
        pl->stats.h2d_ms = 0;
    }
}

// One pass of the batched pedigree sweep.  pass 0: unit input vectors, values only (transfer matrices);
// pass 1: true input vectors, back-pointers written.
int ped_pass(whmec_plan *pl, int pass, uint32_t &launches, std::string &msg) {
    Packed &pk = pl->pk;
    const uint32_t T = pk.T, tb = pk.tb;
    if (pass == 0) {
        const uint32_t unit_slots = ((uint32_t)pk.chain_begin.size() - 1) * T;
        ped_init_kernel<<<(unit_slots * T + 255) / 256, 256, 0, pl->stream>>>(pl->d_ped_vals.p, pl->ped_max_ent, T, unit_slots);
        ++launches;
    }
    const size_t nsteps = pl->ped_grid[pass].size();
    for (size_t st = 0; st < nsteps; ++st) {
        const uint32_t b0 = pl->ped_begin[pass][st], b1 = pl->ped_begin[pass][st + 1];
        if (b1 > b0) {
            dim3 grid(pl->ped_grid[pass][st], b1 - b0);
            col_batched_kernel<<<grid, 256, 0, pl->stream>>>(pl->d_ped_steps.p + b0, pl->d_ped_vals.p, pl->ped_max_ent, T, tb,
                                                               pl->d_fn_c0.p, pl->d_fn_delta.p, pl->d_fn_group.p, pl->d_arena.p,
                                                               (uint32_t)(st & 1), pl->d_ped_args.p);
            ++launches;
        }
        if (pass == 0 && pl->ped_multi && st < pl->ped_grid[2].size()) {
            const uint32_t m0 = pl->ped_begin[2][st], m1 = pl->ped_begin[2][st + 1];
            if (m1 > m0) {
                dim3 grid(pl->ped_grid[2][st], m1 - m0);
                col_multi_kernel<<<grid, 256, 0, pl->stream>>>(pl->d_ped_steps.p + m0, pl->d_ped_vals.p, pl->ped_max_ent, T, tb,
                                                                 pl->d_fn_c0.p, pl->d_fn_delta.p, pl->d_fn_group.p, (uint32_t)(st & 1));
                ++launches;
            }
        }
    }
    CUDA_TRY(cudaGetLastError());
    return WHMEC_OK;
}

// every chain's true input vector from the transfer matrices (in_vec: see ped_prefix_kernel)
int ped_prefix(whmec_plan *pl, const uint32_t *d_in_vec, uint32_t &launches, std::string &msg) {
    const uint32_t C = (uint32_t)pl->pk.chain_begin.size() - 1;
    ped_prefix_kernel<<<1, 32, 0, pl->stream>>>(pl->d_ped_vals.p, pl->ped_max_ent, pl->pk.T, C, pl->d_chain_len.p, d_in_vec,
                                                 pl->segment == 2, nullptr);
    ++launches;
    CUDA_TRY(cudaGetLastError());
    return WHMEC_OK;
}

// the fused sweep in pieces: pass 1 (unit input e_0 of every chain, values only), prefix, pass 2 (true inputs, back-pointers)
PedFusedArgs ped_fused_args(whmec_plan *pl, bool unit) {
    return PedFusedArgs{pl->d_cols.p, pl->d_chain_begin.p, pl->d_fn_c0.p, pl->d_fn_group.p, pl->d_fn_delta.p, pl->d_arena.p,
                        pl->d_chain_in.p, unit ? pl->d_chain_rows.p : pl->d_chain_out.p, unit ? 1u : 0u};
}

int ped_fused_pass(whmec_plan *pl, bool unit, std::string &msg) {
    const uint32_t C = (uint32_t)pl->pk.chain_begin.size() - 1;
    if (pl->ped_cluster > 1) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(C * pl->ped_cluster);
        cfg.blockDim = dim3(PF_THREADS);
        cfg.dynamicSmemBytes = PF_CLUSTER_SMEM;
        cfg.stream = pl->stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeClusterDimension;
        attr[0].val.clusterDim.x = pl->ped_cluster;
        attr[0].val.clusterDim.y = 1;
        attr[0].val.clusterDim.z = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        CUDA_TRY(cudaLaunchKernelEx(&cfg, ped_fused_cluster_kernel, ped_fused_args(pl, unit)));
    } else {
        ped_fused_kernel<<<C, PF_THREADS, PF_SMEM, pl->stream>>>(ped_fused_args(pl, unit));
    }
    CUDA_TRY(cudaGetLastError());
    return WHMEC_OK;
}

int ped_fused_prefix(whmec_plan *pl, const uint32_t *d_in_vec, uint32_t *d_matrix, std::string &msg) {
    const uint32_t C = (uint32_t)pl->pk.chain_begin.size() - 1;
    ped_fused_prefix_kernel<<<1, 32, 0, pl->stream>>>(pl->d_chain_rows.p, C, d_in_vec, pl->segment == 2, pl->d_chain_in.p, d_matrix);
    CUDA_TRY(cudaGetLastError());
    return WHMEC_OK;
}

// three launches for the whole table
int ped_fused_sweep(whmec_plan *pl, std::string &msg) {
    int rc = ped_fused_pass(pl, true, msg);
    if (rc == WHMEC_OK) rc = ped_fused_prefix(pl, nullptr, nullptr, msg);
    if (rc == WHMEC_OK) rc = ped_fused_pass(pl, false, msg);
    pl->stats.kernel_launches = 3;
    return rc;
}

int ped_batched_sweep(whmec_plan *pl, std::string &msg) {
    if (pl->use_ped_fused) return ped_fused_sweep(pl, msg);
    uint32_t launches = 0;
    int rc = ped_pass(pl, 0, launches, msg);
    if (rc == WHMEC_OK) rc = ped_prefix(pl, nullptr, launches, msg);
    if (rc == WHMEC_OK) rc = ped_pass(pl, 1, launches, msg);
    pl->stats.kernel_launches = launches;
    return rc;
}

// The column path issues one (small) kernel per column; a sweep of the same plan is replayed from a
// CUDA graph from the second time on (launch-bound inner loop, captured once).
int column_sweep(whmec_plan *pl, std::string &msg) {
    Packed &pk = pl->pk;
    const uint32_t n = pk.n, T = pk.T, tb = pk.tb;
    if (pl->graph_exec) {
        CUDA_TRY(cudaGraphLaunch(pl->graph_exec, pl->stream));
        return WHMEC_OK;
    }
    const bool capture = pl->sweeps_done >= 1 && n >= 64;
    if (capture) CUDA_TRY(cudaStreamBeginCapture(pl->stream, cudaStreamCaptureModeThreadLocal));
    uint32_t launches = 0;
    uint32_t curb = 0;
    for (uint32_t k = 0; k < n; ++k) {
        const ColMeta &m = pk.cols[k];
        const uint64_t nent = ((uint64_t)1 << m.f) * T;
        const uint32_t *prev = pl->d_val[curb ^ 1].p;
        uint32_t *out = pl->d_val[curb].p;
        if (m.d <= 6) {
            const uint32_t lc = col_lane_bits(m.f + tb, m.d);
            const uint64_t ent_per_block = 256u >> lc;
            const unsigned blocks = (unsigned)((nent + ent_per_block - 1) / ent_per_block);
            col_direct_kernel<<<blocks, 256, 0, pl->stream>>>(m, pk.fn_group[m.grp_off + T], T, tb, pl->d_fn_c0.p, pl->d_fn_delta.p,
                                                               pl->d_fn_group.p, prev, out, pl->d_arena.p);
            launches += 1;
        } else {
            const uint32_t log_chunks = m.d - 6;
            if (cudaError_t e = cudaMemsetAsync(pl->d_keys.p, 0xFF, nent * 8, pl->stream); e != cudaSuccess) {
                if (capture) {  // do not leave the stream in capture mode
                    cudaGraph_t dead = nullptr;
                    cudaStreamEndCapture(pl->stream, &dead);
                    if (dead) cudaGraphDestroy(dead);
                }
                msg = std::string("cudaMemsetAsync (column sweep): ") + cudaGetErrorString(e);
                return WHMEC_ERR_CUDA;
            }
            const uint64_t threads = nent << log_chunks;
            const unsigned blocks = (unsigned)((threads + 255) / 256);
            col_chunk_kernel<<<blocks, 256, 0, pl->stream>>>(m, pk.fn_group[m.grp_off + T], T, tb, pl->d_fn_c0.p, pl->d_fn_delta.p,
                                                              pl->d_fn_group.p, prev, log_chunks, pl->d_keys.p);
            col_finalize_kernel<<<(unsigned)((nent + 255) / 256), 256, 0, pl->stream>>>(pl->d_cols.p, k, T, tb, pl->d_keys.p,
                                                                                          out, pl->d_arena.p);
            launches += 2;
        }
        curb ^= 1;
    }
    pl->last_buf = curb ^ 1;
    pl->stats.kernel_launches = launches;
    if (capture) {
        cudaGraph_t graph = nullptr;
        CUDA_TRY(cudaStreamEndCapture(pl->stream, &graph));
        CUDA_TRY(cudaGraphInstantiate(&pl->graph_exec, graph, 0));
        cudaGraphDestroy(graph);
        CUDA_TRY(cudaGraphLaunch(pl->graph_exec, pl->stream));
    }
    CUDA_TRY(cudaGetLastError());
    pl->sweeps_done++;
    return WHMEC_OK;
}

// wait == false: the sweep is only enqueued on the plan's stream; plan_finish_impl (same stream) collects it
int plan_sweep_impl(whmec_plan *pl, std::string &msg, bool wait = true) {
    if (pl->pk.n == 0) {
        pl->swept = true;
        return WHMEC_OK;
    }
    CUDA_TRY(cudaSetDevice(pl->device));
    CUDA_TRY(cudaEventRecord(pl->ev0, pl->stream));
    int rc;
    if (pl->use_tiles) {
        rc = pl->tiles.sweep(pl->pk, pl->stream, msg);
        pl->stats.kernel_launches = pl->tiles.launches;
        pl->stats.state_bytes = pl->tiles.state_bytes;
    } else if (pl->use_ped_batch) {
        rc = ped_batched_sweep(pl, msg);
    } else {
        rc = column_sweep(pl, msg);
    }
    if (rc != WHMEC_OK) return rc;
    CUDA_TRY(cudaEventRecord(pl->ev1, pl->stream));
    pl->swept = true;
    pl->exits_mode = 0;
    pl->sweep_pending = !wait;
    if (!wait) return WHMEC_OK;
    CUDA_TRY(cudaStreamSynchronize(pl->stream));
    CUDA_TRY(cudaEventElapsedTime(&pl->stats.sweep_ms, pl->ev0, pl->ev1));
    read_h2d_time(pl);
    return WHMEC_OK;
}

BtArgs bt_args(const whmec_plan *pl, int entry) {
    const Packed &pk = pl->pk;
    return BtArgs{pl->d_cols.p, pl->d_arena.p, pl->d_chain_begin.p, pl->use_ped_batch ? pl->d_last_vals : pl->d_val[pl->last_buf].p,
                  pk.T, pk.tb, (uint32_t)pk.chain_begin.size() - 1, entry};
}

// exits of every (chain, entry value): the first of the three backtrace kernels for T > 1
int pedigree_exits(whmec_plan *pl, int entry, std::string &msg) {
    const BtArgs a = bt_args(pl, entry);
    const uint32_t threads = a.n_chains * a.T;
    bt_exits_kernel<<<threads, 32, 0, pl->stream>>>(a, pl->d_bt_exits.p);
    CUDA_TRY(cudaGetLastError());
    pl->exits_mode = entry < 0 ? 1 : 2;
    return WHMEC_OK;
}

// entry < 0: the plan ends the table (start from the optimum of the last column); otherwise the
// transmission value handed over by the segment that follows.
int pedigree_backtrace(whmec_plan *pl, int entry, std::string &msg) {
    if (pl->exits_mode != (entry < 0 ? 1 : 2)) {  // the table of exits depends only on how the last chain is entered
        int rc = pedigree_exits(pl, entry, msg);
        if (rc != WHMEC_OK) return rc;
    }
    const BtArgs a = bt_args(pl, entry);
    bt_entries_kernel<<<1, 32, 0, pl->stream>>>(a, pl->d_bt_exits.p, pl->d_bt_entries.p, nullptr);
    bt_paths_kernel<<<a.n_chains, 32, 0, pl->stream>>>(a, pl->d_bt_entries.p, pl->d_path_index.p, pl->d_path_tv.p, pl->d_result.p);
    CUDA_TRY(cudaGetLastError());
    return WHMEC_OK;
}

int plan_finish_impl(whmec_plan *pl, whmec_solution *s, std::string &msg, int entry = -1) {
    Packed &pk = pl->pk;
    const uint32_t n = pk.n;
    if (n == 0) {  // pedigreedptable.cpp:88-92
        s->cost = 0;
        if (s->partition) std::memset(s->partition, 1, pk.n_reads);
        return WHMEC_OK;
    }
    if (!pl->swept) {
        msg = "whmec_plan_finish called before whmec_plan_sweep";
        return WHMEC_ERR_INPUT;
    }
    CUDA_TRY(cudaSetDevice(pl->device));
    using fclk = std::chrono::steady_clock;
    const bool timing = std::getenv("WHMEC_TIMING") != nullptr;
    const auto tf0 = fclk::now();
    if (pl->sweep_pending) {  // enqueued by plan_sweep_impl(wait = false): its events are reused below
        CUDA_TRY(cudaEventSynchronize(pl->ev1));
        CUDA_TRY(cudaEventElapsedTime(&pl->stats.sweep_ms, pl->ev0, pl->ev1));
        pl->sweep_pending = false;
    }
    CUDA_TRY(cudaEventRecord(pl->ev0, pl->stream));
    if (pl->use_tiles) {
        int rc = pl->tiles.backtrace(pk, pl->stream, pl->d_path_index.p, pl->d_result.p, msg);
        if (rc != WHMEC_OK) return rc;
        pl->stats.kernel_launches = pl->tiles.launches;  // a memory-bounded sweep re-sweeps segments during the backtrace
        CUDA_TRY(cudaMemsetAsync(pl->d_path_tv.p, 0, (size_t)n * 4, pl->stream));
    } else {
        const uint32_t n_chains = (uint32_t)pk.chain_begin.size() - 1;
        const uint32_t *last_vals = pl->use_ped_batch ? pl->d_last_vals : pl->d_val[pl->last_buf].p;
        if (pk.T == 1) {
            backtrace_kernel<<<(n_chains + 63) / 64, 64, 0, pl->stream>>>(pl->d_cols.p, pl->d_arena.p, pl->d_chain_begin.p, n_chains, n,
                                                                           last_vals, pl->d_path_index.p, pl->d_path_tv.p, pl->d_result.p);
        } else {
            int rc = pedigree_backtrace(pl, entry, msg);
            if (rc != WHMEC_OK) return rc;
        }
        CUDA_TRY(cudaGetLastError());
    }
    std::vector<uint32_t> pidx(n), ptv(n);
    uint32_t result[4] = {0, 0, 0, 0};
    CUDA_TRY(cudaMemcpyAsync(pidx.data(), pl->d_path_index.p, (size_t)n * 4, cudaMemcpyDeviceToHost, pl->stream));
    CUDA_TRY(cudaMemcpyAsync(ptv.data(), pl->d_path_tv.p, (size_t)n * 4, cudaMemcpyDeviceToHost, pl->stream));
    CUDA_TRY(cudaMemcpyAsync(result, pl->d_result.p, 16, cudaMemcpyDeviceToHost, pl->stream));
    CUDA_TRY(cudaEventRecord(pl->ev1, pl->stream));
    CUDA_TRY(cudaStreamSynchronize(pl->stream));
    CUDA_TRY(cudaEventElapsedTime(&pl->stats.d2h_ms, pl->ev0, pl->ev1));
    read_h2d_time(pl);
    pl->stats.d2h_bytes = (uint64_t)n * 8 + 16;
    s->cost = result[0];
    const auto tf1 = fclk::now();
    const int orc = build_outputs(pk, pidx.data(), ptv.data(), s, msg);
    if (timing)
        std::fprintf(stderr, "[whmec] finish: backtrace + D2H %.2f ms, outputs %.2f ms\n", std::chrono::duration<double, std::milli>(tf1 - tf0).count(),
                     std::chrono::duration<double, std::milli>(fclk::now() - tf1).count());
    return orc;
}

// ---- segments of a pedigree table (include/whmec.h) ----
int segment_check(const whmec_plan *pl, std::string &msg) {
    if (!pl || !pl->segment || !pl->use_ped_batch) {
        msg = "not a segment plan (use whmec_segment_create)";
        return WHMEC_ERR_INPUT;
    }
    return WHMEC_OK;
}

int segment_transfer_impl(whmec_plan *pl, uint32_t *matrix, std::string &msg) {
    int rc = segment_check(pl, msg);
    if (rc != WHMEC_OK) return rc;
    const Packed &pk = pl->pk;
    const uint32_t C = (uint32_t)pk.chain_begin.size() - 1;
    CUDA_TRY(cudaSetDevice(pl->device));
    CUDA_TRY(cudaEventRecord(pl->ev0, pl->stream));
    uint32_t launches = 0;
    if (pl->use_ped_fused) {
        rc = ped_fused_pass(pl, true, msg);
        if (rc == WHMEC_OK) rc = ped_fused_prefix(pl, nullptr, pl->d_matrix.p, msg);
        if (rc != WHMEC_OK) return rc;
        launches = 2;
    } else {
        rc = ped_pass(pl, 0, launches, msg);
        if (rc != WHMEC_OK) return rc;
        ped_prefix_kernel<<<(pk.T + 31) / 32, 32, 0, pl->stream>>>(pl->d_ped_vals.p, pl->ped_max_ent, pk.T, C, pl->d_chain_len.p, nullptr,
                                                                    pl->segment == 2, pl->d_matrix.p);
        ++launches;
    }
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(matrix, pl->d_matrix.p, (size_t)pk.T * pk.T * 4, cudaMemcpyDeviceToHost, pl->stream));
    CUDA_TRY(cudaEventRecord(pl->ev1, pl->stream));
    CUDA_TRY(cudaStreamSynchronize(pl->stream));
    CUDA_TRY(cudaEventElapsedTime(&pl->stats.sweep_ms, pl->ev0, pl->ev1));
    pl->stats.kernel_launches = launches;
    pl->transferred = true;
    return WHMEC_OK;
}

int segment_sweep_impl(whmec_plan *pl, const uint32_t *in_vec, uint32_t *out_vec, std::string &msg) {
    int rc = segment_check(pl, msg);
    if (rc != WHMEC_OK) return rc;
    if (!pl->transferred) {
        msg = "whmec_segment_sweep called before whmec_segment_transfer";
        return WHMEC_ERR_INPUT;
    }
    if ((pl->segment == 2) != (in_vec != nullptr)) {
        msg = "a continuing segment needs an input vector, the first segment of a table takes none";
        return WHMEC_ERR_INPUT;
    }
    const uint32_t T = pl->pk.T;
    CUDA_TRY(cudaSetDevice(pl->device));
    CUDA_TRY(cudaEventRecord(pl->ev0, pl->stream));
    if (in_vec) CUDA_TRY(cudaMemcpyAsync(pl->d_in_vec.p, in_vec, (size_t)T * 4, cudaMemcpyHostToDevice, pl->stream));
    uint32_t launches = 0;
    if (pl->use_ped_fused) {
        rc = ped_fused_prefix(pl, in_vec ? pl->d_in_vec.p : nullptr, nullptr, msg);
        if (rc == WHMEC_OK) rc = ped_fused_pass(pl, false, msg);
        launches = 2;
    } else {
        rc = ped_prefix(pl, in_vec ? pl->d_in_vec.p : nullptr, launches, msg);
        if (rc == WHMEC_OK) rc = ped_pass(pl, 1, launches, msg);
    }
    if (rc != WHMEC_OK) return rc;
    CUDA_TRY(cudaMemcpyAsync(out_vec, pl->d_last_vals, (size_t)T * 4, cudaMemcpyDeviceToHost, pl->stream));
    CUDA_TRY(cudaEventRecord(pl->ev1, pl->stream));
    CUDA_TRY(cudaStreamSynchronize(pl->stream));
    float ms = 0;
    CUDA_TRY(cudaEventElapsedTime(&ms, pl->ev0, pl->ev1));
    pl->stats.sweep_ms += ms;
    pl->stats.kernel_launches += launches;
    pl->swept = true;
    pl->exits_mode = 0;
    return WHMEC_OK;
}

int segment_exits_impl(whmec_plan *pl, int is_last, uint32_t *exits, std::string &msg) {
    int rc = segment_check(pl, msg);
    if (rc != WHMEC_OK) return rc;
    if (!pl->swept) {
        msg = "whmec_segment_exits called before whmec_segment_sweep";
        return WHMEC_ERR_INPUT;
    }
    CUDA_TRY(cudaSetDevice(pl->device));
    rc = pedigree_exits(pl, is_last ? -1 : 0, msg);
    if (rc != WHMEC_OK) return rc;
    const BtArgs a = bt_args(pl, is_last ? -1 : 0);
    bt_entries_kernel<<<(a.T + 31) / 32, 32, 0, pl->stream>>>(a, pl->d_bt_exits.p, nullptr, pl->d_in_vec.p);  // d_in_vec is free again
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(exits, pl->d_in_vec.p, (size_t)a.T * 4, cudaMemcpyDeviceToHost, pl->stream));
    CUDA_TRY(cudaStreamSynchronize(pl->stream));
    return WHMEC_OK;
}

// Backend of solve_in_groups (grouped.h): one plan per group of chains, sweeps enqueued without waiting
struct CudaGroups {
    using Handle = whmec_plan;
    int device;
    whmec_stats total{};
    uint32_t groups = 0;
    int start(const whmec_problem &q, whmec_plan *&h, std::string &msg) {
        h = nullptr;
        std::unique_ptr<whmec_plan> pl(new whmec_plan());
        int rc = plan_create_impl(&q, device, pl.get(), msg);
        if (rc == WHMEC_OK) rc = plan_sweep_impl(pl.get(), msg, false);
        if (rc == WHMEC_OK) h = pl.release();
        return rc;
    }
    int finish(whmec_plan *h, whmec_solution *sub, std::string &msg) {
        const int rc = plan_finish_impl(h, sub, msg);
        if (rc != WHMEC_OK) return rc;
        const whmec_stats &st = h->stats;
        total.cells += st.cells;
        total.algorithmic_bytes += st.algorithmic_bytes;
        total.backptr_bytes += st.backptr_bytes;
        total.state_bytes += st.state_bytes;
        total.kernel_launches += st.kernel_launches;
        total.n_chains += st.n_chains;
        total.max_active = std::max(total.max_active, st.max_active);
        total.transmissions = st.transmissions;
        total.sweep_ms += st.sweep_ms;
        total.h2d_ms += st.h2d_ms;
        total.d2h_ms += st.d2h_ms;
        total.h2d_bytes += st.h2d_bytes;
        total.d2h_bytes += st.d2h_bytes;
        total.path_kind = (groups == 0 || total.path_kind == st.path_kind) ? st.path_kind : 3;
        ++groups;
        return WHMEC_OK;
    }
    void destroy(whmec_plan *h) { delete h; }
};

// Same driver, one group at a time: nothing of group g stays on the device when group g+1 is created.
// Used when a whole problem does not fit the HBM budget but its groups of chains do.
struct SequentialGroups {
    struct Handle {
        const whmec_problem *prob;
    };
    CudaGroups inner{0};
    int start(const whmec_problem &q, Handle *&h, std::string &) {
        h = new Handle{&q};
        return WHMEC_OK;
    }
    int finish(Handle *h, whmec_solution *sub, std::string &msg) {
        whmec_plan *pl = nullptr;
        int rc = inner.start(*h->prob, pl, msg);
        if (rc != WHMEC_OK) return rc;
        rc = inner.finish(pl, sub, msg);
        inner.destroy(pl);
        return rc;
    }
    void destroy(Handle *h) { delete h; }
};

}  // namespace

// No C++ exception may cross the C ABI (a failed host allocation inside the packer or planner would otherwise
// unwind into the caller's C / ctypes frame): entry points that allocate run their body through this.
template <class Body>
int guarded(char *err, size_t errlen, Body body) {
    try {
        return body();
    } catch (const std::bad_alloc &) {
        set_err(err, errlen, "out of host memory");
        return WHMEC_ERR_UNSUPPORTED;
    } catch (const std::exception &e) {
        set_err(err, errlen, std::string("internal error: ") + e.what());
        return WHMEC_ERR_INPUT;
    }
}

extern "C" {

int whmec_abi_version(void) { return WHMEC_ABI_VERSION; }

const char *whmec_build_info(void) { return "whmec: CUDA sm_90a weighted-MEC/PedMEC DP (column + tile kernels), no CPU path"; }

int whmec_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

int whmec_plan_create(const whmec_problem *p, int device, whmec_plan **out, char *err, size_t errlen) {
    return guarded(err, errlen, [&]() -> int {
        std::string msg;
        *out = nullptr;
        std::unique_ptr<whmec_plan> pl(new whmec_plan());  // released (device buffers too) if anything below throws
        const int rc = plan_create_impl(p, device, pl.get(), msg);
        if (rc != WHMEC_OK) {
            set_err(err, errlen, msg);
            return rc;
        }
        *out = pl.release();
        return WHMEC_OK;
    });
}

int whmec_plan_sweep(whmec_plan *plan, char *err, size_t errlen) {
    return guarded(err, errlen, [&]() -> int {
        std::string msg;
        int rc = plan_sweep_impl(plan, msg);
        if (rc != WHMEC_OK) set_err(err, errlen, msg);
        return rc;
    });
}

int whmec_plan_finish(whmec_plan *plan, whmec_solution *s, char *err, size_t errlen) {
    return guarded(err, errlen, [&]() -> int {
        std::string msg;
        int rc = plan_finish_impl(plan, s, msg);
        if (rc != WHMEC_OK) set_err(err, errlen, msg);
        return rc;
    });
}

int whmec_plan_stats(const whmec_plan *plan, whmec_stats *st) {
    *st = plan->stats;
    return WHMEC_OK;
}

void whmec_plan_destroy(whmec_plan *plan) { delete plan; }

int whmec_segment_create(const whmec_problem *p, int device, int continues, whmec_plan **out, char *err, size_t errlen) {
    return guarded(err, errlen, [&]() -> int {
        std::string msg;
        *out = nullptr;
        std::unique_ptr<whmec_plan> pl(new whmec_plan());
        const int rc = plan_create_impl(p, device, pl.get(), msg, continues ? 2 : 1);
        if (rc != WHMEC_OK) {
            set_err(err, errlen, msg);
            return rc;
        }
        *out = pl.release();
        return WHMEC_OK;
    });
}

int whmec_segment_transfer(whmec_plan *plan, uint32_t *matrix, char *err, size_t errlen) {
    return guarded(err, errlen, [&]() -> int {
        std::string msg;
        int rc = segment_transfer_impl(plan, matrix, msg);
        if (rc != WHMEC_OK) set_err(err, errlen, msg);
        return rc;
    });
}

int whmec_segment_sweep(whmec_plan *plan, const uint32_t *in_vec, uint32_t *out_vec, char *err, size_t errlen) {
    return guarded(err, errlen, [&]() -> int {
        std::string msg;
        int rc = segment_sweep_impl(plan, in_vec, out_vec, msg);
        if (rc != WHMEC_OK) set_err(err, errlen, msg);
        return rc;
    });
}

int whmec_segment_exits(whmec_plan *plan, int is_last, uint32_t *exits, char *err, size_t errlen) {
    return guarded(err, errlen, [&]() -> int {
        std::string msg;
        int rc = segment_exits_impl(plan, is_last, exits, msg);
        if (rc != WHMEC_OK) set_err(err, errlen, msg);
        return rc;
    });
}

int whmec_segment_finish(whmec_plan *plan, int entry, whmec_solution *s, char *err, size_t errlen) {
    return guarded(err, errlen, [&]() -> int {
        std::string msg;
        int rc = segment_check(plan, msg);
        if (rc == WHMEC_OK && entry >= (int)plan->pk.T) {
            msg = "entry transmission value out of range";
            rc = WHMEC_ERR_INPUT;
        }
        if (rc == WHMEC_OK) rc = plan_finish_impl(plan, s, msg, entry);
        if (rc != WHMEC_OK) set_err(err, errlen, msg);
        return rc;
    });
}

static int solve_impl(const whmec_problem *p, whmec_solution *s, int device, whmec_stats *st, char *err, size_t errlen) {
    using clk = std::chrono::steady_clock;
    const bool timing = std::getenv("WHMEC_TIMING") != nullptr;
    auto ms = [](clk::time_point a, clk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    const auto t0 = clk::now();
    // WHMEC_SOLVE_GROUPS=G (G >= 2): single-individual problems with many chains are cut into G groups of chains;
    // the host packs / plans / uploads group g+1 while the GPU sweeps group g (grouped.h).  Off by default.
    if (const char *e = std::getenv("WHMEC_SOLVE_GROUPS")) {
        const int G = std::atoi(e);
        if (G >= 2 && G <= 64) {
            keep_host_memory();
            CudaGroups be{device};
            std::string msg;
            bool handled = false;
            solve_in_groups(p, s, (uint32_t)G, be, msg, &handled);
            if (handled) {
                if (st) *st = be.total;
                if (timing) std::fprintf(stderr, "[whmec] solve: %u groups, %.2f ms (device sweeps %.2f ms)\n", be.groups, ms(t0, clk::now()), (double)be.total.sweep_ms);
                return WHMEC_OK;
            }
        }
    }
    whmec_plan *pl = nullptr;
    int rc = whmec_plan_create(p, device, &pl, err, errlen);
    if (rc == WHMEC_ERR_UNSUPPORTED && err && std::strstr(err, "exceeds the free HBM")) {
        // the back-pointers of the whole table do not fit: chains of a single individual are independent problems,
        // solve them group after group (2, 4, ... groups until a group fits)
        for (uint32_t G = 2; G <= 1024; G *= 2) {
            SequentialGroups be;
            be.inner.device = device;
            std::string msg;
            bool handled = false;
            solve_in_groups(p, s, G, be, msg, &handled);
            if (handled) {
                if (st) *st = be.inner.total;
                if (errlen) err[0] = 0;
                return WHMEC_OK;
            }
        }
    }
    if (rc != WHMEC_OK) return rc;
    const auto t1 = clk::now();
    rc = whmec_plan_sweep(pl, err, errlen);
    const auto t2 = clk::now();
    if (rc == WHMEC_OK) rc = whmec_plan_finish(pl, s, err, errlen);
    const auto t3 = clk::now();
    const whmec_stats stats = pl->stats;
    if (st) *st = stats;
    whmec_plan_destroy(pl);
    if (timing)
        std::fprintf(stderr, "[whmec] solve: create %.2f ms (h2d %.2f), sweep %.2f ms (device %.2f), finish %.2f ms (device %.2f), destroy %.2f ms\n",
                     ms(t0, t1), (double)stats.h2d_ms, ms(t1, t2), (double)stats.sweep_ms, ms(t2, t3), (double)stats.d2h_ms, ms(t3, clk::now()));
    return rc;
}

int whmec_solve(const whmec_problem *p, whmec_solution *s, int device, whmec_stats *st, char *err, size_t errlen) {
    return guarded(err, errlen, [&]() -> int { return solve_impl(p, s, device, st, err, errlen); });
}

}  // extern "C"
