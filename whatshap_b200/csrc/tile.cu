// Tile kernel: single-individual weighted MEC with the projection column held in shared memory.
//
// One CTA owns one tile (2^s entries of the projection column, all bipartitions of the s
// tile-local reads for one fixed assignment of the global reads) and sweeps a whole panel of
// consecutive columns without touching HBM except for the packed back-pointer stream; see
// tile_plan.h for the decomposition and tile_device.h for the per-cell arithmetic.
// Replaces PedigreeDPTable::compute_column (src/pedigreedptable.cpp:177-335) for T == 1.
#include "tile.cuh"

#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <utility>
#include <vector>

#include "../../include/whmec.h"
#include "tile_device.h"
#include "tile_fast.h"
#include "tile_plan.h"

namespace whmec {

namespace {

constexpr int NT = 1024;  // threads per tile
constexpr uint32_t TILE_ENTRIES = 1u << TILE_SMAX;

constexpr uint32_t TC_CHUNK = 16;  // column descriptors staged in shared memory at a time
constexpr uint32_t BULK_MAX_GA = 6;     // bulk-copy hand-off: at most 2^6 chunks ...
constexpr uint32_t BULK_MIN_J = 5;      // ... of at least 2^5 entries (128 bytes)
constexpr uint32_t BULK_SKEW = 4;       // words of skew between consecutive chunks in the staging buffer (keeps 16-byte alignment)
constexpr uint32_t STAGE_PAD_WORDS = BULK_SKEW << BULK_MAX_GA;

// Arrivals at the split column barrier.  1 (default): every thread arrives -- its release covers its own stores, which is also
// what compute-sanitizer's racecheck can follow (0 hazards); 0: one arrival per warp (lane 0 after __syncwarp: correct by
// cumulativity, but racecheck then reports the other lanes' stores as unordered).
#ifndef WHMEC_COL_ARRIVE_ALL
#define WHMEC_COL_ARRIVE_ALL 1
#endif

struct TileSmem {
    uint32_t buf[3][TILE_ENTRIES];  // [0],[1]: ping-pong projection; [2]: staging / prefetch of the next tile's input
    uint32_t stage_pad[STAGE_PAD_WORDS];  // directly behind buf[2]: bulk-copied chunks are laid out with a 16-byte skew each
    unsigned long long stage_bar;   // mbarrier of the bulk copies into the staging buffer
    unsigned long long col_bar;     // column barrier of the steady-state panels (split: arrive, prepare the next column, wait)
    int32_t TL[2][TILE_TL_SIZE];
    int32_t TH[2][TILE_TH_SIZE];
    int32_t TW[2][32];    // fast path, per warp: K2 + E(global bits of the tile) + weights of the warp's output bits
    int32_t T5[2][32];    // fast path, per lane: weights of output bits 0..4
    unsigned long long keys[NT];
    unsigned long long keys2[NT];  // mirrored panels: keys of the mirror outputs (few-output columns)
    TileCol tcs[TC_CHUNK];
    int32_t TWs[TC_CHUNK][32];  // steady-state panels: the tables of every column of the panel, built once
    int32_t T5s[TC_CHUNK][32];
    uint32_t cgs[TC_CHUNK];
    SteadyCol scs[TC_CHUNK];            // steady-state panels: the per-column constants of column_fast, 32 bytes each
    unsigned long long bp_at[TC_CHUNK]; // steady-state panels: first back-pointer word of this tile in column j (bp_off + tile * stride)
    Panel P;
    uint32_t cg[2];
    uint32_t a_col[TC_CHUNK];
    uint32_t panel_index;
};
static_assert(sizeof(TileSmem) <= 227 * 1024, "TileSmem exceeds the shared memory of one CTA on sm_90");

// The steady-state column of a coverage-capped ReadSet: the oldest local read (local bit 0) ends and
// there are enough outputs for every thread.  The planner marks such columns (TileCol::pad0):
//   1  fast:        every thread produces 2^LG outputs
//   2  fast+share:  exactly one read starts in this column: outputs o and o + nout/2 (new read on side
//                   0 / 1) use the same two previous values, so one thread produces both from one load
// TileCol::pad1 = LG.  Output index o = cell index without the dropped bit 0: o bit q <-> local bit q+1.
__device__ __forceinline__ uint32_t fast_kind(const TileCol &tc) { return tc.pad0; }

// Tables of one column: the x-indexed TL/TH pair of tile_device.h (threads 0..384, one entry each) or, for
// fast columns, the two 32-entry tables of column_fast.
__device__ __forceinline__ void build_tables(TileSmem &S, const TileCol &tc, uint32_t tile, uint32_t which, uint32_t tid) {
    if (fast_kind(tc)) {
        if (tid < 32) {
            S.TW[which][tid] = tile_fast_warp_entry(tc, tile, tid);
        } else if (tid < 64) {
            S.T5[which][tid - 32] = tile_fast_lane_entry(tc, tid - 32);
        } else if (tid == 64) {
            S.cg[which] = tile_cg(tc, tile);
        }
        return;
    }
    if (tid < TILE_TL_SIZE) S.TL[which][tid] = tile_tl_entry(tc, tid);
    else if (tid < TILE_TL_SIZE + TILE_TH_SIZE) S.TH[which][tid - TILE_TL_SIZE] = tile_th_entry(tc, tile, tid - TILE_TL_SIZE);
    else if (tid == TILE_TL_SIZE + TILE_TH_SIZE) S.cg[which] = tile_cg(tc, tile);
}

// Steady-state column: exactly one read ends (d == 1), at least one output per thread.
// Per output: two candidate cells that differ in the dropped bit; the reference's visiting order
// makes the candidate whose dropped bit equals the parity of the bits above it the earlier one.
__device__ __forceinline__ void column_drop1(const TileCol &tc, const int32_t *__restrict__ TL, const int32_t *__restrict__ TH,
                                             uint32_t cg, const uint32_t *__restrict__ Sin, uint32_t *__restrict__ Sout,
                                             uint32_t *__restrict__ bpw, uint32_t tid) {
    const uint32_t p = tc.dpos[0];
    const uint32_t lowm = (1u << p) - 1u;
    const uint32_t pbit = 1u << p;
    const uint32_t inmask = low_mask(tc.l_in);
    const uint32_t wp = (uint32_t)tc.w_local[p];
    const uint32_t K0 = tc.K0, K12 = tc.K12, cg0 = cg & 1u;
    const uint32_t nout = 1u << tc.l_out;
    const bool mirror = tc.half && tc.km != 0;
#pragma unroll 4
    for (uint32_t o = tid; o < nout; o += NT) {
        const uint32_t hi = o >> p;
        const uint32_t x0 = ((hi << 1) << p) | (o & lowm);
        const uint32_t u0 = (uint32_t)(TL[x0 & (TILE_TL_SIZE - 1)] + TH[x0 >> TILE_TL_BITS]);
        const uint32_t u1 = u0 + wp;
        const uint32_t c0 = min(K0, min(u0, K12 - u0));
        const uint32_t c1 = min(K0, min(u1, K12 - u1));
        const uint32_t v0 = c0 + Sin[x0 & inmask];
        const uint32_t v1 = c1 + Sin[(x0 | pbit) & inmask];
        const uint32_t par = (__popc(hi) + cg0) & 1u;
        const uint32_t pick1 = par ? (v1 <= v0) : (v1 < v0);
        Sout[o] = min(v0, v1);
        const uint32_t ballot = __ballot_sync(0xFFFFFFFFu, (pick1 ^ par) != 0);
        if ((tid & 31u) == 0) bpw[o >> 5] = ballot;
        if (mirror) {  // the mirror output's winner: same comparison, tie-break parity par ^ km (tile_device.h)
            const uint32_t q = par ^ 1u;
            const uint32_t pickm = q ? (v1 <= v0) : (v1 < v0);
            const uint32_t mballot = __ballot_sync(0xFFFFFFFFu, (pickm ^ q) != 0);
            if ((tid & 31u) == 0) bpw[tc.bp_tile_words + (o >> 5)] = mballot;
        }
    }
}

// Back-pointer words of the fast path leave as warp ballots: all lanes store the same word to the same address (one
// transaction, no divergence).
struct BallotEmit {
    uint32_t *bp;
    uint32_t section;  // words from the tile's own section to its mirror section (mirrored panels, tile_device.h)
    __device__ __forceinline__ void operator()(uint32_t word, bool bit) const { bp[word] = __ballot_sync(0xFFFFFFFFu, bit); }
    __device__ __forceinline__ void mirror(uint32_t word, bool bit) const { bp[section + word] = __ballot_sync(0xFFFFFFFFu, bit); }
    __device__ __forceinline__ void store(uint32_t) const {}
    __device__ __forceinline__ void store_mirror(uint32_t) const {}
};

// Thread-packed layout (TileCol::pad2 == 1, the default): thread `tid` owns element `tid` of BITS bits; a warp's 32
// elements are contiguous (one 32- or 64-byte transaction).
template <int BITS>
struct PackedEmit {
    uint32_t *bpw;  // the tile's slice of the arena
    uint32_t tid;
    uint32_t section;
    __device__ __forceinline__ void operator()(uint32_t, bool) const {}
    __device__ __forceinline__ void mirror(uint32_t, bool) const {}
    __device__ __forceinline__ void store(uint32_t bits) const {
        if (BITS == 8) reinterpret_cast<uint8_t *>(bpw)[tid] = (uint8_t)bits;
        else reinterpret_cast<uint16_t *>(bpw)[tid] = (uint16_t)bits;
    }
    __device__ __forceinline__ void store_mirror(uint32_t bits) const {
        if (BITS == 8) reinterpret_cast<uint8_t *>(bpw + section)[tid] = (uint8_t)bits;
        else reinterpret_cast<uint16_t *>(bpw + section)[tid] = (uint16_t)bits;
    }
};

// Column in which no read ends (coverage still growing): one cell per output, no back-pointer.
__device__ __forceinline__ void column_drop0(const TileCol &tc, const int32_t *__restrict__ TL, const int32_t *__restrict__ TH,
                                             const uint32_t *__restrict__ Sin, uint32_t *__restrict__ Sout, uint32_t tid) {
    const uint32_t inmask = low_mask(tc.l_in);
    const uint32_t K0 = tc.K0, K12 = tc.K12;
    const uint32_t nout = 1u << tc.l_out;
#pragma unroll 4
    for (uint32_t o = tid; o < nout; o += NT) {
        const uint32_t u = (uint32_t)(TL[o & (TILE_TL_SIZE - 1)] + TH[o >> TILE_TL_BITS]);
        Sout[o] = min(K0, min(u, K12 - u)) + Sin[o & inmask];
    }
}

#define CUDA_TRY(expr)                                                    \
    do {                                                                  \
        cudaError_t _e = (expr);                                          \
        if (_e != cudaSuccess) {                                          \
            msg = std::string(#expr) + ": " + cudaGetErrorString(_e);     \
            return WHMEC_ERR_CUDA;                                        \
        }                                                                 \
    } while (0)

__device__ __forceinline__ void bp_store_warp_tile(uint32_t *words, uint32_t width, uint32_t e, uint32_t value, bool valid) {
    if (width == 0) return;
    const uint32_t per = 32u / width;
    const uint32_t lane = threadIdx.x & 31u;
    const uint32_t sub = lane % per;
    uint32_t word = valid ? (value << (sub * width)) : 0u;
    for (uint32_t off = 1; off < per; off <<= 1) word |= __shfl_xor_sync(0xFFFFFFFFu, word, off);
    if (sub == 0 && valid) words[e / per] = word;
}

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long key) {
    for (int off = 16; off > 0; off >>= 1) {
        unsigned long long other = __shfl_xor_sync(0xFFFFFFFFu, key, off);
        key = other < key ? other : key;
    }
    return key;
}

// pdep of an index whose low 10 bits are the thread id: split so that only the high part is
// recomputed per iteration.
__device__ __forceinline__ uint32_t mask_without_low_bits(uint32_t mask, uint32_t nbits) {
    for (uint32_t i = 0; i < nbits && mask; ++i) mask &= mask - 1;
    return mask;
}

// Staging index of element (producer tile tA, offset ll) of a tile-major hand-off: a bijection of
// [0, 2^s_in) chosen so that 32 consecutive (tA, ll) in either order hit 32 different banks.
__device__ __forceinline__ uint32_t stage_index(uint32_t gA, uint32_t jb, uint32_t tA, uint32_t ll) {
    if (gA == 0) return ll;
    if (jb >= 5) return (tA << jb) + (ll ^ ((tA << (gA <= 5 ? 5 - gA : 0)) & 31u));
    const uint32_t idx = (tA << jb) + ll;
    return idx ^ ((idx >> 5) & ((1u << jb) - 1u));
}

__device__ __forceinline__ void cp_async4(uint32_t *smem_dst, const uint32_t *gsrc) {
    const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// ---- bulk asynchronous copies (TMA engine, cp.async.bulk) completing on an mbarrier
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void *dst, const void *src, uint32_t bytes, unsigned long long *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(src),
                 "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile("{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
                     : "=r"(done)
                     : "r"(smem_u32(bar)), "r"(parity)
                     : "memory");
    } while (!done);
}

__device__ __forceinline__ void mbar_arrive(unsigned long long *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// Steady-state panel (see tile_panel_kernel): `ncol` fast twin columns of one tile size, tables already in shared memory.
// One barrier per column, split: a warp ARRIVES when its outputs of column j are stored, computes everything of column j + 1
// that does not read the projection (addresses, constants, the subset sums of its outputs: column_fast_prep), and only then
// WAITS for the other warps -- the block's drift at the barrier is filled with work instead of idle issue slots.
// The barrier is an mbarrier (arrive = release, try_wait = acquire at CTA scope) with one arrival per thread (or per warp, see
// WHMEC_COL_ARRIVE_ALL).  Every thread of the block runs the same number of iterations.
template <int LG, bool MR>
__device__ __forceinline__ void steady_columns(TileSmem &S, uint32_t ncol, uint32_t *__restrict__ arena, uint32_t &cur, uint32_t &col_phase,
                                               uint32_t tid) {
    constexpr int BITS = 2 << LG;  // outputs (= back-pointer bits) per thread and column: 2^LG twins
    constexpr uint32_t IT = 1u << LG;
    // constants of the panel (l_in, l_out are those of its first column)
    const uint32_t lane = tid & 31u, warp = tid >> 5;
    const uint32_t obase = warp * (IT * 32u) + lane;
    const uint32_t pair_off = obase & ((1u << (S.tcs[0].l_in - 1)) - 1u);
    const uint32_t half = 1u << (S.tcs[0].l_out - 1);
    const uint32_t pop = popc32(obase);
    const uint32_t section = S.tcs[0].bp_tile_words;
    FastPrep<LG> pr;
    steady_prep<LG>(pr, S.scs[0], S.TWs[0][warp], S.T5s[0][lane], S.buf[cur], S.buf[cur ^ 1], obase, pair_off, half, pop);
    uint32_t *bpw = arena + S.bp_at[0];
    for (uint32_t j = 0; j < ncol; ++j) {
        column_fast_body<LG, false, true, true, MR>(pr, PackedEmit<BITS>{bpw, tid, section});
#if WHMEC_COL_ARRIVE_ALL
        mbar_arrive(&S.col_bar);  // every thread releases its own stores
#else
        __syncwarp();
        if (lane == 0) mbar_arrive(&S.col_bar);
#endif
        cur ^= 1;
        if (j + 1 < ncol) {
            steady_prep<LG>(pr, S.scs[j + 1], S.TWs[j + 1][warp], S.T5s[j + 1][lane], S.buf[cur], S.buf[cur ^ 1], obase, pair_off, half, pop);
            bpw = arena + S.bp_at[j + 1];
        }
        mbar_wait(&S.col_bar, col_phase);
        col_phase ^= 1u;
    }
}

// Tile-major hand-offs whose chunks are at least 128 bytes travel as one bulk copy per producer tile.
__device__ __forceinline__ bool bulk_handoff(uint32_t gA, uint32_t jb) { return gA <= BULK_MAX_GA && jb >= BULK_MIN_J; }

// Bulk version of stage_tile_async (called by warp 0 only): chunk tA lands at stage + tA * (2^j + BULK_SKEW), in the
// producer's order -- ascending for a computed producer tile, for an uncomputed one (mirrored producer) the chunk of the
// mirror tile, which holds the wanted entries in DESCENDING order (the reader flips the offset).
__device__ __forceinline__ void stage_tile_bulk(uint32_t *stage, unsigned long long *bar, const Panel *pp, uint32_t ptile, const uint32_t *state) {
    const uint32_t gA = __ldg(&pp->in_gA), jb = __ldg(&pp->in_j), sA = __ldg(&pp->in_sA);
    const uint32_t told = ptile & low_mask(__ldg(&pp->in_gold));
    const uint32_t top = __ldg(&pp->in_half) ? (1u << (gA - 1)) : 0u;
    const uint32_t amask = (1u << gA) - 1u, tmask = (1u << (sA - jb)) - 1u;
    const uint32_t *base = state + __ldg(&pp->in_off);
    const uint32_t lane = threadIdx.x & 31u, bytes = 4u << jb;
    if (lane == 0) mbar_expect_tx(bar, bytes << gA);
    __syncwarp();
    for (uint32_t tA = lane; tA <= amask; tA += 32) {
        const uint32_t *from = (tA & top) ? base + ((uint64_t)(~tA & amask) << sA) + ((uint64_t)(~told & tmask) << jb)
                                          : base + ((uint64_t)tA << sA) + ((uint64_t)told << jb);
        bulk_copy_g2s(stage + tA * ((1u << jb) + BULK_SKEW), from, bytes, bar);
    }
}

// Asynchronous gather of one tile's input (tile-major hand-off) into the staging buffer: one contiguous
// 2^j chunk from each of the 2^gA producer tiles.  `pp` points to the panel in global memory.
__device__ __forceinline__ void stage_tile_async(uint32_t *stage, const Panel *pp, uint32_t ptile, const uint32_t *state) {
    const uint32_t gA = __ldg(&pp->in_gA), jb = __ldg(&pp->in_j), sA = __ldg(&pp->in_sA);
    const uint32_t nin = 1u << __ldg(&pp->s_in);
    const uint32_t told = ptile & low_mask(__ldg(&pp->in_gold));
    const uint32_t *src = state + __ldg(&pp->in_off) + ((uint64_t)told << jb);
    const uint32_t jmask = (1u << jb) - 1u;
    // mirrored producer (Panel::half): its tiles with top tile-id bit 1 were not computed; their entries are the
    // complemented index of the mirror tile (descending inside the chunk)
    const uint32_t top = __ldg(&pp->in_half) ? (1u << (gA - 1)) : 0u;
    const uint32_t amask = (1u << gA) - 1u, smask = (1u << sA) - 1u;
    const uint32_t *base = state + __ldg(&pp->in_off);
    const uint32_t chunk0 = told << jb;
    for (uint32_t e = threadIdx.x; e < nin; e += NT) {
        const uint32_t tA = e >> jb, ll = e & jmask;
        const uint32_t *from = (tA & top) ? base + ((uint64_t)(~tA & amask) << sA) + (~(chunk0 + ll) & smask)
                                          : src + ((uint64_t)tA << sA) + ll;
        cp_async4(&stage[stage_index(gA, jb, tA, ll)], from);
    }
    cp_async_commit();
}

__global__ void __launch_bounds__(NT, 1)
tile_panel_kernel(const Panel *__restrict__ panels, uint32_t n_panels, uint32_t total_tiles, int32_t tile_log, const TileCol *__restrict__ tcols,
                  const ColMeta *__restrict__ cols, uint32_t *__restrict__ state, uint32_t *__restrict__ arena,
                  unsigned long long *__restrict__ chain_keys) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    TileSmem &S = *reinterpret_cast<TileSmem *>(smem_raw);
    const uint32_t tid = threadIdx.x;

    // Persistent CTAs: each walks the launch's tiles with stride gridDim.x and, while it sweeps one
    // tile's panel, the input of its next tile is already streaming into the third buffer (cp.async).
    uint32_t pi = 0;            // panel of the current work item; panels[] is sorted by tile_begin
    uint32_t staged = 0;        // the staging buffer holds (or is receiving) the current tile's input: 1 = cp.async, 2 = bulk copies
    uint32_t bar_phase = 0;     // parity of the staging mbarrier's current phase
    uint32_t col_phase = 0;     // parity of the column barrier's current phase
    if (tid == 0) {
        mbar_init(&S.stage_bar, 1);
        mbar_init(&S.col_bar, WHMEC_COL_ARRIVE_ALL ? NT : NT / 32);
    }
    __syncthreads();
    for (uint32_t work = blockIdx.x; work < total_tiles; work += gridDim.x) {
    if (tile_log >= 0) pi = work >> tile_log;  // every panel of this launch has 2^tile_log tiles
    else while (pi + 1 < n_panels && __ldg(&panels[pi + 1].tile_begin) <= work) ++pi;
    __syncthreads();  // previous work item completely done (its stores read the buffers, S.P is reused)
    if (tid < sizeof(Panel) / 4) ((uint32_t *)&S.P)[tid] = ((const uint32_t *)&panels[pi])[tid];
    __syncthreads();
    const Panel &P = S.P;
    const uint32_t tile = work - P.tile_begin;
    uint32_t cur = 0;

    // ---- the tile's slice of the incoming projection column
    if (P.fresh) {
        if (tid == 0) S.buf[0][0] = 0;
    } else if (P.in_layout == 1 && bulk_handoff(P.in_gA, P.in_j)) {
        // tile-major hand-off, one bulk copy per producer tile (issued by warp 0, normally already while the previous tile
        // was swept); every thread waits on the mbarrier, then the chunks are transposed into the canonical local order
        //   index = (chunk offset << gA) | producer tile.
        if (!staged && tid < 32) stage_tile_bulk(S.buf[2], &S.stage_bar, &panels[pi], tile, state);
        mbar_wait(&S.stage_bar, bar_phase);
        bar_phase ^= 1u;
        const uint32_t gA = P.in_gA, jb = P.in_j, nin = 1u << P.s_in;
        const uint32_t cs = (1u << jb) + BULK_SKEW, jmask = (1u << jb) - 1u;
        const uint32_t top = P.in_half ? (1u << (gA - 1)) : 0u;  // chunks of uncomputed producer tiles arrive reversed
        const uint32_t *stage = S.buf[2];
        if (gA >= 5) {
            // a warp moves 32 producer tiles x 4 offsets per step; lane L takes offset (L / 8 + r) % 4 in rotation r, so that
            // the 32 reads (chunk stride = 4 banks) and the 32 writes (consecutive words) of a rotation hit 32 different banks
            const uint32_t lane = tid & 31u, warp = tid >> 5;
            for (uint32_t blk = warp; blk < (nin >> 7); blk += NT / 32) {
                const uint32_t tA = ((blk & ((1u << (gA - 5)) - 1u)) << 5) + lane;
                const uint32_t ll0 = (blk >> (gA - 5)) << 2;
                const uint32_t *row = stage + tA * cs;
#pragma unroll
                for (uint32_t r = 0; r < 4; ++r) {
                    const uint32_t ll = ll0 + (((lane >> 3) + r) & 3u);
                    S.buf[0][(ll << gA) | tA] = row[(tA & top) ? (jmask - ll) : ll];
                }
            }
        } else {
            const uint32_t amask = (1u << gA) - 1u;
            for (uint32_t i = tid; i < nin; i += NT) {
                const uint32_t tA = i & amask, ll = i >> gA;
                S.buf[0][i] = stage[tA * cs + ((tA & top) ? (jmask - ll) : ll)];
            }
        }
    } else if (P.in_layout == 1) {
        // tile-major hand-off with small chunks: gathered element by element into the staging buffer (XOR-swizzled so that
        // both passes are bank-conflict free), then transposed into the canonical local order
        if (!staged) stage_tile_async(S.buf[2], &panels[pi], tile, state);
        cp_async_wait_all();
        __syncthreads();
        const uint32_t gA = P.in_gA, jb = P.in_j, nin = 1u << P.s_in;
        const uint32_t amask = (1u << gA) - 1u;
        for (uint32_t i = tid; i < nin; i += NT) S.buf[0][i] = S.buf[2][stage_index(gA, jb, i & amask, i >> gA)];
    } else {
        const uint32_t nin = 1u << P.s_in;
        const uint32_t gpart = pdep32(tile, P.gmask_in);
        const uint32_t lo = pdep32(tid, P.lmask_in);
        const uint32_t himask = mask_without_low_bits(P.lmask_in, 10);
        const uint32_t *src = state + P.in_off;
        const uint32_t top = P.in_half ? P.in_top : 0u, fmask_in = P.lmask_in | P.gmask_in;
        for (uint32_t l = tid, it = 0; l < nin; l += NT, ++it) {
            uint32_t e = lo | pdep32(it, himask) | gpart;
            if (e & top) e = ~e & fmask_in;  // entry of an uncomputed tile of a mirrored producer
            S.buf[0][l] = src[e];
        }
    }
    __syncthreads();  // staging buffer free again
    // ---- prefetch the input of this CTA's next tile
    staged = 0;
    {
        const uint32_t nwork = work + gridDim.x;
        if (nwork < total_tiles) {
            uint32_t pn = pi;
            if (tile_log >= 0) pn = nwork >> tile_log;
            else while (pn + 1 < n_panels && __ldg(&panels[pn + 1].tile_begin) <= nwork) ++pn;
            if (__ldg(&panels[pn].in_layout) == 1 && !__ldg(&panels[pn].fresh)) {
                const uint32_t ntile = nwork - __ldg(&panels[pn].tile_begin);
                if (bulk_handoff(__ldg(&panels[pn].in_gA), __ldg(&panels[pn].in_j))) {
                    if (tid < 32) {
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic reads of the buffer above -> async writes
                        stage_tile_bulk(S.buf[2], &S.stage_bar, &panels[pn], ntile, state);
                    }
                    staged = 2;
                } else {
                    stage_tile_async(S.buf[2], &panels[pn], ntile, state);
                    staged = 1;
                }
            }
        }
    }

    if (P.steady) {
        // ---- steady-state panel: every column is the twin fast column of one tile size.  Descriptors and ALL tables of
        // the panel are built once, in parallel (thread (column, entry)); then one barrier and one call per column.
        const uint32_t kb = P.col_begin, ncol = P.col_end - kb;
        {
            constexpr uint32_t WORDS = sizeof(TileCol) / 4;
            for (uint32_t w = tid; w < ncol * WORDS; w += NT) ((uint32_t *)S.tcs)[w] = ((const uint32_t *)(tcols + kb))[w];
        }
        __syncthreads();
        {
            const uint32_t j = tid >> 6, idx = tid & 63u;
            if (j < ncol) {
                if (idx < 32) S.TWs[j][idx] = tile_fast_warp_entry(S.tcs[j], tile, idx);
                else S.T5s[j][idx - 32] = tile_fast_lane_entry(S.tcs[j], idx - 32);
                if (idx == 63) {
                    const uint32_t cg = tile_cg(S.tcs[j], tile);
                    S.cgs[j] = cg;
                    S.scs[j] = steady_col(S.tcs[j], cg);
                    S.bp_at[j] = S.tcs[j].bp_off + (uint64_t)tile * S.tcs[j].bp_tile_stride;
                }
            }
        }
        const bool mirror = S.tcs[0].half && S.tcs[0].km != 0;
        const uint32_t lg = P.steady - 1u;
        __syncthreads();  // tables ready; the tile's input is in place
        if (lg == 3) {
            if (mirror) steady_columns<3, true>(S, ncol, arena, cur, col_phase, tid);
            else steady_columns<3, false>(S, ncol, arena, cur, col_phase, tid);
        } else {
            if (mirror) steady_columns<2, true>(S, ncol, arena, cur, col_phase, tid);
            else steady_columns<2, false>(S, ncol, arena, cur, col_phase, tid);
        }
    } else
    for (uint32_t k = P.col_begin; k < P.col_end; ++k) {
        const uint32_t j = (k - P.col_begin) % TC_CHUNK;
        if (j == 0) {
            // stage the next TC_CHUNK column descriptors (previous chunk is no longer referenced)
            __syncthreads();
            const uint32_t ncol = min(TC_CHUNK, P.col_end - k);
            constexpr uint32_t WORDS = sizeof(TileCol) / 4;
            for (uint32_t w = tid; w < ncol * WORDS; w += NT)
                ((uint32_t *)S.tcs)[w] = ((const uint32_t *)(tcols + k))[w];
            if (tid < ncol) S.a_col[tid] = cols[k + tid].a;
            __syncthreads();
            build_tables(S, S.tcs[0], tile, k & 1u, tid);
        }
        __syncthreads();  // tables of column k ready; previous column's outputs complete
        // tables of column k+1 are produced while column k is evaluated (double buffered)
        if (j + 1 < TC_CHUNK && k + 1 < P.col_end) build_tables(S, S.tcs[j + 1], tile, (k + 1) & 1u, tid);
        const TileCol &tc = S.tcs[j];
        const uint32_t tb = k & 1u;
        TileCtx c{&tc, tile, S.TL[tb], S.TH[tb], S.cg[tb], S.buf[cur]};
        uint32_t *Sout = S.buf[cur ^ 1];
        const uint32_t m = tc.l_in + tc.n_new;

        if (tc.kind == 1) {
            // chain end: every read ends here -> one global minimum per chain, ordered by the
            // reference's Gray-code visiting rank of the canonical index
            const uint32_t ncell = 1u << m;
            const uint32_t gpart = pdep32(tile, ~tc.lmask_col & low_mask(S.a_col[j]));
            const uint32_t per = ncell >= NT ? ncell / NT : 1;
            unsigned long long key = KEY_INF;
            if (tid * per < ncell) key = tile_eval_end(c, gpart, tid * per, tid * per + per);
            key = warp_min_u64(key);
            if ((tid & 31) == 0) S.keys[tid >> 5] = key;
            __syncthreads();
            if (tid < 32) {
                key = warp_min_u64(S.keys[tid]);
                if (tid == 0) atomicMin(&chain_keys[P.chain], key);
            }
        } else {
            const uint32_t nout = 1u << tc.l_out;
            const uint32_t ncand = 1u << tc.d;
            uint32_t *bpw = arena + tc.bp_off + (uint64_t)tile * tc.bp_tile_stride;
            const bool mirror = tc.half && tc.km != 0;  // the mirror outputs' back-pointers differ: second section
            if (fast_kind(tc)) {
#define WHMEC_FAST_ARGS tc, S.TW[tb], S.T5[tb], S.cg[tb], S.buf[cur], Sout
#define WHMEC_FAST(LGV, SH)                                                                                      \
    {                                                                                                            \
        const BallotEmit em{bpw + (tid >> 5) * (1u << LGV), tc.bp_tile_words};                                   \
        if (mirror) {                                                                                            \
            if (tc.K0 >= TILE_KINF) column_fast<LGV, false, SH, false, true>(WHMEC_FAST_ARGS, em, tid);           \
            else column_fast<LGV, true, SH, false, true>(WHMEC_FAST_ARGS, em, tid);                               \
        } else if (tc.K0 >= TILE_KINF) column_fast<LGV, false, SH>(WHMEC_FAST_ARGS, em, tid);                     \
        else column_fast<LGV, true, SH>(WHMEC_FAST_ARGS, em, tid);                                                \
    }
#define WHMEC_FAST_PACKED(LGV, SH, BITS)                                                                          \
    {                                                                                                            \
        const PackedEmit<BITS> em{bpw, tid, tc.bp_tile_words};                                                   \
        if (mirror) {                                                                                            \
            if (tc.K0 >= TILE_KINF) column_fast<LGV, false, SH, true, true>(WHMEC_FAST_ARGS, em, tid);            \
            else column_fast<LGV, true, SH, true, true>(WHMEC_FAST_ARGS, em, tid);                                \
        } else if (tc.K0 >= TILE_KINF) column_fast<LGV, false, SH, true>(WHMEC_FAST_ARGS, em, tid);               \
        else column_fast<LGV, true, SH, true>(WHMEC_FAST_ARGS, em, tid);                                          \
    }
                if (tc.pad2 & 1u) {  // thread-packed back-pointer bits (planner: 8 or 16 outputs per thread only)
                    if (fast_kind(tc) == 2) {
                        if (tc.pad1 == 2) { WHMEC_FAST_PACKED(2, true, 8) } else { WHMEC_FAST_PACKED(3, true, 16) }
                    } else {
                        if (tc.pad1 == 3) { WHMEC_FAST_PACKED(3, false, 8) } else { WHMEC_FAST_PACKED(4, false, 16) }
                    }
                } else if (fast_kind(tc) == 2) {
                    switch (tc.pad1) {
                        case 0: WHMEC_FAST(0, true) break;
                        case 1: WHMEC_FAST(1, true) break;
                        case 2: WHMEC_FAST(2, true) break;
                        default: WHMEC_FAST(3, true) break;
                    }
                } else {
                    switch (tc.pad1) {
                        case 0: WHMEC_FAST(0, false) break;
                        case 1: WHMEC_FAST(1, false) break;
                        case 2: WHMEC_FAST(2, false) break;
                        case 3: WHMEC_FAST(3, false) break;
                        default: WHMEC_FAST(4, false) break;
                    }
                }
#undef WHMEC_FAST_PACKED
#undef WHMEC_FAST
#undef WHMEC_FAST_ARGS
            } else if (nout >= NT && tc.d == 1) {
                column_drop1(tc, S.TL[tb], S.TH[tb], S.cg[tb], S.buf[cur], Sout, bpw, tid);
            } else if (nout >= NT && tc.d == 0) {
                column_drop0(tc, S.TL[tb], S.TH[tb], S.buf[cur], Sout, tid);
            } else if (nout >= NT) {
                for (uint32_t o = tid; o < nout; o += NT) {
                    uint64_t mkey;
                    const unsigned long long key = tile_eval(c, o, 0, ncand, &mkey);
                    Sout[o] = (uint32_t)(key >> 32);
                    bp_store_warp_tile(bpw, tc.bp_width, o, (uint32_t)key, true);
                    if (mirror) bp_store_warp_tile(bpw + tc.bp_tile_words, tc.bp_width, o, (uint32_t)mkey, true);
                }
            } else {
                // few outputs: split every output's candidates over several threads
                const uint32_t spare = 10u - tc.l_out;
                const uint32_t log_chunks = spare < tc.d ? spare : tc.d;
                const uint32_t items = nout << log_chunks;
                if (tid < nout) S.keys[tid] = S.keys2[tid] = KEY_INF;
                __syncthreads();
                unsigned long long key = KEY_INF, mkey = KEY_INF;
                const uint32_t o = tid >> log_chunks;
                if (tid < items) {
                    const uint32_t ch = tid & ((1u << log_chunks) - 1);
                    const uint32_t per = ncand >> log_chunks;
                    uint64_t mk;
                    key = tile_eval(c, o, ch * per, (ch + 1) * per, &mk);
                    mkey = mk;
                }
                if (log_chunks >= 5) {
                    key = warp_min_u64(key);
                    if (mirror) mkey = warp_min_u64(mkey);
                    if ((tid & 31) == 0 && tid < items) {
                        atomicMin(&S.keys[o], key);
                        if (mirror) atomicMin(&S.keys2[o], mkey);
                    }
                } else if (tid < items) {
                    atomicMin(&S.keys[o], key);
                    if (mirror) atomicMin(&S.keys2[o], mkey);
                }
                __syncthreads();
                key = tid < nout ? S.keys[tid] : 0ull;
                if (tid < nout) Sout[tid] = (uint32_t)(key >> 32);
                bp_store_warp_tile(bpw, tc.bp_width, tid, (uint32_t)key, tid < nout);
                if (mirror) bp_store_warp_tile(bpw + tc.bp_tile_words, tc.bp_width, tid, tid < nout ? (uint32_t)S.keys2[tid] : 0u, tid < nout);
            }
            cur ^= 1;
        }
    }

    // ---- write the tile back in canonical layout for the next panel
    if (!P.ends_chain && P.out_layout == 1) {
        __syncthreads();
        const uint32_t nout = 1u << P.s_out;
        uint32_t *dst = state + P.out_off + ((uint64_t)tile << P.s_out);
        if (P.s_out >= 2) {
            const uint4 *b4 = reinterpret_cast<const uint4 *>(S.buf[cur]);
            uint4 *d4 = reinterpret_cast<uint4 *>(dst);
            for (uint32_t v = tid; v < (nout >> 2); v += NT) d4[v] = b4[v];
        } else {
            if (tid < nout) dst[tid] = S.buf[cur][tid];
        }
    } else if (!P.ends_chain) {
        __syncthreads();
        const uint32_t nout = 1u << P.s_out;
        const uint32_t gpart = pdep32(tile, P.gmask_out);
        const uint32_t lo = pdep32(tid, P.lmask_out);
        const uint32_t himask = mask_without_low_bits(P.lmask_out, 10);
        uint32_t *dst = state + P.out_off;
        for (uint32_t l = tid, it = 0; l < nout; l += NT, ++it) dst[lo | pdep32(it, himask) | gpart] = S.buf[cur][l];
    }
    }  // work loop
}

// Backtrace: one warp per DP-independent chain.  The walk itself is sequential (the cell of column k - 1 is read through the
// cell of column k), but the per-column records it needs (ColMeta + TileCol, ~360 bytes) are not: the lanes stage them 16
// columns at a time into shared memory, lane 0 then walks those 16 columns paying only for the dependent back-pointer loads.
// seg_lo / seg_hi: the chain's columns whose back-pointers are resident (the whole chain, or its part inside the segment of
// a memory-bounded sweep; the walk then continues from path_index[hi + 1], written by the segment before).
constexpr uint32_t BT_CHUNK = 16;

__global__ void __launch_bounds__(32) tile_backtrace_kernel(const ColMeta *__restrict__ cols, const TileCol *__restrict__ tcols,
                                                            const uint32_t *__restrict__ arena, const uint32_t *__restrict__ chain_begin,
                                                            const uint32_t *__restrict__ seg_lo, const uint32_t *__restrict__ seg_hi,
                                                            uint32_t n_chains, const unsigned long long *__restrict__ chain_keys,
                                                            uint32_t *__restrict__ path_index, uint32_t *__restrict__ result) {
    __shared__ ColMeta s_cols[BT_CHUNK + 1];  // columns lo .. lo + n (the extra one supplies cols[k].bw of the chunk's top step)
    __shared__ TileCol s_tcols[BT_CHUNK];
    __shared__ uint32_t s_path[BT_CHUNK];
    const uint32_t c = blockIdx.x, lane = threadIdx.x;
    if (c >= n_chains) return;
    const uint32_t k_first = seg_lo[c], k_res = seg_hi[c];
    if (k_first > k_res) return;  // no column of this chain in the segment
    const uint32_t chain_last = chain_begin[c + 1] - 1;
    uint32_t x, k_last;
    if (k_res == chain_last) {
        const unsigned long long key = chain_keys[c];
        const uint32_t r = (uint32_t)key;
        x = r ^ (r >> 1);  // Gray code of the winning rank = canonical index in the last column
        k_last = k_res;
        if (lane == 0) {
            path_index[k_last] = x;
            atomicAdd(&result[0], (uint32_t)(key >> 32));  // cost = sum over DP-independent chains
        }
    } else {
        x = path_index[k_res + 1];  // the walk arrives from the columns of the following segment
        k_last = k_res + 1;
    }
    for (uint32_t hi = k_last; hi > k_first;) {  // steps hi -> hi - 1, ..., lo + 1 -> lo
        const uint32_t lo = hi - k_first > BT_CHUNK ? hi - BT_CHUNK : k_first, n = hi - lo;
        constexpr uint32_t CW = sizeof(ColMeta) / 4, TW = sizeof(TileCol) / 4;
        for (uint32_t w = lane; w < (n + 1) * CW; w += 32) ((uint32_t *)s_cols)[w] = ((const uint32_t *)(cols + lo))[w];
        for (uint32_t w = lane; w < n * TW; w += 32) ((uint32_t *)s_tcols)[w] = ((const uint32_t *)(tcols + lo))[w];
        __syncwarp();
        // The walk is a chain of dependent loads (one back-pointer per column, ~1 us each from HBM).  Runs of columns with 1-bit
        // back-pointers (the steady state) are walked SPECULATIVELY, up to 5 columns per memory round trip: lane l stands for
        // the node (level L, hypothesis h) of the binary tree of possible paths, l + 1 = 2^L + h; it applies the L assumed
        // back-pointer bits of h to x (index arithmetic only) and loads the back-pointer its node would read; the true path is
        // then picked out of the 2^D - 1 loaded bits with D shuffles.  Other columns take the ordinary step (all lanes alike).
        for (uint32_t k = hi; k > lo;) {
            uint32_t D = 0;
            while (D < 5 && k - D > lo && s_tcols[k - 1 - D - lo].bp_width == 1) ++D;
            if (D >= 2) {
                const uint32_t L = 31u - (uint32_t)__clz((int)(lane + 1)), h = lane + 1 - (1u << L);
                uint32_t xl = x, b = 0;
                if (L < D) {
                    for (uint32_t i = 0; i < L; ++i)
                        xl = candidate_index(s_cols[k - 1 - i - lo], xl & low_mask(s_cols[k - i - lo].bw), (h >> i) & 1u);
                    b = tile_backtrace_bp(s_cols[k - L - lo].bw, s_cols[k - 1 - L - lo], s_tcols[k - 1 - L - lo], arena, xl);
                }
                uint32_t hh = 0, xi = x, bi = 0;
                for (uint32_t i = 0; i < D; ++i) {  // level i of the true path: column k - i, whose cell is xi
                    const uint32_t src = (1u << i) - 1u + hh;
                    xi = __shfl_sync(0xFFFFFFFFu, xl, src);
                    bi = __shfl_sync(0xFFFFFFFFu, b, src);
                    if (i > 0 && lane == 0) s_path[k - i - lo] = xi;
                    hh |= bi << i;
                }
                x = candidate_index(s_cols[k - D - lo], xi & low_mask(s_cols[k - D + 1 - lo].bw), bi);
                if (lane == 0) s_path[k - D - lo] = x;
                k -= D;
            } else {
                x = tile_backtrace_step(s_cols[k - lo].bw, s_cols[k - 1 - lo], s_tcols[k - 1 - lo], arena, x);
                if (lane == 0) s_path[k - 1 - lo] = x;
                --k;
            }
        }
        __syncwarp();
        if (lane < n) path_index[lo + lane] = s_path[lane];
        __syncwarp();
        hi = lo;
    }
}

struct TileSeg {
    uint32_t r0, r1;       // rounds [r0, r1)
    uint64_t words;        // back-pointer words of the segment
};

struct TileImpl {
    TileSchedule ts;
    std::vector<TileSeg> segs;          // one segment: everything resident (the usual case)
    uint32_t *d_ckpt = nullptr;         // projection state before segments 1 .. K-1 (state_words each)
    uint32_t *d_seg_lo = nullptr, *d_seg_hi = nullptr;  // [segment][chain]: columns of the chain inside the segment (lo > hi: none)
    std::vector<uint32_t> seg_lo, seg_hi;  // their host copies (kept: the upload is asynchronous)
    uint64_t arena_words = 0;
    const ColMeta *d_cols = nullptr;  // owned by the plan that owns this schedule (uploaded before the planner ran)
    TileCol *d_tcols = nullptr;
    Panel *d_panels = nullptr;
    uint32_t *d_state = nullptr, *d_arena = nullptr, *d_chain_begin = nullptr;
    unsigned long long *d_chain_keys = nullptr;
    uint32_t n_chains = 0;
    uint32_t n_sm = 132;
};

}  // namespace

size_t device_available_bytes() {
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) return 0;
    int dev = 0;
    cudaMemPool_t pool;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
        uint64_t reserved = 0, used = 0;
        if (cudaMemPoolGetAttribute(pool, cudaMemPoolAttrReservedMemCurrent, &reserved) == cudaSuccess &&
            cudaMemPoolGetAttribute(pool, cudaMemPoolAttrUsedMemCurrent, &used) == cudaSuccess && reserved > used)
            free_b += (size_t)(reserved - used);
    }
    return free_b;
}

bool TilePlan::plan(const Packed &pk) {
    TileImpl *I = new TileImpl();
    plan_tiles(pk, I->ts);
    if (!I->ts.eligible) {
        why = I->ts.why;
        delete I;
        return false;
    }
    impl = I;
    backptr_bytes = I->ts.bp_words * 4;
    state_bytes = I->ts.state_traffic_bytes;
    return true;
}

int TilePlan::create(const Packed &pk, cudaStream_t stream, uint64_t &h2d, std::string &msg, const ColMeta *d_cols) {
    TileImpl *I = (TileImpl *)impl;
    TileSchedule &ts = I->ts;
    I->n_chains = (uint32_t)pk.chain_begin.size() - 1;
    const size_t free_b = device_available_bytes();
    const uint64_t fixed = (ts.state_words + 2) * 4 + (uint64_t)pk.n * (sizeof(TileCol) + sizeof(ColMeta)) + ts.panels.size() * sizeof(Panel) +
                           (512ull << 20);
    // Memory-bounded sweep.  The reference bounds its memory by keeping every sqrt(n)-th column and recomputing
    // (pedigreedptable.cpp:103-134,146-173).  Here the 1-bit back-pointers of ALL columns normally stay resident; when they do
    // not fit (coverage 25 beyond ~90k columns, coverage 26+), the launch rounds are cut into segments whose back-pointers share
    // one arena: the forward sweep keeps the projection state in front of every segment (a checkpoint) and the back-pointers of
    // the last segment; the backtrace walks the last segment, then re-sweeps the one before from its checkpoint, and so on.
    // The last segment is made as large as fits, so the re-swept fraction is small.  WHMEC_TILE_ARENA_BUDGET (bytes): test hook.
    uint64_t budget = free_b > fixed ? free_b - fixed : 0;
    uint64_t arena_override = 0;  // test hook: bytes the ARENA may take (checkpoints are not counted against it)
    if (const char *e = std::getenv("WHMEC_TILE_ARENA_BUDGET")) arena_override = std::max<uint64_t>(8, std::strtoull(e, nullptr, 10));
    const size_t n_rounds = ts.round_tiles.size();
    I->segs.clear();
    const uint64_t resident_limit = arena_override ? std::min(arena_override, budget) : budget;
    if ((ts.bp_words + 1) * 4 <= resident_limit || n_rounds <= 1) {
        if ((ts.bp_words + 1) * 4 > resident_limit) {
            msg = "tile path: state + back-pointer storage exceeds the free HBM of this device";
            return WHMEC_ERR_UNSUPPORTED;
        }
        I->segs.push_back(TileSeg{0, (uint32_t)n_rounds, ts.bp_words});
        I->arena_words = ts.bp_words;
    } else {
        std::vector<uint64_t> round_words(n_rounds, 0);
        for (size_t r = 0; r < n_rounds; ++r)
            for (uint32_t q = ts.round_begin[r]; q < ts.round_begin[r + 1]; ++q) {
                const Panel &P = ts.panels[q];
                for (uint32_t k = P.col_begin; k < P.col_end; ++k)
                    round_words[r] += (uint64_t)ts.cols[k].bp_tile_stride << (ts.cols[k].g - ts.cols[k].half);
            }
        bool ok = false;
        for (uint32_t guess = 2; guess <= n_rounds && !ok; ++guess) {  // `guess` segments -> guess - 1 checkpoints
            const uint64_t ckpt = (uint64_t)(guess - 1) * ts.state_words * 4;
            if (ckpt + 4096 >= budget) break;
            const uint64_t cap = (arena_override ? std::min(arena_override, budget - ckpt) : budget - ckpt) / 4 - 1;  // arena words
            std::vector<TileSeg> segs;
            size_t r1 = n_rounds;
            bool fits = true;
            while (r1 > 0) {  // greedy from the end: the segment that is swept only once is the largest
                uint64_t words = 0;
                size_t r0 = r1;
                while (r0 > 0 && words + round_words[r0 - 1] <= cap) words += round_words[--r0];
                if (r0 == r1) {
                    fits = false;
                    break;
                }
                segs.push_back(TileSeg{(uint32_t)r0, (uint32_t)r1, words});
                r1 = r0;
            }
            if (fits && segs.size() <= guess) {
                std::reverse(segs.begin(), segs.end());
                I->segs = segs;
                ok = true;
            }
        }
        if (!ok) {
            msg = "tile path: state + back-pointer storage exceeds the free HBM of this device";
            return WHMEC_ERR_UNSUPPORTED;
        }
        // segment-local back-pointer offsets: the columns of a segment are laid out round by round, panel by panel
        I->arena_words = 0;
        for (const TileSeg &sg : I->segs) {
            uint64_t at = 0;
            for (uint32_t r = sg.r0; r < sg.r1; ++r)
                for (uint32_t q = ts.round_begin[r]; q < ts.round_begin[r + 1]; ++q) {
                    const Panel &P = ts.panels[q];
                    for (uint32_t k = P.col_begin; k < P.col_end; ++k) {
                        ts.cols[k].bp_off = at;
                        at += (uint64_t)ts.cols[k].bp_tile_stride << (ts.cols[k].g - ts.cols[k].half);
                    }
                }
            I->arena_words = std::max(I->arena_words, at);
        }
        backptr_bytes = I->arena_words * 4;
    }
    // columns of every chain inside every segment
    const size_t K = I->segs.size();
    std::vector<uint32_t> &seg_lo = I->seg_lo, &seg_hi = I->seg_hi;
    seg_lo.assign(K * I->n_chains, 1);
    seg_hi.assign(K * I->n_chains, 0);
    for (size_t sgi = 0; sgi < K; ++sgi)
        for (uint32_t r = I->segs[sgi].r0; r < I->segs[sgi].r1; ++r)
            for (uint32_t q = ts.round_begin[r]; q < ts.round_begin[r + 1]; ++q) {
                const Panel &P = ts.panels[q];
                uint32_t &lo = seg_lo[sgi * I->n_chains + P.chain], &hi = seg_hi[sgi * I->n_chains + P.chain];
                if (lo > hi) {
                    lo = P.col_begin;
                    hi = P.col_end - 1;
                } else {
                    lo = std::min(lo, P.col_begin);
                    hi = std::max(hi, P.col_end - 1);
                }
            }
    using cclk = std::chrono::steady_clock;
    const bool timing = std::getenv("WHMEC_TIMING") != nullptr;
    const auto tq0 = cclk::now();
    CUDA_TRY(cudaMallocAsync((void **)&I->d_seg_lo, seg_lo.size() * 4, stream));
    CUDA_TRY(cudaMallocAsync((void **)&I->d_seg_hi, seg_hi.size() * 4, stream));
    CUDA_TRY(cudaMemcpyAsync(I->d_seg_lo, seg_lo.data(), seg_lo.size() * 4, cudaMemcpyHostToDevice, stream));
    CUDA_TRY(cudaMemcpyAsync(I->d_seg_hi, seg_hi.data(), seg_hi.size() * 4, cudaMemcpyHostToDevice, stream));
    if (K > 1) CUDA_TRY(cudaMallocAsync((void **)&I->d_ckpt, (uint64_t)(K - 1) * (ts.state_words + 1) * 4, stream));
    I->d_cols = d_cols;
    CUDA_TRY(cudaMallocAsync((void **)&I->d_tcols, (size_t)pk.n * sizeof(TileCol), stream));
    CUDA_TRY(cudaMallocAsync((void **)&I->d_panels, ts.panels.size() * sizeof(Panel), stream));
    CUDA_TRY(cudaMallocAsync((void **)&I->d_state, (ts.state_words + 1) * 4, stream));
    CUDA_TRY(cudaMallocAsync((void **)&I->d_arena, (I->arena_words + 1) * 4, stream));
    CUDA_TRY(cudaMallocAsync((void **)&I->d_chain_begin, pk.chain_begin.size() * 4, stream));
    CUDA_TRY(cudaMallocAsync((void **)&I->d_chain_keys, (size_t)I->n_chains * 8, stream));
    const auto tq1 = cclk::now();
    auto up = [&](void *dst, const void *src, size_t bytes) {
        h2d += bytes;
        return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream);
    };
    struct Piece {
        void *dst;
        const void *src;
        size_t bytes, off;
    };
    Piece pieces[3] = {{I->d_tcols, ts.cols.data(), (size_t)pk.n * sizeof(TileCol), 0},
                       {I->d_panels, ts.panels.data(), ts.panels.size() * sizeof(Panel), 0},
                       {I->d_chain_begin, pk.chain_begin.data(), pk.chain_begin.size() * 4, 0}};
    size_t total = 0;
    for (Piece &q : pieces) {
        q.off = total;
        total += (q.bytes + 255) & ~(size_t)255;
    }
    // the records sit in page-locked memory when the library's staging pool is installed (hostpool.h: StagedVec): each array
    // is then ONE asynchronous DMA transfer that the sweep's first launch queues behind; from pageable memory (pool off or
    // exhausted) the same calls go through the driver's bounce buffer
    for (const Piece &q : pieces) CUDA_TRY(up(q.dst, q.src, q.bytes));
    {
        int dev = 0, sms = 132;
        CUDA_TRY(cudaGetDevice(&dev));
        CUDA_TRY(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        I->n_sm = (uint32_t)sms;
    }
    CUDA_TRY(cudaFuncSetAttribute(tile_panel_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TileSmem)));
    if (timing) {
        auto qms = [](cclk::time_point a, cclk::time_point b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
        std::fprintf(stderr, "[whmec] tiles.create: segments + seg tables + %.1f MB of allocations %.2f ms, upload calls (%.1f MB) %.2f ms\n",
                     (double)((I->arena_words + ts.state_words) * 4) / 1e6, qms(tq0, tq1), (double)total / 1e6, qms(tq1, cclk::now()));
    }
    return WHMEC_OK;
}

namespace {
// the launch rounds [r0, r1) of a schedule
void launch_rounds(TileImpl *I, uint32_t r0, uint32_t r1, cudaStream_t stream, uint32_t &launches) {
    const TileSchedule &ts = I->ts;
    for (uint32_t r = r0; r < r1; ++r) {
        const uint32_t p0 = ts.round_begin[r], p1 = ts.round_begin[r + 1];
        const uint32_t grid = std::min<uint32_t>(ts.round_tiles[r], I->n_sm);
        tile_panel_kernel<<<grid, NT, sizeof(TileSmem), stream>>>(I->d_panels + p0, p1 - p0, ts.round_tiles[r], ts.round_tile_log[r], I->d_tcols, I->d_cols,
                                                                                I->d_state, I->d_arena, I->d_chain_keys);
        ++launches;
    }
}
}  // namespace

int TilePlan::sweep(const Packed &pk, cudaStream_t stream, std::string &msg) {
    TileImpl *I = (TileImpl *)impl;
    const TileSchedule &ts = I->ts;
    CUDA_TRY(cudaMemsetAsync(I->d_chain_keys, 0xFF, (size_t)I->n_chains * 8, stream));
    launches = 0;
    for (size_t sgi = 0; sgi < I->segs.size(); ++sgi) {
        if (sgi > 0)  // checkpoint: the projection state in front of segment sgi
            CUDA_TRY(cudaMemcpyAsync(I->d_ckpt + (sgi - 1) * (ts.state_words + 1), I->d_state, (ts.state_words + 1) * 4, cudaMemcpyDeviceToDevice, stream));
        launch_rounds(I, I->segs[sgi].r0, I->segs[sgi].r1, stream, launches);
    }
    CUDA_TRY(cudaGetLastError());
    return WHMEC_OK;
}

int TilePlan::backtrace(const Packed &pk, cudaStream_t stream, uint32_t *d_path_index, uint32_t *d_result, std::string &msg) {
    TileImpl *I = (TileImpl *)impl;
    const TileSchedule &ts = I->ts;
    CUDA_TRY(cudaMemsetAsync(d_result, 0, 16, stream));
    for (size_t sgi = I->segs.size(); sgi-- > 0;) {
        if (sgi + 1 < I->segs.size()) {  // its back-pointers were overwritten by the later segments: sweep it again from its checkpoint
            if (sgi > 0)
                CUDA_TRY(cudaMemcpyAsync(I->d_state, I->d_ckpt + (sgi - 1) * (ts.state_words + 1), (ts.state_words + 1) * 4, cudaMemcpyDeviceToDevice, stream));
            uint32_t again = 0;
            launch_rounds(I, I->segs[sgi].r0, I->segs[sgi].r1, stream, again);
            launches += again;
        }
        tile_backtrace_kernel<<<I->n_chains, 32, 0, stream>>>(I->d_cols, I->d_tcols, I->d_arena, I->d_chain_begin, I->d_seg_lo + sgi * I->n_chains,
                                                              I->d_seg_hi + sgi * I->n_chains, I->n_chains, I->d_chain_keys, d_path_index, d_result);
    }
    CUDA_TRY(cudaGetLastError());
    return WHMEC_OK;
}

void TilePlan::release(cudaStream_t stream) {
    TileImpl *I = (TileImpl *)impl;
    if (!I) return;
    for (void *q : {(void *)I->d_tcols, (void *)I->d_panels, (void *)I->d_state, (void *)I->d_arena,
                    (void *)I->d_chain_begin, (void *)I->d_chain_keys, (void *)I->d_ckpt, (void *)I->d_seg_lo, (void *)I->d_seg_hi})
        if (q) cudaFreeAsync(q, stream);
    delete I;
    impl = nullptr;
}

}  // namespace whmec
