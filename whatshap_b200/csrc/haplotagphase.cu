// Votes of `whatshap haplotagphase` on the GPU (whmec_haplotagphase, DESIGN §4.16): the kernels of one chunk and its buffers
// (hp_run_votes, hp_run_runs).  The per-entry lookup, the per-position walk and the choice are haplotagphase.h's, shared with the
// host emulation.  A vote-form chunk is: emit one (position, phase set, x) key per entry with its chunk index (and find the
// first error), radix-sort the keys over their used bits, let one thread per position walk its runs and choose, and sort the
// positions and their (position, phase set) records by first entry.  A runs-form chunk is one thread per position choosing.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cub/cub.cuh>
#include <string>
#include <vector>

#include "haplotagphase_plan.h"
#include "tile.cuh"  // device_available_bytes

namespace whmec {

namespace {

constexpr uint32_t HP_BLOCK = 256;

// one thread per entry: its key and chunk index; an entry error goes to the 64-bit minimum of (ordinal, kind)
__global__ void __launch_bounds__(HP_BLOCK) hp_emit_kernel(const HpEntry *en, uint32_t n, HpTable t, uint64_t p0, uint32_t ps_bits,
                                                           uint64_t *keys, uint32_t *vals, unsigned long long *error) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const HpEntry e = en[i];
    uint32_t x = 0;
    const uint32_t kind = hp_lookup(e, t, p0 + e.pos, x);
    if (kind != HP_OK) atomicMin(error, (unsigned long long)hp_error_code(e.ordinal, kind));
    keys[i] = (uint64_t)e.pos << (ps_bits + 1) | (uint64_t)e.ps << 1 | x;
    vals[i] = i;
}

// one thread per chunk position: the walk of its sorted keys, the choice and the filters; its sort key by first entry
__global__ void __launch_bounds__(HP_BLOCK) hp_walk_kernel(const uint64_t *keys, const uint32_t *vals, const uint32_t *pstart, uint32_t np,
                                                           const HpEntry *en, HpTable t, uint64_t p0, uint32_t ps_bits, uint32_t ib,
                                                           double gap, int only_indels, HpRecord *rec, uint64_t *rkey, uint32_t *rval,
                                                           HpChoice *choice, uint32_t *pkey, uint32_t *pval) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= np) return;
    HpPick k;
    HpChoice ch = hp_walk(keys, vals, pstart[c], pstart[c + 1], en, ps_bits, ib, rec, rkey, rval, k);
    if (ch.voted) hp_finish(k, t, p0 + c, gap, only_indels, ch);
    choice[c] = ch;
    pkey[c] = ch.voted ? ch.first : UINT32_MAX;
    pval[c] = c;
}

// the records in sorted order
__global__ void __launch_bounds__(HP_BLOCK) hp_gather_kernel(const HpRecord *rec, const uint32_t *slot, uint32_t n, HpRecord *out) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n) out[j] = rec[slot[j]];
}

// runs form: one thread per position
__global__ void __launch_bounds__(HP_BLOCK) hp_runs_kernel(const uint64_t *roff, const uint64_t *tpos, uint32_t np, const int64_t *ps,
                                                           const int64_t *h, const int64_t *score, HpTable t, double gap, int only_indels,
                                                           HpChoice *choice) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= np) return;
    HpPick k;
    hp_pick_runs(ps, h, score, roff[c] - roff[0], roff[c + 1] - roff[0], k);
    HpChoice ch{};
    ch.voted = 1;
    hp_finish(k, t, tpos[c], gap, only_indels, ch);
    choice[c] = ch;
}

#define HP_CUDA(expr)                                                 \
    do {                                                              \
        cudaError_t _e = (expr);                                      \
        if (_e != cudaSuccess) {                                      \
            msg = std::string(#expr) + ": " + cudaGetErrorString(_e); \
            return WHMEC_ERR_CUDA;                                    \
        }                                                             \
    } while (0)

// per call: the position tables on the device, a stream, events, the chunk buffers (grown to the largest chunk) and CUB's scratch
struct HpDev {
    cudaStream_t s = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    HpTable t{};
    uint8_t *flags = nullptr;
    uint64_t *a2i_off = nullptr, *i2a_off = nullptr;
    int64_t *a2i_allele = nullptr, *a2i_id = nullptr, *i2a_id = nullptr, *i2a_allele = nullptr;
    uint8_t *arena = nullptr, *temp = nullptr;
    uint64_t arena_bytes = 0, temp_bytes = 0;
    unsigned long long *error = nullptr;
};

uint64_t align_up(uint64_t b) { return (b + 255) / 256 * 256; }

uint32_t bits_for(uint64_t max_value) {
    uint32_t b = 0;
    while (b < 64 && (max_value >> b)) ++b;
    return b;
}

template <class T>
int upload(HpDev &D, HpCall &call, T *&dst, const T *src, uint64_t n, std::string &msg) {
    HP_CUDA(cudaMalloc(&dst, std::max<uint64_t>(n, 1) * sizeof(T)));
    if (n) HP_CUDA(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyHostToDevice, D.s));
    call.st.h2d_bytes += n * sizeof(T);
    return WHMEC_OK;
}

int grow(uint8_t *&p, uint64_t &have, uint64_t need, std::string &msg) {
    if (have >= need) return WHMEC_OK;
    if (p) HP_CUDA(cudaFree(p));
    p = nullptr;
    HP_CUDA(cudaMalloc(&p, need));
    have = need;
    return WHMEC_OK;
}

int open(int device, HpCall &call, std::string &msg) {
    if (!call.dev) call.dev = new HpDev();
    HpDev &D = *(HpDev *)call.dev;
    HP_CUDA(cudaSetDevice(device));
    if (D.s) return WHMEC_OK;
    HP_CUDA(cudaStreamCreateWithFlags(&D.s, cudaStreamNonBlocking));
    HP_CUDA(cudaEventCreate(&D.e0));
    HP_CUDA(cudaEventCreate(&D.e1));
    HP_CUDA(cudaMalloc(&D.error, 8));
    const HpTable &h = call.host;
    const uint64_t np = call.n_pos, na = np ? h.a2i_off[np] : 0, ni = np ? h.i2a_off[np] : 0;
    int rc = WHMEC_OK;
    if ((rc = upload(D, call, D.flags, h.flags, np, msg)) || (rc = upload(D, call, D.a2i_off, h.a2i_off, np ? np + 1 : 0, msg)) ||
        (rc = upload(D, call, D.a2i_allele, h.a2i_allele, na, msg)) || (rc = upload(D, call, D.a2i_id, h.a2i_id, na, msg)) ||
        (rc = upload(D, call, D.i2a_off, h.i2a_off, np ? np + 1 : 0, msg)) || (rc = upload(D, call, D.i2a_id, h.i2a_id, ni, msg)) ||
        (rc = upload(D, call, D.i2a_allele, h.i2a_allele, ni, msg)))
        return rc;
    D.t = HpTable{D.flags, D.a2i_off, D.a2i_allele, D.a2i_id, D.i2a_off, D.i2a_id, D.i2a_allele};
    return WHMEC_OK;
}

}  // namespace

uint64_t hp_budget(int device, std::string &msg) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e == cudaSuccess && (device < 0 || device >= count)) e = cudaErrorInvalidDevice;
    if (e == cudaSuccess) e = cudaSetDevice(device);
    if (e != cudaSuccess) {
        msg = std::string("whmec_haplotagphase: ") + cudaGetErrorString(e);
        return 0;
    }
    const uint64_t free_b = device_available_bytes(), margin = 512ull << 20;
    uint64_t budget = free_b > margin ? free_b - margin : 0;
    // WHMEC_HAPLOTAGPHASE_ARENA_BUDGET=bytes (test hook): the device bytes a call may take
    if (const char *h = std::getenv("WHMEC_HAPLOTAGPHASE_ARENA_BUDGET")) budget = std::min<uint64_t>(budget, std::strtoull(h, nullptr, 10));
    return budget;
}

int hp_run_votes(int device, HpCall &call, std::string &msg) {
    int rc;
    if ((rc = open(device, call, msg))) return rc;
    HpDev &D = *(HpDev *)call.dev;
    const uint32_t ne = call.n_entries, np = call.n_cpos;
    const uint32_t ib = bits_for(ne), pos_bits = bits_for(np - 1);
    // the arena: entries, two key / value buffers for each sort, records and their gathered copy, positions' starts, choices and
    // sort buffers
    const uint64_t b_en = align_up((uint64_t)ne * sizeof(HpEntry)), b_k = align_up((uint64_t)ne * 8), b_v = align_up((uint64_t)ne * 4);
    const uint64_t b_rec = align_up((uint64_t)ne * sizeof(HpRecord)), b_ps = align_up(((uint64_t)np + 1) * 4);
    const uint64_t b_ch = align_up((uint64_t)np * sizeof(HpChoice)), b_p = align_up((uint64_t)np * 4);
    if ((rc = grow(D.arena, D.arena_bytes, b_en + 4 * b_k + 4 * b_v + 2 * b_rec + b_ps + b_ch + 4 * b_p, msg))) return rc;
    uint8_t *a = D.arena;
    auto take = [&](uint64_t b) { uint8_t *p = a; a += b; return p; };
    HpEntry *d_en = (HpEntry *)take(b_en);
    uint64_t *k_a = (uint64_t *)take(b_k), *k_b = (uint64_t *)take(b_k), *rk_a = (uint64_t *)take(b_k), *rk_b = (uint64_t *)take(b_k);
    uint32_t *v_a = (uint32_t *)take(b_v), *v_b = (uint32_t *)take(b_v), *rv_a = (uint32_t *)take(b_v), *rv_b = (uint32_t *)take(b_v);
    HpRecord *d_rec = (HpRecord *)take(b_rec), *d_rec_out = (HpRecord *)take(b_rec);
    uint32_t *d_pstart = (uint32_t *)take(b_ps);
    HpChoice *d_choice = (HpChoice *)take(b_ch);
    uint32_t *pk_a = (uint32_t *)take(b_p), *pk_b = (uint32_t *)take(b_p), *pv_a = (uint32_t *)take(b_p), *pv_b = (uint32_t *)take(b_p);
    HP_CUDA(cudaMemcpyAsync(d_en, call.entries, (uint64_t)ne * sizeof(HpEntry), cudaMemcpyHostToDevice, D.s));
    HP_CUDA(cudaMemcpyAsync(d_pstart, call.pstart.data(), ((uint64_t)np + 1) * 4, cudaMemcpyHostToDevice, D.s));
    call.st.h2d_bytes += (uint64_t)ne * sizeof(HpEntry) + ((uint64_t)np + 1) * 4;
    cub::DoubleBuffer<uint64_t> dk(k_a, k_b), drk(rk_a, rk_b);
    cub::DoubleBuffer<uint32_t> dv(v_a, v_b), drv(rv_a, rv_b), dpk(pk_a, pk_b), dpv(pv_a, pv_b);
    const int key_bits = (int)(pos_bits + call.ps_bits + 1);
    size_t t1 = 0, t2 = 0, t3 = 0;
    HP_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t1, dk, dv, (int)ne, 0, key_bits, D.s));
    HP_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t2, drk, drv, (int)ne, 0, (int)(2 * ib), D.s));
    HP_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t3, dpk, dpv, (int)np, 0, (int)ib, D.s));
    if ((rc = grow(D.temp, D.temp_bytes, std::max<size_t>({t1, t2, t3, (size_t)1}), msg))) return rc;
    HP_CUDA(cudaMemsetAsync(D.error, 0xFF, 8, D.s));
    HP_CUDA(cudaEventRecord(D.e0, D.s));
    hp_emit_kernel<<<(ne + HP_BLOCK - 1) / HP_BLOCK, HP_BLOCK, 0, D.s>>>(d_en, ne, D.t, call.p0, call.ps_bits, k_a, v_a, D.error);
    HP_CUDA(cudaGetLastError());
    size_t tb = D.temp_bytes;
    HP_CUDA(cub::DeviceRadixSort::SortPairs(D.temp, tb, dk, dv, (int)ne, 0, key_bits, D.s));
    hp_walk_kernel<<<(np + HP_BLOCK - 1) / HP_BLOCK, HP_BLOCK, 0, D.s>>>(dk.Current(), dv.Current(), d_pstart, np, d_en, D.t, call.p0,
                                                                         call.ps_bits, ib, call.gap, call.only_indels, d_rec, rk_a, rv_a,
                                                                         d_choice, pk_a, pv_a);
    HP_CUDA(cudaGetLastError());
    tb = D.temp_bytes;
    HP_CUDA(cub::DeviceRadixSort::SortPairs(D.temp, tb, drk, drv, (int)ne, 0, (int)(2 * ib), D.s));
    tb = D.temp_bytes;
    HP_CUDA(cub::DeviceRadixSort::SortPairs(D.temp, tb, dpk, dpv, (int)np, 0, (int)ib, D.s));
    hp_gather_kernel<<<(ne + HP_BLOCK - 1) / HP_BLOCK, HP_BLOCK, 0, D.s>>>(d_rec, drv.Current(), ne, d_rec_out);
    HP_CUDA(cudaGetLastError());
    HP_CUDA(cudaEventRecord(D.e1, D.s));
    call.st.kernel_launches += 6;
    call.choice.resize(np);
    call.order.resize(np);
    unsigned long long err = 0;
    HP_CUDA(cudaMemcpyAsync(call.choice.data(), d_choice, (uint64_t)np * sizeof(HpChoice), cudaMemcpyDeviceToHost, D.s));
    HP_CUDA(cudaMemcpyAsync(call.order.data(), dpv.Current(), (uint64_t)np * 4, cudaMemcpyDeviceToHost, D.s));
    HP_CUDA(cudaMemcpyAsync(&err, D.error, 8, cudaMemcpyDeviceToHost, D.s));
    HP_CUDA(cudaStreamSynchronize(D.s));
    call.st.d2h_bytes += (uint64_t)np * (sizeof(HpChoice) + 4) + 8;
    float ms = 0;
    HP_CUDA(cudaEventElapsedTime(&ms, D.e0, D.e1));
    call.st.device_ms += ms;
    call.error = err;
    uint64_t nr = 0, nv = 0;
    for (const HpChoice &c : call.choice) nr += c.n_ps, nv += c.voted;
    call.order.resize(nv);  // the unvoted positions sort last
    call.records.resize(nr);
    HP_CUDA(cudaMemcpyAsync(call.records.data(), d_rec_out, nr * sizeof(HpRecord), cudaMemcpyDeviceToHost, D.s));
    HP_CUDA(cudaStreamSynchronize(D.s));
    call.st.d2h_bytes += nr * sizeof(HpRecord);
    return WHMEC_OK;
}

int hp_run_runs(int device, HpCall &call, std::string &msg) {
    int rc;
    if ((rc = open(device, call, msg))) return rc;
    HpDev &D = *(HpDev *)call.dev;
    const uint32_t np = call.n_cpos;
    const uint64_t r0 = call.roff[0], nr = call.roff[np] - r0;
    const uint64_t b_off = align_up(((uint64_t)np + 1) * 8), b_r = align_up(nr * 8), b_ch = align_up((uint64_t)np * sizeof(HpChoice));
    if ((rc = grow(D.arena, D.arena_bytes, 2 * b_off + 3 * b_r + b_ch, msg))) return rc;
    uint64_t *d_off = (uint64_t *)D.arena, *d_tpos = (uint64_t *)(D.arena + b_off);
    int64_t *d_ps = (int64_t *)(D.arena + 2 * b_off), *d_h = (int64_t *)(D.arena + 2 * b_off + b_r), *d_sc = (int64_t *)(D.arena + 2 * b_off + 2 * b_r);
    HpChoice *d_choice = (HpChoice *)(D.arena + 2 * b_off + 3 * b_r);
    HP_CUDA(cudaMemcpyAsync(d_off, call.roff.data(), ((uint64_t)np + 1) * 8, cudaMemcpyHostToDevice, D.s));
    HP_CUDA(cudaMemcpyAsync(d_tpos, call.tpos.data(), (uint64_t)np * 8, cudaMemcpyHostToDevice, D.s));
    if (nr) {
        HP_CUDA(cudaMemcpyAsync(d_ps, call.run_ps + r0, nr * 8, cudaMemcpyHostToDevice, D.s));
        HP_CUDA(cudaMemcpyAsync(d_h, call.run_h + r0, nr * 8, cudaMemcpyHostToDevice, D.s));
        HP_CUDA(cudaMemcpyAsync(d_sc, call.run_score + r0, nr * 8, cudaMemcpyHostToDevice, D.s));
    }
    call.st.h2d_bytes += ((uint64_t)np * 2 + 1) * 8 + nr * 24;
    HP_CUDA(cudaEventRecord(D.e0, D.s));
    hp_runs_kernel<<<(np + HP_BLOCK - 1) / HP_BLOCK, HP_BLOCK, 0, D.s>>>(d_off, d_tpos, np, d_ps, d_h, d_sc, D.t, call.gap, call.only_indels,
                                                                         d_choice);
    HP_CUDA(cudaGetLastError());
    HP_CUDA(cudaEventRecord(D.e1, D.s));
    ++call.st.kernel_launches;
    call.choice.resize(np);
    HP_CUDA(cudaMemcpyAsync(call.choice.data(), d_choice, (uint64_t)np * sizeof(HpChoice), cudaMemcpyDeviceToHost, D.s));
    HP_CUDA(cudaStreamSynchronize(D.s));
    call.st.d2h_bytes += (uint64_t)np * sizeof(HpChoice);
    float ms = 0;
    HP_CUDA(cudaEventElapsedTime(&ms, D.e0, D.e1));
    call.st.device_ms += ms;
    return WHMEC_OK;
}

void hp_close(HpCall &call) {
    HpDev *D = (HpDev *)call.dev;
    if (!D) return;
    if (D->s) cudaStreamSynchronize(D->s);
    for (void *p : {(void *)D->flags, (void *)D->a2i_off, (void *)D->a2i_allele, (void *)D->a2i_id, (void *)D->i2a_off, (void *)D->i2a_id,
                    (void *)D->i2a_allele, (void *)D->arena, (void *)D->temp, (void *)D->error})
        cudaFree(p);
    for (cudaEvent_t e : {D->e0, D->e1})
        if (e) cudaEventDestroy(e);
    if (D->s) cudaStreamDestroy(D->s);
    delete D;
    call.dev = nullptr;
}

}  // namespace whmec
