// Read assignment of `whatshap haplotag` on the GPU (whmec_haplotag, DESIGN §4.15): the kernels of one chunk and its buffers
// (ht_run_chunk).  The per-entry visit and the per-group choice are haplotag.h's, shared with the host emulation.  A chunk is:
// count each entry's matches (and find the first error), scan the counts, emit one (group, block, haplotype) key per match with
// the entry's ordinal, radix-sort the keys over their used bits, and let one thread per group choose from its sorted keys.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cub/cub.cuh>
#include <string>
#include <vector>

#include "haplotag_plan.h"
#include "tile.cuh"  // device_available_bytes

namespace whmec {

namespace {

constexpr uint32_t HT_BLOCK = 256;

// one thread per entry: its match count and, on a visit error, the error's code
__global__ void __launch_bounds__(HT_BLOCK) ht_count_kernel(const HtEntry *en, uint32_t n, HtTable t, int64_t ploidy, uint64_t e0,
                                                            uint32_t *counts, unsigned long long *error) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t c = 0;
    const uint32_t kind = ht_visit(en[i], t, ploidy, [&](uint32_t, uint32_t) { ++c; });
    counts[i] = c;
    if (kind != HT_OK) atomicMin(error, (unsigned long long)ht_error_code(2 * (e0 + i), kind));
}

// one thread per entry: its keys from koff[i] on, each with the entry's ordinal
__global__ void __launch_bounds__(HT_BLOCK) ht_emit_kernel(const HtEntry *en, uint32_t n, HtTable t, int64_t ploidy, const uint32_t *koff,
                                                           uint32_t hap_bits, uint32_t rank_bits, uint64_t *keys, uint32_t *ords) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const HtEntry e = en[i];
    const uint64_t g = (uint64_t)e.group << (hap_bits + rank_bits);
    uint32_t k = koff[i];
    ht_visit(e, t, ploidy, [&](uint32_t rank, uint32_t h) {
        keys[k] = g | (uint64_t)rank << hap_bits | h;
        ords[k] = i;
        ++k;
    });
}

// one thread per group: the choice from its sorted keys, which occupy the same range as its emitted keys
__global__ void __launch_bounds__(HT_BLOCK) ht_choose_kernel(const uint64_t *keys, const uint32_t *ords, const uint32_t *koff, const uint32_t *gstart,
                                                             uint32_t ng, const HtEntry *en, int64_t ploidy, uint32_t hap_bits,
                                                             uint32_t rank_bits, uint64_t e0, HtChoice *choice, unsigned long long *error) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= ng) return;
    const HtChoice c = ht_choose(keys, ords, koff[gstart[g]], koff[gstart[g + 1]], en, ploidy, hap_bits, rank_bits);
    choice[g] = c;
    if (c.n_blocks && ploidy < 2) atomicMin(error, (unsigned long long)ht_error_code(2 * (e0 + gstart[g + 1]) - 1, HT_INDEX));
}

#define HT_CUDA(expr)                                                 \
    do {                                                              \
        cudaError_t _e = (expr);                                      \
        if (_e != cudaSuccess) {                                      \
            msg = std::string(#expr) + ": " + cudaGetErrorString(_e); \
            return WHMEC_ERR_CUDA;                                    \
        }                                                             \
    } while (0)

// per call: the phase tables on the device, a stream, events, the chunk buffers (grown to the largest chunk) and CUB's scratch
struct HtDev {
    cudaStream_t s = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr, e2 = nullptr, e3 = nullptr;  // around the counting half and the keys' half of a chunk
    HtTable t{};
    uint64_t *soff = nullptr, *aoff = nullptr;
    int64_t *pos = nullptr;
    uint32_t *rank = nullptr;
    int32_t *allele = nullptr;
    uint8_t *arena = nullptr, *keys = nullptr, *temp = nullptr;
    uint64_t arena_bytes = 0, keys_bytes = 0, temp_bytes = 0;
    unsigned long long *error = nullptr;
};

uint64_t align_up(uint64_t b) { return (b + 255) / 256 * 256; }

template <class T>
int upload(HtDev &D, HtCall &call, T *&dst, const T *src, uint64_t n, std::string &msg) {
    HT_CUDA(cudaMalloc(&dst, std::max<uint64_t>(n, 1) * sizeof(T)));
    if (n) HT_CUDA(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyHostToDevice, D.s));
    call.st.h2d_bytes += n * sizeof(T);
    return WHMEC_OK;
}

int grow(uint8_t *&p, uint64_t &have, uint64_t need, std::string &msg) {
    if (have >= need) return WHMEC_OK;
    if (p) HT_CUDA(cudaFree(p));
    p = nullptr;
    HT_CUDA(cudaMalloc(&p, need));
    have = need;
    return WHMEC_OK;
}

int run(HtCall &call, HtDev &D, std::string &msg) {
    const uint32_t ne = (uint32_t)call.entries.size(), ng = (uint32_t)call.gstart.size() - 1;
    const uint64_t b_en = align_up((uint64_t)ne * sizeof(HtEntry)), b_cnt = align_up(((uint64_t)ne + 1) * 4), b_gs = align_up(((uint64_t)ng + 1) * 4);
    int rc;
    if ((rc = grow(D.arena, D.arena_bytes, b_en + 2 * b_cnt + b_gs + align_up((uint64_t)ng * sizeof(HtChoice)), msg))) return rc;
    HtEntry *d_en = (HtEntry *)D.arena;
    uint32_t *d_cnt = (uint32_t *)(D.arena + b_en), *d_koff = (uint32_t *)(D.arena + b_en + b_cnt);
    uint32_t *d_gs = (uint32_t *)(D.arena + b_en + 2 * b_cnt);
    HtChoice *d_choice = (HtChoice *)(D.arena + b_en + 2 * b_cnt + b_gs);
    HT_CUDA(cudaMemcpyAsync(d_en, call.entries.data(), (uint64_t)ne * sizeof(HtEntry), cudaMemcpyHostToDevice, D.s));
    HT_CUDA(cudaMemcpyAsync(d_gs, call.gstart.data(), ((uint64_t)ng + 1) * 4, cudaMemcpyHostToDevice, D.s));
    call.st.h2d_bytes += (uint64_t)ne * sizeof(HtEntry) + ((uint64_t)ng + 1) * 4;
    size_t t_scan = 0;
    HT_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t_scan, d_cnt, d_koff, (int)ne + 1, D.s));
    if ((rc = grow(D.temp, D.temp_bytes, std::max<size_t>(t_scan, 1), msg))) return rc;
    HT_CUDA(cudaMemsetAsync(D.error, 0xFF, 8, D.s));
    HT_CUDA(cudaMemsetAsync(d_cnt + ne, 0, 4, D.s));
    HT_CUDA(cudaEventRecord(D.e0, D.s));
    if (ne) {
        ht_count_kernel<<<(ne + HT_BLOCK - 1) / HT_BLOCK, HT_BLOCK, 0, D.s>>>(d_en, ne, D.t, call.ploidy, call.e0, d_cnt, D.error);
        HT_CUDA(cudaGetLastError());
        ++call.st.kernel_launches;
    }
    size_t tb = D.temp_bytes;
    HT_CUDA(cub::DeviceScan::ExclusiveSum(D.temp, tb, d_cnt, d_koff, (int)ne + 1, D.s));
    ++call.st.kernel_launches;
    HT_CUDA(cudaEventRecord(D.e1, D.s));
    uint32_t nk = 0;
    unsigned long long err = 0;
    HT_CUDA(cudaMemcpyAsync(&nk, d_koff + ne, 4, cudaMemcpyDeviceToHost, D.s));
    HT_CUDA(cudaMemcpyAsync(&err, D.error, 8, cudaMemcpyDeviceToHost, D.s));
    HT_CUDA(cudaStreamSynchronize(D.s));
    call.st.d2h_bytes += 12;
    float ms = 0;
    HT_CUDA(cudaEventElapsedTime(&ms, D.e0, D.e1));
    call.st.device_ms += ms;
    call.error = err;
    // an entry error ends the call; only with ploidy < 2 can an earlier group's choice fail before it
    if (err != ~0ull && call.ploidy >= 2) return WHMEC_OK;
    call.st.keys += nk;
    const uint64_t b_keys = align_up((uint64_t)nk * 8), b_ords = align_up((uint64_t)nk * 4);
    if ((rc = grow(D.keys, D.keys_bytes, 2 * b_keys + 2 * b_ords, msg))) return rc;
    uint64_t *k_a = (uint64_t *)D.keys, *k_b = (uint64_t *)(D.keys + b_keys);
    uint32_t *o_a = (uint32_t *)(D.keys + 2 * b_keys), *o_b = (uint32_t *)(D.keys + 2 * b_keys + b_ords);
    const uint32_t end_bit = call.hap_bits + call.rank_bits + std::max<uint32_t>(1, 32 - __builtin_clz(std::max<uint32_t>(ng - 1, 1)));
    cub::DoubleBuffer<uint64_t> dk(k_a, k_b);
    cub::DoubleBuffer<uint32_t> dv(o_a, o_b);
    size_t t_sort = 0;
    HT_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t_sort, dk, dv, (int)nk, 0, (int)end_bit, D.s));
    if ((rc = grow(D.temp, D.temp_bytes, std::max<size_t>(t_sort, 1), msg))) return rc;
    HT_CUDA(cudaEventRecord(D.e2, D.s));
    if (nk) {
        ht_emit_kernel<<<(ne + HT_BLOCK - 1) / HT_BLOCK, HT_BLOCK, 0, D.s>>>(d_en, ne, D.t, call.ploidy, d_koff, call.hap_bits, call.rank_bits,
                                                                             k_a, o_a);
        HT_CUDA(cudaGetLastError());
        tb = D.temp_bytes;
        HT_CUDA(cub::DeviceRadixSort::SortPairs(D.temp, tb, dk, dv, (int)nk, 0, (int)end_bit, D.s));
        call.st.kernel_launches += 2;
    }
    ht_choose_kernel<<<(ng + HT_BLOCK - 1) / HT_BLOCK, HT_BLOCK, 0, D.s>>>(dk.Current(), dv.Current(), d_koff, d_gs, ng, d_en, call.ploidy,
                                                                           call.hap_bits, call.rank_bits, call.e0, d_choice, D.error);
    HT_CUDA(cudaGetLastError());
    ++call.st.kernel_launches;
    HT_CUDA(cudaEventRecord(D.e3, D.s));
    call.choice.resize(ng);
    HT_CUDA(cudaMemcpyAsync(call.choice.data(), d_choice, (uint64_t)ng * sizeof(HtChoice), cudaMemcpyDeviceToHost, D.s));
    HT_CUDA(cudaMemcpyAsync(&err, D.error, 8, cudaMemcpyDeviceToHost, D.s));
    HT_CUDA(cudaStreamSynchronize(D.s));
    call.st.d2h_bytes += (uint64_t)ng * sizeof(HtChoice) + 8;
    HT_CUDA(cudaEventElapsedTime(&ms, D.e2, D.e3));
    call.st.device_ms += ms;
    call.error = err;
    for (const HtChoice &c : call.choice) call.st.runs += c.runs;
    return WHMEC_OK;
}

}  // namespace

uint64_t ht_budget(int device, std::string &msg) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e == cudaSuccess && (device < 0 || device >= count)) e = cudaErrorInvalidDevice;
    if (e == cudaSuccess) e = cudaSetDevice(device);
    if (e != cudaSuccess) {
        msg = std::string("whmec_haplotag: ") + cudaGetErrorString(e);
        return 0;
    }
    const uint64_t free_b = device_available_bytes(), margin = 512ull << 20;
    uint64_t budget = free_b > margin ? free_b - margin : 0;
    // WHMEC_HAPLOTAG_ARENA_BUDGET=bytes (test hook): the device bytes a call may take
    if (const char *h = std::getenv("WHMEC_HAPLOTAG_ARENA_BUDGET")) budget = std::min<uint64_t>(budget, std::strtoull(h, nullptr, 10));
    return budget;
}

int ht_run_chunk(int device, HtCall &call, std::string &msg) {
    if (!call.dev) call.dev = new HtDev();
    HtDev &D = *(HtDev *)call.dev;
    HT_CUDA(cudaSetDevice(device));
    if (!D.s) {
        HT_CUDA(cudaStreamCreateWithFlags(&D.s, cudaStreamNonBlocking));
        HT_CUDA(cudaEventCreate(&D.e0));
        HT_CUDA(cudaEventCreate(&D.e1));
        HT_CUDA(cudaEventCreate(&D.e2));
        HT_CUDA(cudaEventCreate(&D.e3));
        HT_CUDA(cudaMalloc(&D.error, 8));
        int rc = WHMEC_OK;
        if ((rc = upload(D, call, D.soff, call.host.soff, (uint64_t)call.n_samples + 1, msg)) ||
            (rc = upload(D, call, D.pos, call.host.pos, call.n_pos, msg)) || (rc = upload(D, call, D.rank, call.rank.data(), call.n_pos, msg)) ||
            (rc = upload(D, call, D.aoff, call.host.aoff, call.n_pos ? call.n_pos + 1 : 0, msg)) ||
            (rc = upload(D, call, D.allele, call.host.allele, call.n_alleles, msg)))
            return rc;
        D.t = HtTable{D.soff, D.pos, D.rank, D.aoff, D.allele};
    }
    return run(call, D, msg);
}

void ht_close(HtCall &call) {
    HtDev *D = (HtDev *)call.dev;
    if (!D) return;
    if (D->s) cudaStreamSynchronize(D->s);
    for (void *p : {(void *)D->soff, (void *)D->aoff, (void *)D->pos, (void *)D->rank, (void *)D->allele, (void *)D->arena, (void *)D->keys,
                    (void *)D->temp, (void *)D->error})
        cudaFree(p);
    for (cudaEvent_t e : {D->e0, D->e1, D->e2, D->e3})
        if (e) cudaEventDestroy(e);
    if (D->s) cudaStreamDestroy(D->s);
    delete D;
    call.dev = nullptr;
}

}  // namespace whmec
