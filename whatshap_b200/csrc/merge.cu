// Read merging of `whatshap phase --merge-reads` on the GPU (whmec_merge_reads, DESIGN §4.17): a set's resident arrays and the
// kernels of its chunks.  Per set: pack the alleles as bits (one thread per word) and start every read as its own root; per pair
// chunk, one thread per pair counts the mismatches of its overlap and sets its flags, hooking blue edges into the parent array
// or writing the flags back for the host's removal loop; the roots are found by pointer jumping.  Per accumulation chunk: one
// (component, position) key per entry, a stable radix sort over the used bits, run heads, a scan, and one thread per run for z0
// and z1.  The per-thread code is merge.h's, shared with the host emulation.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cub/cub.cuh>
#include <string>

#include "merge_plan.h"
#include "tile.cuh"  // device_available_bytes

namespace whmec {

namespace {

constexpr uint32_t MG_BLOCK = 256;

__global__ void __launch_bounds__(MG_BLOCK) mg_pack_kernel(const uint64_t *woff, const uint64_t *roff, const uint8_t *allele,
                                                           uint32_t n_reads, uint64_t n_words, uint64_t *words) {
    const uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (w < n_words) words[w] = mg_pack_word(w, woff, roff, allele, n_reads);
    if (w == n_words) words[w] = 0;  // the padding word
}

__global__ void __launch_bounds__(MG_BLOCK) mg_init_kernel(uint32_t *parent, uint32_t n) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x < n) parent[x] = x;
}

// one thread per pair of [p0, p0 + n): its flags and m - mm (hook = 0), or the hook of a blue edge (hook = 1)
__global__ void __launch_bounds__(MG_BLOCK) mg_pair_kernel(uint64_t p0, uint32_t n, const uint64_t *pstart, uint32_t n_reads,
                                                           const int64_t *begin, const uint64_t *roff, const uint64_t *woff,
                                                           const uint64_t *words, int64_t thr_diff, int64_t thr_neg_diff, double max_e,
                                                           int hook, uint32_t *parent, uint8_t *flag, int64_t *diff,
                                                           unsigned long long *blue) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n) return;
    uint32_t j, i;
    mg_pair(p0 + t, pstart, n_reads, j, i);
    int64_t d;
    const uint8_t f = mg_eval(j, i, begin, roff, woff, words, thr_diff, thr_neg_diff, max_e, d);
    if (!hook) {
        flag[t] = f, diff[t] = d;
    } else if (f & MG_BLUE) {
        mg_hook(parent, j, i);
        atomicAdd(blue, 1ull);
    }
}

__global__ void __launch_bounds__(MG_BLOCK) mg_compress_kernel(uint32_t *parent, uint32_t n) {
    const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x < n) parent[x] = mg_find(parent, x);
}

__global__ void __launch_bounds__(MG_BLOCK) mg_key_kernel(const MgEntry *en, uint32_t n, int32_t pmin, uint32_t pos_bits, uint64_t *keys,
                                                          uint32_t *vals) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    keys[k] = mg_key(en[k], pmin, pos_bits);
    vals[k] = k;
}

__global__ void __launch_bounds__(MG_BLOCK) mg_head_kernel(const uint64_t *keys, uint32_t n, uint32_t *head) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) head[k] = k == 0 || keys[k] != keys[k - 1];
}

__global__ void __launch_bounds__(MG_BLOCK) mg_start_kernel(const uint32_t *head, const uint32_t *rank, uint32_t n, uint32_t *start) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n && head[k]) start[rank[k]] = k;
    if (k == n - 1) start[rank[k] + head[k]] = n;
}

__global__ void __launch_bounds__(MG_BLOCK) mg_sum_kernel(const MgEntry *en, const uint32_t *order, const uint32_t *start, uint32_t n_runs,
                                                          MgRun *runs) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r < n_runs) runs[r] = mg_sum_run(en, order, start[r], start[r + 1]);
}

#define MG_CUDA(expr)                                                 \
    do {                                                              \
        cudaError_t _e = (expr);                                      \
        if (_e != cudaSuccess) {                                      \
            msg = std::string(#expr) + ": " + cudaGetErrorString(_e); \
            return WHMEC_ERR_CUDA;                                    \
        }                                                             \
    } while (0)

// per call: a stream, events, a counter, the resident set (freed at the next set), the chunk arena and CUB's scratch
struct MgDev {
    cudaStream_t s = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    unsigned long long *blue = nullptr;
    uint8_t *set = nullptr, *arena = nullptr, *temp = nullptr;
    uint64_t arena_bytes = 0, temp_bytes = 0;
    uint64_t *pstart = nullptr, *roff = nullptr, *woff = nullptr, *words = nullptr;
    int64_t *begin = nullptr;
    uint32_t *parent = nullptr;
};

uint64_t align_up(uint64_t b) { return (b + 255) / 256 * 256; }

uint32_t bits_for(uint64_t max_value) {
    uint32_t b = 0;
    while (b < 64 && (max_value >> b)) ++b;
    return b;
}

uint32_t blocks(uint64_t n) { return (uint32_t)((n + MG_BLOCK - 1) / MG_BLOCK); }

int grow(uint8_t *&p, uint64_t &have, uint64_t need, std::string &msg) {
    if (have >= need) return WHMEC_OK;
    if (p) MG_CUDA(cudaFree(p));
    p = nullptr;
    MG_CUDA(cudaMalloc(&p, need));
    have = need;
    return WHMEC_OK;
}

int timed(MgDev &D, MgCall &call, std::string &msg) {  // after the launches between the two events
    MG_CUDA(cudaStreamSynchronize(D.s));
    float ms = 0;
    MG_CUDA(cudaEventElapsedTime(&ms, D.e0, D.e1));
    call.st.device_ms += ms;
    return WHMEC_OK;
}

}  // namespace

uint64_t mg_budget(int device, std::string &msg) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e == cudaSuccess && (device < 0 || device >= count)) e = cudaErrorInvalidDevice;
    if (e == cudaSuccess) e = cudaSetDevice(device);
    if (e != cudaSuccess) {
        msg = std::string("whmec_merge_reads: ") + cudaGetErrorString(e);
        return 0;
    }
    const uint64_t free_b = device_available_bytes(), margin = 512ull << 20;
    uint64_t budget = free_b > margin ? free_b - margin : 0;
    // WHMEC_MERGE_ARENA_BUDGET=bytes (test hook): the device bytes a call may take
    if (const char *h = std::getenv("WHMEC_MERGE_ARENA_BUDGET")) budget = std::min<uint64_t>(budget, std::strtoull(h, nullptr, 10));
    return budget;
}

int mg_open_set(int device, MgCall &call, std::string &msg) {
    if (!call.dev) call.dev = new MgDev();
    MgDev &D = *(MgDev *)call.dev;
    MG_CUDA(cudaSetDevice(device));
    if (!D.s) {
        MG_CUDA(cudaStreamCreateWithFlags(&D.s, cudaStreamNonBlocking));
        MG_CUDA(cudaEventCreate(&D.e0));
        MG_CUDA(cudaEventCreate(&D.e1));
        MG_CUDA(cudaMalloc(&D.blue, 8));
    }
    if (D.set) MG_CUDA(cudaFree(D.set));
    D.set = nullptr;
    const uint64_t n = call.n_reads, nw = call.woff[n], ne = call.n_entries;
    const uint64_t b_off = align_up((n + 1) * 8), b_begin = align_up(n * 8), b_words = align_up((nw + 1) * 8);
    const uint64_t b_parent = align_up(n * 4), b_allele = align_up(std::max<uint64_t>(ne, 1));
    MG_CUDA(cudaMalloc(&D.set, 3 * b_off + b_begin + b_words + b_parent + b_allele));
    uint8_t *a = D.set;
    auto take = [&](uint64_t b) { uint8_t *p = a; a += b; return p; };
    D.pstart = (uint64_t *)take(b_off), D.roff = (uint64_t *)take(b_off), D.woff = (uint64_t *)take(b_off);
    D.begin = (int64_t *)take(b_begin), D.words = (uint64_t *)take(b_words), D.parent = (uint32_t *)take(b_parent);
    uint8_t *d_allele = take(b_allele);
    MG_CUDA(cudaMemcpyAsync(D.pstart, call.pstart.data(), (n + 1) * 8, cudaMemcpyHostToDevice, D.s));
    MG_CUDA(cudaMemcpyAsync(D.roff, call.roff.data(), (n + 1) * 8, cudaMemcpyHostToDevice, D.s));
    MG_CUDA(cudaMemcpyAsync(D.woff, call.woff.data(), (n + 1) * 8, cudaMemcpyHostToDevice, D.s));
    MG_CUDA(cudaMemcpyAsync(D.begin, call.begin.data(), n * 8, cudaMemcpyHostToDevice, D.s));
    if (ne) MG_CUDA(cudaMemcpyAsync(d_allele, call.allele, ne, cudaMemcpyHostToDevice, D.s));
    call.st.h2d_bytes += 3 * (n + 1) * 8 + n * 8 + ne;
    MG_CUDA(cudaEventRecord(D.e0, D.s));
    mg_pack_kernel<<<blocks(nw + 1), MG_BLOCK, 0, D.s>>>(D.woff, D.roff, d_allele, (uint32_t)n, nw, D.words);
    MG_CUDA(cudaGetLastError());
    mg_init_kernel<<<blocks(n), MG_BLOCK, 0, D.s>>>(D.parent, (uint32_t)n);
    MG_CUDA(cudaGetLastError());
    MG_CUDA(cudaEventRecord(D.e1, D.s));
    call.st.kernel_launches += 2;
    return timed(D, call, msg);
}

int mg_run_pairs(int device, MgCall &call, std::string &msg) {
    MgDev &D = *(MgDev *)call.dev;
    const uint32_t np = (uint32_t)(call.p1 - call.p0);
    const int hook = !call.host_edges;
    int rc;
    if (!hook && (rc = grow(D.arena, D.arena_bytes, align_up(np) + align_up((uint64_t)np * 8), msg))) return rc;
    uint8_t *d_flag = hook ? nullptr : D.arena;
    int64_t *d_diff = hook ? nullptr : (int64_t *)(D.arena + align_up(np));
    MG_CUDA(cudaMemsetAsync(D.blue, 0, 8, D.s));
    MG_CUDA(cudaEventRecord(D.e0, D.s));
    mg_pair_kernel<<<blocks(np), MG_BLOCK, 0, D.s>>>(call.p0, np, D.pstart, call.n_reads, D.begin, D.roff, D.woff, D.words, call.thr_diff,
                                                     call.thr_neg_diff, call.max_error_rate, hook, D.parent, d_flag, d_diff, D.blue);
    MG_CUDA(cudaGetLastError());
    MG_CUDA(cudaEventRecord(D.e1, D.s));
    ++call.st.kernel_launches;
    unsigned long long blue = 0;
    MG_CUDA(cudaMemcpyAsync(&blue, D.blue, 8, cudaMemcpyDeviceToHost, D.s));
    call.st.d2h_bytes += 8;
    if (!hook) {
        call.flag.resize(np);
        call.diff.resize(np);
        MG_CUDA(cudaMemcpyAsync(call.flag.data(), d_flag, np, cudaMemcpyDeviceToHost, D.s));
        MG_CUDA(cudaMemcpyAsync(call.diff.data(), d_diff, (uint64_t)np * 8, cudaMemcpyDeviceToHost, D.s));
        call.st.d2h_bytes += (uint64_t)np * 9;
    }
    if ((rc = timed(D, call, msg))) return rc;
    call.blue += blue;
    return WHMEC_OK;
}

int mg_roots(int device, MgCall &call, std::string &msg) {
    MgDev &D = *(MgDev *)call.dev;
    const uint32_t n = call.n_reads;
    MG_CUDA(cudaEventRecord(D.e0, D.s));
    mg_compress_kernel<<<blocks(n), MG_BLOCK, 0, D.s>>>(D.parent, n);
    MG_CUDA(cudaGetLastError());
    MG_CUDA(cudaEventRecord(D.e1, D.s));
    ++call.st.kernel_launches;
    call.parent.resize(n);
    MG_CUDA(cudaMemcpyAsync(call.parent.data(), D.parent, (uint64_t)n * 4, cudaMemcpyDeviceToHost, D.s));
    call.st.d2h_bytes += (uint64_t)n * 4;
    return timed(D, call, msg);
}

int mg_run_accumulate(int device, MgCall &call, std::string &msg) {
    MgDev &D = *(MgDev *)call.dev;
    const uint32_t ne = (uint32_t)call.entries.size();
    const uint64_t b_en = align_up((uint64_t)ne * sizeof(MgEntry)), b_k = align_up((uint64_t)ne * 8), b_v = align_up((uint64_t)ne * 4);
    const uint64_t b_s = align_up(((uint64_t)ne + 1) * 4), b_r = align_up((uint64_t)ne * sizeof(MgRun));
    int rc;
    if ((rc = grow(D.arena, D.arena_bytes, b_en + 2 * b_k + 4 * b_v + b_s + b_r, msg))) return rc;
    uint8_t *a = D.arena;
    auto take = [&](uint64_t b) { uint8_t *p = a; a += b; return p; };
    MgEntry *d_en = (MgEntry *)take(b_en);
    uint64_t *k_a = (uint64_t *)take(b_k), *k_b = (uint64_t *)take(b_k);
    uint32_t *v_a = (uint32_t *)take(b_v), *v_b = (uint32_t *)take(b_v), *head = (uint32_t *)take(b_v), *rank = (uint32_t *)take(b_v);
    uint32_t *start = (uint32_t *)take(b_s);
    MgRun *d_runs = (MgRun *)take(b_r);
    MG_CUDA(cudaMemcpyAsync(d_en, call.entries.data(), (uint64_t)ne * sizeof(MgEntry), cudaMemcpyHostToDevice, D.s));
    call.st.h2d_bytes += (uint64_t)ne * sizeof(MgEntry);
    cub::DoubleBuffer<uint64_t> dk(k_a, k_b);
    cub::DoubleBuffer<uint32_t> dv(v_a, v_b);
    const int key_bits = (int)std::max<uint32_t>(1, call.pos_bits + bits_for(call.n_comp - 1));
    size_t t1 = 0, t2 = 0;
    MG_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t1, dk, dv, (int)ne, 0, key_bits, D.s));
    MG_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t2, head, rank, (int)ne, D.s));
    if ((rc = grow(D.temp, D.temp_bytes, std::max<size_t>({t1, t2, (size_t)1}), msg))) return rc;
    MG_CUDA(cudaEventRecord(D.e0, D.s));
    mg_key_kernel<<<blocks(ne), MG_BLOCK, 0, D.s>>>(d_en, ne, call.pmin, call.pos_bits, k_a, v_a);
    MG_CUDA(cudaGetLastError());
    size_t tb = D.temp_bytes;
    MG_CUDA(cub::DeviceRadixSort::SortPairs(D.temp, tb, dk, dv, (int)ne, 0, key_bits, D.s));
    mg_head_kernel<<<blocks(ne), MG_BLOCK, 0, D.s>>>(dk.Current(), ne, head);
    MG_CUDA(cudaGetLastError());
    tb = D.temp_bytes;
    MG_CUDA(cub::DeviceScan::ExclusiveSum(D.temp, tb, head, rank, (int)ne, D.s));
    mg_start_kernel<<<blocks(ne), MG_BLOCK, 0, D.s>>>(head, rank, ne, start);
    MG_CUDA(cudaGetLastError());
    uint32_t last[2] = {0, 0};
    MG_CUDA(cudaMemcpyAsync(&last[0], rank + ne - 1, 4, cudaMemcpyDeviceToHost, D.s));
    MG_CUDA(cudaMemcpyAsync(&last[1], head + ne - 1, 4, cudaMemcpyDeviceToHost, D.s));
    MG_CUDA(cudaStreamSynchronize(D.s));
    const uint32_t n_runs = last[0] + last[1];
    mg_sum_kernel<<<blocks(n_runs), MG_BLOCK, 0, D.s>>>(d_en, dv.Current(), start, n_runs, d_runs);
    MG_CUDA(cudaGetLastError());
    MG_CUDA(cudaEventRecord(D.e1, D.s));
    call.st.kernel_launches += 6;
    call.runs.resize(n_runs);
    MG_CUDA(cudaMemcpyAsync(call.runs.data(), d_runs, (uint64_t)n_runs * sizeof(MgRun), cudaMemcpyDeviceToHost, D.s));
    call.st.d2h_bytes += 8 + (uint64_t)n_runs * sizeof(MgRun);
    return timed(D, call, msg);
}

void mg_close(MgCall &call) {
    MgDev *D = (MgDev *)call.dev;
    if (!D) return;
    if (D->s) cudaStreamSynchronize(D->s);
    for (void *p : {(void *)D->blue, (void *)D->set, (void *)D->arena, (void *)D->temp}) cudaFree(p);
    for (cudaEvent_t e : {D->e0, D->e1})
        if (e) cudaEventDestroy(e);
    if (D->s) cudaStreamDestroy(D->s);
    delete D;
    call.dev = nullptr;
}

}  // namespace whmec
