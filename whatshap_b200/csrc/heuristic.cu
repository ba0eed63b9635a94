// The row-limited heuristic on the GPU (whmec_heuristic_batch, DESIGN §4.10): heur_batch_kernel sweeps a group of tables, one
// CTA per table taken from a work list, with the sweep of heuristic_device.h; this file also holds the group's arena, upload,
// launch and download (heur_run_group).  Compiled with -fmad=false: every float expression must round as heuristic.cpp's does.
#include <cuda_runtime.h>

#include <algorithm>
#include <string>
#include <vector>

#include "heuristic_batch.h"
#include "tile.cuh"  // device_available_bytes

namespace whmec {

namespace {

// the executor of heur_sweep on the device: the rows of a phase spread over the CTA's threads
struct DevExec {
    HeurShared &sh;
    template <class F>
    __device__ void rows(uint32_t n, F f) {
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) f(i);
    }
    template <class F>
    __device__ void single(F f) {
        if (threadIdx.x == 0) f();
    }
    __device__ void sync() { __syncthreads(); }
    __device__ int32_t atomic_cas(int32_t *p, int32_t cmp, int32_t v) { return atomicCAS(p, cmp, v); }
    __device__ void atomic_min(int32_t *p, int32_t v) { atomicMin(p, v); }
    __device__ void atomic_min(uint32_t *p, uint32_t v) { atomicMin(p, v); }
    __device__ void atomic_min(unsigned long long *p, unsigned long long v) { atomicMin(p, v); }
    __device__ void atomic_add(uint32_t *p, uint32_t v) { atomicAdd(p, v); }
    __device__ void store(uint32_t *p, uint32_t v) { *p = v; }
    // exclusive prefix sums of a[0..n) in place, chunk by chunk of the CTA; returns the total (every thread)
    __device__ uint32_t scan(uint32_t *a, uint32_t n) {
        const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = blockDim.x >> 5;
        uint32_t carry = 0;
        for (uint32_t base = 0; base < n; base += blockDim.x) {
            const uint32_t i = base + threadIdx.x;
            const uint32_t v = i < n ? a[i] : 0u;
            uint32_t incl = v;
            for (uint32_t o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
                if (lane >= o) incl += y;
            }
            if (lane == 31) sh.warp_sums[warp] = incl;
            __syncthreads();
            if (warp == 0) {
                uint32_t w = lane < n_warps ? sh.warp_sums[lane] : 0u;
                for (uint32_t o = 1; o < 32; o <<= 1) {
                    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, w, o);
                    if (lane >= o) w += y;
                }
                if (lane < n_warps) sh.warp_sums[lane] = w;
            }
            __syncthreads();
            if (i < n) a[i] = carry + (warp ? sh.warp_sums[warp - 1] : 0u) + incl - v;
            carry += sh.warp_sums[n_warps - 1];
            __syncthreads();
        }
        return carry;
    }
};

__global__ void __launch_bounds__(HEUR_THREADS) heur_batch_kernel(const HeurDevTable *tables, uint32_t n_tables, uint32_t *next) {
    __shared__ HeurShared sh;
    __shared__ uint32_t s_table;
    DevExec x{sh};
    for (;;) {
        if (threadIdx.x == 0) s_table = atomicAdd(next, 1u);
        __syncthreads();
        const uint32_t t = s_table;
        __syncthreads();
        if (t >= n_tables) return;
        heur_sweep(x, sh, tables[t]);
    }
}

#define HEUR_CUDA(expr)                                               \
    do {                                                              \
        cudaError_t _e = (expr);                                      \
        if (_e != cudaSuccess) {                                      \
            msg = std::string(#expr) + ": " + cudaGetErrorString(_e); \
            rc = WHMEC_ERR_CUDA;                                      \
            goto done;                                                \
        }                                                             \
    } while (0)

}  // namespace

uint64_t heur_budget(int device, std::string &msg) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e == cudaSuccess && (device < 0 || device >= count)) e = cudaErrorInvalidDevice;
    if (e == cudaSuccess) e = cudaSetDevice(device);
    if (e != cudaSuccess) {
        msg = std::string("whmec_heuristic_batch: ") + cudaGetErrorString(e);
        return 0;
    }
    const uint64_t free_b = device_available_bytes();
    const uint64_t margin = 512ull << 20;
    return free_b > margin ? free_b - margin : 0;
}

int heur_run_group(int device, const std::vector<HeurLayout> &layouts, const HeurGroup &g, std::vector<uint8_t> &in, std::vector<uint8_t> &out,
                   float *ms, std::string &msg) {
    int rc = WHMEC_OK;
    uint8_t *arena = nullptr;
    cudaStream_t s = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    int sms = 0;
    const uint32_t n = (uint32_t)g.members.size();
    const uint64_t in_b = g.in_bytes, work_b = g.work_bytes, out_b = g.out_bytes;
    HEUR_CUDA(cudaSetDevice(device));
    HEUR_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    HEUR_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    HEUR_CUDA(cudaEventCreate(&e0));
    HEUR_CUDA(cudaEventCreate(&e1));
    // one arena: [inputs (descriptors first) | work counter | rows, scratch and records | outputs]
    HEUR_CUDA(cudaMalloc(&arena, in_b + 16 + work_b + out_b));
    {
        uint8_t *d_in = arena, *d_next = arena + in_b, *d_work = d_next + 16, *d_out = d_work + work_b;
        HeurDevTable *desc = (HeurDevTable *)in.data();
        for (uint32_t j = 0; j < n; ++j) desc[j] = heur_bind(layouts[g.members[j]], d_in, d_work, d_out);
        HEUR_CUDA(cudaMemcpyAsync(d_in, in.data(), in_b, cudaMemcpyHostToDevice, s));
        HEUR_CUDA(cudaMemsetAsync(d_next, 0, 16, s));
        const uint32_t grid = std::min<uint32_t>(n, 2u * (uint32_t)sms);
        HEUR_CUDA(cudaEventRecord(e0, s));
        heur_batch_kernel<<<grid, HEUR_THREADS, 0, s>>>((const HeurDevTable *)d_in, n, (uint32_t *)d_next);
        HEUR_CUDA(cudaGetLastError());
        HEUR_CUDA(cudaEventRecord(e1, s));
        out.assign(out_b, 0);
        HEUR_CUDA(cudaMemcpyAsync(out.data(), d_out, out_b, cudaMemcpyDeviceToHost, s));
        HEUR_CUDA(cudaStreamSynchronize(s));
        HEUR_CUDA(cudaEventElapsedTime(ms, e0, e1));
    }
done:
    if (arena) cudaFree(arena);
    if (e0) cudaEventDestroy(e0);
    if (e1) cudaEventDestroy(e1);
    if (s) cudaStreamDestroy(s);
    if (rc != WHMEC_OK) msg = "CUDA failure in whmec_heuristic_batch: " + msg;
    return rc;
}

}  // namespace whmec
