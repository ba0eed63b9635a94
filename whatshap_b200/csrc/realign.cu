// Allele detection by re-alignment on the GPU (whmec_realign, DESIGN §4.11; k-mer mode, §4.12): the kernels of one chunk and its
// arena, uploads and downloads (ra_run_chunk).  Per-job code: realign.h, kmerald.h.  Compiled with -fmad=false: the affine and
// k-mer recurrences must round one float operation at a time, as align.pyx does.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <string>
#include <vector>

#include "realign_plan.h"
#include "tile.cuh"  // device_available_bytes

namespace whmec {

namespace {

constexpr uint32_t RA_BLOCK = 128;
constexpr unsigned FULL = 0xFFFFFFFFu;

// one thread per one-thread job
__global__ void __launch_bounds__(RA_BLOCK) ra_short_kernel(RaBufs b, const RaItem *items, uint32_t item0, const RaJob *jobs, uint32_t n_jobs,
                                                            RaParams pr, int64_t *dist, uint8_t *status) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const RaJob jb = jobs[k];
    if (jb.scratch != RA_NO_SCRATCH) return;
    int64_t d = 0;
    status[k] = !ra_short_job(b, items[jb.item - item0], jb.allele, pr, d);
    dist[k] = d;
}

// one warp per longer job: an anti-diagonal wavefront, lane L one column behind lane L - 1
__global__ void __launch_bounds__(RA_BLOCK) ra_long_kernel(RaBufs b, const RaItem *items, uint32_t item0, const RaJob *jobs, const uint32_t *list,
                                                           uint32_t n_list, RaParams pr, uint8_t *scratch, int64_t *dist, uint8_t *status) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warps = gridDim.x * (blockDim.x / 32);
    for (uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) / 32; w < n_list; w += warps) {
        const uint32_t k = list[w];
        const RaJob jb = jobs[k];
        const RaItem it = items[jb.item - item0];
        RaSeq q = ra_query(b, it), t = ra_target(b, it, jb.allele);
        ra_trim(q, t);
        int64_t d = 0;
        bool ok = true;
        if (!pr.affine) {
            const RaSeq &p = q.len <= t.len ? q : t, &x = q.len <= t.len ? t : q;
            if (p.len <= RA_SHORT) {
                if (lane == 0) d = ra_unit_short(q, t);
            } else {
                int8_t *hrow = (int8_t *)(scratch + jb.scratch);  // bottom deltas of a 32-word group, for the next group
                const uint32_t words = (p.len + 63) / 64, groups = (words + 31) / 32;
                for (uint32_t g = 0; g < groups; ++g) {
                    RaUnitLane ln;
                    ln.init(p, 32 * g + lane);
                    int out = 0;
                    for (uint32_t s = 0; s < x.len + 31; ++s) {
                        const int recv = __shfl_up_sync(FULL, out, 1);
                        const int64_t j = (int64_t)s - lane;
                        if (ln.active && j >= 0 && j < x.len) {
                            const int hin = lane ? recv : g ? hrow[j] : 1;
                            out = ln.step(p, x.at((uint32_t)j), hin);
                            if (lane == 31 && g + 1 < groups) hrow[j] = (int8_t)out;
                        }
                    }
                    __syncwarp();
                    if (g + 1 == groups) d = __shfl_sync(FULL, (long long)ln.score, (words - 1) % 32);
                }
            }
        } else if (q.len <= RA_SHORT) {
            if (lane == 0) ok = ra_trunc(ra_affine_short(q, t, pr), d);
        } else {
            const uint32_t m = q.len;
            float *A = (float *)(scratch + jb.scratch), *B = A + (m + 1), *C = B + (m + 1);
            RaAffLane ln;
            ln.init(m, lane, 32, A, B, C, pr);
            RaCell out{0.0f, 0.0f, 0.0f};
            for (uint32_t s = 0; s < t.len + 31; ++s) {
                const RaCell recv{__shfl_up_sync(FULL, out.a, 1), __shfl_up_sync(FULL, out.b, 1), __shfl_up_sync(FULL, out.c, 1)};
                const int64_t j = (int64_t)s - lane + 1;
                if (ln.active() && j >= 1 && j <= t.len) out = ln.step(A, B, C, lane ? recv : ra_affine_top((uint32_t)j, pr), q, t.at((uint32_t)(j - 1)), pr);
            }
            __syncwarp();
            if (lane == 0) ok = ra_trunc(ra_min3(A[m], B[m], C[m]), d);
        }
        if (lane == 0) {
            dist[k] = d;
            status[k] = !ok;
        }
    }
}

// one thread per item: the call from the item's distances
__global__ void __launch_bounds__(RA_BLOCK) ra_decide_kernel(const RaItem *items, uint32_t n_items, uint32_t job0, const int64_t *dist, int affine,
                                                             int32_t *call, int64_t *quality) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_items) return;
    const RaItem it = items[i];
    int64_t q = 0;
    call[i] = ra_decide(dist + (it.job0 - job0), it.n_jobs, affine, q);
    quality[i] = q;
}

// ---- k-mer mode (kmerald.h) ----------------------------------------------------------------------------------------------------

// one thread per one-thread k-mer job
__global__ void __launch_bounds__(RA_BLOCK) ka_short_kernel(RaBufs b, const RaItem *items, uint32_t item0, const RaJob *jobs, uint32_t n_jobs,
                                                            KaParams p, float *dist) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_jobs) return;
    const RaJob jb = jobs[k];
    if (jb.scratch != RA_NO_SCRATCH) return;
    dist[k] = ka_short_job(b, items[jb.item - item0], jb.allele, p);
}

// one warp per longer k-mer job: lane 0 lists the k-mers into the job's scratch, every lane finds its rows' costs, then an
// anti-diagonal wavefront over row bands, lane L one column behind lane L - 1
__global__ void __launch_bounds__(RA_BLOCK) ka_long_kernel(RaBufs b, const RaItem *items, uint32_t item0, const RaJob *jobs, const uint32_t *list,
                                                           uint32_t n_list, KaParams p, uint8_t *scratch, float *dist) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warps = gridDim.x * (blockDim.x / 32);
    for (uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) / 32; w < n_list; w += warps) {
        const uint32_t k = list[w];
        const RaJob jb = jobs[k];
        const RaItem it = items[jb.item - item0];
        const RaSeq q = ra_query(b, it), t = ra_target(b, it, jb.allele);
        const KaScratch s(scratch + jb.scratch, q.len, t.len);
        uint32_t m = 0, n = 0, x = 0;
        if (lane == 0) m = ka_kmers(t, p.k, s.a), n = ka_kmers(q, p.k, s.b);
        m = __shfl_sync(FULL, m, 0);
        n = __shfl_sync(FULL, n, 0);
        __syncwarp();
        float d = 0.0f;
        if (ka_trim(s.a, s.b, m, n, x)) {
            if (m == 0) {
                d = p.gap * (float)n;
            } else {
                const uint32_t *a = s.a + x, *bq = s.b + x;
                KaLane ln;
                ln.init(m, lane, 32, a, s.row, s.S, p);
                float out = 0.0f;
                for (uint32_t st = 0; st < n + 31; ++st) {
                    const float recv = __shfl_up_sync(FULL, out, 1);
                    const int64_t j = (int64_t)st - lane + 1;
                    if (ln.active() && j >= 1 && j <= n) out = ln.step(a, s.row, s.S, lane ? recv : p.gap * (float)j, bq[j - 1], p);
                }
                __syncwarp();
                d = s.S[m];
            }
        }
        if (lane == 0) dist[k] = d;
    }
}

// one thread per item: the call from the distances of allele 0 and alternative_allele
__global__ void __launch_bounds__(RA_BLOCK) ka_decide_kernel(const RaItem *items, uint32_t n_items, uint32_t job0, const float *dist, int32_t *call,
                                                             int64_t *quality) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_items) return;
    const RaItem it = items[i];
    call[i] = ka_decide(dist[it.job0 - job0], dist[it.job0 - job0 + 1]);
    quality[i] = 30;
}

#define RA_CUDA(expr)                                                 \
    do {                                                              \
        cudaError_t _e = (expr);                                      \
        if (_e != cudaSuccess) {                                      \
            msg = std::string(#expr) + ": " + cudaGetErrorString(_e); \
            return WHMEC_ERR_CUDA;                                    \
        }                                                             \
    } while (0)

// per call: the variants' alleles on the device, a stream, events and an arena that grows to the largest chunk
struct RaDev {
    cudaStream_t s = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    uint8_t *al = nullptr;
    uint64_t *al_off = nullptr;
    uint32_t *al_first = nullptr;
    uint64_t *key = nullptr;  // k-mer mode: the costs table
    float *cost = nullptr;
    uint8_t *arena = nullptr;
    uint64_t arena_bytes = 0;
    int sms = 0;
};

uint64_t align_up(uint64_t b) { return (b + 255) / 256 * 256; }

// the launches and downloads of a k-mer chunk (ra_run_chunk after its uploads): float distances, no status
int ka_launch(RaCall &call, const RaChunk &c, RaDev &D, const RaBufs &b, const RaItem *d_items, const RaJob *d_jobs, const uint32_t *d_list,
              size_t n_list, uint8_t *d_scratch, float *d_dist, int32_t *d_call, int64_t *d_quality, std::string &msg) {
    const uint32_t ni = c.item1 - c.item0, nj = c.job1 - c.job0;
    const KaParams p{call.kparams.k, call.kparams.gap, D.key, D.cost, call.kparams.n};
    RA_CUDA(cudaEventRecord(D.e0, D.s));
    ka_short_kernel<<<(nj + RA_BLOCK - 1) / RA_BLOCK, RA_BLOCK, 0, D.s>>>(b, d_items, c.item0, d_jobs, nj, p, d_dist);
    RA_CUDA(cudaGetLastError());
    ++call.st.kernel_launches;
    if (n_list) {
        const uint32_t per_block = RA_BLOCK / 32;
        const uint32_t grid = (uint32_t)std::min<uint64_t>((n_list + per_block - 1) / per_block, 64ull * D.sms);
        ka_long_kernel<<<grid, RA_BLOCK, 0, D.s>>>(b, d_items, c.item0, d_jobs, d_list, (uint32_t)n_list, p, d_scratch, d_dist);
        RA_CUDA(cudaGetLastError());
        ++call.st.kernel_launches;
    }
    if (call.decide) {
        ka_decide_kernel<<<(ni + RA_BLOCK - 1) / RA_BLOCK, RA_BLOCK, 0, D.s>>>(d_items, ni, c.job0, d_dist, d_call, d_quality);
        RA_CUDA(cudaGetLastError());
        ++call.st.kernel_launches;
    }
    RA_CUDA(cudaEventRecord(D.e1, D.s));
    if (call.decide) {
        RA_CUDA(cudaMemcpyAsync(call.call + c.item0, d_call, ni * 4, cudaMemcpyDeviceToHost, D.s));
        RA_CUDA(cudaMemcpyAsync(call.quality + c.item0, d_quality, ni * 8, cudaMemcpyDeviceToHost, D.s));
        call.st.d2h_bytes += ni * 12;
    } else {
        RA_CUDA(cudaMemcpyAsync(call.kdist + c.job0, d_dist, nj * 4, cudaMemcpyDeviceToHost, D.s));
        call.st.d2h_bytes += nj * 4;
    }
    RA_CUDA(cudaStreamSynchronize(D.s));
    float ms = 0;
    RA_CUDA(cudaEventElapsedTime(&ms, D.e0, D.e1));
    call.st.device_ms += ms;
    return WHMEC_OK;
}

}  // namespace

uint64_t ra_budget(int device, std::string &msg) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e == cudaSuccess && (device < 0 || device >= count)) e = cudaErrorInvalidDevice;
    if (e == cudaSuccess) e = cudaSetDevice(device);
    if (e != cudaSuccess) {
        msg = std::string("whmec_realign: ") + cudaGetErrorString(e);
        return 0;
    }
    install_pinned_staging();
    const uint64_t free_b = device_available_bytes(), margin = 512ull << 20;
    uint64_t budget = free_b > margin ? free_b - margin : 0;
    // WHMEC_REALIGN_ARENA_BUDGET=bytes (test hook): the device bytes a call may take
    if (const char *h = std::getenv("WHMEC_REALIGN_ARENA_BUDGET")) budget = std::min<uint64_t>(budget, std::strtoull(h, nullptr, 10));
    return budget;
}

int ra_run_chunk(int device, RaCall &call, const RaChunk &c, std::string &msg) {
    if (!call.dev) call.dev = new RaDev();
    RaDev &D = *(RaDev *)call.dev;
    RA_CUDA(cudaSetDevice(device));
    if (!D.s) {
        RA_CUDA(cudaDeviceGetAttribute(&D.sms, cudaDevAttrMultiProcessorCount, device));
        RA_CUDA(cudaStreamCreateWithFlags(&D.s, cudaStreamNonBlocking));
        RA_CUDA(cudaEventCreate(&D.e0));
        RA_CUDA(cudaEventCreate(&D.e1));
        if (call.n_alleles) {
            const uint64_t nb = call.host.al_off[call.n_alleles];
            RA_CUDA(cudaMalloc(&D.al, std::max<uint64_t>(nb, 1)));
            RA_CUDA(cudaMalloc(&D.al_off, (call.n_alleles + 1) * 8));
            RA_CUDA(cudaMalloc(&D.al_first, (uint64_t)(call.n_variants + 1) * 4));
            RA_CUDA(cudaMemcpyAsync(D.al, call.host.al, nb, cudaMemcpyHostToDevice, D.s));
            RA_CUDA(cudaMemcpyAsync(D.al_off, call.host.al_off, (call.n_alleles + 1) * 8, cudaMemcpyHostToDevice, D.s));
            RA_CUDA(cudaMemcpyAsync(D.al_first, call.host.al_first, (uint64_t)(call.n_variants + 1) * 4, cudaMemcpyHostToDevice, D.s));
            call.st.h2d_bytes += nb + (call.n_alleles + 1) * 8 + (uint64_t)(call.n_variants + 1) * 4;
        }
        if (call.kmerald && call.kparams.n) {
            const uint64_t nk = call.kparams.n;
            RA_CUDA(cudaMalloc(&D.key, nk * 8));
            RA_CUDA(cudaMalloc(&D.cost, nk * 4));
            RA_CUDA(cudaMemcpyAsync(D.key, call.kparams.key, nk * 8, cudaMemcpyHostToDevice, D.s));
            RA_CUDA(cudaMemcpyAsync(D.cost, call.kparams.cost, nk * 4, cudaMemcpyHostToDevice, D.s));
            call.st.h2d_bytes += nk * 12;
        }
    }
    if (D.arena_bytes < c.bytes) {
        if (D.arena) RA_CUDA(cudaFree(D.arena));
        D.arena = nullptr;
        RA_CUDA(cudaMalloc(&D.arena, c.bytes));
        D.arena_bytes = c.bytes;
    }
    const uint32_t ni = c.item1 - c.item0, nj = c.job1 - c.job0;
    std::vector<uint32_t> list;  // the chunk's warp jobs
    for (uint32_t k = c.job0; k < c.job1; ++k)
        if (call.jobs[k].scratch != RA_NO_SCRATCH) list.push_back(k - c.job0);
    // the arena in the order of ra_chunk_bytes
    uint8_t *p = D.arena;
    auto take = [&p](uint64_t bytes) {
        uint8_t *r = p;
        p += align_up(bytes);
        return r;
    };
    RaItem *d_items = (RaItem *)take(ni * sizeof(RaItem));
    RaJob *d_jobs = (RaJob *)take(nj * sizeof(RaJob));
    uint32_t *d_list = (uint32_t *)take(nj * 4);
    int64_t *d_dist = (int64_t *)take(nj * 8);
    uint8_t *d_status = take(nj);
    int32_t *d_call = (int32_t *)take(ni * 4);
    int64_t *d_quality = (int64_t *)take(ni * 8);
    uint8_t *d_q = take(c.q_hi - c.q_lo);
    uint8_t *d_r = take((uint64_t)(c.r_hi - c.r_lo));
    uint8_t *d_scratch = take(c.scratch);
    RA_CUDA(cudaMemcpyAsync(d_items, call.items + c.item0, ni * sizeof(RaItem), cudaMemcpyHostToDevice, D.s));
    RA_CUDA(cudaMemcpyAsync(d_jobs, call.jobs + c.job0, nj * sizeof(RaJob), cudaMemcpyHostToDevice, D.s));
    if (!list.empty()) RA_CUDA(cudaMemcpyAsync(d_list, list.data(), list.size() * 4, cudaMemcpyHostToDevice, D.s));
    RA_CUDA(cudaMemcpyAsync(d_q, call.host.q + c.q_lo, c.q_hi - c.q_lo, cudaMemcpyHostToDevice, D.s));
    RA_CUDA(cudaMemcpyAsync(d_r, call.host.ref + c.r_lo, (uint64_t)(c.r_hi - c.r_lo), cudaMemcpyHostToDevice, D.s));
    call.st.h2d_bytes += ni * sizeof(RaItem) + nj * sizeof(RaJob) + list.size() * 4 + (c.q_hi - c.q_lo) + (uint64_t)(c.r_hi - c.r_lo);
    const RaBufs b{d_q, c.q_lo, d_r, c.r_lo, D.al, D.al_off, D.al_first};
    if (call.kmerald) return ka_launch(call, c, D, b, d_items, d_jobs, d_list, list.size(), d_scratch, (float *)d_dist, d_call, d_quality, msg);
    RA_CUDA(cudaEventRecord(D.e0, D.s));
    ra_short_kernel<<<(nj + RA_BLOCK - 1) / RA_BLOCK, RA_BLOCK, 0, D.s>>>(b, d_items, c.item0, d_jobs, nj, call.params, d_dist, d_status);
    RA_CUDA(cudaGetLastError());
    ++call.st.kernel_launches;
    if (!list.empty()) {
        const uint32_t per_block = RA_BLOCK / 32;
        const uint32_t grid = (uint32_t)std::min<uint64_t>((list.size() + per_block - 1) / per_block, 64ull * D.sms);
        ra_long_kernel<<<grid, RA_BLOCK, 0, D.s>>>(b, d_items, c.item0, d_jobs, d_list, (uint32_t)list.size(), call.params, d_scratch, d_dist,
                                                   d_status);
        RA_CUDA(cudaGetLastError());
        ++call.st.kernel_launches;
    }
    if (call.decide) {
        ra_decide_kernel<<<(ni + RA_BLOCK - 1) / RA_BLOCK, RA_BLOCK, 0, D.s>>>(d_items, ni, c.job0, d_dist, call.params.affine, d_call, d_quality);
        RA_CUDA(cudaGetLastError());
        ++call.st.kernel_launches;
    }
    RA_CUDA(cudaEventRecord(D.e1, D.s));
    RA_CUDA(cudaMemcpyAsync(call.status + c.job0, d_status, nj, cudaMemcpyDeviceToHost, D.s));
    call.st.d2h_bytes += nj;
    if (call.decide) {
        RA_CUDA(cudaMemcpyAsync(call.call + c.item0, d_call, ni * 4, cudaMemcpyDeviceToHost, D.s));
        RA_CUDA(cudaMemcpyAsync(call.quality + c.item0, d_quality, ni * 8, cudaMemcpyDeviceToHost, D.s));
        call.st.d2h_bytes += ni * 12;
    } else {
        RA_CUDA(cudaMemcpyAsync(call.dist + c.job0, d_dist, nj * 8, cudaMemcpyDeviceToHost, D.s));
        call.st.d2h_bytes += nj * 8;
    }
    RA_CUDA(cudaStreamSynchronize(D.s));
    float ms = 0;
    RA_CUDA(cudaEventElapsedTime(&ms, D.e0, D.e1));
    call.st.device_ms += ms;
    return WHMEC_OK;
}

void ra_close(RaCall &call) {
    RaDev *D = (RaDev *)call.dev;
    if (!D) return;
    if (D->s) cudaStreamSynchronize(D->s);
    cudaFree(D->arena);
    cudaFree(D->al);
    cudaFree(D->al_off);
    cudaFree(D->al_first);
    cudaFree(D->key);
    cudaFree(D->cost);
    if (D->e0) cudaEventDestroy(D->e0);
    if (D->e1) cudaEventDestroy(D->e1);
    if (D->s) cudaStreamDestroy(D->s);
    delete D;
    call.dev = nullptr;
}

}  // namespace whmec
