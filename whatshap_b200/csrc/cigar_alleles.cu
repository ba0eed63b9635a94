// Allele detection from the CIGAR alone on the GPU (whmec_detect_alleles_cigar, DESIGN §4.14): the kernels of one chunk and its arena,
// uploads and downloads (ca_run_chunk).  Per-thread code: cigar_alleles.h.
//
// A chunk is a run of alignments.  ca_count_kernel walks each alignment's CIGAR (one thread per alignment) and counts its items; a
// scan gives every alignment its first item.  The items are then handled in windows that fit the budget: ca_emit_kernel walks again
// and writes the window's items, ca_resolve_kernel resolves each item (one thread per item), and a select keeps the calls, which are
// already in alignment and enqueue order.
#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include <algorithm>
#include <string>

#include "cigar_alleles_plan.h"

namespace whmec {

uint64_t ra_budget(int device, std::string &msg);  // realign.cu: the free HBM less 512 MB, or WHMEC_REALIGN_ARENA_BUDGET

namespace {

constexpr uint32_t CA_BLOCK = 128;

__global__ void __launch_bounds__(CA_BLOCK) ca_count_kernel(CaBufs b, uint32_t n, uint64_t *count) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a > n) return;
    CaCount c;
    if (a < n) ca_walk(b, a, c);
    count[a] = c.n;  // count[n] = 0: the exclusive scan's last entry is the chunk's total
}

__global__ void __launch_bounds__(CA_BLOCK) ca_emit_kernel(CaBufs b, uint32_t n, const uint64_t *first, uint64_t lo, uint64_t hi, CaItem *items) {
    const uint32_t a = blockIdx.x * blockDim.x + threadIdx.x;
    if (a >= n || first[a + 1] <= lo || first[a] >= hi) return;
    CaEmit e{items, first[a], lo, hi};
    ca_walk(b, a, e);
}

__global__ void __launch_bounds__(CA_BLOCK, 1) ca_resolve_kernel(CaBufs b, const CaItem *items, uint32_t m, uint32_t a0, CaCall *calls,
                                                              uint32_t *raised, unsigned long long *alleles) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t n_alleles = 0;
    if (k < m) {
        const CaItem it = items[k];
        CaCall c{a0 + it.aln, b.vars[it.var].id, -1, 0, 0};
        if (!ca_resolve(b, it, c.allele, c.quality, n_alleles)) {
            atomicMin(raised, a0 + it.aln);
            c.allele = -1;
        }
        calls[k] = c;
    }
    const uint32_t sum = __reduce_add_sync(0xFFFFFFFFu, n_alleles);
    if ((threadIdx.x & 31) == 0 && sum) atomicAdd(alleles, (unsigned long long)sum);
}

struct IsCall {
    __host__ __device__ bool operator()(const CaCall &c) const { return c.allele >= 0; }
};

#define CA_CUDA(expr)                                                 \
    do {                                                              \
        cudaError_t _e = (expr);                                      \
        if (_e != cudaSuccess) {                                      \
            msg = std::string(#expr) + ": " + cudaGetErrorString(_e); \
            return WHMEC_ERR_CUDA;                                    \
        }                                                             \
    } while (0)

// per call: the variants and their alleles on the device, a stream, events, an arena that grows to the largest chunk and window, the
// scan and select scratch, and three device scalars (the window's call count, the first raising alignment, the allele count)
struct CaDev {
    cudaStream_t s = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    CaVar *vars = nullptr;
    CaAllele *alleles = nullptr;
    uint8_t *ab = nullptr;
    uint8_t *arena = nullptr;  // the chunk's alignments, operations and bytes
    uint64_t arena_bytes = 0;
    uint8_t *win = nullptr;    // a window's items and outcomes
    uint64_t win_bytes = 0;
    void *temp = nullptr;
    size_t temp_bytes = 0;
    uint64_t *scalars = nullptr;  // [0] calls (int), [1] raised (uint32), [2] alleles
    uint64_t *host = nullptr;     // page-locked copy of the scalars
};

uint64_t align_up(uint64_t b) { return (b + 255) / 256 * 256; }

int ensure_temp(CaDev &D, size_t bytes, std::string &msg) {
    if (bytes <= D.temp_bytes) return WHMEC_OK;
    if (D.temp) CA_CUDA(cudaFree(D.temp));
    D.temp = nullptr;
    CA_CUDA(cudaMalloc(&D.temp, bytes));
    D.temp_bytes = bytes;
    return WHMEC_OK;
}

int grow(uint8_t *&buf, uint64_t &have, uint64_t need, std::string &msg) {
    if (need <= have) return WHMEC_OK;
    if (buf) CA_CUDA(cudaFree(buf));
    buf = nullptr;
    CA_CUDA(cudaMalloc(&buf, need));
    have = need;
    return WHMEC_OK;
}

int ca_setup(int device, CaRun &run, CaDev &D, std::string &msg) {
    const CaPlan &P = *run.plan;
    CA_CUDA(cudaSetDevice(device));
    CA_CUDA(cudaStreamCreateWithFlags(&D.s, cudaStreamNonBlocking));
    CA_CUDA(cudaEventCreate(&D.e0));
    CA_CUDA(cudaEventCreate(&D.e1));
    CA_CUDA(cudaMalloc(&D.scalars, 3 * sizeof(uint64_t)));
    CA_CUDA(cudaMallocHost(&D.host, 3 * sizeof(uint64_t)));
    const uint64_t nv = P.vars.size(), nal = P.alleles.size();
    const uint32_t n_var = run.in->n_variants;
    const uint64_t nb = n_var ? run.in->allele_off[run.in->allele_first[n_var]] : 0;
    CA_CUDA(cudaMalloc(&D.vars, nv * sizeof(CaVar)));
    CA_CUDA(cudaMalloc(&D.alleles, std::max<uint64_t>(nal, 1) * sizeof(CaAllele)));
    CA_CUDA(cudaMalloc(&D.ab, std::max<uint64_t>(nb, 1)));
    CA_CUDA(cudaMemcpyAsync(D.vars, P.vars.data(), nv * sizeof(CaVar), cudaMemcpyHostToDevice, D.s));
    if (nal) CA_CUDA(cudaMemcpyAsync(D.alleles, P.alleles.data(), nal * sizeof(CaAllele), cudaMemcpyHostToDevice, D.s));
    if (nb) CA_CUDA(cudaMemcpyAsync(D.ab, run.in->allele_bytes, nb, cudaMemcpyHostToDevice, D.s));
    run.st.h2d_bytes += nv * sizeof(CaVar) + nal * sizeof(CaAllele) + nb;
    return WHMEC_OK;
}

}  // namespace

uint64_t ca_budget(int device, std::string &msg) {
    const uint64_t b = ra_budget(device, msg);
    if (!msg.empty()) msg = "whmec_detect_alleles_cigar" + msg.substr(msg.find(':'));
    return b;
}

int ca_run_chunk(int device, CaRun &run, const CaChunk &c, std::string &msg) {
    if (!run.dev) {
        run.dev = new CaDev();
        if (const int rc = ca_setup(device, run, *(CaDev *)run.dev, msg)) return rc;
    }
    CaDev &D = *(CaDev *)run.dev;
    const CaPlan &P = *run.plan;
    const whmec_realign_input &in = *run.in;
    const uint32_t na = c.a1 - c.a0;
    // the chunk's arena, in the order of ca_chunk_bytes (its scratch is D.temp)
    size_t t_scan = 0, t_sel = 0;
    CA_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t_scan, (uint64_t *)nullptr, (uint64_t *)nullptr, (int)na + 1, D.s));
    if (const int rc = ensure_temp(D, t_scan, msg)) return rc;
    if (const int rc = grow(D.arena, D.arena_bytes, c.bytes, msg)) return rc;
    uint8_t *p = D.arena;
    auto take = [&p](uint64_t bytes) {
        uint8_t *r = p;
        p += align_up(bytes);
        return r;
    };
    CaAln *d_alns = (CaAln *)take(na * sizeof(CaAln));
    uint64_t *d_count = (uint64_t *)take((na + 1) * 8);
    uint64_t *d_first = (uint64_t *)take((na + 1) * 8);
    uint8_t *d_op = take(c.op_hi - c.op_lo);
    int32_t *d_len = (int32_t *)take((c.op_hi - c.op_lo) * 4);
    uint8_t *d_q = take(c.q_hi - c.q_lo);
    uint8_t *d_qual = take(c.qual_hi - c.qual_lo);
    CA_CUDA(cudaMemcpyAsync(d_alns, P.alns.data() + c.a0, na * sizeof(CaAln), cudaMemcpyHostToDevice, D.s));
    if (c.op_hi > c.op_lo) {
        CA_CUDA(cudaMemcpyAsync(d_op, in.cigar_op + c.op_lo, c.op_hi - c.op_lo, cudaMemcpyHostToDevice, D.s));
        CA_CUDA(cudaMemcpyAsync(d_len, in.cigar_len + c.op_lo, (c.op_hi - c.op_lo) * 4, cudaMemcpyHostToDevice, D.s));
    }
    if (c.q_hi > c.q_lo) CA_CUDA(cudaMemcpyAsync(d_q, in.query + c.q_lo, c.q_hi - c.q_lo, cudaMemcpyHostToDevice, D.s));
    if (c.qual_hi > c.qual_lo) CA_CUDA(cudaMemcpyAsync(d_qual, run.q->qual + c.qual_lo, c.qual_hi - c.qual_lo, cudaMemcpyHostToDevice, D.s));
    run.st.h2d_bytes += na * sizeof(CaAln) + (c.op_hi - c.op_lo) * 5 + (c.q_hi - c.q_lo) + (c.qual_hi - c.qual_lo);
    const CaBufs b{d_op, d_len, c.op_lo, d_q, c.q_lo, d_qual, c.qual_lo, d_alns, D.vars, (uint32_t)(P.vars.size() - 1), D.alleles, D.ab};
    float ms = 0;
    CA_CUDA(cudaEventRecord(D.e0, D.s));
    ca_count_kernel<<<(na + CA_BLOCK) / CA_BLOCK, CA_BLOCK, 0, D.s>>>(b, na, d_count);
    CA_CUDA(cudaGetLastError());
    size_t tb = D.temp_bytes;
    CA_CUDA(cub::DeviceScan::ExclusiveSum(D.temp, tb, d_count, d_first, (int)na + 1, D.s));
    CA_CUDA(cudaMemcpyAsync(D.host, d_first + na, 8, cudaMemcpyDeviceToHost, D.s));
    CA_CUDA(cudaEventRecord(D.e1, D.s));
    CA_CUDA(cudaStreamSynchronize(D.s));
    CA_CUDA(cudaEventElapsedTime(&ms, D.e0, D.e1));
    run.st.device_ms += ms;
    run.st.kernel_launches += 2;
    run.st.d2h_bytes += 8;
    const uint64_t items = D.host[0];
    run.st.items += items;
    if (!items) return WHMEC_OK;
    // the windows' buffers: items, their outcomes, the selected calls
    const uint64_t window = std::min<uint64_t>({ca_window(c, run.budget), items, 1ull << 30});
    CA_CUDA(cub::DeviceSelect::If(nullptr, t_sel, (CaCall *)nullptr, (CaCall *)nullptr, (int *)nullptr, (int)window, IsCall(), D.s));
    if (const int rc = ensure_temp(D, t_sel, msg)) return rc;
    if (const int rc = grow(D.win, D.win_bytes, 3 * 256 + window * (sizeof(CaItem) + 2 * sizeof(CaCall)), msg)) return rc;
    p = D.win;
    CaItem *d_items = (CaItem *)take(window * sizeof(CaItem));
    CaCall *d_calls = (CaCall *)take(window * sizeof(CaCall));
    CaCall *d_sel = (CaCall *)take(window * sizeof(CaCall));
    for (uint64_t lo = 0; lo < items; lo += window) {
        const uint64_t hi = std::min(items, lo + window), m = hi - lo;
        CA_CUDA(cudaMemsetAsync(D.scalars, 0xFF, 2 * sizeof(uint64_t), D.s));
        CA_CUDA(cudaMemsetAsync(D.scalars + 2, 0, sizeof(uint64_t), D.s));
        CA_CUDA(cudaEventRecord(D.e0, D.s));
        ca_emit_kernel<<<(na + CA_BLOCK - 1) / CA_BLOCK, CA_BLOCK, 0, D.s>>>(b, na, d_first, lo, hi, d_items);
        CA_CUDA(cudaGetLastError());
        ca_resolve_kernel<<<(uint32_t)((m + CA_BLOCK - 1) / CA_BLOCK), CA_BLOCK, 0, D.s>>>(b, d_items, (uint32_t)m, c.a0, d_calls,
                                                                                            (uint32_t *)(D.scalars + 1), (unsigned long long *)(D.scalars + 2));
        CA_CUDA(cudaGetLastError());
        tb = D.temp_bytes;
        CA_CUDA(cub::DeviceSelect::If(D.temp, tb, d_calls, d_sel, (int *)D.scalars, (int)m, IsCall(), D.s));
        CA_CUDA(cudaEventRecord(D.e1, D.s));
        CA_CUDA(cudaMemcpyAsync(D.host, D.scalars, 3 * sizeof(uint64_t), cudaMemcpyDeviceToHost, D.s));
        CA_CUDA(cudaStreamSynchronize(D.s));
        const uint32_t n_calls = *(uint32_t *)D.host, raised = *(uint32_t *)(D.host + 1);
        run.st.jobs += D.host[2];
        if (n_calls) {
            const size_t w = run.calls.size();
            run.calls.resize(w + n_calls);
            CA_CUDA(cudaMemcpyAsync(run.calls.data() + w, d_sel, (uint64_t)n_calls * sizeof(CaCall), cudaMemcpyDeviceToHost, D.s));
            CA_CUDA(cudaStreamSynchronize(D.s));
        }
        CA_CUDA(cudaEventElapsedTime(&ms, D.e0, D.e1));
        run.st.device_ms += ms;
        run.st.kernel_launches += 3;
        run.st.d2h_bytes += 3 * sizeof(uint64_t) + (uint64_t)n_calls * sizeof(CaCall);
        ++run.st.chunks;
        run.raised = std::min(run.raised, raised);
        if (raised != UMAX) break;  // the chunk's first raising alignment is in this window or an earlier one
    }
    return WHMEC_OK;
}

void ca_close(CaRun &run) {
    CaDev *D = (CaDev *)run.dev;
    if (!D) return;
    if (D->s) cudaStreamSynchronize(D->s);
    cudaFree(D->arena);
    cudaFree(D->win);
    cudaFree(D->temp);
    cudaFree(D->vars);
    cudaFree(D->alleles);
    cudaFree(D->ab);
    cudaFree(D->scalars);
    cudaFreeHost(D->host);
    if (D->e0) cudaEventDestroy(D->e0);
    if (D->e1) cudaEventDestroy(D->e1);
    if (D->s) cudaStreamDestroy(D->s);
    delete D;
    run.dev = nullptr;
}

}  // namespace whmec
