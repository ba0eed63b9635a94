// K-mer pair counts of `whatshap learn` on the GPU (whmec_learn, DESIGN §4.13): the kernels of one chunk and its arena, uploads
// and downloads (ln_run_chunk).  The per-read emit and the reference k-mer are learn.h's, shared with the host emulation.  A chunk
// is: emit every kept k-mer's key, radix-sort the keys over their used bits, run-length encode them, turn each run into a row
// (filtered by the output intervals) and compact the rows.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdlib>
#include <cub/cub.cuh>
#include <string>
#include <vector>

#include "learn_plan.h"
#include "tile.cuh"  // device_available_bytes

namespace whmec {

void install_pinned_staging();  // whmec.cu

namespace {

constexpr uint32_t LN_BLOCK = 128;
constexpr unsigned FULL = 0xFFFFFFFFu;

// An entry writes at most the n_keys keys the plan gave it, from key_off; `bad` is set where the keys disagree with that count.

// one thread per entry of at most LN_SHORT bytes
template <class K>
__global__ void __launch_bounds__(LN_BLOCK) ln_short_kernel(const LnEntry *en, uint32_t n, const LnRead *reads, const LnOp *ops,
                                                            const uint8_t *query, LnRange g, K *keys, uint32_t *bad) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const LnEntry e = en[i];
    if (e.b1 - e.b0 > LN_SHORT) return;
    const LnRead r = reads[e.read];
    if (ln_emit<K>(r, ops + r.op0, query + r.q, e.b0, e.b1, g, keys + e.key_off, e.n_keys) != e.n_keys) *bad = 1;
}

// one warp per longer entry: each lane counts the keys of its share of the bytes, a warp scan gives its offset, then it writes them
template <class K>
__global__ void __launch_bounds__(LN_BLOCK) ln_long_kernel(const LnEntry *en, const uint32_t *list, uint32_t n_list, const LnRead *reads,
                                                           const LnOp *ops, const uint8_t *query, LnRange g, K *keys, uint32_t *bad) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warps = gridDim.x * (blockDim.x / 32);
    for (uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) / 32; w < n_list; w += warps) {
        const LnEntry e = en[list[w]];
        const LnRead r = reads[e.read];
        uint32_t i0, i1;
        ln_lane_span(e.b0, e.b1, lane, i0, i1);
        const uint64_t n = ln_emit<K>(r, ops + r.op0, query + r.q, i0, i1, g, (K *)nullptr, 0);
        uint64_t incl = n;
        for (uint32_t d = 1; d < 32; d *= 2) {
            const uint64_t v = __shfl_up_sync(FULL, (unsigned long long)incl, d);
            if (lane >= d) incl += v;
        }
        const uint64_t before = incl - n;
        ln_emit<K>(r, ops + r.op0, query + r.q, i0, i1, g, keys + e.key_off + before, e.n_keys > before ? e.n_keys - before : 0);
        if (lane == 31 && incl != e.n_keys) *bad = 1;
    }
}

// one thread per run: its row (column, reference k-mer, read k-mer, count) and whether its column is output
template <class K>
__global__ void __launch_bounds__(LN_BLOCK) ln_row_kernel(const K *unique, const uint32_t *counts, uint32_t n_runs, LnRange g, LnRef f,
                                                          const int64_t *iv, uint32_t n_iv, int4 *rows, uint8_t *flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_runs) return;
    const K key = unique[i];
    const int64_t col = g.lo + (int64_t)(key >> (2 * g.k));
    const uint32_t kmer = (uint32_t)(key & (K)((1u << (2 * g.k)) - 1));
    flag[i] = ln_output(iv, n_iv, col);
    rows[i] = make_int4((int)col, (int)ln_ref_kmer(f, col, g.k), (int)kmer, (int)counts[i]);
}

#define LN_CUDA(expr)                                                 \
    do {                                                              \
        cudaError_t _e = (expr);                                      \
        if (_e != cudaSuccess) {                                      \
            msg = std::string(#expr) + ": " + cudaGetErrorString(_e); \
            return WHMEC_ERR_CUDA;                                    \
        }                                                             \
    } while (0)

// per call: the reads, their runs and queries, the reference's codes and the output intervals on the device, a stream, events,
// an arena that grows to the largest chunk and CUB's scratch
struct LnDev {
    cudaStream_t s = nullptr;
    cudaEvent_t e0 = nullptr, e1 = nullptr, e2 = nullptr, e3 = nullptr;  // around the keys' half and the rows' half of a chunk
    uint8_t *query = nullptr;
    LnOp *ops = nullptr;
    LnRead *reads = nullptr;
    uint8_t *code = nullptr;
    uint32_t *base = nullptr, *mask = nullptr;
    int64_t *iv = nullptr;
    uint8_t *arena = nullptr, *temp = nullptr;
    uint64_t arena_bytes = 0, temp_bytes = 0;
    uint32_t *scalars = nullptr;  // [3]: runs, selected rows, an entry whose keys disagree with the plan
    int sms = 0;
};

uint64_t align_up(uint64_t b) { return (b + 255) / 256 * 256; }

template <class T>
int upload(LnDev &D, LnCall &call, T *&dst, const T *src, uint64_t n, std::string &msg) {
    LN_CUDA(cudaMalloc(&dst, std::max<uint64_t>(n, 1) * sizeof(T)));
    if (n) LN_CUDA(cudaMemcpyAsync(dst, src, n * sizeof(T), cudaMemcpyHostToDevice, D.s));
    call.st.h2d_bytes += n * sizeof(T);
    return WHMEC_OK;
}

template <class K>
int run(LnCall &call, const LnChunk &c, LnDev &D, std::string &msg) {
    const uint32_t ne = c.e1 - c.e0, n = (uint32_t)c.n_keys;
    std::vector<uint32_t> list;  // the chunk's warp entries
    for (uint32_t i = c.e0; i < c.e1; ++i)
        if (call.entries[i].b1 - call.entries[i].b0 > LN_SHORT) list.push_back(i - c.e0);
    uint8_t *p = D.arena;
    auto take = [&p](uint64_t bytes) {
        uint8_t *r = p;
        p += align_up(bytes);
        return r;
    };
    // the arena as LN_KEY_BYTES counts it: entries, warp list, two key buffers, the runs, their counts, the rows and their flags
    LnEntry *d_en = (LnEntry *)take(ne * sizeof(LnEntry));
    uint32_t *d_list = (uint32_t *)take(ne * 4);
    K *d_a = (K *)take(n * sizeof(K)), *d_b = (K *)take(n * sizeof(K)), *d_unique = (K *)take(n * sizeof(K));
    uint32_t *d_counts = (uint32_t *)take(n * 4);
    int4 *d_rows = (int4 *)take(n * 16), *d_sel = (int4 *)take(n * 16);
    uint8_t *d_flag = take(n);
    LN_CUDA(cudaMemcpyAsync(d_en, call.entries.data() + c.e0, ne * sizeof(LnEntry), cudaMemcpyHostToDevice, D.s));
    if (!list.empty()) LN_CUDA(cudaMemcpyAsync(d_list, list.data(), list.size() * 4, cudaMemcpyHostToDevice, D.s));
    call.st.h2d_bytes += ne * sizeof(LnEntry) + list.size() * 4;
    const LnRange g{c.lo, c.hi, call.k};
    uint32_t bits = 2 * call.k;
    while (bits < 8 * sizeof(K) && (uint64_t)(c.hi - c.lo) >> (bits - 2 * call.k)) ++bits;
    cub::DoubleBuffer<K> db(d_a, d_b);
    size_t t_sort = 0, t_rle = 0, t_sel = 0;
    LN_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, t_sort, db, (int)n, 0, (int)bits, D.s));
    LN_CUDA(cub::DeviceRunLengthEncode::Encode(nullptr, t_rle, d_a, d_unique, d_counts, D.scalars, (int)n, D.s));
    LN_CUDA(cub::DeviceSelect::Flagged(nullptr, t_sel, d_rows, d_flag, d_sel, D.scalars + 1, (int)n, D.s));
    const uint64_t t_need = std::max({t_sort, t_rle, t_sel, (size_t)1});
    if (D.temp_bytes < t_need) {
        if (D.temp) LN_CUDA(cudaFree(D.temp));
        D.temp = nullptr;
        LN_CUDA(cudaMalloc(&D.temp, t_need));
        D.temp_bytes = t_need;
    }
    LN_CUDA(cudaMemsetAsync(D.scalars, 0, 12, D.s));
    LN_CUDA(cudaEventRecord(D.e0, D.s));
    ln_short_kernel<K><<<(ne + LN_BLOCK - 1) / LN_BLOCK, LN_BLOCK, 0, D.s>>>(d_en, ne, D.reads, D.ops, D.query, g, d_a, D.scalars + 2);
    LN_CUDA(cudaGetLastError());
    ++call.st.kernel_launches;
    if (!list.empty()) {
        const uint32_t per_block = LN_BLOCK / 32;
        const uint32_t grid = (uint32_t)std::min<uint64_t>((list.size() + per_block - 1) / per_block, 64ull * D.sms);
        ln_long_kernel<K><<<grid, LN_BLOCK, 0, D.s>>>(d_en, d_list, (uint32_t)list.size(), D.reads, D.ops, D.query, g, d_a, D.scalars + 2);
        LN_CUDA(cudaGetLastError());
        ++call.st.kernel_launches;
    }
    size_t tb = D.temp_bytes;
    LN_CUDA(cub::DeviceRadixSort::SortKeys(D.temp, tb, db, (int)n, 0, (int)bits, D.s));
    tb = D.temp_bytes;
    LN_CUDA(cub::DeviceRunLengthEncode::Encode(D.temp, tb, db.Current(), d_unique, d_counts, D.scalars, (int)n, D.s));
    call.st.kernel_launches += 2;
    LN_CUDA(cudaEventRecord(D.e1, D.s));
    uint32_t sc[3] = {0, 0, 0};
    LN_CUDA(cudaMemcpyAsync(sc, D.scalars, 12, cudaMemcpyDeviceToHost, D.s));
    LN_CUDA(cudaStreamSynchronize(D.s));
    if (sc[2]) {
        msg = "whmec_learn: a read's keys disagree with the plan's count (internal error)";
        return WHMEC_ERR_CUDA;
    }
    const uint32_t runs = sc[0];
    LN_CUDA(cudaEventRecord(D.e2, D.s));
    const LnRef f{D.code, D.base, D.mask, call.b0};
    ln_row_kernel<K><<<(runs + LN_BLOCK - 1) / LN_BLOCK, LN_BLOCK, 0, D.s>>>(d_unique, d_counts, runs, g, f, D.iv, (uint32_t)(call.iv.size() / 2),
                                                                            d_rows, d_flag);
    LN_CUDA(cudaGetLastError());
    tb = D.temp_bytes;
    LN_CUDA(cub::DeviceSelect::Flagged(D.temp, tb, d_rows, d_flag, d_sel, D.scalars + 1, (int)runs, D.s));
    call.st.kernel_launches += 2;
    LN_CUDA(cudaEventRecord(D.e3, D.s));
    uint32_t sel = 0;
    LN_CUDA(cudaMemcpyAsync(&sel, D.scalars + 1, 4, cudaMemcpyDeviceToHost, D.s));
    LN_CUDA(cudaStreamSynchronize(D.s));
    const size_t at = call.rows.size();
    call.rows.resize(at + 4 * (size_t)sel);
    if (sel) LN_CUDA(cudaMemcpyAsync(call.rows.data() + at, d_sel, (size_t)sel * 16, cudaMemcpyDeviceToHost, D.s));
    LN_CUDA(cudaStreamSynchronize(D.s));
    call.st.d2h_bytes += 16 + (uint64_t)sel * 16;
    call.st.distinct += runs;
    float ms = 0, ms2 = 0;  // the host's read of the run count between the halves is not device time
    LN_CUDA(cudaEventElapsedTime(&ms, D.e0, D.e1));
    LN_CUDA(cudaEventElapsedTime(&ms2, D.e2, D.e3));
    call.st.device_ms += ms + ms2;
    return WHMEC_OK;
}

}  // namespace

uint64_t ln_budget(int device, std::string &msg) {
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e == cudaSuccess && (device < 0 || device >= count)) e = cudaErrorInvalidDevice;
    if (e == cudaSuccess) e = cudaSetDevice(device);
    if (e != cudaSuccess) {
        msg = std::string("whmec_learn: ") + cudaGetErrorString(e);
        return 0;
    }
    install_pinned_staging();
    const uint64_t free_b = device_available_bytes(), margin = 512ull << 20;
    uint64_t budget = free_b > margin ? free_b - margin : 0;
    // WHMEC_LEARN_ARENA_BUDGET=bytes (test hook): the device bytes a call may take
    if (const char *h = std::getenv("WHMEC_LEARN_ARENA_BUDGET")) budget = std::min<uint64_t>(budget, std::strtoull(h, nullptr, 10));
    return budget;
}

int ln_run_chunk(int device, LnCall &call, const LnChunk &c, std::string &msg) {
    if (!call.dev) call.dev = new LnDev();
    LnDev &D = *(LnDev *)call.dev;
    LN_CUDA(cudaSetDevice(device));
    if (!D.s) {
        LN_CUDA(cudaDeviceGetAttribute(&D.sms, cudaDevAttrMultiProcessorCount, device));
        LN_CUDA(cudaStreamCreateWithFlags(&D.s, cudaStreamNonBlocking));
        LN_CUDA(cudaEventCreate(&D.e0));
        LN_CUDA(cudaEventCreate(&D.e1));
        LN_CUDA(cudaEventCreate(&D.e2));
        LN_CUDA(cudaEventCreate(&D.e3));
        LN_CUDA(cudaMalloc(&D.scalars, 12));
        int rc = WHMEC_OK;
        if ((rc = upload(D, call, D.query, call.query, call.query_bytes, msg)) || (rc = upload(D, call, D.ops, call.ops, call.n_ops, msg)) ||
            (rc = upload(D, call, D.reads, call.reads, call.n_reads, msg)) ||
            (rc = upload(D, call, D.code, call.code.data(), call.code.size(), msg)) ||
            (rc = upload(D, call, D.base, call.base.data(), call.base.size(), msg)) ||
            (rc = upload(D, call, D.mask, call.mask.data(), call.mask.size(), msg)) ||
            (rc = upload(D, call, D.iv, call.iv.data(), call.iv.size(), msg)))
            return rc;
    }
    const uint64_t ne = c.e1 - c.e0, n = c.n_keys, ks = c.wide ? 8 : 4;
    const uint64_t need = align_up(ne * sizeof(LnEntry)) + align_up(ne * 4) + 3 * align_up(n * ks) + align_up(n * 4) + 2 * align_up(n * 16) +
                          align_up(n);
    if (D.arena_bytes < need) {
        if (D.arena) LN_CUDA(cudaFree(D.arena));
        D.arena = nullptr;
        LN_CUDA(cudaMalloc(&D.arena, need));
        D.arena_bytes = need;
    }
    return c.wide ? run<uint64_t>(call, c, D, msg) : run<uint32_t>(call, c, D, msg);
}

void ln_close(LnCall &call) {
    LnDev *D = (LnDev *)call.dev;
    if (!D) return;
    if (D->s) cudaStreamSynchronize(D->s);
    for (void *p : {(void *)D->query, (void *)D->ops, (void *)D->reads, (void *)D->code, (void *)D->base, (void *)D->mask, (void *)D->iv,
                    (void *)D->arena, (void *)D->temp, (void *)D->scalars})
        cudaFree(p);
    for (cudaEvent_t e : {D->e0, D->e1, D->e2, D->e3})
        if (e) cudaEventDestroy(e);
    if (D->s) cudaStreamDestroy(D->s);
    delete D;
    call.dev = nullptr;
}

}  // namespace whmec
