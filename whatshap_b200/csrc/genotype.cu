// whmec_genotype: forward-backward genotype likelihoods (the reference's GenotypeDPTable,
// src/genotypedptable.cpp) on the device.  Sibling DP of the MEC sweep (SURVEY.md 8(f) rank 4): same packer,
// same column / projection structure, sums of products in double precision instead of u32 min-plus.
//
// One thread per DP cell (bipartition x of a column); a cell adds its contribution to the projection entry it
// maps to with a double-precision atomicAdd (several cells share an entry when reads end / start in the column).
// Per step: backward pass  gl_backward_kernel + gl_scale_kernel,  forward pass  gl_forward_kernel + gl_scale_kernel;
// one launch advances every table of a group by one column (gl_schedule, gl_pack.cpp): for a single individual the
// DP-independent chains are tables of their own, so the launch count is 4 x (longest chain), not 4 x (columns).
// The backward tables of all columns of a group stay in HBM.  A table whose backward tables do not fit runs alone in
// memory-bounded mode (gl_bounded, DESIGN §4.5): its columns are cut into segments that share one arena, and every
// segment but the first is swept backward again from a checkpoint before its forward steps (the reference keeps every
// sqrt(n)-th column and recomputes, genotypedptable.cpp:139-166,326-343).
// A pedigree table can also be split into segments of whole chains, one per GPU (whmec_genotype_segment_*, DESIGN §4.5): a
// forward-only transfer pass per segment (gl_transfer_kernel) gives the T x T matrix that carries the T values across the
// cut, the caller folds the matrices, and each segment runs the passes above from its true inputs.
// Many tables in one call (whmec_genotype_batch, DESIGN §4.9): the sub-tables of every table of a group (a single individual's
// chains, a pedigree's whole table) share one step list, swept by gl_batch_backward_kernel / gl_batch_forward_kernel, which read
// each step's table from a descriptor (gl_batch.h), and the same gl_scale_kernel.
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <vector>

#include "gl_batch.h"
#include "gl_pack.h"
#include "tile.cuh"  // device_available_bytes

using namespace whmec;

namespace {

#define CUDA_TRY(expr)                                                    \
    do {                                                                  \
        cudaError_t _e = (expr);                                          \
        if (_e != cudaSuccess) {                                          \
            msg = std::string(#expr) + ": " + cudaGetErrorString(_e);     \
            return WHMEC_ERR_CUDA;                                        \
        }                                                                 \
    } while (0)

constexpr int GL_THREADS = 256;

struct AtomicAdd {
    __device__ void operator()(double *addr, double v) const { atomicAdd(addr, v); }
};

// grid.y = the tables advanced by this launch (GlStep each); grid.x covers the widest column among them
__global__ void __launch_bounds__(GL_THREADS) gl_backward_kernel(GlView v, const GlStep *steps, double *beta, uint64_t beta_base) {
    const GlStep st = steps[blockIdx.y];
    const uint64_t x = (uint64_t)blockIdx.x * GL_THREADS + threadIdx.x;
    if (x >= ((uint64_t)1 << st.cells_log2)) return;
    gl_backward_cell(v, st.k, (uint32_t)x, beta + (v.cols[st.k].beta_off - beta_base), beta + st.cur_off, AtomicAdd());
}

// lacc: [n_cols][n_ind * 3] posterior accumulators
__global__ void __launch_bounds__(GL_THREADS) gl_forward_kernel(GlView v, const GlStep *steps, double *F, const double *beta, uint64_t beta_base,
                                                                double *lacc_out) {
    __shared__ double s_acc[GL_MAX_IND * 3];
    const GlStep st = steps[blockIdx.y];
    if ((uint64_t)blockIdx.x * GL_THREADS >= ((uint64_t)1 << st.cells_log2)) return;  // whole block beyond this column (uniform)
    const uint32_t n_acc = v.n_ind * 3;
    if (threadIdx.x < n_acc) s_acc[threadIdx.x] = 0.0;
    __syncthreads();
    double lacc[GL_MAX_IND * 3];
    for (uint32_t e = 0; e < n_acc; ++e) lacc[e] = 0.0;
    const uint64_t x = (uint64_t)blockIdx.x * GL_THREADS + threadIdx.x;
    if (x < ((uint64_t)1 << st.cells_log2))
        gl_forward_cell(v, st.k, (uint32_t)x, F + st.prev_off, F + st.cur_off, beta + (v.cols[st.k].beta_off - beta_base), lacc, AtomicAdd());
    for (uint32_t e = 0; e < n_acc; ++e) {
        double s = lacc[e];
        for (int off = 16; off > 0; off >>= 1) s += __shfl_down_sync(0xFFFFFFFFu, s, off);
        if ((threadIdx.x & 31) == 0 && s != 0.0) atomicAdd(&s_acc[e], s);
    }
    __syncthreads();
    if (threadIdx.x < n_acc && s_acc[threadIdx.x] != 0.0) atomicAdd(&lacc_out[(size_t)st.k * n_acc + threadIdx.x], s_acc[threadIdx.x]);
}

// One block per table of the launch: divides the finished projection column (pool + cur_off, n_scale entries) by its
// largest entry (gl_scale_host) and clears the buffer the table's next column accumulates into (pool + prev_off).
__global__ void __launch_bounds__(1024) gl_scale_kernel(const GlStep *steps, double *pool) {
    __shared__ double s_max[32];
    const GlStep st = steps[blockIdx.x];
    double *v = pool + st.cur_off;
    const uint64_t n = st.n_scale;
    double mx = 0.0;
    for (uint64_t i = threadIdx.x; i < n; i += blockDim.x) mx = fmax(mx, v[i]);
    for (int off = 16; off > 0; off >>= 1) mx = fmax(mx, __shfl_down_sync(0xFFFFFFFFu, mx, off));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
        mx = threadIdx.x < (blockDim.x >> 5) ? s_max[threadIdx.x] : 0.0;
        for (int off = 16; off > 0; off >>= 1) mx = fmax(mx, __shfl_down_sync(0xFFFFFFFFu, mx, off));
        if (threadIdx.x == 0) s_max[0] = mx;
    }
    __syncthreads();
    mx = s_max[0];
    if (mx > 0.0) {
        const double inv = 1.0 / mx;
        for (uint64_t i = threadIdx.x; i < n; i += blockDim.x) v[i] *= inv;
    }
    double *c = pool + st.prev_off;
    for (uint64_t i = threadIdx.x; i < st.n_clear; i += blockDim.x) c[i] = 0.0;
}

// A group of whmec_genotype_batch (gl_batch_plan): grid.y = the steps of this launch, each of its own table (tables[step_table[y]]:
// singles, trios and larger pedigrees share a launch; a CTA never mixes tables); grid.x covers the widest column among them.
// The cells are those of gl_backward_kernel / gl_forward_kernel on the table's view of the group's concatenated inputs.
__global__ void __launch_bounds__(GL_THREADS) gl_batch_backward_kernel(GlBatchInputs in, const GlBatchTable *tables, const GlStep *steps,
                                                                       const uint32_t *step_table, double *beta) {
    const GlStep st = steps[blockIdx.y];
    const uint64_t x = (uint64_t)blockIdx.x * GL_THREADS + threadIdx.x;
    if (x >= ((uint64_t)1 << st.cells_log2)) return;
    const GlBatchTable d = tables[step_table[blockIdx.y]];
    const GlView v = gl_batch_view(in, d);
    gl_backward_cell(v, st.k, (uint32_t)x, beta + d.beta_base + v.cols[st.k].beta_off, beta + st.cur_off, AtomicAdd());
}

// acc: every table's posterior accumulators, [n_cols][n_ind * 3] from its acc_base
__global__ void __launch_bounds__(GL_THREADS) gl_batch_forward_kernel(GlBatchInputs in, const GlBatchTable *tables, const GlStep *steps,
                                                                      const uint32_t *step_table, double *F, const double *beta, double *acc) {
    __shared__ double s_acc[GL_MAX_IND * 3];
    const GlStep st = steps[blockIdx.y];
    if ((uint64_t)blockIdx.x * GL_THREADS >= ((uint64_t)1 << st.cells_log2)) return;  // whole block beyond this column (uniform)
    const GlBatchTable d = tables[step_table[blockIdx.y]];
    const GlView v = gl_batch_view(in, d);
    const uint32_t n_acc = v.n_ind * 3;
    const double *beta_k = beta + d.beta_base + v.cols[st.k].beta_off;
    double *acc_k = acc + d.acc_base + (size_t)st.k * n_acc;
    if (threadIdx.x < n_acc) s_acc[threadIdx.x] = 0.0;
    __syncthreads();
    double lacc[GL_MAX_IND * 3];
    for (uint32_t e = 0; e < n_acc; ++e) lacc[e] = 0.0;
    const uint64_t x = (uint64_t)blockIdx.x * GL_THREADS + threadIdx.x;
    if (x < ((uint64_t)1 << st.cells_log2))
        gl_forward_cell(v, st.k, (uint32_t)x, F + st.prev_off, F + st.cur_off, beta_k, lacc, AtomicAdd());
    for (uint32_t e = 0; e < n_acc; ++e) {
        double s = lacc[e];
        for (int off = 16; off > 0; off >>= 1) s += __shfl_down_sync(0xFFFFFFFFu, s, off);
        if ((threadIdx.x & 31) == 0 && s != 0.0) atomicAdd(&s_acc[e], s);
    }
    __syncthreads();
    if (threadIdx.x < n_acc && s_acc[threadIdx.x] != 0.0) atomicAdd(&acc_k[threadIdx.x], s_acc[threadIdx.x]);
}

// Transfer pass of a segment (gl_transfer_plan): one column for the n_in input rows of a batch.  grid.x covers the column.
__global__ void __launch_bounds__(GL_THREADS) gl_transfer_kernel(GlView v, const GlStep *step, double *F, uint32_t n_in) {
    const GlStep st = *step;
    const uint64_t x = (uint64_t)blockIdx.x * GL_THREADS + threadIdx.x;
    if (x >= ((uint64_t)1 << st.cells_log2)) return;
    gl_transfer_cell(v, st.k, (uint32_t)x, n_in, F + st.prev_off, F + st.cur_off, AtomicAdd());
}

// Writes the largest entry of the finished column (pool + cur_off, n_scale entries; 0 when all are 0) to *col_max, before
// gl_scale_kernel divides by it: the transfer pass of a segment with several batches puts their rows on one scale with these
// (gl_transfer_combine).
__global__ void __launch_bounds__(1024) gl_column_max_kernel(const GlStep *step, const double *pool, double *col_max) {
    __shared__ double s_max[32];
    const GlStep st = *step;
    const double *v = pool + st.cur_off;
    double mx = 0.0;
    for (uint64_t i = threadIdx.x; i < st.n_scale; i += blockDim.x) mx = fmax(mx, v[i]);
    for (int off = 16; off > 0; off >>= 1) mx = fmax(mx, __shfl_down_sync(0xFFFFFFFFu, mx, off));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x < 32) {
        mx = threadIdx.x < (blockDim.x >> 5) ? s_max[threadIdx.x] : 0.0;
        for (int off = 16; off > 0; off >>= 1) mx = fmax(mx, __shfl_down_sync(0xFFFFFFFFu, mx, off));
        if (threadIdx.x == 0) *col_max = mx;
    }
}

struct Buffers {  // freed on every exit path
    cudaStream_t stream = nullptr;
    bool owns_stream = true;  // false: the stream belongs to a longer-lived Buffers
    std::vector<void *> ptrs;
    template <class Tp>
    cudaError_t alloc(Tp **p, size_t count) {
        cudaError_t e = cudaMallocAsync((void **)p, std::max<size_t>(count, 1) * sizeof(Tp), stream);
        if (e == cudaSuccess) ptrs.push_back((void *)*p);
        return e;
    }
    ~Buffers() {
        for (void *p : ptrs) cudaFreeAsync(p, stream);
        if (stream) {
            cudaStreamSynchronize(stream);
            if (owns_stream) cudaStreamDestroy(stream);
        }
    }
};

// The packed problem in HBM: per-column records, error probabilities, alleles, pedigree indices, transition and prior tables.
int upload_inputs(Buffers &B, const Packed &pk, const GlPacked &g, GlView &v, uint64_t &h2d, std::string &msg) {
    const uint32_t n = pk.n;
    cudaStream_t s = B.stream;
    GlCol *d_cols = nullptr;
    double *d_eps = nullptr, *d_trans = nullptr, *d_q = nullptr;
    uint8_t *d_allele = nullptr, *d_ind = nullptr;
    int8_t *d_h2p = nullptr;
    CUDA_TRY(B.alloc(&d_cols, n));
    CUDA_TRY(B.alloc(&d_eps, g.eps.size()));
    CUDA_TRY(B.alloc(&d_allele, pk.act_allele.size()));
    CUDA_TRY(B.alloc(&d_ind, pk.act_ind.size()));
    CUDA_TRY(B.alloc(&d_h2p, pk.h2p.size()));
    CUDA_TRY(B.alloc(&d_trans, g.trans.size()));
    CUDA_TRY(B.alloc(&d_q, g.q.size()));
    auto up = [&](void *dst, const void *src, size_t bytes) {
        h2d += bytes;
        return bytes ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s) : cudaSuccess;
    };
    CUDA_TRY(up(d_cols, g.cols.data(), (size_t)n * sizeof(GlCol)));
    CUDA_TRY(up(d_eps, g.eps.data(), g.eps.size() * 8));
    CUDA_TRY(up(d_allele, pk.act_allele.data(), pk.act_allele.size()));
    CUDA_TRY(up(d_ind, pk.act_ind.data(), pk.act_ind.size()));
    CUDA_TRY(up(d_h2p, pk.h2p.data(), pk.h2p.size()));
    CUDA_TRY(up(d_trans, g.trans.data(), g.trans.size() * 8));
    CUDA_TRY(up(d_q, g.q.data(), g.q.size() * 8));
    v = GlView{d_cols, d_eps, d_allele, d_ind, d_h2p, d_trans, d_q, pk.T, pk.P, pk.n_ind};
    return WHMEC_OK;
}

// Bytes the inputs above and the per-call arrays take; the budget for backward tables + projection buffers is what remains of
// the free HBM (or WHMEC_GENOTYPE_ARENA_BUDGET, whichever is smaller), in doubles.
int work_budget(const Packed &pk, const GlPacked &g, uint64_t &budget, std::string &msg) {
    const uint32_t n = pk.n, n_ind = pk.n_ind;
    const size_t free_b = device_available_bytes();
    const uint64_t fixed = (uint64_t)n * sizeof(GlCol) + g.eps.size() * 10 + (g.trans.size() + g.q.size()) * 8 + (uint64_t)n * sizeof(GlStep) * 2 +
                           (uint64_t)n * n_ind * 3 * 8 + (512ull << 20);
    if (fixed > free_b) {
        msg = "genotyping: problem exceeds the free HBM of this device";
        return WHMEC_ERR_UNSUPPORTED;
    }
    budget = (free_b - fixed) / 8;  // doubles available for backward tables + projection buffers
    // WHMEC_GENOTYPE_ARENA_BUDGET=bytes (test hook): the budget for backward tables, checkpoints and projection buffers
    if (const char *e = std::getenv("WHMEC_GENOTYPE_ARENA_BUDGET")) budget = std::min<uint64_t>(budget, std::strtoull(e, nullptr, 10) / 8);
    return WHMEC_OK;
}

// Runs the units of gl_plan on stream s, accumulating the posteriors into d_acc ([n_cols][n_ind * 3]).  d_work holds the largest
// unit's work_doubles (per unit: its backward store, then its projection buffers), d_steps its step list.  A segment of a table
// passes alpha_in / beta_in (T doubles each, or null), which go where the unit's plan says (GlUnit::alpha_at, beta_at).
int run_units(cudaStream_t s, const GlView &v, const std::vector<GlUnit> &units, const double *alpha_in, const double *beta_in, double *d_work,
              GlStep *d_steps, double *d_acc, uint32_t &launches, uint64_t &h2d, std::string &msg) {
    auto up = [&](void *dst, const void *src, size_t bytes) {
        h2d += bytes;
        return bytes ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s) : cudaSuccess;
    };
    auto inputs = [&](const GlUnit &u) {  // after the unit's buffers are cleared
        cudaError_t e = cudaSuccess;
        if (alpha_in) e = up(d_work + u.alpha_at, alpha_in, (size_t)v.T * 8);
        if (e == cudaSuccess && beta_in) e = up(d_work + u.beta_at, beta_in, (size_t)v.T * 8);
        return e;
    };
    constexpr uint32_t MAX_GRID_Y = 65535;
    for (size_t q = 0; q < units.size(); ++q) {
        if (q > 0) CUDA_TRY(cudaStreamSynchronize(s));  // the step list of the previous unit is still being read
        if (units[q].bounded) {
            const GlBounded &bd = units[q].bd;
            const uint64_t store = bd.arena_doubles + bd.ckpt_doubles;
            double *d_beta = d_work, *d_F = d_work + store;
            CUDA_TRY(up(d_steps, bd.steps.data(), bd.steps.size() * sizeof(GlStep)));
            CUDA_TRY(cudaMemsetAsync(d_work, 0, (store + bd.f_pool_doubles) * 8, s));
            CUDA_TRY(inputs(units[q]));
            auto blocks = [&](uint32_t e) { return (unsigned)((((uint64_t)1 << bd.steps[e].cells_log2) + GL_THREADS - 1) / GL_THREADS); };
            for (const GlSweep &sw : bd.sweeps) {
                if (sw.clear) CUDA_TRY(cudaMemsetAsync(d_beta, 0, sw.clear * 8, s));
                if (sw.copy_n) CUDA_TRY(cudaMemcpyAsync(d_beta + sw.copy_dst, d_beta + sw.copy_src, sw.copy_n * 8, cudaMemcpyDeviceToDevice, s));
                for (uint32_t e = sw.bwd_begin; e < sw.bwd_end; ++e) {
                    gl_backward_kernel<<<blocks(e), GL_THREADS, 0, s>>>(v, d_steps + e, d_beta, sw.beta_base);
                    gl_scale_kernel<<<1, 1024, 0, s>>>(d_steps + e, d_beta);
                    launches += 2;
                }
                for (uint32_t e = sw.fwd_begin; e < sw.fwd_end; ++e) {
                    gl_forward_kernel<<<blocks(e), GL_THREADS, 0, s>>>(v, d_steps + e, d_F, d_beta, sw.beta_base, d_acc);
                    gl_scale_kernel<<<1, 1024, 0, s>>>(d_steps + e, d_F);
                    launches += 2;
                }
            }
            continue;
        }
        const GlSchedule &sc = units[q].sc;
        double *d_beta = d_work, *d_F = d_work + sc.beta_doubles + 1;
        CUDA_TRY(up(d_steps, sc.steps.data(), sc.steps.size() * sizeof(GlStep)));
        CUDA_TRY(cudaMemsetAsync(d_beta, 0, (sc.beta_doubles + 1) * 8, s));
        CUDA_TRY(cudaMemsetAsync(d_F, 0, sc.f_pool_doubles * 8, s));
        CUDA_TRY(inputs(units[q]));
        auto widest = [&](uint32_t e0, uint32_t e1) {
            uint32_t a_max = 0;
            for (uint32_t e = e0; e < e1; ++e) a_max = std::max(a_max, sc.steps[e].cells_log2);
            return (unsigned)((((uint64_t)1 << a_max) + GL_THREADS - 1) / GL_THREADS);
        };
        for (size_t l = 0; l + 1 < sc.bwd_begin.size(); ++l)
            for (uint32_t e0 = sc.bwd_begin[l]; e0 < sc.bwd_begin[l + 1]; e0 += MAX_GRID_Y) {
                const uint32_t e1 = std::min(sc.bwd_begin[l + 1], e0 + MAX_GRID_Y);
                gl_backward_kernel<<<dim3(widest(e0, e1), e1 - e0), GL_THREADS, 0, s>>>(v, d_steps + e0, d_beta, sc.beta_base);
                gl_scale_kernel<<<e1 - e0, 1024, 0, s>>>(d_steps + e0, d_beta);
                launches += 2;
            }
        for (size_t l = 0; l + 1 < sc.fwd_begin.size(); ++l)
            for (uint32_t e0 = sc.fwd_begin[l]; e0 < sc.fwd_begin[l + 1]; e0 += MAX_GRID_Y) {
                const uint32_t e1 = std::min(sc.fwd_begin[l + 1], e0 + MAX_GRID_Y);
                gl_forward_kernel<<<dim3(widest(e0, e1), e1 - e0), GL_THREADS, 0, s>>>(v, d_steps + e0, d_F, d_beta, sc.beta_base, d_acc);
                gl_scale_kernel<<<e1 - e0, 1024, 0, s>>>(d_steps + e0, d_F);
                launches += 2;
            }
    }
    return WHMEC_OK;
}

struct Timer {  // CUDA events around the work enqueued between start() and stop()
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    ~Timer() {
        if (ev0) cudaEventDestroy(ev0);
        if (ev1) cudaEventDestroy(ev1);
    }
    cudaError_t start(cudaStream_t s) {
        cudaError_t e = cudaEventCreate(&ev0);
        if (e == cudaSuccess) e = cudaEventCreate(&ev1);
        return e == cudaSuccess ? cudaEventRecord(ev0, s) : e;
    }
};

int open_device(int device, std::string &msg) {
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
        msg = "no CUDA device (whatshap_b200 has no CPU path)";
        return WHMEC_ERR_CUDA;
    }
    CUDA_TRY(cudaSetDevice(device));
    return WHMEC_OK;
}

// Groups of tables or bounded tables (gl_plan) of one packed problem on the device, posteriors normalised into `likelihoods`.
// Shared by whmec_genotype (alpha_in = beta_in = null) and whmec_genotype_segment_run.
int run_packed(Buffers &B, const Packed &pk, const GlPacked &g, const GlView &v, uint64_t budget, const double *alpha_in, const double *beta_in,
               double *likelihoods, whmec_stats *st, uint64_t h2d, std::string &msg) {
    const uint32_t n = pk.n, n_ind = pk.n_ind;
    cudaStream_t s = B.stream;
    // groups of tables on launch schedules (one launch advances every table of a group by one column); a table whose
    // backward tables do not fit runs alone in memory-bounded mode (gl_bounded)
    std::vector<GlUnit> units;
    int rc = gl_plan(g, pk.T, budget, units, msg);
    if (rc != WHMEC_OK) return rc;
    uint64_t max_work = 1, max_steps = 1, max_store = 0;  // max_store: the largest backward store of a unit (doubles)
    bool bounded = false;
    for (const GlUnit &u : units) {
        max_work = std::max(max_work, u.work_doubles);
        max_steps = std::max<uint64_t>(max_steps, u.bounded ? u.bd.steps.size() : u.sc.steps.size());
        max_store = std::max(max_store, u.bounded ? u.bd.arena_doubles + u.bd.ckpt_doubles : u.sc.beta_doubles);
        bounded = bounded || u.bounded;
    }
    Buffers W;  // this call's buffers, on the same stream, allocated before the timed region
    W.stream = s;
    W.owns_stream = false;
    double *d_work = nullptr, *d_acc = nullptr;
    GlStep *d_steps = nullptr;
    CUDA_TRY(W.alloc(&d_work, max_work));
    CUDA_TRY(W.alloc(&d_steps, max_steps));
    CUDA_TRY(W.alloc(&d_acc, (size_t)n * n_ind * 3));
    CUDA_TRY(cudaMemsetAsync(d_acc, 0, (size_t)n * n_ind * 3 * 8, s));
    Timer tm;
    CUDA_TRY(tm.start(s));
    uint32_t launches = 0;
    rc = run_units(s, v, units, alpha_in, beta_in, d_work, d_steps, d_acc, launches, h2d, msg);
    if (rc != WHMEC_OK) return rc;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaEventRecord(tm.ev1, s));
    std::vector<double> acc((size_t)n * n_ind * 3);
    CUDA_TRY(cudaMemcpyAsync(acc.data(), d_acc, acc.size() * 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    float ms = 0.f;
    CUDA_TRY(cudaEventElapsedTime(&ms, tm.ev0, tm.ev1));
    gl_normalise(acc.data(), n, n_ind, likelihoods);
    if (st) {
        *st = pk.stats;
        st->kernel_launches = launches;
        st->sweep_ms = ms;
        st->h2d_bytes = h2d;
        st->d2h_bytes = acc.size() * 8;
        // here: bytes of backward tables kept in HBM; with a table in bounded mode, the largest store allocated for them
        // (arena + checkpoints of a bounded table, the backward tables of a group)
        st->backptr_bytes = bounded ? max_store * 8 : g.beta_doubles * 8;
        st->path_kind = 4;
    }
    return WHMEC_OK;
}

int genotype_impl(const whmec_problem *p, double *likelihoods, int device, whmec_stats *st, std::string &msg) {
    if (!p || !likelihoods) {
        msg = "null argument";
        return WHMEC_ERR_INPUT;
    }
    Packed pk;
    GlPacked g;
    int rc = gl_pack(p, pk, g, msg);
    if (rc != WHMEC_OK) return rc;
    if (st) *st = pk.stats;
    if (pk.n == 0) return WHMEC_OK;
    rc = open_device(device, msg);
    if (rc != WHMEC_OK) return rc;
    Buffers B;
    CUDA_TRY(cudaStreamCreateWithFlags(&B.stream, cudaStreamNonBlocking));
    uint64_t budget = 0;
    rc = work_budget(pk, g, budget, msg);
    if (rc != WHMEC_OK) return rc;
    uint64_t h2d = 0;
    GlView v{};
    rc = upload_inputs(B, pk, g, v, h2d, msg);
    if (rc != WHMEC_OK) return rc;
    return run_packed(B, pk, g, v, budget, nullptr, nullptr, likelihoods, st, h2d, msg);
}

template <class F>
int guarded(F &&fn, char *err, size_t errlen) {
    std::string msg;
    int rc;
    try {
        rc = fn(msg);
    } catch (const std::exception &e) {  // no C++ exception crosses the C boundary
        msg = e.what();
        rc = WHMEC_ERR_INPUT;
    }
    if (rc != WHMEC_OK && err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = 0;
    }
    return rc;
}

void set_err(char *err, size_t errlen, const std::string &msg) {
    if (err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = 0;
    }
}

void add_stats(whmec_stats &total, const whmec_stats &st) {
    total.cells += st.cells;
    total.algorithmic_bytes += st.algorithmic_bytes;
    total.backptr_bytes += st.backptr_bytes;
    total.kernel_launches += st.kernel_launches;
    total.n_chains += st.n_chains;
    total.max_active = std::max(total.max_active, st.max_active);
    total.transmissions = std::max(total.transmissions, st.transmissions);
    total.sweep_ms += st.sweep_ms;
    total.h2d_bytes += st.h2d_bytes;
    total.d2h_bytes += st.d2h_bytes;
    total.path_kind = 4;
}

// One group of whmec_genotype_batch on stream s: one upload (concatenated inputs, descriptors, step list), one clear of the work
// buffer (backward store, F pool, accumulators), the launches of the group's step list, one copy of every member's posteriors
// back, each normalised into its caller's array.
int run_batch_group(cudaStream_t s, const GlBatchGroup &gp, const std::vector<Packed> &pks, const std::vector<GlPacked> &gs, double *const *likelihoods,
                    whmec_stats *stats, whmec_stats &total, std::string &msg) {
    std::vector<uint8_t> blob;
    auto put = [&](const void *src, size_t bytes) {  // 16-byte aligned sections
        const size_t at = (blob.size() + 15) & ~(size_t)15;
        blob.resize(at + bytes);
        if (bytes) std::memcpy(blob.data() + at, src, bytes);
        return at;
    };
    const size_t o_cols = put(gp.cols.data(), gp.cols.size() * sizeof(GlCol)), o_eps = put(gp.eps.data(), gp.eps.size() * 8),
                 o_trans = put(gp.trans.data(), gp.trans.size() * 8), o_q = put(gp.q.data(), gp.q.size() * 8),
                 o_allele = put(gp.allele.data(), gp.allele.size()), o_ind = put(gp.ind.data(), gp.ind.size()), o_h2p = put(gp.h2p.data(), gp.h2p.size()),
                 o_tables = put(gp.tables.data(), gp.tables.size() * sizeof(GlBatchTable)),
                 o_steps = put(gp.steps.data(), gp.steps.size() * sizeof(GlStep)),
                 o_step_table = put(gp.step_table.data(), gp.step_table.size() * 4);
    const uint64_t work = gp.store_doubles + gp.f_pool_doubles + gp.acc_doubles;
    Buffers W;
    W.stream = s;
    W.owns_stream = false;
    uint8_t *d_blob = nullptr;
    double *d_work = nullptr;
    CUDA_TRY(W.alloc(&d_blob, blob.size()));
    CUDA_TRY(W.alloc(&d_work, work));
    CUDA_TRY(cudaMemcpyAsync(d_blob, blob.data(), blob.size(), cudaMemcpyHostToDevice, s));
    CUDA_TRY(cudaMemsetAsync(d_work, 0, work * 8, s));
    const GlBatchInputs in{(const GlCol *)(d_blob + o_cols),  (const double *)(d_blob + o_eps), d_blob + o_allele,          d_blob + o_ind,
                           (const int8_t *)(d_blob + o_h2p), (const double *)(d_blob + o_trans), (const double *)(d_blob + o_q)};
    const GlBatchTable *d_tables = (const GlBatchTable *)(d_blob + o_tables);
    const GlStep *d_steps = (const GlStep *)(d_blob + o_steps);
    const uint32_t *d_step_table = (const uint32_t *)(d_blob + o_step_table);
    double *d_beta = d_work, *d_F = d_work + gp.store_doubles, *d_acc = d_F + gp.f_pool_doubles;
    auto widest = [&](uint32_t e0, uint32_t e1) {
        uint32_t a_max = 0;
        for (uint32_t e = e0; e < e1; ++e) a_max = std::max(a_max, gp.steps[e].cells_log2);
        return (unsigned)((((uint64_t)1 << a_max) + GL_THREADS - 1) / GL_THREADS);
    };
    Timer tm;
    CUDA_TRY(tm.start(s));
    uint32_t launches = 0;
    for (size_t l = 0; l + 1 < gp.bwd_begin.size(); ++l)
        for (uint32_t e0 = gp.bwd_begin[l]; e0 < gp.bwd_begin[l + 1]; e0 += GL_MAX_GRID_Y) {
            const uint32_t e1 = std::min(gp.bwd_begin[l + 1], e0 + GL_MAX_GRID_Y);
            gl_batch_backward_kernel<<<dim3(widest(e0, e1), e1 - e0), GL_THREADS, 0, s>>>(in, d_tables, d_steps + e0, d_step_table + e0, d_beta);
            gl_scale_kernel<<<e1 - e0, 1024, 0, s>>>(d_steps + e0, d_beta);
            launches += 2;
        }
    for (size_t l = 0; l + 1 < gp.fwd_begin.size(); ++l)
        for (uint32_t e0 = gp.fwd_begin[l]; e0 < gp.fwd_begin[l + 1]; e0 += GL_MAX_GRID_Y) {
            const uint32_t e1 = std::min(gp.fwd_begin[l + 1], e0 + GL_MAX_GRID_Y);
            gl_batch_forward_kernel<<<dim3(widest(e0, e1), e1 - e0), GL_THREADS, 0, s>>>(in, d_tables, d_steps + e0, d_step_table + e0, d_F, d_beta,
                                                                                         d_acc);
            gl_scale_kernel<<<e1 - e0, 1024, 0, s>>>(d_steps + e0, d_F);
            launches += 2;
        }
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaEventRecord(tm.ev1, s));
    std::vector<double> acc(gp.acc_doubles);
    CUDA_TRY(cudaMemcpyAsync(acc.data(), d_acc, acc.size() * 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    whmec_stats group{};
    CUDA_TRY(cudaEventElapsedTime(&group.sweep_ms, tm.ev0, tm.ev1));
    group.kernel_launches = launches;
    group.h2d_bytes = blob.size();
    group.d2h_bytes = acc.size() * 8;
    add_stats(total, group);
    for (size_t m = 0; m < gp.members.size(); ++m) {
        const uint32_t t = gp.members[m];
        const GlBatchTable &d = gp.tables[m];
        gl_normalise(acc.data() + d.acc_base, d.n_cols, d.n_ind, likelihoods[t]);
        whmec_stats st = pks[t].stats;  // times and launches: the group's, in `total`
        st.path_kind = 4;
        st.backptr_bytes = gs[t].beta_doubles * 8;
        add_stats(total, st);
        if (stats) stats[t] = st;
    }
    return WHMEC_OK;
}

// whmec_genotype_batch: every table packed (a table that fails keeps its status and message), then groups of tables on one step
// list each (gl_batch_groups under the budget work_budget applies), and every table that does not fit a group alone through the
// single-table path.  A CUDA failure returns WHMEC_ERR_CUDA with `msg` (the caller reports it for every table).
int genotype_batch_impl(const whmec_problem *const *problems, double *const *likelihoods, uint32_t n_tables, int device, int *status, char *errs,
                        size_t errlen, whmec_stats *stats, whmec_stats &total, std::string &msg) {
    auto err_of = [&](uint32_t t) { return errs ? errs + (size_t)t * errlen : nullptr; };
    std::vector<Packed> pks(n_tables);
    std::vector<GlPacked> gs(n_tables);
    std::vector<uint64_t> cost(n_tables, 0);  // 0: not on the device (an error, or no columns)
    bool any = false;
    for (uint32_t t = 0; t < n_tables; ++t) {
        status[t] = WHMEC_OK;
        if (stats) stats[t] = whmec_stats{};
        std::string m;
        int rc = WHMEC_ERR_INPUT;
        if (!problems[t] || !likelihoods[t]) m = "null argument";
        else {
            try {
                rc = gl_pack(problems[t], pks[t], gs[t], m);
            } catch (const std::exception &e) {
                m = e.what();
                rc = WHMEC_ERR_INPUT;
            }
        }
        if (rc != WHMEC_OK) {
            status[t] = rc;
            set_err(err_of(t), errlen, m);
            pks[t] = Packed();
            gs[t] = GlPacked();
            continue;
        }
        if (stats) stats[t] = pks[t].stats;
        if (pks[t].n == 0) continue;
        any = true;
    }
    if (!any) return WHMEC_OK;
    int rc = open_device(device, msg);
    if (rc != WHMEC_OK) return rc;
    Buffers S;
    CUDA_TRY(cudaStreamCreateWithFlags(&S.stream, cudaStreamNonBlocking));
    const size_t free_b = device_available_bytes();
    const uint64_t reserve = 512ull << 20;
    uint64_t budget = free_b > reserve ? (free_b - reserve) / 8 : 0;
    if (const char *e = std::getenv("WHMEC_GENOTYPE_ARENA_BUDGET")) budget = std::min<uint64_t>(budget, std::strtoull(e, nullptr, 10) / 8);
    for (uint32_t t = 0; t < n_tables; ++t)
        if (status[t] == WHMEC_OK && pks[t].n > 0) cost[t] = gl_batch_cost(pks[t], gs[t]);
    std::vector<std::vector<uint32_t>> groups;
    std::vector<uint32_t> alone;
    gl_batch_groups(cost, budget, groups, alone);
    for (const std::vector<uint32_t> &members : groups) {
        GlBatchGroup gp;
        gl_batch_plan(pks, gs, members, gp);
        rc = run_batch_group(S.stream, gp, pks, gs, likelihoods, stats, total, msg);
        if (rc != WHMEC_OK) return rc;
        for (uint32_t t : members) {
            pks[t] = Packed();
            gs[t] = GlPacked();
        }
    }
    for (uint32_t t : alone) {  // packed again there; its result, code and text are whmec_genotype's
        pks[t] = Packed();
        gs[t] = GlPacked();
        whmec_stats st{};
        std::string m;
        try {
            rc = genotype_impl(problems[t], likelihoods[t], device, &st, m);
        } catch (const std::exception &e) {
            m = e.what();
            rc = WHMEC_ERR_INPUT;
        }
        if (rc == WHMEC_ERR_CUDA) {
            msg = m;
            return rc;
        }
        status[t] = rc;
        set_err(err_of(t), errlen, m);
        if (rc != WHMEC_OK) continue;
        add_stats(total, st);
        st.sweep_ms = st.h2d_ms = st.d2h_ms = 0;
        if (stats) stats[t] = st;
    }
    return WHMEC_OK;
}

}  // namespace

// A segment of a pedigree table on one device (include/whmec.h): packed and uploaded once, then the transfer pass and the run.
struct whmec_gl_segment {
    int device = 0;
    bool continues = false, continued = false;
    Packed pk;
    GlPacked g;
    Buffers B;  // the stream and the uploaded inputs
    GlView v{};
    uint64_t h2d = 0;
};

extern "C" int whmec_genotype(const whmec_problem *p, double *likelihoods, int device, whmec_stats *st, char *err, size_t errlen) {
    return guarded([&](std::string &msg) { return genotype_impl(p, likelihoods, device, st, msg); }, err, errlen);
}

extern "C" int whmec_genotype_batch(const whmec_problem *const *problems, double *const *likelihoods, uint32_t n_tables, int device, int *status,
                                    char *errs, size_t errlen, whmec_stats *stats, whmec_stats *total) {
    if (total) *total = whmec_stats{};
    if (n_tables == 0) return WHMEC_OK;
    if (!problems || !likelihoods || !status) return WHMEC_ERR_INPUT;
    whmec_stats sum{};
    std::string msg;
    int rc;
    try {
        rc = genotype_batch_impl(problems, likelihoods, n_tables, device, status, errs, errlen, stats, sum, msg);
    } catch (const std::exception &e) {  // out of host memory: the call failed
        msg = e.what();
        rc = WHMEC_ERR_UNSUPPORTED;
    }
    if (rc != WHMEC_OK) {  // the call failed: every table reports why
        for (uint32_t t = 0; t < n_tables; ++t) {
            status[t] = rc;
            set_err(errs ? errs + (size_t)t * errlen : nullptr, errlen, msg);
        }
        return rc;
    }
    if (total) *total = sum;
    return WHMEC_OK;
}

extern "C" int whmec_genotype_segment_create(const whmec_problem *p, int device, int continues, int continued, whmec_gl_segment **out, char *err,
                                             size_t errlen) {
    return guarded(
        [&](std::string &msg) {
            if (!p || !out) {
                msg = "null argument";
                return WHMEC_ERR_INPUT;
            }
            *out = nullptr;
            auto sg = std::make_unique<whmec_gl_segment>();
            sg->device = device;
            sg->continues = continues != 0;
            sg->continued = continued != 0;
            int rc = gl_pack_segment(p, sg->continues, sg->continued, sg->pk, sg->g, msg);
            if (rc != WHMEC_OK) return rc;
            if (sg->pk.n == 0) {
                msg = "genotyping segments: a segment needs at least one column";
                return WHMEC_ERR_INPUT;
            }
            rc = open_device(device, msg);
            if (rc != WHMEC_OK) return rc;
            CUDA_TRY(cudaStreamCreateWithFlags(&sg->B.stream, cudaStreamNonBlocking));
            rc = upload_inputs(sg->B, sg->pk, sg->g, sg->v, sg->h2d, msg);
            if (rc != WHMEC_OK) return rc;
            CUDA_TRY(cudaStreamSynchronize(sg->B.stream));
            *out = sg.release();
            return WHMEC_OK;
        },
        err, errlen);
}

extern "C" int whmec_genotype_segment_transfer(whmec_gl_segment *sg, double *matrix, whmec_stats *st, char *err, size_t errlen) {
    return guarded(
        [&](std::string &msg) {
            if (!sg || !matrix) {
                msg = "null argument";
                return WHMEC_ERR_INPUT;
            }
            CUDA_TRY(cudaSetDevice(sg->device));
            const uint32_t T = sg->pk.T, n = sg->pk.n;
            GlTransfer tp;
            gl_transfer_plan(sg->g, T, sg->continues, tp);
            cudaStream_t s = sg->B.stream;
            Buffers W;
            W.stream = s;
            W.owns_stream = false;
            // the batches' inputs, rows and column scales stay on the device until the timed region is over: no host work
            // between the batches
            const size_t batch = (size_t)tp.n_in * T, n_max = tp.n_batches > 1 ? (size_t)tp.n_batches * n : 0;
            double *d_F = nullptr, *d_in = nullptr, *d_rows = nullptr, *d_max = nullptr;
            GlStep *d_steps = nullptr;
            CUDA_TRY(W.alloc(&d_F, tp.f_pool_doubles));
            CUDA_TRY(W.alloc(&d_steps, n));
            CUDA_TRY(W.alloc(&d_rows, tp.n_batches * batch));
            CUDA_TRY(W.alloc(&d_max, n_max));
            std::vector<double> rows(tp.n_batches * batch), col_max(n_max), inputs;
            uint64_t h2d = (uint64_t)n * sizeof(GlStep);
            CUDA_TRY(cudaMemcpyAsync(d_steps, tp.steps.data(), (size_t)n * sizeof(GlStep), cudaMemcpyHostToDevice, s));
            if (sg->continues) {  // batch b's inputs: e_u for u = b * n_in + r, one row each
                inputs.assign(tp.n_batches * batch, 0.0);
                for (uint32_t u = 0; u < tp.n_batches * tp.n_in; ++u) inputs[(size_t)u * T + u] = 1.0;
                CUDA_TRY(W.alloc(&d_in, inputs.size()));
                CUDA_TRY(cudaMemcpyAsync(d_in, inputs.data(), inputs.size() * 8, cudaMemcpyHostToDevice, s));
                h2d += inputs.size() * 8;
            }
            Timer tm;
            CUDA_TRY(tm.start(s));
            uint32_t launches = 0;
            for (uint32_t b = 0; b < tp.n_batches; ++b) {
                CUDA_TRY(cudaMemsetAsync(d_F, 0, tp.f_pool_doubles * 8, s));
                if (d_in) CUDA_TRY(cudaMemcpyAsync(d_F + tp.in_off, d_in + b * batch, batch * 8, cudaMemcpyDeviceToDevice, s));
                for (uint32_t k = 0; k < n; ++k) {
                    const unsigned blocks = (unsigned)((((uint64_t)1 << tp.steps[k].cells_log2) + GL_THREADS - 1) / GL_THREADS);
                    gl_transfer_kernel<<<blocks, GL_THREADS, 0, s>>>(sg->v, d_steps + k, d_F, tp.n_in);
                    if (n_max) gl_column_max_kernel<<<1, 1024, 0, s>>>(d_steps + k, d_F, d_max + (size_t)b * n + k);
                    gl_scale_kernel<<<1, 1024, 0, s>>>(d_steps + k, d_F);
                    launches += n_max ? 3 : 2;
                }
                CUDA_TRY(cudaMemcpyAsync(d_rows + b * batch, d_F + tp.out_off, batch * 8, cudaMemcpyDeviceToDevice, s));
            }
            CUDA_TRY(cudaGetLastError());
            CUDA_TRY(cudaEventRecord(tm.ev1, s));
            CUDA_TRY(cudaMemcpyAsync(rows.data(), d_rows, rows.size() * 8, cudaMemcpyDeviceToHost, s));
            if (n_max) CUDA_TRY(cudaMemcpyAsync(col_max.data(), d_max, n_max * 8, cudaMemcpyDeviceToHost, s));
            CUDA_TRY(cudaStreamSynchronize(s));
            float ms = 0.f;
            CUDA_TRY(cudaEventElapsedTime(&ms, tm.ev0, tm.ev1));
            gl_transfer_combine(tp, T, rows, col_max, matrix);
            if (st) {
                *st = sg->pk.stats;
                st->kernel_launches = launches;
                st->sweep_ms = ms;
                st->h2d_bytes = h2d;
                st->d2h_bytes = (rows.size() + col_max.size()) * 8;
                st->backptr_bytes = 0;  // no backward tables in this pass
                st->path_kind = 4;
            }
            return WHMEC_OK;
        },
        err, errlen);
}

extern "C" int whmec_genotype_segment_run(whmec_gl_segment *sg, const double *alpha_in, const double *beta_in, double *likelihoods, whmec_stats *st,
                                          char *err, size_t errlen) {
    return guarded(
        [&](std::string &msg) {
            if (!sg || !likelihoods) {
                msg = "null argument";
                return WHMEC_ERR_INPUT;
            }
            if (sg->continues && !alpha_in) {
                msg = "genotyping segments: a segment that continues the table needs alpha_in (the forward vector in front of it)";
                return WHMEC_ERR_INPUT;
            }
            if (sg->continued && !beta_in) {
                msg = "genotyping segments: a segment that the table continues after needs beta_in (the backward vector behind it)";
                return WHMEC_ERR_INPUT;
            }
            CUDA_TRY(cudaSetDevice(sg->device));
            uint64_t budget = 0;  // the inputs are resident already: counted twice, which errs on the safe side
            const int rc = work_budget(sg->pk, sg->g, budget, msg);
            if (rc != WHMEC_OK) return rc;
            return run_packed(sg->B, sg->pk, sg->g, sg->v, budget, sg->continues ? alpha_in : nullptr, sg->continued ? beta_in : nullptr, likelihoods, st,
                              sg->h2d, msg);
        },
        err, errlen);
}

extern "C" void whmec_genotype_segment_destroy(whmec_gl_segment *sg) {
    if (!sg) return;
    cudaSetDevice(sg->device);
    delete sg;
}
