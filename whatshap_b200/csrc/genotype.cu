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
#include <cuda_runtime.h>

#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

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

struct Buffers {  // freed on every exit path
    cudaStream_t stream = nullptr;
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
            cudaStreamDestroy(stream);
        }
    }
};

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
    const uint32_t n = pk.n, T = pk.T, n_ind = pk.n_ind;
    if (n == 0) return WHMEC_OK;
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
        msg = "no CUDA device (whatshap_b200 has no CPU path)";
        return WHMEC_ERR_CUDA;
    }
    CUDA_TRY(cudaSetDevice(device));
    Buffers B;
    CUDA_TRY(cudaStreamCreateWithFlags(&B.stream, cudaStreamNonBlocking));
    cudaStream_t s = B.stream;

    // groups of whole tables (T == 1: chains; otherwise the one table) whose backward tables fit the device together
    const size_t free_b = device_available_bytes();
    const uint64_t fixed = (uint64_t)n * sizeof(GlCol) + g.eps.size() * 10 + (g.trans.size() + g.q.size()) * 8 + (uint64_t)n * sizeof(GlStep) * 2 +
                           (uint64_t)n * n_ind * 3 * 8 + (512ull << 20);
    if (fixed > free_b) {
        msg = "genotyping: problem exceeds the free HBM of this device";
        return WHMEC_ERR_UNSUPPORTED;
    }
    uint64_t budget = (free_b - fixed) / 8;  // doubles available for backward tables + projection buffers
    // WHMEC_GENOTYPE_ARENA_BUDGET=bytes (test hook): the budget for backward tables, checkpoints and projection buffers
    if (const char *e = std::getenv("WHMEC_GENOTYPE_ARENA_BUDGET")) budget = std::min<uint64_t>(budget, std::strtoull(e, nullptr, 10) / 8);
    // groups of tables on launch schedules (one launch advances every table of a group by one column); a table whose
    // backward tables do not fit runs alone in memory-bounded mode (gl_bounded)
    std::vector<GlUnit> units;
    rc = gl_plan(g, T, budget, units, msg);
    if (rc != WHMEC_OK) return rc;
    uint64_t max_work = 1, max_steps = 1, max_store = 0;  // max_store: the largest backward store of a unit (doubles)
    bool bounded = false;
    for (const GlUnit &u : units) {
        max_work = std::max(max_work, u.work_doubles);
        max_steps = std::max<uint64_t>(max_steps, u.bounded ? u.bd.steps.size() : u.sc.steps.size());
        max_store = std::max(max_store, u.bounded ? u.bd.arena_doubles + u.bd.ckpt_doubles : u.sc.beta_doubles);
        bounded = bounded || u.bounded;
    }
    GlCol *d_cols = nullptr;
    double *d_eps = nullptr, *d_trans = nullptr, *d_q = nullptr, *d_work = nullptr, *d_acc = nullptr;
    GlStep *d_steps = nullptr;
    uint8_t *d_allele = nullptr, *d_ind = nullptr;
    int8_t *d_h2p = nullptr;
    CUDA_TRY(B.alloc(&d_cols, n));
    CUDA_TRY(B.alloc(&d_eps, g.eps.size()));
    CUDA_TRY(B.alloc(&d_allele, pk.act_allele.size()));
    CUDA_TRY(B.alloc(&d_ind, pk.act_ind.size()));
    CUDA_TRY(B.alloc(&d_h2p, pk.h2p.size()));
    CUDA_TRY(B.alloc(&d_trans, g.trans.size()));
    CUDA_TRY(B.alloc(&d_q, g.q.size()));
    CUDA_TRY(B.alloc(&d_work, max_work));  // per unit: its backward store, then its projection buffers
    CUDA_TRY(B.alloc(&d_steps, max_steps));
    CUDA_TRY(B.alloc(&d_acc, (size_t)n * n_ind * 3));
    uint64_t h2d = 0;
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
    CUDA_TRY(cudaMemsetAsync(d_acc, 0, (size_t)n * n_ind * 3 * 8, s));
    const GlView v{d_cols, d_eps, d_allele, d_ind, d_h2p, d_trans, d_q, T, pk.P, n_ind};

    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    CUDA_TRY(cudaEventCreate(&ev0));
    CUDA_TRY(cudaEventCreate(&ev1));
    CUDA_TRY(cudaEventRecord(ev0, s));
    uint32_t launches = 0;
    constexpr uint32_t MAX_GRID_Y = 65535;
    for (size_t q = 0; q < units.size(); ++q) {
        if (q > 0) CUDA_TRY(cudaStreamSynchronize(s));  // the step list of the previous unit is still being read
        if (units[q].bounded) {
            const GlBounded &bd = units[q].bd;
            const uint64_t store = bd.arena_doubles + bd.ckpt_doubles;
            double *d_beta = d_work, *d_F = d_work + store;
            CUDA_TRY(up(d_steps, bd.steps.data(), bd.steps.size() * sizeof(GlStep)));
            CUDA_TRY(cudaMemsetAsync(d_work, 0, (store + bd.f_pool_doubles) * 8, s));
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
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaEventRecord(ev1, s));
    std::vector<double> acc((size_t)n * n_ind * 3);
    CUDA_TRY(cudaMemcpyAsync(acc.data(), d_acc, acc.size() * 8, cudaMemcpyDeviceToHost, s));
    CUDA_TRY(cudaStreamSynchronize(s));
    float ms = 0.f;
    CUDA_TRY(cudaEventElapsedTime(&ms, ev0, ev1));
    cudaEventDestroy(ev0);
    cudaEventDestroy(ev1);
    gl_normalise(acc.data(), n, n_ind, likelihoods);
    if (st) {
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

}  // namespace

extern "C" int whmec_genotype(const whmec_problem *p, double *likelihoods, int device, whmec_stats *st, char *err, size_t errlen) {
    std::string msg;
    int rc;
    try {
        rc = genotype_impl(p, likelihoods, device, st, msg);
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
