// TEST-ONLY host emulation of whmec_genotype under a memory budget (genotype.cu, gl_plan): groups of tables on their launch
// schedules and tables in memory-bounded mode, with the host packer (gl_pack.cpp) and the __host__ __device__ per-cell
// functions of gl_device.h stepped serially, in the kernels' launch order (as emul_gl.cpp does for the resident path).
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "../../whatshap_b200/csrc/gl_pack.h"

using namespace whmec;

namespace {

int fail(int rc, const std::string &msg, char *err, size_t errlen) {
    if (err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = 0;
    }
    return rc;
}

auto add = [](double *addr, double val) { *addr += val; };

// the cells of one backward / forward step, then its rescale (and, forward, the clear of the other projection buffer)
void backward_step(const GlView &v, const GlStep &st, const double *beta_k, double *beta) {
    for (uint64_t x = 0; x < ((uint64_t)1 << st.cells_log2); ++x) gl_backward_cell(v, st.k, (uint32_t)x, beta_k, beta + st.cur_off, add);
}
void forward_step(const GlView &v, const GlStep &st, double *F, const double *beta_k, double *acc) {
    for (uint64_t x = 0; x < ((uint64_t)1 << st.cells_log2); ++x)
        gl_forward_cell(v, st.k, (uint32_t)x, F + st.prev_off, F + st.cur_off, beta_k, acc + (size_t)st.k * v.n_ind * 3, add);
}
void forward_finish(const GlStep &st, double *F) {
    gl_scale_host(F + st.cur_off, st.n_scale);
    std::fill(F + st.prev_off, F + st.prev_off + st.n_clear, 0.0);
}

// one group of whole tables on its launch schedule (gl_schedule)
void run_schedule(const GlPacked &g, const GlView &v, const GlSchedule &sc, double *acc) {
    std::vector<double> beta(sc.beta_doubles + 1, 0.0), F(sc.f_pool_doubles, 0.0);
    auto table_of = [&](uint32_t k) { return beta.data() + (g.cols[k].beta_off - sc.beta_base); };
    for (size_t l = 0; l + 1 < sc.bwd_begin.size(); ++l) {
        for (uint32_t e = sc.bwd_begin[l]; e < sc.bwd_begin[l + 1]; ++e) backward_step(v, sc.steps[e], table_of(sc.steps[e].k), beta.data());
        for (uint32_t e = sc.bwd_begin[l]; e < sc.bwd_begin[l + 1]; ++e) gl_scale_host(beta.data() + sc.steps[e].cur_off, sc.steps[e].n_scale);
    }
    for (size_t l = 0; l + 1 < sc.fwd_begin.size(); ++l) {
        for (uint32_t e = sc.fwd_begin[l]; e < sc.fwd_begin[l + 1]; ++e) forward_step(v, sc.steps[e], F.data(), table_of(sc.steps[e].k), acc);
        for (uint32_t e = sc.fwd_begin[l]; e < sc.fwd_begin[l + 1]; ++e) forward_finish(sc.steps[e], F.data());
    }
}

// one table in memory-bounded mode (gl_bounded): the sweeps of pass A and pass B, one step per launch
void run_bounded(const GlPacked &g, const GlView &v, const GlBounded &bd, double *acc) {
    std::vector<double> store(bd.arena_doubles + bd.ckpt_doubles, 0.0), F(bd.f_pool_doubles, 0.0);
    for (const GlSweep &sw : bd.sweeps) {
        std::fill(store.begin(), store.begin() + sw.clear, 0.0);
        std::copy(store.begin() + sw.copy_src, store.begin() + sw.copy_src + sw.copy_n, store.begin() + sw.copy_dst);
        auto table_of = [&](uint32_t k) { return store.data() + (g.cols[k].beta_off - sw.beta_base); };
        for (uint32_t e = sw.bwd_begin; e < sw.bwd_end; ++e) {
            backward_step(v, bd.steps[e], table_of(bd.steps[e].k), store.data());
            gl_scale_host(store.data() + bd.steps[e].cur_off, bd.steps[e].n_scale);
        }
        for (uint32_t e = sw.fwd_begin; e < sw.fwd_end; ++e) {
            forward_step(v, bd.steps[e], F.data(), table_of(bd.steps[e].k), acc);
            forward_finish(bd.steps[e], F.data());
        }
    }
}

}  // namespace

// What whmec_genotype runs under a budget of `budget_doubles` for backward tables, checkpoints and projection buffers
// (gl_plan): groups of tables as above, and a table that alone exceeds the budget in memory-bounded mode.  n_segments: the
// most segments any table was cut into (1: none was).
extern "C" int whemul_genotype_bounded(const whmec_problem *p, double *likelihoods, uint64_t budget_doubles, uint32_t *n_segments,
                                       char *err, size_t errlen) {
    Packed pk;
    GlPacked g;
    std::string msg;
    int rc = gl_pack(p, pk, g, msg);
    if (rc != WHMEC_OK) return fail(rc, msg, err, errlen);
    const uint32_t n = pk.n, n_ind = pk.n_ind;
    if (n_segments) *n_segments = 1;
    if (n == 0) return WHMEC_OK;
    std::vector<GlUnit> units;
    rc = gl_plan(g, pk.T, budget_doubles, units, msg);
    if (rc != WHMEC_OK) return fail(rc, msg, err, errlen);
    const GlView v = g.view(pk);
    std::vector<double> acc((size_t)n * n_ind * 3, 0.0);
    for (const GlUnit &u : units) {
        if (u.bounded) {
            run_bounded(g, v, u.bd, acc.data());
            if (n_segments) *n_segments = std::max<uint32_t>(*n_segments, (uint32_t)u.bd.cuts.size() - 1);
        } else {
            run_schedule(g, v, u.sc, acc.data());
        }
    }
    gl_normalise(acc.data(), n, n_ind, likelihoods);
    return WHMEC_OK;
}

// The plan of the table with the most segments under `budget_doubles`: its cuts (n_cuts <= cuts_cap entries, absolute
// columns), sizes = {arena, checkpoints, projection buffers} (doubles), and own[k] = doubles of column k's backward table
// (0 for a table's last column) for every column.  n_cuts = 0 when no table needs cutting.
extern "C" int whemul_genotype_bounded_plan(const whmec_problem *p, uint64_t budget_doubles, uint32_t *cuts, uint32_t cuts_cap, uint32_t *n_cuts,
                                            uint64_t *sizes, uint64_t *own, char *err, size_t errlen) {
    Packed pk;
    GlPacked g;
    std::string msg;
    int rc = gl_pack(p, pk, g, msg);
    if (rc != WHMEC_OK) return fail(rc, msg, err, errlen);
    *n_cuts = 0;
    for (uint32_t k = 0; k < pk.n; ++k) own[k] = g.cols[k].last ? 0 : ((uint64_t)1 << g.cols[k].f) * pk.T;
    if (pk.n == 0) return WHMEC_OK;
    std::vector<GlUnit> units;
    rc = gl_plan(g, pk.T, budget_doubles, units, msg);
    if (rc != WHMEC_OK) return fail(rc, msg, err, errlen);
    for (const GlUnit &u : units)
        if (u.bounded && u.bd.cuts.size() > *n_cuts && u.bd.cuts.size() <= cuts_cap) {
            *n_cuts = (uint32_t)u.bd.cuts.size();
            std::copy(u.bd.cuts.begin(), u.bd.cuts.end(), cuts);
            sizes[0] = u.bd.arena_doubles;
            sizes[1] = u.bd.ckpt_doubles;
            sizes[2] = u.bd.f_pool_doubles;
        }
    return WHMEC_OK;
}
