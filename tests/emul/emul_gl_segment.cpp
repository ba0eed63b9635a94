// TEST-ONLY host emulation of the genotyping segments (whmec_genotype_segment_*, genotype.cu): the host packer and plans
// (gl_pack_segment, gl_transfer_plan, gl_plan) and the __host__ __device__ per-cell functions of gl_device.h stepped serially,
// in the kernels' launch order (as emul_gl_bounded.cpp does for whmec_genotype).
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

void backward_step(const GlView &v, const GlStep &st, const double *beta_k, double *beta) {
    for (uint64_t x = 0; x < ((uint64_t)1 << st.cells_log2); ++x) gl_backward_cell(v, st.k, (uint32_t)x, beta_k, beta + st.cur_off, add);
}
void forward_step(const GlView &v, const GlStep &st, double *F, const double *beta_k, double *acc) {
    for (uint64_t x = 0; x < ((uint64_t)1 << st.cells_log2); ++x)
        gl_forward_cell(v, st.k, (uint32_t)x, F + st.prev_off, F + st.cur_off, beta_k, acc + (size_t)st.k * v.n_ind * 3, add);
}
void finish_step(const GlStep &st, double *F) {  // gl_scale_kernel
    gl_scale_host(F + st.cur_off, st.n_scale);
    std::fill(F + st.prev_off, F + st.prev_off + st.n_clear, 0.0);
}

// one unit of gl_plan in its work buffer (store, then F pool), with the segment's inputs placed after the buffer is cleared
void run_unit(const GlPacked &g, const GlView &v, const GlUnit &u, const double *alpha, const double *beta, double *acc) {
    std::vector<double> work(u.work_doubles, 0.0);
    if (alpha) std::copy(alpha, alpha + v.T, work.begin() + u.alpha_at);
    if (beta) std::copy(beta, beta + v.T, work.begin() + u.beta_at);
    if (u.bounded) {
        const GlBounded &bd = u.bd;
        double *store = work.data(), *F = store + bd.arena_doubles + bd.ckpt_doubles;
        for (const GlSweep &sw : bd.sweeps) {
            std::fill(store, store + sw.clear, 0.0);
            std::copy(store + sw.copy_src, store + sw.copy_src + sw.copy_n, store + sw.copy_dst);
            auto table_of = [&](uint32_t k) { return store + (g.cols[k].beta_off - sw.beta_base); };
            for (uint32_t e = sw.bwd_begin; e < sw.bwd_end; ++e) {
                backward_step(v, bd.steps[e], table_of(bd.steps[e].k), store);
                gl_scale_host(store + bd.steps[e].cur_off, bd.steps[e].n_scale);
            }
            for (uint32_t e = sw.fwd_begin; e < sw.fwd_end; ++e) {
                forward_step(v, bd.steps[e], F, table_of(bd.steps[e].k), acc);
                finish_step(bd.steps[e], F);
            }
        }
        return;
    }
    const GlSchedule &sc = u.sc;
    double *store = work.data(), *F = store + sc.beta_doubles + 1;
    auto table_of = [&](uint32_t k) { return store + (g.cols[k].beta_off - sc.beta_base); };
    for (size_t l = 0; l + 1 < sc.bwd_begin.size(); ++l) {
        for (uint32_t e = sc.bwd_begin[l]; e < sc.bwd_begin[l + 1]; ++e) backward_step(v, sc.steps[e], table_of(sc.steps[e].k), store);
        for (uint32_t e = sc.bwd_begin[l]; e < sc.bwd_begin[l + 1]; ++e) gl_scale_host(store + sc.steps[e].cur_off, sc.steps[e].n_scale);
    }
    for (size_t l = 0; l + 1 < sc.fwd_begin.size(); ++l) {
        for (uint32_t e = sc.fwd_begin[l]; e < sc.fwd_begin[l + 1]; ++e) forward_step(v, sc.steps[e], F, table_of(sc.steps[e].k), acc);
        for (uint32_t e = sc.fwd_begin[l]; e < sc.fwd_begin[l + 1]; ++e) finish_step(sc.steps[e], F);
    }
}

struct Segment {
    bool continues, continued;
    Packed pk;
    GlPacked g;
};

}  // namespace

extern "C" int whemul_gl_segment_create(const whmec_problem *p, int continues, int continued, void **out, char *err, size_t errlen) {
    auto *s = new Segment{continues != 0, continued != 0, Packed(), GlPacked()};
    std::string msg;
    int rc = gl_pack_segment(p, s->continues, s->continued, s->pk, s->g, msg);
    if (rc == WHMEC_OK && s->pk.n == 0) {
        rc = WHMEC_ERR_INPUT;
        msg = "genotyping segments: a segment needs at least one column";
    }
    if (rc != WHMEC_OK) {
        delete s;
        return fail(rc, msg, err, errlen);
    }
    *out = s;
    return WHMEC_OK;
}

// whmec_genotype_segment_transfer: the batches of gl_transfer_plan, each column a transfer step, then (with several batches)
// the column's scale recorded, then the scale itself
extern "C" int whemul_gl_segment_transfer(void *h, double *matrix, uint32_t *n_batches) {
    const Segment &s = *(const Segment *)h;
    const uint32_t T = s.pk.T, n = s.pk.n;
    const GlView v = s.g.view(s.pk);
    GlTransfer tp;
    gl_transfer_plan(s.g, T, s.continues, tp);
    std::vector<double> F(tp.f_pool_doubles), rows((size_t)tp.n_batches * tp.n_in * T), col_max((size_t)tp.n_batches * n, 0.0);
    for (uint32_t b = 0; b < tp.n_batches; ++b) {
        std::fill(F.begin(), F.end(), 0.0);
        if (s.continues)
            for (uint32_t r = 0; r < tp.n_in; ++r) F[tp.in_off + (size_t)r * T + b * tp.n_in + r] = 1.0;
        for (uint32_t k = 0; k < n; ++k) {
            const GlStep &st = tp.steps[k];
            for (uint64_t x = 0; x < ((uint64_t)1 << st.cells_log2); ++x)
                gl_transfer_cell(v, k, (uint32_t)x, tp.n_in, F.data() + st.prev_off, F.data() + st.cur_off, add);
            if (tp.n_batches > 1)
                for (uint64_t i = 0; i < st.n_scale; ++i) col_max[(size_t)b * n + k] = std::max(col_max[(size_t)b * n + k], F[st.cur_off + i]);
            finish_step(st, F.data());
        }
        std::copy(F.begin() + tp.out_off, F.begin() + tp.out_off + (size_t)tp.n_in * T, rows.begin() + (size_t)b * tp.n_in * T);
    }
    gl_transfer_combine(tp, T, rows, col_max, matrix);
    if (n_batches) *n_batches = tp.n_batches;
    return WHMEC_OK;
}

// whmec_genotype_segment_run under `budget_doubles` for backward tables, checkpoints and projection buffers (gl_plan); n_segments:
// the segments of the memory-bounded mode (1: resident)
extern "C" int whemul_gl_segment_run(void *h, const double *alpha, const double *beta, double *likelihoods, uint64_t budget_doubles,
                                     uint32_t *n_segments, char *err, size_t errlen) {
    const Segment &s = *(const Segment *)h;
    if (s.continues && !alpha)
        return fail(WHMEC_ERR_INPUT, "genotyping segments: a segment that continues the table needs alpha_in (the forward vector in front of it)", err,
                    errlen);
    if (s.continued && !beta)
        return fail(WHMEC_ERR_INPUT, "genotyping segments: a segment that the table continues after needs beta_in (the backward vector behind it)", err,
                    errlen);
    std::vector<GlUnit> units;
    std::string msg;
    int rc = gl_plan(s.g, s.pk.T, budget_doubles, units, msg);
    if (rc != WHMEC_OK) return fail(rc, msg, err, errlen);
    const GlView v = s.g.view(s.pk);
    std::vector<double> acc((size_t)s.pk.n * s.pk.n_ind * 3, 0.0);
    if (n_segments) *n_segments = 1;
    for (const GlUnit &u : units) {
        run_unit(s.g, v, u, s.continues ? alpha : nullptr, s.continued ? beta : nullptr, acc.data());
        if (u.bounded && n_segments) *n_segments = std::max<uint32_t>(*n_segments, (uint32_t)u.bd.cuts.size() - 1);
    }
    gl_normalise(acc.data(), s.pk.n, s.pk.n_ind, likelihoods);
    return WHMEC_OK;
}

extern "C" void whemul_gl_segment_destroy(void *h) { delete (Segment *)h; }
