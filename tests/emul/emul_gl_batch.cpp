// TEST-ONLY host emulation of whmec_genotype_batch (genotype.cu): the host packer (gl_pack.cpp), the batch plan (gl_batch.cpp)
// and the __host__ __device__ per-cell functions of gl_device.h, stepped serially in the kernels' launch order.  Within a launch
// the steps of the different tables run in a seeded random order, so a table whose step read or wrote another table's part of the
// work buffer would not give what it gives alone (the tests compare bit for bit with the single-table emulation).  The device clears
// the whole work buffer (backward store, projection buffers, accumulators); here the spare double behind the group's backward store,
// which the plan never reads, and a guard behind the buffer stay NaN, so a read past the store or past the buffer shows as NaN.
// A table that fits no group runs whmec_genotype's path under the same budget (emul_gl_bounded.cpp).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <limits>
#include <random>
#include <string>
#include <vector>

#include "../../whatshap_b200/csrc/gl_batch.h"

using namespace whmec;

extern "C" int whemul_genotype_bounded(const whmec_problem *p, double *likelihoods, uint64_t budget_doubles, uint32_t *n_segments, char *err,
                                       size_t errlen);

namespace {

void set_err(char *err, size_t errlen, const std::string &msg) {
    if (err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = 0;
    }
}

constexpr uint64_t GUARD = 64;  // NaN doubles behind the work buffer

// one group: one clear of the work buffer, the launches of its step list, the posteriors normalised into the callers' arrays
void run_group(const GlBatchGroup &gp, double *const *likelihoods, std::mt19937_64 &rng) {
    const double nan = std::numeric_limits<double>::quiet_NaN();
    const uint64_t work = gp.store_doubles + gp.f_pool_doubles + gp.acc_doubles;
    std::vector<double> buf(work + GUARD, nan);
    std::fill(buf.begin(), buf.begin() + work, 0.0);
    buf[gp.store_doubles - 1] = nan;  // the spare double behind the last table's backward tables (a last column points there)
    double *beta = buf.data(), *F = beta + gp.store_doubles, *acc = F + gp.f_pool_doubles;
    const GlBatchInputs in{gp.cols.data(), gp.eps.data(), gp.allele.data(), gp.ind.data(), gp.h2p.data(), gp.trans.data(), gp.q.data()};
    auto add = [](double *addr, double val) { *addr += val; };
    auto order = [&](uint32_t e0, uint32_t e1) {
        std::vector<uint32_t> o(e1 - e0);
        for (uint32_t e = e0; e < e1; ++e) o[e - e0] = e;
        std::shuffle(o.begin(), o.end(), rng);
        return o;
    };
    for (size_t l = 0; l + 1 < gp.bwd_begin.size(); ++l) {
        for (uint32_t e : order(gp.bwd_begin[l], gp.bwd_begin[l + 1])) {  // gl_batch_backward_kernel
            const GlStep &st = gp.steps[e];
            const GlBatchTable &d = gp.tables[gp.step_table[e]];
            const GlView v = gl_batch_view(in, d);
            for (uint64_t x = 0; x < ((uint64_t)1 << st.cells_log2); ++x)
                gl_backward_cell(v, st.k, (uint32_t)x, beta + d.beta_base + v.cols[st.k].beta_off, beta + st.cur_off, add);
        }
        for (uint32_t e : order(gp.bwd_begin[l], gp.bwd_begin[l + 1])) gl_scale_host(beta + gp.steps[e].cur_off, gp.steps[e].n_scale);
    }
    for (size_t l = 0; l + 1 < gp.fwd_begin.size(); ++l) {
        for (uint32_t e : order(gp.fwd_begin[l], gp.fwd_begin[l + 1])) {  // gl_batch_forward_kernel
            const GlStep &st = gp.steps[e];
            const GlBatchTable &d = gp.tables[gp.step_table[e]];
            const GlView v = gl_batch_view(in, d);
            for (uint64_t x = 0; x < ((uint64_t)1 << st.cells_log2); ++x)
                gl_forward_cell(v, st.k, (uint32_t)x, F + st.prev_off, F + st.cur_off, beta + d.beta_base + v.cols[st.k].beta_off,
                                acc + d.acc_base + (size_t)st.k * d.n_ind * 3, add);
        }
        for (uint32_t e : order(gp.fwd_begin[l], gp.fwd_begin[l + 1])) {  // gl_scale_kernel
            const GlStep &st = gp.steps[e];
            gl_scale_host(F + st.cur_off, st.n_scale);
            std::fill(F + st.prev_off, F + st.prev_off + st.n_clear, 0.0);
        }
    }
    for (size_t m = 0; m < gp.members.size(); ++m) {
        const GlBatchTable &d = gp.tables[m];
        gl_normalise(acc + d.acc_base, d.n_cols, d.n_ind, likelihoods[gp.members[m]]);
    }
}

}  // namespace

// What whmec_genotype_batch runs when `budget_doubles` (0: no limit) is the budget of a group.  status / errs as the C ABI;
// group_of[t] = the group of table t (UINT32_MAX: none; an error, no columns, or a table run alone); info = {groups, launches
// of the groups, tables run alone}.
extern "C" int whemul_genotype_batch(const whmec_problem *const *problems, double *const *likelihoods, uint32_t n, uint64_t budget_doubles,
                                     uint64_t seed, int *status, char *errs, size_t errlen, uint32_t *group_of, uint32_t *info) {
    std::vector<Packed> pks(n);
    std::vector<GlPacked> gs(n);
    std::vector<uint64_t> cost(n, 0);
    auto err_of = [&](uint32_t t) { return errs ? errs + (size_t)t * errlen : nullptr; };
    for (uint32_t t = 0; t < n; ++t) {
        group_of[t] = UINT32_MAX;
        std::string m;
        const int rc = problems[t] && likelihoods[t] ? gl_pack(problems[t], pks[t], gs[t], m) : (m = "null argument", WHMEC_ERR_INPUT);
        status[t] = rc;
        set_err(err_of(t), errlen, rc == WHMEC_OK ? "" : m);
        if (rc == WHMEC_OK && pks[t].n > 0) cost[t] = gl_batch_cost(pks[t], gs[t]);
    }
    std::vector<std::vector<uint32_t>> groups;
    std::vector<uint32_t> alone;
    gl_batch_groups(cost, budget_doubles ? budget_doubles : ~0ull, groups, alone);
    std::mt19937_64 rng(seed);
    info[0] = (uint32_t)groups.size();
    info[1] = 0;
    info[2] = (uint32_t)alone.size();
    for (uint32_t q = 0; q < groups.size(); ++q) {
        GlBatchGroup gp;
        gl_batch_plan(pks, gs, groups[q], gp);
        run_group(gp, likelihoods, rng);
        info[1] += gp.launches;
        for (uint32_t t : groups[q]) group_of[t] = q;
    }
    for (uint32_t t : alone) {
        std::vector<char> e(errlen ? errlen : 1, 0);
        status[t] = whemul_genotype_bounded(problems[t], likelihoods[t], budget_doubles, nullptr, e.data(), e.size());
        set_err(err_of(t), errlen, e.data());
    }
    return WHMEC_OK;
}

// Doubles table `p` takes in a group (gl_batch_cost); 0 for a table with an input error or without columns.
extern "C" uint64_t whemul_gl_batch_cost(const whmec_problem *p) {
    Packed pk;
    GlPacked g;
    std::string msg;
    return gl_pack(p, pk, g, msg) == WHMEC_OK && pk.n > 0 ? gl_batch_cost(pk, g) : 0;
}
