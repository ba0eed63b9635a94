// TEST-ONLY plan inspector of the column-kernel paths: runs the host planner col_plan (col_plan.cpp) on a packed problem for
// given device figures and switches, so that tests/test_col_plan.py checks path choice and memory-bounded segments on the CPU.
// Built into tests/emul/libwhemul_col_plan.so by tests/emul/col_plan.mk.
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>

#include "../../whatshap_b200/csrc/col_plan.h"

using namespace whmec;

namespace {

int fail_with(const std::string &msg, char *err, size_t errlen, int code) {
    if (err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = 0;
    }
    return code;
}

}  // namespace

// Packs `p` with deltas, as plan creation does once the tile planner declines, and
// runs col_plan on the given device figures and switches.  info[9]: path (0 column, 1 batched, 2 fused), bounded, over_hbm,
// arena words, checkpoint words, the budget the segments were cut under (bytes), the plan's fixed bytes, the resident
// back-pointer words, the fused sweep's cluster size.  cuts: the chain cuts of a two-pass plan, else the column cuts; bp_off:
// every column's back-pointer offset as planned (rebased per segment when bounded).  Arrays hold `cap` >= columns + 1 entries.
extern "C" int whemul_col_plan(const whmec_problem *p, uint64_t free_bytes, uint64_t hook, int fused, int sequential, int segment,
                               int bounded_t1, uint32_t sms, uint32_t cluster, uint64_t *info, uint32_t *cuts, uint32_t *n_cuts,
                               uint32_t *chain_begin, uint32_t *n_chain_begin, uint64_t *bp_off, uint32_t cap, char *err, size_t errlen) {
    Packed pk;
    std::string msg;
    int rc = pack_problem(p, pk, msg, true);
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    if (pk.n == 0 || pk.n + 1 > cap) return fail_with("no columns, or arrays too small", err, errlen, WHMEC_ERR_INPUT);
    ColPlanInput in;
    in.free_bytes = free_bytes;
    in.hook = hook;
    in.fused = fused != 0;
    in.sequential = sequential != 0;
    in.segment = segment;
    in.bounded_t1 = bounded_t1 != 0;
    in.sms = sms;
    in.cluster = cluster;
    ColPlan plan;
    const uint64_t bp_words = pk.bp_words;
    rc = col_plan(pk, in, plan, msg);
    const uint64_t out[9] = {(uint64_t)plan.path, plan.bounded, plan.over_hbm, plan.arena_words, plan.ckpt_words, plan.budget_bytes,
                             plan.fixed_bytes, bp_words, plan.cluster};
    std::copy(out, out + 9, info);
    const std::vector<uint32_t> &c = plan.seg_chain.empty() ? plan.seg_col : plan.seg_chain;
    *n_cuts = (uint32_t)c.size();
    std::copy(c.begin(), c.end(), cuts);
    *n_chain_begin = (uint32_t)pk.chain_begin.size();
    std::copy(pk.chain_begin.begin(), pk.chain_begin.end(), chain_begin);
    for (uint32_t k = 0; k < pk.n; ++k) bp_off[k] = pk.cols[k].bp_off;
    if (rc != WHMEC_OK) return fail_with(msg, err, errlen, rc);
    return WHMEC_OK;
}
