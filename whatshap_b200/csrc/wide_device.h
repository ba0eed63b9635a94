// Per-thread pieces of the wide column sweep (T = 1024, five trios; DESIGN §4.7), host/device so that the test-only emulation
// (tests/emul/emul_wide.cpp) steps the same code the kernels run (whmec.cu: wide_xform_kernel, wide_step_kernel).
#pragma once
#include "common.h"
#include "dp_device.h"

namespace whmec {

constexpr uint32_t WIDE_TB = 10;  // log2(WIDE_T)

// Transition transform key of one previous value: (value, j) compared lexicographically, +inf as KEY_INF.
WHMEC_HD uint64_t wide_key(uint32_t value, uint32_t j) { return value == UMAX ? KEY_INF : ((uint64_t)value << 32) | j; }

// One hypercube relaxation step of the transform, key(i) <- min(key(i), key(i ^ 2^q) + rc).  After the rounds q = 0 .. tb-1 every j
// has reached i along exactly one path, with popcount(i ^ j) additions of rc: key(i) = min_j (prev[j] + popcount(i ^ j) * rc, j),
// which is transition_min (dp_device.h) with its smallest-j tie rule, as long as no sum reaches 2^32 - 1 (Packed::nowrap).
WHMEC_HD uint64_t wide_relax(uint64_t key, uint64_t other, uint32_t rc) {
    if (other == KEY_INF) return key;
    const uint64_t cand = other + ((uint64_t)rc << 32);
    return cand < key ? cand : key;
}

// Result of the transform: the transition minimum and its argmin (0 for an all-infinite row, as transition_min).
WHMEC_HD uint32_t wide_key_value(uint64_t key) { return (uint32_t)(key >> 32); }
WHMEC_HD uint16_t wide_key_arg(uint64_t key) { return key == KEY_INF ? (uint16_t)0 : (uint16_t)(key & 0xFFFFu); }

// log2 of the threads that share one projection entry of a wide column: at most 64 candidates per thread, and at least 2^20 threads
// per column where the entry's 2^d candidates allow it.
WHMEC_HD uint32_t wide_chunk_bits(uint32_t f, uint32_t d) {
    const uint32_t log_ent = f + WIDE_TB;
    uint32_t L = d > 6 ? d - 6 : 0;
    if (log_ent < 20 && 20 - log_ent > L) L = 20 - log_ent;
    return L < d ? L : d;
}

// Candidates [c * 2^(d - L), (c + 1) * 2^(d - L)) of entry (o, i): a min-key over them (dp_device.h: eval_candidates).
WHMEC_HD uint64_t wide_entry_key(const ColView &v, uint32_t o, uint32_t i, uint32_t c, uint32_t L) {
    const uint32_t per = 1u << (v.m->d - L);
    return eval_candidates<true>(v, o, i, c * per, (c + 1) * per);
}

}  // namespace whmec
