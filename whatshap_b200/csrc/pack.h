// Host-side packer and result builder (C++; no CUDA in this translation unit).
#pragma once
#include <stdint.h>
#include <string>
#include <vector>

#include "../../include/whmec.h"
#include "common.h"
#include "hostpool.h"

namespace whmec {

struct Packed {
    uint32_t n = 0, n_reads = 0, n_ind = 0, n_trios = 0;
    uint32_t T = 1, tb = 0, P = 2;
    bool has_deltas = true;              // fn_delta filled
    bool safe31 = false;                 // every reachable cost value < 2^30 (tile-kernel arithmetic is exact)
    bool nowrap = false;                 // every reachable value plus a column's transition cost < 2^32 - 1: no 32-bit sum wraps
                                         // (the wide path's transition transform is exact, DESIGN §4.7)
    // (RawVec: resize() does not zero-fill; every element is written by the packer)
    StagedVec<ColMeta> cols;             // [n]  (uploaded as it is: page-locked when the CUDA side installed its pool)
    // active reads per column, CSR aligned with cols[k].a
    RawVec<uint64_t> act_off;            // [n+1]
    RawVec<uint32_t> act_read;           // read index of bit j
    RawVec<uint8_t> act_allele;          // 0/1/2
    RawVec<uint32_t> act_phred;
    RawVec<uint8_t> act_ind;
    // cost functions (see common.h), grouped per column and transmission value
    StagedVec<uint32_t> fn_c0;
    StagedVec<int32_t> fn_delta;         // [nf][FN_STRIDE]
    RawVec<uint32_t> fn_asg;             // allele assignment A of the function
    RawVec<uint32_t> fn_base;            // genotype-likelihood base cost of A
    StagedVec<uint32_t> fn_group;        // per column T+1 offsets relative to cols[k].fn_off
    std::vector<int8_t> h2p;             // [T][n_ind][2]
    std::vector<uint32_t> read_first, read_last;  // column span of every read
    // chains: maximal runs of columns with f > 0 between them (T == 1 only uses them)
    std::vector<uint32_t> chain_begin;   // first column of each chain; chain c = [begin[c], begin[c+1])
    uint32_t max_d = 0;                  // most reads that end in one column
    uint64_t bp_words = 0;               // arena size in 32-bit words (column-kernel layout)
    whmec_stats stats{};
};

// Returns WHMEC_OK or an error code with a reference-compatible message in `err`.
// `want_deltas == false` skips the per-read deltas of the cost functions (the tile kernel does not use them).
int pack_problem(const whmec_problem *p, Packed &out, std::string &err, bool want_deltas = true);

// get_optimal_partitioning + get_super_reads from the optimal path (pedigreedptable.cpp:344-406).
int build_outputs(const Packed &pk, const uint32_t *path_index, const uint32_t *path_tv,
                  whmec_solution *s, std::string &err);

}  // namespace whmec
