// The parts of the row-limited heuristic (heuristic.cpp) that whmec_heuristic and whmec_heuristic_batch share: the constructor
// part of a table (validation, sample ids, recombination and mutation costs, where reads start) and the output pass (votes of
// the chosen bipartition, best phasing of every column).  Host C++.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/whmec.h"

namespace whmec {

using HeurScore = float;                       // MecScore (src/mecheader.h)
constexpr uint32_t HEUR_MAX_ROWS = 65535;      // MAX_ROW_LIMIT

struct HeurTable {
    const whmec_problem *p = nullptr;
    uint32_t n = 0, m = 0, S = 0, n_trios = 0, tm_bits = 0;
    bool distrust = false, allow_mut = true;
    std::vector<HeurScore> rc, mc;         // recombination / mutation cost per column
    std::vector<uint32_t> first, last;     // column span of every read
    std::vector<uint32_t> sample_of_read;  // index into the sorted sample list
    std::vector<uint32_t> trios;           // [3 * n_trios] as sample indices
    std::vector<int> gt;                   // [S][n]  0 / 1 / 2
    std::vector<uint32_t> start;           // [n + 1] first read that starts after column k - 1
    std::vector<uint8_t> seen;             // [S] the first read of a sample that is not a child always goes to side 0

    // best joint phasing of one column given the votes of all sample haplotypes (getOptPhasing, :462-560)
    HeurScore best_phasing(const std::vector<HeurScore> &v, uint32_t t, uint32_t col, int8_t *alleles, uint8_t *mutated) const;
};

// The constructor part (:9-81): fills `tb` from `p`, writes out->n_samples and out->score.  An error code (message in `err`) for
// malformed input.  With S == 0 (no reads and no trios) the table is complete: out->transmission is zeroed, `start` and `seen`
// stay empty.
int heur_prepare(HeurTable &tb, const whmec_problem *p, bool allow_mut, whmec_heuristic_solution *out, std::string &err);

// The output pass after the backtrace: `part` [m] and `tv` [n] (masked to the trio bits) go to out->partition /
// out->transmission, then the votes of every read under `part` give each column's best phasing (haplotypes, mutations).
void heur_finish(const HeurTable &tb, const uint8_t *part, const uint32_t *tv, whmec_heuristic_solution *out);

}  // namespace whmec
