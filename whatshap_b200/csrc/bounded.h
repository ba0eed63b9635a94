// Segment cutter of the memory-bounded column / pedigree sweep (col_plan.cpp, DESIGN §4.2): when the back-pointers of the whole
// table exceed the budget, the table is cut into segments that share one arena.  Host only, so that the test harness
// (tests/emul) checks the cuts on the CPU.
//
//   col_off[k]  word offset of column k's back-pointers in the resident layout (pack.cpp), col_off[n] = the resident size:
//               column k owns words [col_off[k], col_off[k + 1]).
//
// Both cutters work greedily from the end of the table, as the tile planner does (§4.1e): the last segment, whose
// back-pointers are left in the arena by the forward sweep, is as large as fits.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

namespace whmec {

// Two-pass paths (fused trio sweep, batched sweep): segments of whole chains, no checkpoints.  chain_begin holds the first
// column of every chain and n at the end.  Fills chain_cuts (ascending chain indices, 0 first, n_chains last) and the arena
// (the largest segment, words).  False when a single chain alone exceeds the budget.
inline bool cut_chain_segments(const std::vector<uint32_t> &chain_begin, const std::vector<uint64_t> &col_off, uint64_t budget_words,
                               std::vector<uint32_t> &chain_cuts, uint64_t &arena_words) {
    const uint32_t C = (uint32_t)chain_begin.size() - 1;
    chain_cuts.assign(1, C);
    arena_words = 0;
    uint32_t hi = C;  // the open segment is chains [c, hi)
    for (uint32_t c = C; c-- > 0;) {
        const uint64_t own = col_off[chain_begin[c + 1]] - col_off[chain_begin[c]];
        if (own > budget_words) return false;
        if (col_off[chain_begin[hi]] - col_off[chain_begin[c]] > budget_words) {
            chain_cuts.push_back(c + 1);
            hi = c + 1;
        }
    }
    chain_cuts.push_back(0);
    std::reverse(chain_cuts.begin(), chain_cuts.end());
    for (size_t s = 0; s + 1 < chain_cuts.size(); ++s)
        arena_words = std::max(arena_words, col_off[chain_begin[chain_cuts[s + 1]]] - col_off[chain_begin[chain_cuts[s]]]);
    return true;
}

// Sequential column path: segments of columns; segment s >= 1 starts from a checkpoint of the values that column
// cuts[s] - 1 hands on (ckpt_words[k]: size of column k's output, 2^f * T).  The budget covers the arena and all
// checkpoints (ckpt_words empty: the arena alone).  Fills col_cuts (0 first, n last), the arena and the checkpoints' total
// (words).  False when no cut fits.
inline bool cut_column_segments(const std::vector<uint64_t> &col_off, const std::vector<uint64_t> &ckpt_words, uint64_t budget_words,
                                std::vector<uint32_t> &col_cuts, uint64_t &arena_words, uint64_t &ckpt_total) {
    const uint32_t n = (uint32_t)col_off.size() - 1;
    uint64_t widest = 0;
    for (uint32_t k = 0; k < n; ++k) widest = std::max(widest, col_off[k + 1] - col_off[k]);
    // cut with an arena of `cap` words; the checkpoints it needs come on top.  A smaller arena means more checkpoints: lower the
    // arena by what the checkpoints overshoot until both fit (cap only decreases, so this ends).
    auto cut = [&](uint64_t cap) {
        col_cuts.assign(1, n);
        arena_words = ckpt_total = 0;
        uint32_t hi = n;
        for (uint32_t k = n; k-- > 0;) {
            if (col_off[hi] - col_off[k] > cap) {
                arena_words = std::max(arena_words, col_off[hi] - col_off[k + 1]);
                if (!ckpt_words.empty()) ckpt_total += ckpt_words[k];  // segment [k + 1, hi) starts from column k's output
                col_cuts.push_back(k + 1);
                hi = k + 1;
            }
        }
        arena_words = std::max(arena_words, col_off[hi] - col_off[0]);
        col_cuts.push_back(0);
        std::reverse(col_cuts.begin(), col_cuts.end());
    };
    uint64_t cap = budget_words;
    for (int round = 0; cap >= widest && cap > 0; ++round) {
        cut(cap);
        if (arena_words + ckpt_total <= budget_words) return true;
        cap = std::min(cap - 1, budget_words > ckpt_total ? budget_words - ckpt_total : 0);
        if (round >= 16) cap = std::min(cap, cap - cap / 16);  // many tiny checkpoints: stop creeping, shrink geometrically
    }
    return false;
}

}  // namespace whmec
