// Row-limited heuristic PedMEC solver: `whmec_heuristic` of include/whmec.h (host C++; no CUDA in this translation unit).
//
// Restates the behaviour of the reference's PedMecHeuristic (src/pedmecheuristic.cpp:9-81 constructor, :121-409 solve,
// :411-630 helpers; Python surface whatshap/core.pyx:674-734) on the flat arrays of `whmec_problem`: a beam search that walks the
// columns left to right, keeps at most `row_limit` partial solutions (a side for every active read, a transmission value, per
// sample and haplotype a window of signed allele votes), extends every solution by the reads that start in the column, prunes by
// score and records back-pointers.  All scores are `float` and every expression below keeps the reference's operand types and
// order, so that the results (bipartition, transmission vector, haplotypes, mutations) are identical bit for bit; the quirks that
// follow from the reference's code are kept and marked (Q1..Q4).
//
//   Q1  getOptScore() returns a member that solve() never assigns: the reported score is 0 (pedmecheuristic.cpp:84-86).
//   Q2  with allow_mutations == false the mutation cost is +inf and `false * inf` is NaN (:463-464, :521-522): kept as computed.
//   Q3  sample s of the sorted id list reads the genotypes of pedigree INDEX s (:72-80): ids must be 0 .. S-1.
//   Q4  a transmission variant of a solution (extendSolutions) carries its new reads' sides twice after finalize(); only the
//       first |active| entries are ever read (:163-166), so the duplicate tail is not represented here.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <string>
#include <unordered_map>
#include <vector>

#include "heuristic.h"

using namespace whmec;

namespace {

using Score = HeurScore;
constexpr uint32_t MAX_ROWS = HEUR_MAX_ROWS;

struct Partial {
    std::vector<uint8_t> side;    // side of every read that was active at the end of the previous column (kept reads first)
    std::vector<uint8_t> placed;  // sides given to the reads that start in the current column, in read order
    uint32_t tv = 0;
    Score score = 0, mut = 0;
    uint16_t from = 0;            // row of the previous column this solution continues
    std::vector<Score> votes;     // [2 * S][W]: signed votes (positive: allele 1) per sample haplotype and window column
};

struct Solver : HeurTable {
    uint32_t row_limit, W = 1;

    Score &vote(Partial &q, uint32_t row, uint32_t i) const { return q.votes[(size_t)row * W + i]; }
    Score vote(const Partial &q, uint32_t row, uint32_t i) const { return q.votes[(size_t)row * W + i]; }

    // votes against the transmission `t` between parents and children over window columns 0 .. ahead (getMutationCost, :429-459)
    Score mutation_cost(const Partial &q, uint32_t t, uint32_t col, bool flips, size_t ahead) const {
        Score cost = 0.0;
        const size_t lastw = std::min(ahead, (size_t)W - 1);
        for (size_t i = 0; i <= lastw; ++i)
            for (uint32_t k = 0; k < n_trios; ++k) {
                const uint32_t a = trios[3 * k], b = trios[3 * k + 1], c = trios[3 * k + 2];
                const uint32_t sel_a = (t >> (2 * k)) & 1, sel_b = (t >> (2 * k + 1)) & 1;
                const Score ca = vote(q, 2 * c, (uint32_t)i), cb = vote(q, 2 * c + 1, (uint32_t)i);
                const Score pa = vote(q, 2 * a + sel_a, (uint32_t)i), pb = vote(q, 2 * b + sel_b, (uint32_t)i);
                if (flips) {
                    if (ca * pa < 0) cost += std::min(mc[col], std::min(std::abs(ca), std::abs(pa)));
                    if (cb * pb < 0) cost += std::min(mc[col], std::min(std::abs(cb), std::abs(pb)));
                } else {
                    cost += (ca * pa < 0) * mc[col];
                    cost += (cb * pb < 0) * mc[col];
                }
            }
        return cost;
    }

    // adds the votes of a read to one haplotype of its sample; returns the score the placement costs (addBalance, :562-585)
    Score add_votes(Partial &q, uint32_t row, uint32_t other, const std::vector<Score> &add, const int *target) const {
        Score penalty = 0;
        for (uint32_t i = 0; i < W; ++i) {
            Score &basis = vote(q, row, i);
            const Score co = vote(q, other, i);
            if (distrust) {
                if (basis * add[i] < 0) penalty += std::min(std::abs(basis), std::abs(add[i]));
            } else if (target[i] == 1) {
                if (add[i] <= 0) penalty += std::min(-add[i], std::max(basis - co, (Score)0));
                else penalty += std::min(add[i], std::max(co - basis, (Score)0));
            } else {
                penalty += std::abs(add[i]) * (add[i] * (target[i] - 1) < 0);
            }
            basis += add[i];
        }
        return penalty;
    }

    // keeps the solutions below the (row_limit + 1)-th best total, and all optimal ones (filterSolutions, :611-630)
    void prune(std::vector<Partial> &sols) const {
        std::vector<Score> totals(sols.size());
        for (size_t i = 0; i < sols.size(); ++i) totals[i] = sols[i].score + sols[i].mut;
        std::vector<Score> sorted = totals;
        std::sort(sorted.begin(), sorted.end());
        const Score too_high = sorted.size() > row_limit ? sorted[row_limit] : std::numeric_limits<Score>::infinity();
        size_t kept = 0;
        for (size_t i = 0; i < sols.size(); ++i)
            if ((totals[i] < too_high || totals[i] == sorted[0]) && kept < MAX_ROWS) {
                if (kept != i) sols[kept] = std::move(sols[i]);
                ++kept;
            }
        sols.resize(kept);
    }

    int run(whmec_heuristic_solution *out, std::string &err);
};

int Solver::run(whmec_heuristic_solution *out, std::string &err) {
    // ---- constructor part (:9-81)
    {
        const int code = heur_prepare(*this, p, allow_mut, out, err);
        if (code != WHMEC_OK || S == 0) return code;
    }

    // ---- solve (:121-409)
    std::vector<Partial> prev(1);
    W = 1;
    prev[0].votes.assign(2 * (size_t)S, 0.0f);
    std::vector<uint32_t> active;
    std::vector<std::vector<uint16_t>> back(n);         // per column: row of the previous column
    std::vector<std::vector<uint8_t>> placed_all(n);    // per column: sides of the new reads of every row
    std::vector<std::vector<uint32_t>> tv_all(n);
    uint32_t right = 0;

    for (uint32_t col = 0; col < n; ++col) {
        // reads that are still active
        std::vector<uint32_t> kept;
        {
            std::vector<uint32_t> still;
            for (uint32_t i = 0; i < active.size(); ++i)
                if (last[active[i]] >= col) {
                    still.push_back(active[i]);
                    kept.push_back(i);
                }
            active.swap(still);
        }
        // solutions of the previous column without the reads that ended; equal ones merge into the first, which takes the
        // lowest score (and the votes and back-pointer that come with it)
        const uint32_t W_prev = W;
        std::vector<Partial> sols;
        {
            std::unordered_map<std::string, uint32_t> where;
            std::string key;
            for (uint32_t i = 0; i < prev.size(); ++i) {
                const Partial &old = prev[i];
                key.assign((const char *)&old.tv, 4);
                for (uint32_t a : kept) key.push_back((char)old.side[a]);
                auto it = where.find(key);
                uint32_t j;
                if (it == where.end()) {
                    j = (uint32_t)sols.size();
                    where.emplace(key, j);
                    sols.emplace_back();
                    Partial &q = sols.back();
                    q.side.assign(key.begin() + 4, key.end());
                    q.tv = old.tv;
                    q.score = std::numeric_limits<Score>::infinity();
                    q.votes.assign(2 * (size_t)S, 0.0f);  // one window column of zeros, replaced below unless the score is NaN
                    q.from = 0;
                } else {
                    j = it->second;
                }
                Partial &q = sols[j];
                if (q.score > old.score) {
                    q.score = old.score;
                    q.from = (uint16_t)i;
                    // the window moves on by one column
                    const uint32_t w = W_prev > 0 ? W_prev - 1 : 0;
                    q.votes.assign(2 * (size_t)S * w, 0.0f);
                    for (uint32_t row = 0; row < 2 * S; ++row)
                        for (uint32_t x = 0; x < w; ++x) q.votes[(size_t)row * w + x] = old.votes[(size_t)row * W_prev + x + 1];
                }
            }
        }
        // window of this column: up to the last column of any read seen so far
        right = std::max(right, col);
        for (uint32_t r = start[col]; r < start[col + 1]; ++r) right = std::max(right, last[r]);
        const uint32_t W_new = right + 1 - col;
        for (Partial &q : sols) {
            const uint32_t w_old = (uint32_t)(q.votes.size() / (2 * (size_t)S));
            std::vector<Score> wide(2 * (size_t)S * W_new, 0.0f);
            for (uint32_t row = 0; row < 2 * S; ++row)
                for (uint32_t x = 0; x < std::min(w_old, W_new); ++x) wide[(size_t)row * W_new + x] = q.votes[(size_t)row * w_old + x];
            q.votes.swap(wide);
        }
        W = W_new;

        // votes of the reads that start here; a read whose votes agree in sign and support with an earlier new read of the
        // same sample is merged into that read and later placed on the same side
        const uint32_t n_new = start[col + 1] - start[col];
        std::vector<int> equal_to(n_new, -1);
        std::vector<std::vector<Score>> add(n_new);
        for (uint32_t i = 0; i < n_new; ++i) {
            const uint32_t r = start[col] + i;
            active.push_back(r);
            std::vector<Score> b(W, 0.0f);
            for (uint64_t e = p->read_off[r]; e < p->read_off[r + 1]; ++e) {
                const uint32_t o = p->ent_col[e] - col;
                const int8_t a = (int8_t)p->ent_allele[e];
                const Score q = (Score)(int)p->ent_phred[e];
                b[o] += q * a - q * (1 - a);
            }
            for (uint32_t j = 0; j < i; ++j) {
                if (equal_to[j] != -1 || sample_of_read[start[col] + j] != sample_of_read[r]) continue;
                bool same = true;
                for (uint32_t x = 0; x < W; ++x)
                    if (add[j][x] * b[x] < 0 || (add[j][x] != 0.0) != (b[x] != 0.0)) {
                        same = false;
                        break;
                    }
                if (same) {
                    equal_to[i] = (int)j;
                    for (uint32_t x = 0; x < W; ++x) add[j][x] += b[x];
                    break;
                }
            }
            add[i] = std::move(b);
        }

        for (uint32_t i = 0; i < n_new; ++i) {
            const uint32_t s = sample_of_read[start[col] + i];
            const int *target = &gt[(size_t)s * n + col];
            const std::vector<Score> &b = add[i];
            const uint32_t count = (uint32_t)sols.size();
            for (uint32_t x = 0; x < count; ++x) {
                if (equal_to[i] >= 0) {
                    sols[x].placed.push_back(sols[x].placed[equal_to[i]]);
                    continue;
                }
                // a read that neither touches a heterozygous column (trusted genotypes) nor can change a consensus (distrusted)
                // is not branched on: it goes where it fits better
                bool useful = false;
                if (distrust) {
                    for (uint32_t j = 0; j < W && !useful; ++j) {
                        const Score s0 = vote(sols[x], 2 * s, j), s1 = vote(sols[x], 2 * s + 1, j);
                        useful |= (b[j] != 0 && s0 * s1 < 0) || ((b[j] + s0) * s0 <= 0 && (b[j] + s1) * s1 <= 0);
                    }
                } else {
                    for (uint32_t j = 0; j < W && !useful; ++j) useful |= (target[j] == 1 && b[j] != 0);
                }
                uint32_t twin = 0;
                if (seen[s]) {
                    Partial copy = sols[x];
                    sols.push_back(std::move(copy));
                    twin = (uint32_t)sols.size() - 1;
                    Partial &t = sols[twin];
                    t.score += add_votes(t, 2 * s + 1, 2 * s, b, target);
                    t.mut = mutation_cost(t, t.tv, col, true, 5);
                    t.placed.push_back(1);
                }
                Partial &q = sols[x];
                q.score += add_votes(q, 2 * s, 2 * s + 1, b, target);
                q.mut = mutation_cost(q, q.tv, col, true, 5);
                q.placed.push_back(0);
                if (twin && !useful) {
                    if (q.score + q.mut > sols[twin].score + sols[twin].mut) sols[x] = sols[twin];
                    sols.pop_back();
                }
            }
            seen[s] = 1;
            if (sols.size() > row_limit) prune(sols);
        }
        // other transmission values for solutions that pay for mutations here (extendSolutions, :587-609)
        {
            const uint32_t count = (uint32_t)sols.size();
            for (uint32_t x = 0; x < count; ++x) {
                sols[x].mut = mutation_cost(sols[x], sols[x].tv, col, false, 0);
                if (sols[x].mut > 0) {
                    for (uint32_t t = 0; t < std::pow(2, tm_bits); ++t) {
                        if (t == sols[x].tv) continue;
                        const Score cost = rc[col] * (Score)__builtin_popcountll((uint64_t)(sols[x].tv ^ t));
                        if (cost >= sols[x].mut) continue;
                        const Score other = mutation_cost(sols[x], t, col, false, 0);
                        if (other + cost >= sols[x].mut) continue;
                        Partial v = sols[x];
                        v.tv = t;
                        v.score = sols[x].score + cost;
                        v.mut = other;
                        sols.push_back(std::move(v));  // (Q4)
                    }
                }
            }
            if (sols.size() > row_limit) prune(sols);
        }
        // the column itself is settled: cost of its best joint phasing under the solution's votes
        {
            std::vector<Score> firsts(2 * (size_t)S);
            for (Partial &q : sols) {
                for (uint32_t row = 0; row < 2 * S; ++row) firsts[row] = vote(q, row, 0);
                q.score += best_phasing(firsts, q.tv, col, nullptr, nullptr);
            }
        }
        if (sols.empty()) {
            // every total is NaN (allow_mutations == false: `false * inf`, Q2) and NaN survives no comparison of the pruning step;
            // the reference walks back through empty columns here (undefined)
            err = "the heuristic kept no solution (scores are not numbers: allow_mutations = false is not usable, as in the reference)";
            return WHMEC_ERR_UNSUPPORTED;
        }
        // record the column
        back[col].reserve(sols.size());
        placed_all[col].reserve(sols.size() * n_new);
        tv_all[col].reserve(sols.size());
        for (Partial &q : sols) {
            back[col].push_back(q.from);
            placed_all[col].insert(placed_all[col].end(), q.placed.begin(), q.placed.end());
            tv_all[col].push_back(q.tv);
            q.side.insert(q.side.end(), q.placed.begin(), q.placed.end());
            q.placed.clear();
        }
        prev.swap(sols);
    }

    // best row of the last column (first minimum), walk back
    uint32_t row = 0;
    {
        Score best = std::numeric_limits<Score>::infinity();
        for (uint32_t i = 0; i < prev.size(); ++i)
            if (prev[i].score < best) {
                best = prev[i].score;
                row = i;
            }
    }
    std::vector<uint8_t> part(m, 0);
    std::vector<uint32_t> tv(n, 0);
    for (uint32_t col = n; col-- > 0;) {
        const uint32_t n_new = start[col + 1] - start[col];
        for (uint32_t i = 0; i < n_new; ++i) part[start[col] + i] = placed_all[col][(size_t)n_new * row + i];
        tv[col] = tm_bits ? (tv_all[col][row] & (uint32_t)((1ull << tm_bits) - 1)) : 0u;
        row = back[col][row];
    }
    heur_finish(*this, part.data(), tv.data(), out);
    return WHMEC_OK;
}

}  // namespace

namespace whmec {

// best joint phasing of one column given the votes of all sample haplotypes (getOptPhasing, :462-560)
HeurScore HeurTable::best_phasing(const std::vector<HeurScore> &v, uint32_t t, uint32_t col, int8_t *alleles, uint8_t *mutated) const {
    using Score = HeurScore;
    std::vector<Score> pc((size_t)S * 5);
    for (uint32_t s = 0; s < S; ++s) {
        const Score a0 = v[2 * s], a1 = v[2 * s + 1];
        Score *c = &pc[(size_t)s * 5];
        c[0] = (a0 * (a0 > 0) + a1 * (a1 > 0));
        c[1] = (-a0 * (a0 < 0) + a1 * (a1 > 0));
        c[2] = (a0 * (a0 > 0) - a1 * (a1 < 0));
        c[3] = (-a0 * (a0 < 0) - a1 * (a1 < 0));
        c[4] = *std::max_element(c, c + 4);
    }
    // allowed phasings per sample: 0 = 0|0, 1 = 0|1, 2 = 1|0, 3 = 1|1
    std::vector<std::vector<int>> ph(S);
    for (uint32_t s = 0; s < S; ++s) {
        if (distrust) {
            for (int i = 0; i < 4; ++i)
                if (pc[(size_t)s * 5 + i] < pc[(size_t)s * 5 + 4] + 2 * mc[col]) ph[s].push_back(i);
        } else {
            const int g = gt[(size_t)s * n + col];
            if (g == 0) ph[s].push_back(0);
            else if (g == 2) ph[s].push_back(3);
            else {
                ph[s].push_back(1);
                ph[s].push_back(2);
            }
        }
    }
    Score best = std::numeric_limits<Score>::infinity();
    // (a sample without any allowed phasing -- possible with distrusted genotypes where the mutation cost is 0 -- makes the
    //  reference index an empty vector, :505-530; here such a column has no finite phasing)
    for (uint32_t s = 0; s < S; ++s)
        if (ph[s].empty()) return best;
    std::vector<size_t> ctr(S, 0);
    std::vector<uint8_t> mut(2 * (size_t)S);
    while (ctr[S - 1] < ph[S - 1].size()) {
        Score cost = 0.0;
        std::fill(mut.begin(), mut.end(), 0);
        for (uint32_t k = 0; k < n_trios; ++k) {
            const uint32_t a = trios[3 * k], b = trios[3 * k + 1], c = trios[3 * k + 2];
            const uint32_t sel_a = (t >> (2 * k)) & 1, sel_b = (t >> (2 * k + 1)) & 1;
            const int child = ph[c][ctr[c]];
            const int8_t ca = child & 1, cb = (child & 2) >> 1;
            const int8_t pa = (ph[a][ctr[a]] & (1 + sel_a)) >> sel_a;
            const int8_t pb = (ph[b][ctr[b]] & (1 + sel_b)) >> sel_b;
            cost += (pa != ca) * mc[col];
            cost += (pb != cb) * mc[col];
            mut[2 * c] = (pa != ca);
            mut[2 * c + 1] = (pb != cb);
        }
        for (uint32_t s = 0; s < S; ++s) cost += pc[(size_t)s * 5 + ph[s][ctr[s]]];
        if (cost < best) {
            best = cost;
            if (alleles)
                for (uint32_t s = 0; s < S; ++s) {
                    alleles[2 * s] = ph[s][ctr[s]] & 1;
                    alleles[2 * s + 1] = (ph[s][ctr[s]] & 2) >> 1;
                }
            if (mutated) std::copy(mut.begin(), mut.end(), mutated);
        }
        ++ctr[0];
        for (uint32_t j = 0; j + 1 < S; ++j)
            if (ctr[j] >= ph[j].size()) {
                ctr[j] = 0;
                ++ctr[j + 1];
            }
    }
    return best;
}

// constructor part (:9-81) and the start of solve (:121-140)
int heur_prepare(HeurTable &tb, const whmec_problem *p, bool allow_mut, whmec_heuristic_solution *out, std::string &err) {
    using Score = HeurScore;
    tb.p = p;
    tb.allow_mut = allow_mut;
    uint32_t &n = tb.n, &m = tb.m, &S = tb.S, &n_trios = tb.n_trios;
    std::vector<Score> &rc = tb.rc, &mc = tb.mc;
    std::vector<uint32_t> &first = tb.first, &last = tb.last, &sample_of_read = tb.sample_of_read, &trios = tb.trios;
    std::vector<int> &gt = tb.gt;
    n = p->n_cols;
    m = p->n_reads;
    n_trios = p->n_trios;
    tb.tm_bits = 2 * n_trios;
    tb.distrust = p->distrust != 0;
    if (n > 0 && (!p->recombcost || !p->gt)) {
        err = "recombcost and genotypes must be given for every column";
        return WHMEC_ERR_INPUT;
    }
    if (m > 0 && (!p->read_off || !p->ent_col || !p->ent_allele || !p->ent_phred || !p->read_ind)) {
        err = "read arrays must not be null";
        return WHMEC_ERR_INPUT;
    }
    if (n_trios > 15) {
        err = "unsupported pedigree: more than 15 trio relationships";
        return WHMEC_ERR_UNSUPPORTED;
    }
    rc.assign(n, 0.0f);
    mc.assign(n, std::numeric_limits<Score>::infinity());
    for (uint32_t i = 1; i < n; ++i) {
        rc[i] = (Score)p->recombcost[i];  // (rc[0] stays 0: recombinations are free in the first column)
        if (allow_mut) mc[i - 1] = 0.75 * (rc[i - 1] + rc[i]);  // double product, stored as float
    }
    if (allow_mut && n > 0) mc[n - 1] = rc[n - 1] * 1.5;
    // sample ids: those of the reads and of the trio members, ascending (Q3)
    {
        std::vector<uint32_t> ids(p->read_ind, p->read_ind + m);
        for (uint32_t i = 0; i < 3 * n_trios; ++i) ids.push_back(p->trios[i]);
        std::sort(ids.begin(), ids.end());
        ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
        S = (uint32_t)ids.size();
        if (S > p->n_ind) {
            err = "sample ids must be the zero-based indices of the pedigree's individuals";
            return WHMEC_ERR_INPUT;
        }
        auto index_of = [&](uint32_t id) { return (uint32_t)(std::lower_bound(ids.begin(), ids.end(), id) - ids.begin()); };
        sample_of_read.resize(m);
        for (uint32_t r = 0; r < m; ++r) sample_of_read[r] = index_of(p->read_ind[r]);
        trios.resize(3 * (size_t)n_trios);
        for (uint32_t i = 0; i < 3 * n_trios; ++i) trios[i] = index_of(p->trios[i]);
    }
    out->n_samples = S;
    out->score = 0;  // Q1
    gt.assign((size_t)S * n, 0);
    for (uint32_t s = 0; s < S; ++s)
        for (uint32_t k = 0; k < n; ++k) {
            const uint8_t g = p->gt[(size_t)s * n + k];
            if (g > 2) {
                err = "the heuristic needs a diploid biallelic genotype for every sample and column";
                return WHMEC_ERR_INPUT;
            }
            gt[(size_t)s * n + k] = g;
        }
    first.resize(m);
    last.resize(m);
    for (uint32_t r = 0; r < m; ++r) {
        const uint64_t b = p->read_off[r], e = p->read_off[r + 1];
        if (e <= b) {
            err = "No variants present";
            return WHMEC_ERR_INPUT;
        }
        first[r] = p->ent_col[b];
        last[r] = p->ent_col[e - 1];
        if (last[r] >= n || first[r] > last[r] || (r > 0 && first[r] < first[r - 1])) {
            err = "reads must be sorted by their first column and lie inside the columns";
            return WHMEC_ERR_INPUT;
        }
    }
    if (S == 0) {  // no reads and no trios: nothing to phase (the reference indexes an empty vector here)
        if (out->transmission) std::fill(out->transmission, out->transmission + n, 0u);
        return WHMEC_OK;
    }
    std::vector<uint32_t> &start = tb.start;
    start.assign(1, 0);  // first read that starts after column k - 1
    {
        uint32_t q = 0;
        for (uint32_t k = 0; k < n; ++k) {
            while (q < m && first[q] <= k) ++q;
            start.push_back(q);
        }
    }
    tb.seen.assign(S, 0);  // the first read of a sample that is not a child always goes to side 0
    for (uint32_t k = 0; k < n_trios; ++k) tb.seen[trios[3 * k + 2]] = 1;
    return WHMEC_OK;
}

void heur_finish(const HeurTable &tb, const uint8_t *part, const uint32_t *tv, whmec_heuristic_solution *out) {
    using Score = HeurScore;
    const whmec_problem *p = tb.p;
    const uint32_t n = tb.n, m = tb.m, S = tb.S;
    const std::vector<uint32_t> &sample_of_read = tb.sample_of_read;
    if (out->partition) std::copy(part, part + m, out->partition);
    if (out->transmission) std::copy(tv, tv + n, out->transmission);

    // votes of all reads under the chosen bipartition, then the best phasing of every column
    std::vector<Score> votes((size_t)n * 2 * S, 0.0f);
    for (uint32_t r = 0; r < m; ++r)
        for (uint64_t e = p->read_off[r]; e < p->read_off[r + 1]; ++e) {
            const int8_t a = (int8_t)p->ent_allele[e];
            const Score q = (Score)(int)p->ent_phred[e];
            if (a >= 0) votes[(size_t)p->ent_col[e] * 2 * S + 2 * sample_of_read[r] + part[r]] += (2 * a - 1) * q;
        }
    std::vector<int8_t> alleles(2 * (size_t)S);
    std::vector<uint8_t> mutated(2 * (size_t)S);
    if (out->mutated) std::memset(out->mutated, 0, (size_t)S * 2 * n);
    for (uint32_t col = 0; col < n; ++col) {
        std::vector<Score> v(votes.begin() + (size_t)col * 2 * S, votes.begin() + (size_t)(col + 1) * 2 * S);
        std::fill(alleles.begin(), alleles.end(), 0);
        std::fill(mutated.begin(), mutated.end(), 0);
        tb.best_phasing(v, tv[col], col, alleles.data(), mutated.data());
        for (uint32_t s = 0; s < S; ++s)
            for (uint32_t h = 0; h < 2; ++h) {
                if (out->haplotypes) out->haplotypes[((size_t)s * 2 + h) * n + col] = alleles[2 * s + h];
                if (out->mutated) out->mutated[((size_t)s * 2 + h) * n + col] = mutated[2 * s + h];
            }
    }
}

}  // namespace whmec

extern "C" int whmec_heuristic(const whmec_problem *p, uint32_t row_limit, int allow_mutations, whmec_heuristic_solution *s, char *err,
                               size_t errlen) {
    std::string msg;
    int rc;
    try {
        Solver sv;
        sv.row_limit = std::min(row_limit, MAX_ROWS);
        sv.p = p;
        sv.allow_mut = allow_mutations != 0;
        rc = sv.run(s, msg);
    } catch (const std::bad_alloc &) {
        msg = "out of host memory";
        rc = WHMEC_ERR_UNSUPPORTED;
    }
    if (rc != WHMEC_OK && err && errlen) {
        std::strncpy(err, msg.c_str(), errlen - 1);
        err[errlen - 1] = 0;
    }
    return rc;
}
