// Votes of `whatshap haplotagphase` (whmec_haplotagphase, DESIGN §4.16): the per-entry key, the per-position walk and the choice
// rule, shared by the kernels of haplotagphase.cu and the host emulation tests/emul/emul_haplotagphase.cpp.
//
// An entry is one (position, allele, quality) of a read whose HP and PS tags count, at a heterozygous position, in read order.
// Its key is position << (ps_bits + 1) | ps rank << 1 | x with x = ht ^ allele_to_id[allele], and its chunk index as the value;
// after a stable sort a position's keys are contiguous, ascending by phase set and x, each run in read order.  A position's
// vote holds, per phase set in the order the reads first reached it, the keys (ps, 0) and (ps, 1); the best key has the highest
// score, ties going to the key inserted first.  The same rule chooses from runs handed over as (ps, h, score) in a dict's order.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define HP_HD __host__ __device__ __forceinline__
#else
#define HP_HD inline
#endif

namespace whmec {

// entry errors of the vote (all KeyError in the reference): a position missing from the table (found by the host plan), an
// allele missing from allele_to_id[position], and an id that makes ht ^ id a key the vote does not hold
enum HpEntryError : uint32_t { HP_OK = 0, HP_KEY_POSITION = 1, HP_KEY_ALLELE = 2, HP_KEY_HAPLOTYPE = 3 };
// position errors of the choice, as whmec_haplotagphase_output.error reports them
enum HpChoiceError : int32_t { HP_ZERO_DIVISION = 1, HP_KEY_ID = 2, HP_TOO_LARGE = 3, HP_EMPTY = 4 };

HP_HD uint64_t hp_error_code(uint64_t ordinal, uint32_t kind) { return ordinal << 2 | kind; }

struct HpEntry {
    int64_t allele;
    uint64_t ordinal;   // call-wide entry index (read order)
    uint32_t pos;       // chunk-local position
    uint32_t ps;        // dense phase-set rank within the sample
    int32_t quality;
    uint32_t ht;        // HP_tag - 1: 0 or 1
};

struct HpTable {               // every sample's positions (call-wide indices)
    const uint8_t *flags;      // HP_HOMOZYGOUS | HP_PHASED | HP_SNV (whmec_haplotagphase_input.pos_flags)
    const uint64_t *a2i_off;   // allele -> id pairs
    const int64_t *a2i_allele, *a2i_id;
    const uint64_t *i2a_off;   // id -> allele pairs
    const int64_t *i2a_id, *i2a_allele;
};
constexpr uint8_t HP_HOMOZYGOUS = 1, HP_PHASED = 2, HP_SNV = 4;

struct HpRecord {              // one (position, phase set) of a vote: its two keys' scores
    int64_t s0, s1;
    uint32_t ps;
    uint32_t first;            // the chunk index of its first entry
};

struct HpChoice {              // one position's outcome
    int64_t score, total;      // the best key's score and the sum of all (total valid below 2^53 in magnitude)
    int64_t ps, h;             // the best key (ps: the phase-set rank in the vote form)
    int64_t allele0, allele1;  // id_to_allele[h], id_to_allele[1 - h] of a kept position
    uint32_t first;            // vote form: the chunk index of the position's first entry
    uint32_t n_ps;             // vote form: its phase sets
    int32_t error;             // 0 or an HpChoiceError
    uint8_t voted, kept;
};

// The allele's id at position p, or an error (KeyError for an allele the position lacks, or for an id outside {0, 1}).
HP_HD uint32_t hp_lookup(const HpEntry &e, const HpTable &t, uint64_t p, uint32_t &x) {
    for (uint64_t a = t.a2i_off[p]; a < t.a2i_off[p + 1]; ++a) {
        if (t.a2i_allele[a] != e.allele) continue;
        const int64_t id = t.a2i_id[a];
        if (id < 0 || id > 1) return HP_KEY_HAPLOTYPE;
        x = e.ht ^ (uint32_t)id;
        return HP_OK;
    }
    return HP_KEY_ALLELE;
}

// The choice rule: the highest score, ties to the least insertion order; the total is exact (128 bits).
struct HpPick {
    int64_t best, ps, h;
    uint64_t order;
    __int128 total;
    uint32_t n;
    HP_HD void reset() { best = 0, ps = 0, h = 0, order = 0, total = 0, n = 0; }
    HP_HD void take(int64_t score, uint64_t ord, int64_t set, int64_t hap) {
        total += score;
        if (n == 0 || score > best || (score == best && ord < order)) best = score, order = ord, ps = set, h = hap;
        ++n;
    }
};

// i2a lookup of one id at position p (found: allele set)
HP_HD bool hp_allele(const HpTable &t, uint64_t p, int64_t id, int64_t &allele) {
    for (uint64_t a = t.i2a_off[p]; a < t.i2a_off[p + 1]; ++a)
        if (t.i2a_id[a] == id) {
            allele = t.i2a_allele[a];
            return true;
        }
    return false;
}

// consensus for one position p: q = score / total as a double, the gap and indel filters (a phased position is always taken),
// and the two alleles of a kept one.  The homopolymer filter of the reference never removes a position (it counts at most
// cut_poly bases and then asks for more than cut_poly), so it has no counterpart here.
HP_HD void hp_finish(const HpPick &k, const HpTable &t, uint64_t p, double gap_threshold, int only_indels, HpChoice &c) {
    c.score = k.best, c.ps = k.ps, c.h = k.h, c.kept = 0, c.error = 0, c.allele0 = c.allele1 = 0;
    const __int128 lim = (__int128)1 << 53;
    c.total = (k.total >= lim || k.total <= -lim) ? (k.total > 0 ? INT64_MAX : INT64_MIN) : (int64_t)k.total;
    if (k.n == 0) {
        c.error = HP_EMPTY;
        return;
    }
    if (k.total == 0) {
        c.error = HP_ZERO_DIVISION;
        return;
    }
    if (k.total >= lim || k.total <= -lim || k.best >= ((int64_t)1 << 53) || k.best <= -((int64_t)1 << 53)) {
        c.error = HP_TOO_LARGE;
        return;
    }
    const uint8_t f = t.flags[p];
    if (!(f & HP_PHASED)) {
        const double q = (double)k.best / (double)k.total;
        if (100.0 * q < gap_threshold) return;
        if (only_indels && (f & HP_SNV)) return;
    }
    c.kept = 1;
    if (!hp_allele(t, p, k.h, c.allele0) || !hp_allele(t, p, (int64_t)(1 - (uint64_t)k.h), c.allele1)) c.error = HP_KEY_ID;
}

// The vote of one chunk position from its sorted keys [k0, k1): per phase set its two scores and first entry, recorded at
// rec[k0 ..] with the sort key (position's first << ib | set's first) at rkey[k0 ..] (all ones on the slots left over), and
// the keys fed to the choice rule with the insertion order (set's first, x).
HP_HD HpChoice hp_walk(const uint64_t *keys, const uint32_t *vals, uint32_t k0, uint32_t k1, const HpEntry *en, uint32_t ps_bits,
                       uint32_t ib, HpRecord *rec, uint64_t *rkey, uint32_t *rval, HpPick &k) {
    k.reset();
    uint32_t n_ps = 0, first = UINT32_MAX;
    const uint64_t mask = ((uint64_t)1 << ps_bits) - 1;
    for (uint32_t i = k0; i < k1;) {
        const uint64_t set = keys[i] >> 1;
        int64_t s0 = 0, s1 = 0;  // (two scalars: an indexed pair would live in local memory)
        uint32_t f = UINT32_MAX;
        for (; i < k1 && keys[i] >> 1 == set; ++i) {
            const int64_t q = en[vals[i]].quality;
            if (keys[i] & 1) s1 += q;
            else s0 += q;
            f = vals[i] < f ? vals[i] : f;
        }
        const uint32_t ps = (uint32_t)(set & mask);
        k.take(s0, (uint64_t)f << 1, ps, 0);
        k.take(s1, (uint64_t)f << 1 | 1, ps, 1);
        rec[k0 + n_ps] = HpRecord{s0, s1, ps, f};
        rkey[k0 + n_ps] = f;
        first = f < first ? f : first;
        ++n_ps;
    }
    for (uint32_t j = k0; j < k1; ++j) {
        rkey[j] = j < k0 + n_ps ? (uint64_t)first << ib | rkey[j] : ~0ull;
        rval[j] = j;
    }
    HpChoice c{};
    c.first = first, c.n_ps = n_ps, c.voted = k1 > k0;
    return c;
}

// The choice from runs [r0, r1) handed over in a mapping's key order (the runs form).
HP_HD void hp_pick_runs(const int64_t *ps, const int64_t *h, const int64_t *score, uint64_t r0, uint64_t r1, HpPick &k) {
    k.reset();
    for (uint64_t r = r0; r < r1; ++r) k.take(score[r], r - r0, ps[r], h[r]);
}

}  // namespace whmec
