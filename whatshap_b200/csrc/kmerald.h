// Allele detection by k-mer re-alignment (whmec_realign_kmerald, whmec_kmer_align_batch, DESIGN §4.12): the per-job code shared
// by the kernels of realign.cu and the host emulation (tests/emul/emul_kmerald.cpp).
//
// A job aligns the k-mer list of one padded allele (rows, seq1 of kmer_align) against the k-mer list of the query window
// (columns, seq2), as ReadSetReader.realign(use_kmerald=True) does (whatshap/variants.py:731-794, align.pyx:199-271):
//   enumerate_all_kmers: a rolling 2-bit hash of the bytes A C G T; other bytes leave it as it is; a k-mer is listed at every
//                        position >= k - 1 whose hash is not 0;
//   kmer_align:          equal lists give 0; else both lists lose their common prefix and then their common suffix, and the
//                        float32 DP score[i][j] = min(match, score[i-1][j] + gap, score[i][j-1] + gap) runs over what is left,
//                        with borders gap * i and gap * j; match is score[i-1][j-1], plus costs[(a, b)], else costs[(a, -5)],
//                        else inf, when the k-mers a (row) and b (column) differ.
// The costs are one sorted table of keys (a << 32 | b), read k-mer 0 standing for -5; the row of ref k-mer a is a contiguous
// range of it, found once per DP row (ka_row), and a mismatching cell is a binary search inside that row (ka_cost).
// Every cell is computed from the same three operands in the same order whatever the traversal, so the one-thread row sweep
// (ka_short) and the warp's anti-diagonal wavefront over row bands (KaLane) give the reference's float32 values bit for bit.
#pragma once
#include <math.h>
#include <stdint.h>

#include "realign.h"

namespace whmec {

constexpr uint32_t KA_SHORT = 64;  // one thread: query window and padded allele both <= 64 bytes (so <= 64 k-mers each)

struct KaParams {
    uint32_t k;           // 1..15
    float gap;            // (float) gap_penalty
    const uint64_t *key;  // [n]: strictly ascending (ref k-mer << 32 | read k-mer), read k-mer 0 = the reference's -5
    const float *cost;    // [n]
    uint32_t n;
};

// enumerate_all_kmers(s, k) into out (at most s.len entries); returns the count
RA_HD uint32_t ka_kmers(const RaSeq &s, uint32_t k, uint32_t *out) {
    const uint32_t mask = (1u << (2 * k)) - 1;
    uint32_t h = 0, n = 0;
    for (uint32_t i = 0; i < s.len; ++i) {
        const uint8_t c = s.at(i);
        const int code = c == 'A' ? 0 : c == 'C' ? 1 : c == 'G' ? 2 : c == 'T' ? 3 : -1;
        if (code >= 0) h = ((h << 2) | (uint32_t)code) & mask;
        if (i + 1 >= k && h != 0) out[n++] = h;
    }
    return n;
}

// The trim of kmer_align on lists a[0..m), b[0..n): the common prefix x, then the common suffix.  Returns false when the lists
// are equal (distance 0); else m and n become the lengths of what is left, from a + x and b + x on.
RA_HD bool ka_trim(const uint32_t *a, const uint32_t *b, uint32_t &m, uint32_t &n, uint32_t &x) {
    x = 0;
    while (x < m && x < n && a[x] == b[x]) ++x;
    if (x == m && x == n) return false;
    while (m > x && n > x && a[m - 1] == b[n - 1]) --m, --n;
    m -= x, n -= x;
    return true;
}

// the first index in [lo, hi) whose key is >= want
RA_HD uint32_t ka_lower(const uint64_t *key, uint32_t lo, uint32_t hi, uint64_t want) {
    while (lo < hi) {
        const uint32_t mid = lo + (hi - lo) / 2;
        if (key[mid] < want) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

// The row of ref k-mer a: its entries [lo, hi) and its default costs[(a, -5)] (inf when missing).
struct KaRow {
    uint32_t lo, hi;
    float def;
};
RA_HD KaRow ka_row(const KaParams &p, uint32_t a) {
    KaRow r;
    r.lo = ka_lower(p.key, 0, p.n, (uint64_t)a << 32);
    r.hi = ka_lower(p.key, r.lo, p.n, (uint64_t)(a + 1) << 32);
    r.def = r.lo < r.hi && p.key[r.lo] == (uint64_t)a << 32 ? p.cost[r.lo] : INFINITY;
    return r;
}

// costs[(a, b)], else the row's default (b != 0: a real k-mer)
RA_HD float ka_cost(const KaParams &p, const KaRow &r, uint32_t a, uint32_t b) {
    const uint64_t want = (uint64_t)a << 32 | b;
    const uint32_t i = ka_lower(p.key, r.lo, r.hi, want);
    return i < r.hi && p.key[i] == want ? p.cost[i] : r.def;
}

// one DP cell in the reference's order: min(match, delete, insert), the first of equal (or unordered) values kept
RA_HD float ka_cell(const KaParams &p, const KaRow &r, uint32_t a, uint32_t b, float diag, float up, float left) {
    const float match = a == b ? diag : diag + ka_cost(p, r, a, b);
    return ra_min3(match, up + p.gap, left + p.gap);
}

// kmer_align of trimmed lists a[0..m), b[0..n) with n <= KA_SHORT, rows outer, in one thread
RA_HD float ka_short(const uint32_t *a, uint32_t m, const uint32_t *b, uint32_t n, const KaParams &p) {
    float S[KA_SHORT + 1];  // score[i][0..n]
    for (uint32_t j = 0; j <= n; ++j) S[j] = p.gap * (float)j;
    for (uint32_t i = 1; i <= m; ++i) {
        const uint32_t ai = a[i - 1];
        const KaRow r = ka_row(p, ai);
        float diag = S[0];
        S[0] = p.gap * (float)i;
        for (uint32_t j = 1; j <= n; ++j) {
            const float up = S[j];
            S[j] = ka_cell(p, r, ai, b[j - 1], diag, up, S[j - 1]);
            diag = up;
        }
    }
    return S[n];
}

// A one-thread job: kmer_align(kmers(target), kmers(query)) for a query window and padded allele of <= KA_SHORT bytes.
RA_HD float ka_short_job(const RaBufs &bf, const RaItem &it, uint32_t allele, const KaParams &p) {
    uint32_t a[KA_SHORT], b[KA_SHORT];
    uint32_t m = ka_kmers(ra_target(bf, it, allele), p.k, a), n = ka_kmers(ra_query(bf, it), p.k, b), x;
    if (!ka_trim(a, b, m, n, x)) return 0.0f;
    return ka_short(a + x, m, b + x, n, p);
}

// The work area of a warp job (ka_job_need bytes): the two k-mer lists, then per row of the trimmed DP its cost row and the
// column values score[i][j - 1] the sweep carries.
struct KaScratch {
    uint32_t *a, *b;  // [t_len], [q_len]
    KaRow *row;       // [t_len]
    float *S;         // [t_len + 1]
    RA_HD KaScratch(uint8_t *base, uint32_t q_len, uint32_t t_len) {
        a = (uint32_t *)base;
        b = a + t_len;
        row = (KaRow *)(b + q_len);
        S = (float *)(row + t_len);
    }
};
RA_HD uint64_t ka_scratch_bytes(uint64_t q_len, uint64_t t_len) {
    return (4 * (t_len + q_len) + sizeof(KaRow) * t_len + 4 * (t_len + 1) + 15) / 16 * 16;
}

// One lane of the warp wavefront of a longer job: rows lo..hi (1-based, of the trimmed lists a, b), over every column.
struct KaLane {
    uint32_t lo, hi;
    float prev_up;  // the lane's row lo - 1 in the previous column
    RA_HD void init(uint32_t m, uint32_t lane, uint32_t lanes, const uint32_t *a, KaRow *row, float *S, const KaParams &p) {
        const uint32_t band = (m + lanes - 1) / lanes;
        lo = 1 + lane * band;
        hi = lo + band - 1 < m ? lo + band - 1 : m;
        for (uint32_t i = lo; i <= hi; ++i) {
            row[i - 1] = ka_row(p, a[i - 1]);
            S[i] = p.gap * (float)i;
        }
        prev_up = p.gap * (float)(lo - 1);
    }
    RA_HD bool active() const { return lo <= hi; }
    // column j (k-mer bj): `up` is score[lo - 1][j] (the upper lane's last row, or gap * j for lane 0).  Returns score[hi][j].
    RA_HD float step(const uint32_t *a, const KaRow *row, float *S, float up, uint32_t bj, const KaParams &p) {
        float diag = prev_up;
        prev_up = up;
        for (uint32_t i = lo; i <= hi; ++i) {
            const float left = S[i];
            up = ka_cell(p, row[i - 1], a[i - 1], bj, diag, up, left);
            S[i] = up;
            diag = left;
        }
        return up;
    }
};

// The call of realign(use_kmerald=True) from the distances of allele 0 and the alternative allele: the smaller one, none on a
// tie or NaN; quality 30.  Returns 0, 1 or -1.
RA_HD int32_t ka_decide(float d_ref, float d_alt) { return d_ref < d_alt ? 0 : d_ref > d_alt ? 1 : -1; }

}  // namespace whmec
