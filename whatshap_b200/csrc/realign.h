// Allele detection by re-alignment (whmec_realign, DESIGN §4.11): the per-item code shared by the kernels of realign.cu and the
// host emulation (tests/emul/emul_realign.cpp), and the host plan of realign_plan.cpp.
//
// An item is one (alignment, variant) pair that whatshap's _iterate_cigar yields and ReadSetReader.realign aligns
// (whatshap/variants.py:685-848); a job is one allele of an item that survives the restricted-genotype filter.  A job's target
// (the padded allele) is never materialised: it is up to three slices, left pad | allele | right pad, of the reference and the
// variant's allele bytes.  Both strings lose their common prefix and suffix first (align.pyx:47-57, 142-153), then
//   unit cost: Myers/Hyyro bit-parallel global edit distance, 64 rows per word (symmetric, so the shorter string is the pattern);
//   affine:    the float32 Gotoh recurrence of align.pyx:160-196, cell for cell, rows over the query.
// A job whose strings are short enough runs in one thread (ra_unit_short, ra_affine_short); a longer one runs on a warp as an
// anti-diagonal wavefront over 64-row words (unit) or row bands (affine), lane L one step behind lane L-1 (RaUnitLane, RaAffLane).
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define RA_HD __host__ __device__ __forceinline__
#else
#define RA_HD inline
#endif

namespace whmec {

constexpr uint32_t RA_SHORT = 64;          // one thread: unit cost min(query, target) <= 64, affine query <= 64 (untrimmed)
constexpr float RA_INT_MAX_F = 2147483648.0f;  // (float)INT_MAX, align.pyx:166
constexpr uint64_t RA_NO_SCRATCH = ~0ull;

struct RaItem {
    uint64_t q;               // first byte of the query window in the query bytes
    int64_t r;                // reference window start (variant position - left reference bases)
    uint32_t q_len;           // query window length
    uint32_t left, right;     // reference bases left of the variant and from the variant on (cigar_prefix_length)
    uint32_t ref_len;         // len(reference_allele)
    uint32_t variant;         // index into the variant list
    uint32_t job0, n_jobs;    // the item's jobs, in allele order
    uint32_t alignment;
};

struct RaJob {
    uint32_t item, allele;
    uint64_t scratch;  // RA_NO_SCRATCH: one-thread job; else the byte offset of its work area in the chunk's scratch
};

// Where a chunk's slices live: item.q - q0 indexes q, item.r - r0 indexes ref.  Allele a of variant v is
// al[al_off[al_first[v] + a] .. al_off[al_first[v] + a + 1]).
struct RaBufs {
    const uint8_t *q;
    uint64_t q0;
    const uint8_t *ref;
    int64_t r0;
    const uint8_t *al;
    const uint64_t *al_off;
    const uint32_t *al_first;
};

struct RaParams {
    int affine;
    float mismatch;  // (float) default_mismatch
    int32_t gap_start, gap_extend;
};

// A view [off, off + len) of the concatenation of up to three byte slices.
struct RaSeq {
    const uint8_t *p0, *p1, *p2;
    uint32_t l0, l1, l2, off, len;
    RA_HD uint8_t at(uint32_t i) const {
        i += off;
        if (i < l0) return p0[i];
        i -= l0;
        return i < l1 ? p1[i] : p2[i - l1];
    }
};

RA_HD RaSeq ra_query(const RaBufs &b, const RaItem &it) {
    RaSeq s{b.q + (it.q - b.q0), nullptr, nullptr, it.q_len, 0, 0, 0, it.q_len};
    return s;
}

// the padded allele: reference[pos - left : pos + right] for allele 0, else left pad + allele + reference[pos + ref_len : pos + right]
RA_HD RaSeq ra_target(const RaBufs &b, const RaItem &it, uint32_t allele) {
    const uint8_t *w = b.ref + (it.r - b.r0);
    if (allele == 0) return RaSeq{w, nullptr, nullptr, it.left + it.right, 0, 0, 0, it.left + it.right};
    const uint32_t slot = b.al_first[it.variant] + allele;
    const uint32_t l1 = (uint32_t)(b.al_off[slot + 1] - b.al_off[slot]);
    const uint32_t l2 = it.right > it.ref_len ? it.right - it.ref_len : 0;
    return RaSeq{w, b.al + b.al_off[slot], w + it.left + it.ref_len, it.left, l1, l2, 0, it.left + l1 + l2};
}

// strips the identical prefix, then the identical suffix
RA_HD void ra_trim(RaSeq &s, RaSeq &t) {
    while (s.len > 0 && t.len > 0 && s.at(0) == t.at(0)) ++s.off, ++t.off, --s.len, --t.len;
    while (s.len > 0 && t.len > 0 && s.at(s.len - 1) == t.at(t.len - 1)) --s.len, --t.len;
}

// ---- unit cost -----------------------------------------------------------------------------------------------------------

// Match masks of up to 64 pattern bytes: the first 8 distinct bytes in registers, a scan of the pattern beyond that.
struct RaPeq {
    uint8_t ch[8];
    uint64_t pm[8];
    uint32_t nd;
    bool many;
    RA_HD void init(const RaSeq &p, uint32_t base, uint32_t len) {
        nd = 0;
        many = false;
#pragma unroll
        for (int k = 0; k < 8; ++k) ch[k] = 0, pm[k] = 0;
        for (uint32_t i = 0; i < len; ++i) {
            const uint8_t c = p.at(base + i);
            bool found = false;
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if ((uint32_t)k < nd && ch[k] == c) pm[k] |= 1ull << i, found = true;
            if (found) continue;
            if (nd == 8) {
                many = true;
                continue;
            }
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if ((uint32_t)k == nd) ch[k] = c, pm[k] = 1ull << i;
            ++nd;
        }
    }
    RA_HD uint64_t eq(const RaSeq &p, uint32_t base, uint32_t len, uint8_t c) const {
        uint64_t e = 0;
        if (!many) {
#pragma unroll
            for (int k = 0; k < 8; ++k)
                if ((uint32_t)k < nd && ch[k] == c) e = pm[k];
            return e;
        }
        for (uint32_t i = 0; i < len; ++i) e |= (uint64_t)(p.at(base + i) == c) << i;
        return e;
    }
};

// One column of one 64-row word (Myers 1999 / Hyyro): hin, hout in {-1, 0, +1} are the horizontal deltas above and at `hb`.
RA_HD int ra_word_step(uint64_t &pv, uint64_t &mv, uint64_t eq, int hin, uint64_t hb) {
    const uint64_t xv = eq | mv;
    if (hin < 0) eq |= 1;
    const uint64_t xh = (((eq & pv) + pv) ^ pv) | eq;
    uint64_t ph = mv | ~(xh | pv), mh = pv & xh;
    const int hout = (ph & hb) ? 1 : (mh & hb) ? -1 : 0;
    ph <<= 1;
    mh <<= 1;
    if (hin < 0) mh |= 1;
    else if (hin > 0) ph |= 1;
    pv = mh | ~(xv | ph);
    mv = ph & xv;
    return hout;
}

// edit distance of trimmed strings with min(len) <= 64, in one thread
RA_HD int64_t ra_unit_short(RaSeq s, RaSeq t) {
    const RaSeq &p = s.len <= t.len ? s : t, &x = s.len <= t.len ? t : s;
    if (p.len == 0) return x.len;
    RaPeq peq;
    peq.init(p, 0, p.len);
    uint64_t pv = ~0ull, mv = 0;
    const uint64_t hb = 1ull << (p.len - 1);
    int64_t score = p.len;
    for (uint32_t j = 0; j < x.len; ++j) score += ra_word_step(pv, mv, peq.eq(p, 0, p.len, x.at(j)), 1, hb);
    return score;
}

// One lane of the warp wavefront for a longer unit-cost job: word `w` of the pattern (rows 64w ..), over the text's columns.
struct RaUnitLane {
    RaPeq peq;
    uint64_t pv, mv, hb;
    uint32_t base, len;
    bool active, last;
    int64_t score;
    RA_HD void init(const RaSeq &p, uint32_t w) {
        const uint32_t words = (p.len + 63) / 64;
        active = w < words;
        last = w + 1 == words;
        base = 64 * w;
        len = active ? (p.len - base < 64 ? p.len - base : 64) : 0;
        if (active) peq.init(p, base, len);
        pv = ~0ull;
        mv = 0;
        hb = 1ull << (len ? len - 1 : 0);
        score = p.len;
    }
    RA_HD int step(const RaSeq &p, uint8_t c, int hin) {
        const int h = ra_word_step(pv, mv, peq.eq(p, base, len, c), hin, hb);
        if (last) score += h;
        return h;
    }
};

// ---- affine gap cost (float32, literal) ------------------------------------------------------------------------------------

RA_HD float ra_min3(float x, float y, float z) {  // Cython's min(x, y, z)
    float r = x;
    if (y < r) r = y;
    if (z < r) r = z;
    return r;
}
RA_HD float ra_gap(int64_t l, const RaParams &pr) {  // f(l) = gap_start + (l-1) * gap_extend, a Python int stored to a float
    return (float)(double)((int64_t)pr.gap_start + (l - 1) * (int64_t)pr.gap_extend);
}

struct RaCell {
    float a, b, c;
};

// Rows lo..hi (1-based) of one column j: `up` holds the column's values in row lo - 1, `diag` those of column j - 1.  A, B, C
// hold column j - 1 on entry and column j on exit (align.pyx:180-195).  Returns row hi's values.
RA_HD RaCell ra_affine_band(float *A, float *B, float *C, uint32_t lo, uint32_t hi, RaCell up, RaCell diag, const RaSeq &q, uint8_t tj,
                           const RaParams &pr) {
    const float gs = (float)pr.gap_start, ge = (float)pr.gap_extend;
    for (uint32_t i = lo; i <= hi; ++i) {
        const float mc = q.at(i - 1) == tj ? 0.0f : pr.mismatch;
        const RaCell cur{ra_min3(diag.a, diag.b, diag.c) + mc, ra_min3(up.a + gs, up.b + ge, up.c + gs), ra_min3(A[i] + gs, B[i] + gs, C[i] + ge)};
        diag = RaCell{A[i], B[i], C[i]};
        A[i] = cur.a, B[i] = cur.b, C[i] = cur.c;
        up = cur;
    }
    return up;
}
RA_HD RaCell ra_affine_top(uint32_t j, const RaParams &pr) {  // row 0 of column j
    return j == 0 ? RaCell{0.0f, 0.0f, 0.0f} : RaCell{RA_INT_MAX_F, RA_INT_MAX_F, ra_gap(j, pr)};
}
RA_HD RaCell ra_affine_init(uint32_t i, const RaParams &pr) {  // column 0 of row i
    return i == 0 ? RaCell{0.0f, 0.0f, 0.0f} : RaCell{RA_INT_MAX_F, ra_gap(i, pr), RA_INT_MAX_F};
}

// the affine distance (before int()) of trimmed strings with q.len <= 64, in one thread
RA_HD float ra_affine_short(const RaSeq &q, const RaSeq &t, const RaParams &pr) {
    float A[RA_SHORT + 1], B[RA_SHORT + 1], C[RA_SHORT + 1];
    const uint32_t m = q.len;
    for (uint32_t i = 0; i <= m; ++i) {
        const RaCell v = ra_affine_init(i, pr);
        A[i] = v.a, B[i] = v.b, C[i] = v.c;
    }
    for (uint32_t j = 1; j <= t.len; ++j) {
        const RaCell top = ra_affine_top(j, pr);
        const RaCell diag{A[0], B[0], C[0]};
        A[0] = top.a, B[0] = top.b, C[0] = top.c;
        if (m) ra_affine_band(A, B, C, 1, m, top, diag, q, t.at(j - 1), pr);
    }
    return ra_min3(A[m], B[m], C[m]);
}

// One lane of the warp wavefront for a longer affine job: rows lo..hi of every column, A/B/C in the job's scratch.
struct RaAffLane {
    uint32_t lo, hi;
    RaCell prev_up;  // the lane's row lo - 1 in the previous column
    RA_HD void init(uint32_t m, uint32_t lane, uint32_t lanes, float *A, float *B, float *C, const RaParams &pr) {
        const uint32_t band = (m + lanes - 1) / lanes;
        lo = 1 + lane * band;
        hi = lo + band - 1 < m ? lo + band - 1 : m;
        for (uint32_t i = lo; i <= hi; ++i) {
            const RaCell v = ra_affine_init(i, pr);
            A[i] = v.a, B[i] = v.b, C[i] = v.c;
        }
        prev_up = ra_affine_init(lo - 1, pr);
    }
    RA_HD bool active() const { return lo <= hi; }
    // column j: `up` is the upper lane's row lo - 1 of this column (lane 0: ra_affine_top(j))
    RA_HD RaCell step(float *A, float *B, float *C, RaCell up, const RaSeq &q, uint8_t tj, const RaParams &pr) {
        const RaCell diag = prev_up;
        prev_up = up;
        return ra_affine_band(A, B, C, lo, hi, up, diag, q, tj, pr);
    }
};

// int(x) of align.pyx:196; false when x is not finite or beyond int64 (the call then fails)
RA_HD bool ra_trunc(float x, int64_t &out) {
    if (!(x > -9.2233720e18f && x < 9.2233720e18f)) return false;
    out = (int64_t)x;
    return true;
}

// A one-thread job (RaJob::scratch == RA_NO_SCRATCH): false when the affine distance has no int64 value.
RA_HD bool ra_short_job(const RaBufs &b, const RaItem &it, uint32_t allele, const RaParams &pr, int64_t &d) {
    RaSeq q = ra_query(b, it), t = ra_target(b, it, allele);
    ra_trim(q, t);
    if (pr.affine) return ra_trunc(ra_affine_short(q, t, pr), d);
    d = ra_unit_short(q, t);
    return true;
}

// The decision of realign() (variants.py:816-848) over the item's distances d[0..n) in allele order: the stable sort's first
// entry is the first minimum, the second entry the minimum of the others.  Returns the position of the called allele among the
// item's jobs, or -1.
RA_HD int32_t ra_decide(const int64_t *d, uint32_t n, int affine, int64_t &quality) {
    uint32_t best = 0;
    for (uint32_t k = 1; k < n; ++k)
        if (d[k] < d[best]) best = k;
    if (n == 1) {
        quality = affine ? d[0] : 30;
        return 0;
    }
    bool have = false;
    int64_t second = 0;
    for (uint32_t k = 0; k < n; ++k)
        if (k != best && (!have || d[k] < second)) second = d[k], have = true;
    if (d[best] < second) {
        quality = affine ? d[best] - second : 30;
        return (int32_t)best;
    }
    return -1;
}

}  // namespace whmec
