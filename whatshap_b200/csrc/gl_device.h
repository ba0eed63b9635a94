// Forward-backward genotyping DP over the same column / projection structure as the MEC sweep
// (sibling DP of SURVEY.md 8(f) rank 4): per-cell code shared by the CUDA kernels (genotype.cu) and the
// test-only host emulation (tests/emul/emul_gl.cpp).
//
// Reference: GenotypeDPTable (src/genotypedptable.cpp:218-443), GenotypeColumnCostComputer
// (src/genotypecolumncostcomputer.cpp:47-103), TransitionProbabilityComputer
// (src/transitionprobabilitycomputer.cpp:10-90).  With  x  a bipartition of column k's active reads,
// i  a transmission value and  A  an allele assignment of the founder haplotypes:
//
//   e_i(x, A)   = prod_p cp_i[p][A_p](x),  cp_i[p][al] = prod over reads in partition p of
//                 (1 - eps) if the read's allele is al, eps otherwise          (cost computer :47-103)
//   forward     F_k(fwd(x), i)   += S_i(x) * e_i(x, A) * q_k(i, A),   S_i(x) = sum_j F_{k-1}(bwd(x), j) * t_k(j, i)   (:385-427)
//   backward    B_{k-1}(bwd(x), j) += B_k(fwd(x), i) * e_i(x, A) * t_k(j, i) * q_k(i, A)                           (:268-293)
//   posterior   L_k(ind, g)      += S_i(x) * e_i(x, A) * q_k(i, A) * B_k(fwd(x), i)   for g = genotype of ind under (i, A)   (:412-421)
//
// and every column's likelihoods are divided by their total (:438-442), so the per-column scale factors of
// F and B cancel: the reference divides by running sums of long doubles (:296-304,407), here every finished
// projection column is divided by its largest entry (exact same posterior up to floating-point rounding;
// doubles instead of the reference's 80-bit long doubles: results agree to ~1e-13, the reference's own tests
// compare with 1e-9, whatshap/testhelpers.py:11-15).
#pragma once
#include <stddef.h>

#include "common.h"

namespace whmec {

constexpr uint32_t GL_MAX_P = 10;    // founder haplotypes (2 * (individuals - trios))
constexpr uint32_t GL_MAX_IND = 16;
constexpr uint32_t GL_T_LOCAL = 16;  // transmission values accumulated in registers by one cell

struct GlCol {
    uint32_t a, bw, keep, f;  // as ColMeta
    uint32_t first, last;     // first column (S = 1) / last column (B = 1) of the table
    uint64_t act_off;         // this column's slice of eps / allele / ind
    uint64_t beta_off;        // doubles: where B_k (2^f * T entries, [fwd * T + i]) starts in the host's layout of all backward tables; a last column owns none
    uint64_t trans_off;       // doubles: t_k, [j * T + i] = P(transmission j in column k-1 -> i in column k)
    uint64_t q_off;           // doubles: q_k, [i * 2^P + A] = prior of allele assignment A given i
};

struct GlView {  // everything a cell needs; device pointers in the kernels, host pointers in the emulation
    const GlCol *cols;
    const double *eps;        // error probability of every (column, active read) entry
    const uint8_t *allele;    // 0 / 1 / 2 (blank)
    const uint8_t *ind;       // pedigree index of the read's sample
    const int8_t *h2p;        // [T][n_ind][2] haplotype -> partition (src/pedigreepartitions.cpp:7-42)
    const double *trans;
    const double *q;
    uint32_t T, P, n_ind;
};

// cp[p][allele] for cell x under transmission value i.  A read whose bit is 0 sits on haplotype 1 of its
// individual, bit 1 on haplotype 0 (genotypecolumncostcomputer.cpp:56,60-61: `entry_in_partition1`).
WHMEC_HD void gl_partition_products(const GlView &v, const GlCol &c, uint32_t x, uint32_t i, double (*cp)[2]) {
    for (uint32_t p = 0; p < v.P; ++p) cp[p][0] = cp[p][1] = 1.0;
    const int8_t *h = v.h2p + (size_t)i * v.n_ind * 2;
    for (uint32_t j = 0; j < c.a; ++j) {
        const uint32_t al = v.allele[c.act_off + j];
        if (al > 1) continue;  // BLANK (:51-53)
        const double e = v.eps[c.act_off + j];
        const uint32_t part = (uint32_t)h[2 * v.ind[c.act_off + j] + (((x >> j) & 1u) ? 0 : 1)];
        cp[part][al] *= 1.0 - e;
        cp[part][al ^ 1u] *= e;
    }
}

WHMEC_HD double gl_emission(const double (*cp)[2], uint32_t P, uint32_t A) {  // get_cost (:93-103)
    double e = 1.0;
    for (uint32_t p = 0; p < P; ++p) e *= cp[p][(A >> p) & 1u];
    return e;
}

// One cell of the backward pass of column k >= 1: reads B_k (`beta_k`, unused for a last column) and adds into
// B_{k-1} (`out`, 2^bw * T doubles).
template <class Add>
WHMEC_HD void gl_backward_cell(const GlView &v, uint32_t k, uint32_t x, const double *beta_k, double *out, Add add) {
    const GlCol &c = v.cols[k];
    const uint32_t T = v.T, nA = 1u << v.P;
    const uint32_t o = pext32(x, c.keep), b = x & low_mask(c.bw);
    double acc[GL_T_LOCAL];
    for (uint32_t j = 0; j < GL_T_LOCAL; ++j) acc[j] = 0.0;
    double cp[GL_MAX_P][2];
    for (uint32_t i = 0; i < T; ++i) {
        const double bi = c.last ? 1.0 : beta_k[(size_t)o * T + i];
        gl_partition_products(v, c, x, i, cp);
        double E = 0.0;
        for (uint32_t A = 0; A < nA; ++A) E += gl_emission(cp, v.P, A) * v.q[c.q_off + (size_t)i * nA + A];
        const double w = bi * E;
        const double *t = v.trans + c.trans_off;
        if (T <= GL_T_LOCAL) {
            for (uint32_t j = 0; j < T; ++j) acc[j] += w * t[(size_t)j * T + i];
        } else {
            for (uint32_t j = 0; j < T; ++j) add(&out[(size_t)b * T + j], w * t[(size_t)j * T + i]);
        }
    }
    if (T <= GL_T_LOCAL)
        for (uint32_t j = 0; j < T; ++j) add(&out[(size_t)b * T + j], acc[j]);
}

// One cell of the forward pass of column k: adds into F_k (`cur`, 2^f * T doubles; not for the last column) and
// into the caller's posterior accumulators lacc[ind * 3 + genotype index] (allele0 + allele1, :414-419).
template <class Add>
WHMEC_HD void gl_forward_cell(const GlView &v, uint32_t k, uint32_t x, const double *prev, double *cur, const double *beta_k,
                              double *lacc, Add add) {
    const GlCol &c = v.cols[k];
    const uint32_t T = v.T, nA = 1u << v.P;
    const uint32_t o = pext32(x, c.keep), b = x & low_mask(c.bw);
    double cp[GL_MAX_P][2];
    for (uint32_t i = 0; i < T; ++i) {
        double S = 1.0;
        if (!c.first) {
            S = 0.0;
            const double *t = v.trans + c.trans_off;
            for (uint32_t j = 0; j < T; ++j) S += prev[(size_t)b * T + j] * t[(size_t)j * T + i];
        }
        const double bi = c.last ? 1.0 : beta_k[(size_t)o * T + i];
        gl_partition_products(v, c, x, i, cp);
        const int8_t *h = v.h2p + (size_t)i * v.n_ind * 2;
        double sum = 0.0;
        for (uint32_t A = 0; A < nA; ++A) {
            const double w = gl_emission(cp, v.P, A) * v.q[c.q_off + (size_t)i * nA + A];
            sum += w;
            const double fb = S * w * bi;
            for (uint32_t n = 0; n < v.n_ind; ++n) lacc[n * 3 + ((A >> h[2 * n]) & 1u) + ((A >> h[2 * n + 1]) & 1u)] += fb;
        }
        if (!c.last) add(&cur[(size_t)o * T + i], S * sum);
    }
}

// One cell of the transfer pass of a segment (gl_transfer_plan): the forward recursion of column k for n_in input rows at
// once, without posterior and without backward tables.  prev / cur hold one row per input, [u][2^f * T] (the row stride of
// column k is 2^f_k * T; before a segment's column 0, prev holds the inputs themselves, [u][T]).  The partition products and
// the emission are computed once per (x, i) and reused for every input.  Unlike gl_forward_cell, the table's last column
// adds its values too: the mass the segment leaves at every transmission value.
template <class Add>
WHMEC_HD void gl_transfer_cell(const GlView &v, uint32_t k, uint32_t x, uint32_t n_in, const double *prev, double *cur, Add add) {
    const GlCol &c = v.cols[k];
    const uint32_t T = v.T, nA = 1u << v.P;
    const uint32_t o = pext32(x, c.keep), b = x & low_mask(c.bw);
    const uint64_t out_w = ((uint64_t)1 << c.f) * T, in_w = k ? ((uint64_t)1 << v.cols[k - 1].f) * T : T;
    const double *t = v.trans + c.trans_off;
    double cp[GL_MAX_P][2];
    for (uint32_t i = 0; i < T; ++i) {
        gl_partition_products(v, c, x, i, cp);
        double E = 0.0;
        for (uint32_t A = 0; A < nA; ++A) E += gl_emission(cp, v.P, A) * v.q[c.q_off + (size_t)i * nA + A];
        for (uint32_t u = 0; u < n_in; ++u) {
            double S = 1.0;
            if (!c.first) {
                S = 0.0;
                const double *p = prev + u * in_w + (size_t)b * T;
                for (uint32_t j = 0; j < T; ++j) S += p[j] * t[(size_t)j * T + i];
            }
            add(&cur[u * out_w + (size_t)o * T + i], S * E);
        }
    }
}

}  // namespace whmec
