/*
 * TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT PATH.
 *
 * Plain-C restatement of WhatsHap's forward-backward genotyping DP (GenotypeDPTable), the checker of
 * whmec_genotype (tests/).  Nothing under whatshap_b200/ links, imports or
 * executes this file.
 *
 * Parity status: PINNED within floating-point tolerance.  Validated against the compiled, unmodified
 * reference (oracle/_ref/libwhref.so: whref_genotype) by tests/test_genotype_oracle.py (max abs difference
 * of the normalised likelihoods ~1e-17, both compute in long double) and against the reference's own known
 * answers (tests/test_genotyping.py:113-190 of the reference, restated in tests/golden/genotype_kat.json).
 *
 * Follows (paths relative to the whatshap tree):
 *   GenotypeDPTable::compute_backward_column   src/genotypedptable.cpp:218-305
 *   GenotypeDPTable::compute_forward_column    src/genotypedptable.cpp:308-443
 *   GenotypeColumnCostComputer                 src/genotypecolumncostcomputer.cpp:24-103
 *   TransitionProbabilityComputer              src/transitionprobabilitycomputer.cpp:10-90
 *   PedigreePartitions                         src/pedigreepartitions.cpp:7-42
 * Differences that do not change results beyond rounding: every backward column is kept (the reference keeps
 * every sqrt(n)-th and recomputes, :139-166,326-343); a cell's partition products are formed directly instead
 * of being updated along the Gray code by multiplications and divisions (cost computer :70-91).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../include/whmec.h"

#define GL_MAX_IND 16
#define GL_MAX_PART 10

typedef long double real;

static void gl_set_err(char *err, size_t errlen, const char *msg) {
    if (err && errlen) {
        strncpy(err, msg, errlen - 1);
        err[errlen - 1] = 0;
    }
}

/* src/pedigreepartitions.cpp:7-42 */
static int gl_h2p(const whmec_problem *p, uint32_t tv, int (*h2p)[2]) {
    int triple_of[GL_MAX_IND];
    for (uint32_t i = 0; i < p->n_ind; ++i) {
        triple_of[i] = -1;
        h2p[i][0] = h2p[i][1] = -1;
    }
    for (uint32_t r = 0; r < p->n_trios; ++r) triple_of[p->trios[3 * r + 2]] = (int)r;
    int q = 0;
    for (uint32_t i = 0; i < p->n_ind; ++i)
        if (triple_of[i] < 0) {
            h2p[i][0] = q;
            h2p[i][1] = q + 1;
            q += 2;
        }
    for (uint32_t round = 0; round <= p->n_ind; ++round) {
        int pending = 0;
        for (uint32_t i = 0; i < p->n_ind; ++i) {
            if (h2p[i][0] != -1) continue;
            const uint32_t f = p->trios[3 * triple_of[i]], m = p->trios[3 * triple_of[i] + 1];
            if (h2p[f][0] == -1 || h2p[m][0] == -1) {
                pending = 1;
                continue;
            }
            h2p[i][0] = h2p[f][((tv >> (2 * triple_of[i])) & 1) ? 0 : 1];
            h2p[i][1] = h2p[m][((tv >> (2 * triple_of[i] + 1)) & 1) ? 0 : 1];
        }
        if (!pending) return 0;
    }
    return -1;
}

/* src/genotypecolumncostcomputer.cpp:24-45 */
static real gl_phred_probability(uint32_t phred) {
    if (phred == 0) return 0.9999L;
    return powl(10.0L, -(real)(int)phred / 10.0L);
}

typedef struct {
    uint32_t a, bw, keep, f;
    uint32_t ind[32];
    uint8_t allele[32];
    real eps[32];
} gl_column;

static uint32_t gl_popcount(uint32_t x) {
    uint32_t c = 0;
    for (; x; x >>= 1) c += x & 1;
    return c;
}

/* forward projection of index x: the bits of the reads that stay, compacted (columnindexingiterator.cpp:26-49) */
static uint32_t gl_forward_index(uint32_t x, uint32_t keep) {
    uint32_t out = 0, o = 0;
    for (uint32_t j = 0; j < 32; ++j)
        if ((keep >> j) & 1) {
            out |= ((x >> j) & 1u) << o;
            ++o;
        }
    return out;
}

/* cost_partition of a cell (set_partitioning, cost computer :47-67): the read of bit j sits on haplotype 1 when the bit is 0 */
static void gl_cell_products(const gl_column *c, uint32_t x, int (*h2p)[2], uint32_t P, real cp[][2]) {
    for (uint32_t q = 0; q < P; ++q) cp[q][0] = cp[q][1] = 1.0L;
    for (uint32_t j = 0; j < c->a; ++j) {
        if (c->allele[j] > 1) continue;
        const int in_partition1 = ((x >> j) & 1u) == 0;
        const int part = h2p[c->ind[j]][in_partition1];
        const int is_ref = c->allele[j] == 0;
        cp[part][!is_ref] *= (1.0L - c->eps[j]);
        cp[part][is_ref] *= c->eps[j];
    }
}

static real gl_cost(real cp[][2], uint32_t P, uint32_t A) { /* get_cost :93-103 */
    real cost = 1.0L;
    for (uint32_t q = 0; q < P; ++q) cost *= cp[q][(A >> q) & 1];
    return cost;
}

int whoracle_genotype(const whmec_problem *p, double *likelihoods, char *err, size_t errlen) {
    const uint32_t n = p->n_cols;
    if (p->n_ind == 0 || p->n_ind > GL_MAX_IND || p->n_trios >= p->n_ind || p->n_trios > 4) {
        gl_set_err(err, errlen, "oracle: unsupported pedigree");
        return WHMEC_ERR_UNSUPPORTED;
    }
    const uint32_t P = 2 * (p->n_ind - p->n_trios), T = 1u << (2 * p->n_trios), nA = 1u << P, tb = 2 * p->n_trios;
    if (P > GL_MAX_PART) {
        gl_set_err(err, errlen, "oracle: pedigree too large");
        return WHMEC_ERR_UNSUPPORTED;
    }
    if (n == 0) return WHMEC_OK;
    if (!p->gl) {
        gl_set_err(err, errlen, "oracle: genotype priors required");
        return WHMEC_ERR_INPUT;
    }
    int (*h2p)[GL_MAX_IND][2] = (int (*)[GL_MAX_IND][2])malloc(sizeof(int) * T * GL_MAX_IND * 2);
    for (uint32_t t = 0; t < T; ++t)
        if (gl_h2p(p, t, h2p[t])) {
            free(h2p);
            gl_set_err(err, errlen, "oracle: malformed pedigree");
            return WHMEC_ERR_INPUT;
        }
    /* columns (ColumnIterator, src/columniterator.cpp:91-139; indexing scheme, src/columnindexingscheme.cpp:7-34,62-85) */
    gl_column *cols = (gl_column *)calloc(n, sizeof(gl_column));
    int rc = WHMEC_OK;
    for (uint32_t r = 0; r < p->n_reads && rc == WHMEC_OK; ++r) {
        const uint64_t b = p->read_off[r], e = p->read_off[r + 1];
        if (e <= b || p->ent_col[e - 1] >= n || p->ent_col[b] >= p->ent_col[e - 1]) {
            /* backwardcolumniterator.cpp:41 asserts first column < last column */
            gl_set_err(err, errlen, "oracle: every read must cover at least two columns");
            rc = WHMEC_ERR_INPUT;
            break;
        }
        if (r > 0 && p->ent_col[b] < p->ent_col[p->read_off[r - 1]]) {
            gl_set_err(err, errlen, "ColumnIterator: reads in ReadSet are not sorted.");
            rc = WHMEC_ERR_INPUT;
            break;
        }
        uint64_t cur = b;
        for (uint32_t k = p->ent_col[b]; k <= p->ent_col[e - 1]; ++k) {
            gl_column *c = &cols[k];
            if (c->a >= 30) {
                gl_set_err(err, errlen, "oracle: too many active reads");
                rc = WHMEC_ERR_UNSUPPORTED;
                break;
            }
            while (p->ent_col[cur] < k) ++cur;
            const uint32_t j = c->a++;
            c->ind[j] = p->read_ind[r];
            if (p->ent_col[cur] == k) {
                c->allele[j] = p->ent_allele[cur];
                c->eps[j] = gl_phred_probability(p->ent_phred[cur]);
            } else { /* gap: BLANK (columniterator.cpp:131) */
                c->allele[j] = 2;
                c->eps[j] = 0.9999L;
            }
            if (k < p->ent_col[e - 1]) c->keep |= 1u << j;
            if (k > p->ent_col[b]) c->bw++; /* reads are sorted by first column: shared reads are the lowest bits */
        }
    }
    if (rc != WHMEC_OK) {
        free(cols);
        free(h2p);
        return rc;
    }
    for (uint32_t k = 0; k < n; ++k) cols[k].f = gl_popcount(cols[k].keep);

    /* transition tables (transitionprobabilitycomputer.cpp:18-89) */
    real *trans = (real *)malloc(sizeof(real) * (size_t)n * T * T);
    real *prior = (real *)malloc(sizeof(real) * (size_t)n * T * nA);
    for (uint32_t k = 0; k < n; ++k) {
        const real r = powl(10.0L, -(real)p->recombcost[k] / 10.0L);
        real bern[9];
        for (uint32_t i = 0; i <= tb; ++i) bern[i] = powl(r, (real)i) * powl(1.0L - r, (real)(tb - i));
        for (uint32_t i = 0; i < T; ++i) {
            real norm = 0.0L;
            for (uint32_t j = 0; j < T; ++j) norm += bern[gl_popcount(i ^ j)];
            for (uint32_t j = 0; j < T; ++j) trans[((size_t)k * T + i) * T + j] = bern[gl_popcount(i ^ j)] / norm;
        }
        for (uint32_t i = 0; i < T; ++i) {
            real *q = prior + ((size_t)k * T + i) * nA;
            uint32_t *code = (uint32_t *)malloc(sizeof(uint32_t) * nA); /* genotype vector, 2 bits per individual */
            for (uint32_t A = 0; A < nA; ++A) {
                real pr = 1.0L;
                uint32_t cd = 0;
                for (uint32_t ind = 0; ind < p->n_ind; ++ind) {
                    const uint32_t g = ((A >> h2p[i][ind][0]) & 1u) + ((A >> h2p[i][ind][1]) & 1u);
                    pr *= p->gl[((size_t)ind * n + k) * 3 + g];
                    cd |= g << (2 * ind);
                }
                q[A] = pr;
                code[A] = cd;
            }
            real norm = 0.0L;
            for (uint32_t A = 0; A < nA; ++A) { /* :76-82 */
                uint32_t same = 0;
                for (uint32_t B = 0; B < nA; ++B) same += code[B] == code[A];
                q[A] /= (real)same;
            }
            for (uint32_t A = 0; A < nA; ++A) norm += q[A];
            for (uint32_t A = 0; A < nA; ++A) q[A] /= norm;
            free(code);
        }
    }

    /* backward pass (:218-305): beta[k] = projection between columns k and k+1, indexed by forward index of column k */
    real **beta = (real **)calloc(n, sizeof(real *));
    real *scaling = (real *)calloc(n, sizeof(real));
    real cp[GL_MAX_PART][2];
    for (uint32_t kk = n; kk-- > 0;) {
        const gl_column *c = &cols[kk];
        real *prev = (kk + 1 < n) ? beta[kk] : NULL;
        real *cur = NULL;
        size_t cur_size = 0;
        if (kk > 0) {
            cur_size = ((size_t)1 << cols[kk - 1].f) * T;
            cur = (real *)calloc(cur_size, sizeof(real));
        }
        real scaling_sum = 0.0L;
        for (uint32_t x = 0; x < (1u << c->a); ++x) {
            const uint32_t fwd = gl_forward_index(x, c->keep), bwd = x & ((1u << c->bw) - 1u);
            for (uint32_t i = 0; i < T; ++i) {
                const real backward_prob = prev ? prev[(size_t)fwd * T + i] : 1.0L;
                gl_cell_products(c, x, h2p[i], P, cp);
                for (uint32_t A = 0; A < nA; ++A) {
                    if (kk > 0) {
                        const real local = gl_cost(cp, P, A);
                        for (uint32_t j = 0; j < T; ++j)
                            cur[(size_t)bwd * T + j] += backward_prob * local * trans[((size_t)kk * T + j) * T + i] * prior[((size_t)kk * T + i) * nA + A];
                    }
                    scaling_sum += backward_prob;
                }
            }
        }
        if (prev)
            for (size_t e = 0; e < ((size_t)1 << c->f) * T; ++e) prev[e] /= scaling_sum;
        if (cur) {
            for (size_t e = 0; e < cur_size; ++e) cur[e] /= scaling_sum;
            beta[kk - 1] = cur;
        }
        scaling[kk] = scaling_sum;
    }

    /* forward pass (:308-443) */
    real *fprev = NULL;
    for (uint32_t k = 0; k < n; ++k) {
        const gl_column *c = &cols[k];
        real *fcur = (k + 1 < n) ? (real *)calloc(((size_t)1 << c->f) * T, sizeof(real)) : NULL;
        real *bk = (k + 1 < n) ? beta[k] : NULL;
        real normalization = 0.0L;
        real lik[GL_MAX_IND][3];
        memset(lik, 0, sizeof lik);
        for (uint32_t x = 0; x < (1u << c->a); ++x) {
            const uint32_t fwd = gl_forward_index(x, c->keep), bwd = x & ((1u << c->bw) - 1u);
            for (uint32_t i = 0; i < T; ++i) {
                real sum_prev = 0.0L;
                if (k > 0) {
                    for (uint32_t j = 0; j < T; ++j) sum_prev += fprev[(size_t)bwd * T + j] * trans[((size_t)k * T + j) * T + i];
                } else {
                    sum_prev = 1.0L;
                }
                gl_cell_products(c, x, h2p[i], P, cp);
                for (uint32_t A = 0; A < nA; ++A) {
                    const real backward_probability = bk ? bk[(size_t)fwd * T + i] : 1.0L;
                    const real forward_probability = (sum_prev * gl_cost(cp, P, A) * prior[((size_t)k * T + i) * nA + A]) / scaling[k];
                    const real fb = forward_probability * backward_probability;
                    normalization += fb;
                    for (uint32_t ind = 0; ind < p->n_ind; ++ind)
                        lik[ind][((A >> h2p[i][ind][0]) & 1u) + ((A >> h2p[i][ind][1]) & 1u)] += fb;
                    if (fcur) fcur[(size_t)fwd * T + i] += forward_probability;
                }
            }
        }
        for (uint32_t ind = 0; ind < p->n_ind; ++ind)
            for (uint32_t g = 0; g < 3; ++g) likelihoods[((size_t)ind * n + k) * 3 + g] = (double)(lik[ind][g] / normalization);
        free(fprev);
        fprev = fcur;
    }
    free(fprev);
    for (uint32_t k = 0; k < n; ++k) free(beta[k]);
    free(beta);
    free(scaling);
    free(trans);
    free(prior);
    free(cols);
    free(h2p);
    return WHMEC_OK;
}
