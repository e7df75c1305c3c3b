/*
 * TEST INFRASTRUCTURE -- NOT PRODUCT CODE.
 *
 * C/OpenMP restatement of the two numeric hot paths the EVcouplings pipeline
 * delegates to the external plmc binary (call site
 * evcouplings/couplings/tools.py:202-266; "compile using make all-openmp32",
 * reference README.md:35-42).  plmc's source is not part of the reference, so this
 * is a *port of the published algorithm* (kind "port"), parallel over sites like
 * plmc's OpenMP build, in fp32 (the all-openmp32 arithmetic) and fp64.
 * Semantics are the ones pinned by the golden plmc run in
 * notebooks/example/ -- see oracle/plm_oracle.py header and SURVEY.md 8(a)
 * rows a5/a7.  Used by tests/ (parity checker at sizes numpy is too slow for)
 * and by bench.py's cpu_baseline / --impl reference legs only.
 *
 * Parameter layout: x = [h (L*q) | J tri blocks (i<j row-major, block[a][b])]
 * = the plmc_v2 .model order (evcouplings/couplings/model.py:354-389).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#ifdef _OPENMP
#include <omp.h>
#endif

/* (b) Hamming neighbour counts: in-tree twin evcouplings/align/alignment.py:1192-1233
 * n_s = #{t : #identical positions >= thr}, self included, gap==gap identical. */
void oracle_hamming_counts(const uint8_t *codes, int64_t N, int32_t L, int32_t thr,
                           int32_t *counts, int32_t nthreads)
{
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#endif
#pragma omp parallel for schedule(dynamic, 16)
    for (int64_t s = 0; s < N; s++) {
        const uint8_t *a = codes + s * L;
        int32_t c = 0;
        for (int64_t t = 0; t < N; t++) {
            const uint8_t *b = codes + t * L;
            int32_t id = 0;
            for (int32_t k = 0; k < L; k++) id += (a[k] == b[k]);
            c += (id >= thr);
        }
        counts[s] = c;
    }
}

/* row-range variant used to time a bounded sample of the N x N comparison */
void oracle_hamming_counts_rows(const uint8_t *codes, int64_t N, int32_t L, int32_t thr,
                                int64_t row0, int64_t row1, int32_t *counts, int32_t nthreads)
{
#ifdef _OPENMP
    if (nthreads > 0) omp_set_num_threads(nthreads);
#endif
#pragma omp parallel for schedule(dynamic, 4)
    for (int64_t s = row0; s < row1; s++) {
        const uint8_t *a = codes + s * L;
        int32_t c = 0;
        for (int64_t t = 0; t < N; t++) {
            const uint8_t *b = codes + t * L;
            int32_t id = 0;
            for (int32_t k = 0; k < L; k++) id += (a[k] == b[k]);
            c += (id >= thr);
        }
        counts[s - row0] = c;
    }
}

#define DEFINE_PLM_EVAL(NAME, REAL, EXPF, LOGF)                                              \
/* (a) PLM negative log-posterior + gradient, site-parallel (SURVEY row a7).          */    \
/* codes >= q mark a gap under ignore_gaps: the site is skipped as a conditional and  */    \
/* contributes nothing as a neighbour.  Returns 0, or -1 on allocation failure.       */    \
int NAME(const uint8_t *codes, int64_t N, int32_t L, int32_t q, const REAL *w,               \
         const REAL *x, REAL lambda_h, REAL lambda_J, REAL *g, double *fx_out,               \
         double *nll_out, int32_t nthreads)                                                  \
{                                                                                            \
    const int64_t qq = (int64_t)q * q;                                                       \
    const int64_t blk = (int64_t)L * qq;            /* one site's row block [j][b][a] */      \
    REAL *W = (REAL *)calloc((size_t)L * blk, sizeof(REAL));                                 \
    REAL *G = (REAL *)calloc((size_t)L * blk, sizeof(REAL));                                 \
    if (!W || !G) { free(W); free(G); return -1; }                                           \
    const REAL *h = x;                                                                       \
    const REAL *J = x + (int64_t)L * q;                                                      \
    /* expand tri blocks into W[i][j][b][a] = J_ij(a,b), both orientations */                \
    {                                                                                        \
        int64_t p = 0;                                                                       \
        for (int32_t i = 0; i < L; i++)                                                      \
            for (int32_t j = i + 1; j < L; j++, p++) {                                       \
                const REAL *B = J + p * qq;                                                  \
                REAL *Wij = W + (int64_t)i * blk + (int64_t)j * qq;                          \
                REAL *Wji = W + (int64_t)j * blk + (int64_t)i * qq;                          \
                for (int32_t a = 0; a < q; a++)                                              \
                    for (int32_t b = 0; b < q; b++) {                                        \
                        Wij[b * q + a] = B[a * q + b];                                       \
                        Wji[a * q + b] = B[a * q + b];                                       \
                    }                                                                        \
            }                                                                                \
    }                                                                                        \
    double fx = 0.0;                                                                         \
    _Pragma("omp parallel for schedule(dynamic, 1) reduction(+ : fx)")                       \
    for (int32_t i = 0; i < L; i++) {                                                        \
        const REAL *Wi = W + (int64_t)i * blk;                                               \
        REAL *Gi = G + (int64_t)i * blk;                                                     \
        REAL gh[64];                                                                         \
        REAL z[64];                                                                          \
        double fxi = 0.0;                                                                    \
        for (int32_t a = 0; a < q; a++) gh[a] = 0;                                           \
        for (int64_t s = 0; s < N; s++) {                                                    \
            const uint8_t *row = codes + s * L;                                              \
            const int32_t si = row[i];                                                       \
            if (si >= q) continue;                                                           \
            for (int32_t a = 0; a < q; a++) z[a] = h[(int64_t)i * q + a];                    \
            for (int32_t j = 0; j < L; j++) {                                                \
                const int32_t sj = row[j];                                                   \
                if (j == i || sj >= q) continue;                                             \
                const REAL *col = Wi + (int64_t)j * qq + (int64_t)sj * q;                    \
                for (int32_t a = 0; a < q; a++) z[a] += col[a];                              \
            }                                                                                \
            REAL zmax = z[0];                                                                \
            for (int32_t a = 1; a < q; a++) zmax = z[a] > zmax ? z[a] : zmax;                \
            REAL sum = 0;                                                                    \
            for (int32_t a = 0; a < q; a++) { z[a] = EXPF(z[a] - zmax); sum += z[a]; }       \
            const REAL ws = w[s];                                                            \
            const REAL inv = (REAL)1 / sum;                                                  \
            fxi -= (double)ws * (double)LOGF(z[si] * inv);                                   \
            for (int32_t a = 0; a < q; a++) z[a] = ws * z[a] * inv;                          \
            z[si] -= ws;                                                                     \
            for (int32_t a = 0; a < q; a++) gh[a] += z[a];                                   \
            for (int32_t j = 0; j < L; j++) {                                                \
                const int32_t sj = row[j];                                                   \
                if (j == i || sj >= q) continue;                                             \
                REAL *col = Gi + (int64_t)j * qq + (int64_t)sj * q;                          \
                for (int32_t a = 0; a < q; a++) col[a] += z[a];                              \
            }                                                                                \
        }                                                                                    \
        for (int32_t a = 0; a < q; a++)                                                      \
            g[(int64_t)i * q + a] = gh[a] + 2 * lambda_h * h[(int64_t)i * q + a];            \
        fx += fxi;                                                                           \
    }                                                                                        \
    double reg = 0.0;                                                                        \
    for (int64_t k = 0; k < (int64_t)L * q; k++) reg += (double)lambda_h * h[k] * h[k];      \
    {                                                                                        \
        REAL *gJ = g + (int64_t)L * q;                                                       \
        int64_t p = 0;                                                                       \
        for (int32_t i = 0; i < L; i++)                                                      \
            for (int32_t j = i + 1; j < L; j++, p++) {                                       \
                const REAL *Gij = G + (int64_t)i * blk + (int64_t)j * qq; /* [b][a] */        \
                const REAL *Gji = G + (int64_t)j * blk + (int64_t)i * qq; /* [a][b] */        \
                const REAL *B = J + p * qq;                                                  \
                REAL *O = gJ + p * qq;                                                       \
                for (int32_t a = 0; a < q; a++)                                              \
                    for (int32_t b = 0; b < q; b++) {                                        \
                        const REAL v = B[a * q + b];                                         \
                        O[a * q + b] = Gij[b * q + a] + Gji[a * q + b] + 2 * lambda_J * v;   \
                        reg += (double)lambda_J * v * v;                                     \
                    }                                                                        \
            }                                                                                \
    }                                                                                        \
    free(W); free(G);                                                                        \
    *nll_out = fx;                                                                           \
    *fx_out = fx + reg;                                                                      \
    return 0;                                                                                \
}

static void set_threads(int32_t n)
{
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

DEFINE_PLM_EVAL(plm_eval_f32_impl, float, expf, logf)
DEFINE_PLM_EVAL(plm_eval_f64_impl, double, exp, log)

int oracle_plm_eval_f32(const uint8_t *codes, int64_t N, int32_t L, int32_t q, const float *w,
                        const float *x, float lambda_h, float lambda_J, float *g,
                        double *fx_out, double *nll_out, int32_t nthreads)
{
    set_threads(nthreads);
    return plm_eval_f32_impl(codes, N, L, q, w, x, lambda_h, lambda_J, g, fx_out, nll_out, nthreads);
}

int oracle_plm_eval_f64(const uint8_t *codes, int64_t N, int32_t L, int32_t q, const double *w,
                        const double *x, double lambda_h, double lambda_J, double *g,
                        double *fx_out, double *nll_out, int32_t nthreads)
{
    set_threads(nthreads);
    return plm_eval_f64_impl(codes, N, L, q, w, x, lambda_h, lambda_J, g, fx_out, nll_out, nthreads);
}

int32_t oracle_max_threads(void)
{
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
