/*
 * gmm_oracle.c — CPU restatement of the Corv/CUDA-GMM-MPI EM hot path.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, bench.py's
 * cpu_baseline / --impl reference legs and __graft_entry__.smoke() may load
 * it, and only as the checker (or as the timed CPU baseline).  The product
 * (libgmm_b200.so) never links, loads or calls anything in oracle/.
 *
 * Parity status: the reference ships NO tests, golden vectors or sample data
 * (SURVEY.md §4) and its EM exists only as CUDA kernels, so it cannot run in
 * the (GPU-less) build container.  The oracle is pinned by
 *   (1) the fixtures in tests/golden/ref_c1_*, produced by the UNMODIFIED
 *       reference sources compiled for sm_90a (oracle/Makefile target `ref`,
 *       oracle/ref_wrapper.cu) and run on an H100 by tests/golden/make_ref_golden.sh;
 *   (2) an independent cross-check against scikit-learn's GaussianMixture
 *       M-step/E-step (tests/test_oracle.py).
 * Until (1) has been generated the header of tests/golden/README.md says
 * "parity unpinned".
 *
 * Every function cites the reference file:line it follows (paths relative to
 * the reference repository).  The arithmetic ORDER of the reference's block/thread
 * decomposition is restated literally where it affects FP32 results
 * (strided per-thread partial sums, butterfly reduction, thread-0 serial sum).
 *
 * Build twice: -DORACLE_REAL=float  (reference arithmetic, the "port" that is
 * timed as the CPU baseline) and -DORACLE_REAL=double (ground truth for
 * parity).  State (clusters_t, memberships) is float in both, as in the
 * reference.
 *
 * Conscious deviations from the reference (SURVEY.md §8 quirks), identical in
 * the product:
 *   Q1  regulariser avgvar is added once (G = 1 semantics) for any GPU count.
 *   Q2  mean / avgvar use the whole data set, not GPU-0's shard.
 *   Q3  per-iteration constants use ln det (device `invert`); the merge
 *       distance uses invert_cpu's log10 det — both mirrored literally.
 *   Q4  compute_pi writes pi[c] (reference writes pi[threadIdx.x]; identical
 *       for K <= 256).
 *   Q5  iteration bounds are arguments (reference: MIN_ITERS = MAX_ITERS = 100).
 */
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#ifndef ORACLE_REAL
#define ORACLE_REAL float
#endif
typedef ORACLE_REAL real;

#define PI 3.1415926535897931            /* gaussian.h:11 */
#define COVARIANCE_DYNAMIC_RANGE 1E3     /* gaussian.h:12 */
#define NUM_BLOCKS 16                    /* gaussian.h:13 */
#define NUM_THREADS_ESTEP 512            /* gaussian.h:14 */
#define NUM_THREADS_MSTEP 256            /* gaussian.h:15 */

typedef struct {                          /* gaussian.h:62-76 */
    float* N; float* pi; float* constant; float* avgvar;
    float* means; float* R; float* Rinv; float* memberships;
} clusters_t;

/* real-typed libm wrappers: logf/expf/fmaxf in the reference */
static inline real r_log(real x)  { return sizeof(real) == 4 ? (real)logf((float)x) : (real)log((double)x); }
static inline real r_exp(real x)  { return sizeof(real) == 4 ? (real)expf((float)x) : (real)exp((double)x); }
static inline real r_max(real a, real b) { return a > b ? a : b; }
static inline real r_abs(real a) { return a < 0 ? -a : a; }

int oracle_real_bytes(void) { return (int)sizeof(real); }

/* parallelSum (gaussian_kernel.cu:332-344): butterfly, ndata power of two.
 * Every slot ends with the same value; returns data[0]. */
static real butterfly_sum(real* data, int ndata) {
    real* t = (real*)malloc(sizeof(real) * (size_t)ndata);
    for (int bit = ndata >> 1; bit > 0; bit >>= 1) {
        for (int tid = 0; tid < ndata; tid++) t[tid] = data[tid] + data[tid ^ bit];
        memcpy(data, t, sizeof(real) * (size_t)ndata);
    }
    free(t);
    return data[0];
}

/* AoS [N][D] -> SoA [D][N] (gaussian.cu:212-218) */
void oracle_transpose(const float* aos, int N, int D, float* soa) {
    for (int e = 0; e < N; e++)
        for (int d = 0; d < D; d++) soa[(size_t)d * N + e] = aos[(size_t)e * D + d];
}

/* ---------------------------------------------------------------------------
 * invert (gaussian_kernel.cu:107-169) == invert_cpu (invert_matrix.cpp:25-101)
 * apart from the logarithm: device uses logf (ln), host uses log10 (quirk Q3).
 * In-place Crout LU without pivoting; expressions kept literally (including
 * the double-typed 1.0 literals).
 * ------------------------------------------------------------------------- */
static void invert_literal(float* data, int actualsize, float* log_determinant, int use_log10) {
    int maxsize = actualsize;
    int n = actualsize;
    *log_determinant = 0.0;
    if (actualsize == 1) {
        *log_determinant = logf(data[0]);
        data[0] = 1.0 / data[0];
    } else if (actualsize >= 2) {
        for (int i = 1; i < actualsize; i++) data[i] /= data[0];
        for (int i = 1; i < actualsize; i++) {
            for (int j = i; j < actualsize; j++) {
                float sum = 0.0;
                for (int k = 0; k < i; k++) sum += data[j * maxsize + k] * data[k * maxsize + i];
                data[j * maxsize + i] -= sum;
            }
            if (i == actualsize - 1) continue;
            for (int j = i + 1; j < actualsize; j++) {
                float sum = 0.0;
                for (int k = 0; k < i; k++) sum += data[i * maxsize + k] * data[k * maxsize + j];
                data[i * maxsize + j] = (data[i * maxsize + j] - sum) / data[i * maxsize + i];
            }
        }
        for (int i = 0; i < actualsize; i++) {
            if (use_log10) *log_determinant += log10(fabs(data[i * n + i]));   /* invert_matrix.cpp:61 */
            else           *log_determinant += logf(fabs(data[i * n + i]));    /* gaussian_kernel.cu:139 */
        }
        for (int i = 0; i < actualsize; i++)
            for (int j = i; j < actualsize; j++) {
                float x = 1.0;
                if (i != j) {
                    x = 0.0;
                    for (int k = i; k < j; k++) x -= data[j * maxsize + k] * data[k * maxsize + i];
                }
                data[j * maxsize + i] = x / data[j * maxsize + j];
            }
        for (int i = 0; i < actualsize; i++)
            for (int j = i; j < actualsize; j++) {
                if (i == j) continue;
                float sum = 0.0;
                for (int k = i; k < j; k++)
                    sum += data[k * maxsize + j] * ((i == k) ? 1.0 : data[i * maxsize + k]);
                data[i * maxsize + j] = -sum;
            }
        for (int i = 0; i < actualsize; i++)
            for (int j = 0; j < actualsize; j++) {
                float sum = 0.0;
                for (int k = ((i > j) ? i : j); k < actualsize; k++)
                    sum += ((j == k) ? 1.0 : data[j * maxsize + k]) * data[k * maxsize + i];
                data[j * maxsize + i] = sum;
            }
    }
}

static void invert_exact(double* data, int actualsize, double* log_determinant, int use_log10) {
    int maxsize = actualsize;
    int n = actualsize;
    *log_determinant = 0.0;
    if (actualsize == 1) {
        *log_determinant = log(data[0]);
        data[0] = 1.0 / data[0];
    } else if (actualsize >= 2) {
        for (int i = 1; i < actualsize; i++) data[i] /= data[0];
        for (int i = 1; i < actualsize; i++) {
            for (int j = i; j < actualsize; j++) {
                double sum = 0.0;
                for (int k = 0; k < i; k++) sum += data[j * maxsize + k] * data[k * maxsize + i];
                data[j * maxsize + i] -= sum;
            }
            if (i == actualsize - 1) continue;
            for (int j = i + 1; j < actualsize; j++) {
                double sum = 0.0;
                for (int k = 0; k < i; k++) sum += data[i * maxsize + k] * data[k * maxsize + j];
                data[i * maxsize + j] = (data[i * maxsize + j] - sum) / data[i * maxsize + i];
            }
        }
        for (int i = 0; i < actualsize; i++) {
            if (use_log10) *log_determinant += log10(fabs(data[i * n + i]));   /* invert_matrix.cpp:61 */
            else           *log_determinant += log(fabs(data[i * n + i]));    /* gaussian_kernel.cu:139 */
        }
        for (int i = 0; i < actualsize; i++)
            for (int j = i; j < actualsize; j++) {
                double x = 1.0;
                if (i != j) {
                    x = 0.0;
                    for (int k = i; k < j; k++) x -= data[j * maxsize + k] * data[k * maxsize + i];
                }
                data[j * maxsize + i] = x / data[j * maxsize + j];
            }
        for (int i = 0; i < actualsize; i++)
            for (int j = i; j < actualsize; j++) {
                if (i == j) continue;
                double sum = 0.0;
                for (int k = i; k < j; k++)
                    sum += data[k * maxsize + j] * ((i == k) ? 1.0 : data[i * maxsize + k]);
                data[i * maxsize + j] = -sum;
            }
        for (int i = 0; i < actualsize; i++)
            for (int j = 0; j < actualsize; j++) {
                double sum = 0.0;
                for (int k = ((i > j) ? i : j); k < actualsize; k++)
                    sum += ((j == k) ? 1.0 : data[j * maxsize + k]) * data[k * maxsize + i];
                data[j * maxsize + i] = sum;
            }
    }
}

/* ORACLE_REAL=float : the reference's FP32 routine, literally.
 * ORACLE_REAL=double: the same elimination (no pivoting) carried out in double on the float
 * input and rounded back to float — the ground-truth build removes the reference's FP32
 * round-off from the inverse (the float LU alone perturbs Rinv by ~cond*2^-24*D). */
void oracle_invert(float* data, int actualsize, float* log_determinant, int use_log10) {
    if (sizeof(real) == 4) { invert_literal(data, actualsize, log_determinant, use_log10); return; }
    double m[32 * 32], ld;
    for (int i = 0; i < actualsize * actualsize; i++) m[i] = data[i];
    invert_exact(m, actualsize, &ld, use_log10);
    for (int i = 0; i < actualsize * actualsize; i++) data[i] = (float)m[i];
    *log_determinant = (float)ld;
}

/* ---------------------------------------------------------------------------
 * constants_kernel (gaussian_kernel.cu:250-259): compute_constants (196-243)
 * for every cluster, then compute_pi (172-193).
 * ------------------------------------------------------------------------- */
void oracle_constants(clusters_t* c, int K, int D) {
    for (int k = 0; k < K; k++) {
        float* m = c->Rinv + (size_t)k * D * D;
        memcpy(m, c->R + (size_t)k * D * D, sizeof(float) * D * D);
        float log_det;
        oracle_invert(m, D, &log_det, 0);
        c->constant[k] = -D * 0.5f * logf(2.0f * PI) - 0.5f * log_det;   /* :241 */
    }
    float sum = 0.0;                                                     /* :176-181 */
    for (int i = 0; i < K; i++) sum += c->N[i];
    for (int k = 0; k < K; k++) {                                        /* :184-190, Q4 */
        if (c->N[k] < 0.5f) c->pi[k] = 1e-10;
        else                c->pi[k] = c->N[k] / sum;
    }
}

/* ---------------------------------------------------------------------------
 * Seeding: seed_clusters kernel (gaussian_kernel.cu:269-328) with mvtmeans
 * (54-69) and averageVariance (71-102); constants_kernel (gaussian.cu:404);
 * host seed_clusters (gaussian.cu:108-123).
 * ------------------------------------------------------------------------- */
void oracle_seed(const float* aos, int N, int D, int K, clusters_t* c) {
    real* means = (real*)calloc((size_t)D, sizeof(real));
    real* var = (real*)calloc((size_t)D, sizeof(real));
    for (int d = 0; d < D; d++) {                      /* mvtmeans: serial per dimension */
        real s = 0;
        for (int i = 0; i < N; i++) s += aos[(size_t)i * D + d];
        means[d] = s / (real)N;
    }
    real total = 0;
    for (int d = 0; d < D; d++) {                      /* averageVariance */
        real s = 0;
        for (int j = 0; j < N; j++) s += (real)aos[(size_t)j * D + d] * (real)aos[(size_t)j * D + d];
        var[d] = s / (real)N - means[d] * means[d];
        total += var[d];
    }
    float avgvar = (float)(total / (real)D);
    float seed = (K > 1) ? (N - 1.0f) / (K - 1.0f) : 0.0f;   /* float arithmetic, Q9 */
    for (int k = 0; k < K; k++) {
        for (int d = 0; d < D; d++) c->means[k * D + d] = aos[(size_t)((int)(k * seed)) * D + d];
        for (int i = 0; i < D * D; i++) c->R[(size_t)k * D * D + i] = (i / D == i % D) ? 1.0f : 0.0f;
        c->pi[k] = 1.0f / ((float)K);
        c->N[k] = ((float)N) / ((float)K);
        c->avgvar[k] = avgvar / COVARIANCE_DYNAMIC_RANGE;
    }
    oracle_constants(c, K, D);                         /* gaussian.cu:404 */
    for (int k = 0; k < K; k++) c->N[k] = N / K;       /* host seed: INTEGER division, gaussian.cu:118 */
    free(means); free(var);
}

/* compute_indices (gaussian_kernel.cu:367-381) */
static void block_range(int N, int nblocks, int b, int* start, int* stop) {
    int per = N / nblocks;
    per = per - (per % 16);
    *start = b * per;
    *stop = (b == nblocks - 1) ? N : (b + 1) * per;
}

/* ---------------------------------------------------------------------------
 * estep1 (gaussian_kernel.cu:383-444): unnormalised log numerators.
 * Full D x D double loop, exactly as written (:435-439).
 * ------------------------------------------------------------------------- */
void oracle_estep1(const float* soa, int N, int D, int K, clusters_t* c) {
    /* every (cluster, event) value is independent: clusters x event chunks are spread over the threads
     * (the arithmetic per value is the reference's, whatever the decomposition) */
    const int EB = 8192, nb = (N + EB - 1) / EB;
#pragma omp parallel for collapse(2) schedule(static)
    for (int k = 0; k < K; k++)
      for (int b = 0; b < nb; b++) {
        const float* means = c->means + (size_t)k * D;
        const float* Rinv = c->Rinv + (size_t)k * D * D;
        real cluster_pi = c->pi[k];
        real constant = c->constant[k];
        real logpi = r_log(cluster_pi);
        const int e1 = (b + 1) * EB < N ? (b + 1) * EB : N;
        for (int e = b * EB; e < e1; e++) {
            real like = 0;
            for (int i = 0; i < D; i++)
                for (int j = 0; j < D; j++)
                    like += ((real)soa[(size_t)i * N + e] - (real)means[i]) *
                            ((real)soa[(size_t)j * N + e] - (real)means[j]) * (real)Rinv[i * D + j];
            c->memberships[(size_t)k * N + e] = (float)((real)-0.5 * like + constant + logpi);
        }
    }
}

/* ---------------------------------------------------------------------------
 * estep2 (gaussian_kernel.cu:446-512): log-sum-exp normalisation in place and
 * the 16 per-block likelihood partials; host sum of the partials in float
 * (gaussian.cu:733-739).  Returns the log-likelihood.
 * ------------------------------------------------------------------------- */
float oracle_estep2(int N, int K, clusters_t* c) {
    float partial[NUM_BLOCKS];
    /* pass 1 (independent per event, spread over all threads): denominators + normalisation in place;
     * pass 2: the per-block / per-thread partial sums of the denominators in the reference's order */
    real* den_all = (real*)malloc(sizeof(real) * (size_t)(N > 0 ? N : 1));
    const int EB = 4096, nb = (N + EB - 1) / EB;
#pragma omp parallel for schedule(static)
    for (int b = 0; b < nb; b++) {
        const int e1 = (b + 1) * EB < N ? (b + 1) * EB : N;
        for (int e = b * EB; e < e1; e++) {
            real mx = c->memberships[e];
            for (int k = 1; k < K; k++) mx = r_max(mx, (real)c->memberships[(size_t)k * N + e]);
            real den = 0;
            for (int k = 0; k < K; k++) den += r_exp((real)c->memberships[(size_t)k * N + e] - mx);
            den = mx + r_log(den);
            den_all[e] = den;
            for (int k = 0; k < K; k++)
                c->memberships[(size_t)k * N + e] = (float)r_exp((real)c->memberships[(size_t)k * N + e] - den);
        }
    }
#pragma omp parallel for schedule(static)
    for (int b = 0; b < NUM_BLOCKS; b++) {
        int start, stop;
        block_range(N, NUM_BLOCKS, b, &start, &stop);
        real thread_ll[NUM_THREADS_ESTEP];
        for (int t = 0; t < NUM_THREADS_ESTEP; t++) thread_ll[t] = 0;
        for (int e = start; e < stop; e++)
            thread_ll[(e - start) % NUM_THREADS_ESTEP] += den_all[e];     /* thread tid owns start+tid+512*i */
        partial[b] = (float)butterfly_sum(thread_ll, NUM_THREADS_ESTEP);
    }
    free(den_all);
    float likelihood = 0.0;
    for (int i = 0; i < NUM_BLOCKS; i++) likelihood += partial[i];
    return likelihood;
}

float oracle_estep(const float* soa, int N, int D, int K, clusters_t* c) {
    oracle_estep1(soa, N, D, K, c);
    return oracle_estep2(N, K, c);
}

/* ---------------------------------------------------------------------------
 * M-step, in the reference's order (gaussian.cu:538-687):
 *   mstep_N (gaussian_kernel.cu:551-577)
 *   mstep_means (522-545) + host division, 0 if N <= 0.5 (gaussian.cu:611-622)
 *   mstep_covariance1 (605-677): centred on the NEW means, 0 if N < 1.0,
 *     += avgvar on the diagonal, then host division / identity
 *     (gaussian.cu:663-679).
 * ------------------------------------------------------------------------- */
void oracle_mstep(const float* soa, int N, int D, int K, clusters_t* c) {
#pragma omp parallel for schedule(static)
    for (int k = 0; k < K; k++) {                                  /* mstep_N */
        real part[NUM_THREADS_MSTEP];
        for (int t = 0; t < NUM_THREADS_MSTEP; t++) part[t] = 0;
        const float* g = c->memberships + (size_t)k * N;
        for (int e = 0; e < N; e++) part[e % NUM_THREADS_MSTEP] += g[e];
        c->N[k] = (float)butterfly_sum(part, NUM_THREADS_MSTEP);
    }
#pragma omp parallel for collapse(2) schedule(static)
    for (int k = 0; k < K; k++)                                    /* mstep_means */
        for (int d = 0; d < D; d++) {
            real part[NUM_THREADS_MSTEP];
            for (int t = 0; t < NUM_THREADS_MSTEP; t++) part[t] = 0;
            const float* g = c->memberships + (size_t)k * N;
            const float* x = soa + (size_t)d * N;
            for (int e = 0; e < N; e++) part[e % NUM_THREADS_MSTEP] += (real)x[e] * (real)g[e];
            float s = (float)butterfly_sum(part, NUM_THREADS_MSTEP);
            if (c->N[k] > 0.5f) c->means[k * D + d] = s / c->N[k];  /* gaussian.cu:614-618 */
            else                c->means[k * D + d] = 0.0f;
        }
    int ntri = D * (D + 1) / 2;
#pragma omp parallel for collapse(2) schedule(static)
    for (int k = 0; k < K; k++)                                    /* mstep_covariance1 */
        for (int t = 0; t < ntri; t++) {
            int row = 0, col = 0, i = 0;                           /* compute_row_col :586-598 */
            for (int r = 0; r < D && i <= t; r++)
                for (int cc = 0; cc <= r; cc++) { if (i == t) { row = r; col = cc; } i++; }
            real part[NUM_THREADS_MSTEP];
            for (int q = 0; q < NUM_THREADS_MSTEP; q++) part[q] = 0;
            const float* g = c->memberships + (size_t)k * N;
            const float* xr = soa + (size_t)row * N;
            const float* xc = soa + (size_t)col * N;
            real mr = c->means[k * D + row], mc = c->means[k * D + col];
            for (int e = 0; e < N; e++)
                part[e % NUM_THREADS_MSTEP] += ((real)xr[e] - mr) * ((real)xc[e] - mc) * (real)g[e];
            real cov = 0;                                          /* thread-0 serial sum :653-657 */
            for (int q = 0; q < NUM_THREADS_MSTEP; q++) cov += part[q];
            float v = (c->N[k] >= 1.0f) ? (float)cov : 0.0f;       /* :658-668 */
            float* Rk = c->R + (size_t)k * D * D;
            Rk[row * D + col] = v;
            Rk[col * D + row] = v;
            if (row == col) Rk[col * D + row] += c->avgvar[k];     /* :673-675 */
        }
    for (int k = 0; k < K; k++) {                                  /* gaussian.cu:663-679 */
        float* Rk = c->R + (size_t)k * D * D;
        if (c->N[k] > 0.5f) {
            for (int d = 0; d < D * D; d++) Rk[d] /= c->N[k];
        } else {
            for (int i = 0; i < D; i++)
                for (int j = 0; j < D; j++) Rk[i * D + j] = (i == j) ? 1.0f : 0.0f;
        }
    }
}

/* epsilon (gaussian.cu:458) */
float oracle_epsilon(int D, int N) {
    return (1 + D + 0.5 * (D + 1) * D) * log((float)N * D) * 0.01;
}

/* ---------------------------------------------------------------------------
 * EM for a fixed K (gaussian.cu:487-755): initial E-step, then
 * while(iters < MIN || (|change| > eps && iters < MAX)) { M; constants; E }.
 * `soa` is the [D][N] transpose.  Returns the final likelihood.
 * ------------------------------------------------------------------------- */
float oracle_em(const float* soa, int N, int D, int K, clusters_t* c,
                int min_iters, int max_iters, float epsilon, int* iters_out) {
    float likelihood = oracle_estep(soa, N, D, K, c);
    float old_likelihood;
    float change = epsilon * 2;
    int iters = 0;
    while (iters < min_iters || (fabs(change) > epsilon && iters < max_iters)) {
        old_likelihood = likelihood;
        oracle_mstep(soa, N, D, K, c);
        oracle_constants(c, K, D);
        likelihood = oracle_estep(soa, N, D, K, c);
        change = likelihood - old_likelihood;
        iters++;
    }
    if (iters_out) *iters_out = iters;
    return likelihood;
}

/* ---- order reduction (gaussian.cu:825-907, 1203-1264) -------------------- */

float oracle_rissanen(float likelihood, int K, int D, int N) {   /* gaussian.cu:826 */
    return -likelihood + 0.5 * (K * (1 + D + 0.5 * (D + 1) * D) - 1) * logf((float)N * D);
}

static void copy_cluster(clusters_t dest, int c_dest, clusters_t src, int c_src, int D) {   /* :1254-1264 */
    dest.N[c_dest] = src.N[c_src];
    dest.pi[c_dest] = src.pi[c_src];
    dest.constant[c_dest] = src.constant[c_src];
    dest.avgvar[c_dest] = src.avgvar[c_src];
    memcpy(&dest.means[c_dest * D], &src.means[c_src * D], sizeof(float) * D);
    memcpy(&dest.R[(size_t)c_dest * D * D], &src.R[(size_t)c_src * D * D], sizeof(float) * D * D);
    memcpy(&dest.Rinv[(size_t)c_dest * D * D], &src.Rinv[(size_t)c_src * D * D], sizeof(float) * D * D);
}

static void add_clusters(clusters_t cl, int c1, int c2, clusters_t tmp, int D) {            /* :1210-1252 */
    float wt1 = (cl.N[c1]) / (cl.N[c1] + cl.N[c2]);
    float wt2 = 1.0f - wt1;
    for (int i = 0; i < D; i++) tmp.means[i] = wt1 * cl.means[c1 * D + i] + wt2 * cl.means[c2 * D + i];
    for (int i = 0; i < D; i++)
        for (int j = i; j < D; j++) {
            tmp.R[i * D + j] = ((tmp.means[i] - cl.means[c1 * D + i]) * (tmp.means[j] - cl.means[c1 * D + j])
                                + cl.R[(size_t)c1 * D * D + i * D + j]) * wt1;
            tmp.R[i * D + j] += ((tmp.means[i] - cl.means[c2 * D + i]) * (tmp.means[j] - cl.means[c2 * D + j])
                                 + cl.R[(size_t)c2 * D * D + i * D + j]) * wt2;
            tmp.R[j * D + i] = tmp.R[i * D + j];
        }
    tmp.pi[0] = cl.pi[c1] + cl.pi[c2];
    tmp.N[0] = cl.N[c1] + cl.N[c2];
    float log_determinant;
    memcpy(tmp.Rinv, tmp.R, sizeof(float) * D * D);
    oracle_invert(tmp.Rinv, D, &log_determinant, 1);               /* invert_cpu: log10, Q3 */
    tmp.constant[0] = (-D) * 0.5 * logf(2 * PI) - 0.5 * log_determinant;
    tmp.avgvar[0] = cl.avgvar[0];
}

static float cluster_distance(clusters_t cl, int c1, int c2, clusters_t tmp, int D) {       /* :1203-1208 */
    add_clusters(cl, c1, c2, tmp, D);
    return cl.N[c1] * cl.constant[c1] + cl.N[c2] * cl.constant[c2] - tmp.N[0] * tmp.constant[0];
}

static void alloc_scratch(clusters_t* s, int D) {
    s->N = (float*)malloc(sizeof(float)); s->pi = (float*)malloc(sizeof(float));
    s->constant = (float*)malloc(sizeof(float)); s->avgvar = (float*)malloc(sizeof(float));
    s->means = (float*)malloc(sizeof(float) * D);
    s->R = (float*)malloc(sizeof(float) * D * D); s->Rinv = (float*)malloc(sizeof(float) * D * D);
    s->memberships = NULL;
}
static void free_scratch(clusters_t* s) {
    free(s->N); free(s->pi); free(s->constant); free(s->avgvar); free(s->means); free(s->R); free(s->Rinv);
}

/* One order-reduction step (gaussian.cu:860-907).  Returns the new K. */
int oracle_reduce_order(clusters_t* c, int K, int D, int* out_c1, int* out_c2) {
    clusters_t scratch; alloc_scratch(&scratch, D);
    for (int i = K - 1; i >= 0; i--) {                              /* empties :866-874 */
        if (c->N[i] < 0.5) {
            for (int j = i; j < K - 1; j++) copy_cluster(*c, j, *c, j + 1, D);
            K--;
        }
    }
    int min_c1 = 0, min_c2 = 1;
    float min_distance = 0.0;
    for (int c1 = 0; c1 < K; c1++)                                  /* :882-894 */
        for (int c2 = c1 + 1; c2 < K; c2++) {
            float distance = cluster_distance(*c, c1, c2, scratch, D);
            if ((c1 == 0 && c2 == 1) || distance < min_distance) {
                min_distance = distance; min_c1 = c1; min_c2 = c2;
            }
        }
    if (K >= 2) {
        add_clusters(*c, min_c1, min_c2, scratch, D);                   /* :899-907 */
        copy_cluster(*c, min_c1, scratch, 0, D);
        for (int i = min_c2; i < K - 1; i++) copy_cluster(*c, i, *c, i + 1, D);
    }
    if (out_c1) *out_c1 = min_c1;
    if (out_c2) *out_c2 = min_c2;
    free_scratch(&scratch);
    return K - 1;      /* the for-loop decrement of gaussian.cu:479 */
}

/* ---------------------------------------------------------------------------
 * The whole outer loop (gaussian.cu:479-960), single GPU semantics.
 * clusters / saved must be sized for K0 (saved->memberships [K0*N] or NULL).
 * Returns ideal_num_clusters; *min_rissanen_out receives the best score.
 * ------------------------------------------------------------------------- */
int oracle_fit(const float* aos, int N, int D, int K0, int target_K,
               int min_iters, int max_iters, clusters_t* c, clusters_t* saved,
               float* min_rissanen_out) {
    float* soa = (float*)malloc(sizeof(float) * (size_t)N * D);
    oracle_transpose(aos, N, D, soa);
    int stop_number = (target_K == 0) ? 1 : target_K;
    oracle_seed(aos, N, D, K0, c);
    float epsilon = oracle_epsilon(D, N);
    float min_rissanen = 0;
    int ideal = K0;
    for (int K = K0; K >= stop_number; ) {
        int iters;
        float likelihood = oracle_em(soa, N, D, K, c, min_iters, max_iters, epsilon, &iters);
        float rissanen = oracle_rissanen(likelihood, K, D, N);
        if (K == K0 || (rissanen < min_rissanen && target_K == 0) || K == target_K) {   /* :839 */
            min_rissanen = rissanen;
            ideal = K;
            memcpy(saved->N, c->N, sizeof(float) * K); memcpy(saved->pi, c->pi, sizeof(float) * K);
            memcpy(saved->constant, c->constant, sizeof(float) * K);
            memcpy(saved->avgvar, c->avgvar, sizeof(float) * K);
            memcpy(saved->means, c->means, sizeof(float) * K * D);
            memcpy(saved->R, c->R, sizeof(float) * (size_t)K * D * D);
            memcpy(saved->Rinv, c->Rinv, sizeof(float) * (size_t)K * D * D);
            if (saved->memberships) memcpy(saved->memberships, c->memberships, sizeof(float) * (size_t)K * N);
        }
        if (K > stop_number) K = oracle_reduce_order(c, K, D, NULL, NULL);
        else break;
    }
    if (min_rissanen_out) *min_rissanen_out = min_rissanen;
    free(soa);
    return ideal;
}
