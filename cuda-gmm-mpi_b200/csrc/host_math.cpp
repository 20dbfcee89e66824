// host_math.cpp — GPU-free host numerics: M-step finalisation, constants
// (DxD inversion stays on the host: BASELINE.json north_star), seeding,
// Rissanen score, order reduction.  Semantics follow the reference
// (file:line cited per function); the code is written from scratch.
#include "host_math.h"

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>

namespace gmm {

static thread_local std::string g_err;
void set_error(const std::string& msg) { g_err = msg; }
int fail(int code, const std::string& msg) { g_err = msg; return code; }
const char* last_error_cstr() { return g_err.c_str(); }

// ---------------------------------------------------------------------------
// LU inverse without pivoting.  Same contract as invert_cpu
// (invert_matrix.cpp:25-101) / device invert (gaussian_kernel.cu:107-169):
// in place, no row exchanges, log|det| accumulated from the pivots.
// Doolittle factorisation A = L U (unit L), then A^-1 column by column.
// ---------------------------------------------------------------------------
template <class T>
void lu_inverse_nopivot(T* __restrict__ a, int n, T* logabsdet, T* __restrict__ w) {
    // Elimination applied to [A | I]: every inner loop is an axpy over a contiguous row (vectorises
    // without reassociation).  Forward pass leaves U in the upper triangle of `a` and L^-1 in `w`;
    // the backward pass turns `w` into U^-1 L^-1 = A^-1.
    for (int i = 0; i < n; i++)
        for (int j = 0; j < n; j++) w[i * n + j] = (i == j) ? T(1) : T(0);
    T ld = 0;
    for (int k = 0; k < n; k++) {
        const T piv = a[k * n + k];
        ld += std::log(std::fabs(piv));
        const T rp = T(1) / piv;
        const T* ak = a + k * n;
        const T* wk = w + k * n;
        for (int i = k + 1; i < n; i++) {
            const T l = a[i * n + k] * rp;
            T* ai = a + i * n;
            T* wi = w + i * n;
            for (int j = k + 1; j < n; j++) ai[j] -= l * ak[j];
            for (int j = 0; j <= k; j++) wi[j] -= l * wk[j];
        }
    }
    for (int k = n - 1; k >= 0; k--) {
        T* wk = w + k * n;
        for (int j = k + 1; j < n; j++) {
            const T u = a[k * n + j];
            const T* wj = w + j * n;
            for (int c = 0; c < n; c++) wk[c] -= u * wj[c];
        }
        const T rp = T(1) / a[k * n + k];
        for (int c = 0; c < n; c++) wk[c] *= rp;
    }
    for (int i = 0; i < n * n; i++) a[i] = w[i];
    *logabsdet = ld;
}
template void lu_inverse_nopivot<float>(float*, int, float*, float*);
template void lu_inverse_nopivot<double>(double*, int, double*, double*);

static const double kPi = 3.1415926535897931;   // gaussian.h:11

// constants_kernel (gaussian_kernel.cu:250-259): compute_constants (196-243)
// per cluster + compute_pi (172-193).  Inversion in double, results stored as
// float like the reference's clusters_t.
void constants_cluster(int k, int D, clusters_t* c) {
    double m[GMM_MAX_DIMENSIONS * GMM_MAX_DIMENSIONS], w[GMM_MAX_DIMENSIONS * GMM_MAX_DIMENSIONS];
    const float* R = c->R + (size_t)k * D * D;
    for (int i = 0; i < D * D; i++) m[i] = R[i];
    double ld;
    lu_inverse_nopivot<double>(m, D, &ld, w);
    float* Ri = c->Rinv + (size_t)k * D * D;
    for (int i = 0; i < D * D; i++) Ri[i] = (float)m[i];
    c->constant[k] = (float)(-D * 0.5 * std::log(2.0 * kPi) - 0.5 * ld);   // :241
}

// The same for a symmetric positive definite R through ONE factorisation: R = U U^T (U upper triangular, "reverse"
// Cholesky), W = U^-1 (upper triangular), Rinv = W^T W, ln det R = 2 sum ln U_ii — a third of the arithmetic of the
// LU inverse plus the separate factorisation of Rinv the tensor E-step's operand needs (W is handed to it directly).
// Returns false (nothing written) when R is not positive definite: the caller then takes the no-pivot LU path, whose
// semantics on such matrices are the reference's (invert_matrix.cpp:25-101).
// Every product is rounded before it is added (no fused multiply-add, whatever the compiler vectorises): the device-side
// finalisation (finalize_params_kernel) evaluates the same operations in the same order with __dmul_rn / __dsub_rn, so the
// two finalisations produce bit-identical factors and E-step operands.
#pragma GCC push_options
#pragma GCC optimize("fp-contract=off")
bool reverse_cholesky(const float* R, int D, double (*U)[GMM_MAX_DIMENSIONS], double* ld_out) {
    double ld = 0.0;
    for (int j = D - 1; j >= 0; j--) {
        double d = R[j * D + j];
        for (int m = j + 1; m < D; m++) d -= U[j][m] * U[j][m];
        if (!(d > 0.0) || !std::isfinite(d)) return false;
        const double piv = std::sqrt(d), rp = 1.0 / piv;
        U[j][j] = piv;
        ld += std::log(piv);
        for (int i = 0; i < j; i++) {
            double v = 0.5 * ((double)R[i * D + j] + (double)R[j * D + i]);
            for (int m = j + 1; m < D; m++) v -= U[i][m] * U[j][m];
            U[i][j] = v * rp;
        }
    }
    *ld_out = ld;
    return true;
}

bool constants_cluster_spd(int k, int D, clusters_t* c, double* W /* [D][D] out */, double* half_ln_det) {
    double U[GMM_MAX_DIMENSIONS][GMM_MAX_DIMENSIONS];
    double ld;
    if (!reverse_cholesky(c->R + (size_t)k * D * D, D, U, &ld)) return false;
    if (half_ln_det) *half_ln_det = ld;
    // W = U^-1 (upper triangular), column by column: W[i][j] = -(sum_{m=i+1..j} U[i][m] W[m][j]) / U[i][i]
    for (int j = 0; j < D; j++) {
        for (int i = D - 1; i > j; i--) W[i * D + j] = 0.0;
        W[j * D + j] = 1.0 / U[j][j];
        for (int i = j - 1; i >= 0; i--) {
            double v = 0.0;
            for (int m = i + 1; m <= j; m++) v -= U[i][m] * W[m * D + j];
            W[i * D + j] = v / U[i][i];
        }
    }
    float* Ri = c->Rinv + (size_t)k * D * D;
    for (int i = 0; i < D; i++)
        for (int j = i; j < D; j++) {                   // (W^T W)[i][j] = sum_{m <= i} W[m][i] W[m][j]
            double v = 0.0;
            for (int m = 0; m <= i; m++) v += W[m * D + i] * W[m * D + j];
            Ri[i * D + j] = (float)v;
            Ri[j * D + i] = (float)v;
        }
    c->constant[k] = (float)(-D * 0.5 * std::log(2.0 * kPi) - 0.5 * (2.0 * ld));   // gaussian_kernel.cu:241
    return true;
}
#pragma GCC pop_options

void mixing_weights(int K, clusters_t* c) {
    double sum = 0;                                                            // :176-181
    for (int k = 0; k < K; k++) sum += c->N[k];
    for (int k = 0; k < K; k++)                                                // :184-190
        c->pi[k] = (c->N[k] < 0.5f) ? 1e-10f : (float)(c->N[k] / sum);
}

void constants_from_R(int K, int D, clusters_t* c, int num_threads) {
    (void)num_threads;
#pragma omp parallel for schedule(static) num_threads(num_threads) if (K >= 8 && num_threads > 1)
    for (int k = 0; k < K; k++) {
        double W[GMM_MAX_DIMENSIONS * GMM_MAX_DIMENSIONS];
        if (!constants_cluster_spd(k, D, c, W)) constants_cluster(k, D, c);     // not positive definite: the no-pivot LU semantics
    }
    mixing_weights(K, c);
}

// Host side of the M-step (gaussian.cu:611-622 means, :663-679 covariance)
// together with the device-side rules of mstep_covariance1
// (gaussian_kernel.cu:658-675: zero if N < 1.0, += avgvar on the diagonal
// BEFORE the division).  Input statistics are taken about `shift`:
//   S0 = sum g, S1 = sum g (x - shift), S2 = sum g (x - shift)(x - shift)^T
// so that  sum g (x - mu)(x - mu)^T = S2 - S1 S1^T / S0  with mu = shift + S1/S0.
void finalize_cluster(const double* stats, const double* shift, int k, int D, clusters_t* c) {
    const int F = num_features(D);
    const double* s = stats + (size_t)k * F;
    const double S0 = s[0];
    const float Nf = (float)S0;
    c->N[k] = Nf;
    float* mu = c->means + (size_t)k * D;
    float* R = c->R + (size_t)k * D * D;
    double m[GMM_MAX_DIMENSIONS];
    for (int d = 0; d < D; d++) {
        m[d] = (S0 != 0.0) ? s[1 + d] / S0 : 0.0;
        mu[d] = (Nf > 0.5f) ? (float)(m[d] + shift[d]) : 0.0f;              // gaussian.cu:614-618
    }
    if (Nf > 0.5f) {
        const double inv = 1.0 / (double)Nf;
        for (int i = 0; i < D; i++)
            for (int j = 0; j <= i; j++) {
                // kernel :658-668; the product is fused with the subtraction explicitly, as finalize_params_kernel fuses it
                // (bit identity of the two finalisations must not hang on whether this compiler contracts the line)
                double cov = (Nf >= 1.0f) ? std::fma(-m[i], s[1 + j], s[feat2(D, i, j)]) : 0.0;
                if (i == j) cov += c->avgvar[k];                                      // kernel :673-675
                const float v = (float)(cov * inv);                                   // gaussian.cu:664-667
                R[i * D + j] = v;
                R[j * D + i] = v;
            }
    } else {                                                                          // gaussian.cu:668-677
        for (int i = 0; i < D; i++)
            for (int j = 0; j < D; j++) R[i * D + j] = (i == j) ? 1.0f : 0.0f;
    }
}

void finalize_from_stats(const double* stats, const double* shift, int K, int D, clusters_t* c,
                         int num_threads, bool with_constants) {
    for (int k = 0; k < K; k++) finalize_cluster(stats, shift, k, D, c);
    if (with_constants) constants_from_R(K, D, c, num_threads);
}

long long seed_event_index(int c, int K, long long N) {
    float seed = (K > 1) ? ((float)N - 1.0f) / ((float)K - 1.0f) : 0.0f;   // gaussian.cu:110-115
    return (long long)(int)((float)c * seed);                              // :120
}

void seed_from_moments(const double* sum_x, const double* sum_x2, long long N, int D, int K,
                       const float* seed_rows, clusters_t* c) {
    double total = 0;                                   // averageVariance, gaussian_kernel.cu:71-102
    for (int d = 0; d < D; d++) {
        const double mean = sum_x[d] / (double)N;
        total += sum_x2[d] / (double)N - mean * mean;
    }
    const float avgvar = (float)(total / D);
    for (int k = 0; k < K; k++) {                       // seed_clusters kernel :304-327
        for (int d = 0; d < D; d++) c->means[k * D + d] = seed_rows[k * D + d];
        float* R = c->R + (size_t)k * D * D;
        for (int i = 0; i < D; i++)
            for (int j = 0; j < D; j++) R[i * D + j] = (i == j) ? 1.0f : 0.0f;
        c->pi[k] = 1.0f / (float)K;
        c->N[k] = (float)N / (float)K;
        c->avgvar[k] = (float)(avgvar / 1e3);           // COVARIANCE_DYNAMIC_RANGE
    }
    constants_from_R(K, D, c, 1);                       // gaussian.cu:404
    for (int k = 0; k < K; k++) c->N[k] = (float)(N / K);   // host seed_clusters: integer division, gaussian.cu:118
}

float rissanen(float loglik, int K, int D, double N) {           // gaussian.cu:826
    return (float)(-loglik + 0.5 * (K * (1 + D + 0.5 * (D + 1) * D) - 1) * logf((float)N * D));
}
float em_epsilon(int D, double N) {                              // gaussian.cu:458
    return (float)((1 + D + 0.5 * (D + 1) * D) * std::log((float)N * D) * 0.01);
}

// ---------------------------------------------------------------------------
// Order reduction (gaussian.cu:860-907).  Merge rule of add_clusters
// (gaussian.cu:1210-1252): weights N1/(N1+N2); merged mean; merged covariance
// = weighted (R_c + (mu - mu_c)(mu - mu_c)^T); pi and N add.  The merged
// constant uses log10(det) exactly as invert_cpu returns it
// (invert_matrix.cpp:61; quirk Q3) so that the merge SEQUENCE matches the
// reference.  Distance (cluster_distance :1203-1208):
//   N1*const1 + N2*const2 - N12*const12.
// ---------------------------------------------------------------------------
namespace {
struct Merged {
    float N, pi, constant;
    std::vector<float> means, R, Rinv;
};

void merge_pair(const clusters_t* c, int a, int b, int D, Merged& out) {
    out.means.resize(D); out.R.resize((size_t)D * D); out.Rinv.resize((size_t)D * D);
    const float wa = c->N[a] / (c->N[a] + c->N[b]);
    const float wb = 1.0f - wa;
    const float* ma = c->means + (size_t)a * D; const float* mb = c->means + (size_t)b * D;
    const float* Ra = c->R + (size_t)a * D * D; const float* Rb = c->R + (size_t)b * D * D;
    for (int i = 0; i < D; i++) out.means[i] = wa * ma[i] + wb * mb[i];
    for (int i = 0; i < D; i++)
        for (int j = i; j < D; j++) {
            float v = ((out.means[i] - ma[i]) * (out.means[j] - ma[j]) + Ra[i * D + j]) * wa;
            v += ((out.means[i] - mb[i]) * (out.means[j] - mb[j]) + Rb[i * D + j]) * wb;
            out.R[i * D + j] = v;
            out.R[j * D + i] = v;
        }
    out.pi = c->pi[a] + c->pi[b];
    out.N = c->N[a] + c->N[b];
    std::vector<float> work((size_t)D * D);
    out.Rinv = out.R;
    float lndet;
    lu_inverse_nopivot<float>(out.Rinv.data(), D, &lndet, work.data());
    const float log10det = (float)(lndet / std::log(10.0));
    out.constant = (float)((-D) * 0.5 * logf((float)(2 * kPi)) - 0.5 * log10det);
}

void move_cluster(clusters_t* c, int dst, int src, int D) {               // copy_cluster :1254-1264
    c->N[dst] = c->N[src]; c->pi[dst] = c->pi[src];
    c->constant[dst] = c->constant[src]; c->avgvar[dst] = c->avgvar[src];
    std::memmove(c->means + (size_t)dst * D, c->means + (size_t)src * D, sizeof(float) * D);
    std::memmove(c->R + (size_t)dst * D * D, c->R + (size_t)src * D * D, sizeof(float) * D * D);
    std::memmove(c->Rinv + (size_t)dst * D * D, c->Rinv + (size_t)src * D * D, sizeof(float) * D * D);
}
}  // namespace

int reduce_order(clusters_t* c, int K, int D, int* out_c1, int* out_c2, int num_threads, const ParallelFor* pfor) {
    (void)num_threads;
    for (int i = K - 1; i >= 0; i--)                                      // empties :866-874
        if (c->N[i] < 0.5f) {
            for (int j = i; j < K - 1; j++) move_cluster(c, j, j + 1, D);
            K--;
        }
    int best_a = 0, best_b = 1;
    if (K >= 2) {
        const int npairs = K * (K - 1) / 2;
        std::vector<float> dist(npairs);
        auto one_pair = [&](int p) {
            int a = 0, rem = p;                                           // p -> (a, b), a < b, row-major
            while (rem >= K - 1 - a) { rem -= K - 1 - a; a++; }
            const int b = a + 1 + rem;
            Merged m;
            merge_pair(c, a, b, D, m);
            dist[p] = c->N[a] * c->constant[a] + c->N[b] * c->constant[b] - m.N * m.constant;
        };
        if (pfor && *pfor && npairs >= 64) {                              // the caller's worker team, 16 pairs per task
            const int ntask = (npairs + 15) / 16;
            (*pfor)(ntask, [&](int t) { for (int p = t * 16; p < npairs && p < t * 16 + 16; p++) one_pair(p); });
        } else {
#pragma omp parallel for schedule(dynamic, 16) num_threads(num_threads) if (npairs >= 64 && num_threads > 1)
            for (int p = 0; p < npairs; p++) one_pair(p);
        }
        float best = 0.0f;
        int p = 0;
        for (int a = 0; a < K; a++)                                       // first strict minimum :882-894
            for (int b = a + 1; b < K; b++, p++)
                if ((a == 0 && b == 1) || dist[p] < best) { best = dist[p]; best_a = a; best_b = b; }
        Merged m;
        merge_pair(c, best_a, best_b, D, m);                              // :899-907
        c->N[best_a] = m.N; c->pi[best_a] = m.pi; c->constant[best_a] = m.constant;
        c->avgvar[best_a] = c->avgvar[0];
        std::memcpy(c->means + (size_t)best_a * D, m.means.data(), sizeof(float) * D);
        std::memcpy(c->R + (size_t)best_a * D * D, m.R.data(), sizeof(float) * D * D);
        std::memcpy(c->Rinv + (size_t)best_a * D * D, m.Rinv.data(), sizeof(float) * D * D);
        for (int i = best_b; i < K - 1; i++) move_cluster(c, i, i + 1, D);
    }
    if (out_c1) *out_c1 = best_a;
    if (out_c2) *out_c2 = best_b;
    return K - 1;                                                         // loop decrement, gaussian.cu:479
}

int epack_stride(int D) {
    const int coef_off = (D + 3) & ~3;
    return (coef_off + D * (D + 1) / 2 + 1 + 3) & ~3;
}

// E-step parameters of estep1 (gaussian_kernel.cu:412-423) pre-combined:
// the full D x D loop of :435-439 equals sum_i dx_i (Rinv_ii dx_i + sum_{j>i}
// (Rinv_ij + Rinv_ji) dx_j); constant + logf(pi) is the additive term of :442.
void build_epack(int K, int D, const clusters_t* c, float* out) {
    const int stride = epack_stride(D), coef_off = (D + 3) & ~3;
    std::memset(out, 0, sizeof(float) * (size_t)K * stride);
    for (int k = 0; k < K; k++) {
        float* p = out + (size_t)k * stride;
        const float* Ri = c->Rinv + (size_t)k * D * D;
        for (int d = 0; d < D; d++) p[d] = c->means[(size_t)k * D + d];
        int idx = coef_off;
        for (int i = 0; i < D; i++)
            for (int j = i; j < D; j++)
                p[idx++] = (i == j) ? Ri[i * D + i] : Ri[i * D + j] + Ri[j * D + i];
        p[idx] = c->constant[k] + logf(c->pi[k]);
    }
}

bool condition_cluster(const clusters_t* c, int k, int D, const int* obs, int n_obs, const int* mis, int nm, float* p_o,
                       float* constant_o, float* g, float* cvar, double* g_d, double* c_d) {
    constexpr int DM = GMM_MAX_DIMENSIONS;
    const float* P = c->Rinv + (size_t)k * D * D;
    auto S = [&](int i, int j) { return 0.5 * ((double)P[i * D + j] + (double)P[j * D + i]); };
    double L[DM][DM], Y[DM][DM], Z[DM][DM], Li[DM][DM];
    double ld = 0.0;
    for (int j = 0; j < nm; j++) {                          // S_MM = L L^T
        double s = S(mis[j], mis[j]);
        for (int t = 0; t < j; t++) s -= L[j][t] * L[j][t];
        if (!(s > 0.0) || !std::isfinite(s)) return false;
        L[j][j] = std::sqrt(s);
        ld += std::log(L[j][j]);
        for (int i = j + 1; i < nm; i++) {
            double v = S(mis[i], mis[j]);
            for (int t = 0; t < j; t++) v -= L[i][t] * L[j][t];
            L[i][j] = v / L[j][j];
        }
    }
    for (int o = 0; o < n_obs; o++) {
        for (int i = 0; i < nm; i++) {                      // Y = L^-1 S_MO
            double v = S(mis[i], obs[o]);
            for (int t = 0; t < i; t++) v -= L[i][t] * Y[t][o];
            Y[i][o] = v / L[i][i];
        }
        for (int i = nm - 1; i >= 0; i--) {                 // Z = L^-T Y = S_MM^-1 S_MO
            double v = Y[i][o];
            for (int t = i + 1; t < nm; t++) v -= L[t][i] * Z[t][o];
            Z[i][o] = v / L[i][i];
        }
    }
    for (int a = 0; a < n_obs; a++)                         // S_OO - S_OM S_MM^-1 S_MO = S_OO - Y^T Y
        for (int b = a; b < n_obs; b++) {
            double v = S(obs[a], obs[b]);
            for (int t = 0; t < nm; t++) v -= Y[t][a] * Y[t][b];
            p_o[a * n_obs + b] = p_o[b * n_obs + a] = (float)v;
        }
    for (int j = 0; j < nm; j++) {                          // L^-1, lower triangular; S_MM^-1 = L^-T L^-1
        Li[j][j] = 1.0 / L[j][j];
        for (int i = j + 1; i < nm; i++) {
            double v = 0.0;
            for (int t = j; t < i; t++) v -= L[i][t] * Li[t][j];
            Li[i][j] = v / L[i][i];
        }
    }
    for (int d = 0; d < nm; d++) {
        double v = 0.0;
        for (int i = d; i < nm; i++) v += Li[i][d] * Li[i][d];
        cvar[d] = (float)v;
        for (int o = 0; o < n_obs; o++) g[d * n_obs + o] = (float)(-Z[d][o]);
    }
    if (g_d)
        for (int d = 0; d < nm; d++)
            for (int o = 0; o < n_obs; o++) g_d[d * n_obs + o] = -Z[d][o];
    if (c_d)
        for (int d = 0; d < nm; d++)
            for (int e = 0; e <= d; e++) {
                double v = 0.0;
                for (int i = d; i < nm; i++) v += Li[i][d] * Li[i][e];
                c_d[d * nm + e] = c_d[e * nm + d] = v;
            }
    *constant_o = (float)((double)c->constant[k] + 0.5 * nm * std::log(2.0 * M_PI) - ld);
    return true;
}

void condition_stats_cluster(double* row, int D, const int* obs, int n_obs, const int* mis, int nm, const float* mu,
                             const double* shift, const double* g, const double* cm) {
    constexpr int DM = GMM_MAX_DIMENSIONS;
    double T1[DM], T2[DM][DM], b[DM], u[DM], GT2[DM][DM];
    const double T0 = row[0];
    for (int a = 0; a < n_obs; a++) {
        T1[a] = row[1 + obs[a]];
        for (int c = 0; c <= a; c++) T2[a][c] = T2[c][a] = row[feat2(D, obs[a], obs[c])];   // obs increasing: obs[a] >= obs[c]
    }
    for (int d = 0; d < nm; d++) {                          // b = (mu_M - s_M) - G (mu_O - s_O),  u = G T1,  G T2
        const double* gd = g + (size_t)d * n_obs;
        double v = (double)mu[mis[d]] - shift[mis[d]], w = 0.0;
        for (int a = 0; a < n_obs; a++) {
            v -= gd[a] * ((double)mu[obs[a]] - shift[obs[a]]);
            w += gd[a] * T1[a];
        }
        b[d] = v;
        u[d] = w;
        for (int a = 0; a < n_obs; a++) {
            double t = 0.0;
            for (int c = 0; c < n_obs; c++) t += gd[c] * T2[c][a];
            GT2[d][a] = t;
        }
    }
    for (int d = 0; d < nm; d++) {
        const int i = mis[d];
        row[1 + i] = b[d] * T0 + u[d];
        for (int a = 0; a < n_obs; a++) {                   // S2_MO = b T1^T + G T2
            const int j = obs[a];
            row[i > j ? feat2(D, i, j) : feat2(D, j, i)] = b[d] * T1[a] + GT2[d][a];
        }
        for (int e = 0; e <= d; e++) {                      // S2_MM = T0 (b b^T + C) + b u^T + u b^T + G T2 G^T
            const double* ge = g + (size_t)e * n_obs;
            double q = 0.0;
            for (int a = 0; a < n_obs; a++) q += GT2[d][a] * ge[a];
            row[feat2(D, i, mis[e])] = T0 * (b[d] * b[e] + cm[(size_t)d * nm + e]) + b[d] * u[e] + u[d] * b[e] + q;
        }
    }
}

// ---------------------------------------------------------------------------
// Variational Bayesian mixture (gmm_vb_em; sklearn's BayesianGaussianMixture with covariance_type='full', restated in
// float64 numpy by tests/_vb_ref.py).
// ---------------------------------------------------------------------------
double digamma(double x) {
    // psi(x) = psi(x + m) - sum_{j<m} 1/(x + j) until x + m >= 10, then the asymptotic series in 1/x^2 (Abramowitz and
    // Stegun 6.3.18) to the x^-14 term, whose truncation error at x >= 10 is about 2e-17 relative.
    if (!(x > 0.0)) return std::numeric_limits<double>::quiet_NaN();
    double acc = 0.0;
    while (x < 10.0) { acc -= 1.0 / x; x += 1.0; }
    const double r = 1.0 / x, r2 = r * r;
    const double series =
        r2 * (1.0 / 12 - r2 * (1.0 / 120 - r2 * (1.0 / 252 - r2 * (1.0 / 240 - r2 * (1.0 / 132 - r2 * (691.0 / 32760 - r2 / 12))))));
    return acc + std::log(x) - 0.5 * r - series;
}

int vb_resolve_prior(const gmm_vb_prior* p, int K, int D, VbPrior* out) {
    if (!p) return fail(GMM_ERR_ARG, "VB prior: NULL prior");
    if (p->weight_prior_type != GMM_VB_DIRICHLET_PROCESS && p->weight_prior_type != GMM_VB_DIRICHLET_DISTRIBUTION)
        return fail(GMM_ERR_ARG, "VB prior: unknown weight_prior_type");
    if (!std::isfinite(p->weight_concentration)) return fail(GMM_ERR_ARG, "VB prior: weight_concentration is not finite");
    if (!std::isfinite(p->mean_precision)) return fail(GMM_ERR_ARG, "VB prior: mean_precision is not finite");
    if (std::isnan(p->dof) || std::isinf(p->dof) || (p->dof > 0.0 && p->dof <= D - 1.0))
        return fail(GMM_ERR_ARG, "VB prior: dof must be > D - 1 (or <= 0 for the default D)");
    if (std::isnan(p->reg_covar) || std::isinf(p->reg_covar)) return fail(GMM_ERR_ARG, "VB prior: reg_covar is not finite");
    out->type = p->weight_prior_type;
    out->gamma0 = p->weight_concentration > 0.0 ? p->weight_concentration : 1.0 / K;
    out->beta0 = p->mean_precision > 0.0 ? p->mean_precision : 1.0;
    out->nu0 = p->dof > 0.0 ? p->dof : (double)D;
    out->reg = p->reg_covar >= 0.0 ? p->reg_covar : 1e-6;
    return GMM_OK;
}

// Cholesky A = L L^T of a symmetric [D][D] double matrix (lower triangle read); *half_ld = sum ln L_jj.  false = not
// positive definite.
static bool cholesky_half_ld(const double* A, int D, double* half_ld) {
    double L[GMM_MAX_DIMENSIONS][GMM_MAX_DIMENSIONS];
    double ld = 0.0;
    for (int j = 0; j < D; j++) {
        double s = A[j * D + j];
        for (int t = 0; t < j; t++) s -= L[j][t] * L[j][t];
        if (!(s > 0.0) || !std::isfinite(s)) return false;
        L[j][j] = std::sqrt(s);
        ld += std::log(L[j][j]);
        for (int i = j + 1; i < D; i++) {
            double v = A[i * D + j];
            for (int t = 0; t < j; t++) v -= L[i][t] * L[j][t];
            L[i][j] = v / L[j][j];
        }
    }
    *half_ld = ld;
    return true;
}

int vb_set_prior_moments(const double* mean, const double* cov, int D, VbPrior* out) {
    for (int d = 0; d < D; d++)
        if (!std::isfinite(mean[d])) return fail(GMM_ERR_ARG, "VB prior: mean is not finite");
    double amax = 0.0;
    for (int i = 0; i < D * D; i++) {
        if (!std::isfinite(cov[i])) return fail(GMM_ERR_ARG, "VB prior: covariance is not finite");
        amax = std::max(amax, std::fabs(cov[i]));
    }
    for (int i = 0; i < D; i++)
        for (int j = 0; j < i; j++)
            if (std::fabs(cov[i * D + j] - cov[j * D + i]) > 1e-12 * amax)
                return fail(GMM_ERR_ARG, "VB prior: covariance is not symmetric");
    double hl;
    if (!cholesky_half_ld(cov, D, &hl)) return fail(GMM_ERR_ARG, "VB prior: covariance is not positive definite");
    std::memcpy(out->m0, mean, sizeof(double) * D);
    std::memcpy(out->psi0, cov, sizeof(double) * D * D);
    return GMM_OK;
}

void vb_finalize_cluster(const double* stats, const double* shift, int k, int D, const VbPrior& p, clusters_t* c, VbCluster* out) {
    const int F = num_features(D);
    const double* s = stats + (size_t)k * F;
    const double S0 = s[0];
    const double nk = S0 + 10.0 * std::numeric_limits<double>::epsilon();      // sklearn: resp.sum(0) + 10 eps
    double xk[GMM_MAX_DIMENSIONS], dd[GMM_MAX_DIMENSIONS], m[GMM_MAX_DIMENSIONS], df[GMM_MAX_DIMENSIONS];
    for (int d = 0; d < D; d++) {
        xk[d] = (S0 * shift[d] + s[1 + d]) / nk;                                 // an empty component gets xk = 0
        dd[d] = xk[d] - shift[d];
    }
    const double beta = p.beta0 + nk, nu = p.nu0 + nk, wmix = nk * p.beta0 / beta;
    for (int d = 0; d < D; d++) {
        m[d] = (p.beta0 * p.m0[d] + nk * xk[d]) / beta;
        df[d] = xk[d] - p.m0[d];
    }
    double C[GMM_MAX_DIMENSIONS * GMM_MAX_DIMENSIONS];
    for (int i = 0; i < D; i++)
        for (int j = 0; j <= i; j++) {
            // nk sk = sum g (x - xk)(x - xk)^T + nk reg I, with sum g (x - xk)(x - xk)^T = S2 - S1 dd^T - dd S1^T + S0 dd dd^T
            double q = s[feat2(D, i, j)] - s[1 + i] * dd[j] - dd[i] * s[1 + j] + S0 * dd[i] * dd[j];
            if (i == j) q += nk * p.reg;
            const double v = (p.psi0[i * D + j] + q + wmix * df[i] * df[j]) / nu;
            C[i * D + j] = C[j * D + i] = v;
        }
    c->N[k] = (float)nk;
    float* mu = c->means + (size_t)k * D;
    float* R = c->R + (size_t)k * D * D;
    for (int d = 0; d < D; d++) mu[d] = (float)m[d];
    for (int i = 0; i < D * D; i++) R[i] = (float)C[i];
    out->nk = nk; out->beta = beta; out->nu = nu;
    double W[GMM_MAX_DIMENSIONS * GMM_MAX_DIMENSIONS], hl_f = 0.0, hl_d = 0.0;
    out->ok = constants_cluster_spd(k, D, c, W, &hl_f) && cholesky_half_ld(C, D, &hl_d);
    if (!out->ok) { out->offset = out->log_wishart = 0.0; return; }
    double sum_psi = 0.0, sum_lg = 0.0;
    for (int i = 0; i < D; i++) {
        sum_psi += digamma(0.5 * (nu - i));
        sum_lg += std::lgamma(0.5 * (nu - i));
    }
    out->offset = -0.5 * D * std::log(2.0 * kPi) - hl_f - 0.5 * D * std::log(nu) + 0.5 * (D * std::log(2.0) + sum_psi) - 0.5 * D / beta;
    const double ldpc = -hl_d - 0.5 * D * std::log(nu);                         // ln det of sklearn's precisions_cholesky_
    out->log_wishart = -(nu * ldpc + nu * D * 0.5 * std::log(2.0) + sum_lg);
}

int vb_finalize_weights(int K, int D, const VbPrior& p, const VbCluster* cl, clusters_t* c, gmm_vb_posterior* post, double* bound,
                        int* bad_k) {
    for (int k = 0; k < K; k++)
        if (!cl[k].ok) { if (bad_k) *bad_k = k; return -1; }
    std::vector<double> a(K), b(K), elog(K), w(K);
    double log_norm_weight = 0.0, wsum = 0.0;
    if (p.type == GMM_VB_DIRICHLET_PROCESS) {
        double tail = 0.0;                                  // sum_{j > k} nk_j, accumulated from the last component down
        for (int k = K - 1; k >= 0; k--) {
            a[k] = 1.0 + cl[k].nk;
            b[k] = p.gamma0 + tail;
            tail += cl[k].nk;
        }
        double run = 0.0, prod = 1.0;
        for (int k = 0; k < K; k++) {
            const double ds = digamma(a[k] + b[k]);
            elog[k] = digamma(a[k]) - ds + run;
            run += digamma(b[k]) - ds;
            w[k] = a[k] / (a[k] + b[k]) * prod;
            prod *= b[k] / (a[k] + b[k]);
            log_norm_weight -= std::lgamma(a[k]) + std::lgamma(b[k]) - std::lgamma(a[k] + b[k]);   // -sum betaln(a, b)
        }
    } else {
        double sa = 0.0, slg = 0.0;
        for (int k = 0; k < K; k++) {
            a[k] = p.gamma0 + cl[k].nk;
            sa += a[k];
            slg += std::lgamma(a[k]);
        }
        const double ds = digamma(sa);
        for (int k = 0; k < K; k++) {
            elog[k] = digamma(a[k]) - ds;
            w[k] = a[k];
        }
        log_norm_weight = std::lgamma(sa) - slg;
    }
    for (int k = 0; k < K; k++) wsum += w[k];
    double log_wishart = 0.0, sum_lb = 0.0;
    for (int k = 0; k < K; k++) {
        w[k] /= wsum;
        const float pf = std::max((float)w[k], std::numeric_limits<float>::min());
        c->pi[k] = pf;
        // constant + ln pi = offset + E[ln pi]: ln pi in double of the float pi (the tensor E-step packs constant + ln pi
        // with ln pi in double, the SIMT E-step with logf; both round to float)
        c->constant[k] = (float)(cl[k].offset + elog[k] - std::log((double)pf));
        log_wishart += cl[k].log_wishart;
        sum_lb += std::log(cl[k].beta);
    }
    if (bound) *bound = -log_wishart - log_norm_weight - 0.5 * D * sum_lb;
    if (post) {
        for (int k = 0; k < K; k++) {
            if (post->weights) post->weights[k] = w[k];
            if (post->weight_concentration) {
                post->weight_concentration[k] = a[k];
                if (p.type == GMM_VB_DIRICHLET_PROCESS) post->weight_concentration[K + k] = b[k];
            }
            if (post->mean_precision) post->mean_precision[k] = cl[k].beta;
            if (post->dof) post->dof[k] = cl[k].nu;
        }
        if (post->mean_prior) std::memcpy(post->mean_prior, p.m0, sizeof(double) * D);
        if (post->covariance_prior) std::memcpy(post->covariance_prior, p.psi0, sizeof(double) * D * D);
    }
    return 0;
}

}  // namespace gmm

// ---------------------------------------------------------------------------
// extern "C" wrappers (include/gmm.h, "host-only numerics")
// ---------------------------------------------------------------------------
namespace gmm { const char* last_error_cstr(); }

extern "C" {

const char* gmm_last_error(void) { return gmm::last_error_cstr(); }

int gmm_host_invert(float* data, int n, float* log_det, int use_log10) {
    if (!data || !log_det || n < 1 || n > GMM_MAX_DIMENSIONS) return gmm::fail(GMM_ERR_ARG, "gmm_host_invert: bad argument");
    std::vector<float> work((size_t)n * n);
    float ln;
    gmm::lu_inverse_nopivot<float>(data, n, &ln, work.data());
    *log_det = use_log10 ? (float)(ln / std::log(10.0)) : ln;
    return GMM_OK;
}

long long gmm_stats_len(int K, int D) { return (long long)K * gmm::num_features(D) + 1; }

int gmm_host_finalize(const double* stats, const double* shift, int K, int D, clusters_t* inout) {
    if (!stats || !shift || !inout || K < 1 || K > GMM_MAX_CLUSTERS || D < 1 || D > GMM_MAX_DIMENSIONS)
        return gmm::fail(GMM_ERR_ARG, "gmm_host_finalize: bad argument");
    gmm::finalize_from_stats(stats, shift, K, D, inout, 1);
    return GMM_OK;
}

int gmm_host_vb_finalize(const double* stats, const double* shift, int K, int D, const gmm_vb_prior* prior,
                         clusters_t* out, gmm_vb_posterior* post_out, double* bound_out) {
    if (!stats || !shift || !out || K < 1 || K > GMM_MAX_CLUSTERS || D < 1 || D > GMM_MAX_DIMENSIONS)
        return gmm::fail(GMM_ERR_ARG, "gmm_host_vb_finalize: bad argument");
    gmm::VbPrior p;
    if (int rc = gmm::vb_resolve_prior(prior, K, D, &p)) return rc;
    if (!prior->mean || !prior->covariance) return gmm::fail(GMM_ERR_ARG, "gmm_host_vb_finalize: the prior's mean and covariance are required");
    if (int rc = gmm::vb_set_prior_moments(prior->mean, prior->covariance, D, &p)) return rc;
    std::vector<gmm::VbCluster> cl((size_t)K);
    for (int k = 0; k < K; k++) gmm::vb_finalize_cluster(stats, shift, k, D, p, out, &cl[(size_t)k]);
    int bad = -1;
    if (gmm::vb_finalize_weights(K, D, p, cl.data(), out, post_out, bound_out, &bad))
        return gmm::fail(GMM_ERR_STATE, "gmm_host_vb_finalize: the covariance of component " + std::to_string(bad) + " is not positive definite");
    return GMM_OK;
}

int gmm_host_digamma(const double* x, double* out, long long n) {
    if ((!x || !out) && n > 0) return gmm::fail(GMM_ERR_ARG, "gmm_host_digamma: bad argument");
    for (long long i = 0; i < n; i++) out[i] = gmm::digamma(x[i]);
    return GMM_OK;
}

int gmm_host_combine_groups(const int* merges, int K, int L, int* group_out) {
    if (K < 1 || K > GMM_MAX_CLUSTERS || L < 1 || L > K || !group_out || (K >= 2 && !merges))
        return gmm::fail(GMM_ERR_ARG, "gmm_host_combine_groups: bad argument (need 1 <= L <= K <= 512, merges and group_out)");
    // rep[k] = the component k was merged into (itself while its group is live); a merge joins two live groups a < b
    std::vector<int> rep((size_t)K);
    for (int k = 0; k < K; k++) rep[(size_t)k] = k;
    for (int s = 0; s < K - 1; s++) {
        const int a = merges[2 * s], b = merges[2 * s + 1];
        if (a < 0 || b >= K || a >= b || rep[(size_t)a] != a || rep[(size_t)b] != b)
            return gmm::fail(GMM_ERR_ARG, "gmm_host_combine_groups: merge " + std::to_string(s) + " is not a pair a < b of live groups");
        if (s < K - L) rep[(size_t)b] = a;
    }
    // a group's smallest component is its root, met first in increasing k: clusters numbered in that order
    std::vector<int> label((size_t)K, -1);
    int next = 0;
    for (int k = 0; k < K; k++) {
        int r = k;
        while (rep[(size_t)r] != r) r = rep[(size_t)r];
        if (label[(size_t)r] < 0) label[(size_t)r] = next++;
        group_out[k] = label[(size_t)r];
    }
    return GMM_OK;
}

// Residual sum of squares of the least-squares line through points [b, e) (the mean when their x are all equal):
// centred sums, in index order.
static double elbow_sse(const double* x, const double* y, int b, int e) {
    const int m = e - b;
    double sx = 0.0, sy = 0.0;
    for (int i = b; i < e; i++) { sx += x[i]; sy += y[i]; }
    const double mx = sx / m, my = sy / m;
    double sxx = 0.0, sxy = 0.0;
    for (int i = b; i < e; i++) { sxx += (x[i] - mx) * (x[i] - mx); sxy += (x[i] - mx) * (y[i] - my); }
    const double beta = sxx > 0.0 ? sxy / sxx : 0.0;
    double sse = 0.0;
    for (int i = b; i < e; i++) {
        const double r = (y[i] - my) - beta * (x[i] - mx);
        sse += r * r;
    }
    return sse;
}

int gmm_host_combine_elbow(const double* entropy, const double* x, int K, int* L_out) {
    if (!entropy || !L_out || K < 3) return gmm::fail(GMM_ERR_ARG, "gmm_host_combine_elbow: bad argument (need entropy, L_out and K >= 3)");
    std::vector<double> xs((size_t)K);
    for (int i = 0; i < K; i++) {
        xs[(size_t)i] = x ? x[i] : (double)(i + 1);
        if (!std::isfinite(xs[(size_t)i]) || !std::isfinite(entropy[i]))
            return gmm::fail(GMM_ERR_ARG, "gmm_host_combine_elbow: a value that is not finite");
    }
    // point L = i + 1 is index i; change point c joins the segments [0, c) and [c - 1, K)
    int best = 2;
    double best_sse = 0.0;
    for (int c = 2; c <= K - 1; c++) {
        const double sse = elbow_sse(xs.data(), entropy, 0, c) + elbow_sse(xs.data(), entropy, c - 1, K);
        if (c == 2 || sse < best_sse) { best = c; best_sse = sse; }
    }
    *L_out = best;
    return GMM_OK;
}

float gmm_host_rissanen(float loglik, int K, int D, long long N) { return gmm::rissanen(loglik, K, D, (double)N); }
float gmm_host_epsilon(int D, long long N) { return gmm::em_epsilon(D, (double)N); }

int gmm_host_reduce_order(clusters_t* clusters, int* K, int D, int* c1, int* c2) {
    if (!clusters || !K || *K < 1 || D < 1 || D > GMM_MAX_DIMENSIONS) return gmm::fail(GMM_ERR_ARG, "gmm_host_reduce_order: bad argument");
    *K = gmm::reduce_order(clusters, *K, D, c1, c2, 1);
    return GMM_OK;
}

void gmm_shard_range(long long n_global, int nranks, int rank, long long* begin, long long* count) {
    const long long per = n_global / nranks;                  // gaussian.cu:348-352 (Q6 fixed)
    if (begin) *begin = per * rank;
    if (count) *count = (rank == nranks - 1) ? per + n_global % nranks : per;
}

}  // extern "C"
