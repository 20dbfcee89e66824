// host_math.h — GPU-free host numerics of the engine (internal C++ API).
// The extern "C" wrappers of include/gmm.h live in host_math.cpp.
#pragma once
#include <cstddef>
#include <functional>
#include <string>
#include <vector>
#include "../../include/gmm.h"

namespace gmm {

void set_error(const std::string& msg);          // thread-local, read by gmm_last_error()
int  fail(int code, const std::string& msg);     // set_error + return code

// Number of per-cluster sufficient statistics: 1 + D + D(D+1)/2.
inline int num_features(int D) { return 1 + D + D * (D + 1) / 2; }
// Index of the second-moment feature (i >= j) inside a cluster's feature row.
inline int feat2(int D, int i, int j) { return 1 + D + i * (i + 1) / 2 + j; }

// In-place inverse by LU factorisation WITHOUT pivoting (the semantics of
// invert_cpu, invert_matrix.cpp:25-101, and of the device `invert`,
// gaussian_kernel.cu:107-169).  Returns sum log|u_ii| in *logabsdet (natural
// log).  T = float or double.
template <class T> void lu_inverse_nopivot(T* a, int n, T* logabsdet, T* work /* n*n */);

// Host finalisation of one M-step from reduced statistics (see gmm.h).
void finalize_from_stats(const double* stats, const double* shift, int K, int D, clusters_t* c,
                         int num_threads, bool with_constants = true);

// constants_kernel semantics on host arrays: Rinv, constant (ln det), pi.
void constants_from_R(int K, int D, clusters_t* c, int num_threads);
// The two parts of constants_from_R, for callers that run their own loop over the clusters:
// inverse + constant of one cluster, and the mixing weights pi (needs every N[k]).
void constants_cluster(int k, int D, clusters_t* c);
// Same results for a symmetric positive definite R from one (reverse) Cholesky factorisation; also returns the
// upper-triangular W with Rinv = W^T W.  false = not positive definite, nothing written (use constants_cluster).
bool constants_cluster_spd(int k, int D, clusters_t* c, double* W, double* half_ln_det = nullptr);
// The factorisation behind it: R = U U^T with U upper triangular, in double from the float R [D][D] (row-major, the
// off-diagonal pairs averaged), pivots from the last one up; *ld = sum ln U_jj.  Only U's upper triangle is written.
// false = not positive definite (a pivot <= 0 or not finite).
bool reverse_cholesky(const float* R, int D, double (*U)[GMM_MAX_DIMENSIONS], double* ld);
// N, mean and covariance of ONE cluster from the packed statistics (the loop body of finalize_from_stats).
void finalize_cluster(const double* stats, const double* shift, int k, int D, clusters_t* c);
void mixing_weights(int K, clusters_t* c);

// Seeding from global column sums (double): sum x, sum x^2 over all N events,
// and the K seed rows (already gathered).  gaussian_kernel.cu:269-328,
// gaussian.cu:108-123.
void seed_from_moments(const double* sum_x, const double* sum_x2, long long N, int D, int K,
                       const float* seed_rows /* [K][D] */, clusters_t* c);
// Row index of seed event c (gaussian.cu:110-120: (int)(c*seed), seed in float).
long long seed_event_index(int c, int K, long long N);

// N: the number of events, or the sum of the weights (gmm_set_weights); (float)N as the reference forms it.
float rissanen(float loglik, int K, int D, double N);
float em_epsilon(int D, double N);

// One order-reduction step (gaussian.cu:860-907).  Returns new K.  The K(K-1)/2 trial merges run on the caller's
// worker team when `pfor` is given (pfor(n, fn) calls fn(0..n-1) in parallel), else on an OpenMP team of num_threads.
using ParallelFor = std::function<void(int, const std::function<void(int)>&)>;
int reduce_order(clusters_t* c, int K, int D, int* c1, int* c2, int num_threads, const ParallelFor* pfor = nullptr);

// Packed E-step parameters for the SIMT kernel: per cluster
//   [ mean(D) | c_ii, 2c_ij (j>i) row by row (D(D+1)/2) | constant + ln(pi) ] padded to stride.
int  epack_stride(int D);
void build_epack(int K, int D, const clusters_t* c, float* out);

// gmm_condition's parameters of cluster k (gmm.h): in double from the float Rinv of c, S = (Rinv + Rinv^T) / 2, split
// into the observed dimensions obs[n_obs] and the missing ones mis[nm] (nm >= 1), rounded to float:
//   p_o [n_obs][n_obs] = S_OO - S_OM S_MM^-1 S_MO    (marginal precision, symmetric)
//   *constant_o        = constant + nm/2 ln 2 pi - 1/2 ln det S_MM
//   g [nm][n_obs]      = -S_MM^-1 S_MO               (regression of the missing dimensions on dx_O)
//   cvar [nm]          = diag(S_MM^-1)                (conditional variances)
//   g_d [nm][n_obs], c_d [nm][nm]: when not NULL, G and the full S_MM^-1 in double (gmm_condition_stats' expansion)
// S_MM is factorised once (Cholesky).  false = S_MM is not positive definite (a pivot <= 0 or not finite); nothing written.
bool condition_cluster(const clusters_t* c, int k, int D, const int* obs, int n_obs, const int* mis, int nm, float* p_o,
                       float* constant_o, float* g, float* cvar, double* g_d = nullptr, double* c_d = nullptr);
// gmm_condition_stats' expansion of one cluster's packed row (F doubles, about `shift`) in place, in double: on entry the
// entries of the observed dimensions hold T0 = sum r, T1 = sum r y, T2 = sum r y y^T (y = x_O - s_O, r the marginal
// posterior); the entries that involve a missing dimension are overwritten with their expectations given x_O,
//   S1_M = b T0 + G T1,  S2_MO = b T1^T + G T2,  S2_MM = T0 (b b^T + C) + b u^T + u b^T + G T2 G^T,  u = G T1,
// with b = (mu_M - s_M) - G (mu_O - s_O).  mu: the cluster's float means [D]; g [nm][n_obs] = G and cm [nm][nm] = C = S_MM^-1
// as condition_cluster returns them in double.
void condition_stats_cluster(double* row, int D, const int* obs, int n_obs, const int* mis, int nm, const float* mu,
                             const double* shift, const double* g, const double* cm);

// ---- variational Bayesian mixture (gmm_vb_em, gmm_host_vb_finalize; gmm.h) ----
double digamma(double x);
// The prior with its defaults applied (m0 / Psi0 by the caller: the events' moments when the user passes NULL).
struct VbPrior {
    int type;                                   // GMM_VB_*
    double gamma0, beta0, nu0, reg;
    double m0[GMM_MAX_DIMENSIONS];
    double psi0[GMM_MAX_DIMENSIONS * GMM_MAX_DIMENSIONS];
};
// Checks the scalars of `p` and applies their defaults (m0 / Psi0 are copied by vb_set_prior_moments).  GMM_OK or
// GMM_ERR_ARG with the message set.
int vb_resolve_prior(const gmm_vb_prior* p, int K, int D, VbPrior* out);
// m0 and Psi0 (row-major [D][D]): finite, Psi0 symmetric and positive definite; GMM_OK or GMM_ERR_ARG.
int vb_set_prior_moments(const double* mean, const double* cov, int D, VbPrior* out);
// What the per-cluster part of the VB M-step leaves for the serial part.
struct VbCluster {
    double nk, beta, nu;
    double offset;          // -D/2 ln 2 pi - 1/2 ln det R(float) - D/2 ln nu + 1/2 (D ln 2 + sum psi) - D / (2 beta)
    double log_wishart;     // sklearn's _log_wishart_norm of the cluster (ln det C of the double C)
    bool ok;                // the float R (and the double C) are positive definite
};
// The per-cluster part of the VB M-step of cluster k from the packed statistics about `shift`: N, means, R, Rinv of c
// (Rinv from the reverse Cholesky factorisation of the float R, as the host finalisation forms it) and `out`.
void vb_finalize_cluster(const double* stats, const double* shift, int k, int D, const VbPrior& p, clusters_t* c, VbCluster* out);
// The serial part: weight posterior, E[ln pi], weights_, pi (float, floored at FLT_MIN), constant, and the parameter part of
// the bound.  post (may be NULL) and its arrays receive the posterior.  Returns -1 if a cluster is not positive definite
// (its index in *bad_k), else 0.
int vb_finalize_weights(int K, int D, const VbPrior& p, const VbCluster* cl, clusters_t* c, gmm_vb_posterior* post, double* bound,
                        int* bad_k);

}  // namespace gmm
