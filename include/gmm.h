/*
 * gmm.h — C ABI of the H100-native GMM-EM engine (libgmm_b200.so).
 *
 * This is the drop-in boundary for the hot path of Corv/CUDA-GMM-MPI.  The
 * reference has no plugin/FFI layer: its seven kernels are #included into the
 * host translation unit (gaussian.cu:16) and launched inline from main().  The
 * boundary a maintainer can bind is therefore (1) the clusters_t / events
 * memory layout, (2) the operator granularity of the kernels, (3) the CLI.
 * Every entry point below names the reference code it replaces (file:line in
 * the reference repository).
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no torch / CUDA types.
 *   - All pointers are HOST pointers owned by the caller unless stated.
 *   - Return 0 on success, a GMM_ERR_* code otherwise; gmm_last_error()
 *     returns a thread-local message.
 *   - One gmm_ctx owns ONE GPU and one contiguous shard of events
 *     (reference: one OpenMP thread per GPU, gaussian.cu:289-377).  A ctx is
 *     not re-entrant; different ctxs may be driven from different threads or
 *     processes.  Multi-GPU = one ctx per GPU joined by gmm_comm_init().
 *   - There is NO CPU fallback: every compute entry point fails with
 *     GMM_ERR_CUDA when no sm_90 device is usable.
 */
#ifndef GMM_B200_H
#define GMM_B200_H

#ifdef __cplusplus
extern "C" {
#endif

/* ---- data layout: verbatim from gaussian.h:62-76 -------------------------
 * K = number of clusters, D = dimensions, N = events.
 *   N[K] pi[K] constant[K] avgvar[K] means[K*D] R[K*D*D] Rinv[K*D*D]
 *   memberships[K*N], CLUSTER-major: memberships[c*N + n].
 * Events are row-major AoS float32 [N][D] (gaussian.cu:188-192).            */
typedef struct {
    float* N;           /* expected # of events in cluster: [K]            */
    float* pi;          /* mixing probability: [K]                         */
    float* constant;    /* -D/2 ln(2 pi) - 1/2 ln det R: [K]               */
    float* avgvar;      /* diagonal regulariser (avg variance / 1e3): [K]  */
    float* means;       /* [K*D]                                           */
    float* R;           /* covariance, row-major DxD per cluster: [K*D*D]  */
    float* Rinv;        /* inverse covariance: [K*D*D]                     */
    float* memberships; /* responsibilities, cluster-major: [K*N]          */
} clusters_t;

typedef struct gmm_ctx gmm_ctx;

enum {
    GMM_OK = 0,
    GMM_ERR_ARG = 1,      /* bad argument (validateArguments returns 1/2/4, gaussian.cu:1111-1166) */
    GMM_ERR_IO = 2,
    GMM_ERR_NOMEM = 3,
    GMM_ERR_CUDA = 4,     /* no device / CUDA error — never falls back to the CPU */
    GMM_ERR_NCCL = 5,
    GMM_ERR_STATE = 6
};

/* Limits of the reference (gaussian.h:10,16). */
#define GMM_MAX_CLUSTERS   512
#define GMM_MAX_DIMENSIONS 32

/* E/M-step implementation selector (gmm_set_option "path").               */
#define GMM_PATH_AUTO   0   /* tensor-core path when the shape allows it    */
#define GMM_PATH_SIMT   1   /* FP32/FP64 CUDA-core kernels                  */
#define GMM_PATH_TENSOR 2   /* wgmma kernels (fails if shape unsupported) */

const char* gmm_last_error(void);
const char* gmm_version(void);

/* ---- context ------------------------------------------------------------
 * Replaces the per-thread device setup of gaussian.cu:298-377: cudaSetDevice,
 * cudaMalloc of the clusters_t arrays and of the event shard, H2D copy of the
 * shard.  `events_aos` holds THIS shard only ([n_local][D]); `n_global` and
 * `offset` place it in the whole data set (reference sharding rule:
 * events_per_gpu = N / G, remainder to the last GPU, gaussian.cu:348-352 —
 * see gmm_shard_range).                                                     */
int  gmm_create(gmm_ctx** out, int device, int n_local, int D, int Kmax,
                const float* events_aos, long long n_global, long long offset);
void gmm_destroy(gmm_ctx*);

/* Replace the events of this shard in an existing context (same n_local and D): the H2D copy
 * of gaussian.cu:370 without re-creating buffers or the communicator.                        */
int  gmm_upload_events(gmm_ctx*, const float* events_aos);

/* The same from a "*.bin" file (readData.cpp:35-47: int32 N, int32 D, float32[N][D]): the rows
 * [offset, offset + n_local) of the file go to the device through two pinned staging buffers,
 * reads and H2D copies overlapped; the host never holds the data set (replaces readData +
 * the host transpose + the per-GPU pageable copy, gaussian.cu:188-218, 360-377).  The header must
 * match the context (N == n_global, D).  A context may be created with events_aos == NULL and
 * filled this way.                                                                             */
int  gmm_upload_events_file(gmm_ctx*, const char* path);
int  gmm_read_bin_header(const char* path, int* ndims, int* nevents);

/* Contiguous event range of shard `rank` of `nranks` (gaussian.cu:348-352,
 * with quirk Q6 fixed: the remainder goes to the LAST shard).              */
void gmm_shard_range(long long n_global, int nranks, int rank,
                     long long* begin, long long* count);

/* ---- multi-GPU: replaces MPI_Allreduce/MPI_Bcast + OpenMP-master sums
 * (gaussian.cu:516,566,605,658,741; 555-559,594-600,647-653).  One
 * ncclAllReduce of the packed sufficient statistics per EM iteration.      */
int  gmm_nccl_unique_id(char id_out[128]);
int  gmm_comm_init(gmm_ctx*, int nranks, int rank, const char id[128]);
int  gmm_comm_rank(const gmm_ctx*, int* rank, int* nranks);

/* ---- options: the reference's compile-time #defines made runtime
 * (gaussian.h:23-38).  Known keys: "path" (GMM_PATH_*: both steps),
 * "estep_path" / "mstep_path" (GMM_PATH_* for one step only, -1 = follow
 * "path"), "verbose", "host_threads" (threads of the host-side
 * finalisation), "profile" (0 = no per-phase CUDA-event timers inside the EM
 * loop; gmm_get_profile then reports zeros for the device phases),
 * "allreduce" (1, default = the per-iteration sum of the packed statistics runs
 * as this library's own kernel over NVLink peer memory when every rank could map
 * every other rank's exchange area — one box, <= 8 GPUs; 0 = ncclAllReduce),
 * "finalize" (1, default = when the tensor E-step serves the parameters, the
 * whole step between the reduced statistics and the next E-step — N, means, R,
 * inverse, constants, pi and the E-step operand — runs as ONE kernel on the
 * device and gmm_em_iterations / the first min_iters iterations of gmm_em queue
 * their iterations back to back without returning to the host; a cluster that
 * needs the host's no-pivot LU semantics (R not positive definite) or leaves the
 * FP16 operand range makes the library replay from the last good parameters
 * through the host path and stay on it; 0 = host finalisation every iteration,
 * invert_matrix.cpp semantics; env GMM_FINALIZE=host|device sets the default),
 * "finalize_fault_iter" (tests: that iteration of the next batch reports a
 * failure although nothing is wrong, -1 = never), "score_chunk" (events per
 * chunk that gmm_score streams through its pinned and device buffers;
 * default 1048576, at most 2^28).  Options have to be set
 * identically on every rank of a communicator.  Unknown keys are an
 * error (GMM_ERR_ARG).  Every E-step materialises the memberships on the
 * device (the reference's behaviour); they reach the host only through
 * gmm_get_clusters / gmm_fit.                                              */
int  gmm_set_option(gmm_ctx*, const char* key, double value);

/* ---- operators (one per reference kernel group) ------------------------- */

/* seed_clusters kernel + host seed_clusters + first constants_kernel
 * (gaussian_kernel.cu:269-328, gaussian.cu:108-123, 390-452).  Fills
 * host_out (all arrays except memberships) and uploads it.                 */
int  gmm_seed(gmm_ctx*, int K, clusters_t* host_out);

/* k-means++ (greedy) seeding + at most max_iter Lloyd iterations on the context's events,
 * then ONE M-step on the one-hot memberships of the final assignment: the mixture
 * sklearn's init_params='kmeans' starts EM from.  Collective (all ranks, same arguments).
 * Leaves the context as gmm_seed does: current parameters for K = the returned ones,
 * no valid memberships; gmm_em / gmm_estep / gmm_score may follow.
 *   host_out     all clusters_t arrays except memberships (may be NULL)
 *   centres_out  [K][D] the centres of the final assignment (may be NULL)
 *   iters_out    Lloyd centre updates performed (may be NULL)
 *   inertia_out  sum over all events of the squared distance to the assigned centre (may be NULL)
 * Semantics (reproducible bit for bit in float64 numpy):
 *   - draws: splitmix64 from `seed`, u = (next() >> 11) * 2^-53, on the host, the same on
 *     every rank.  First centre: global event min(floor(u n_global), n_global - 1).
 *   - d(x, c) = sum_d (double(x_d) - double(c_d))^2 in dimension order, no FMA; d2[i] = min
 *     over the chosen centres.  Block sums of d2 add blocks of 1024 consecutive events of a
 *     shard in index order; T and the running prefix add the block sums in block order and
 *     the shards in rank order.
 *   - each further centre: L = 2 + floor(ln K) draws, targets u_l T; candidate l = the first
 *     event whose inclusive prefix of d2 exceeds u_l T (rounding leaving none: the last event
 *     with d2 > 0); the candidate of smallest potential sum min(d2, d(x, c_l)) wins, lowest l
 *     on ties.  T = 0 (fewer distinct events than K): the remaining centres repeat the first.
 *   - Lloyd: nearest centre in FP32 (sum of (x - c)^2, ties to the lowest k); the centre
 *     update is shift + S1/S0 of the context's own M-step (wgmma or FP64 SIMT, as gmm_mstep
 *     chooses; counted in gmm_get_profile's launch counters); S0 = 0 keeps the centre.  Stops
 *     after max_iter updates or when an assignment changes no label.  max_iter = 0: the
 *     k-means++ centres, one assignment, one M-step (sklearn's 'k-means++' init).
 *   - result: N, pi, means, R, Rinv, constant from the last M-step's statistics with avgvar
 *     from the global variance as gmm_seed sets it (clusters without events: the N < 0.5
 *     rules), uploaded as gmm_set_clusters uploads them.  Overwrites the device memberships.
 * Device memory: 12 bytes per event (allocated on the first call, freed by gmm_destroy).
 * Errors: K outside [1, Kmax], K > n_global or max_iter < 0 -> GMM_ERR_ARG; a failed
 * collective -> GMM_ERR_NCCL.  The k-means++ centres are deterministic for a seed; so is the
 * rest where the wgmma M-step runs (the FP64 SIMT M-step adds with atomics in varying order). */
int  gmm_seed_kmeans(gmm_ctx*, int K, int max_iter, unsigned long long seed,
                     clusters_t* host_out, float* centres_out, int* iters_out, double* inertia_out);

/* H2D of N,pi,constant,avgvar,means,R,Rinv (gaussian.cu:446-452, 935-941). */
int  gmm_set_clusters(gmm_ctx*, int K, const clusters_t* host_in);

/* Per-event weights of THIS shard ([n_local] floats, finite, >= 0), used by every later E-step log-likelihood and
 * M-step statistic of the context's own shard.  NULL clears them (back to unit weights).  Collective with several
 * ranks.  *total_out (may be NULL) = the global sum of the weights (n_global after NULL).
 * Semantics: EM over the multiset in which event n appears w_n times, extended to real w >= 0 (integer weights give
 * the EM of replicated rows):
 *   - gmm_estep's log-likelihood is sum w logp; the M-step statistics of gmm_mstep, gmm_em, gmm_em_iterations (host
 *     and device-side finalisation) and gmm_fit are S0 = sum w g, S1 = sum w g (x - s), S2 = sum w g (x - s)(x - s)^T;
 *     everything after them (the all-reduce, N, pi = N / sum N, the N thresholds, the order reduction) is unchanged.
 *   - gmm_em's default epsilon and gmm_fit's Rissanen score use N = sum w in place of n_global (the public
 *     gmm_host_epsilon / gmm_host_rissanen do not change).
 *   - ignored: gmm_seed and gmm_seed_kmeans (initialisation only), the memberships (posteriors do not depend on the
 *     weights), and gmm_score, gmm_score_stats, gmm_sample, gmm_condition, gmm_condition_stats (they do not read the shard;
 *     their kernels, outputs and profiles are the same with and without weights set).
 *   - kernels: weighted instances of the context's own E- and M-step kernels.  The wgmma M-step divides the weights by
 *     the largest one; it serves weights whose positive values are all equal (dynamic range
 *     max w / min positive w = 1: a constant factor, zeros allowed), the range its fixed-point operand holds to the
 *     per-cluster accuracy bar (DESIGN.md §5.11).  Other weights run the FP64 SIMT M-step, or fail with GMM_ERR_ARG at the next M-step when "mstep_path" (or "path") is
 *     GMM_PATH_TENSOR.  The decision uses the global extremes: every rank takes the same path.
 *   - setting or clearing weights marks the memberships stale, as gmm_set_clusters does: gmm_mstep and
 *     gmm_em_iterations then need a gmm_estep first.  gmm_upload_events / gmm_upload_events_file keep the weights (they
 *     belong to event positions).
 * Device memory: one [n_local rounded up to 32] float buffer, allocated on the first call, freed by gmm_destroy.
 * Errors: a weight that is NaN, infinite or negative on any rank, a global sum of 0, or weights on some ranks and NULL on
 * others -> GMM_ERR_ARG on every rank, and the weights in effect before the call stay unchanged; a failed collective ->
 * GMM_ERR_NCCL.                                      */
int  gmm_set_weights(gmm_ctx*, const float* weights, double* total_out);

/* D2H of the parameters, optionally the memberships of THIS shard into
 * host_out->memberships laid out [K][n_local] (gaussian.cu:761-774).       */
int  gmm_get_clusters(gmm_ctx*, int K, clusters_t* host_out, int with_memberships);

/* estep1 + estep2 + likelihood reduction (gaussian_kernel.cu:383-512,
 * gaussian.cu:713-746).  Writes memberships (device), returns the GLOBAL
 * log-likelihood (summed over ranks).  A cluster with pi = 0 (logit constant
 * + ln pi = -inf) gets a membership of exactly 0 and adds nothing to any
 * event's density, as in estep2, on every path and at every K, also when it
 * comes first or fills a whole 64-cluster pass.  Every pi = 0 (no finite
 * logit) is not supported.                                                   */
int  gmm_estep(gmm_ctx*, int K, float* loglik_out);

/* mstep_N + mstep_means + mstep_covariance1 + the three reductions and host
 * normalisations (gaussian_kernel.cu:522-677, gaussian.cu:538-687).
 * Reads the device memberships; leaves N, means, R updated on host+device. */
int  gmm_mstep(gmm_ctx*, int K);

/* constants_kernel semantics: Rinv, constant (ln det), pi
 * (gaussian_kernel.cu:107-259, gaussian.cu:698-708).  The DxD inversion runs
 * on the host here (invert_matrix.cpp semantics); inside gmm_em /
 * gmm_em_iterations see option "finalize".                                  */
int  gmm_constants(gmm_ctx*, int K);

/* The EM loop of gaussian.cu:532-755 (preceded by the initial E-step of
 * :487-523): while(iters < min_iters || (|change| > epsilon && iters <
 * max_iters)).  Returns the final global log-likelihood and iteration count.
 * epsilon < 0 selects the reference value (gaussian.cu:458).                */
int  gmm_em(gmm_ctx*, int K, int min_iters, int max_iters, float epsilon,
            float* loglik_out, int* iters_out);

/* Exactly `iters` passes of the loop body of gaussian.cu:532-755 (M-step,
 * reductions, constants, E-step) with no convergence test; needs a preceding
 * gmm_estep()/gmm_em() for the same K.  Returns the global log-likelihood of
 * the last E-step.  This is the unit bench.py times.                        */
int  gmm_em_iterations(gmm_ctx*, int K, int iters, float* loglik_out);

/* ---- using a fitted mixture (sklearn's predict / score_samples) ---------
 * Evaluate n events (host, row-major [n][D], NOT the context's shard) against
 * the parameter set the next gmm_estep(ctx, K) would use.  Per event:
 *   labels[i]   = argmax_k of the posterior (lowest k on ties, -1 if every
 *                 logit is NaN),
 *   max_resp[i] = that posterior (NaN when labels[i] = -1),
 *   logp[i]     = ln sum_k pi_k N(x_i | k) (the E-step's log-denominator).
 * Any of the three output pointers may be NULL.  *loglik_out (may be NULL) =
 * sum of logp in double over this call, THIS context only (no collective).
 * The kernels are the ones the E-step would use (wgmma for D in {8, 16, 24}
 * when its operand serves the parameters, else SIMT); a chunk holding an event
 * beyond 2^14 standard deviations of the training data (or not finite) is
 * re-scored by the SIMT kernel, or fails with GMM_ERR_STATE under
 * GMM_PATH_TENSOR.  On the training shard the outputs equal the E-step's
 * (max_resp bit for bit).  A cluster with pi = 0 is never a label and adds
 * nothing to logp (gmm_estep).  The batch streams through two pinned
 * buffers in chunks of option "score_chunk" events; nothing of the EM state
 * (memberships, statistics, log-likelihood, gmm_get_profile) changes.
 * Errors: K outside [1, Kmax], n < 0 or events_aos == NULL with n > 0 ->
 * GMM_ERR_ARG; K != the K of the current parameters, or a call between
 * gmm_mstep and gmm_constants (half-updated parameters) -> GMM_ERR_STATE.
 * After gmm_fit, score against the best model with
 * gmm_set_clusters(ctx, ideal_K, saved) followed by gmm_score.               */
int  gmm_score(gmm_ctx*, int K, const float* events_aos, long long n,
               int* labels, float* max_resp, float* logp, double* loglik_out);
/* Since the last reset: out[0] score-kernel ms, out[1] wall ms inside
 * gmm_score, out[2] chunks scored by the wgmma kernel, out[3] chunks scored
 * by the SIMT kernel (including re-scored ones, which out[2] then omits).   */
int  gmm_get_score_profile(gmm_ctx*, double out[4], int reset);

/* E-step + M-step statistics of n new events (host, row-major [n][D], NOT
 * the context's shard) under the parameter set the next gmm_estep(ctx, K)
 * would use.  No collective; nothing of the EM state changes (memberships,
 * statistics, log-likelihood, gmm_get_profile, gmm_get_score_profile).
 *   stats_out   [gmm_stats_len(K, D)] doubles: S0 | S1 | S2 per cluster about
 *               the context's centre (the packed layout of gmm_host_finalize),
 *               then the sum of the events' log-densities.  Overwritten, not
 *               accumulated.  May be NULL (then no M-step work is done).
 *   shift_out   [D] the centre s the statistics are about (the float-rounded
 *               value the kernels use); may be NULL.
 *   memberships [K][n] cluster-major (the clusters_t layout, so
 *               gmm_write_results can write them); may be NULL.
 * At least one of stats_out / memberships must be non-NULL.  Statistics of
 * several calls (batches, ranks) about the same centre add up: summed and
 * passed to gmm_host_finalize, then gmm_set_clusters, they make one EM
 * iteration over data that never has to fit on the device.
 * Kernels: those the context's own steps would use, chosen per chunk of option
 * "score_chunk" events.  A chunk with an event beyond 2^14 standard
 * deviations runs the SIMT E-step; one with an event at or beyond the
 * training data's power-of-two bound zb (the tensor M-step's fixed-point
 * range) runs the FP64 SIMT M-step; either fails with GMM_ERR_STATE when the
 * step concerned is forced to GMM_PATH_TENSOR.  On the training shard, in one
 * chunk, the memberships equal gmm_estep's bit for bit, and so do the
 * statistics gmm_mstep's wgmma M-step forms.
 * Errors: K outside [1, Kmax], n < 0, events_aos == NULL with n > 0, both
 * outputs NULL, or a coordinate that is not finite -> GMM_ERR_ARG; K != the K
 * of the current parameters, a call between gmm_mstep and gmm_constants, or a
 * multi-rank context whose centre is not fixed yet (a SIMT-only context
 * before its first gmm_mstep / gmm_em) -> GMM_ERR_STATE.  n = 0 gives zero
 * statistics and fills shift_out.                                            */
int  gmm_score_stats(gmm_ctx*, int K, const float* events_aos, long long n,
                     double* stats_out, double* shift_out, float* memberships);
/* Since the last reset: out[0] kernel ms (prep + E + M), out[1] wall ms,
 * out[2] / out[3] chunks whose responsibilities came from the wgmma / SIMT
 * E-step, out[4] / out[5] chunks whose statistics came from the wgmma /
 * FP64 SIMT M-step, out[6] ms the compute stream stood between a chunk's prep
 * kernel and its E-step: the range-flag round trip to the host plus the
 * host's staging of the next chunk, which is issued before the flag is read. */
int  gmm_get_score_stats_profile(gmm_ctx*, double out[7], int reset);

/* Draw n events from the mixture (sklearn's sample(n)): events_out [n][D] row-major, labels_out [n] the
 * component of each event (may be NULL).  The parameters are the set the next gmm_estep(ctx, K) would use:
 * pi, means and R of the context's host copy.  No collective; nothing of the EM state changes (memberships,
 * statistics, log-likelihood, gmm_get_profile, gmm_get_score_profile, gmm_get_score_stats_profile).
 * Event i of the call is the event of global index g = first + i, a function of (parameters, seed, g)
 * alone: options "path" and "score_chunk" and the number of ranks do not change it, and calls (first, n1)
 * and (first + n1, n2) give the bits of one call (first, n1 + n2) — ranks or batches split one sample so.
 * Semantics (restated in float64 numpy by tests/_sample_ref.py):
 *   - words: Philox4x32-10 (Salmon et al. 2011, the Random123 definition), key (lo32(seed), hi32(seed));
 *     block j of event g uses counter (lo32(g), hi32(g), j, 0); the event's words are block 0's four
 *     words (x, y, z, w), then block 1's, and so on.
 *   - component: u = ((w0 >> 5) 2^26 + (w1 >> 6)) 2^-53 (53 bits, [0, 1)).  C_k = running sum in double
 *     of the float pi in cluster order, T = C_{K-1}; the label is the first k with u*T < C_k (product
 *     rounded in double), or, if rounding leaves none, the last k with pi_k > 0.  A cluster with pi = 0
 *     is never drawn; one that carries the reference's pi = 1e-10 (N < 0.5) is drawn with that weight.
 *   - normals: pair p = 0 .. ceil(D/2) - 1 uses words a = w_{2+2p}, b = w_{3+2p}, in float:
 *     u1 = ((float)a + 0.5f) 2^-32 in (0, 1], r = sqrtf(-2 logf(u1)) (at most ~6.8),
 *     (s, c) = sincospif((float)b 2^-31), z_{2p} = r c, z_{2p+1} = r s (the last s dropped for odd D).
 *     Conversions round to nearest; no fast-math approximations.
 *   - event: x = mu_k + U_k z, with U_k the upper-triangular factor R_k = U_k U_k^T that the host
 *     finalisation computes in double from the float R (off-diagonal pairs averaged, pivots from the last
 *     one up), rounded to float: x_d = fmaf-accumulation of U_dj z_j for j = d .. D-1 onto mu_d, in float.
 *   This is sklearn's distribution, except that events come i.i.d. in index order where sklearn sorts
 *   them by component.
 * The kernel writes chunks of option "score_chunk" events through gmm_score's two device chunks and pinned
 * stages; the parameter block ([K] double + [K][D + D(D+1)/2] float, padded) is allocated for Kmax on the
 * first call and freed by gmm_destroy.
 * Errors: K outside [1, Kmax], n < 0, first < 0, first + n > 2^62, or events_out == NULL with n > 0 ->
 * GMM_ERR_ARG; K != the K of the current parameters, a call between gmm_mstep and gmm_constants, a cluster
 * whose R is not positive definite, a pi that is negative or not finite (the first such cluster is named
 * in the message), or T <= 0 -> GMM_ERR_STATE.  n = 0 returns GMM_OK and writes nothing.              */
int  gmm_sample(gmm_ctx*, int K, long long n, unsigned long long seed, long long first,
                float* events_out, int* labels_out);
/* Since the last reset: out[0] sampling-kernel ms, out[1] wall ms inside gmm_sample.                   */
int  gmm_get_sample_profile(gmm_ctx*, double out[2], int reset);

/* Score n events measured on a subset O of the dimensions, and impute the others, under the parameter set the next
 * gmm_estep(ctx, K) would use (statistical file matching of panels that share a backbone; Gaussian-mixture regression).
 *   obs_dims [n_obs]   strictly increasing indices in [0, D): the set O.  M = the other dimensions in increasing
 *                      order, NM = D - n_obs of them.
 *   events_obs         [n][n_obs] row-major, the coordinates of O in the order of obs_dims.
 *   labels, max_resp, logp   as gmm_score defines them, for the MARGINAL mixture sum_k pi_k N(x_O | mu_kO, R_kOO).
 *   cond_mean [n][NM]  E[x_M | x_O];  cond_var [n][NM]  the diagonal of Cov[x_M | x_O].  Ignored when NM = 0.
 *   *loglik_out        sum of logp in double over this call, THIS context only.
 * Every output pointer may be NULL.  No collective; nothing of the EM state changes (memberships, statistics,
 * log-likelihood, the SIMT E-step's parameters, gmm_get_profile, gmm_get_score_profile, gmm_get_score_stats_profile,
 * gmm_get_sample_profile).
 * Semantics (restated in float64 numpy by tests/_condition_ref.py), from the float means, Rinv (P), constant and pi of
 * the context's host copy, per cluster k:
 *   - NM = 0: the marginal set is (means, Rinv, constant, pi) itself, so the outputs are gmm_score's SIMT kernel's.
 *   - NM >= 1, in double: S = (P + P^T) / 2; S_MM = L L^T (Cholesky; a pivot <= 0 or not finite -> GMM_ERR_STATE);
 *       P_O        = S_OO - S_OM S_MM^-1 S_MO                      (the inverse of R_OO)
 *       constant_O = constant + (NM/2) ln 2 pi - (1/2) ln det S_MM  (ln det R_OO = ln det R + ln det P_MM)
 *       G          = -S_MM^-1 S_MO  [NM][n_obs],   c_d = (S_MM^-1)_dd
 *     each rounded to float.  The marginal set (mu_O, P_O, constant_O, pi) is packed as the SIMT E-step packs its
 *     parameters (coefficients P_ii and P_ij + P_ji, constant_O + logf(pi) in float).
 *   - scoring: gmm_score's SIMT kernel on the marginal set: dx = x_O - mu_kO, l_k = constant_O + ln pi_k - dx^T P_O dx / 2
 *     in float, online log-sum-exp and arg-max.  Computing the imputations too changes no bit of labels, max_resp, logp.
 *   - imputation, in float: m_k = mu_kM + G_k dx (G_k dx summed first), r_k = exp(l_k - logp);
 *     cond_mean = sum_k r_k m_k,  cond_var = sum_k r_k (c_k + (m_k - cond_mean)^2), merged cluster by cluster with a
 *     weighted running mean and sum of squares (West 1979), rescaled when the running maximum logit moves.
 *   Events with a coordinate that is not finite give what gmm_score's SIMT kernel gives (label -1, NaN) and NaN
 *   imputations.  The result of an event does not depend on the chunking or on the split into calls.
 * Rows stream in chunks of option "score_chunk" events through gmm_score's two device chunks, pinned stages and copy
 * stream.  A parameter block for Kmax clusters (at most 700 floats per cluster, at D = 32) and its pinned mirror are
 * allocated on the first call; an imputing call adds per slot 2 x score_chunk x NM floats on the device and pinned,
 * grown to the largest chunk x NM seen.  gmm_destroy frees them.
 * Errors: K outside [1, Kmax], n < 0, events_obs == NULL with n > 0, obs_dims == NULL, n_obs outside [1, D], or indices
 * that are not strictly increasing or out of range -> GMM_ERR_ARG; K != the K of the current parameters, a call between
 * gmm_mstep and gmm_constants, or a cluster whose block P_MM is not positive definite (the first one is named in the
 * message) -> GMM_ERR_STATE.  n = 0 returns GMM_OK after these checks and writes nothing, *loglik_out included.        */
int  gmm_condition(gmm_ctx*, int K, const int* obs_dims, int n_obs, const float* events_obs, long long n,
                   int* labels, float* max_resp, float* logp, float* cond_mean, float* cond_var, double* loglik_out);
/* Since the last reset: out[0] kernel ms, out[1] wall ms inside gmm_condition.                                        */
int  gmm_get_condition_profile(gmm_ctx*, double out[2], int reset);

/* M-step statistics of n events measured on a subset O of the dimensions: the E-step of EM with values missing at
 * random (Ghahramani and Jordan 1994), so that EM can fit a full-D mixture to tubes of a split panel that share a
 * backbone.  The statistics are gmm_score_stats' (packed, about the context's centre, summable over calls, ranks and
 * missing patterns) with every entry that involves a missing dimension replaced by its expectation given x_O under the
 * parameter set the next gmm_estep(ctx, K) would use.  One EM iteration over tubes t: stats = sum_t
 * gmm_condition_stats(tube t) (+ gmm_score_stats of complete rows), gmm_host_finalize, gmm_set_clusters.
 *   obs_dims, n_obs, events_obs   as gmm_condition defines them (rows [n][n_obs] in the order of obs_dims).
 *   stats_out   [gmm_stats_len(K, D)], full-D layout of gmm_host_finalize about the centre; overwritten, not
 *               accumulated; the last slot is the sum of the events' marginal log-densities (the observed-data
 *               log-likelihood).  May be NULL (then no M-step work is done).
 *   shift_out   [D] the centre s (float-rounded when the wgmma M-step can run); may be NULL.
 *   memberships [K][n] cluster-major: the posteriors under the MARGINAL mixture of gmm_condition; may be NULL.
 * At least one of stats_out / memberships must be non-NULL.  No collective; nothing of the EM state or of another
 * call's profile changes.
 * Semantics (restated in float64 numpy by tests/_condition_stats_ref.py), with NM = D - n_obs >= 1:
 *   - the marginal parameters are gmm_condition's (same derivation, same float rounding, same packing); the
 *     memberships come from the SIMT E-step on them, so their row maximum is gmm_condition's max_resp bit for bit.
 *   - T0 = sum r, T1 = sum r y, T2 = sum r y y^T (y = x_O - s_O) come from the context's own M-step run over all D
 *     dimensions on rows whose missing dimensions contribute zeros.
 *   - per cluster, in double from the float Rinv (P), with S = (P + P^T) / 2: G = -S_MM^-1 S_MO, C = S_MM^-1 (the full
 *     conditional covariance), b = (mu_M - s_M) - G (mu_O - s_O), u = G T1.  Then E[x_M | x_O, k] - s_M = b + G y and
 *       S0 = T0, S1_O = T1, S2_OO = T2,  S1_M = b T0 + u,  S2_MO = b T1^T + G T2,
 *       S2_MM = T0 (b b^T + C) + b u^T + u b^T + G T2 G^T.
 *   - n_obs = D is gmm_score_stats: the same code path and the same bits.
 * Kernels: a prep kernel, the SIMT E-step on the observed dimensions, and the M-step gmm_score_stats would choose, per
 * chunk of option "score_chunk" events (a chunk with an observed coordinate at or beyond the tensor M-step's bound zb
 * runs the FP64 SIMT M-step, or fails with GMM_ERR_STATE under mstep_path = GMM_PATH_TENSOR).  Rows stream through
 * gmm_score's slots; the chunk buffers are gmm_score_stats', plus an observed copy of D x score_chunk floats allocated on
 * the first call with NM >= 1 and freed by gmm_destroy.
 * Errors: K outside [1, Kmax], n < 0, events_obs == NULL with n > 0, obs_dims == NULL, n_obs outside [1, D], indices
 * that are not strictly increasing or out of range, both outputs NULL, or a coordinate that is not finite ->
 * GMM_ERR_ARG; K != the K of the current parameters, a call between gmm_mstep and gmm_constants, a cluster whose block
 * P_MM is not positive definite (the first one is named in the message), or a multi-rank context whose centre is not
 * fixed yet -> GMM_ERR_STATE.  n = 0 gives zero statistics and fills shift_out.                                       */
int  gmm_condition_stats(gmm_ctx*, int K, const int* obs_dims, int n_obs, const float* events_obs, long long n,
                         double* stats_out, double* shift_out, float* memberships);
/* Since the last reset: out[0] kernel ms (prep + E + M), out[1] wall ms inside gmm_condition_stats, out[2] / out[3]
 * chunks whose statistics came from the wgmma / FP64 SIMT M-step.                                                    */
int  gmm_get_condition_stats_profile(gmm_ctx*, double out[4], int reset);

/* ---- variational Bayesian mixture (sklearn's BayesianGaussianMixture, covariance_type='full') ------------------------
 * One fit at an upper bound K; a Dirichlet-process (or Dirichlet) prior on the weights empties the components the data do
 * not need, where gmm_fit instead runs EM at every model order and keeps the smallest Rissanen score.                */
#define GMM_VB_DIRICHLET_PROCESS      0   /* sklearn's default weight_concentration_prior_type */
#define GMM_VB_DIRICHLET_DISTRIBUTION 1

typedef struct {
    int           weight_prior_type;      /* GMM_VB_*                                                    */
    double        weight_concentration;   /* gamma0 > 0;  <= 0 selects 1/K                               */
    double        mean_precision;         /* beta0 > 0;   <= 0 selects 1                                 */
    double        dof;                    /* nu0 > D-1;   <= 0 selects D                                 */
    const double* mean;                   /* [D] m0;      NULL selects the events' mean                  */
    const double* covariance;             /* [D][D] Psi0, symmetric positive definite; NULL selects the
                                             events' covariance with ddof = 1 (np.cov(X.T))              */
    double        reg_covar;              /* >= 0 added to each sk's diagonal; < 0 selects 1e-6          */
} gmm_vb_prior;

typedef struct {                          /* every pointer may be NULL                                   */
    double* weights;                      /* [K]  sklearn's weights_ (normalised E[pi])                  */
    double* weight_concentration;         /* [2][K] (DP: the Beta parameters) or [K] (Dirichlet)         */
    double* mean_precision;               /* [K]  beta                                                   */
    double* dof;                          /* [K]  nu                                                     */
    double* mean_prior;                   /* [D]  the m0 used (after defaults)                           */
    double* covariance_prior;             /* [D][D] the Psi0 used                                        */
} gmm_vb_posterior;

/* Variational Bayesian EM at K components.  Collective over the ranks of a communicator, like gmm_em (same arguments on
 * every rank).  Semantics (restated in float64 numpy by tests/_vb_ref.py):
 *   - start: the context's current parameter set for K (gmm_seed, gmm_seed_kmeans, gmm_set_clusters or an earlier fit).
 *     One E-step under it gives the responsibilities g0 (sklearn's initial resp); a VB M-step on g0 gives posterior 0.
 *     Iteration i = 1, 2, ...: an E-step under posterior i-1, the VB M-step that gives posterior i, the lower bound LB_i of
 *     that E-step's responsibilities and posterior i.  The loop stops after iteration i when i >= min_iters and
 *     |LB_i - LB_{i-1}| < tol (LB_0 = -inf), or at max_iters; a last E-step under the final posterior leaves valid
 *     memberships: iters + 2 E-steps and iters + 1 M-steps.  tol is absolute on the total bound (sklearn's tol).
 *   - VB M-step, in double, from the packed statistics S0, S1, S2 about the centre s that the E- and M-step kernels
 *     form (wgmma or FP64 SIMT, weights included, summed over the ranks): nk = S0 + 10 * 2^-52, xk = (S0 s + S1) / nk,
 *     nk sk = sum g (x - xk)(x - xk)^T + nk reg_covar I (expanded about s); then sklearn's _estimate_weights,
 *     _estimate_means, _estimate_wishart_full: beta = beta0 + nk, m = (beta0 m0 + nk xk) / beta, nu = nu0 + nk,
 *     C = (Psi0 + nk sk + nk beta0 / beta (xk - m0)(xk - m0)^T) / nu, and weights_ as _set_parameters forms it.
 *   - the parameter set left in the context and in host_out: N = nk, means = m, R = C (float), Rinv from the reverse
 *     Cholesky factorisation of the float R (as the host finalisation forms it), pi = weights_ rounded to float and
 *     floored at FLT_MIN, and constant such that constant + ln pi (the additive term every E-step packs) is sklearn's
 *       -D/2 ln 2 pi - 1/2 ln det R - D/2 ln nu + 1/2 (D ln 2 + sum_{i<D} psi((nu - i) / 2)) - D / (2 beta) + E[ln pi_k]
 *     with ln det R from the same factorisation.  So gmm_estep, gmm_score and gmm_score_stats on the fitted context give
 *     sklearn's predict_proba, predict and score_samples, and gmm_sample draws from weights_.  avgvar is left as it was.
 *   - bound: LB = -sum_n w_n sum_k g ln g (0 ln 0 = 0) - log_wishart - log_norm_weight - D/2 sum_k ln beta_k
 *     (sklearn's _compute_lower_bound, with ln det C from a Cholesky factorisation of the double C); psi is the library's
 *     own double digamma (recurrence + asymptotic series), lgamma / betaln from libm.  The entropy term is one pass of
 *     resp_entropy_kernel over the memberships (block partials added in block order, then one ncclAllReduce of one
 *     double), run only in iterations whose bound is used (i >= min_iters - 1, or all when lower_bounds_out != NULL).
 *   - weights (gmm_set_weights) enter the statistics as in gmm_em, the entropy as w_n, and the default prior as the
 *     weighted mean and covariance with denominator sum w - 1: integer weights give the fit of replicated rows.
 *   - the default m0 / Psi0 come from the context's own M-step at K = 1 on unit responsibilities (written by the k-means
 *     assignment kernel with one centre), which allocates gmm_seed_kmeans' buffers.
 *   - afterwards: cur_K = K, memberships valid, gmm_get_profile counts the iterations; the set counts as one given from
 *     outside (as after gmm_set_clusters): a later replay of the device-side finalisation keeps its Rinv and constant.
 *   host_out          all clusters_t arrays except memberships (may be NULL)
 *   post_out          the posterior (may be NULL; so may each of its pointers)
 *   lower_bound_out   LB of the last iteration (-inf when max_iters = 0); lower_bounds_out [max_iters]: LB_1 .. LB_iters
 *   iters_out         iterations run; converged_out 1 when the tol test stopped the loop
 * Errors: K outside [1, Kmax], a NULL prior, an unknown prior type, gamma0 / beta0 / reg_covar / m0 not finite, nu0 in
 * (0, D - 1] or NaN, Psi0 not symmetric positive definite, min_iters < 0, max_iters < min_iters, or tol < 0 or NaN ->
 * GMM_ERR_ARG; a default prior over a total weight <= 1 -> GMM_ERR_ARG; K != the K of the current parameters, a call
 * between gmm_mstep and gmm_constants, or a posterior whose float covariance is not positive definite -> GMM_ERR_STATE;
 * a failed collective -> GMM_ERR_NCCL.
 * Device memory: [4 x SMs + 1] doubles of entropy partials (and their pinned mirror), allocated on first use, freed by
 * gmm_destroy.                                                                                                        */
int  gmm_vb_em(gmm_ctx*, int K, const gmm_vb_prior* prior, int min_iters, int max_iters, double tol,
               clusters_t* host_out, gmm_vb_posterior* post_out,
               double* lower_bound_out, double* lower_bounds_out /* [max_iters] or NULL */,
               int* iters_out, int* converged_out);

/* Host-only, usable without a GPU (as gmm_host_finalize): packed statistics about `shift` (gmm_stats_len(K, D) doubles,
 * e.g. the sum of gmm_score_stats over batches) -> the VB parameter set of gmm_vb_em in `out` (N, pi, constant, means,
 * R, Rinv; avgvar untouched) and the posterior; *bound_out (may be NULL) = -log_wishart - log_norm_weight
 * - D/2 sum ln beta (the lower bound without its entropy term).  prior->mean and prior->covariance are required.
 * Errors: as gmm_vb_em's argument errors, NULL stats / shift / out / prior mean or covariance -> GMM_ERR_ARG; a float
 * covariance that is not positive definite -> GMM_ERR_STATE.                                                          */
int  gmm_host_vb_finalize(const double* stats, const double* shift, int K, int D, const gmm_vb_prior* prior,
                          clusters_t* out, gmm_vb_posterior* post_out, double* bound_out);

/* The library's digamma in double (recurrence to x >= 10, then the asymptotic series): n values, x > 0.             */
int  gmm_host_digamma(const double* x, double* out, long long n);

/* Since the last reset: out[0] entropy-kernel ms, out[1] host VB finalisation ms, out[2] wall ms inside gmm_vb_em.    */
int  gmm_get_vb_profile(gmm_ctx*, double out[3], int reset);

/* ---- combining mixture components into clusters (Baudry, Raftery, Celeux, Lo and Gottardo, JCGS 19 (2010); mclust's
 * clustCombi, flowMerge) ----------------------------------------------------------------------------------------------
 * A population that is skewed, curved or heavy-tailed is fitted by several Gaussian components.  These calls keep the
 * K-component density and merge components into clusters hierarchically, each merge chosen by the largest drop in
 * classification entropy; a cluster is a union of components, so the density never changes (unlike the order reduction
 * of gmm_fit, which re-fits one Gaussian per merged pair).  Workflow: a fit (gmm_em, gmm_fit, gmm_vb_em), gmm_estep,
 * gmm_combine, a level L (gmm_host_combine_elbow or the caller's choice), gmm_host_combine_groups, gmm_combine_labels.
 * After gmm_fit the current memberships are those of the last order it ran, not of ideal_K: to combine the best model,
 * call gmm_set_clusters(ideal_K, saved) and gmm_estep first.
 * Notation (restated in float64 / float32 numpy by tests/_combine_ref.py):
 *   - tau_k(n) is the stored float membership of event n in component k; w_n the weight of gmm_set_weights (1 without).
 *   - group sum: tau_A(n) of a group A is the float sum of its members' rows, added left to right in increasing component
 *     index (no FMA, no reassociation); a singleton is the stored value.
 *   - pair gain: dEnt(A, B) = sum_n w_n phi(tau_A(n), tau_B(n)), phi(a, b) = (a+b) ln(a+b) - a ln a - b ln b, computed in
 *     float as M h(m / M) with M = max(a, b), m = min(a, b), h(r) = (1 + r) log1pf(r) - r logf(r), and phi = 0 when
 *     m = 0; both terms of h are >= 0 on (0, 1], so nothing cancels.  Events are summed in double.
 *   - hierarchy: step s = 0 .. K-2 merges the live pair (A, B) of largest all-reduced gain, ties between equal doubles to
 *     the lexicographically smallest (a, b).  A group is named by its smallest component: a < b, and the merged group
 *     keeps a.  The choice is made from the reduced gains, identically on every rank.
 * Kernels (csrc/kernels_combine.cuh, sm_90a): one all-pairs pass over the singletons (32 x 32 component tiles times event
 * ranges, the rows staged in shared memory), then after each merge one pass of the merged group against every live group,
 * each group sum formed on the fly from the original rows (one read of all K rows per step).  The memberships are never
 * copied or rewritten.  No atomics: repeated calls give the same bits.
 * Device memory: per-(range, value) partials of at most about 4 MB (K = 512), the reduced values with a pinned mirror
 * (K(K-1)/2 + K doubles), the group lists (2 x 512 + 1 ints, pinned mirror), allocated on the first call and grown with
 * K; gmm_combine_labels adds an int and a float per event (the pitched row length).  gmm_destroy frees them.          */

/* The entropy-criterion hierarchy over the memberships of the last E-step for K.  Collective over the ranks of a
 * communicator, like gmm_em (same K on every rank).
 *   merges_out  [K-1][2]: step s merged groups {a, b}, a < b
 *   gain_out    [K-1]:    that pair's gain dEnt
 *   entropy_out [K]:      entropy_out[L-1] = the classification entropy at L clusters; entropy_out[K-1] =
 *                         -sum_n w_n sum_k tau ln tau (0 ln 0 = 0) from resp_entropy_kernel, as gmm_vb_em sums it;
 *                         entropy_out[L-2] = entropy_out[L-1] - gain_out[K-L] in double
 *   mass_out    [K-1]:    m_A + m_B, where m_k = sum_n w_n tau_k(n) in double and a group's mass is the sum of its
 *                         members' masses in member order (Baudry's abscissa: entropy against cumulative merged mass)
 * Every output except merges_out may be NULL; K = 1 writes only entropy_out[0] (and merges_out may be NULL).
 * Nothing of the state changes: not the memberships, not the parameters, not gmm_get_profile nor any other profile.
 * Errors: K outside [1, Kmax] or a NULL merges_out with K >= 2 -> GMM_ERR_ARG; K != the K of the current parameters,
 * memberships that are not valid (before any E-step, or after gmm_set_clusters or gmm_set_weights), a call between
 * gmm_mstep and gmm_constants, or a membership that is not finite (the first component concerned is named) ->
 * GMM_ERR_STATE; a failed collective -> GMM_ERR_NCCL.                                                                */
int  gmm_combine(gmm_ctx*, int K, int* merges_out, double* gain_out, double* entropy_out, double* mass_out);

/* Labels of THIS shard's events under a grouping of the K components into G clusters (group[k] in [0, G), e.g. from
 * gmm_host_combine_groups): label = argmax over g of the group sum of {k : group[k] = g} (a cluster without members sums
 * to 0), the lowest g on ties, -1 when every sum is NaN; max_out = that sum (NaN for -1).  One read of the K rows.  No
 * collective; nothing of the state changes.  labels_out [n_local] (may be NULL only when n_local = 0), max_out [n_local]
 * or NULL.
 * Errors: K outside [1, Kmax], a NULL group, G outside [1, K], a group index outside [0, G) or a NULL labels_out ->
 * GMM_ERR_ARG; the state errors of gmm_combine -> GMM_ERR_STATE.                                                     */
int  gmm_combine_labels(gmm_ctx*, int K, const int* group, int G, int* labels_out, float* max_out);

/* Host-only, no GPU needed.  The cluster of each component at level L (1 <= L <= K) of a hierarchy: the first K-L
 * merges of merges [K-1][2] applied; clusters numbered 0 .. L-1 in increasing order of their smallest component.
 * Errors: K outside [1, 512], L outside [1, K], a NULL group_out, a NULL merges with K >= 2, or a merge list that is
 * not a valid hierarchy (every step a pair a < b of groups still live, named by their smallest components) -> GMM_ERR_ARG. */
int  gmm_host_combine_groups(const int* merges, int K, int L, int* group_out);

/* Host-only.  The change point flowMerge and Baudry use to pick the level: points P_L = (x_L, entropy[L-1]) for L = 1 .. K,
 * x_L = L when x is NULL.  For each c in 2 .. K-1, least-squares lines are fitted to {P_L : L <= c} and to {P_L : L >= c}
 * (a segment whose x are all equal uses its mean); *L_out = the c of the smallest total residual sum of squares, the
 * smaller c on ties.  Sums are centred and in index order, in double.
 * Errors: K < 3, a NULL entropy or L_out, or a value that is not finite -> GMM_ERR_ARG.                              */
int  gmm_host_combine_elbow(const double* entropy, const double* x /* [K] or NULL */, int K, int* L_out);

/* Since the last reset: out[0] kernel ms (gmm_combine's and gmm_combine_labels' passes), out[1] wall ms inside
 * gmm_combine, out[2] wall ms inside gmm_combine_labels.                                                             */
int  gmm_get_combine_profile(gmm_ctx*, double out[3], int reset);

/* ---- EM over several samples with shared components (the maximum-likelihood counterpart of Cron et al., PLoS Comput
 * Biol 9 (2013) e1003130, without the HDP prior) ----------------------------------------------------------------------
 * A study is many samples (patients, time points, stimulations) measured on the same panel.  Separate fits give components
 * that are not aligned; one pooled fit classifies every event under the pool's mixing weights, biasing each sample's
 * counts toward the pool where populations overlap.  This model keeps the means and covariances shared and gives each
 * sample s its own mixing weights pi_{s,k}: aligned populations and per-sample abundances from one fit.  ("Sample" is a
 * set of events measured together, not a draw of gmm_sample.)
 * Semantics (restated in float64 / float32 numpy by tests/_multisample_ref.py):
 *   - sample s is the global event range [offsets[s], offsets[s+1]); w_n is the weight of gmm_set_weights (1 without).
 *   - the library's E-step under the pooled set (pi_k) gives r_nk ~ pi_k N(x_n | k).  With rho_{s,k} = pi_{s,k} / pi_k the
 *     per-sample posterior is r'_nk = r_nk rho_{s,k} / S_n, S_n = sum_j r_nj rho_{s,j}, and ln p'(x_n) = ln p(x_n) + ln S_n.
 *     The pooled pi keeps rho <= N / n_s, so no responsibility the reweight needs has underflowed.
 *   - reweight, per event of sample s, in float with one rounding per operation: t_k = r_k * rho_{s,k}, S = t_0 + t_1 + ...
 *     in increasing k, r'_k = t_k / S; the log-likelihood correction is w_n log((double)S), summed in double.  Only rows
 *     k < K of the shard's events are written.  An event whose every t_k is 0 (possible only with zeros in pi_init) gets
 *     NaN memberships and a -inf log-likelihood.
 *   - masses M_{s,k} = sum_{n in s} w_n r'_nk and n_s = sum_{n in s} w_n, in double in a fixed order without atomics,
 *     zeros for samples outside a rank's shard, summed over the ranks by one ncclAllReduce.
 *   - start: an E-step under the current parameter set for K, then the reweight with pi^0_{s,k} = pi_init[s][k] / sum_j
 *     pi_init[s][j] (rows need not be normalised).  pi_init = NULL: pi^0_{s,k} = pi_k and rho = 1; the pass then only forms
 *     the masses, writes no membership and adds nothing to the log-likelihood, so the start equals gmm_estep bit for bit.
 *   - loop: gmm_em's (the same stop rule, epsilon < 0 selecting the same default, min_iters / max_iters as there), with the
 *     reweight after every E-step.  Each iteration: the M-step statistics over r', one reduction of them (its
 *     log-likelihood slot already holds sum w ln p + sum w ln S), the stop test, the host finalisation of gmm_em (N, means,
 *     R, avgvar rules, constants, the pooled pi with its 0.5 / 1e-10 rules), pi_{s,k} = max(M_{s,k} / n_s, 1e-10) in double
 *     (floored, not renormalised), rho_{s,k} = (float)(pi_{s,k} / (double)pi_k), then the E-step and the reweight.  Every
 *     iteration takes the host finalisation (the device-side one of option "finalize" is not used).
 *   - afterwards: the context holds the pooled parameter set (a valid gmm_em set: gmm_score, gmm_sample and
 *     gmm_get_clusters see it), cur_K = K, and the memberships are the per-sample posteriors of the last E-step:
 *     gmm_combine and gmm_combine_labels work on them, a later gmm_estep replaces them with pooled ones.  gmm_get_profile
 *     counts the iterations.
 *   - scoring new events of sample s: put pi_out[s] (as float) into the clusters' pi, gmm_set_clusters, then gmm_score.
 * Collective over the ranks of a communicator, like gmm_em: the same K, S, offsets, pi_init and iteration arguments on
 * every rank.  A sample may straddle shards.
 *   offsets      [S+1] global event offsets: offsets[0] = 0, offsets[S] = n_global, strictly increasing; 1 <= S <= 4096
 *   pi_init      [S][K] starting weights, or NULL
 *   pi_out       [S][K] the pi_{s,k} the last E-step used, or NULL
 *   n_out        [S] n_s, or NULL
 *   loglik_out   the last E-step's multi-sample log-likelihood sum_n w_n ln p'(x_n)
 *   logliks_out  [max_iters + 1] or NULL: that of E-step i, E-step 0 being the start
 *   iters_out    iterations run
 * Kernels (csrc/kernels_multisample.cuh, sm_90a): one reweight pass that reads and writes each membership once (windows of
 * E events staged in shared memory, persistent CTAs over units that never cross a sample boundary, one partial per CTA and
 * sample segment) and a finishing kernel that adds the partials per sample in order and the correction into the
 * statistics' log-likelihood slot.  The E- and M-step kernels, the K > 64 passes and the all-reduce are the library's own.
 * Errors: K outside [1, Kmax], S outside [1, 4096], bad offsets, a pi_init row with a negative or non-finite entry or a zero
 * sum, a pi_init entry > 0 where the current pi_k is 0, min_iters < 0 or max_iters < min_iters -> GMM_ERR_ARG; a sample
 * whose total weight is 0 -> GMM_ERR_ARG (found after the start E-step; the memberships are then valid only when pi_init is
 * NULL); K != the K of the current parameters or a call between gmm_mstep and gmm_constants -> GMM_ERR_STATE; a failed
 * collective -> GMM_ERR_NCCL.
 * Device memory: rho [S][K] floats, the work units (about n_local / E + S), the CTA and sample indices, the partial records
 * ((CTAs + S) x (K + 2) doubles at most) and the masses [S][K + 1] doubles, with pinned mirrors; reserved on first use,
 * grown with S, K and the shard, freed by gmm_destroy.                                                                */
int  gmm_em_multisample(gmm_ctx*, int K, int S, const long long* offsets /* [S+1] global */,
                        const double* pi_init /* [S][K] or NULL */, int min_iters, int max_iters, float epsilon,
                        double* pi_out /* [S][K] or NULL */, double* n_out /* [S] or NULL */,
                        float* loglik_out, float* logliks_out /* [max_iters + 1] or NULL */, int* iters_out);

/* Since the last reset: out[0] reweight and finishing kernels ms (0 with option "profile" = 0), out[1] host ms of the
 * finalisations and the pi / rho updates, out[2] wall ms inside gmm_em_multisample.                                  */
int  gmm_get_multisample_profile(gmm_ctx*, double out[3], int reset);

/* Modal clustering of a fitted mixture (Carreira-Perpinan, TPAMI 2000; Li, Ray and Lindsay, JMLR 2007): the modes of the
 * density p(x) = sum_k pi_k N(x | mu_k, R_k) and the mode each event's hill-climb reaches (its basin of attraction).  A
 * population is a hill of p: several components may cover one hill, and a basin may split a component that straddles two.
 * Parameters: the set the next gmm_estep(ctx, K) would use (float means, Rinv = P, constant, pi of the host copy).
 * Components with pi = 0 take no part.  The host derives, in double, then rounds to float: the centre c = sum_k pi_k mu_k
 * (rounded to float first; every device coordinate is relative to it), mu~_k = mu_k - c, S_k = (P_k + P_k^T) / 2, the
 * logit constant constant_k + ln pi_k and sigma_d = sqrt(sum_k pi_k R_k[d][d]).
 * Iteration (step form of the fixed point; csrc/kernels_modes.cuh, FP32 on sm_90a): for a point x,
 *   dx_k = x - mu~_k,  l_k = const_k - dx_k^T S_k dx_k / 2,  r_k = exp(l_k - ln sum_j exp l_j)  (online log-sum-exp),
 *   g = sum_k r_k S_k (-dx_k)  (the gradient of ln p, formed from each dx_k, in increasing k),
 *   A = sum_k r_k S_k,  delta = A^-1 g by a Cholesky factorisation,  x <- x + delta.
 * This is MEM's x <- A^-1 sum_k r_k S_k mu~_k and keeps its monotone ascent.  A fixed point is g = 0 for any nonsingular
 * A, so A's rounding changes only the speed of convergence, never a mode.  A point stops after the first iteration in
 * which every |delta_d| < max(tol sigma_d, 2^-22 |x_d|), x relative to c before the step (converged): beyond about
 * tol 2^22 spreads from the centre a float coordinate cannot resolve tol sigma_d, and the second term stops a point that
 * has reached the float resolution there instead of letting it hop between neighbouring floats until max_iter; one that has not stopped after max_iter iterations, or whose A is not
 * positive definite in float, is unconverged.  A point with a coordinate that is not finite runs no iteration.
 * Distance: rho(a, b) = max_d |a_d - b_d| / sigma_d.  Each point's arithmetic is fixed: the same bits whatever its CTA,
 * chunk, round or source, and across calls.
 * gmm_modes runs the iteration from every mean mu~_k with pi_k > 0 and deduplicates the endpoints in component order on the
 * host, in double: an endpoint joins the first mode with rho <= merge_tol, else starts a new mode at that endpoint.
 *   n_modes_out    the number of modes found
 *   modes_out      [K][D] the modes in absolute coordinates (c added back in double); the first *n_modes_out rows are set
 *   mode_logp_out  [K] ln p at each mode, in double, or NULL
 *   comp_mode_out  [K] the mode component k reaches; -1 for pi_k = 0 or an unconverged start
 *   is_max_out     [K] 1 when the double-precision Hessian of ln p at the mode is negative definite, or NULL.  A mean can sit
 *                  exactly on a saddle in a symmetric mixture, so this is reported rather than assumed
 *   iters_out      [K] iterations run from each mean (0 for pi_k = 0), or NULL
 * Not collective: every rank computes the same bits.
 * gmm_mode_labels runs the iteration from every event: events_aos [n][D] rows streamed in chunks of option "score_chunk",
 * or events_aos = NULL for the context's own shard (n must equal n_local), read in place from its device copy.
 *   labels       [n] the listed mode of smallest rho <= merge_tol from a converged endpoint, ties to the lower index; -2 for a
 *                converged event near no listed mode; -1 for an unconverged event or one that is not finite
 *   endpoints    [n][D] where each event's ascent stopped (absolute float coordinates: the relative endpoint plus the float
 *                centre, rounded once); NaN for an event that is not finite; or NULL
 *   logp_end     [n] ln p at the endpoint (float; a pass of its own over the records, not the iteration's last value);
 *                NaN for an event that is not finite; or NULL
 *   iters        [n] iterations run, or NULL
 *   unmatched_out / unconverged_out   the counts of labels -2 / -1, or NULL
 * A mixture can have modes that no mean climbs to (three equal isotropic components at the vertices of an equilateral
 * triangle have a fourth mode at the centroid for a range of spreads, Carreira-Perpinan and Williams 2003).  Events in such
 * a basin get -2; their endpoints show where they went (gmm_modes' list plus those endpoints, deduplicated, is a fuller
 * list).  Labelling by component instead: map the -1 entries of comp_mode to any group, then
 * gmm_combine_labels(ctx, K, comp_mode, n_modes, ...) labels each event by the mode of its most likely component.  That
 * differs from the basins where a component straddles two hills, and for events in a basin no mean reaches.
 * tol < 0 selects 1e-5, merge_tol < 0 selects 1e-2.  Weights (gmm_set_weights) are ignored.  Nothing of the EM state
 * changes: memberships, statistics, log-likelihood and every other profile stay as they are.
 * Errors: K outside [1, Kmax], n < 0, max_iter < 1, tol or merge_tol not finite, merge_tol < 10 tol, a mode list that is
 * NULL or has n_modes < 1, NULL shard with n != n_local, a required output NULL -> GMM_ERR_ARG; K != the K of the current
 * parameters, a call between gmm_mstep and gmm_constants, no component with pi > 0, or an S_k that is not positive
 * definite (the first such component is named in the message) -> GMM_ERR_STATE.
 * Device memory: the component records (DP + DP^2 + 4 floats each, DP = D rounded up to a multiple of 4), the mode list,
 * per point of a chunk DP + 4 floats of state, and per slot of two (12 + 4 D) bytes of outputs with a pinned mirror;
 * reserved on first use, grown with the chunk, freed by gmm_destroy.                                                  */
int  gmm_modes(gmm_ctx*, int K, int max_iter, double tol /* <0: 1e-5 */, double merge_tol /* <0: 1e-2 */,
               int* n_modes_out, double* modes_out /* [K][D] */, double* mode_logp_out /* [K] */,
               int* comp_mode_out /* [K] */, int* is_max_out /* [K] */, int* iters_out /* [K] */);
int  gmm_mode_labels(gmm_ctx*, int K, const float* events_aos, long long n,
                     const double* modes /* [n_modes][D] */, int n_modes,
                     int max_iter, double tol, double merge_tol,
                     int* labels, float* endpoints /* [n][D] or NULL */, float* logp_end /* [n] or NULL */,
                     int* iters /* [n] or NULL */, long long* unmatched_out, long long* unconverged_out);

/* Since the last reset: out[0] kernel ms (gmm_modes and gmm_mode_labels), out[1] wall ms in gmm_modes, out[2] wall ms in
 * gmm_mode_labels, out[3] event-iterations run.                                                                          */
int  gmm_get_modes_profile(gmm_ctx*, double out[4], int reset);

/* Per-phase device/host time accumulated since the last reset, in ms
 * (replaces profile_t, gaussian.cu:76-106,967).
 * out[0]=estep out[1]=mstep out[2]=constants(host) out[3]=allreduce
 * out[4]=parameter finalisation + operand upload (host time, or the device
 * kernel's time with option "finalize") out[6]=iterations
 * out[5] / out[7] = M-step launches of the tensor / the SIMT kernel         */
int  gmm_get_profile(gmm_ctx*, double out[8], int reset);

/* Host-side phases of gmm_fit since the last gmm_get_profile(reset=1), in ms:
 * out[0]=order reduction (gaussian.cu:860-907: empties, pair search, merge)
 * out[1]=seeding (:390-452) out[2]=saving the best configuration (:839-851)
 * out[3]=launches of the device-side finalisation since the context was
 * created + 0.001 x the number of host replays (see option "finalize")     */
int  gmm_get_fit_profile(gmm_ctx*, double out[4]);

/* Model-order reduction driver (gaussian.cu:479-960): for K = K0 .. stop:
 * EM, Rissanen score, save-best, drop empty clusters, merge closest pair.
 * `saved` receives the best configuration (memberships [K][n_local] if
 * saved->memberships != NULL).  Returns ideal K and min Rissanen.           */
int  gmm_fit(gmm_ctx*, int K0, int target_K, int min_iters, int max_iters,
             clusters_t* saved, int* ideal_K, float* min_rissanen);

/* ---- host-only numerics (usable without a GPU) --------------------------- */

/* invert_cpu (invert_matrix.cpp:25-101): in-place Crout LU inverse without
 * pivoting.  use_log10 = 1 reproduces invert_cpu's log10(det) (quirk Q3);
 * 0 gives ln det as the device `invert` does (gaussian_kernel.cu:138-140). */
int  gmm_host_invert(float* data, int n, float* log_det, int use_log10);

/* Packed sufficient statistics of K clusters in D dims (doubles), the buffer
 * that is all-reduced once per iteration: K rows of F = 1 + D + D(D+1)/2
 *   [ S0 = sum g | S1_d = sum g (x-shift)_d | S2_ij = sum g (x-shift)_i (x-shift)_j, i>=j row-wise ]
 * followed by one slot for the log-likelihood.  Length = K*F + 1.           */
long long gmm_stats_len(int K, int D);

/* Host M-step finalisation from (already reduced) statistics: the host
 * normalisations of gaussian.cu:611-622,663-679 + mstep_covariance1's
 * N>=1 / avgvar rules (gaussian_kernel.cu:658-675) + constants
 * (gaussian_kernel.cu:172-243).  Updates N, means, R, Rinv, constant, pi.   */
int  gmm_host_finalize(const double* stats, const double* shift, int K, int D,
                       clusters_t* inout);

/* Self-test of the host worker team behind the per-iteration finalisation
 * (`jobs` parallel loops of n items on `threads` threads); 0 = every item
 * ran exactly once per loop.                                                 */
int  gmm_host_pool_selftest(int threads, int jobs, int n);

/* Rissanen / MDL score (gaussian.cu:826) and convergence epsilon (:458).   */
float gmm_host_rissanen(float loglik, int K, int D, long long N);
float gmm_host_epsilon(int D, long long N);

/* One order-reduction step on host parameters (gaussian.cu:860-907 +
 * cluster_distance/add_clusters/copy_cluster :1203-1264): removes clusters
 * with N < 0.5, merges the closest pair, compacts.  *K is updated.
 * Returns the merged pair through c1/c2 (may be NULL).                      */
int  gmm_host_reduce_order(clusters_t* clusters, int* K, int D, int* c1, int* c2);

/* readData (readData.cpp:25-129): "*.bin" = int32 N, int32 D, float32[N*D];
 * anything else = comma-separated text with one header line.  Caller frees
 * with gmm_free().                                                          */
float* gmm_read_data(const char* path, int* ndims, int* nevents);
void   gmm_free(void*);

/* .summary / .results writers (gaussian.cu:998-1061, 1180-1201).            */
int  gmm_write_summary(const char* path, const clusters_t* c, int K, int D);
int  gmm_write_results(const char* path, const float* events_aos, long long N, int D,
                       const clusters_t* c, int K);

/* The reference program: argv = {prog, num_clusters, infile, outfile,
 * [target_num_clusters]} (gaussian.cu:128-1106, 1111-1178).  Same return
 * codes.  Extra options come from the environment (GMM_ITERS, GMM_GPUS,
 * GMM_OUTPUT, GMM_PATH).                                                    */
int  gmm_main(int argc, char** argv);

#ifdef __cplusplus
}
#endif
#endif /* GMM_B200_H */
