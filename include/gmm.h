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
 * failure although nothing is wrong, -1 = never).  Options have to be set
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

/* H2D of N,pi,constant,avgvar,means,R,Rinv (gaussian.cu:446-452, 935-941). */
int  gmm_set_clusters(gmm_ctx*, int K, const clusters_t* host_in);

/* D2H of the parameters, optionally the memberships of THIS shard into
 * host_out->memberships laid out [K][n_local] (gaussian.cu:761-774).       */
int  gmm_get_clusters(gmm_ctx*, int K, clusters_t* host_out, int with_memberships);

/* estep1 + estep2 + likelihood reduction (gaussian_kernel.cu:383-512,
 * gaussian.cu:713-746).  Writes memberships (device), returns the GLOBAL
 * log-likelihood (summed over ranks).                                       */
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
