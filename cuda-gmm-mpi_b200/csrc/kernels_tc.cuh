// kernels_tc.cuh — warpgroup-MMA (wgmma) tensor-core path of the EM hot
// path.  Interface used by gmm_api.cu; implementation in kernels_tc.cu.
#pragma once
#include <cuda_runtime.h>
#include "../../include/gmm.h"

namespace gmm {

struct TcState;

// Shapes the tensor-core kernels cover (independently for the two steps).
bool tc_mstep_supported(int D, int K);
bool tc_estep_supported(int D, int K);

// memb_pitch: row pitch (in floats) of the cluster-major responsibilities buffer AND of the SoA event copy.
int  tc_create(TcState** out, const float* d_x_aos, const float* d_x_soa, int n, int D, int Kmax, float* d_memb, size_t memb_pitch,
               int num_sms, cudaStream_t stream);
void tc_destroy(TcState*);
void tc_set_host_threads(TcState*, int n);
// Centre/scale used inside the tensor kernels: z = (x - shift) * inv_scale, both rounded to
// float; `shift` is updated in place to the float-rounded values actually used.  xmin / xmax: per-dimension extremes
// of the WHOLE data set (all ranks): they fix the power-of-two quanta of the M-step's fixed-point operand parts.
int  tc_set_shift_scale(TcState*, double* shift, const double* scale, const double* xmin, const double* xmax, cudaStream_t stream);
// True once the quanta are set and the data range fits the fixed-point budget (|z| <= 64 global standard deviations);
// otherwise the caller uses the FP64 SIMT M-step.
bool tc_mstep_ready(const TcState*);
// False when an event lies beyond 2^14 global standard deviations (its standardised coordinates would overflow FP16).
bool tc_estep_range_ok(const TcState*);
int  tc_upload_params(TcState*, const clusters_t* host, int K, cudaStream_t stream);
// The same in three steps, so that the caller can fuse the per-cluster work with its own per-cluster
// finalisation in ONE parallel loop: begin (serial), cluster k in [0, tc_params_padded) (independent, thread
// safe; returns 0 or a defect code to be max-reduced), commit (serial: error report or H2D of the operand).
int  tc_params_begin(TcState*, int K, cudaStream_t stream);
int  tc_params_padded(const TcState*, int K);
int  tc_params_cluster(TcState*, const clusters_t* host, int k, int K);
// The same with the upper-triangular factor W (Rinv = W^T W, double, row-major [D][D]) supplied by the caller
// (constants_cluster_spd): no second factorisation of the inverse.
int  tc_params_cluster_w(TcState*, const clusters_t* host, int k, int K, const double* W);
int  tc_params_commit(TcState*, int K, int bad, cudaStream_t stream);
// d_w (optional): per-event weights of the shard ([n] floats): the log-likelihood adds w * denominator (gmm_set_weights).
int  tc_launch_estep(TcState*, int K, double* d_ll, cudaStream_t stream, const float* d_w = nullptr);
// Scoring of a chunk of new events ([n][D] on the device) against the resident operand of the current parameters
// (score_tc_kernel): labels / max_resp / logp per event, ll += sum of logp, *flag = 1 when an event is outside the FP16
// operand range.  run_*: per-event running state of the passes, n entries each (needed for K > 64 only).
struct TcScoreIo {
    const float* x;
    int n;
    int* labels;
    float* max_resp;
    float* logp;
    double* ll;
    int* flag;
    float* run_den;
    float* run_bl;
    int* run_bk;
};
int  tc_launch_score(TcState*, int K, const TcScoreIo& io, cudaStream_t stream);
// Device-side M-step finalisation: reduced statistics -> parameter set `d_set` (floats, tc_param_set_floats(); arrays at
// tc_param_set_off(which = 0 N, 1 pi, 2 constant, 3 means, 4 R, 5 Rinv), stride Kmax) + the E-step operand, no host round
// trip.  d_ll[0] receives the log-likelihood slot of the statistics.  d_bad[0] = first iteration (`iter`) that met a cluster
// the host path must handle (-1: none; later launches then return immediately), d_bad[1] = its code (1 not positive
// definite, 2 outside FP16, 4 statistics not finite).
bool tc_finalize_supported(const TcState*, int K);
size_t tc_param_set_floats(int Kmax, int D);
size_t tc_param_set_off(int Kmax, int D, int which);
// fault_iter: the launch with iter == fault_iter reports code 1 although nothing is wrong (-1: never; test hook).
int  tc_launch_finalize(TcState*, int K, const double* d_stats, const float* d_avgvar, float* d_set, double* d_ll, int* d_bad, int iter,
                        int fault_iter, cudaStream_t stream);
// Accumulates sum_n g[k][n] * phi_f(x_n - shift) into d_stats[k*F + f] (double, original units).
// d_w (optional): per-event weights of the shard ([memb_pitch] floats, zero beyond n), wscale = the largest of them: the
// sums are of w g phi.
int  tc_launch_mstep(TcState*, int K, double* d_stats, cudaStream_t stream, const float* d_w = nullptr, double wscale = 1.0);

// The same two steps on caller-owned buffers (gmm_score_stats: chunks of new events, nothing of the state's buffers is
// written except the M-step's per-launch scratch).  pitch: row pitch in floats of memb (and of z), a multiple of 32.
//   estep: events [n][D] (device, AoS) -> memb [8 * ceil(K / 8)][pitch]; den: [n] floats of running log-denominator
//          (K > 64 only); *d_ll += sum of the events' log-denominators.
//   mstep: standardised SoA copy z [D][pitch] (tc_shift_f / tc_inv_scale_f) and memb [>= Kmax rows][pitch] of n events;
//          adds into d_stats[0 .. K*F).  The tensor maps are encoded with n as their event extent (TMA's zero fill masks
//          the tail), re-encoded only when the buffers or n change.
int  tc_launch_estep_on(TcState*, int K, const float* d_x_aos, int n, float* d_memb, size_t pitch, float* d_den, double* d_ll,
                        cudaStream_t stream);
int  tc_launch_mstep_on(TcState*, int K, const float* d_z, const float* d_memb, size_t pitch, int n, double* d_stats, cudaStream_t stream);
// Device copies of the float centre and inverse scale the tensor kernels use (NULL before tc_set_shift_scale), and the
// power-of-two bound zb of |z| the M-step's fixed-point quanta were set from (max over the dimensions).
const float* tc_shift_f(const TcState*);
const float* tc_inv_scale_f(const TcState*);
float tc_mstep_zbound(const TcState*);

}  // namespace gmm
