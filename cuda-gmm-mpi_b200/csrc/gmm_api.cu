// gmm_api.cu — the C ABI of include/gmm.h: context, operators, EM loop,
// model-order reduction.  Host orchestration in C++, compute in the CUDA
// kernels of kernels_simt.cuh / kernels_tc.cuh, cross-GPU reduction with one
// ncclAllReduce of the packed sufficient statistics per iteration.
//
// Reference being replaced: gaussian.cu:289-960 (the OpenMP-thread-per-GPU body
// of main()).  There is no CPU fallback: every compute entry point needs a
// CUDA device of compute capability 10.x.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <fcntl.h>
#include <unistd.h>
#include <nccl.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <memory>
#include <string>
#include <thread>
#include <vector>

#include "../../include/gmm.h"
#include "cuda_owned.h"
#include "host_math.h"
#include "kernels_simt.cuh"
#include "kernels_condition.cuh"
#include "kernels_sample.cuh"
#include "kernels_seed.cuh"
#include "kernels_tc.cuh"
#include "kernels_vb.cuh"
#include "kernels_combine.cuh"

namespace gmm {

// ---- NCCL, loaded lazily so that the library imports without it -----------
struct NcclApi {
    void* handle = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    bool ok = false;
};
static NcclApi& nccl() {
    static NcclApi api;
    static bool tried = false;
    if (!tried) {
        tried = true;
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* nm : names) {
            api.handle = dlopen(nm, RTLD_NOW | RTLD_GLOBAL);
            if (api.handle) break;
        }
        if (api.handle) {
            api.GetUniqueId = (decltype(api.GetUniqueId))dlsym(api.handle, "ncclGetUniqueId");
            api.CommInitRank = (decltype(api.CommInitRank))dlsym(api.handle, "ncclCommInitRank");
            api.AllReduce = (decltype(api.AllReduce))dlsym(api.handle, "ncclAllReduce");
            api.AllGather = (decltype(api.AllGather))dlsym(api.handle, "ncclAllGather");
            api.CommDestroy = (decltype(api.CommDestroy))dlsym(api.handle, "ncclCommDestroy");
            api.GetErrorString = (decltype(api.GetErrorString))dlsym(api.handle, "ncclGetErrorString");
            api.ok = api.GetUniqueId && api.CommInitRank && api.AllReduce && api.AllGather && api.CommDestroy && api.GetErrorString;
        }
    }
    return api;
}
#define NCCL_TRY(expr)                                                                         \
    do {                                                                                       \
        ncclResult_t r_ = (expr);                                                              \
        if (r_ != ncclSuccess)                                                                 \
            return fail(GMM_ERR_NCCL, std::string(#expr) + ": " + nccl().GetErrorString(r_));  \
    } while (0)

struct PhaseTimer {          // replaces cudaTimer_t / profile_t (gaussian.cu:33-106)
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pending;
    double total_ms = 0;
};
// Timing events are recycled: cudaEventCreate / Destroy cost microseconds each and sat inside the EM loop.  The pool owns
// every event it made, lent or not.
struct EventPool {
    std::vector<Event> owned;
    std::vector<cudaEvent_t> free_list;
    cudaEvent_t get() {
        if (!free_list.empty()) { cudaEvent_t e = free_list.back(); free_list.pop_back(); return e; }
        Event e;
        if (e.create(cudaEventDefault) != GMM_OK) return nullptr;
        owned.push_back(std::move(e));
        return owned.back();
    }
    void put(cudaEvent_t e) { if (e) free_list.push_back(e); }
};

// Persistent worker team for the per-iteration host finalisation (K independent clusters, a few microseconds each).
// The workers SPIN on a generation counter for a few milliseconds after each job — an EM iteration hands them the
// next one within that window — and only then block on a condition variable.  An OpenMP parallel region costs a
// futex wake-up per thread and iteration when the runtime's wait policy is passive (torchrun exports OMP_NUM_THREADS=1
// and the measured finalisation went from 0.05 ms to 0.33 ms per iteration at 2 ranks).
class HostPool {
public:
    explicit HostPool(int nthreads) { resize(nthreads); }
    ~HostPool() { stop(); }
    int size() const { return (int)workers_.size() + 1; }
    void resize(int nthreads) {
        if (nthreads < 1) nthreads = 1;
        if (nthreads == size() && started_) return;
        stop();
        quit_.store(false);
        started_ = true;
        for (int i = 1; i < nthreads; i++) workers_.emplace_back([this] { worker(); });
    }
    // fn(i) for i in [0, n), spread dynamically over the team (the caller takes part); returns when all are done
    void run(int n, const std::function<void(int)>& fn) {
        if (n <= 0) return;
        if (workers_.empty() || n == 1) { for (int i = 0; i < n; i++) fn(i); return; }
        // Items are claimed by counting `remaining_` DOWN: a claim is valid iff the value it saw was positive, so a worker
        // still on its way out of the previous job's loop either sees <= 0 (before the store below) or a genuine item of
        // THIS job (after it) — there is no window in which a stale claim can be mistaken for a new one (an index
        // counted up against a separately published bound had one: found by gmm_host_pool_selftest).  Everything a
        // claimer reads is published before the store (release / acquire on `remaining_`).
        fn_ = &fn; n_ = n;
        done_.store(0, std::memory_order_relaxed);
        remaining_.store(n, std::memory_order_release);
        {
            std::lock_guard<std::mutex> lk(m_);
            gen_.fetch_add(1, std::memory_order_release);
        }
        cv_.notify_all();
        work();
        while (done_.load(std::memory_order_acquire) < n_) cpu_relax();
    }
private:
    static void cpu_relax() {
#if defined(__x86_64__) || defined(__i386__)
        __builtin_ia32_pause();
#endif
    }
    void work() {
        for (;;) {
            const int r = remaining_.fetch_sub(1, std::memory_order_acq_rel);
            if (r <= 0) break;
            (*fn_)(r - 1);
            done_.fetch_add(1, std::memory_order_release);
        }
    }
    void worker() {
        unsigned long long seen = gen_.load(std::memory_order_acquire);
        for (;;) {
            // spin for up to ~4 ms, then sleep
            const auto t0 = std::chrono::steady_clock::now();
            unsigned long long g;
            int spins = 0;
            while ((g = gen_.load(std::memory_order_acquire)) == seen && !quit_.load(std::memory_order_relaxed)) {
                cpu_relax();
                if ((++spins & 1023) == 0 && std::chrono::steady_clock::now() - t0 > std::chrono::milliseconds(4)) {
                    std::unique_lock<std::mutex> lk(m_);
                    cv_.wait(lk, [&] { return gen_.load(std::memory_order_acquire) != seen || quit_.load(); });
                }
            }
            if (quit_.load()) return;
            seen = g;
            work();
        }
    }
    void stop() {
        if (!started_) return;
        {
            std::lock_guard<std::mutex> lk(m_);
            quit_.store(true);
        }
        cv_.notify_all();
        for (auto& t : workers_) t.join();
        workers_.clear();
        started_ = false;
    }
    std::vector<std::thread> workers_;
    std::mutex m_;
    std::condition_variable cv_;
    std::atomic<unsigned long long> gen_{0};
    std::atomic<int> remaining_{0}, done_{0};
    std::atomic<bool> quit_{false};
    const std::function<void(int)>* fn_ = nullptr;
    int n_ = 0;
    bool started_ = false;
};

// ---------------------------------------------------------------------------------------------------------------
// All-reduce of the packed statistics over NVLink peer memory (one box, <= 8 GPUs): replaces the per-iteration
// ncclAllReduce (and with it the four MPI_Allreduce of gaussian.cu:566,605,658,741) by ONE kernel of this library.
// Every rank owns an exchange area [2 parities][len doubles] + flags, mapped into every other rank (cudaIpc between
// processes, peer access between the threads of one process; NCCL only carries the 100-byte handles once, at
// gmm_comm_init).  Per call and CTA: copy the CTA's chunk of the local statistics into the own area, fence, raise
// the chunk's flag in every peer (posted remote writes), wait for the G flags of the chunk in LOCAL memory, then sum
// the chunk over the ranks' areas in rank order (remote loads) — the same order on every rank, so the replicated host
// finalisation sees bit-identical statistics.  Two parities: a rank can be at most one call ahead of the slowest one.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kXMaxRanks = 8;
constexpr int kXCtas = 24;                      // chunks of the vector, one CTA each (flags per chunk: no grid barrier)
struct PeerTable {
    double* buf[kXMaxRanks];                    // exchange area of rank p as mapped HERE: [2][cap] doubles
    unsigned long long* flags[kXMaxRanks];      // flags of rank p as mapped here: [2][kXMaxRanks][kXCtas]
    int nranks, rank;
    size_t cap;
};
struct PeerExchange {
    PeerTable tab{};
    DeviceArray<char> base;                     // own allocation: [2][cap] doubles, then the flags
    void* opened[kXMaxRanks] = {nullptr};       // cudaIpcOpenMemHandle results to close
    unsigned long long epoch = 0;
    bool ok = false;
};
struct PeerHello {                              // what every rank tells the others (carried by ncclAllGather once)
    cudaIpcMemHandle_t handle;
    unsigned long long ptr;
    long long pid;
    int device, ok;
    int dev_fin, pad;                           // this rank can finalise on the device (it has events and the buffers)
};

__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ double ld_relaxed_sys(const double* p) {
    double v;
    asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
    return v;
}

__global__ void __launch_bounds__(1024)
allreduce_peer_kernel(PeerTable t, double* __restrict__ stats, int len, int parity, unsigned long long epoch) {
    const int per = (len + kXCtas - 1) / kXCtas;
    const int i0 = blockIdx.x * per, i1 = min(len, i0 + per);
    double* mine = t.buf[t.rank] + (size_t)parity * t.cap;
    for (int i = i0 + threadIdx.x; i < i1; i += blockDim.x) mine[i] = stats[i];
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < t.nranks)                  // tell rank threadIdx.x that this chunk of rank t.rank is in place
        st_release_sys(t.flags[threadIdx.x] + ((size_t)parity * kXMaxRanks + t.rank) * kXCtas + blockIdx.x, epoch);
    __shared__ int timed_out;
    if (threadIdx.x == 0) timed_out = 0;
    __syncthreads();
    if (threadIdx.x < t.nranks) {
        const unsigned long long* f = t.flags[t.rank] + ((size_t)parity * kXMaxRanks + threadIdx.x) * kXCtas + blockIdx.x;
        const long long t0 = clock64();
        while (ld_acquire_sys(f) < epoch) {
            __nanosleep(20);
            if (clock64() - t0 > 20000000000LL) { timed_out = 1; break; }      // ~10 s: a peer is gone; do not hang the GPU
        }
    }
    __syncthreads();
    for (int i = i0 + threadIdx.x; i < i1; i += blockDim.x) {
        double s = 0.0;
        for (int p = 0; p < t.nranks; p++) s += ld_relaxed_sys(t.buf[p] + (size_t)parity * t.cap + i);
        stats[i] = timed_out ? __longlong_as_double(0x7ff8000000000000LL) : s;   // NaN: the host reports the failure
    }
}

// gmm_score's own buffers (nothing of the EM state is touched): per slot s of two, a pinned input stage and a device
// chunk of events, device outputs and their pinned mirror laid out [ll double | flag int | pad][labels][max_resp][logp],
// plus the running state of the tensor kernel's passes (K > 64).
struct ScoreBuffers {
    long long cap = 0;                          // events per chunk
    PinnedArray<float> h_in[2];
    DeviceArray<float> d_in[2];
    DeviceArray<char> d_out[2];
    PinnedArray<char> h_out[2];
    DeviceArray<float> d_run_den;
    DeviceArray<float> d_run_bl;
    DeviceArray<int> d_run_bk;
    Stream copy;                                // H2D of the next chunk / D2H of the last one, beside the kernels
    Event h2d[2], kern[2], d2h[2];
    Event t0[2], t1[2];
    double kernel_ms = 0, wall_ms = 0;          // gmm_get_score_profile
    long long tensor_chunks = 0, simt_chunks = 0;
    static constexpr size_t kHeader = 16;
    static size_t out_bytes(long long cap) { return kHeader + (size_t)cap * 12; }
};

// Time and kernel counts of the calls that stream E- and M-steps over chunks (gmm_get_score_stats_profile,
// gmm_get_condition_stats_profile).
struct StatsProfile {
    double kernel_ms = 0, wall_ms = 0, wait_ms = 0;
    long long e_tensor = 0, e_simt = 0, m_tensor = 0, m_simt = 0;
};

// gmm_score_stats' own buffers (its input stage is gmm_score's two pinned slots and device chunks): ONE compute-side chunk
// (the kernels of consecutive chunks are serialised on the compute stream), the statistics it adds up, the range flag and,
// on the first call that asks for memberships, their pinned mirror.  gmm_condition_stats uses the same buffers, plus its
// observed copy (allocated on its first call) and the float centre.
struct ScoreStatsBuffers {
    long long cap = 0;                          // events per chunk
    size_t pitch = 0;                           // row pitch in floats of the SoA copies and the responsibilities (multiple of 32)
    DeviceArray<float> d_z;                     // [D][pitch] standardised SoA copy (tensor M-step)
    DeviceArray<float> d_xs;                    // [D][pitch] raw SoA copy (SIMT kernels)
    DeviceArray<float> d_xo;                    // [D][pitch] observed SoA copy of gmm_condition_stats (its n_obs rows)
    DeviceArray<float> d_shift_f;               // [GMM_MAX_DIMENSIONS] the centre in float (gmm_condition_stats' missing rows)
    DeviceArray<float> d_memb;                  // [8 ceil(Kmax / 8)][pitch] responsibilities of the chunk
    PinnedArray<float> h_memb;                  // [Kmax][cap]
    DeviceArray<double> d_stats;                // [Kmax F + 1]
    PinnedArray<double> h_stats;
    DeviceArray<int> d_flag;
    PinnedArray<int> h_flag;
    Event ev_flag;
    Event p0[2], p1[2], k0[2], k1[2];
    StatsProfile prof;                          // gmm_get_score_stats_profile
    StatsProfile cond_prof;                     // gmm_get_condition_stats_profile
};

// gmm_seed_kmeans' buffers, allocated on its first call (the shard's size is fixed; the transfer slots follow the rank count).
struct KmeansBuffers {
    int nb = 0, nba = 0;                        // blocks of the k-means++ kernels / of the assignment
    DeviceArray<double> d_d2;                   // [n] squared distance to the nearest chosen centre
    DeviceArray<int> d_labels;                  // [n] Lloyd labels
    DeviceArray<double> d_bsum;                 // [nb] per-block sums of d2
    DeviceArray<double> d_bpot;                 // [nb][kSeedMaxCand] per-block candidate potentials
    DeviceArray<int> d_bchanged;                // [nba] changed labels per assignment block
    DeviceArray<double> d_binertia;             // [nba] distances per assignment block
    DeviceArray<float> d_cand;                  // [kSeedMaxCand][D] candidate rows
    DeviceArray<SeedPick> d_pick;               // [kSeedMaxCand]
    DeviceArray<int> d_pick_idx;                // [kSeedMaxCand]
    DeviceArray<float> d_centres;               // [Kmax][D]
    DeviceArray<double> d_xfer;                 // [nranks][16] zero-padded per-rank values
    PinnedArray<double> h_bsum;                 // pinned mirrors
    PinnedArray<double> h_bpot;
    PinnedArray<int> h_bchanged;
    PinnedArray<double> h_binertia;
    PinnedArray<SeedPick> h_pick;
    PinnedArray<double> h_xfer;
};

// gmm_sample's parameter block (kernels_sample.cuh layout, sized for Kmax) and its pinned staging, allocated on the first
// call.  Its chunks stream through gmm_score's slots.
struct SampleBuffers {
    DeviceArray<double> d_block;
    PinnedArray<char> h_block;
    double kernel_ms = 0, wall_ms = 0;          // gmm_get_sample_profile
};

// gmm_condition's parameter block (sized for Kmax and the largest record any observed set of this D needs) and its
// pinned mirror, allocated on the first call; per slot of gmm_score's two, the imputations of a chunk (device and pinned:
// cond_mean [chunk][NM] then cond_var [chunk][NM]), allocated on the first imputing call and grown with chunk x NM, never
// shrunk.  Its chunks stream through gmm_score's slots.
struct ConditionBuffers {
    DeviceArray<float> d_block;
    PinnedArray<float> h_block;
    DeviceArray<float> d_imp[2];
    PinnedArray<float> h_imp[2];
    double kernel_ms = 0, wall_ms = 0;          // gmm_get_condition_profile
};

// gmm_combine / gmm_combine_labels: per-(range, value) partials of the passes, their reduced sums and pinned mirror (sized
// for the largest pass seen), the live groups' member lists, and the labels' device outputs; allocated on first use.
struct CombineBuffers {
    DeviceArray<double> d_part;
    DeviceArray<double> d_sum;
    PinnedArray<double> h_sum;
    DeviceArray<int> d_groups;                  // [2 kCombMaxK + 1]: members, then offsets
    PinnedArray<int> h_groups;
    DeviceArray<int> d_lab;                     // [memb_pitch]
    DeviceArray<float> d_max;                   // [memb_pitch]
    Event t0, t1;
    double kernel_ms = 0, wall_ms = 0, labels_wall_ms = 0;   // gmm_get_combine_profile
};

}  // namespace gmm

using namespace gmm;

struct gmm_ctx {
    Stream stream;               // first member: destroyed last, after every buffer and event its work may use
    int device = 0, n = 0, D = 0, Kmax = 0, F = 0;
    long long n_global = 0, offset = 0;
    int num_sms = 132;
    // events
    DeviceArray<float> d_x_aos;  // [n][D]  as supplied (TMA source of the tensor path)
    DeviceArray<float> d_x_soa;  // [D][n]  transpose for the SIMT kernels
    // responsibilities, cluster-major [Kmax][n]
    DeviceArray<float> d_memb;
    size_t memb_pitch = 0;           // row pitch in floats (multiple of 32: TMA-aligned rows)
    DeviceArray<float> d_memb_saved; // best configuration during gmm_fit
    Event ev_stats;                  // statistics have reached the host
    // parameters
    DeviceArray<float> d_epack;  // SIMT E-step parameters [Kmax][epack_stride]
    PinnedArray<float> h_epack;  // staging
    DeviceArray<double> d_stats; // [Kmax*F + 1]
    PinnedArray<double> h_stats;
    DeviceArray<double> d_shift; // [32]
    double shift[GMM_MAX_DIMENSIONS] = {0};
    bool have_shift = false;
    double scale[GMM_MAX_DIMENSIONS] = {0};   // global per-dimension standard deviation
    double sum_x[GMM_MAX_DIMENSIONS] = {0}, sum_x2[GMM_MAX_DIMENSIONS] = {0};
    // host copy of the current parameters (all arrays sized for Kmax)
    std::vector<float> hN, hpi, hconst, havgvar, hmeans, hR, hRinv;
    clusters_t host{};
    int cur_K = 0;
    bool memb_valid = false;     // d_memb holds the responsibilities of the current parameters
    int stats_clean_K = 0;       // d_stats[0 .. K*F) is known to be zero for this K (0 = not known)
    // communication
    ncclComm_t comm = nullptr;
    int rank = 0, nranks = 1;
    // options
    int path = GMM_PATH_AUTO;
    int estep_path = -1, mstep_path = -1;   // per-step override of `path` (options "estep_path" / "mstep_path"; -1 = follow `path`)
    int verbose = 0;
    int host_threads = 1;
    bool host_threads_fixed = false; // set by GMM_HOST_THREADS / gmm_set_option: not re-derived from the rank count
    // profile
    PhaseTimer t_estep, t_mstep, t_reduce, t_fused;
    EventPool events;
    bool profile_phases = true;  // per-phase CUDA-event timers inside the EM loop (option "profile")
    double host_const_ms = 0, memcpy_ms = 0;
    double fit_reduce_ms = 0, fit_seed_ms = 0, fit_save_ms = 0;   // gmm_fit phases (gmm_get_fit_profile)
    long long mstep_tensor = 0, mstep_simt = 0;                   // M-step launches by kernel
    long long iterations = 0;
    std::unique_ptr<TcState, TcStateDelete> tc;   // tensor-core path state (kernels_tc.cuh)
    std::unique_ptr<HostPool> pool;              // worker team of the per-iteration host finalisation (created on first use)
    PeerExchange xchg;           // peer-memory all-reduce of the statistics (gmm_comm_init; falls back to NCCL)
    int allreduce_mode = 1;      // option "allreduce": 1 = peer-memory kernel when available, 0 = ncclAllReduce
    bool estep_tensor_ready = false;   // the tensor E-step operand of the current parameters is uploaded
    // device-side finalisation (kernels_tc.cu: finalize_params_kernel): EM iterations without a host round trip
    int finalize_mode = 1;       // option "finalize": 1 = on the device when the tensor E-step serves the state, 0 = host
    bool dev_fin_failed = false; // a cluster needed the host path once: this context stays on it
    bool dev_fin_agreed = true;  // every rank of the communicator can (gmm_comm_init): the replay re-issues collectives
    DeviceArray<float> d_pset[2];   // parameter sets written by the kernel (iteration parity)
    PinnedArray<float> h_pset;   // staging of one set
    DeviceArray<float> d_avgvar; // [Kmax]
    DeviceArray<int> d_bad;      // [2] first failed iteration (-1), code
    DeviceArray<double> d_llprev;   // [2] log-likelihood slot seen by the finalisation of iteration parity
    PinnedArray<char> h_small;   // int bad[2] | double ll[2] | float avgvar[Kmax]
    PhaseTimer t_final;
    long long dev_finalize_launches = 0, dev_replays = 0;
    int fin_fault_iter = -1;     // option "finalize_fault_iter" (tests): that iteration of the next batch reports a failure
    bool params_partial = false; // gmm_mstep has updated N, means, R but not yet Rinv / constants / the operand (upload_params clears)
    bool set_from_finalize = false;  // the host copy came from a finalisation (device or host): Rinv, constant, pi and the
                                     // E-step operand were derived from R, not given (seed, gmm_set_clusters, order reduction)
    ScoreBuffers score;          // gmm_score: streaming buffers, allocated on first use
    long long score_chunk = 1 << 20;   // option "score_chunk": events per streamed chunk of gmm_score / gmm_score_stats
    ScoreStatsBuffers sstats;    // gmm_score_stats: chunk buffers, allocated on first use
    KmeansBuffers kmeans;        // gmm_seed_kmeans: allocated on first use
    SampleBuffers sample;        // gmm_sample: parameter block, allocated on first use
    ConditionBuffers cond;       // gmm_condition: parameter block and imputation buffers, allocated on first use
    // gmm_set_weights: per-event weights of the shard, used by the E-step log-likelihood and the M-step statistics
    DeviceArray<float> d_w;      // [memb_pitch], zero beyond n (allocated on the first call)
    bool weighted = false;       // d_w is in effect
    double w_total = 0;          // global sum of the weights (the N of the default epsilon and of the Rissanen score)
    double w_scale = 1;          // the global largest weight (the tensor M-step divides the weights by it)
    bool w_tensor_ok = true;     // the weights' dynamic range fits the tensor M-step (kWeightRangeTc)
    bool seeding = false;        // gmm_seed_kmeans: its M-steps ignore the weights
    // gmm_vb_em: block partials of the responsibility entropy (resp_entropy_kernel), allocated on first use
    DeviceArray<double> d_ent;   // [ent_blocks + 1]: the partials, then the rank's sum for the all-reduce
    PinnedArray<double> h_ent;
    int ent_blocks = 0;
    PhaseTimer t_entropy;
    double vb_final_ms = 0, vb_wall_ms = 0;   // gmm_get_vb_profile
    CombineBuffers comb;         // gmm_combine / gmm_combine_labels: allocated on first use
};

namespace gmm {

static void timer_begin(gmm_ctx* c, PhaseTimer& t) {
    if (!c->profile_phases) return;
    cudaEvent_t a = c->events.get(), b = c->events.get();
    cudaEventRecord(a, c->stream);
    t.pending.push_back({a, b});
}
static void timer_end(gmm_ctx* c, PhaseTimer& t) {
    if (!c->profile_phases || t.pending.empty()) return;
    cudaEventRecord(t.pending.back().second, c->stream);
}
static void timer_collect(gmm_ctx* c, PhaseTimer& t) {          // call after a stream sync
    for (auto& p : t.pending) {
        float ms = 0;
        if (cudaEventElapsedTime(&ms, p.first, p.second) == cudaSuccess) t.total_ms += ms;
        c->events.put(p.first); c->events.put(p.second);
    }
    t.pending.clear();
}
static void collect_all(gmm_ctx* c) {
    timer_collect(c, c->t_estep); timer_collect(c, c->t_mstep); timer_collect(c, c->t_reduce); timer_collect(c, c->t_fused);
    timer_collect(c, c->t_final); timer_collect(c, c->t_entropy);
}

static void bind_host(gmm_ctx* c) {
    c->host.N = c->hN.data(); c->host.pi = c->hpi.data(); c->host.constant = c->hconst.data();
    c->host.avgvar = c->havgvar.data(); c->host.means = c->hmeans.data(); c->host.R = c->hR.data();
    c->host.Rinv = c->hRinv.data(); c->host.memberships = nullptr;
}

static void copy_params(clusters_t* dst, const clusters_t* src, int K, int D) {
    std::memcpy(dst->N, src->N, sizeof(float) * K);
    std::memcpy(dst->pi, src->pi, sizeof(float) * K);
    std::memcpy(dst->constant, src->constant, sizeof(float) * K);
    std::memcpy(dst->avgvar, src->avgvar, sizeof(float) * K);
    std::memcpy(dst->means, src->means, sizeof(float) * (size_t)K * D);
    std::memcpy(dst->R, src->R, sizeof(float) * (size_t)K * D * D);
    std::memcpy(dst->Rinv, src->Rinv, sizeof(float) * (size_t)K * D * D);
}

// Threads of the replicated host finalisation (K independent D x D inversions + factorizations, ~5 us each): at most
// 16 (beyond that the fork/join costs more than it saves) and at most HALF of this rank's share of the hardware
// threads — with every hardware thread of the box claimed by spinning OpenMP teams (8 ranks x 16 on 128) the
// NCCL proxy threads starve: measured 3.4 ms per all-reduce and 1.8 ms per finalisation instead of 0.05 / 0.1 ms.
static int default_host_threads(int ranks_on_box) {
    const int hw = (int)std::thread::hardware_concurrency();
    int t = hw > 0 ? hw / (2 * (ranks_on_box > 0 ? ranks_on_box : 1)) : 8;
    if (t > 16) t = 16;
    if (t < 1) t = 1;
    return t;
}

static int estep_path_of(const gmm_ctx* c) { return c->estep_path >= 0 ? c->estep_path : c->path; }
static int mstep_path_of(const gmm_ctx* c) { return c->mstep_path >= 0 ? c->mstep_path : c->path; }
static bool use_tensor_estep(const gmm_ctx* c, int K) { return estep_path_of(c) != GMM_PATH_SIMT && c->n > 0 && tc_estep_supported(c->D, K); }
// Weights of the shard for the E- and M-step kernels (NULL: unit weights; seeding ignores them).
static const float* step_weights(const gmm_ctx* c) { return c->weighted && !c->seeding ? c->d_w.get() : nullptr; }
// Largest dynamic range max w / min positive w of the weights that the tensor M-step serves.  A weight whose scaled value
// is not 1 moves a whole group of confident events off the points the operand's fixed-point part holds exactly, and their
// common FP16 rounding then biases the statistics: the CPU emulation (tests/test_weights_error_model.py, DESIGN §5.11)
// leaves a quarter of the per-cluster bar with two values 1 and 1.4 at the widest legal data range.  So the tensor M-step
// serves one positive value (a constant factor, zeros allowed); any other weights are served by the FP64 SIMT M-step.
// Only the steps of the context's own shard read the weights (run_mstep_accumulate); gmm_score_stats and
// gmm_condition_stats choose their M-step without them.
constexpr double kWeightRangeTc = 1.0;
// (the tensor M-step also needs the data range to fit its fixed-point operand budget: known once the moments are)
static bool use_tensor_mstep(const gmm_ctx* c, int K) {
    return mstep_path_of(c) != GMM_PATH_SIMT && c->n > 0 && tc_mstep_supported(c->D, K) && (!c->have_shift || tc_mstep_ready(c->tc.get()));
}
// N of the default epsilon and of the Rissanen score: the number of events, or the sum of the weights
static double em_count(const gmm_ctx* c) { return c->weighted ? c->w_total : (double)c->n_global; }
// GMM_PATH_TENSOR never degrades silently: the M-step (the covariance contraction) must be covered.
static int check_path(const gmm_ctx* c, int K) {
    if (mstep_path_of(c) == GMM_PATH_TENSOR && !tc_mstep_supported(c->D, K))
        return fail(GMM_ERR_ARG, "GMM_PATH_TENSOR requested but the wgmma kernels do not cover this (D, K)");
    if (mstep_path_of(c) == GMM_PATH_TENSOR && c->n > 0 && c->have_shift && !tc_mstep_ready(c->tc.get()))
        return fail(GMM_ERR_ARG, "GMM_PATH_TENSOR requested but the data range (outliers beyond 64 standard deviations) exceeds the "
                                 "tensor M-step's fixed-point operand budget");
    return GMM_OK;
}

static int ensure_moments(gmm_ctx* c);
// Doubles of d_stats / h_stats: the packed statistics and the log-likelihood slot, and at least the 4 D column moments
// that ensure_moments stages there (more than K F + 1 at Kmax = 1 and D = 2 or 3)
static size_t stats_capacity(const gmm_ctx* c) { return std::max((size_t)c->Kmax * c->F + 1, 4 * (size_t)c->D); }

// The worker team of the host finalisation, created on first use and resized to the context's host_threads.
static HostPool* host_pool(gmm_ctx* c) {
    if (!c->pool) c->pool.reset(new HostPool(c->host_threads));
    else c->pool->resize(c->host_threads);
    return c->pool.get();
}

// fn(i) for i in [0, n), the items of a loop over K clusters: on the worker team when K >= 8, serially below.
static void run_clusters(gmm_ctx* c, int K, int n, const std::function<void(int)>& fn) {
    if (K >= 8) host_pool(c)->run(n, fn);
    else for (int i = 0; i < n; i++) fn(i);
}

// Upload the current host parameters in the form the E-step kernels consume
// (gaussian.cu:446-452 / 935-941 upload the seven raw arrays; here the E-step
// operand is pre-packed on the host once per iteration).
// with_constants: the inverse / constant / pi of every cluster still have to be derived from R (M-step
// finalisation).  On the tensor path that work shares ONE parallel loop over the clusters with the E-step
// operand (Cholesky + FP16 split): one thread-team wake-up per EM iteration instead of two.
static int upload_params(gmm_ctx* c, int K, bool with_constants = false, bool with_finalize = false) {
    if (int rc = check_path(c, K)) return rc;
    auto t0 = std::chrono::steady_clock::now();
    const bool from_outside = !with_finalize;          // seed / set_clusters / order reduction: avgvar may have changed
    const bool from_R = with_constants;                // (with_constants is cleared below once the loop has done that work)
    c->estep_tensor_ready = false;
    if (use_tensor_estep(c, K)) {
        if (int rc = ensure_moments(c)) return rc;
        // events further than 2^14 global standard deviations from the centre would overflow the FP16 event operand
        int rc = tc_estep_range_ok(c->tc.get()) ? tc_params_begin(c->tc.get(), K, c->stream)
                                          : fail(GMM_ERR_STATE, "tensor E-step: the data range exceeds the FP16 event operand");
        if (rc == GMM_OK) {
            if (with_finalize)                     // pi needs every N[k] = (float)S0 before the per-cluster loop
                for (int k = 0; k < K; k++) c->host.N[k] = (float)c->h_stats[(size_t)k * c->F];
            if (with_constants) mixing_weights(K, &c->host);
            const int kp = tc_params_padded(c->tc.get(), K), D = c->D;
            std::atomic<int> bad_all{0};
            const std::function<void(int)> per_cluster = [&](int k) {
                if (with_finalize && k < K) finalize_cluster(c->h_stats, c->shift, k, D, &c->host);
                int b;
                double W[GMM_MAX_DIMENSIONS * GMM_MAX_DIMENSIONS];
                if (with_constants && k < K && constants_cluster_spd(k, D, &c->host, W)) {
                    b = tc_params_cluster_w(c->tc.get(), &c->host, k, K, W);      // one factorisation serves Rinv, ln det and the operand
                } else {
                    if (with_constants && k < K) constants_cluster(k, D, &c->host);
                    b = tc_params_cluster(c->tc.get(), &c->host, k, K);
                }
                int cur = bad_all.load(std::memory_order_relaxed);
                while (b > cur && !bad_all.compare_exchange_weak(cur, b)) {}
            };
            run_clusters(c, K, kp, per_cluster);
            const int bad = bad_all.load();
            with_constants = with_finalize = false;
            rc = tc_params_commit(c->tc.get(), K, bad, c->stream);
        }
        if (rc == GMM_OK) c->estep_tensor_ready = true;
        else if (rc != GMM_ERR_STATE || estep_path_of(c) == GMM_PATH_TENSOR) return rc;
        // GMM_ERR_STATE under GMM_PATH_AUTO: a cluster whose inverse covariance is not positive definite
        // (or does not fit FP16) — this parameter set is evaluated by the FP32 SIMT kernel instead.
    }
    if (with_finalize) finalize_from_stats(c->h_stats, c->shift, K, c->D, &c->host, c->host_threads, /*with_constants=*/false);
    if (with_constants) constants_from_R(K, c->D, &c->host, c->host_threads);
    if (!c->estep_tensor_ready) {
        build_epack(K, c->D, &c->host, c->h_epack);
        CUDA_TRY(cudaMemcpyAsync(c->d_epack, c->h_epack, sizeof(float) * (size_t)K * epack_stride(c->D),
                                 cudaMemcpyHostToDevice, c->stream));
    }
    if (c->d_avgvar && c->estep_tensor_ready && from_outside) {   // the device-side finalisation adds avgvar to the diagonals
        float* stage = reinterpret_cast<float*>(c->h_small + 32);
        std::memcpy(stage, c->host.avgvar, sizeof(float) * (size_t)K);
        CUDA_TRY(cudaMemcpyAsync(c->d_avgvar, stage, sizeof(float) * (size_t)K, cudaMemcpyHostToDevice, c->stream));
    }
    c->cur_K = K;
    c->params_partial = false;
    c->set_from_finalize = from_R;
    c->memcpy_ms +=std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return GMM_OK;
}

// ---- kernel dispatch -------------------------------------------------------
// SIMT E-step over n events of the SoA copy xs [D][pitch] into memb [K][pitch] against the epack records `epack` (the
// shard's or a gmm_score_stats chunk's with the context's D and d_epack; a gmm_condition_stats chunk's with the observed
// dimensions and its marginal block)
template <int D>
static void launch_estep_simt_d(gmm_ctx* c, int K, const float* epack, const float* xs, int n, float* memb, size_t pitch, double* ll,
                                const float* w) {
    const int blocks = (n + kEstepThreads - 1) / kEstepThreads;
    if (w) estep_simt_kernel<D, true><<<blocks, kEstepThreads, 0, c->stream>>>(xs, pitch, n, K, epack, memb, pitch, ll, w);
    else estep_simt_kernel<D><<<blocks, kEstepThreads, 0, c->stream>>>(xs, pitch, n, K, epack, memb, pitch, ll);
}
static int launch_estep_simt_on(gmm_ctx* c, int D, int K, const float* epack, const float* xs, int n, float* memb, size_t pitch,
                                double* ll, const float* w = nullptr) {
    if (n == 0) return GMM_OK;
    switch (D) {
#define GMM_CASE(d) case d: launch_estep_simt_d<d>(c, K, epack, xs, n, memb, pitch, ll, w); break;
        GMM_CASE(1) GMM_CASE(2) GMM_CASE(3) GMM_CASE(4) GMM_CASE(5) GMM_CASE(6) GMM_CASE(7) GMM_CASE(8)
        GMM_CASE(9) GMM_CASE(10) GMM_CASE(11) GMM_CASE(12) GMM_CASE(13) GMM_CASE(14) GMM_CASE(15) GMM_CASE(16)
        GMM_CASE(17) GMM_CASE(18) GMM_CASE(19) GMM_CASE(20) GMM_CASE(21) GMM_CASE(22) GMM_CASE(23) GMM_CASE(24)
        GMM_CASE(25) GMM_CASE(26) GMM_CASE(27) GMM_CASE(28) GMM_CASE(29) GMM_CASE(30) GMM_CASE(31) GMM_CASE(32)
#undef GMM_CASE
        default: return fail(GMM_ERR_ARG, "unsupported dimension count");
    }
    CUDA_TRY(cudaGetLastError());
    return GMM_OK;
}
static int launch_estep_simt(gmm_ctx* c, int K) {
    return launch_estep_simt_on(c, c->D, K, c->d_epack, c->d_x_soa, c->n, c->d_memb, c->memb_pitch, c->d_stats + (size_t)K * c->F,
                                step_weights(c));
}

// SIMT scoring of io.n rows of D coordinates against the epack records `epack` (gmm_score: the context's D and d_epack;
// gmm_condition: the observed dimensions and its marginal block)
template <int D>
static void launch_score_simt_d(gmm_ctx* c, int K, const float* epack, const TcScoreIo& io) {
    score_simt_kernel<D><<<(io.n + kEstepThreads - 1) / kEstepThreads, kEstepThreads, 0, c->stream>>>(io.x, io.n, K, epack, io.labels,
                                                                                                     io.max_resp, io.logp, io.ll);
}
static int launch_score_simt(gmm_ctx* c, int D, int K, const float* epack, const TcScoreIo& io) {
    if (io.n <= 0) return GMM_OK;
    switch (D) {
#define GMM_CASE(d) case d: launch_score_simt_d<d>(c, K, epack, io); break;
        GMM_CASE(1) GMM_CASE(2) GMM_CASE(3) GMM_CASE(4) GMM_CASE(5) GMM_CASE(6) GMM_CASE(7) GMM_CASE(8)
        GMM_CASE(9) GMM_CASE(10) GMM_CASE(11) GMM_CASE(12) GMM_CASE(13) GMM_CASE(14) GMM_CASE(15) GMM_CASE(16)
        GMM_CASE(17) GMM_CASE(18) GMM_CASE(19) GMM_CASE(20) GMM_CASE(21) GMM_CASE(22) GMM_CASE(23) GMM_CASE(24)
        GMM_CASE(25) GMM_CASE(26) GMM_CASE(27) GMM_CASE(28) GMM_CASE(29) GMM_CASE(30) GMM_CASE(31) GMM_CASE(32)
#undef GMM_CASE
        default: return fail(GMM_ERR_ARG, "unsupported dimension count");
    }
    CUDA_TRY(cudaGetLastError());
    return GMM_OK;
}

// FP64 SIMT M-step over n events of the SoA copy xs and the responsibilities memb (both [..][pitch]), adding into stats;
// w (optional): per-event weights
template <int JMAX, int CPT>
static int launch_mstep_simt_t(gmm_ctx* c, int K, const float* xs, int n, const float* memb, size_t pitch, double* stats,
                               const float* w) {
    constexpr int FP = 16 * JMAX, KT = 16 * CPT, GS = KT + 2;
    const size_t smem = sizeof(double) * (size_t)(kMstepTE * FP + kMstepTE * GS + kMstepTE * GMM_MAX_DIMENSIONS) +
                        sizeof(short) * 2 * FP;
    // the attribute is per device (context): one flag per device, not per process (a thread per GPU in the CLI)
    static bool attr_set[64] = {false};
    if (c->device >= 64 || !attr_set[c->device]) {
        CUDA_TRY(cudaFuncSetAttribute(mstep_simt_kernel<JMAX, CPT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        CUDA_TRY(cudaFuncSetAttribute(mstep_simt_kernel<JMAX, CPT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if (c->device < 64) attr_set[c->device] = true;
    }
    int gx = c->num_sms;
    int per = (n + gx - 1) / gx;
    per = (per + kMstepTE - 1) / kMstepTE * kMstepTE;
    if (per < kMstepTE) per = kMstepTE;
    gx = (n + per - 1) / per;
    dim3 grid(gx, (K + KT - 1) / KT);
    if (w) mstep_simt_kernel<JMAX, CPT, true><<<grid, kMstepThreads, smem, c->stream>>>(xs, pitch, n, c->D, K, memb, pitch, c->d_shift, stats, per, w);
    else mstep_simt_kernel<JMAX, CPT><<<grid, kMstepThreads, smem, c->stream>>>(xs, pitch, n, c->D, K, memb, pitch, c->d_shift, stats, per);
    CUDA_TRY(cudaGetLastError());
    return GMM_OK;
}
static int launch_mstep_simt_on(gmm_ctx* c, int K, const float* xs, int n, const float* memb, size_t pitch, double* stats,
                                const float* w = nullptr) {
    if (n == 0) return GMM_OK;
    const int F = c->F;
    const int cpt = K <= 16 ? 1 : (K <= 32 ? 2 : 4);
#define GMM_MS(j, p) return launch_mstep_simt_t<j, p>(c, K, xs, n, memb, pitch, stats, w)
    if (F <= 48) {
        if (cpt == 1) GMM_MS(3, 1);
        if (cpt == 2) GMM_MS(3, 2);
        GMM_MS(3, 4);
    } else if (F <= 160) {
        if (cpt == 1) GMM_MS(10, 1);
        if (cpt == 2) GMM_MS(10, 2);
        GMM_MS(10, 4);
    } else if (F <= 336) {
        if (cpt == 1) GMM_MS(21, 1);
        if (cpt == 2) GMM_MS(21, 2);
        GMM_MS(21, 4);
    } else {
        if (cpt == 1) GMM_MS(36, 1);
        GMM_MS(36, 2);
    }
#undef GMM_MS
}
static int launch_mstep_simt(gmm_ctx* c, int K) {
    return launch_mstep_simt_on(c, K, c->d_x_soa, c->n, c->d_memb, c->memb_pitch, c->d_stats, step_weights(c));
}

static int zero_stats(gmm_ctx* c, int K) {
    CUDA_TRY(cudaMemsetAsync(c->d_stats, 0, sizeof(double) * ((size_t)K * c->F + 1), c->stream));
    c->stats_clean_K = K;
    return GMM_OK;
}

// E-step on the current device parameters: responsibilities -> d_memb, local
// log-likelihood added to stats[K*F].
static int run_estep(gmm_ctx* c, int K) {
    timer_begin(c, c->t_estep);
    int rc = c->estep_tensor_ready ? tc_launch_estep(c->tc.get(), K, c->d_stats + (size_t)K * c->F, c->stream, step_weights(c))
                                   : launch_estep_simt(c, K);
    timer_end(c, c->t_estep);
    c->memb_valid = (rc == GMM_OK);
    return rc;
}

// M-step accumulation of the local statistics into stats[0 .. K*F).
static int run_mstep_accumulate(gmm_ctx* c, int K) {
    // Both M-step kernels ADD into stats[0 .. K*F): whatever an earlier call left there (column moments, seed rows,
    // the reduced statistics of a finished gmm_em / gmm_mstep) has to go; the log-likelihood slot [K*F] stays.
    const float* w = step_weights(c);
    if (w && !c->w_tensor_ok && mstep_path_of(c) == GMM_PATH_TENSOR)
        return fail(GMM_ERR_ARG, "GMM_PATH_TENSOR requested but the weights' dynamic range (max / min positive) exceeds what the "
                                 "tensor M-step's fixed-point operand serves");
    if (c->stats_clean_K != K) CUDA_TRY(cudaMemsetAsync(c->d_stats, 0, sizeof(double) * (size_t)K * c->F, c->stream));
    c->stats_clean_K = 0;
    timer_begin(c, c->t_mstep);
    int rc;
    if (use_tensor_mstep(c, K) && (!w || c->w_tensor_ok)) {
        rc = tc_launch_mstep(c->tc.get(), K, c->d_stats, c->stream, w, w ? c->w_scale : 1.0);
        c->mstep_tensor++;
    }
    else { rc = launch_mstep_simt(c, K); c->mstep_simt++; }
    timer_end(c, c->t_mstep);
    return rc;
}

// Sum the packed statistics over all ranks (replaces the four MPI_Allreduce of
// gaussian.cu:516,566,605,658,741 and the OpenMP-master sums) and bring them
// to the host.
static int reduce_stats_device(gmm_ctx* c, int K) {
    const size_t len = (size_t)K * c->F + 1;
    timer_begin(c, c->t_reduce);
    if (c->nranks > 1) {
        if (c->xchg.ok && c->allreduce_mode == 1 && len <= c->xchg.tab.cap) {
            c->xchg.epoch++;
            allreduce_peer_kernel<<<kXCtas, 1024, 0, c->stream>>>(c->xchg.tab, c->d_stats, (int)len, (int)(c->xchg.epoch & 1), c->xchg.epoch);
            CUDA_TRY(cudaGetLastError());
        } else {
            ncclResult_t r = nccl().AllReduce(c->d_stats, c->d_stats, len, ncclDouble, ncclSum, c->comm, c->stream);
            if (r != ncclSuccess) return fail(GMM_ERR_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
        }
    }
    timer_end(c, c->t_reduce);
    return GMM_OK;
}
static int reduce_stats_to_host(gmm_ctx* c, int K) {
    const size_t len = (size_t)K * c->F + 1;
    if (int rc = reduce_stats_device(c, K)) return rc;
    CUDA_TRY(cudaMemcpyAsync(c->h_stats, c->d_stats, sizeof(double) * len, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaEventRecord(c->ev_stats, c->stream));
    CUDA_TRY(cudaEventSynchronize(c->ev_stats));
    if (c->nranks > 1 && std::isnan(c->h_stats[0]))
        return fail(GMM_ERR_NCCL, "statistics all-reduce failed (a rank did not arrive, or a cluster's statistics are not finite)");
    return GMM_OK;
}

static int finalize_and_upload(gmm_ctx* c, int K) {
    // N, means, R (gaussian.cu:611-622, 663-679), inverse + constants + pi (:698-708) and the E-step operand: on the
    // tensor path ONE parallel loop over the clusters (timed as "upload"), else the serial + parallel pieces
    return upload_params(c, K, /*with_constants=*/true, /*with_finalize=*/true);
}

// Global column moments (sum x, sum x^2 over ALL events of all ranks), computed once per
// context.  They give (a) the seeding mean / average variance (gaussian_kernel.cu:54-102, with
// quirk Q2 fixed: whole data set, double accumulation) and (b) the centre `shift` and per-
// dimension `scale` about which the M-step statistics are accumulated (DESIGN.md).
static int ensure_moments(gmm_ctx* c) {
    if (c->have_shift) return GMM_OK;
    const int D = c->D;
    c->stats_clean_K = 0;
    // d_stats[0..D) sum x, [D..2D) sum x^2, [2D..3D) max x, [3D..4D) max (-x)
    std::vector<double> init(4 * (size_t)D, 0.0);
    for (int d = 0; d < 2 * D; d++) init[2 * D + d] = -std::numeric_limits<double>::max();
    if (4 * (size_t)D > stats_capacity(c)) return fail(GMM_ERR_STATE, "stats buffer too small for the column moments");
    CUDA_TRY(cudaMemcpyAsync(c->d_stats, init.data(), sizeof(double) * 4 * D, cudaMemcpyHostToDevice, c->stream));
    if (c->n > 0) {
        dim3 grid(std::min(4 * c->num_sms, (c->n + 255) / 256), D);
        column_moments_kernel<<<grid, 256, 0, c->stream>>>(c->d_x_soa, c->memb_pitch, c->n, D, c->d_stats);
        CUDA_TRY(cudaGetLastError());
    }
    if (c->nranks > 1) {
        ncclResult_t r = nccl().AllReduce(c->d_stats, c->d_stats, 2 * D, ncclDouble, ncclSum, c->comm, c->stream);
        if (r == ncclSuccess) r = nccl().AllReduce(c->d_stats + 2 * D, c->d_stats + 2 * D, 2 * D, ncclDouble, ncclMax, c->comm, c->stream);
        if (r != ncclSuccess) return fail(GMM_ERR_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
    }
    CUDA_TRY(cudaMemcpyAsync(c->h_stats, c->d_stats, sizeof(double) * 4 * D, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    double xmin[GMM_MAX_DIMENSIONS], xmax[GMM_MAX_DIMENSIONS];
    for (int d = 0; d < D; d++) {
        c->sum_x[d] = c->h_stats[d];
        c->sum_x2[d] = c->h_stats[D + d];
        xmax[d] = c->h_stats[2 * D + d];
        xmin[d] = -c->h_stats[3 * D + d];
        const double mean = c->sum_x[d] / (double)c->n_global;
        const double var = c->sum_x2[d] / (double)c->n_global - mean * mean;
        c->shift[d] = mean;
        c->scale[d] = var > 0 ? std::sqrt(var) : 1.0;
    }
    if (int rc = tc_set_shift_scale(c->tc.get(), c->shift, c->scale, xmin, xmax, c->stream)) return rc;   // rounds shift to float in place
    CUDA_TRY(cudaMemcpyAsync(c->d_shift, c->shift, sizeof(double) * D, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    c->have_shift = true;
    return GMM_OK;
}

static int check_K(const gmm_ctx* c, int K, const char* who) {
    if (!c) return fail(GMM_ERR_ARG, std::string(who) + ": null context");
    if (K < 1 || K > c->Kmax) return fail(GMM_ERR_ARG, std::string(who) + ": K out of range");
    return GMM_OK;
}

// The calls that apply the current parameter set to new events need a complete one for this K.
static int check_fitted(const gmm_ctx* c, int K, const char* who) {
    if (K != c->cur_K) return fail(GMM_ERR_STATE, std::string(who) + ": parameters for this K have not been set");
    if (c->params_partial)
        return fail(GMM_ERR_STATE, std::string(who) + ": gmm_mstep has updated N, means and R but not the inverses; run gmm_constants first");
    return GMM_OK;
}

// obs_dims of the conditioning calls (strictly increasing indices in [0, D), 1 to D of them), and the rest of [0, D): the
// missing dimensions mis[0 .. *nm) and a bit per observed dimension in *obs_mask.
static int split_obs(const gmm_ctx* c, const int* obs_dims, int n_obs, const char* who, int* mis, int* nm, unsigned* obs_mask) {
    if (!obs_dims || n_obs < 1 || n_obs > c->D)
        return fail(GMM_ERR_ARG, std::string(who) + ": obs_dims must hold between 1 and D dimension indices");
    for (int i = 0; i < n_obs; i++)
        if (obs_dims[i] < 0 || obs_dims[i] >= c->D || (i > 0 && obs_dims[i] <= obs_dims[i - 1]))
            return fail(GMM_ERR_ARG, std::string(who) + ": obs_dims must be strictly increasing indices in [0, D)");
    *nm = 0;
    *obs_mask = 0;
    for (int d = 0, i = 0; d < c->D; d++) {
        if (i < n_obs && obs_dims[i] == d) { *obs_mask |= 1u << d; i++; }
        else mis[(*nm)++] = d;
    }
    return GMM_OK;
}

// The centre the statistics of new events are taken about.  Before the context's first M-step it comes from the global
// column moments, an all-reduce over the ranks: computed here on one rank, never issued from here on several.
static int ensure_centre(gmm_ctx* c, const char* who) {
    if (c->have_shift) return GMM_OK;
    if (c->nranks > 1)
        return fail(GMM_ERR_STATE, std::string(who) + ": the context's centre is not fixed yet (run gmm_mstep or gmm_em first on every rank)");
    return ensure_moments(c);
}

// Nothing of a streaming call may still be in flight when it returns (also after a failure): both streams are drained, and
// an error they report becomes the call's when rc is still GMM_OK.
static int drain_streams(gmm_ctx* c, int rc, const char* who) {
    const cudaError_t e1 = c->score.copy ? cudaStreamSynchronize(c->score.copy) : cudaSuccess, e2 = cudaStreamSynchronize(c->stream);
    if (rc == GMM_OK && (e1 != cudaSuccess || e2 != cudaSuccess))
        rc = fail(GMM_ERR_CUDA, std::string(who) + ": " + cudaGetErrorString(e1 != cudaSuccess ? e1 : e2));
    return rc;
}

}  // namespace gmm

// ===========================================================================
extern "C" {

static int peer_exchange_setup(gmm_ctx* c);
static void peer_exchange_destroy(gmm_ctx* c);

const char* gmm_version(void) { return "cuda-gmm-mpi_b200 0.1 (sm_90a)"; }

int gmm_create(gmm_ctx** out, int device, int n_local, int D, int Kmax, const float* events_aos,
               long long n_global, long long offset) {
    if (!out) return fail(GMM_ERR_ARG, "gmm_create: null out");
    *out = nullptr;
    if (D < 1 || D > GMM_MAX_DIMENSIONS) return fail(GMM_ERR_ARG, "gmm_create: D must be in [1,32] (gaussian.h:16)");
    if (Kmax < 1 || Kmax > GMM_MAX_CLUSTERS) return fail(GMM_ERR_ARG, "gmm_create: Kmax must be in [1,512] (gaussian.h:10)");
    if (n_local < 0) return fail(GMM_ERR_ARG, "gmm_create: bad events");   // events_aos == NULL: supplied later (gmm_upload_events*)
    if (n_global <= 0) n_global = n_local;
    if (n_global < 1) return fail(GMM_ERR_ARG, "gmm_create: no events");
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1)
        return fail(GMM_ERR_CUDA, "ERROR: No CUDA capable GPUs detected (this engine has no CPU fallback).");
    if (device < 0 || device >= ndev) return fail(GMM_ERR_ARG, "gmm_create: device index out of range");
    CUDA_TRY(cudaSetDevice(device));
    cudaDeviceProp prop;
    CUDA_TRY(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)
        return fail(GMM_ERR_CUDA, std::string("device '") + prop.name + "' is not sm_90 (H100); kernels are built for sm_90a only");

    // a failed step returns: gmm_destroy drains the stream, and the owners free whatever was made
    std::unique_ptr<gmm_ctx, void (*)(gmm_ctx*)> own(new gmm_ctx(), gmm_destroy);
    gmm_ctx* c = own.get();
    c->device = device; c->n = n_local; c->D = D; c->Kmax = Kmax; c->F = num_features(D);
    c->n_global = n_global; c->offset = offset; c->num_sms = prop.multiProcessorCount;
    const char* ht = getenv("GMM_HOST_THREADS");
    c->host_threads_fixed = ht != nullptr;
    c->host_threads = ht ? atoi(ht) : default_host_threads(1);
    if (c->host_threads < 1) c->host_threads = 1;
    c->hN.assign(Kmax, 0); c->hpi.assign(Kmax, 0); c->hconst.assign(Kmax, 0); c->havgvar.assign(Kmax, 0);
    c->hmeans.assign((size_t)Kmax * D, 0); c->hR.assign((size_t)Kmax * D * D, 0); c->hRinv.assign((size_t)Kmax * D * D, 0);
    bind_host(c);
    if (int rc = c->stream.create(cudaStreamNonBlocking)) return rc;
    if (int rc = c->ev_stats.create(cudaEventDisableTiming)) return rc;
    const size_t nmax = n_local > 0 ? (size_t)n_local : 1;
    if (int rc = c->d_x_aos.reserve(nmax * D)) return rc;
    c->memb_pitch = (nmax + 31) / 32 * 32;         // also the row pitch of the SoA event copy
    if (int rc = c->d_x_soa.reserve(c->memb_pitch * D)) return rc;
    // rows in multiples of 8: the tensor E-step stores whole 8-cluster groups (zeros for the padding clusters)
    if (int rc = c->d_memb.reserve(c->memb_pitch * (size_t)((Kmax + 7) / 8 * 8))) return rc;
    if (int rc = c->d_epack.reserve((size_t)Kmax * epack_stride(D))) return rc;
    if (int rc = c->h_epack.reserve((size_t)Kmax * epack_stride(D))) return rc;
    if (int rc = c->d_stats.reserve(stats_capacity(c))) return rc;
    CUDA_TRY(cudaMemsetAsync(c->d_stats, 0, sizeof(double) * ((size_t)Kmax * c->F + 1), c->stream));
    if (int rc = c->h_stats.reserve(stats_capacity(c))) return rc;
    if (int rc = c->d_shift.reserve(GMM_MAX_DIMENSIONS)) return rc;
    CUDA_TRY(cudaMemsetAsync(c->d_shift, 0, sizeof(double) * GMM_MAX_DIMENSIONS, c->stream));
    if (n_local > 0 && events_aos) {
        CUDA_TRY(cudaMemcpyAsync(c->d_x_aos, events_aos, sizeof(float) * (size_t)n_local * D, cudaMemcpyHostToDevice, c->stream));
        dim3 blk(32, 8);
        transpose_aos_to_soa_kernel<<<(n_local + 31) / 32, blk, 0, c->stream>>>(c->d_x_aos, c->d_x_soa, c->memb_pitch, n_local, D);
        CUDA_TRY(cudaGetLastError());
    }
    {
        TcState* tc = nullptr;
        const int rc = tc_create(&tc, c->d_x_aos, c->d_x_soa, n_local, D, Kmax, c->d_memb, c->memb_pitch, c->num_sms, c->stream);
        c->tc.reset(tc);
        if (rc) return rc;
        tc_set_host_threads(c->tc.get(), c->host_threads);
    }
    if (const char* fm = getenv("GMM_FINALIZE")) c->finalize_mode = (std::string(fm) == "host") ? 0 : 1;
    if (n_local > 0 && tc_estep_supported(D, Kmax)) {
        const size_t setf = tc_param_set_floats(Kmax, D);
        for (int b = 0; b < 2; b++)
            if (int rc = c->d_pset[b].reserve(setf)) return rc;
        if (int rc = c->h_pset.reserve(setf)) return rc;
        if (int rc = c->d_avgvar.reserve(Kmax)) return rc;
        CUDA_TRY(cudaMemsetAsync(c->d_avgvar, 0, sizeof(float) * (size_t)Kmax, c->stream));
        if (int rc = c->d_bad.reserve(2)) return rc;
        if (int rc = c->d_llprev.reserve(2)) return rc;
        if (int rc = c->h_small.reserve(32 + sizeof(float) * (size_t)Kmax)) return rc;
    }
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    *out = own.release();
    return GMM_OK;
}

// Replace the events of this shard (same n_local, D): H2D copy + device transpose.  The global
// moments (shift / scale, seeding statistics) are recomputed on the next collective call.
int gmm_upload_events(gmm_ctx* c, const float* events_aos) {
    if (!c || (c->n > 0 && !events_aos)) return fail(GMM_ERR_ARG, "gmm_upload_events: bad argument");
    CUDA_TRY(cudaSetDevice(c->device));
    if (c->n > 0) {
        CUDA_TRY(cudaMemcpyAsync(c->d_x_aos, events_aos, sizeof(float) * (size_t)c->n * c->D, cudaMemcpyHostToDevice, c->stream));
        dim3 blk(32, 8);
        transpose_aos_to_soa_kernel<<<(c->n + 31) / 32, blk, 0, c->stream>>>(c->d_x_aos, c->d_x_soa, c->memb_pitch, c->n, c->D);
        CUDA_TRY(cudaGetLastError());
    }
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    c->have_shift = false;
    c->memb_valid = false;
    // the resident E-step operand was built in the coordinates (shift / scale) of the previous data set:
    // the caller has to set parameters again (gmm_seed / gmm_set_clusters) before the next E-step
    c->estep_tensor_ready = false;
    c->cur_K = 0;
    return GMM_OK;
}

// The shard's rows of a "*.bin" file (readData.cpp:35-47 format) straight to the device: pread into two pinned
// staging buffers, each chunk's H2D copy overlapping the read of the next (replaces whole-file malloc + fread on the
// host, gaussian.cu:188-218, followed by a pageable copy per GPU, :360-377).
int gmm_upload_events_file(gmm_ctx* c, const char* path) {
    if (!c || !path) return fail(GMM_ERR_ARG, "gmm_upload_events_file: bad argument");
    CUDA_TRY(cudaSetDevice(c->device));
    const int fd = open(path, O_RDONLY);
    if (fd < 0) return fail(GMM_ERR_IO, std::string("cannot open ") + path);
    int32_t hdr[2] = {0, 0};
    if (pread(fd, hdr, sizeof(hdr), 0) != (ssize_t)sizeof(hdr) || hdr[0] <= 0 || hdr[1] != c->D || (long long)hdr[0] != c->n_global) {
        close(fd);
        return fail(GMM_ERR_IO, "gmm_upload_events_file: header does not match the context (events / dimensions)");
    }
    const size_t row = sizeof(float) * (size_t)c->D;
    const size_t total = row * (size_t)c->n;
    const size_t chunk = std::max<size_t>(row, ((size_t)32 << 20) / row * row);
    PinnedArray<char> stage[2];
    Event done[2];
    int rc = GMM_OK;
    for (int b = 0; b < 2 && rc == GMM_OK; b++) {
        if (stage[b].reserve(chunk) != GMM_OK || done[b].create(cudaEventDisableTiming) != GMM_OK)
            rc = fail(GMM_ERR_CUDA, "gmm_upload_events_file: pinned staging allocation failed");
    }
    size_t off = 0;
    for (int i = 0; rc == GMM_OK && off < total; i++) {
        const int b = i & 1;
        const size_t len = std::min(chunk, total - off);
        if (i >= 2 && cudaEventSynchronize(done[b]) != cudaSuccess) { rc = fail(GMM_ERR_CUDA, "gmm_upload_events_file: copy failed"); break; }
        size_t got = 0;
        while (got < len) {
            const ssize_t r = pread(fd, stage[b] + got, len - got, (off_t)(sizeof(hdr) + row * (size_t)c->offset + off + got));
            if (r <= 0) { rc = fail(GMM_ERR_IO, "truncated .bin file"); break; }
            got += (size_t)r;
        }
        if (rc != GMM_OK) break;
        if (cudaMemcpyAsync(reinterpret_cast<char*>(c->d_x_aos.get()) + off, stage[b], len, cudaMemcpyHostToDevice, c->stream) != cudaSuccess ||
            cudaEventRecord(done[b], c->stream) != cudaSuccess) { rc = fail(GMM_ERR_CUDA, "gmm_upload_events_file: copy failed"); break; }
        off += len;
    }
    close(fd);
    if (rc == GMM_OK && c->n > 0) {
        dim3 blk(32, 8);
        transpose_aos_to_soa_kernel<<<(c->n + 31) / 32, blk, 0, c->stream>>>(c->d_x_aos, c->d_x_soa, c->memb_pitch, c->n, c->D);
        if (cudaGetLastError() != cudaSuccess) rc = fail(GMM_ERR_CUDA, "transpose launch failed");
    }
    if (cudaStreamSynchronize(c->stream) != cudaSuccess && rc == GMM_OK) rc = fail(GMM_ERR_CUDA, "gmm_upload_events_file: copy failed");
    c->have_shift = false;
    c->memb_valid = false;
    c->estep_tensor_ready = false;
    c->cur_K = 0;
    return rc;
}

void gmm_destroy(gmm_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    collect_all(c);
    peer_exchange_destroy(c);
    if (c->comm && nccl().ok) nccl().CommDestroy(c->comm);
    delete c;
}

// Maps every rank's exchange area into this rank (see allreduce_peer_kernel).  Never fatal: whatever goes wrong on
// any rank (no peer access, IPC refused, more than 8 ranks) leaves ALL ranks on ncclAllReduce — the decision is itself
// agreed through the gathered `ok` fields.
static int peer_exchange_setup(gmm_ctx* c) {
    PeerExchange& x = c->xchg;
    x.ok = false;
    const int G = c->nranks;
    const size_t cap = (size_t)c->Kmax * c->F + 1;
    const size_t flag_count = (size_t)2 * kXMaxRanks * kXCtas;
    const size_t bytes = sizeof(double) * 2 * cap + sizeof(unsigned long long) * flag_count;
    PeerHello me{};
    me.pid = (long long)getpid();
    me.device = c->device;
    me.ok = (G <= kXMaxRanks && getenv("GMM_NO_PEER_ALLREDUCE") == nullptr) ? 1 : 0;
    me.dev_fin = c->d_pset[0] ? 1 : 0;
    if (me.ok && x.base.reserve(bytes) != GMM_OK) me.ok = 0;
    if (me.ok) {
        cudaMemset(x.base, 0, bytes);
        me.ptr = (unsigned long long)(uintptr_t)x.base.get();
        if (cudaIpcGetMemHandle(&me.handle, x.base) != cudaSuccess) { me.ok = 0; cudaGetLastError(); }
    }
    // gather the hellos (device staging; NCCL is the only channel the C ABI has between ranks)
    DeviceArray<PeerHello> d_all;
    std::vector<PeerHello> all((size_t)G);
    if (int rc = d_all.reserve(G)) return rc;
    CUDA_TRY(cudaMemcpyAsync(d_all + c->rank, &me, sizeof(PeerHello), cudaMemcpyHostToDevice, c->stream));
    {
        ncclResult_t r = nccl().AllGather(d_all + c->rank, d_all, sizeof(PeerHello), ncclChar, c->comm, c->stream);
        if (r != ncclSuccess) return fail(GMM_ERR_NCCL, std::string("ncclAllGather: ") + nccl().GetErrorString(r));
    }
    CUDA_TRY(cudaMemcpyAsync(all.data(), d_all, sizeof(PeerHello) * G, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    int ok = 1;
    for (int p = 0; p < G; p++) ok &= all[p].ok;
    c->dev_fin_agreed = true;
    for (int p = 0; p < G; p++) c->dev_fin_agreed = c->dev_fin_agreed && all[p].dev_fin != 0;
    x.tab.nranks = G; x.tab.rank = c->rank; x.tab.cap = cap;
    for (int p = 0; p < G && ok; p++) {
        void* mapped = nullptr;
        if (p == c->rank) mapped = x.base;
        else if (all[p].pid == me.pid) {                 // a thread of this process: plain peer access
            int can = 0;
            if (cudaDeviceCanAccessPeer(&can, c->device, all[p].device) != cudaSuccess || !can) ok = 0;
            else {
                cudaError_t e = cudaDeviceEnablePeerAccess(all[p].device, 0);
                if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) ok = 0;
                cudaGetLastError();
                mapped = (void*)(uintptr_t)all[p].ptr;
            }
        } else {
            if (cudaIpcOpenMemHandle(&mapped, all[p].handle, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { ok = 0; cudaGetLastError(); }
            else x.opened[p] = mapped;
        }
        if (ok) {
            x.tab.buf[p] = reinterpret_cast<double*>(mapped);
            x.tab.flags[p] = reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(mapped) + sizeof(double) * 2 * cap);
        }
    }
    // a rank that failed to map somebody must take everybody back to NCCL: agree on the minimum
    {
        DeviceArray<double> d_ok;
        double h_ok = ok ? 1.0 : 0.0;
        if (int rc = d_ok.reserve(1)) return rc;
        CUDA_TRY(cudaMemcpyAsync(d_ok, &h_ok, sizeof(double), cudaMemcpyHostToDevice, c->stream));
        ncclResult_t r = nccl().AllReduce(d_ok, d_ok, 1, ncclDouble, ncclMin, c->comm, c->stream);
        if (r != ncclSuccess) return fail(GMM_ERR_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
        CUDA_TRY(cudaMemcpyAsync(&h_ok, d_ok, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));
        ok = h_ok > 0.5;
    }
    x.ok = ok != 0;
    if (c->verbose) std::printf("[gmm rank %d] statistics all-reduce: %s\n", c->rank, x.ok ? "peer-memory kernel (NVLink)" : "ncclAllReduce");
    return GMM_OK;
}

static void peer_exchange_destroy(gmm_ctx* c) {
    PeerExchange& x = c->xchg;
    for (int p = 0; p < kXMaxRanks; p++)
        if (x.opened[p]) { cudaIpcCloseMemHandle(x.opened[p]); x.opened[p] = nullptr; }
    x.base.reset();
    x.ok = false;
}

int gmm_nccl_unique_id(char id_out[128]) {
    if (!id_out) return fail(GMM_ERR_ARG, "gmm_nccl_unique_id: null");
    if (!nccl().ok) return fail(GMM_ERR_NCCL, "libnccl.so.2 not found");
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId size");
    ncclUniqueId id;
    NCCL_TRY(nccl().GetUniqueId(&id));
    std::memcpy(id_out, &id, 128);
    return GMM_OK;
}

int gmm_comm_init(gmm_ctx* c, int nranks, int rank, const char id_in[128]) {
    if (!c || nranks < 1 || rank < 0 || rank >= nranks) return fail(GMM_ERR_ARG, "gmm_comm_init: bad argument");
    c->rank = rank; c->nranks = nranks;
    if (!c->host_threads_fixed) {                   // the ranks of one box share its cores
        c->host_threads = default_host_threads(nranks);
        tc_set_host_threads(c->tc.get(), c->host_threads);
    }
    if (nranks == 1) return GMM_OK;
    if (!id_in) return fail(GMM_ERR_ARG, "gmm_comm_init: null id");
    if (!nccl().ok) return fail(GMM_ERR_NCCL, "libnccl.so.2 not found");
    CUDA_TRY(cudaSetDevice(c->device));
    ncclUniqueId id;
    std::memcpy(&id, id_in, 128);
    NCCL_TRY(nccl().CommInitRank(&c->comm, nranks, id, rank));
    return peer_exchange_setup(c);
}

int gmm_comm_rank(const gmm_ctx* c, int* rank, int* nranks) {
    if (!c) return fail(GMM_ERR_ARG, "gmm_comm_rank: null context");
    if (rank) *rank = c->rank;
    if (nranks) *nranks = c->nranks;
    return GMM_OK;
}

int gmm_set_option(gmm_ctx* c, const char* key, double value) {
    if (!c || !key) return fail(GMM_ERR_ARG, "gmm_set_option: bad argument");
    const std::string k(key);
    if (k == "path") {
        const int p = (int)value;
        if (p < GMM_PATH_AUTO || p > GMM_PATH_TENSOR) return fail(GMM_ERR_ARG, "gmm_set_option: bad path");
        c->path = p;
    } else if (k == "verbose") c->verbose = (int)value;
    else if (k == "host_threads") {
        c->host_threads = value < 1 ? 1 : (int)value;
        c->host_threads_fixed = true;
        tc_set_host_threads(c->tc.get(), c->host_threads);
    }
    else if (k == "estep_path" || k == "mstep_path") {
        const int p = (int)value;
        if (p < -1 || p > GMM_PATH_TENSOR) return fail(GMM_ERR_ARG, "gmm_set_option: bad path");
        (k == "estep_path" ? c->estep_path : c->mstep_path) = p;
    }
    else if (k == "profile") c->profile_phases = value != 0;
    else if (k == "allreduce") c->allreduce_mode = value != 0 ? 1 : 0;
    else if (k == "finalize") { c->finalize_mode = value != 0 ? 1 : 0; if (value != 0) c->dev_fin_failed = false; }
    else if (k == "finalize_fault_iter") c->fin_fault_iter = (int)value;
    else if (k == "score_chunk") {
        if (!(value >= 1 && value <= 268435456.0)) return fail(GMM_ERR_ARG, "gmm_set_option: score_chunk must be in [1, 2^28] events");
        c->score_chunk = (long long)value;
    }
    else return fail(GMM_ERR_ARG, "gmm_set_option: unknown key '" + k + "'");
    return GMM_OK;
}

// --- seeding ---------------------------------------------------------------
int gmm_seed(gmm_ctx* c, int K, clusters_t* host_out) {
    if (int rc = check_K(c, K, "gmm_seed")) return rc;
    CUDA_TRY(cudaSetDevice(c->device));
    if (int rc = ensure_moments(c)) return rc;
    const int D = c->D;
    // seed rows (evenly spaced events, gaussian.cu:110-120): the owning shard contributes, the others add zeros
    const size_t len = (size_t)K * D;
    if (len > (size_t)c->Kmax * c->F + 1) return fail(GMM_ERR_STATE, "gmm_seed: stats buffer too small");
    std::vector<double> rows(len, 0.0);
    std::vector<float> tmp(D);
    for (int k = 0; k < K; k++) {
        const long long g = seed_event_index(k, K, c->n_global);
        if (g >= c->offset && g < c->offset + c->n) {
            CUDA_TRY(cudaMemcpyAsync(tmp.data(), c->d_x_aos + (size_t)(g - c->offset) * D, sizeof(float) * D,
                                     cudaMemcpyDeviceToHost, c->stream));
            CUDA_TRY(cudaStreamSynchronize(c->stream));
            for (int d = 0; d < D; d++) rows[(size_t)k * D + d] = tmp[d];
        }
    }
    if (c->nranks > 1) {
        c->stats_clean_K = 0;
        CUDA_TRY(cudaMemcpyAsync(c->d_stats, rows.data(), sizeof(double) * len, cudaMemcpyHostToDevice, c->stream));
        ncclResult_t r = nccl().AllReduce(c->d_stats, c->d_stats, len, ncclDouble, ncclSum, c->comm, c->stream);
        if (r != ncclSuccess) return fail(GMM_ERR_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
        CUDA_TRY(cudaMemcpyAsync(rows.data(), c->d_stats, sizeof(double) * len, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    std::vector<float> seed_rows(len);
    for (size_t i = 0; i < len; i++) seed_rows[i] = (float)rows[i];
    seed_from_moments(c->sum_x, c->sum_x2, c->n_global, D, K, seed_rows.data(), &c->host);
    if (int rc = upload_params(c, K)) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    c->memb_valid = false;
    if (host_out) copy_params(host_out, &c->host, K, D);
    return GMM_OK;
}

int gmm_set_clusters(gmm_ctx* c, int K, const clusters_t* in) {
    if (int rc = check_K(c, K, "gmm_set_clusters")) return rc;
    if (!in) return fail(GMM_ERR_ARG, "gmm_set_clusters: null clusters");
    CUDA_TRY(cudaSetDevice(c->device));
    copy_params(&c->host, in, K, c->D);
    c->memb_valid = false;
    if (int rc = upload_params(c, K)) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    return GMM_OK;
}

// Per-event weights of the shard.  Validated and agreed before anything changes: every rank learns the global sum, the
// largest weight and the smallest positive one, whether any rank saw an invalid weight and how many ranks passed weights
// from two all-reduces, so a rejected call leaves the weights in effect on every rank, and a call that passes NULL on some
// ranks only is rejected on all of them (the ranks would otherwise disagree on N = sum w, and so on gmm_em's stopping test).
int gmm_set_weights(gmm_ctx* c, const float* weights, double* total_out) {
    if (!c) return fail(GMM_ERR_ARG, "gmm_set_weights: null context");
    CUDA_TRY(cudaSetDevice(c->device));
    double sum = 0.0, wmax = 0.0, wmin = std::numeric_limits<double>::infinity(), bad = 0.0, has = weights ? 1.0 : 0.0;
    if (weights) {
        for (int e = 0; e < c->n; e++) {
            const float w = weights[e];
            if (!(w >= 0.0f) || !std::isfinite(w)) { bad = 1.0; continue; }
            sum += (double)w;
            wmax = std::max(wmax, (double)w);
            if (w > 0.0f) wmin = std::min(wmin, (double)w);
        }
    }
    if (c->nranks > 1) {
        double h[5] = {sum, bad, has, wmax, -wmin};   // summed | maximised
        DeviceArray<double> d_h;
        if (int rc = d_h.reserve(5)) return rc;
        ncclResult_t r = ncclSuccess;
        cudaError_t e = cudaMemcpyAsync(d_h, h, sizeof(h), cudaMemcpyHostToDevice, c->stream);
        if (e == cudaSuccess) {
            r = nccl().AllReduce(d_h, d_h, 3, ncclDouble, ncclSum, c->comm, c->stream);
            if (r == ncclSuccess) r = nccl().AllReduce(d_h + 3, d_h + 3, 2, ncclDouble, ncclMax, c->comm, c->stream);
            if (r == ncclSuccess) e = cudaMemcpyAsync(h, d_h, sizeof(h), cudaMemcpyDeviceToHost, c->stream);
            if (e == cudaSuccess) e = cudaStreamSynchronize(c->stream);
        }
        if (r != ncclSuccess) return fail(GMM_ERR_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
        if (e != cudaSuccess) return fail(GMM_ERR_CUDA, std::string("gmm_set_weights: ") + cudaGetErrorString(e));
        sum = h[0]; bad = h[1]; has = h[2]; wmax = h[3]; wmin = -h[4];
        if (has != 0.0 && has != (double)c->nranks)
            return fail(GMM_ERR_ARG, "gmm_set_weights: weights on some ranks and NULL on others (pass weights on all ranks, or NULL on all)");
    }
    if (!weights) {
        c->weighted = false;
        c->memb_valid = false;
        if (total_out) *total_out = (double)c->n_global;
        return GMM_OK;
    }
    if (bad != 0.0) return fail(GMM_ERR_ARG, "gmm_set_weights: a weight is negative or not finite");
    if (!(sum > 0.0)) return fail(GMM_ERR_ARG, "gmm_set_weights: the weights sum to zero");
    if (c->d_w.size() < c->memb_pitch) {
        if (int rc = c->d_w.reserve(c->memb_pitch)) return rc;
        CUDA_TRY(cudaMemsetAsync(c->d_w, 0, sizeof(float) * c->memb_pitch, c->stream));   // the M-step reads whole 32-event tiles
    }
    if (c->n > 0) CUDA_TRY(cudaMemcpyAsync(c->d_w, weights, sizeof(float) * (size_t)c->n, cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    c->w_scale = wmax;
    c->w_tensor_ok = wmax <= kWeightRangeTc * wmin;
    c->w_total = sum;
    c->weighted = true;
    c->memb_valid = false;
    if (total_out) *total_out = sum;
    return GMM_OK;
}

int gmm_get_clusters(gmm_ctx* c, int K, clusters_t* out, int with_memberships) {
    if (int rc = check_K(c, K, "gmm_get_clusters")) return rc;
    if (!out) return fail(GMM_ERR_ARG, "gmm_get_clusters: null clusters");
    CUDA_TRY(cudaSetDevice(c->device));
    copy_params(out, &c->host, K, c->D);
    if (with_memberships) {
        if (!out->memberships) return fail(GMM_ERR_ARG, "gmm_get_clusters: memberships requested but pointer is null");
        if (!c->memb_valid) return fail(GMM_ERR_STATE, "gmm_get_clusters: no E-step has run for the current parameters");
        if (c->n > 0)
            CUDA_TRY(cudaMemcpy2DAsync(out->memberships, sizeof(float) * (size_t)c->n, c->d_memb, sizeof(float) * c->memb_pitch,
                                       sizeof(float) * (size_t)c->n, K, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));
    }
    return GMM_OK;
}

int gmm_estep(gmm_ctx* c, int K, float* loglik_out) {
    if (int rc = check_K(c, K, "gmm_estep")) return rc;
    if (K != c->cur_K) return fail(GMM_ERR_STATE, "gmm_estep: parameters for this K have not been set");
    CUDA_TRY(cudaSetDevice(c->device));
    const size_t ll = (size_t)K * c->F;
    CUDA_TRY(cudaMemsetAsync(c->d_stats + ll, 0, sizeof(double), c->stream));
    if (int rc = run_estep(c, K)) return rc;
    if (c->nranks > 1) {
        ncclResult_t r = nccl().AllReduce(c->d_stats + ll, c->d_stats + ll, 1, ncclDouble, ncclSum, c->comm, c->stream);
        if (r != ncclSuccess) return fail(GMM_ERR_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
    }
    CUDA_TRY(cudaMemcpyAsync(c->h_stats + ll, c->d_stats + ll, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    collect_all(c);
    if (loglik_out) *loglik_out = (float)c->h_stats[ll];
    return GMM_OK;
}

int gmm_mstep(gmm_ctx* c, int K) {
    if (int rc = check_K(c, K, "gmm_mstep")) return rc;
    if (!c->memb_valid || K != c->cur_K) return fail(GMM_ERR_STATE, "gmm_mstep: run gmm_estep first");
    CUDA_TRY(cudaSetDevice(c->device));
    if (int rc = ensure_moments(c)) return rc;
    const double ll_keep = c->h_stats[(size_t)K * c->F];
    if (int rc = run_mstep_accumulate(c, K)) return rc;         // zeroes stats[0 .. K*F) first
    if (int rc = reduce_stats_to_host(c, K)) return rc;
    c->h_stats[(size_t)K * c->F] = ll_keep;
    // gmm_mstep stops before constants_kernel: N, means, R only (gaussian.cu:538-687)
    finalize_from_stats(c->h_stats, c->shift, K, c->D, &c->host, c->host_threads, /*with_constants=*/false);
    c->params_partial = true;
    collect_all(c);
    return GMM_OK;
}

int gmm_constants(gmm_ctx* c, int K) {
    if (int rc = check_K(c, K, "gmm_constants")) return rc;
    CUDA_TRY(cudaSetDevice(c->device));
    auto t0 = std::chrono::steady_clock::now();
    constants_from_R(K, c->D, &c->host, c->host_threads);
    c->host_const_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (int rc = upload_params(c, K)) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    return GMM_OK;
}

// One pass of the loop body of gaussian.cu:532-755 on the device-resident
// responsibilities: M-step statistics -> all-reduce -> host normalisation and
// constants -> parameter upload -> E-step.  The log-likelihood of the E-step
// that produced the responsibilities rides in the packed buffer and is returned
// through *prev_loglik.
static int em_iteration(gmm_ctx* c, int K, float* prev_loglik) {
    if (int rc = run_mstep_accumulate(c, K)) return rc;
    if (int rc = reduce_stats_to_host(c, K)) return rc;
    if (prev_loglik) *prev_loglik = (float)c->h_stats[(size_t)K * c->F];
    if (int rc = finalize_and_upload(c, K)) return rc;    // gaussian.cu:611-622, 663-679, 698-708
    if (int rc = zero_stats(c, K)) return rc;
    if (int rc = run_estep(c, K)) return rc;              // gaussian.cu:713-714
    c->iterations++;
    return GMM_OK;
}

// ---- EM iterations with the finalisation on the device --------------------------------------------------------
static bool dev_finalize_ok(const gmm_ctx* c, int K) {
    return c->finalize_mode == 1 && !c->dev_fin_failed && c->dev_fin_agreed && c->d_pset[0] && c->n > 0 && c->estep_tensor_ready && K == c->cur_K &&
           use_tensor_estep(c, K) && tc_finalize_supported(c->tc.get(), K);
}

// Parameter set `which` (K-prefixes of its arrays) -> pinned staging; valid after the next stream synchronisation.
static int fetch_param_set(gmm_ctx* c, int K, int which) {
    const int D = c->D, Kmax = c->Kmax;
    const size_t cnt[6] = {(size_t)K, (size_t)K, (size_t)K, (size_t)K * D, (size_t)K * D * D, (size_t)K * D * D};
    for (int a = 0; a < 6; a++) {
        const size_t off = tc_param_set_off(Kmax, D, a);
        CUDA_TRY(cudaMemcpyAsync(c->h_pset + off, c->d_pset[which] + off, sizeof(float) * cnt[a], cudaMemcpyDeviceToHost, c->stream));
    }
    return GMM_OK;
}
static void scatter_param_set(gmm_ctx* c, int K) {
    const int D = c->D, Kmax = c->Kmax;
    float* dst[6] = {c->host.N, c->host.pi, c->host.constant, c->host.means, c->host.R, c->host.Rinv};
    const size_t cnt[6] = {(size_t)K, (size_t)K, (size_t)K, (size_t)K * D, (size_t)K * D * D, (size_t)K * D * D};
    for (int a = 0; a < 6; a++) std::memcpy(dst[a], c->h_pset + tc_param_set_off(Kmax, D, a), sizeof(float) * cnt[a]);
}

static int em_iteration(gmm_ctx* c, int K, float* prev_loglik);

// `iters` EM iterations queued back to back: M-step -> all-reduce -> finalize_params_kernel -> E-step, nothing returns to
// the host in between.  Afterwards the host copy of the parameters is refreshed from the last set.  *ll_prev receives the
// log-likelihood slot the LAST finalisation saw (the E-step before the last one; gmm_em's convergence test needs it).
// If a finalisation met a cluster only the host path serves (not positive definite, outside FP16), the work queued after
// it was discarded by the kernels themselves: the host takes the last good set, re-creates the responsibilities that
// iteration started from and runs the remaining iterations through its own path; the context then stays on the host path.
static int run_dev_iterations(gmm_ctx* c, int K, int iters, float* ll_prev) {
    if (iters <= 0) return GMM_OK;
    int* h_bad = reinterpret_cast<int*>(c->h_small.get());
    double* h_ll = reinterpret_cast<double*>(c->h_small + 16);
    h_bad[0] = -1; h_bad[1] = 0;
    CUDA_TRY(cudaMemcpyAsync(c->d_bad, h_bad, 2 * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    for (int i = 0; i < iters; i++) {
        if (int rc = run_mstep_accumulate(c, K)) return rc;
        if (int rc = reduce_stats_device(c, K)) return rc;
        timer_begin(c, c->t_final);
        int rc = tc_launch_finalize(c->tc.get(), K, c->d_stats, c->d_avgvar, c->d_pset[i & 1], c->d_llprev + (i & 1), c->d_bad, i, c->fin_fault_iter, c->stream);
        timer_end(c, c->t_final);
        if (rc) return rc;
        c->dev_finalize_launches++;
        if (int rc2 = zero_stats(c, K)) return rc2;
        if (int rc2 = run_estep(c, K)) return rc2;
        c->iterations++;
    }
    CUDA_TRY(cudaMemcpyAsync(h_bad + 2, c->d_bad, 2 * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaMemcpyAsync(h_ll, c->d_llprev, 2 * sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    if (int rc = fetch_param_set(c, K, (iters - 1) & 1)) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    const int first_bad = h_bad[2], code = h_bad[3];
    if (first_bad < 0) {
        scatter_param_set(c, K);
        c->set_from_finalize = true;
        if (ll_prev) *ll_prev = (float)h_ll[(iters - 1) & 1];
        return GMM_OK;
    }
    if (code == 4) return fail(GMM_ERR_NCCL, "statistics all-reduce failed (a rank did not arrive, or a cluster's statistics are not finite)");
    c->dev_fin_failed = true;
    c->dev_replays++;
    if (c->verbose && c->rank == 0)
        std::printf("[gmm] device-side finalisation met a cluster for the host path at iteration %d (code %d): replaying on the host\n", first_bad, code);
    if (first_bad > 0) {                                   // (first_bad == 0: the host copy is still the state before the batch)
        if (int rc = fetch_param_set(c, K, (first_bad - 1) & 1)) return rc;
        CUDA_TRY(cudaStreamSynchronize(c->stream));
        scatter_param_set(c, K);
    }
    c->iterations -= iters - first_bad;
    // A set left by a finalisation (this batch's device set, or at first_bad == 0 the set an earlier device batch or host
    // iteration finalised) is rebuilt as the host path builds it after its own finalisation: inverse, constant, pi and the
    // E-step operand from ONE factorisation of R (the device set is bit-identical to it); refactorising the stored float
    // Rinv would hand the E-step a slightly different operand.  A set that came from outside (seed, gmm_set_clusters, order
    // reduction) keeps its Rinv, as the host path did when it was uploaded.
    if (int rc = upload_params(c, K, /*with_constants=*/first_bad > 0 || c->set_from_finalize)) return rc;
    if (int rc = zero_stats(c, K)) return rc;
    if (int rc = run_estep(c, K)) return rc;
    float prev = 0.f;
    for (int i = first_bad; i < iters; i++)
        if (int rc = em_iteration(c, K, &prev)) return rc;
    if (ll_prev) *ll_prev = prev;
    return GMM_OK;
}

// Bring only the log-likelihood slot of the last E-step to the host (summed over ranks).
static int reduce_loglik_to_host(gmm_ctx* c, int K, float* out) {
    const size_t ll = (size_t)K * c->F;
    if (c->nranks > 1) {
        ncclResult_t r = nccl().AllReduce(c->d_stats + ll, c->d_stats + ll, 1, ncclDouble, ncclSum, c->comm, c->stream);
        if (r != ncclSuccess) return fail(GMM_ERR_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
    }
    CUDA_TRY(cudaMemcpyAsync(c->h_stats + ll, c->d_stats + ll, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    if (out) *out = (float)c->h_stats[ll];
    return GMM_OK;
}

int gmm_em_iterations(gmm_ctx* c, int K, int iters, float* loglik_out) {
    if (int rc = check_K(c, K, "gmm_em_iterations")) return rc;
    if (!c->memb_valid || K != c->cur_K) return fail(GMM_ERR_STATE, "gmm_em_iterations: run gmm_estep first");
    CUDA_TRY(cudaSetDevice(c->device));
    if (int rc = ensure_moments(c)) return rc;
    if (dev_finalize_ok(c, K)) {
        if (int rc = run_dev_iterations(c, K, iters, nullptr)) return rc;
    } else {
        for (int i = 0; i < iters; i++)
            if (int rc = em_iteration(c, K, nullptr)) return rc;
    }
    if (int rc = reduce_loglik_to_host(c, K, loglik_out)) return rc;
    collect_all(c);
    return GMM_OK;
}

// The EM loop (gaussian.cu:487-755): initial E-step, then
// while(iters < min_iters || (|change| > epsilon && iters < max_iters)).
// The convergence test needs the log-likelihood of the E-step that just ran;
// it rides in the same packed buffer as the M-step statistics, so when the
// test can still go either way the next M-step accumulation is issued before
// the test (and discarded if the loop ends there).
int gmm_em(gmm_ctx* c, int K, int min_iters, int max_iters, float epsilon, float* loglik_out, int* iters_out) {
    if (int rc = check_K(c, K, "gmm_em")) return rc;
    if (K != c->cur_K) return fail(GMM_ERR_STATE, "gmm_em: parameters for this K have not been set (gmm_seed / gmm_set_clusters)");
    CUDA_TRY(cudaSetDevice(c->device));
    if (int rc = ensure_moments(c)) return rc;
    if (epsilon < 0) epsilon = em_epsilon(c->D, em_count(c));
    const size_t ll_idx = (size_t)K * c->F;
    if (int rc = zero_stats(c, K)) return rc;
    if (int rc = run_estep(c, K)) return rc;                 // initial E-step, gaussian.cu:487-523
    float likelihood = 0, old_likelihood = 0, change = epsilon * 2;
    int iters = 0;
    if (min_iters > 0 && dev_finalize_ok(c, K)) {
        // the first min_iters iterations run whatever the likelihood does (gaussian.cu:532): no convergence test, so no
        // reason to come back to the host between them
        if (int rc = run_dev_iterations(c, K, min_iters, &old_likelihood)) return rc;
        iters = min_iters;
    }
    for (;;) {
        const bool must_continue = iters < min_iters;
        const bool may_continue = iters < max_iters;
        if (!must_continue && !may_continue) {               // the loop ends whatever the change is
            if (int rc = reduce_loglik_to_host(c, K, &likelihood)) return rc;
            break;
        }
        if (int rc = run_mstep_accumulate(c, K)) return rc;
        if (int rc = reduce_stats_to_host(c, K)) return rc;
        likelihood = (float)c->h_stats[ll_idx];
        if (iters > 0) change = likelihood - old_likelihood;
        if (!(must_continue || (std::fabs(change) > epsilon && may_continue))) break;   // gaussian.cu:532
        old_likelihood = likelihood;
        if (int rc = finalize_and_upload(c, K)) return rc;   // host normalisation + constants
        if (int rc = zero_stats(c, K)) return rc;
        if (int rc = run_estep(c, K)) return rc;             // gaussian.cu:713-714
        iters++;
        c->iterations++;
        if (c->verbose > 1) std::printf("[gmm rank %d] K=%d iter %d\n", c->rank, K, iters);
    }
    collect_all(c);
    if (loglik_out) *loglik_out = likelihood;
    if (iters_out) *iters_out = iters;
    return GMM_OK;
}

// ---- scoring of new events ------------------------------------------------------------------------------------------
// Buffers for chunks of c->score_chunk events: allocated on first use, grown (never shrunk) when the option grows.
static int score_buffers(gmm_ctx* c) {
    ScoreBuffers& s = c->score;
    if (int rc = s.copy.create(cudaStreamNonBlocking)) return rc;
    for (int b = 0; b < 2; b++) {
        for (Event* e : {&s.h2d[b], &s.kern[b], &s.d2h[b]})
            if (int rc = e->create(cudaEventDisableTiming)) return rc;
        for (Event* e : {&s.t0[b], &s.t1[b]})
            if (int rc = e->create(cudaEventDefault)) return rc;
    }
    const long long want = std::max(s.cap, c->score_chunk);
    for (int b = 0; b < 2; b++) {
        if (int rc = s.h_in[b].reserve((size_t)want * c->D)) return rc;
        if (int rc = s.d_in[b].reserve((size_t)want * c->D)) return rc;
        if (int rc = s.d_out[b].reserve(ScoreBuffers::out_bytes(want))) return rc;
        if (int rc = s.h_out[b].reserve(ScoreBuffers::out_bytes(want))) return rc;
    }
    if (c->Kmax > 64) {
        if (int rc = s.d_run_den.reserve(want)) return rc;
        if (int rc = s.d_run_bl.reserve(want)) return rc;
        if (int rc = s.d_run_bk.reserve(want)) return rc;
    }
    s.cap = want;
    return GMM_OK;
}

// Output pointers of slot b (device or pinned host image of the same layout).
static TcScoreIo score_io(gmm_ctx* c, char* base, int b, int n) {
    ScoreBuffers& s = c->score;
    TcScoreIo io{};
    io.x = s.d_in[b];
    io.n = n;
    io.ll = reinterpret_cast<double*>(base);
    io.flag = reinterpret_cast<int*>(base + 8);
    io.labels = reinterpret_cast<int*>(base + ScoreBuffers::kHeader);
    io.max_resp = reinterpret_cast<float*>(base + ScoreBuffers::kHeader + 4 * (size_t)s.cap);
    io.logp = reinterpret_cast<float*>(base + ScoreBuffers::kHeader + 8 * (size_t)s.cap);
    io.run_den = s.d_run_den; io.run_bl = s.d_run_bl; io.run_bk = s.d_run_bk;
    return io;
}

// Kernel time of slot b's last launch (between its timing events), added to *acc.
static void add_slot_ms(gmm_ctx* c, int b, double* acc) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, c->score.t0[b], c->score.t1[b]) == cudaSuccess) *acc += ms;
}

// Input half of slot b: m host rows of `width` floats -> pinned stage -> (copy stream) device chunk.
static int stage_chunk(gmm_ctx* c, int b, const float* rows, int m, int width) {
    ScoreBuffers& s = c->score;
    CUDA_TRY(cudaEventSynchronize(s.h2d[b]));                 // the stage's previous H2D has left it
    std::memcpy(s.h_in[b], rows, sizeof(float) * (size_t)m * width);
    CUDA_TRY(cudaStreamWaitEvent(s.copy, s.kern[b], 0));      // the device chunk's previous readers are done with it
    CUDA_TRY(cudaMemcpyAsync(s.d_in[b], s.h_in[b], sizeof(float) * (size_t)m * width, cudaMemcpyHostToDevice, s.copy));
    CUDA_TRY(cudaEventRecord(s.h2d[b], s.copy));
    return GMM_OK;
}

// The chunk pipeline of the calls that stream outputs back (gmm_score, gmm_condition, gmm_sample).  Chunk i of
// c->score_chunk events goes through slot b = i & 1: with `in`, its host rows (`width` floats each) -> pinned stage ->
// (copy stream) device chunk; then (compute stream) launch(b, e0, m), which records the slot's timing events around its
// kernels -> (copy stream) fetch(b, m, stream) into the slot's pinned mirrors -> hand_over(b, e0, m) to the caller's
// arrays.  Chunk i is issued before chunk i - 1 is finished, so chunk i's H2D and the host staging of chunk i + 1 overlap
// chunk i - 1's kernel and D2H.  Finishing a chunk adds its kernel time to *kernel_ms before the hand-over.
using ChunkFn = std::function<int(int b, long long e0, int m)>;
static int stream_chunks(gmm_ctx* c, long long n, const float* in, int width, double* kernel_ms, const ChunkFn& launch,
                         const std::function<int(int b, int m, cudaStream_t st)>& fetch, const ChunkFn& hand_over) {
    ScoreBuffers& s = c->score;
    const long long chunk = c->score_chunk, nchunks = (n + chunk - 1) / chunk;     // (the buffers hold at least this many)
    auto rows_of = [&](long long i) { return (int)std::min(chunk, n - i * chunk); };
    for (long long i = 0; i <= nchunks; i++) {
        if (i < nchunks) {                                        // issue chunk i
            const int b = (int)(i & 1), m = rows_of(i);
            if (in) {
                if (int rc = stage_chunk(c, b, in + (size_t)(i * chunk) * width, m, width)) return rc;
                CUDA_TRY(cudaStreamWaitEvent(c->stream, s.h2d[b], 0));
            }
            CUDA_TRY(cudaStreamWaitEvent(c->stream, s.d2h[b], 0));    // the slot's previous outputs have left the device
            if (int rc = launch(b, i * chunk, m)) return rc;
            CUDA_TRY(cudaEventRecord(s.kern[b], c->stream));
            CUDA_TRY(cudaStreamWaitEvent(s.copy, s.kern[b], 0));
            if (int rc = fetch(b, m, s.copy)) return rc;
            CUDA_TRY(cudaEventRecord(s.d2h[b], s.copy));
        }
        if (i > 0) {                                              // finish chunk i - 1
            const int b = (int)((i - 1) & 1);
            CUDA_TRY(cudaEventSynchronize(s.d2h[b]));
            add_slot_ms(c, b, kernel_ms);
            if (int rc = hand_over(b, (i - 1) * chunk, rows_of(i - 1))) return rc;
        }
    }
    return GMM_OK;
}

// The outputs gmm_score and gmm_condition return per event (NULL: not requested) and the sum of the chunks' log-likelihoods.
struct ScoreOut {
    int* labels;
    float* max_resp;
    float* logp;
    double* ll_sum;
};

// D2H of slot b's header and requested outputs on stream st.
static int fetch_scores(gmm_ctx* c, const ScoreOut& o, int b, int m, cudaStream_t st) {
    ScoreBuffers& s = c->score;
    const TcScoreIo dv = score_io(c, s.d_out[b], b, m), hv = score_io(c, s.h_out[b], b, m);
    CUDA_TRY(cudaMemcpyAsync(s.h_out[b], s.d_out[b], ScoreBuffers::kHeader, cudaMemcpyDeviceToHost, st));
    if (o.labels) CUDA_TRY(cudaMemcpyAsync(hv.labels, dv.labels, sizeof(int) * (size_t)m, cudaMemcpyDeviceToHost, st));
    if (o.max_resp) CUDA_TRY(cudaMemcpyAsync(hv.max_resp, dv.max_resp, sizeof(float) * (size_t)m, cudaMemcpyDeviceToHost, st));
    if (o.logp) CUDA_TRY(cudaMemcpyAsync(hv.logp, dv.logp, sizeof(float) * (size_t)m, cudaMemcpyDeviceToHost, st));
    return GMM_OK;
}

// Slot b's fetched outputs of the chunk at event e0 to the caller.
static void hand_over_scores(gmm_ctx* c, const ScoreOut& o, int b, long long e0, int m) {
    const TcScoreIo hv = score_io(c, c->score.h_out[b], b, m);
    *o.ll_sum += *hv.ll;
    if (o.labels) std::memcpy(o.labels + e0, hv.labels, sizeof(int) * (size_t)m);
    if (o.max_resp) std::memcpy(o.max_resp + e0, hv.max_resp, sizeof(float) * (size_t)m);
    if (o.logp) std::memcpy(o.logp + e0, hv.logp, sizeof(float) * (size_t)m);
}

// d_epack of the current parameters for a SIMT kernel: while the tensor operand serves them it is not maintained, so the
// first SIMT kernel of a call builds it from the host copy (*ready: it is current).
static int ensure_epack(gmm_ctx* c, int K, bool* ready) {
    if (*ready) return GMM_OK;
    const int D = c->D;
    build_epack(K, D, &c->host, c->h_epack);
    CUDA_TRY(cudaMemcpyAsync(c->d_epack, c->h_epack, sizeof(float) * (size_t)K * epack_stride(D), cudaMemcpyHostToDevice, c->stream));
    *ready = true;
    return GMM_OK;
}

// gmm_score's chunks through the pipeline, on the E-step's kernel family for the current parameters.  A tensor chunk that
// flags an event is scored again by the SIMT kernel before it is handed over.
static int score_batch(gmm_ctx* c, int K, const float* ev, long long n, const ScoreOut& out) {
    ScoreBuffers& s = c->score;
    const int D = c->D;
    const bool tensor = c->estep_tensor_ready;
    bool epack_ready = !tensor;
    auto launch = [&](int b, int m, bool on_tensor) -> int {
        const TcScoreIo io = score_io(c, s.d_out[b], b, m);
        CUDA_TRY(cudaMemsetAsync(s.d_out[b], 0, ScoreBuffers::kHeader, c->stream));
        if (!on_tensor)
            if (int rc = ensure_epack(c, K, &epack_ready)) return rc;
        CUDA_TRY(cudaEventRecord(s.t0[b], c->stream));
        int rc = on_tensor ? tc_launch_score(c->tc.get(), K, io, c->stream) : launch_score_simt(c, D, K, c->d_epack, io);
        if (rc) return rc;
        CUDA_TRY(cudaEventRecord(s.t1[b], c->stream));
        (on_tensor ? s.tensor_chunks : s.simt_chunks)++;
        return GMM_OK;
    };
    auto fetch = [&](int b, int m, cudaStream_t st) { return fetch_scores(c, out, b, m, st); };
    auto hand_over = [&](int b, long long e0, int m) -> int {
        if (tensor && *score_io(c, s.h_out[b], b, m).flag) {
            // an event beyond the FP16 event operand's range (or not finite): the SIMT kernel scores the chunk again
            // (its rows are still in the slot's device buffer: the next H2D into it is issued after this)
            if (estep_path_of(c) == GMM_PATH_TENSOR)
                return fail(GMM_ERR_STATE, "gmm_score: an event lies outside the tensor E-step's FP16 operand range (beyond 2^14 "
                                           "standard deviations, or not finite) and the path is GMM_PATH_TENSOR");
            s.tensor_chunks--;                                    // its outputs come from the SIMT kernel
            if (int rc = launch(b, m, false)) return rc;
            if (int rc = fetch(b, m, c->stream)) return rc;
            CUDA_TRY(cudaStreamSynchronize(c->stream));
            add_slot_ms(c, b, &s.kernel_ms);
        }
        hand_over_scores(c, out, b, e0, m);
        return GMM_OK;
    };
    return stream_chunks(c, n, ev, D, &s.kernel_ms, [&](int b, long long, int m) { return launch(b, m, tensor); }, fetch, hand_over);
}

int gmm_score(gmm_ctx* c, int K, const float* events_aos, long long n, int* labels, float* max_resp, float* logp, double* loglik_out) {
    if (int rc = check_K(c, K, "gmm_score")) return rc;
    if (n < 0 || (n > 0 && !events_aos)) return fail(GMM_ERR_ARG, "gmm_score: bad events (n < 0, or no rows)");
    if (int rc = check_fitted(c, K, "gmm_score")) return rc;
    CUDA_TRY(cudaSetDevice(c->device));
    const auto t0 = std::chrono::steady_clock::now();
    double ll = 0.0;
    int rc = GMM_OK;
    if (n > 0) {
        rc = score_buffers(c);
        if (rc == GMM_OK) rc = score_batch(c, K, events_aos, n, {labels, max_resp, logp, &ll});
        rc = drain_streams(c, rc, "gmm_score");
    }
    c->score.wall_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (rc == GMM_OK && loglik_out) *loglik_out = ll;
    return rc;
}

int gmm_get_score_profile(gmm_ctx* c, double out[4], int reset) {
    if (!c || !out) return fail(GMM_ERR_ARG, "gmm_get_score_profile: bad argument");
    ScoreBuffers& s = c->score;
    out[0] = s.kernel_ms; out[1] = s.wall_ms; out[2] = (double)s.tensor_chunks; out[3] = (double)s.simt_chunks;
    if (reset) { s.kernel_ms = s.wall_ms = 0; s.tensor_chunks = s.simt_chunks = 0; }
    return GMM_OK;
}

// ---- E-step + M-step statistics of new events ---------------------------------------------------------------------------
static int score_stats_buffers(gmm_ctx* c, bool with_memberships, bool with_observed = false) {
    ScoreStatsBuffers& t = c->sstats;
    if (int rc = t.ev_flag.create(cudaEventDisableTiming)) return rc;
    for (int b = 0; b < 2; b++)
        for (Event* e : {&t.p0[b], &t.p1[b], &t.k0[b], &t.k1[b]})
            if (int rc = e->create(cudaEventDefault)) return rc;
    if (int rc = t.d_stats.reserve((size_t)c->Kmax * c->F + 1)) return rc;
    if (int rc = t.h_stats.reserve((size_t)c->Kmax * c->F + 1)) return rc;
    if (int rc = t.d_flag.reserve(1)) return rc;
    if (int rc = t.h_flag.reserve(1)) return rc;
    if (int rc = t.d_shift_f.reserve(GMM_MAX_DIMENSIONS)) return rc;
    const long long want = std::max(t.cap, c->score_chunk);
    const size_t pitch = ((size_t)want + 31) / 32 * 32, rows = (size_t)(c->Kmax + 7) / 8 * 8;
    if (int rc = t.d_z.reserve(pitch * c->D)) return rc;
    if (int rc = t.d_xs.reserve(pitch * c->D)) return rc;
    if (t.d_memb.size() < pitch * rows) {
        if (int rc = t.d_memb.reserve(pitch * rows)) return rc;
        // rows above K that no E-step of this call writes are read by the tensor M-step's 32-cluster boxes (their columns
        // are discarded): keep them finite
        CUDA_TRY(cudaMemsetAsync(t.d_memb, 0, sizeof(float) * pitch * rows, c->stream));
    }
    t.cap = want;
    t.pitch = pitch;
    if (with_memberships)
        if (int rc = t.h_memb.reserve((size_t)c->Kmax * t.cap)) return rc;
    if (with_observed)
        if (int rc = t.d_xo.reserve(t.pitch * c->D)) return rc;
    return GMM_OK;
}

// The chunk loop of the calls that return E- and M-step statistics of streamed events (gmm_score_stats,
// gmm_condition_stats).  Per chunk i (slot b = i & 1 of gmm_score's input stage, rows of `width` floats), in order on the
// compute stream: prep(b, m), the call's prep kernel (its SoA copies and the range flag) -> flag to the host, while chunk
// i + 1 is staged and its H2D issued -> estep(b, m, ce, cm), the fallback image the flag calls for and the E-step into the
// chunk's responsibilities -> M-step adding into the call's statistics -> (memberships) pitched D2H and rows to the caller.
// e_tensor / m_tensor: the call puts the wgmma E- / M-step on the chunks whose flag allows it (ce / cm).  `who` names the
// call in errors.
static int stats_batch(gmm_ctx* c, int K, const float* ev, int width, long long n, bool with_stats, float* memberships,
                       bool e_tensor, bool m_tensor, StatsProfile& pr, const char* who, const std::function<int(int b, int m)>& prep,
                       const std::function<int(int b, int m, bool ce, bool cm)>& estep) {
    ScoreBuffers& s = c->score;
    ScoreStatsBuffers& t = c->sstats;
    const size_t KF = (size_t)K * c->F;
    const long long chunk = c->score_chunk, nchunks = (n + chunk - 1) / chunk;
    bool epack_ready = !e_tensor;          // (a chunk the wgmma E-step cannot take runs the SIMT one on d_epack)
    CUDA_TRY(cudaMemsetAsync(t.d_stats, 0, sizeof(double) * (KF + 1), c->stream));
    auto rows_of = [&](long long i) { return (int)std::min(chunk, n - i * chunk); };
    auto stage = [&](long long i) { return stage_chunk(c, (int)(i & 1), ev + (size_t)(i * chunk) * width, rows_of(i), width); };
    auto collect = [&](int b) {                                   // timings of a chunk whose kernels have finished
        float a = 0, k = 0, w = 0;
        if (cudaEventElapsedTime(&a, t.p0[b], t.p1[b]) == cudaSuccess && cudaEventElapsedTime(&k, t.k0[b], t.k1[b]) == cudaSuccess)
            pr.kernel_ms += (double)a + (double)k;
        if (cudaEventElapsedTime(&w, t.p1[b], t.k0[b]) == cudaSuccess) pr.wait_ms += w;
    };
    if (nchunks > 0)
        if (int rc = stage(0)) return rc;
    for (long long i = 0; i < nchunks; i++) {
        const int b = (int)(i & 1), m = rows_of(i);
        const long long e0 = i * chunk;
        CUDA_TRY(cudaStreamWaitEvent(c->stream, s.h2d[b], 0));
        CUDA_TRY(cudaMemsetAsync(t.d_flag, 0, sizeof(int), c->stream));
        CUDA_TRY(cudaEventRecord(t.p0[b], c->stream));
        if (int rc = prep(b, m)) return rc;
        CUDA_TRY(cudaEventRecord(t.p1[b], c->stream));
        CUDA_TRY(cudaMemcpyAsync(t.h_flag, t.d_flag, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(cudaEventRecord(t.ev_flag, c->stream));
        if (i + 1 < nchunks)
            if (int rc = stage(i + 1)) return rc;
        CUDA_TRY(cudaEventSynchronize(t.ev_flag));
        if (i > 0) collect(b ^ 1);                                // (the prep of chunk i ran after chunk i - 1's kernels)
        const int flag = *t.h_flag;
        if (flag & kScoreStatsNotFinite) return fail(GMM_ERR_ARG, std::string(who) + ": an event has a coordinate that is not finite");
        const bool ce = e_tensor && !(flag & kScoreStatsBeyondFp16);
        const bool cm = m_tensor && !(flag & kScoreStatsBeyondZb);
        if (e_tensor && !ce && estep_path_of(c) == GMM_PATH_TENSOR)
            return fail(GMM_ERR_STATE, std::string(who) + ": an event lies beyond 2^14 standard deviations (the tensor E-step's "
                                                           "FP16 operand range) and estep_path is GMM_PATH_TENSOR");
        if (m_tensor && !cm && mstep_path_of(c) == GMM_PATH_TENSOR)
            return fail(GMM_ERR_STATE, std::string(who) + ": an event lies beyond the tensor M-step's fixed-point range (|z| >= "
                                                           "the training data's bound) and mstep_path is GMM_PATH_TENSOR");
        if (!ce)
            if (int rc = ensure_epack(c, K, &epack_ready)) return rc;
        CUDA_TRY(cudaEventRecord(t.k0[b], c->stream));
        int rc = estep(b, m, ce, cm);
        if (rc) return rc;
        (ce ? pr.e_tensor : pr.e_simt)++;
        CUDA_TRY(cudaEventRecord(s.kern[b], c->stream));          // the device input chunk is free again
        if (with_stats) {
            rc = cm ? tc_launch_mstep_on(c->tc.get(), K, t.d_z, t.d_memb, t.pitch, m, t.d_stats, c->stream)
                    : launch_mstep_simt_on(c, K, t.d_xs, m, t.d_memb, t.pitch, t.d_stats);
            if (rc) return rc;
            (cm ? pr.m_tensor : pr.m_simt)++;
        }
        CUDA_TRY(cudaEventRecord(t.k1[b], c->stream));
        if (memberships) {
            CUDA_TRY(cudaMemcpy2DAsync(t.h_memb, sizeof(float) * (size_t)m, t.d_memb, sizeof(float) * t.pitch, sizeof(float) * (size_t)m, K,
                                       cudaMemcpyDeviceToHost, c->stream));
            CUDA_TRY(cudaStreamSynchronize(c->stream));
            for (int k = 0; k < K; k++)
                std::memcpy(memberships + (size_t)k * n + e0, t.h_memb + (size_t)k * m, sizeof(float) * (size_t)m);
        }
    }
    if (with_stats) CUDA_TRY(cudaMemcpyAsync(t.h_stats, t.d_stats, sizeof(double) * (KF + 1), cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    if (nchunks > 0) collect((int)((nchunks - 1) & 1));
    return GMM_OK;
}

// gmm_score_stats' chunks through the statistics loop, on the context's own kernel selection: the prep kernel writes the
// standardised SoA copy for the wgmma M-step and the raw one when the selection already puts a SIMT kernel on every chunk;
// a chunk that falls back only because of its flag gets its raw copy after the flag is read.
static int score_stats_batch(gmm_ctx* c, int K, const float* ev, long long n, bool with_stats, float* memberships, StatsProfile& pr) {
    ScoreBuffers& s = c->score;
    ScoreStatsBuffers& t = c->sstats;
    const int D = c->D;
    const size_t KF = (size_t)K * c->F;
    const bool e_tensor = c->estep_tensor_ready;
    const bool m_tensor = with_stats && use_tensor_mstep(c, K);
    const bool raw_always = !e_tensor || (with_stats && !m_tensor);   // the context's own selection puts a SIMT kernel on every chunk
    const float* shift_f = (e_tensor || m_tensor) ? tc_shift_f(c->tc.get()) : nullptr;
    const float zb = m_tensor ? tc_mstep_zbound(c->tc.get()) : INFINITY;
    if ((e_tensor || m_tensor) && !shift_f) return fail(GMM_ERR_STATE, "gmm_score_stats: the tensor kernels have no centre");
    auto prep = [&](int b, int m) -> int {
        score_stats_prep_kernel<<<(m + 31) / 32, dim3(32, 8), 0, c->stream>>>(
            s.d_in[b], m, D, shift_f, shift_f ? tc_inv_scale_f(c->tc.get()) : nullptr, zb, m_tensor ? t.d_z.get() : nullptr,
            raw_always ? t.d_xs.get() : nullptr, t.pitch, t.d_flag);
        CUDA_TRY(cudaGetLastError());
        return GMM_OK;
    };
    auto estep = [&](int b, int m, bool ce, bool cm) -> int {
        if (!raw_always && (!ce || (with_stats && !cm))) {       // a fallback of this chunk only: its raw SoA copy now
            transpose_aos_to_soa_kernel<<<(m + 31) / 32, dim3(32, 8), 0, c->stream>>>(s.d_in[b], t.d_xs, t.pitch, m, D);
            CUDA_TRY(cudaGetLastError());
        }
        return ce ? tc_launch_estep_on(c->tc.get(), K, s.d_in[b], m, t.d_memb, t.pitch, s.d_run_den, t.d_stats + KF, c->stream)
                  : launch_estep_simt_on(c, D, K, c->d_epack, t.d_xs, m, t.d_memb, t.pitch, t.d_stats + KF);
    };
    return stats_batch(c, K, ev, D, n, with_stats, memberships, e_tensor, m_tensor, pr, "gmm_score_stats", prep, estep);
}

int gmm_score_stats(gmm_ctx* c, int K, const float* events_aos, long long n, double* stats_out, double* shift_out, float* memberships) {
    if (int rc = check_K(c, K, "gmm_score_stats")) return rc;
    if (n < 0 || (n > 0 && !events_aos)) return fail(GMM_ERR_ARG, "gmm_score_stats: bad events (n < 0, or no rows)");
    if (!stats_out && !memberships) return fail(GMM_ERR_ARG, "gmm_score_stats: neither statistics nor memberships requested");
    if (int rc = check_fitted(c, K, "gmm_score_stats")) return rc;
    CUDA_TRY(cudaSetDevice(c->device));
    const auto t0 = std::chrono::steady_clock::now();
    if (int rc = ensure_centre(c, "gmm_score_stats")) return rc;
    const size_t len = (size_t)K * c->F + 1;
    int rc = GMM_OK;
    if (n > 0) {
        rc = score_buffers(c);
        if (rc == GMM_OK) rc = score_stats_buffers(c, memberships != nullptr);
        if (rc == GMM_OK) rc = score_stats_batch(c, K, events_aos, n, stats_out != nullptr, memberships, c->sstats.prof);
        rc = drain_streams(c, rc, "gmm_score_stats");
    }
    if (rc == GMM_OK) {
        if (stats_out) {
            if (n > 0) std::memcpy(stats_out, c->sstats.h_stats, sizeof(double) * len);
            else std::fill(stats_out, stats_out + len, 0.0);
        }
        if (shift_out) std::memcpy(shift_out, c->shift, sizeof(double) * (size_t)c->D);
    }
    c->sstats.prof.wall_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return rc;
}

int gmm_get_score_stats_profile(gmm_ctx* c, double out[7], int reset) {
    if (!c || !out) return fail(GMM_ERR_ARG, "gmm_get_score_stats_profile: bad argument");
    StatsProfile& t = c->sstats.prof;
    out[0] = t.kernel_ms; out[1] = t.wall_ms;
    out[2] = (double)t.e_tensor; out[3] = (double)t.e_simt; out[4] = (double)t.m_tensor; out[5] = (double)t.m_simt;
    out[6] = t.wait_ms;
    if (reset) t = StatsProfile();
    return GMM_OK;
}

// ---- k-means++ and Lloyd seeding ------------------------------------------------------------------------------------------
static int kmeans_buffers(gmm_ctx* c) {
    KmeansBuffers& b = c->kmeans;
    const size_t n = (size_t)std::max(c->n, 1), D = (size_t)c->D, xfer = 16 * (size_t)c->nranks;
    b.nb = (int)((n + kSeedBlockEvents - 1) / kSeedBlockEvents);
    b.nba = (int)((n + kAssignThreads - 1) / kAssignThreads);
    if (int rc = b.d_d2.reserve(n)) return rc;
    if (int rc = b.d_labels.reserve(n)) return rc;
    if (int rc = b.d_bsum.reserve(b.nb)) return rc;
    if (int rc = b.d_bpot.reserve((size_t)b.nb * kSeedMaxCand)) return rc;
    if (int rc = b.d_bchanged.reserve(b.nba)) return rc;
    if (int rc = b.d_binertia.reserve(b.nba)) return rc;
    if (int rc = b.d_cand.reserve(kSeedMaxCand * D)) return rc;
    if (int rc = b.d_pick.reserve(kSeedMaxCand)) return rc;
    if (int rc = b.d_pick_idx.reserve(kSeedMaxCand)) return rc;
    if (int rc = b.d_centres.reserve((size_t)c->Kmax * D)) return rc;
    if (int rc = b.d_xfer.reserve(xfer)) return rc;
    if (int rc = b.h_bsum.reserve(b.nb)) return rc;
    if (int rc = b.h_bpot.reserve((size_t)b.nb * kSeedMaxCand)) return rc;
    if (int rc = b.h_bchanged.reserve(b.nba)) return rc;
    if (int rc = b.h_binertia.reserve(b.nba)) return rc;
    if (int rc = b.h_pick.reserve(kSeedMaxCand)) return rc;
    if (int rc = b.h_xfer.reserve(xfer)) return rc;
    return GMM_OK;
}

// Every rank's m (<= 16) values on every host: one all-reduce of a zero-padded [nranks][m] vector (each slot has one
// non-zero contributor, so the sum is exact).  Callers add the ranks' values in rank order: every rank forms the same bits.
static int kmeans_rank_values(gmm_ctx* c, const double* mine, int m, std::vector<double>& all) {
    KmeansBuffers& b = c->kmeans;
    all.assign((size_t)c->nranks * m, 0.0);
    std::copy(mine, mine + m, all.begin() + (size_t)c->rank * m);
    if (c->nranks == 1) return GMM_OK;
    const size_t len = (size_t)c->nranks * m;
    std::copy(all.begin(), all.end(), b.h_xfer.get());
    CUDA_TRY(cudaMemcpyAsync(b.d_xfer, b.h_xfer, sizeof(double) * len, cudaMemcpyHostToDevice, c->stream));
    ncclResult_t r = nccl().AllReduce(b.d_xfer, b.d_xfer, len, ncclDouble, ncclSum, c->comm, c->stream);
    if (r != ncclSuccess) return fail(GMM_ERR_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
    CUDA_TRY(cudaMemcpyAsync(b.h_xfer, b.d_xfer, sizeof(double) * len, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    std::copy(b.h_xfer.get(), b.h_xfer + len, all.begin());
    return GMM_OK;
}

// Sum of `count` floats over the ranks (rows that only their owner filled in, zeros elsewhere).
static int kmeans_sum_rows(gmm_ctx* c, float* d_rows, size_t count) {
    if (c->nranks == 1) return GMM_OK;
    ncclResult_t r = nccl().AllReduce(d_rows, d_rows, count, ncclFloat, ncclSum, c->comm, c->stream);
    if (r != ncclSuccess) return fail(GMM_ERR_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
    return GMM_OK;
}

#define GMM_SEED_DISPATCH(D, CALL)                                                                                         \
    switch (D) {                                                                                                           \
        GMM_SEED_CASE(1, CALL) GMM_SEED_CASE(2, CALL) GMM_SEED_CASE(3, CALL) GMM_SEED_CASE(4, CALL)                      \
        GMM_SEED_CASE(5, CALL) GMM_SEED_CASE(6, CALL) GMM_SEED_CASE(7, CALL) GMM_SEED_CASE(8, CALL)                      \
        GMM_SEED_CASE(9, CALL) GMM_SEED_CASE(10, CALL) GMM_SEED_CASE(11, CALL) GMM_SEED_CASE(12, CALL)                   \
        GMM_SEED_CASE(13, CALL) GMM_SEED_CASE(14, CALL) GMM_SEED_CASE(15, CALL) GMM_SEED_CASE(16, CALL)                  \
        GMM_SEED_CASE(17, CALL) GMM_SEED_CASE(18, CALL) GMM_SEED_CASE(19, CALL) GMM_SEED_CASE(20, CALL)                  \
        GMM_SEED_CASE(21, CALL) GMM_SEED_CASE(22, CALL) GMM_SEED_CASE(23, CALL) GMM_SEED_CASE(24, CALL)                  \
        GMM_SEED_CASE(25, CALL) GMM_SEED_CASE(26, CALL) GMM_SEED_CASE(27, CALL) GMM_SEED_CASE(28, CALL)                  \
        GMM_SEED_CASE(29, CALL) GMM_SEED_CASE(30, CALL) GMM_SEED_CASE(31, CALL) GMM_SEED_CASE(32, CALL)                  \
        default: return fail(GMM_ERR_ARG, "unsupported dimension count");                                                 \
    }
#define GMM_SEED_CASE(d, CALL) case d: CALL(d); break;

static int kmeanspp_update(gmm_ctx* c, const float* d_centre, bool first) {
    KmeansBuffers& b = c->kmeans;
    if (c->n == 0) return GMM_OK;
#define GMM_CALL(d) kmeanspp_update_kernel<d><<<b.nb, kSeedThreads, 0, c->stream>>>(c->d_x_soa, c->memb_pitch, c->n, d_centre, \
                                                                                      first ? 1 : 0, b.d_d2, b.d_bsum)
    GMM_SEED_DISPATCH(c->D, GMM_CALL)
#undef GMM_CALL
    CUDA_TRY(cudaGetLastError());
    return GMM_OK;
}

static int kmeanspp_potential(gmm_ctx* c, int L) {
    KmeansBuffers& b = c->kmeans;
    if (c->n == 0) return GMM_OK;
#define GMM_CALL(d) kmeanspp_potential_kernel<d><<<b.nb, kSeedThreads, 0, c->stream>>>(c->d_x_soa, c->memb_pitch, c->n, b.d_cand, L, \
                                                                                         b.d_d2, b.d_bpot)
    GMM_SEED_DISPATCH(c->D, GMM_CALL)
#undef GMM_CALL
    CUDA_TRY(cudaGetLastError());
    return GMM_OK;
}

static int kmeans_assign_launch(gmm_ctx* c, int K, int Kw) {
    KmeansBuffers& b = c->kmeans;
    if (c->n == 0) return GMM_OK;
#define GMM_CALL(d) kmeans_assign_kernel<d><<<b.nba, kAssignThreads, 0, c->stream>>>(c->d_x_soa, c->memb_pitch, c->n, b.d_centres, K, \
                                                                                       Kw, c->d_memb, c->memb_pitch, b.d_labels,    \
                                                                                       b.d_bchanged, b.d_binertia)
    GMM_SEED_DISPATCH(c->D, GMM_CALL)
#undef GMM_CALL
    CUDA_TRY(cudaGetLastError());
    return GMM_OK;
}

// splitmix64; each draw u = (next >> 11) * 2^-53 in [0, 1).  Every rank draws the same sequence.
struct SplitMix64 {
    unsigned long long s;
    double uniform() {
        unsigned long long z = (s += 0x9E3779B97F4A7C15ULL);
        z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
        z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
        z ^= z >> 31;
        return (double)(z >> 11) * 0x1.0p-53;
    }
};

// Greedy k-means++ (sklearn's rule) into kmeans.d_centres [K][D].  Per round: block sums of d2 -> host, T summed in rank
// then block order; L = 2 + floor(ln K) targets u T, each resolved on the rank that owns it (first event whose inclusive
// prefix exceeds the target; if rounding leaves none, the last event with d2 > 0); the candidates' potentials
// sum min(d2, d(x, c_l)) all-reduced; the lowest potential wins (lowest l on ties); d2 takes the winner in.
static int kmeanspp_run(gmm_ctx* c, int K, unsigned long long seed) {
    KmeansBuffers& b = c->kmeans;
    const int D = c->D, L = std::min(kSeedMaxCand, 2 + (int)std::floor(std::log((double)K)));
    SplitMix64 rng{seed};
    const long long g0 = std::min((long long)(rng.uniform() * (double)c->n_global), c->n_global - 1);
    CUDA_TRY(cudaMemsetAsync(b.d_centres, 0, sizeof(float) * (size_t)K * D, c->stream));
    if (g0 >= c->offset && g0 < c->offset + c->n)
        CUDA_TRY(cudaMemcpyAsync(b.d_centres, c->d_x_aos + (size_t)(g0 - c->offset) * D, sizeof(float) * D, cudaMemcpyDeviceToDevice, c->stream));
    if (int rc = kmeans_sum_rows(c, b.d_centres, (size_t)D)) return rc;
    if (K > 1)
        if (int rc = kmeanspp_update(c, b.d_centres, true)) return rc;
    std::vector<double> all, prefix((size_t)b.nb);
    for (int k = 1; k < K; k++) {
        // T: this rank's block sums in block order, then the ranks in rank order
        if (c->n > 0) CUDA_TRY(cudaMemcpyAsync(b.h_bsum, b.d_bsum, sizeof(double) * b.nb, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));
        const int nb = c->n > 0 ? b.nb : 0;
        double Tr = 0.0;
        for (int i = 0; i < nb; i++) Tr += b.h_bsum[i];
        if (int rc = kmeans_rank_values(c, &Tr, 1, all)) return rc;
        double T = 0.0, base = 0.0;
        std::vector<double> Q((size_t)c->nranks);
        for (int r = 0; r < c->nranks; r++) {
            if (r == c->rank) base = T;
            T += all[(size_t)r];
            Q[(size_t)r] = T;
        }
        if (!(T > 0.0)) {                                  // fewer distinct events than K: the rest repeat the first centre
            for (int j = k; j < K; j++)
                CUDA_TRY(cudaMemcpyAsync(b.d_centres + (size_t)j * D, b.d_centres, sizeof(float) * D, cudaMemcpyDeviceToDevice, c->stream));
            break;
        }
        {                                                  // this rank's inclusive block prefixes, continuing from the ranks before it
            double run = base;
            for (int i = 0; i < nb; i++) prefix[(size_t)i] = (run += b.h_bsum[i]);
        }
        int last_block = -1;                               // last block of this rank with a positive sum
        for (int i = nb - 1; i >= 0 && last_block < 0; i--)
            if (b.h_bsum[i] > 0.0) last_block = i;
        int last_rank = -1;
        for (int r = c->nranks - 1; r >= 0 && last_rank < 0; r--)
            if (all[(size_t)r] > 0.0) last_rank = r;
        for (int l = 0; l < L; l++) {
            const double t = rng.uniform() * T;
            SeedPick p{-1, 0, 0.0, 0.0};
            int owner = -1;
            for (int r = 0; r < c->nranks && owner < 0; r++)
                if (Q[(size_t)r] > t) owner = r;
            const bool fallback = owner < 0;
            if (fallback) owner = last_rank;
            if (owner == c->rank) {
                const int blk = fallback ? nb : (int)(std::upper_bound(prefix.begin(), prefix.begin() + nb, t) - prefix.begin());
                if (blk < nb) { p.block = blk; p.start = blk > 0 ? prefix[(size_t)blk - 1] : base; p.target = t; }
                else { p.block = last_block; p.start = 0.0; p.target = INFINITY; }
            }
            b.h_pick[l] = p;
        }
        CUDA_TRY(cudaMemcpyAsync(b.d_pick, b.h_pick, sizeof(SeedPick) * L, cudaMemcpyHostToDevice, c->stream));
        CUDA_TRY(cudaMemsetAsync(b.d_cand, 0, sizeof(float) * (size_t)L * D, c->stream));
        if (c->n > 0) {
            kmeanspp_pick_kernel<<<L, 32, 0, c->stream>>>(b.d_d2, c->n, b.d_pick, c->d_x_aos, D, b.d_cand, b.d_pick_idx);
            CUDA_TRY(cudaGetLastError());
        }
        if (int rc = kmeans_sum_rows(c, b.d_cand, (size_t)L * D)) return rc;
        if (int rc = kmeanspp_potential(c, L)) return rc;
        if (c->n > 0) CUDA_TRY(cudaMemcpyAsync(b.h_bpot, b.d_bpot, sizeof(double) * b.nb * kSeedMaxCand, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));
        double pot[kSeedMaxCand] = {0};
        for (int i = 0; i < nb; i++)
            for (int l = 0; l < L; l++) pot[l] += b.h_bpot[(size_t)i * kSeedMaxCand + l];
        if (int rc = kmeans_rank_values(c, pot, L, all)) return rc;
        int best = 0;
        double best_pot = INFINITY;
        for (int l = 0; l < L; l++) {
            double s = 0.0;
            for (int r = 0; r < c->nranks; r++) s += all[(size_t)r * L + l];
            if (s < best_pot) { best_pot = s; best = l; }
        }
        CUDA_TRY(cudaMemcpyAsync(b.d_centres + (size_t)k * D, b.d_cand + (size_t)best * D, sizeof(float) * D, cudaMemcpyDeviceToDevice, c->stream));
        if (k + 1 < K)
            if (int rc = kmeanspp_update(c, b.d_centres + (size_t)k * D, false)) return rc;
    }
    return GMM_OK;
}

// One Lloyd assignment to kmeans.d_centres: one-hot rows into d_memb, labels; global changed count and inertia.
static int kmeans_assign(gmm_ctx* c, int K, long long* changed, double* inertia) {
    KmeansBuffers& b = c->kmeans;
    const int Kw = std::min((c->Kmax + 7) / 8 * 8, (K + 31) / 32 * 32);
    if (int rc = kmeans_assign_launch(c, K, Kw)) return rc;
    if (c->n > 0) {
        CUDA_TRY(cudaMemcpyAsync(b.h_bchanged, b.d_bchanged, sizeof(int) * b.nba, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(cudaMemcpyAsync(b.h_binertia, b.d_binertia, sizeof(double) * b.nba, cudaMemcpyDeviceToHost, c->stream));
    }
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    double mine[2] = {0.0, 0.0};
    if (c->n > 0)
        for (int i = 0; i < b.nba; i++) { mine[0] += (double)b.h_bchanged[i]; mine[1] += b.h_binertia[i]; }
    std::vector<double> all;
    if (int rc = kmeans_rank_values(c, mine, 2, all)) return rc;
    double ch = 0.0, in = 0.0;
    for (int r = 0; r < c->nranks; r++) { ch += all[(size_t)r * 2]; in += all[(size_t)r * 2 + 1]; }
    *changed = (long long)ch;
    *inertia = in;
    return GMM_OK;
}

int gmm_seed_kmeans(gmm_ctx* c, int K, int max_iter, unsigned long long seed, clusters_t* host_out, float* centres_out,
                    int* iters_out, double* inertia_out) {
    if (int rc = check_K(c, K, "gmm_seed_kmeans")) return rc;
    if ((long long)K > c->n_global) return fail(GMM_ERR_ARG, "gmm_seed_kmeans: K exceeds the number of events");
    if (max_iter < 0) return fail(GMM_ERR_ARG, "gmm_seed_kmeans: max_iter < 0");
    CUDA_TRY(cudaSetDevice(c->device));
    if (int rc = ensure_moments(c)) return rc;             // centre and avgvar fixed before the first M-step
    if (int rc = kmeans_buffers(c)) return rc;
    KmeansBuffers& b = c->kmeans;
    const int D = c->D, F = c->F;
    c->memb_valid = false;
    struct Unweighted {                                    // seeding ignores the weights (gmm.h), on every return path
        gmm_ctx* c;
        explicit Unweighted(gmm_ctx* cc) : c(cc) { c->seeding = true; }
        ~Unweighted() { c->seeding = false; }
    } unweighted(c);
    if (int rc = kmeanspp_run(c, K, seed)) return rc;
    std::vector<float> cent((size_t)K * D);
    CUDA_TRY(cudaMemcpyAsync(cent.data(), b.d_centres, sizeof(float) * cent.size(), cudaMemcpyDeviceToHost, c->stream));
    if (c->n > 0) CUDA_TRY(cudaMemsetAsync(b.d_labels, 0xff, sizeof(int) * (size_t)c->n, c->stream));   // -1: every label changes once
    if (int rc = zero_stats(c, K)) return rc;
    // Lloyd: assignment + M-step on its one-hot memberships; the centre update is shift + S1 / S0 (S0 = 0 keeps the centre)
    long long changed = 0;
    double inertia = 0.0;
    if (int rc = kmeans_assign(c, K, &changed, &inertia)) return rc;
    if (int rc = run_mstep_accumulate(c, K)) return rc;
    if (int rc = reduce_stats_to_host(c, K)) return rc;
    int iters = 0;
    while (iters < max_iter) {
        for (int k = 0; k < K; k++) {
            const double* s = c->h_stats + (size_t)k * F;
            if (s[0] != 0.0)
                for (int d = 0; d < D; d++) cent[(size_t)k * D + d] = (float)(c->shift[d] + s[1 + d] / s[0]);
        }
        CUDA_TRY(cudaMemcpyAsync(b.d_centres, cent.data(), sizeof(float) * cent.size(), cudaMemcpyHostToDevice, c->stream));
        iters++;
        if (int rc = kmeans_assign(c, K, &changed, &inertia)) return rc;
        if (changed == 0) break;                           // same labels: the last M-step's statistics still hold
        if (int rc = run_mstep_accumulate(c, K)) return rc;
        if (int rc = reduce_stats_to_host(c, K)) return rc;
    }
    // the mixture of the final assignment: avgvar as gmm_seed sets it, then the M-step finalisation and the constants;
    // uploaded as gmm_set_clusters uploads parameters
    seed_from_moments(c->sum_x, c->sum_x2, c->n_global, D, K, cent.data(), &c->host);
    finalize_from_stats(c->h_stats, c->shift, K, D, &c->host, c->host_threads, /*with_constants=*/false);
    constants_from_R(K, D, &c->host, c->host_threads);
    if (int rc = upload_params(c, K)) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    c->memb_valid = false;
    collect_all(c);
    if (host_out) copy_params(host_out, &c->host, K, D);
    if (centres_out) std::memcpy(centres_out, cent.data(), sizeof(float) * cent.size());
    if (iters_out) *iters_out = iters;
    if (inertia_out) *inertia_out = inertia;
    return GMM_OK;
}

// ---- variational Bayesian mixture (gmm_vb_em) -----------------------------------------------------------------------------
// The default prior moments from the context's own M-step at K = 1 on unit responsibilities: the Lloyd assignment kernel
// with one centre writes a row of ones (and zeros in the rows the tensor M-step's cluster boxes read), and the weights
// enter as in every M-step.  mean = s + S1 / S0, covariance = (S2 - S1 S1^T / S0) / (S0 - 1): np.cov's ddof = 1, with
// denominator sum w - 1 under weights.  Overwrites the device memberships.
static int vb_default_moments(gmm_ctx* c, double* mean, double* cov) {
    if (int rc = kmeans_buffers(c)) return rc;
    const int D = c->D, Kw = std::min((c->Kmax + 7) / 8 * 8, 32);
    CUDA_TRY(cudaMemsetAsync(c->kmeans.d_centres, 0, sizeof(float) * D, c->stream));
    c->memb_valid = false;
    if (int rc = kmeans_assign_launch(c, 1, Kw)) return rc;
    if (int rc = run_mstep_accumulate(c, 1)) return rc;
    if (int rc = reduce_stats_to_host(c, 1)) return rc;
    const double* s = c->h_stats;
    const double S0 = s[0];
    if (!(S0 > 1.0)) return fail(GMM_ERR_ARG, "gmm_vb_em: the default prior covariance needs a total weight above 1");
    for (int i = 0; i < D; i++) {
        mean[i] = c->shift[i] + s[1 + i] / S0;
        for (int j = 0; j <= i; j++) cov[i * D + j] = cov[j * D + i] = (s[feat2(D, i, j)] - s[1 + i] * s[1 + j] / S0) / (S0 - 1.0);
    }
    return GMM_OK;
}

// resp_entropy_kernel over the current memberships, its partials queued to the pinned mirror (read after the next stream
// synchronisation by vb_entropy_sum).  timer: the profile the kernel counts in (NULL: none).
static int vb_entropy_launch(gmm_ctx* c, int K, int* grid_out, PhaseTimer* timer) {
    c->ent_blocks = kEntropyBlocksPerSm * c->num_sms;
    if (int rc = c->d_ent.reserve((size_t)c->ent_blocks + 1)) return rc;
    if (int rc = c->h_ent.reserve((size_t)c->ent_blocks + 1)) return rc;
    const int nq = (c->n + 3) / 4;
    const int grid = std::max(1, std::min(c->ent_blocks, (nq + kEntropyThreads - 1) / kEntropyThreads));
    *grid_out = c->n > 0 ? grid : 0;
    if (c->n == 0) return GMM_OK;
    const float* w = step_weights(c);
    if (timer) timer_begin(c, *timer);
    if (w) resp_entropy_kernel<true><<<grid, kEntropyThreads, 0, c->stream>>>(c->d_memb, c->memb_pitch, c->n, K, w, c->d_ent);
    else resp_entropy_kernel<false><<<grid, kEntropyThreads, 0, c->stream>>>(c->d_memb, c->memb_pitch, c->n, K, nullptr, c->d_ent);
    if (timer) timer_end(c, *timer);
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaMemcpyAsync(c->h_ent, c->d_ent, sizeof(double) * grid, cudaMemcpyDeviceToHost, c->stream));
    return GMM_OK;
}

// sum_n w_n sum_k g ln g over all ranks: this rank's partials in block order, then one ncclAllReduce of one double.
static int vb_entropy_sum(gmm_ctx* c, int grid, double* out) {
    double s = 0.0;
    for (int i = 0; i < grid; i++) s += c->h_ent[i];
    if (c->nranks > 1) {
        double* slot = c->d_ent + c->ent_blocks;
        c->h_ent[c->ent_blocks] = s;
        CUDA_TRY(cudaMemcpyAsync(slot, c->h_ent + c->ent_blocks, sizeof(double), cudaMemcpyHostToDevice, c->stream));
        ncclResult_t r = nccl().AllReduce(slot, slot, 1, ncclDouble, ncclSum, c->comm, c->stream);
        if (r != ncclSuccess) return fail(GMM_ERR_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
        CUDA_TRY(cudaMemcpyAsync(c->h_ent + c->ent_blocks, slot, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));
        s = c->h_ent[c->ent_blocks];
    }
    *out = s;
    return GMM_OK;
}

// VB M-step from the reduced statistics in h_stats: the per-cluster part on the finalisation's worker team (K >= 8), the
// weights and the bound serially, then the parameter set uploaded as gmm_set_clusters uploads one (Rinv and constant kept).
static int vb_finalize_upload(gmm_ctx* c, int K, const VbPrior& p, std::vector<VbCluster>& cl, gmm_vb_posterior* post, double* bound) {
    auto t0 = std::chrono::steady_clock::now();
    const int D = c->D;
    run_clusters(c, K, K, [&](int k) { vb_finalize_cluster(c->h_stats, c->shift, k, D, p, &c->host, &cl[(size_t)k]); });
    int bad = -1;
    const int rc = vb_finalize_weights(K, D, p, cl.data(), &c->host, post, bound, &bad);
    c->vb_final_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (rc) {
        c->memb_valid = false;
        return fail(GMM_ERR_STATE, "gmm_vb_em: the covariance of component " + std::to_string(bad) + " is not positive definite in float");
    }
    return upload_params(c, K);
}

int gmm_vb_em(gmm_ctx* c, int K, const gmm_vb_prior* prior, int min_iters, int max_iters, double tol, clusters_t* host_out,
              gmm_vb_posterior* post_out, double* lower_bound_out, double* lower_bounds_out, int* iters_out, int* converged_out) {
    if (int rc = check_K(c, K, "gmm_vb_em")) return rc;
    if (!prior) return fail(GMM_ERR_ARG, "gmm_vb_em: NULL prior");
    if (min_iters < 0 || max_iters < min_iters) return fail(GMM_ERR_ARG, "gmm_vb_em: need 0 <= min_iters <= max_iters");
    if (!(tol >= 0.0)) return fail(GMM_ERR_ARG, "gmm_vb_em: tol must be >= 0");
    const int D = c->D;
    VbPrior p;
    if (int rc = vb_resolve_prior(prior, K, D, &p)) return rc;
    std::vector<double> mean((size_t)D, 0.0), cov((size_t)D * D, 0.0);
    for (int d = 0; d < D; d++) cov[(size_t)d * D + d] = 1.0;
    // the caller's moments are checked before anything runs (a NULL one stands in as 0 / I until the default is known)
    if (int rc = vb_set_prior_moments(prior->mean ? prior->mean : mean.data(), prior->covariance ? prior->covariance : cov.data(), D, &p))
        return rc;
    if (K != c->cur_K) return fail(GMM_ERR_STATE, "gmm_vb_em: parameters for this K have not been set (gmm_seed / gmm_set_clusters)");
    if (c->params_partial) return fail(GMM_ERR_STATE, "gmm_vb_em: called between gmm_mstep and gmm_constants");
    CUDA_TRY(cudaSetDevice(c->device));
    const auto t0 = std::chrono::steady_clock::now();
    if (int rc = ensure_moments(c)) return rc;
    if (!prior->mean || !prior->covariance) {
        if (int rc = vb_default_moments(c, mean.data(), cov.data())) return rc;
        if (int rc = vb_set_prior_moments(prior->mean ? prior->mean : mean.data(), prior->covariance ? prior->covariance : cov.data(), D, &p))
            return rc;
    }
    std::vector<VbCluster> cl((size_t)K);
    double bound_par = 0.0, lb = -std::numeric_limits<double>::infinity(), lb_prev = lb;
    // g0 under the starting set, posterior 0 from it (sklearn's _initialize)
    if (int rc = zero_stats(c, K)) return rc;
    if (int rc = run_estep(c, K)) return rc;
    if (int rc = run_mstep_accumulate(c, K)) return rc;
    if (int rc = reduce_stats_to_host(c, K)) return rc;
    if (int rc = vb_finalize_upload(c, K, p, cl, post_out, &bound_par)) return rc;
    int iters = 0, converged = 0;
    for (int i = 1; i <= max_iters; i++) {
        if (int rc = zero_stats(c, K)) return rc;
        if (int rc = run_estep(c, K)) return rc;
        if (int rc = run_mstep_accumulate(c, K)) return rc;
        // the bound of iteration i is used by the tol test of iterations i and i + 1
        const bool need_bound = lower_bounds_out != nullptr || i >= min_iters - 1;
        int grid = 0;
        if (need_bound)
            if (int rc = vb_entropy_launch(c, K, &grid, &c->t_entropy)) return rc;
        if (int rc = reduce_stats_to_host(c, K)) return rc;
        if (int rc = vb_finalize_upload(c, K, p, cl, post_out, &bound_par)) return rc;
        iters = i;
        c->iterations++;
        if (need_bound) {
            double ent = 0.0;
            if (int rc = vb_entropy_sum(c, grid, &ent)) return rc;
            lb = -ent + bound_par;
            if (lower_bounds_out) lower_bounds_out[i - 1] = lb;
        }
        if (i >= min_iters && std::fabs(lb - lb_prev) < tol) { converged = 1; break; }
        lb_prev = lb;
    }
    // the memberships of the final posterior (sklearn's last _e_step)
    if (int rc = zero_stats(c, K)) return rc;
    if (int rc = run_estep(c, K)) return rc;
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    collect_all(c);
    c->vb_wall_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (host_out) copy_params(host_out, &c->host, K, D);
    if (lower_bound_out) *lower_bound_out = lb;
    if (iters_out) *iters_out = iters;
    if (converged_out) *converged_out = converged;
    return GMM_OK;
}

int gmm_get_vb_profile(gmm_ctx* c, double out[3], int reset) {
    if (!c || !out) return fail(GMM_ERR_ARG, "gmm_get_vb_profile: bad argument");
    cudaStreamSynchronize(c->stream);
    collect_all(c);
    out[0] = c->t_entropy.total_ms; out[1] = c->vb_final_ms; out[2] = c->vb_wall_ms;
    if (reset) { c->t_entropy.total_ms = 0; c->vb_final_ms = c->vb_wall_ms = 0; }
    return GMM_OK;
}

// ---- combining mixture components (gmm_combine) ----------------------------------------------------------------------
// The memberships of the last E-step for K, complete and current.
static int check_memberships(const gmm_ctx* c, int K, const char* who) {
    if (int rc = check_fitted(c, K, who)) return rc;
    if (!c->memb_valid) return fail(GMM_ERR_STATE, std::string(who) + ": no E-step has run for the current parameters and weights");
    return GMM_OK;
}

static int combine_buffers(gmm_ctx* c, size_t part, size_t sum) {
    CombineBuffers& b = c->comb;
    if (int rc = b.d_groups.reserve(2 * kCombMaxK + 1)) return rc;
    if (int rc = b.h_groups.reserve(2 * kCombMaxK + 1)) return rc;
    if (int rc = b.t0.create(cudaEventDefault)) return rc;
    if (int rc = b.t1.create(cudaEventDefault)) return rc;
    if (int rc = b.d_part.reserve(part)) return rc;
    if (int rc = b.d_sum.reserve(sum)) return rc;
    if (int rc = b.h_sum.reserve(sum)) return rc;
    return GMM_OK;
}

// Groups as member lists for the step and label kernels: members of group i at [off[i], off[i + 1]) of the pinned staging,
// offsets after the kCombMaxK member slots; queued to the device.
static int combine_upload_groups(gmm_ctx* c, const std::vector<std::vector<int>>& groups) {
    int* h = c->comb.h_groups;
    int* off = h + kCombMaxK;
    int pos = 0;
    for (size_t i = 0; i < groups.size(); i++) {
        off[i] = pos;
        for (int k : groups[i]) h[pos++] = k;
    }
    off[groups.size()] = pos;
    CUDA_TRY(cudaMemcpyAsync(c->comb.d_groups, h, sizeof(int) * (2 * kCombMaxK + 1), cudaMemcpyHostToDevice, c->stream));
    return GMM_OK;
}

// partial [ranges][P] -> d_sum [P] summed in range order, all-reduced over the ranks, -> h_sum; the kernels since t0 are
// timed to t1 and the host waits.
static int combine_finish(gmm_ctx* c, int ranges, int P) {
    CombineBuffers& b = c->comb;
    if (ranges > 0) {
        const int grid = std::max(1, std::min(c->num_sms, (P + kCombSumThreads - 1) / kCombSumThreads));
        combine_sum_ranges_kernel<<<grid, kCombSumThreads, 0, c->stream>>>(b.d_part, ranges, P, b.d_sum);
        CUDA_TRY(cudaGetLastError());
    } else {
        CUDA_TRY(cudaMemsetAsync(b.d_sum, 0, sizeof(double) * P, c->stream));
    }
    if (c->nranks > 1) {
        ncclResult_t r = nccl().AllReduce(b.d_sum, b.d_sum, (size_t)P, ncclDouble, ncclSum, c->comm, c->stream);
        if (r != ncclSuccess) return fail(GMM_ERR_NCCL, std::string("ncclAllReduce: ") + nccl().GetErrorString(r));
    }
    CUDA_TRY(cudaEventRecord(b.t1, c->stream));
    CUDA_TRY(cudaMemcpyAsync(b.h_sum, b.d_sum, sizeof(double) * P, cudaMemcpyDeviceToHost, c->stream));
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    float ms = 0;
    if (cudaEventElapsedTime(&ms, b.t0, b.t1) == cudaSuccess) b.kernel_ms += ms;
    return GMM_OK;
}

static int combine_run(gmm_ctx* c, int K, int* merges_out, double* gain_out, double* entropy_out, double* mass_out) {
    CombineBuffers& b = c->comb;
    const int n = c->n, npairs = K * (K - 1) / 2, P = npairs + K;
    const float* w = step_weights(c);
    // all-pairs pass: ranges of 64-event multiples, about 4 CTAs per SM in all
    const int T = (K + kCombTile - 1) / kCombTile, tiles = T * (T + 1) / 2;
    const int max_ranges = std::max(1, (4 * c->num_sms + tiles - 1) / tiles);
    const long long n_units = ((long long)n + kCombPairEvents - 1) / kCombPairEvents;
    const int range_events = (int)std::max<long long>(1, (n_units + max_ranges - 1) / max_ranges) * kCombPairEvents;
    const int ranges1 = n > 0 ? (n + range_events - 1) / range_events : 0;
    // step pass: blocks of kCombStepEvents grid-strided over the CTAs one wave holds
    int per_sm = 0;
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, w ? combine_step_kernel<true> : combine_step_kernel<false>,
                                                           kCombStepThreads, 0));
    const int nblocks = (n + kCombStepEvents - 1) / kCombStepEvents;
    const int ranges2 = std::min(nblocks, std::max(per_sm, 1) * c->num_sms);
    if (int rc = combine_buffers(c, std::max({(size_t)ranges1 * P, (size_t)ranges2 * K, (size_t)1}), (size_t)P)) return rc;

    CUDA_TRY(cudaEventRecord(b.t0, c->stream));
    int egrid = 0;
    if (int rc = vb_entropy_launch(c, K, &egrid, nullptr)) return rc;
    if (ranges1 > 0) {
        const dim3 grid(tiles, ranges1);
        if (w) combine_pairs_kernel<true><<<grid, kCombPairThreads, 0, c->stream>>>(c->d_memb, c->memb_pitch, n, K, w, range_events, b.d_part, P);
        else combine_pairs_kernel<false><<<grid, kCombPairThreads, 0, c->stream>>>(c->d_memb, c->memb_pitch, n, K, nullptr, range_events, b.d_part, P);
        CUDA_TRY(cudaGetLastError());
    }
    if (int rc = combine_finish(c, ranges1, P)) return rc;
    double ent = 0.0;
    if (int rc = vb_entropy_sum(c, egrid, &ent)) return rc;
    std::vector<double> mk(b.h_sum + npairs, b.h_sum + P);
    for (int k = 0; k < K; k++)
        if (!std::isfinite(mk[(size_t)k]))
            return fail(GMM_ERR_STATE, "gmm_combine: the memberships of component " + std::to_string(k) + " are not finite");
    std::vector<double> gain((size_t)K * K, 0.0);           // gain[a K + b], a < b the groups' smallest components
    for (int a = 0; a < K; a++)
        for (int bb = a + 1; bb < K; bb++) gain[(size_t)a * K + bb] = b.h_sum[combine_pair_index(a, bb, K)];
    std::vector<std::vector<int>> members((size_t)K);
    for (int k = 0; k < K; k++) members[(size_t)k] = {k};
    std::vector<int> live((size_t)K);
    for (int k = 0; k < K; k++) live[(size_t)k] = k;
    std::vector<double> gains((size_t)std::max(K - 1, 0));
    auto group_mass = [&](int r) {
        double m = 0.0;
        for (int k : members[(size_t)r]) m += mk[(size_t)k];
        return m;
    };
    for (int s = 0; s < K - 1; s++) {
        // the live pair of largest gain; strict > over the pairs in lexicographic order keeps the smallest (a, b) of a tie
        int ba = -1, bb = -1;
        double bg = 0.0;
        for (size_t i = 0; i < live.size(); i++)
            for (size_t j = i + 1; j < live.size(); j++) {
                const double g = gain[(size_t)live[i] * K + live[j]];
                if (ba < 0 || g > bg) { ba = live[i]; bb = live[j]; bg = g; }
            }
        merges_out[2 * s] = ba;
        merges_out[2 * s + 1] = bb;
        gains[(size_t)s] = bg;
        if (mass_out) mass_out[s] = group_mass(ba) + group_mass(bb);
        std::vector<int>& ma = members[(size_t)ba];
        ma.insert(ma.end(), members[(size_t)bb].begin(), members[(size_t)bb].end());
        std::sort(ma.begin(), ma.end());
        members[(size_t)bb].clear();
        live.erase(std::find(live.begin(), live.end(), bb));
        if (s == K - 2) break;
        // step pass: the merged group against every other live group
        const int L = (int)live.size();
        const int gi = (int)(std::find(live.begin(), live.end(), ba) - live.begin());
        std::vector<std::vector<int>> groups((size_t)L);
        for (int i = 0; i < L; i++) groups[(size_t)i] = members[(size_t)live[(size_t)i]];
        if (int rc = combine_upload_groups(c, groups)) return rc;
        CUDA_TRY(cudaEventRecord(b.t0, c->stream));
        if (ranges2 > 0) {
            const int* mem = b.d_groups;
            const int* off = b.d_groups + kCombMaxK;
            if (w) combine_step_kernel<true><<<ranges2, kCombStepThreads, 0, c->stream>>>(c->d_memb, c->memb_pitch, n, w, mem, off, L, gi, b.d_part);
            else combine_step_kernel<false><<<ranges2, kCombStepThreads, 0, c->stream>>>(c->d_memb, c->memb_pitch, n, nullptr, mem, off, L, gi, b.d_part);
            CUDA_TRY(cudaGetLastError());
        }
        if (int rc = combine_finish(c, ranges2, L)) return rc;
        for (int i = 0; i < L; i++) {
            if (i == gi) continue;
            const int h = live[(size_t)i];
            gain[(size_t)std::min(ba, h) * K + std::max(ba, h)] = b.h_sum[i];
        }
    }
    if (gain_out) std::copy(gains.begin(), gains.end(), gain_out);
    if (entropy_out) {
        entropy_out[K - 1] = -ent;
        for (int L = K; L >= 2; L--) entropy_out[L - 2] = entropy_out[L - 1] - gains[(size_t)(K - L)];
    }
    return GMM_OK;
}

int gmm_combine(gmm_ctx* c, int K, int* merges_out, double* gain_out, double* entropy_out, double* mass_out) {
    if (int rc = check_K(c, K, "gmm_combine")) return rc;
    if (K >= 2 && !merges_out) return fail(GMM_ERR_ARG, "gmm_combine: NULL merges_out with K >= 2");
    if (int rc = check_memberships(c, K, "gmm_combine")) return rc;
    CUDA_TRY(cudaSetDevice(c->device));
    const auto t0 = std::chrono::steady_clock::now();
    const int rc = combine_run(c, K, merges_out, gain_out, entropy_out, mass_out);
    c->comb.wall_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return rc;
}

int gmm_combine_labels(gmm_ctx* c, int K, const int* group, int G, int* labels_out, float* max_out) {
    if (int rc = check_K(c, K, "gmm_combine_labels")) return rc;
    if (!group || G < 1 || G > K || (c->n > 0 && !labels_out))
        return fail(GMM_ERR_ARG, "gmm_combine_labels: bad argument (need group, 1 <= G <= K and labels_out)");
    std::vector<std::vector<int>> groups((size_t)G);
    for (int k = 0; k < K; k++) {
        if (group[k] < 0 || group[k] >= G)
            return fail(GMM_ERR_ARG, "gmm_combine_labels: group[" + std::to_string(k) + "] is outside [0, G)");
        groups[(size_t)group[k]].push_back(k);
    }
    if (int rc = check_memberships(c, K, "gmm_combine_labels")) return rc;
    CUDA_TRY(cudaSetDevice(c->device));
    const auto t0 = std::chrono::steady_clock::now();
    CombineBuffers& b = c->comb;
    if (int rc = combine_buffers(c, 1, 1)) return rc;
    if (int rc = b.d_lab.reserve(c->memb_pitch)) return rc;
    if (int rc = b.d_max.reserve(c->memb_pitch)) return rc;
    if (c->n > 0) {
        if (int rc = combine_upload_groups(c, groups)) return rc;
        const int nq = (c->n + 3) / 4;
        const int grid = std::max(1, std::min(8 * c->num_sms, (nq + kCombLabelThreads - 1) / kCombLabelThreads));
        CUDA_TRY(cudaEventRecord(b.t0, c->stream));
        combine_labels_kernel<<<grid, kCombLabelThreads, 0, c->stream>>>(c->d_memb, c->memb_pitch, c->n, b.d_groups, b.d_groups + kCombMaxK,
                                                                         G, b.d_lab, b.d_max);
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaEventRecord(b.t1, c->stream));
        CUDA_TRY(cudaMemcpyAsync(labels_out, b.d_lab, sizeof(int) * c->n, cudaMemcpyDeviceToHost, c->stream));
        if (max_out) CUDA_TRY(cudaMemcpyAsync(max_out, b.d_max, sizeof(float) * c->n, cudaMemcpyDeviceToHost, c->stream));
        CUDA_TRY(cudaStreamSynchronize(c->stream));
        float ms = 0;
        if (cudaEventElapsedTime(&ms, b.t0, b.t1) == cudaSuccess) b.kernel_ms += ms;
    }
    b.labels_wall_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return GMM_OK;
}

int gmm_get_combine_profile(gmm_ctx* c, double out[3], int reset) {
    if (!c || !out) return fail(GMM_ERR_ARG, "gmm_get_combine_profile: bad argument");
    out[0] = c->comb.kernel_ms; out[1] = c->comb.wall_ms; out[2] = c->comb.labels_wall_ms;
    if (reset) c->comb.kernel_ms = c->comb.wall_ms = c->comb.labels_wall_ms = 0;
    return GMM_OK;
}

// ---- sampling from the mixture ------------------------------------------------------------------------------------------
// The parameter block of the current K clusters (kernels_sample.cuh layout) in the pinned staging, with the checks of
// gmm.h in cluster order.  *klast = the last cluster with pi > 0.
static int sample_params(gmm_ctx* c, int K, int* klast) {
    const int D = c->D, REC = sample_rec_floats(D);
    double* cum = reinterpret_cast<double*>(c->sample.h_block.get());
    float* rec = reinterpret_cast<float*>(cum + sample_cum_len(K));
    double run = 0.0;
    *klast = -1;
    for (int k = 0; k < K; k++) {
        const float p = c->host.pi[k];
        if (!(p >= 0.0f) || !std::isfinite(p))
            return fail(GMM_ERR_STATE, "gmm_sample: pi of cluster " + std::to_string(k) + " is negative or not finite");
        double U[GMM_MAX_DIMENSIONS][GMM_MAX_DIMENSIONS], ld;
        if (!reverse_cholesky(c->host.R + (size_t)k * D * D, D, U, &ld))
            return fail(GMM_ERR_STATE, "gmm_sample: R of cluster " + std::to_string(k) + " is not positive definite");
        run += (double)p;
        cum[k] = run;
        if (p > 0.0f) *klast = k;
        float* r = rec + (size_t)k * REC;
        int e = 0;
        for (int d = 0; d < D; d++) {
            r[e++] = c->host.means[(size_t)k * D + d];
            for (int j = d; j < D; j++) r[e++] = (float)U[d][j];
        }
        for (; e < REC; e++) r[e] = 0.0f;
    }
    if (!(run > 0.0)) return fail(GMM_ERR_STATE, "gmm_sample: the mixing weights pi sum to zero");
    return GMM_OK;
}

// gmm_sample's chunks through the pipeline without its input half: sample_kernel writes the slot's device chunk (rows) and
// label area, the copy stream brings them to the slot's pinned stages, the host copies them to the caller's arrays.
static int sample_batch(gmm_ctx* c, int K, int klast, unsigned long long seed, long long first, long long n, float* events,
                        int* labels) {
    ScoreBuffers& s = c->score;
    const int D = c->D;
    CUDA_TRY(cudaMemcpyAsync(c->sample.d_block, c->sample.h_block, sample_block_bytes(K, D), cudaMemcpyHostToDevice, c->stream));
    // the parameters go to shared memory when they fit beside the output tile with two blocks per SM (D = 24: K <= 66)
    const size_t staged = sample_tile_bytes(D) + sample_block_bytes(K, D);
    const int stage = staged <= (size_t)kSampleStageBytes ? 1 : 0;
    const size_t smem = stage ? staged : sample_tile_bytes(D);
    int per_sm = 0;
#define GMM_CALL(d)                                                                                                   \
    do {                                                                                                              \
        CUDA_TRY(cudaFuncSetAttribute(sample_kernel<d>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));    \
        CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sample_kernel<d>, kSampleThreads, smem));    \
    } while (0)
    GMM_SEED_DISPATCH(D, GMM_CALL)
#undef GMM_CALL
    const long long max_grid = (long long)std::max(per_sm, 1) * c->num_sms;
    auto labels_of = [&](char* base) { return reinterpret_cast<int*>(base + ScoreBuffers::kHeader); };
    auto launch = [&](int b, long long e0, int m) -> int {
        const int grid = (int)std::min<long long>((m + kSampleThreads - 1) / kSampleThreads, max_grid);
        int* d_lab = labels_of(s.d_out[b]);
        CUDA_TRY(cudaEventRecord(s.t0[b], c->stream));
#define GMM_CALL(d) \
    sample_kernel<d><<<grid, kSampleThreads, smem, c->stream>>>(c->sample.d_block, K, klast, stage, seed, first + e0, m, s.d_in[b], d_lab)
        GMM_SEED_DISPATCH(D, GMM_CALL)
#undef GMM_CALL
        CUDA_TRY(cudaGetLastError());
        CUDA_TRY(cudaEventRecord(s.t1[b], c->stream));
        return GMM_OK;
    };
    auto fetch = [&](int b, int m, cudaStream_t st) -> int {
        CUDA_TRY(cudaMemcpyAsync(s.h_in[b], s.d_in[b], sizeof(float) * (size_t)m * D, cudaMemcpyDeviceToHost, st));
        if (labels) CUDA_TRY(cudaMemcpyAsync(labels_of(s.h_out[b]), labels_of(s.d_out[b]), sizeof(int) * (size_t)m, cudaMemcpyDeviceToHost, st));
        return GMM_OK;
    };
    auto hand_over = [&](int b, long long e0, int m) -> int {
        std::memcpy(events + (size_t)e0 * D, s.h_in[b], sizeof(float) * (size_t)m * D);
        if (labels) std::memcpy(labels + e0, labels_of(s.h_out[b]), sizeof(int) * (size_t)m);
        return GMM_OK;
    };
    return stream_chunks(c, n, nullptr, 0, &c->sample.kernel_ms, launch, fetch, hand_over);
}
#undef GMM_SEED_CASE
#undef GMM_SEED_DISPATCH

int gmm_sample(gmm_ctx* c, int K, long long n, unsigned long long seed, long long first, float* events_out, int* labels_out) {
    if (int rc = check_K(c, K, "gmm_sample")) return rc;
    if (n < 0 || first < 0 || first > (1LL << 62) - n || (n > 0 && !events_out))
        return fail(GMM_ERR_ARG, "gmm_sample: bad range or output (n < 0, first < 0, first + n > 2^62, or no event array)");
    if (int rc = check_fitted(c, K, "gmm_sample")) return rc;
    CUDA_TRY(cudaSetDevice(c->device));
    const auto t0 = std::chrono::steady_clock::now();
    SampleBuffers& sb = c->sample;
    if (int rc = sb.d_block.reserve(sample_block_bytes(c->Kmax, c->D) / sizeof(double))) return rc;   // a multiple of 16 bytes
    if (int rc = sb.h_block.reserve(sample_block_bytes(c->Kmax, c->D))) return rc;
    int klast = 0;
    int rc = sample_params(c, K, &klast);
    if (rc == GMM_OK && n > 0) {
        rc = score_buffers(c);
        if (rc == GMM_OK) rc = sample_batch(c, K, klast, seed, first, n, events_out, labels_out);
        rc = drain_streams(c, rc, "gmm_sample");
    }
    sb.wall_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return rc;
}

int gmm_get_sample_profile(gmm_ctx* c, double out[2], int reset) {
    if (!c || !out) return fail(GMM_ERR_ARG, "gmm_get_sample_profile: bad argument");
    out[0] = c->sample.kernel_ms; out[1] = c->sample.wall_ms;
    if (reset) c->sample.kernel_ms = c->sample.wall_ms = 0;
    return GMM_OK;
}

// ---- events measured on a subset of the dimensions ----------------------------------------------------------------------
// Floats of one cluster's record in gmm_condition's block: the marginal epack record (no imputation), or the
// kernels_condition.cuh record.
static int condition_rec_floats(int n_obs, int nm, bool impute) {
    return impute ? cond_rec_floats(cond_round4(n_obs), cond_round4(nm)) : epack_stride(n_obs);
}
static size_t condition_block_floats(int Kmax, int D) {
    int rec = epack_stride(D);
    for (int o = 1; o < D; o++) rec = std::max(rec, condition_rec_floats(o, D - o, true));
    return (size_t)Kmax * rec;
}

// gmm_condition's parameter block and its pinned mirror, allocated on the first call of either conditioning call.
static int condition_block(gmm_ctx* c) {
    ConditionBuffers& cb = c->cond;
    if (int rc = cb.d_block.reserve(condition_block_floats(c->Kmax, c->D))) return rc;
    if (int rc = cb.h_block.reserve(condition_block_floats(c->Kmax, c->D))) return rc;
    return GMM_OK;
}

// The parameter block of the current K clusters in the pinned mirror (gmm.h): the marginal set (mu_O, P_O, constant_O,
// pi) goes through build_epack, at n_obs dimensions for score_simt_kernel, or zero-padded to a multiple of 4 and followed
// by mu_M, G and c for condition_simt_kernel.  With nm = 0 the marginal set is the context's own arrays.  g_d [K][nm][n_obs]
// and c_d [K][nm][nm], when not NULL, receive G and S_MM^-1 in double (gmm_condition_stats); `who` names the caller in errors.
static int condition_params(gmm_ctx* c, int K, const int* obs, int n_obs, const int* mis, int nm, bool impute,
                            const char* who = "gmm_condition", double* g_d = nullptr, double* c_d = nullptr) {
    const int D = c->D;
    float* block = c->cond.h_block;
    if (nm == 0) {
        build_epack(K, D, &c->host, block);
        return GMM_OK;
    }
    const int DO = impute ? cond_round4(n_obs) : n_obs, NM = cond_round4(nm);
    std::vector<float> mo((size_t)K * DO, 0.0f), po((size_t)K * DO * DO, 0.0f), co(K), g((size_t)K * nm * n_obs), cv((size_t)K * nm);
    std::atomic<int> first_bad{K};
    const std::function<void(int)> per_cluster = [&](int k) {
        std::vector<float> p((size_t)n_obs * n_obs);
        if (!condition_cluster(&c->host, k, D, obs, n_obs, mis, nm, p.data(), &co[k], &g[(size_t)k * nm * n_obs], &cv[(size_t)k * nm],
                               g_d ? g_d + (size_t)k * nm * n_obs : nullptr, c_d ? c_d + (size_t)k * nm * nm : nullptr)) {
            int cur = first_bad.load();
            while (k < cur && !first_bad.compare_exchange_weak(cur, k)) {}
            return;
        }
        for (int a = 0; a < n_obs; a++) {
            mo[(size_t)k * DO + a] = c->host.means[(size_t)k * D + obs[a]];
            for (int b = 0; b < n_obs; b++) po[(size_t)k * DO * DO + a * DO + b] = p[(size_t)a * n_obs + b];
        }
    };
    run_clusters(c, K, K, per_cluster);
    if (first_bad.load() < K)
        return fail(GMM_ERR_STATE, std::string(who) + ": the block P_MM of cluster " + std::to_string(first_bad.load()) +
                                       " (inverse covariance on the missing dimensions) is not positive definite");
    clusters_t marg{};
    marg.means = mo.data(); marg.Rinv = po.data(); marg.constant = co.data(); marg.pi = c->host.pi;
    if (!impute) {
        build_epack(K, DO, &marg, block);
        return GMM_OK;
    }
    const int EP = epack_stride(DO), REC = condition_rec_floats(n_obs, nm, true);
    std::vector<float> ep((size_t)K * EP);
    build_epack(K, DO, &marg, ep.data());
    std::memset(block, 0, sizeof(float) * (size_t)K * REC);
    for (int k = 0; k < K; k++) {
        float* r = block + (size_t)k * REC;
        std::memcpy(r, &ep[(size_t)k * EP], sizeof(float) * EP);
        float* mu = r + EP;
        float* G = mu + NM;
        float* cvar = G + (size_t)NM * DO;
        for (int d = 0; d < nm; d++) {
            mu[d] = c->host.means[(size_t)k * D + mis[d]];
            for (int o = 0; o < n_obs; o++) G[d * DO + o] = g[((size_t)k * nm + d) * n_obs + o];
            cvar[d] = cv[(size_t)k * nm + d];
        }
    }
    return GMM_OK;
}

// condition_simt_kernel<NO, NM> for the observed / imputed counts rounded up to multiples of 4 (NO + NM <= 36: 36 instances)
static int launch_condition(gmm_ctx* c, int n_obs, int nm, int K, const float* block, const TcScoreIo& io, float* mean, float* var) {
    if (io.n <= 0) return GMM_OK;
    const int grid = (io.n + kEstepThreads - 1) / kEstepThreads;
    switch (cond_round4(n_obs) / 4 * 16 + cond_round4(nm) / 4) {
#define GMM_CASE(a, b)                                                                                                          \
    case (a) * 16 + (b):                                                                                                        \
        condition_simt_kernel<4 * (a), 4 * (b)><<<grid, kEstepThreads, 0, c->stream>>>(io.x, io.n, n_obs, nm, K, block, io.labels, \
                                                                                      io.max_resp, io.logp, io.ll, mean, var);  \
        break;
        GMM_CASE(1, 1) GMM_CASE(1, 2) GMM_CASE(1, 3) GMM_CASE(1, 4) GMM_CASE(1, 5) GMM_CASE(1, 6) GMM_CASE(1, 7) GMM_CASE(1, 8)
        GMM_CASE(2, 1) GMM_CASE(2, 2) GMM_CASE(2, 3) GMM_CASE(2, 4) GMM_CASE(2, 5) GMM_CASE(2, 6) GMM_CASE(2, 7)
        GMM_CASE(3, 1) GMM_CASE(3, 2) GMM_CASE(3, 3) GMM_CASE(3, 4) GMM_CASE(3, 5) GMM_CASE(3, 6)
        GMM_CASE(4, 1) GMM_CASE(4, 2) GMM_CASE(4, 3) GMM_CASE(4, 4) GMM_CASE(4, 5)
        GMM_CASE(5, 1) GMM_CASE(5, 2) GMM_CASE(5, 3) GMM_CASE(5, 4)
        GMM_CASE(6, 1) GMM_CASE(6, 2) GMM_CASE(6, 3)
        GMM_CASE(7, 1) GMM_CASE(7, 2)
        GMM_CASE(8, 1)
#undef GMM_CASE
        default: return fail(GMM_ERR_ARG, "gmm_condition: unsupported split of the dimensions");
    }
    CUDA_TRY(cudaGetLastError());
    return GMM_OK;
}

// gmm_condition's chunks through the pipeline: the marginal score kernel, or the imputing one whose conditional means and
// variances come back beside the scores.
static int condition_batch(gmm_ctx* c, int K, int n_obs, int nm, bool impute, const float* ev, long long n, const ScoreOut& out,
                           float* cmean, float* cvar) {
    ScoreBuffers& s = c->score;
    ConditionBuffers& cb = c->cond;
    const size_t var_off = (size_t)c->score_chunk * nm;    // cond_var's offset in a slot's imputation buffer
    CUDA_TRY(cudaMemcpyAsync(cb.d_block, cb.h_block, sizeof(float) * (size_t)K * condition_rec_floats(n_obs, nm, impute),
                             cudaMemcpyHostToDevice, c->stream));
    auto launch = [&](int b, long long, int m) -> int {
        const TcScoreIo dv = score_io(c, s.d_out[b], b, m);
        CUDA_TRY(cudaMemsetAsync(s.d_out[b], 0, ScoreBuffers::kHeader, c->stream));
        CUDA_TRY(cudaEventRecord(s.t0[b], c->stream));
        const int rc = impute ? launch_condition(c, n_obs, nm, K, cb.d_block, dv, cb.d_imp[b], cvar ? cb.d_imp[b] + var_off : nullptr)
                              : launch_score_simt(c, n_obs, K, cb.d_block, dv);
        if (rc) return rc;
        CUDA_TRY(cudaEventRecord(s.t1[b], c->stream));
        return GMM_OK;
    };
    auto fetch = [&](int b, int m, cudaStream_t st) -> int {
        if (int rc = fetch_scores(c, out, b, m, st)) return rc;
        if (impute && cmean) CUDA_TRY(cudaMemcpyAsync(cb.h_imp[b], cb.d_imp[b], sizeof(float) * (size_t)m * nm, cudaMemcpyDeviceToHost, st));
        if (impute && cvar)
            CUDA_TRY(cudaMemcpyAsync(cb.h_imp[b] + var_off, cb.d_imp[b] + var_off, sizeof(float) * (size_t)m * nm, cudaMemcpyDeviceToHost, st));
        return GMM_OK;
    };
    auto hand_over = [&](int b, long long e0, int m) -> int {
        hand_over_scores(c, out, b, e0, m);
        if (impute && cmean) std::memcpy(cmean + (size_t)e0 * nm, cb.h_imp[b], sizeof(float) * (size_t)m * nm);
        if (impute && cvar) std::memcpy(cvar + (size_t)e0 * nm, cb.h_imp[b] + var_off, sizeof(float) * (size_t)m * nm);
        return GMM_OK;
    };
    return stream_chunks(c, n, ev, n_obs, &cb.kernel_ms, launch, fetch, hand_over);
}

int gmm_condition(gmm_ctx* c, int K, const int* obs_dims, int n_obs, const float* events_obs, long long n, int* labels,
                  float* max_resp, float* logp, float* cond_mean, float* cond_var, double* loglik_out) {
    if (int rc = check_K(c, K, "gmm_condition")) return rc;
    if (n < 0 || (n > 0 && !events_obs)) return fail(GMM_ERR_ARG, "gmm_condition: bad events (n < 0, or no rows)");
    int mis[GMM_MAX_DIMENSIONS], nm = 0;
    unsigned obs_mask = 0;
    if (int rc = split_obs(c, obs_dims, n_obs, "gmm_condition", mis, &nm, &obs_mask)) return rc;
    if (int rc = check_fitted(c, K, "gmm_condition")) return rc;
    CUDA_TRY(cudaSetDevice(c->device));
    const auto t0 = std::chrono::steady_clock::now();
    ConditionBuffers& cb = c->cond;
    if (int rc = condition_block(c)) return rc;
    const bool impute = nm > 0 && (cond_mean || cond_var);
    double ll = 0.0;
    int rc = condition_params(c, K, obs_dims, n_obs, mis, nm, impute);
    if (rc == GMM_OK && n > 0) {
        rc = score_buffers(c);
        for (int b = 0; b < 2 && rc == GMM_OK && impute; b++) {
            rc = cb.d_imp[b].reserve(2 * (size_t)c->score_chunk * nm);
            if (rc == GMM_OK) rc = cb.h_imp[b].reserve(2 * (size_t)c->score_chunk * nm);
        }
        if (rc == GMM_OK)
            rc = condition_batch(c, K, n_obs, nm, impute, events_obs, n, {labels, max_resp, logp, &ll}, cond_mean, cond_var);
        rc = drain_streams(c, rc, "gmm_condition");
        if (rc == GMM_OK && loglik_out) *loglik_out = ll;
    }
    cb.wall_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return rc;
}

int gmm_get_condition_profile(gmm_ctx* c, double out[2], int reset) {
    if (!c || !out) return fail(GMM_ERR_ARG, "gmm_get_condition_profile: bad argument");
    out[0] = c->cond.kernel_ms; out[1] = c->cond.wall_ms;
    if (reset) c->cond.kernel_ms = c->cond.wall_ms = 0;
    return GMM_OK;
}

// ---- M-step statistics of events measured on a subset of the dimensions ----------------------------------------------------
// gmm_condition_stats' chunks through the statistics loop: the prep kernel writes the observed SoA copy and the D-row image
// of the M-step that will run (a chunk that falls back only because of its flag gets the raw image after the flag is read),
// then the marginal SIMT E-step of the observed copy and the context's M-step on the D-row image.  The statistics hold T0,
// T1 and T2 in the entries of the observed dimensions; the caller expands the others on the host (condition_stats_cluster).
static int condition_stats_batch(gmm_ctx* c, int K, int n_obs, unsigned obs_mask, const float* ev, long long n, bool with_stats,
                                 float* memberships) {
    ScoreBuffers& s = c->score;
    ScoreStatsBuffers& t = c->sstats;
    const int D = c->D;
    const size_t KF = (size_t)K * c->F;
    const bool m_tensor = with_stats && use_tensor_mstep(c, K);
    const float* inv_scale_f = m_tensor ? tc_inv_scale_f(c->tc.get()) : nullptr;
    const float zb = m_tensor ? tc_mstep_zbound(c->tc.get()) : INFINITY;
    if (m_tensor && !inv_scale_f) return fail(GMM_ERR_STATE, "gmm_condition_stats: the tensor M-step has no centre");
    float shift_f[GMM_MAX_DIMENSIONS] = {0};               // the float centre the M-steps use (c->shift is rounded to it
    for (int d = 0; d < D; d++) shift_f[d] = (float)c->shift[d];   // whenever the wgmma M-step can run)
    CUDA_TRY(cudaMemcpyAsync(t.d_shift_f, shift_f, sizeof(shift_f), cudaMemcpyHostToDevice, c->stream));
    CUDA_TRY(cudaMemcpyAsync(c->cond.d_block, c->cond.h_block, sizeof(float) * (size_t)K * epack_stride(n_obs), cudaMemcpyHostToDevice,
                             c->stream));
    auto prep = [&](int b, int m, float* xo, float* z, float* x) -> int {
        condition_stats_prep_kernel<<<(m + 31) / 32, dim3(32, 8), 0, c->stream>>>(s.d_in[b], m, n_obs, D, obs_mask, t.d_shift_f, inv_scale_f,
                                                                                   zb, xo, z, x, t.pitch, t.d_flag);
        CUDA_TRY(cudaGetLastError());
        return GMM_OK;
    };
    auto estep = [&](int b, int m, bool, bool cm) -> int {
        if (m_tensor && !cm)                                      // a fallback of this chunk only: its raw image now
            if (int rc = prep(b, m, nullptr, nullptr, t.d_xs)) return rc;
        return launch_estep_simt_on(c, n_obs, K, c->cond.d_block, t.d_xo, m, t.d_memb, t.pitch, t.d_stats + KF);
    };
    return stats_batch(c, K, ev, n_obs, n, with_stats, memberships, false, m_tensor, t.cond_prof, "gmm_condition_stats",
                       [&](int b, int m) { return prep(b, m, t.d_xo, m_tensor ? t.d_z.get() : nullptr, with_stats && !m_tensor ? t.d_xs.get() : nullptr); },
                       estep);
}

int gmm_condition_stats(gmm_ctx* c, int K, const int* obs_dims, int n_obs, const float* events_obs, long long n, double* stats_out,
                        double* shift_out, float* memberships) {
    if (int rc = check_K(c, K, "gmm_condition_stats")) return rc;
    if (n < 0 || (n > 0 && !events_obs)) return fail(GMM_ERR_ARG, "gmm_condition_stats: bad events (n < 0, or no rows)");
    int mis[GMM_MAX_DIMENSIONS], nm = 0;
    unsigned obs_mask = 0;
    if (int rc = split_obs(c, obs_dims, n_obs, "gmm_condition_stats", mis, &nm, &obs_mask)) return rc;
    if (!stats_out && !memberships) return fail(GMM_ERR_ARG, "gmm_condition_stats: neither statistics nor memberships requested");
    if (int rc = check_fitted(c, K, "gmm_condition_stats")) return rc;
    CUDA_TRY(cudaSetDevice(c->device));
    const auto t0 = std::chrono::steady_clock::now();
    if (int rc = ensure_centre(c, "gmm_condition_stats")) return rc;
    const int D = c->D;
    const size_t len = (size_t)K * c->F + 1;
    std::vector<double> g, cm;                              // per cluster G [nm][n_obs] and C = S_MM^-1 [nm][nm], in double
    int rc = GMM_OK;
    if (nm > 0) {
        if (int rc = condition_block(c)) return rc;
        g.resize((size_t)K * nm * n_obs);
        cm.resize((size_t)K * nm * nm);
        rc = condition_params(c, K, obs_dims, n_obs, mis, nm, false, "gmm_condition_stats", g.data(), cm.data());
    }
    if (rc == GMM_OK && n > 0) {
        rc = score_buffers(c);
        if (rc == GMM_OK) rc = score_stats_buffers(c, memberships != nullptr, nm > 0);
        if (rc == GMM_OK)
            rc = nm > 0 ? condition_stats_batch(c, K, n_obs, obs_mask, events_obs, n, stats_out != nullptr, memberships)
                        : score_stats_batch(c, K, events_obs, n, stats_out != nullptr, memberships, c->sstats.cond_prof);
        rc = drain_streams(c, rc, "gmm_condition_stats");
    }
    if (rc == GMM_OK) {
        if (stats_out) {
            if (n > 0) std::memcpy(stats_out, c->sstats.h_stats, sizeof(double) * len);
            else std::fill(stats_out, stats_out + len, 0.0);
            if (n > 0 && nm > 0)
                run_clusters(c, K, K, [&](int k) {
                    condition_stats_cluster(stats_out + (size_t)k * c->F, D, obs_dims, n_obs, mis, nm, c->host.means + (size_t)k * D, c->shift,
                                            &g[(size_t)k * nm * n_obs], &cm[(size_t)k * nm * nm]);
                });
        }
        if (shift_out) std::memcpy(shift_out, c->shift, sizeof(double) * (size_t)D);
    }
    c->sstats.cond_prof.wall_ms += std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    return rc;
}

int gmm_get_condition_stats_profile(gmm_ctx* c, double out[4], int reset) {
    if (!c || !out) return fail(GMM_ERR_ARG, "gmm_get_condition_stats_profile: bad argument");
    StatsProfile& t = c->sstats.cond_prof;
    out[0] = t.kernel_ms; out[1] = t.wall_ms; out[2] = (double)t.m_tensor; out[3] = (double)t.m_simt;
    if (reset) t = StatsProfile();
    return GMM_OK;
}

int gmm_get_profile(gmm_ctx* c, double out[8], int reset) {
    if (!c || !out) return fail(GMM_ERR_ARG, "gmm_get_profile: bad argument");
    cudaStreamSynchronize(c->stream);
    collect_all(c);
    out[0] = c->t_estep.total_ms; out[1] = c->t_mstep.total_ms; out[2] = c->host_const_ms;
    out[3] = c->t_reduce.total_ms; out[4] = c->memcpy_ms + c->t_final.total_ms; out[5] = (double)c->mstep_tensor;
    out[6] = (double)c->iterations; out[7] = (double)c->mstep_simt;
    if (reset) {
        c->t_estep.total_ms = c->t_mstep.total_ms = c->t_reduce.total_ms = c->t_fused.total_ms = 0;
        c->host_const_ms = c->memcpy_ms = 0; c->iterations = 0; c->t_final.total_ms = 0;
        c->mstep_tensor = c->mstep_simt = 0;
        c->fit_reduce_ms = c->fit_seed_ms = c->fit_save_ms = 0;
    }
    return GMM_OK;
}

// Host-only self-test of the worker team used by the per-iteration finalisation (tests/test_host.py): `jobs` back-to-back
// parallel loops of n items on `threads` threads, every item must run exactly once per job.  Returns 0 when it did.
int gmm_host_pool_selftest(int threads, int jobs, int n) {
    if (threads < 1 || jobs < 1 || n < 0) return fail(GMM_ERR_ARG, "gmm_host_pool_selftest: bad argument");
    HostPool pool(threads);
    std::vector<std::atomic<int>> hits((size_t)(n > 0 ? n : 1));
    for (auto& h : hits) h.store(0);
    for (int j = 0; j < jobs; j++) {
        const int m = (j % 3 == 0) ? n : (j % 3 == 1 ? (n + 1) / 2 : 1);
        const std::function<void(int)> fn = [&](int i) { hits[(size_t)i].fetch_add(1, std::memory_order_relaxed); };
        pool.run(m, fn);
        for (int i = 0; i < n; i++) {
            const int want = i < m ? 1 : 0;
            if (hits[(size_t)i].exchange(0) != want) return fail(GMM_ERR_STATE, "gmm_host_pool_selftest: an item ran the wrong number of times");
        }
        if (j % 64 == 63) pool.resize(1 + (j / 64) % threads);          // exercise team re-creation as well
        if (j % 200 == 199) std::this_thread::sleep_for(std::chrono::milliseconds(6));   // let the workers fall asleep once in a while
    }
    return GMM_OK;
}

int gmm_get_fit_profile(gmm_ctx* c, double out[4]) {
    if (!c || !out) return fail(GMM_ERR_ARG, "gmm_get_fit_profile: bad argument");
    out[0] = c->fit_reduce_ms; out[1] = c->fit_seed_ms; out[2] = c->fit_save_ms;
    out[3] = (double)c->dev_finalize_launches + 1e-3 * (double)(c->dev_replays > 999 ? 999 : c->dev_replays);
    return GMM_OK;
}

// Model-order reduction loop (gaussian.cu:479-960).
int gmm_fit(gmm_ctx* c, int K0, int target_K, int min_iters, int max_iters, clusters_t* saved, int* ideal_K,
            float* min_rissanen_out) {
    if (int rc = check_K(c, K0, "gmm_fit")) return rc;
    if (target_K < 0 || target_K > K0) return fail(GMM_ERR_ARG, "target_num_clusters must be less than equal to num_clusters");
    if (!saved) return fail(GMM_ERR_ARG, "gmm_fit: null saved clusters");
    CUDA_TRY(cudaSetDevice(c->device));
    const int D = c->D;
    const int stop_number = target_K == 0 ? 1 : target_K;                  // gaussian.cu:177-181
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto ms_since = [](std::chrono::steady_clock::time_point t0) {
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    };
    {
        const auto t0 = now();
        if (int rc = gmm_seed(c, K0, nullptr)) return rc;
        c->fit_seed_ms += ms_since(t0);
    }
    const float epsilon = em_epsilon(D, em_count(c));
    float min_rissanen = 0;
    int ideal = K0;
    if (saved->memberships && c->n > 0)
        if (int rc = c->d_memb_saved.reserve(c->memb_pitch * c->Kmax)) return rc;
    for (int K = K0; K >= stop_number;) {
        float likelihood; int iters;
        if (int rc = gmm_em(c, K, min_iters, max_iters, epsilon, &likelihood, &iters)) return rc;
        const float r = rissanen(likelihood, K, D, em_count(c));          // :826
        if (c->verbose && c->rank == 0) std::printf("K=%d loglik=%e Rissanen Score: %e\n", K, likelihood, r);
        if (K == K0 || (r < min_rissanen && target_K == 0) || K == target_K) {   // :839
            const auto t0 = now();
            min_rissanen = r;
            ideal = K;
            copy_params(saved, &c->host, K, D);
            if (saved->memberships && c->n > 0)
                CUDA_TRY(cudaMemcpyAsync(c->d_memb_saved, c->d_memb, sizeof(float) * (size_t)K * c->memb_pitch, cudaMemcpyDeviceToDevice, c->stream));
            c->fit_save_ms += ms_since(t0);
        }
        if (K > stop_number) {                                            // :860-950
            const auto t0 = now();
            HostPool* pool = host_pool(c);
            const ParallelFor pfor = [&](int n, const std::function<void(int)>& fn) { pool->run(n, fn); };
            K = reduce_order(&c->host, K, D, nullptr, nullptr, c->host_threads, &pfor);
            c->fit_reduce_ms += ms_since(t0);
            if (K < 1) break;
            c->memb_valid = false;
            if (int rc = upload_params(c, K)) return rc;
        } else break;
    }
    if (saved->memberships && c->n > 0) {
        CUDA_TRY(cudaMemcpy2DAsync(saved->memberships, sizeof(float) * (size_t)c->n, c->d_memb_saved, sizeof(float) * c->memb_pitch,
                                   sizeof(float) * (size_t)c->n, ideal, cudaMemcpyDeviceToHost, c->stream));
    }
    CUDA_TRY(cudaStreamSynchronize(c->stream));
    if (ideal_K) *ideal_K = ideal;
    if (min_rissanen_out) *min_rissanen_out = min_rissanen;
    return GMM_OK;
}

}  // extern "C"
