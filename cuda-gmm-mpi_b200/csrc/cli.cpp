// cli.cpp — the reference program's command line on top of the C ABI:
//   gaussianMPI num_clusters infile outfile [target_num_clusters]
// (gaussian.cu:128-1106; argument rules of validateArguments :1111-1166 and
// usage text of printUsage :1171-1178).  One host thread per GPU, like the
// reference's OpenMP team (gaussian.cu:289-301), joined by NCCL instead of
// MPI + shared-memory sums.
//
// Environment (the reference's compile-time switches, gaussian.h:23-38):
//   GMM_ITERS   MIN_ITERS = MAX_ITERS (default 100)
//   GMM_GPUS    number of GPUs to use (default: all visible)
//   GMM_OUTPUT  1 = write .summary/.results content (ENABLE_OUTPUT), default 1
//   GMM_PRINT   1 = ENABLE_PRINT messages, default 0
//   GMM_PATH    0 auto, 1 SIMT kernels, 2 wgmma kernels
#include <cuda_runtime.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/gmm.h"

static void print_usage(char** argv) {
    std::printf("Usage: %s num_clusters infile outfile [target_num_clusters]\n", argv[0]);
    std::printf("\t num_clusters: The number of starting clusters\n");
    std::printf("\t infile: ASCII space-delimited FCS data file\n");
    std::printf("\t outfile: Clustering results output file\n");
    std::printf("\t target_num_clusters: A desired number of clusters. Must be less than or equal to num_clusters\n");
}

// Return codes as validateArguments: 1 bad K / usage, 2 infile, 4 target.
static int validate_arguments(int argc, char** argv, int* num_clusters, int* target) {
    if (argc < 4 || argc > 5) { print_usage(argv); return 1; }
    if (std::sscanf(argv[1], "%d", num_clusters) != 1 || *num_clusters < 1 || *num_clusters > GMM_MAX_CLUSTERS) {
        std::printf("Invalid number of starting clusters\n\n");
        print_usage(argv);
        return 1;
    }
    FILE* in = std::fopen(argv[2], "r");
    if (!in) { std::printf("Invalid infile.\n\n"); print_usage(argv); return 2; }
    std::fclose(in);
    *target = 0;
    if (argc == 5) {
        if (std::sscanf(argv[4], "%d", target) != 1) {
            std::printf("Invalid number of desired clusters.\n\n");
            print_usage(argv);
            return 4;
        }
        if (*target > *num_clusters) {
            std::printf("target_num_clusters must be less than equal to num_clusters\n\n");
            print_usage(argv);
            return 4;
        }
    }
    return 0;
}

// All worker threads meet here once (the reference's `#pragma omp barrier` after its per-GPU setup, gaussian.cu:378).
struct OneShotBarrier {
    std::mutex m; std::condition_variable cv; int waiting = 0; const int total;
    explicit OneShotBarrier(int n) : total(n) {}
    void arrive_and_wait() {
        std::unique_lock<std::mutex> lk(m);
        if (++waiting == total) cv.notify_all();
        else cv.wait(lk, [&] { return waiting == total; });
    }
};

static int env_int(const char* name, int dflt) { const char* s = std::getenv(name); return s ? std::atoi(s) : dflt; }

struct HostClusters {
    std::vector<float> N, pi, constant, avgvar, means, R, Rinv, memb;
    clusters_t c{};
    HostClusters(int K, int D, size_t n_memb) : N(K), pi(K), constant(K), avgvar(K), means((size_t)K * D),
        R((size_t)K * D * D), Rinv((size_t)K * D * D), memb(n_memb) {
        c.N = N.data(); c.pi = pi.data(); c.constant = constant.data(); c.avgvar = avgvar.data();
        c.means = means.data(); c.R = R.data(); c.Rinv = Rinv.data(); c.memberships = n_memb ? memb.data() : nullptr;
    }
};

extern "C" int gmm_main(int argc, char** argv) {
    const auto t_start = std::chrono::steady_clock::now();
    int K0 = 0, target = 0;
    if (validate_arguments(argc, argv, &K0, &target)) return 1;        // gaussian.cu:169-174

    const int print = env_int("GMM_PRINT", 0);
    int D = 0, N = 0;
    if (print) std::printf("Parsing input file...");
    // "*.bin" (readData.cpp:28): only the header is read here; every GPU thread streams its own rows from the file to its
    // device through pinned staging buffers (gmm_upload_events_file) and the .results writer maps the file — the host
    // never allocates the data set.  Anything else (CSV) is parsed into host memory as in the reference.
    const size_t plen = std::strlen(argv[2]);
    const bool is_bin = plen >= 3 && std::strcmp(argv[2] + plen - 3, "bin") == 0;
    float* events = nullptr;
    if (is_bin) {
        if (gmm_read_bin_header(argv[2], &D, &N)) { D = 0; N = 0; }
    } else {
        events = gmm_read_data(argv[2], &D, &N);
    }
    if ((!is_bin && !events) || D <= 0 || N <= 0) {
        std::printf("Error parsing input file. This could be due to an empty file ");
        std::printf("or an inconsistent number of dimensions. Aborting.\n");
        gmm_free(events);
        return 1;
    }
    if (D > GMM_MAX_DIMENSIONS) { std::printf("ERROR: at most %d dimensions are supported.\n", GMM_MAX_DIMENSIONS); gmm_free(events); return 1; }
    if (print) {
        std::printf("Number of events: %d\nNumber of dimensions: %d\n\n", N, D);
        std::printf("Starting with %d cluster(s), will stop at %d cluster(s).\n", K0, target == 0 ? 1 : target);
    }
    const auto t_io = std::chrono::steady_clock::now();

    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev < 1) {
        std::printf("ERROR: No CUDA capable GPUs detected.\n");
        gmm_free(events);
        return -1;
    }
    int G = env_int("GMM_GPUS", ndev);
    if (G < 1) G = 1;
    if (G > ndev) G = ndev;
    if ((long long)G > N) G = 1;
    const int iters = env_int("GMM_ITERS", 100);
    const int want_output = env_int("GMM_OUTPUT", 1);
    const int path = env_int("GMM_PATH", GMM_PATH_AUTO);

    char id[128];
    if (G > 1 && gmm_nccl_unique_id(id)) { std::printf("ERROR: %s\n", gmm_last_error()); gmm_free(events); return -1; }

    HostClusters saved(K0, D, want_output ? (size_t)K0 * N : 0);   // best configuration, memberships [K][N]
    std::vector<int> rcs(G, 0), ideal(G, 0);
    std::vector<float> minr(G, 0.f);
    std::vector<std::string> errs(G);
    std::vector<std::vector<double>> prof(G, std::vector<double>(8, 0.0));

    // Every context is created (and checked) BEFORE any thread enters the communicator bootstrap: ncclCommInitRank
    // needs all G ranks, so a rank that failed earlier (no sm_90 device, out of memory, bad GMM_PATH) would leave
    // the others blocked for ever; the reference exits the whole process on a CUDA failure (CUDA_SAFE_CALL).
    OneShotBarrier created(G);
    std::atomic<int> setup_failed{0};
    auto worker = [&](int g) {
        long long begin, count;
        gmm_shard_range(N, G, g, &begin, &count);
        gmm_ctx* ctx = nullptr;
        int rc = gmm_create(&ctx, g, (int)count, D, K0, events ? events + (size_t)begin * D : nullptr, N, begin);
        if (!rc && is_bin) rc = gmm_upload_events_file(ctx, argv[2]);
        if (!rc) rc = gmm_set_option(ctx, "path", path);
        if (!rc) rc = gmm_set_option(ctx, "verbose", print);
        if (rc) { errs[g] = gmm_last_error(); setup_failed.store(1); }
        created.arrive_and_wait();
        if (setup_failed.load()) {
            if (!rc) { rc = GMM_ERR_STATE; errs[g] = "another GPU failed during setup"; }
            rcs[g] = rc;
            gmm_destroy(ctx);
            return;
        }
        rc = gmm_comm_init(ctx, G, g, id);
        if (!rc) {
            HostClusters mine(K0, D, want_output ? (size_t)K0 * count : 0);
            rc = gmm_fit(ctx, K0, target, iters, iters, &mine.c, &ideal[g], &minr[g]);
            if (!rc) {
                if (g == 0) {
                    const int Ki = ideal[0];
                    std::memcpy(saved.c.N, mine.c.N, sizeof(float) * Ki); std::memcpy(saved.c.pi, mine.c.pi, sizeof(float) * Ki);
                    std::memcpy(saved.c.constant, mine.c.constant, sizeof(float) * Ki);
                    std::memcpy(saved.c.avgvar, mine.c.avgvar, sizeof(float) * Ki);
                    std::memcpy(saved.c.means, mine.c.means, sizeof(float) * (size_t)Ki * D);
                    std::memcpy(saved.c.R, mine.c.R, sizeof(float) * (size_t)Ki * D * D);
                    std::memcpy(saved.c.Rinv, mine.c.Rinv, sizeof(float) * (size_t)Ki * D * D);
                }
                if (want_output)       // gather of gaussian.cu:772-774: shard [K][count] -> global [K][N]
                    for (int k = 0; k < ideal[g]; k++)
                        std::memcpy(saved.c.memberships + (size_t)k * N + begin, mine.c.memberships + (size_t)k * count,
                                    sizeof(float) * (size_t)count);
                gmm_get_profile(ctx, prof[g].data(), 0);
            }
        }
        if (rc) {
            // an error between collectives on one rank would leave the peers inside ncclAllReduce: like the reference
            // (CUDA_SAFE_CALL exits), the process ends here instead of joining threads that can never return
            std::printf("ERROR (GPU %d): %s\n", g, gmm_last_error());
            std::fflush(stdout);
            if (G > 1) std::_Exit(rc == GMM_ERR_CUDA ? 255 : 1);
            errs[g] = gmm_last_error();
        }
        rcs[g] = rc;
        gmm_destroy(ctx);
    };
    std::vector<std::thread> threads;
    for (int g = 0; g < G; g++) threads.emplace_back(worker, g);
    for (auto& t : threads) t.join();
    for (int g = 0; g < G; g++)
        if (rcs[g]) {
            std::printf("ERROR (GPU %d): %s\n", g, errs[g].c_str());
            gmm_free(events);
            return rcs[g] == GMM_ERR_CUDA ? -1 : 1;
        }
    const int ideal_K = ideal[0];
    if (print) std::printf("\nFinal rissanen score was: %f, with %d clusters.\n", minr[0], ideal_K);
    for (int g = 0; g < G; g++)      // profile line in the spirit of gaussian.cu:967
        std::printf("GPU %d:\n\tE-step Kernel:\t%7.4f\n\tM-step Kernel:\t%7.4f\n\tConsts (host):\t%7.4f\n\tAllreduce:\t%7.4f\n\tParam upload:\t%7.4f\n\tEM iterations:\t%d\n",
                    g, prof[g][0] / 1e3, prof[g][1] / 1e3, prof[g][2] / 1e3, prof[g][3] / 1e3, prof[g][4] / 1e3, (int)prof[g][6]);

    const auto t_out = std::chrono::steady_clock::now();
    const std::string summary = std::string(argv[3]) + ".summary", results = std::string(argv[3]) + ".results";
    if (gmm_write_summary(summary.c_str(), want_output ? &saved.c : nullptr, want_output ? ideal_K : 0, D)) {   // :1015-1019
        std::printf("ERROR: Unable to open file '%s' for writing.\n", argv[3]);
        gmm_free(events);
        return -1;
    }
    if (want_output) {
        const float* ev = events;
        void* map = MAP_FAILED;
        size_t map_len = 0;
        if (is_bin) {                                   // the event columns of the .results file come straight from the mapped input
            const int fd = open(argv[2], O_RDONLY);
            struct stat st;
            if (fd >= 0 && fstat(fd, &st) == 0 && (size_t)st.st_size >= 8 + sizeof(float) * (size_t)N * D) {
                map_len = (size_t)st.st_size;
                map = mmap(nullptr, map_len, PROT_READ, MAP_PRIVATE, fd, 0);
            }
            if (fd >= 0) close(fd);
            if (map == MAP_FAILED) { std::printf("ERROR: Unable to map '%s'.\n", argv[2]); return -1; }
            ev = reinterpret_cast<const float*>(static_cast<const char*>(map) + 8);
        }
        gmm_write_results(results.c_str(), ev, N, D, &saved.c, ideal_K);
        if (map != MAP_FAILED) munmap(map, map_len);
    }
    gmm_free(events);
    const auto t_end = std::chrono::steady_clock::now();
    auto ms = [](auto a, auto b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    std::printf("I/O time: %f (ms)\n", ms(t_start, t_io) + ms(t_out, t_end));
    std::printf("Total time: %f (ms)\n", ms(t_start, t_end));
    return 0;
}
