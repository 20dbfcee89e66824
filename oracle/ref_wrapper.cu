/* Wrapper translation unit that compiles the UNMODIFIED reference program
 * (gaussian.cu of the reference repository, which #includes gaussian_kernel.cu) for
 * sm_90a.  No reference source is copied: the files are #included from where
 * they lie.  The only intervention is to pre-include gaussian.h and re-define
 * three of its compile-time switches, which its include guard then protects:
 *   ENABLE_OUTPUT 1          -> the .summary/.results files are written
 *   MIN_ITERS / MAX_ITERS    -> env GMM_REF_ITERS (default 100, the shipped value)
 * With -DGMM_REF_PERF (second binary, gaussianMPI_ref_perf) ENABLE_OUTPUT keeps the shipped value 0 — the
 * reference's own "performance evaluation" configuration (gaussian.h:34-38): that is the build bench.py times
 * on the GPU ("reference_gpu"), the output files of 10M events would be gigabytes of text.
 * Test infrastructure only (see oracle/gmm_oracle.c header). */
#include <stdio.h>
#include <stdlib.h>
#include "gaussian.h"            /* found through -I$(REF) */
static int gmm_ref_iters() { const char* s = getenv("GMM_REF_ITERS"); return s ? atoi(s) : 100; }
#ifndef GMM_REF_PERF
#undef ENABLE_OUTPUT
#define ENABLE_OUTPUT 1
#endif
#undef MAX_ITERS
#define MAX_ITERS gmm_ref_iters()
#undef MIN_ITERS
#define MIN_ITERS gmm_ref_iters()
#include "gaussian.cu"           /* found through -I$(REF) */
