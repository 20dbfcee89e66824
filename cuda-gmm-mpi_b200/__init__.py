"""cuda-gmm-mpi_b200 — H100-native GMM-EM engine (drop-in for the EM hot path of
Corv/CUDA-GMM-MPI).  The product is the C-ABI shared library
``libgmm_b200.so`` (include/gmm.h) built from ``csrc/``; this package is the
thin ctypes mirror used by the tests, bench.py and __graft_entry__.py.

The directory name carries a hyphen (it mirrors the reference repository's
name); import it through ``__graft_entry__.load_package()``, which registers
it as ``cuda_gmm_mpi_b200``.
"""
from .clusters import Clusters, clusters_t          # noqa: F401
from .engine import (Engine, GmmError, build_library, load_library, library_path,   # noqa: F401
                     host_invert, host_finalize, host_rissanen, host_epsilon,
                     host_reduce_order, shard_range, stats_len, read_data,
                     write_summary, write_results, nccl_unique_id,
                     PATH_AUTO, PATH_SIMT, PATH_TENSOR)
from . import synth                                  # noqa: F401
