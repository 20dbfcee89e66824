"""ctypes mirror of include/gmm.h.

Method names and argument meaning follow the C ABI one to one, which in turn
follows the reference's operator granularity (seed / E-step / M-step /
constants / EM loop / order reduction — gaussian.cu:390-960).  Nothing here
computes: every call goes to ``libgmm_b200.so``; a missing library or a
missing GPU raises, there is no fallback.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from .clusters import Clusters, clusters_t

_HERE = os.path.dirname(os.path.abspath(__file__))
_FP = C.POINTER(C.c_float)
_DP = C.POINTER(C.c_double)
_IP = C.POINTER(C.c_int)
_CP = C.POINTER(clusters_t)

PATH_AUTO, PATH_SIMT, PATH_TENSOR = 0, 1, 2

_lib = None


class GmmError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"gmm error {code}: {msg}")
        self.code = code


def library_path():
    # GMM_B200_LIB: development override (kernel variants for experiments); the product is libgmm_b200.so
    return os.environ.get("GMM_B200_LIB") or os.path.join(_HERE, "libgmm_b200.so")


def build_library(force=False):
    """Compile csrc/ for sm_90a (nvcc cross-compiles without a GPU)."""
    args = ["make", "-s", "-C", os.path.join(_HERE, "csrc"), "-j8"]
    if force:
        subprocess.check_call(args[:4] + ["clean"])
    subprocess.check_call(args)


def load_library():
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.exists(path):
        raise FileNotFoundError(f"{path} is missing: run __graft_entry__.build() (there is no fallback path)")
    L = C.CDLL(path, mode=C.RTLD_GLOBAL)
    L.gmm_last_error.restype = C.c_char_p
    L.gmm_version.restype = C.c_char_p
    L.gmm_create.argtypes = [C.POINTER(C.c_void_p), C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                             C.c_longlong, C.c_longlong]
    L.gmm_upload_events.argtypes = [C.c_void_p, C.c_void_p]
    L.gmm_upload_events_file.argtypes = [C.c_void_p, C.c_char_p]
    L.gmm_read_bin_header.argtypes = [C.c_char_p, _IP, _IP]
    L.gmm_destroy.argtypes = [C.c_void_p]
    L.gmm_destroy.restype = None
    L.gmm_shard_range.argtypes = [C.c_longlong, C.c_int, C.c_int, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]
    L.gmm_shard_range.restype = None
    L.gmm_nccl_unique_id.argtypes = [C.c_char_p]
    L.gmm_comm_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_char_p]
    L.gmm_comm_rank.argtypes = [C.c_void_p, _IP, _IP]
    L.gmm_set_option.argtypes = [C.c_void_p, C.c_char_p, C.c_double]
    L.gmm_seed.argtypes = [C.c_void_p, C.c_int, _CP]
    L.gmm_set_clusters.argtypes = [C.c_void_p, C.c_int, _CP]
    L.gmm_get_clusters.argtypes = [C.c_void_p, C.c_int, _CP, C.c_int]
    L.gmm_estep.argtypes = [C.c_void_p, C.c_int, _FP]
    L.gmm_mstep.argtypes = [C.c_void_p, C.c_int]
    L.gmm_constants.argtypes = [C.c_void_p, C.c_int]
    L.gmm_em.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, _FP, _IP]
    L.gmm_em_iterations.argtypes = [C.c_void_p, C.c_int, C.c_int, _FP]
    L.gmm_get_profile.argtypes = [C.c_void_p, _DP, C.c_int]
    L.gmm_get_fit_profile.argtypes = [C.c_void_p, _DP]
    L.gmm_fit.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, _CP, _IP, _FP]
    L.gmm_host_pool_selftest.argtypes = [C.c_int, C.c_int, C.c_int]
    L.gmm_host_invert.argtypes = [_FP, C.c_int, _FP, C.c_int]
    L.gmm_stats_len.argtypes = [C.c_int, C.c_int]
    L.gmm_stats_len.restype = C.c_longlong
    L.gmm_host_finalize.argtypes = [_DP, _DP, C.c_int, C.c_int, _CP]
    L.gmm_host_rissanen.argtypes = [C.c_float, C.c_int, C.c_int, C.c_longlong]
    L.gmm_host_rissanen.restype = C.c_float
    L.gmm_host_epsilon.argtypes = [C.c_int, C.c_longlong]
    L.gmm_host_epsilon.restype = C.c_float
    L.gmm_host_reduce_order.argtypes = [_CP, _IP, C.c_int, _IP, _IP]
    L.gmm_read_data.argtypes = [C.c_char_p, _IP, _IP]
    L.gmm_read_data.restype = C.c_void_p
    L.gmm_free.argtypes = [C.c_void_p]
    L.gmm_free.restype = None
    L.gmm_write_summary.argtypes = [C.c_char_p, _CP, C.c_int, C.c_int]
    L.gmm_write_results.argtypes = [C.c_char_p, _FP, C.c_longlong, C.c_int, _CP, C.c_int]
    L.gmm_main.argtypes = [C.c_int, C.POINTER(C.c_char_p)]
    _lib = L
    return L


def _check(rc):
    if rc != 0:
        raise GmmError(rc, load_library().gmm_last_error().decode(errors="replace"))


# ---- host-only numerics (no GPU needed) -----------------------------------
def host_invert(m, use_log10=False):
    """invert_cpu semantics (invert_matrix.cpp:25-101); returns (inverse, log det)."""
    a = np.ascontiguousarray(m, np.float32).copy()
    ld = C.c_float()
    _check(load_library().gmm_host_invert(a.ctypes.data_as(_FP), a.shape[0], C.byref(ld), int(use_log10)))
    return a, ld.value


def stats_len(K, D):
    return int(load_library().gmm_stats_len(K, D))


def host_finalize(stats, shift, cl, K):
    stats = np.ascontiguousarray(stats, np.float64)
    shift = np.ascontiguousarray(shift, np.float64)
    assert stats.size >= stats_len(K, cl.D) and shift.size >= cl.D
    s = cl.struct()
    _check(load_library().gmm_host_finalize(stats.ctypes.data_as(_DP), shift.ctypes.data_as(_DP), K, cl.D, C.byref(s)))


def host_rissanen(ll, K, D, N):
    return float(load_library().gmm_host_rissanen(ll, K, D, N))


def host_epsilon(D, N):
    return float(load_library().gmm_host_epsilon(D, N))


def host_reduce_order(cl, K):
    k = C.c_int(K)
    c1, c2 = C.c_int(), C.c_int()
    s = cl.struct()
    _check(load_library().gmm_host_reduce_order(C.byref(s), C.byref(k), cl.D, C.byref(c1), C.byref(c2)))
    return k.value, (c1.value, c2.value)


def shard_range(n_global, nranks, rank):
    b, n = C.c_longlong(), C.c_longlong()
    load_library().gmm_shard_range(n_global, nranks, rank, C.byref(b), C.byref(n))
    return b.value, n.value


def read_data(path):
    L = load_library()
    nd, ne = C.c_int(), C.c_int()
    p = L.gmm_read_data(os.fsencode(path), C.byref(nd), C.byref(ne))
    if not p:
        raise GmmError(2, L.gmm_last_error().decode(errors="replace"))
    try:
        arr = np.ctypeslib.as_array(C.cast(p, _FP), shape=(ne.value, nd.value)).copy()
    finally:
        L.gmm_free(p)
    return arr


def write_summary(path, cl, K):
    s = cl.struct()
    _check(load_library().gmm_write_summary(os.fsencode(path), C.byref(s), K, cl.D))


def write_results(path, events, cl, K):
    ev = np.ascontiguousarray(events, np.float32)
    s = cl.struct()
    _check(load_library().gmm_write_results(os.fsencode(path), ev.ctypes.data_as(_FP), ev.shape[0], ev.shape[1], C.byref(s), K))


def nccl_unique_id():
    buf = C.create_string_buffer(128)
    _check(load_library().gmm_nccl_unique_id(buf))
    return buf.raw


class Engine:
    """One GPU, one contiguous shard of events (gmm_ctx)."""

    def __init__(self, events, Kmax, device=0, n_global=None, offset=0, events_ptr=None, n_local=None, D=None):
        """``events``: float32 [n_local][D] host array (numpy).  Alternatively pass a raw
        host pointer (``events_ptr``, e.g. pinned memory) with ``n_local`` and ``D``."""
        self.lib = load_library()
        if events is not None:
            events = np.ascontiguousarray(events, np.float32)
            n_local, D = events.shape
            events_ptr = events.ctypes.data
        self.n, self.D, self.Kmax = int(n_local), int(D), int(Kmax)
        self.n_global = int(n_global) if n_global else self.n
        self.offset = int(offset)
        h = C.c_void_p()
        _check(self.lib.gmm_create(C.byref(h), device, self.n, self.D, self.Kmax, events_ptr, self.n_global, self.offset))
        self.h = h

    def close(self):
        if getattr(self, "h", None):
            self.lib.gmm_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def upload_events(self, events=None, events_ptr=None):
        if events is not None:
            events = np.ascontiguousarray(events, np.float32)
            assert events.shape == (self.n, self.D)
            events_ptr = events.ctypes.data
        _check(self.lib.gmm_upload_events(self.h, events_ptr))

    def upload_events_file(self, path):
        _check(self.lib.gmm_upload_events_file(self.h, os.fsencode(path)))

    def new_clusters(self, with_memberships=False):
        return Clusters(self.Kmax, self.D, self.n if with_memberships else 0)

    def comm_init(self, nranks, rank, unique_id):
        _check(self.lib.gmm_comm_init(self.h, nranks, rank, unique_id))

    def set_option(self, key, value):
        _check(self.lib.gmm_set_option(self.h, key.encode(), float(value)))

    def seed(self, K, out=None):
        out = out or self.new_clusters()
        s = out.struct()
        _check(self.lib.gmm_seed(self.h, K, C.byref(s)))
        return out

    def set_clusters(self, K, cl):
        s = cl.struct()
        _check(self.lib.gmm_set_clusters(self.h, K, C.byref(s)))

    def get_clusters(self, K, out=None, with_memberships=False):
        out = out or self.new_clusters(with_memberships)
        s = out.struct()
        _check(self.lib.gmm_get_clusters(self.h, K, C.byref(s), int(with_memberships)))
        return out

    def estep(self, K):
        ll = C.c_float()
        _check(self.lib.gmm_estep(self.h, K, C.byref(ll)))
        return ll.value

    def mstep(self, K):
        _check(self.lib.gmm_mstep(self.h, K))

    def constants(self, K):
        _check(self.lib.gmm_constants(self.h, K))

    def em(self, K, min_iters, max_iters, epsilon=-1.0):
        ll, it = C.c_float(), C.c_int()
        _check(self.lib.gmm_em(self.h, K, min_iters, max_iters, epsilon, C.byref(ll), C.byref(it)))
        return ll.value, it.value

    def em_iterations(self, K, iters):
        ll = C.c_float()
        _check(self.lib.gmm_em_iterations(self.h, K, iters, C.byref(ll)))
        return ll.value

    def profile(self, reset=False):
        out = (C.c_double * 8)()
        _check(self.lib.gmm_get_profile(self.h, out, int(reset)))
        keys = ("estep_ms", "mstep_ms", "constants_host_ms", "allreduce_ms", "upload_ms", "mstep_tensor_launches", "iterations",
                "mstep_simt_launches")
        return dict(zip(keys, list(out)[:8]))

    def fit_profile(self):
        out = (C.c_double * 4)()
        _check(self.lib.gmm_get_fit_profile(self.h, out))
        return dict(reduce_order_ms=out[0], seed_ms=out[1], save_ms=out[2], device_finalize_launches=int(out[3]),
                    host_replays=int(round((out[3] - int(out[3])) * 1000)))

    def comm_rank(self):
        r, n = C.c_int(), C.c_int()
        _check(self.lib.gmm_comm_rank(self.h, C.byref(r), C.byref(n)))
        return r.value, n.value

    def fit(self, K0, target_K, min_iters, max_iters, saved=None, with_memberships=False):
        saved = saved or self.new_clusters(with_memberships)
        ideal, mr = C.c_int(), C.c_float()
        s = saved.struct()
        _check(self.lib.gmm_fit(self.h, K0, target_K, min_iters, max_iters, C.byref(s), C.byref(ideal), C.byref(mr)))
        return ideal.value, mr.value, saved
