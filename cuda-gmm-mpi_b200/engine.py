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
VB_DIRICHLET_PROCESS, VB_DIRICHLET_DISTRIBUTION = 0, 1


class gmm_vb_prior(C.Structure):
    _fields_ = [("weight_prior_type", C.c_int), ("weight_concentration", C.c_double), ("mean_precision", C.c_double),
                ("dof", C.c_double), ("mean", _DP), ("covariance", _DP), ("reg_covar", C.c_double)]


class gmm_vb_posterior(C.Structure):
    _fields_ = [("weights", _DP), ("weight_concentration", _DP), ("mean_precision", _DP), ("dof", _DP), ("mean_prior", _DP),
                ("covariance_prior", _DP)]


def _vb_prior(D, prior_type, weight_concentration, mean_precision, dof, mean, covariance, reg_covar):
    """gmm_vb_prior and the arrays it points to (keep both alive for the call).  None selects the library's default."""
    keep = []

    def arr(a, shape):
        if a is None:
            return None
        a = np.ascontiguousarray(a, np.float64)
        if a.shape != shape:
            raise ValueError(f"prior array must be {shape}, got {a.shape}")
        keep.append(a)
        return a.ctypes.data_as(_DP)

    p = gmm_vb_prior(int(prior_type), -1.0 if weight_concentration is None else float(weight_concentration),
                     -1.0 if mean_precision is None else float(mean_precision), -1.0 if dof is None else float(dof),
                     arr(mean, (D,)), arr(covariance, (D, D)), -1.0 if reg_covar is None else float(reg_covar))
    return p, keep


def _vb_posterior(K, D, prior_type):
    post = dict(weights=np.zeros(K), weight_concentration=np.zeros((2, K) if prior_type == VB_DIRICHLET_PROCESS else K),
                mean_precision=np.zeros(K), dof=np.zeros(K), mean_prior=np.zeros(D), covariance_prior=np.zeros((D, D)))
    s = gmm_vb_posterior(*(post[f[0]].ctypes.data_as(_DP) for f in gmm_vb_posterior._fields_))
    return post, s

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
    L.gmm_seed_kmeans.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_ulonglong, _CP, _FP, _IP, _DP]
    L.gmm_set_clusters.argtypes = [C.c_void_p, C.c_int, _CP]
    L.gmm_set_weights.argtypes = [C.c_void_p, C.c_void_p, _DP]
    L.gmm_get_clusters.argtypes = [C.c_void_p, C.c_int, _CP, C.c_int]
    L.gmm_estep.argtypes = [C.c_void_p, C.c_int, _FP]
    L.gmm_mstep.argtypes = [C.c_void_p, C.c_int]
    L.gmm_constants.argtypes = [C.c_void_p, C.c_int]
    L.gmm_em.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, _FP, _IP]
    L.gmm_em_iterations.argtypes = [C.c_void_p, C.c_int, C.c_int, _FP]
    L.gmm_get_profile.argtypes = [C.c_void_p, _DP, C.c_int]
    L.gmm_get_fit_profile.argtypes = [C.c_void_p, _DP]
    L.gmm_score.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p, _DP]
    L.gmm_get_score_profile.argtypes = [C.c_void_p, _DP, C.c_int]
    L.gmm_score_stats.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gmm_get_score_stats_profile.argtypes = [C.c_void_p, _DP, C.c_int]
    L.gmm_sample.argtypes = [C.c_void_p, C.c_int, C.c_longlong, C.c_ulonglong, C.c_longlong, C.c_void_p, C.c_void_p]
    L.gmm_get_sample_profile.argtypes = [C.c_void_p, _DP, C.c_int]
    L.gmm_condition.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p, _DP]
    L.gmm_get_condition_profile.argtypes = [C.c_void_p, _DP, C.c_int]
    L.gmm_condition_stats.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p,
                                      C.c_void_p]
    L.gmm_get_condition_stats_profile.argtypes = [C.c_void_p, _DP, C.c_int]
    L.gmm_fit.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, _CP, _IP, _FP]
    L.gmm_vb_em.argtypes = [C.c_void_p, C.c_int, C.POINTER(gmm_vb_prior), C.c_int, C.c_int, C.c_double, _CP,
                            C.POINTER(gmm_vb_posterior), _DP, _DP, _IP, _IP]
    L.gmm_host_vb_finalize.argtypes = [_DP, _DP, C.c_int, C.c_int, C.POINTER(gmm_vb_prior), _CP, C.POINTER(gmm_vb_posterior), _DP]
    L.gmm_host_digamma.argtypes = [_DP, _DP, C.c_longlong]
    L.gmm_get_vb_profile.argtypes = [C.c_void_p, _DP, C.c_int]
    L.gmm_combine.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.gmm_combine_labels.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.gmm_host_combine_groups.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.gmm_host_combine_elbow.argtypes = [C.c_void_p, C.c_void_p, C.c_int, _IP]
    L.gmm_get_combine_profile.argtypes = [C.c_void_p, _DP, C.c_int]
    L.gmm_em_multisample.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p,
                                     C.c_void_p, _FP, C.c_void_p, _IP]
    L.gmm_get_multisample_profile.argtypes = [C.c_void_p, _DP, C.c_int]
    L.gmm_modes.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_double, C.c_double, _IP, C.c_void_p, C.c_void_p, C.c_void_p,
                            C.c_void_p, C.c_void_p]
    L.gmm_mode_labels.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p, C.c_int, C.c_int, C.c_double,
                                  C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_longlong),
                                  C.POINTER(C.c_longlong)]
    L.gmm_get_modes_profile.argtypes = [C.c_void_p, _DP, C.c_int]
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


def host_vb_finalize(stats, shift, cl, K, mean, covariance, prior_type=VB_DIRICHLET_PROCESS, weight_concentration=None,
                     mean_precision=None, dof=None, reg_covar=None):
    """VB M-step on the host (gmm_host_vb_finalize): packed statistics about `shift` -> the VB parameter set in cl (N, pi,
    constant, means, R, Rinv) and the posterior.  The prior's mean and covariance are required here.
    Returns (posterior dict, bound without its entropy term)."""
    stats = np.ascontiguousarray(stats, np.float64)
    shift = np.ascontiguousarray(shift, np.float64)
    assert stats.size >= stats_len(K, cl.D) and shift.size >= cl.D
    p, keep = _vb_prior(cl.D, prior_type, weight_concentration, mean_precision, dof, mean, covariance, reg_covar)
    post, ps = _vb_posterior(K, cl.D, prior_type)
    bound = C.c_double()
    s = cl.struct()
    _check(load_library().gmm_host_vb_finalize(stats.ctypes.data_as(_DP), shift.ctypes.data_as(_DP), K, cl.D, C.byref(p), C.byref(s),
                                               C.byref(ps), C.byref(bound)))
    del keep
    return post, bound.value


def host_digamma(x):
    """The library's double digamma (the psi of gmm_vb_em's bound and E-step offsets)."""
    x = np.ascontiguousarray(x, np.float64).reshape(-1)
    out = np.empty_like(x)
    _check(load_library().gmm_host_digamma(x.ctypes.data_as(_DP), out.ctypes.data_as(_DP), x.size))
    return out


def host_combine_groups(merges, K, L):
    """The cluster of each of K components at level L of a gmm_combine hierarchy (gmm_host_combine_groups): int32 [K],
    clusters numbered 0 .. L-1 in increasing order of their smallest component."""
    m = np.ascontiguousarray(merges, np.int32).reshape(-1)
    out = np.empty(max(int(K), 1), np.int32)
    _check(load_library().gmm_host_combine_groups(m.ctypes.data if m.size else None, int(K), int(L), out.ctypes.data))
    return out[:K]


def host_combine_elbow(entropy, x=None):
    """The level L of the change point of entropy [K] against x [K] (default 1 .. K) (gmm_host_combine_elbow)."""
    e = np.ascontiguousarray(entropy, np.float64).reshape(-1)
    xa = None if x is None else np.ascontiguousarray(x, np.float64).reshape(-1)
    if xa is not None and xa.size != e.size:
        raise ValueError(f"x must have {e.size} values, got {xa.size}")
    L = C.c_int()
    _check(load_library().gmm_host_combine_elbow(e.ctypes.data if e.size else None, xa.ctypes.data if xa is not None else None,
                                                 int(e.size), C.byref(L)))
    return L.value


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

    def seed_kmeans(self, K, max_iter=300, seed=0, out=None):
        """k-means++ + Lloyd initialisation (gmm_seed_kmeans): sklearn's init_params='kmeans' mixture.
        Returns (clusters, centres [K][D] float32, Lloyd centre updates, inertia)."""
        out = out or self.new_clusters()
        s = out.struct()
        cent = np.empty((K, self.D), np.float32)
        it, inertia = C.c_int(), C.c_double()
        _check(self.lib.gmm_seed_kmeans(self.h, K, max_iter, C.c_ulonglong(seed & 0xFFFFFFFFFFFFFFFF), C.byref(s),
                                        cent.ctypes.data_as(_FP), C.byref(it), C.byref(inertia)))
        return out, cent, it.value, inertia.value

    def set_clusters(self, K, cl):
        s = cl.struct()
        _check(self.lib.gmm_set_clusters(self.h, K, C.byref(s)))

    def set_weights(self, w=None):
        """Per-event weights of this shard (gmm_set_weights): float32 [n_local], finite, >= 0; None clears them.
        Returns the global sum of the weights."""
        ptr = None
        if w is not None:
            w = np.ascontiguousarray(w, np.float32)
            if w.shape != (self.n,):
                raise ValueError(f"weights must be [{self.n}], got {w.shape}")
            ptr = w.ctypes.data if w.size else None
            if ptr is None:                                 # an empty shard still sets (zero) weights
                w = np.zeros(1, np.float32)
                ptr = w.ctypes.data
        total = C.c_double()
        _check(self.lib.gmm_set_weights(self.h, ptr, C.byref(total)))
        return total.value

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

    def score(self, K, events, labels=True, max_resp=True, logp=True):
        """Assign and score new events (gmm_score) against the current K-cluster parameters.
        Returns (labels int32, max_resp float32, logp float32, loglik) with None for outputs not asked for."""
        ev = np.ascontiguousarray(events, np.float32)
        if ev.ndim != 2 or ev.shape[1] != self.D:
            raise ValueError(f"events must be [n][{self.D}], got {ev.shape}")
        n = ev.shape[0]
        lab = np.empty(n, np.int32) if labels else None
        mr = np.empty(n, np.float32) if max_resp else None
        lp = np.empty(n, np.float32) if logp else None
        ptr = lambda a: a.ctypes.data if a is not None and a.size else None  # noqa: E731
        ll = C.c_double()
        _check(self.lib.gmm_score(self.h, K, ptr(ev), n, ptr(lab), ptr(mr), ptr(lp), C.byref(ll)))
        return lab, mr, lp, ll.value

    def score_profile(self, reset=False):
        out = (C.c_double * 4)()
        _check(self.lib.gmm_get_score_profile(self.h, out, int(reset)))
        return dict(kernel_ms=out[0], wall_ms=out[1], tensor_chunks=int(out[2]), simt_chunks=int(out[3]))

    def score_stats(self, K, events, stats=True, memberships=False):
        """E-step + M-step statistics of new events (gmm_score_stats) under the current K-cluster parameters.
        Returns (stats [K*F+1] float64 or None, shift [D] float64, memberships [K][n] float32 or None).
        host_finalize(stats, shift, cl, K) turns the statistics into N, pi, means, R, Rinv and constants
        (regularised by cl.avgvar: set it to 0 for the raw per-sample covariances)."""
        ev = np.ascontiguousarray(events, np.float32)
        if ev.ndim != 2 or ev.shape[1] != self.D:
            raise ValueError(f"events must be [n][{self.D}], got {ev.shape}")
        n = ev.shape[0]
        st = np.empty(stats_len(K, self.D), np.float64) if stats else None
        sh = np.empty(self.D, np.float64)
        mb = np.empty((K, n), np.float32) if memberships else None
        ptr = lambda a: a.ctypes.data if a is not None else None  # noqa: E731
        _check(self.lib.gmm_score_stats(self.h, K, ev.ctypes.data if n else None, n, ptr(st), ptr(sh), ptr(mb)))
        return st, sh, mb

    def score_stats_profile(self, reset=False):
        out = (C.c_double * 7)()
        _check(self.lib.gmm_get_score_stats_profile(self.h, out, int(reset)))
        return dict(kernel_ms=out[0], wall_ms=out[1], estep_tensor_chunks=int(out[2]), estep_simt_chunks=int(out[3]),
                    mstep_tensor_chunks=int(out[4]), mstep_simt_chunks=int(out[5]), flag_wait_ms=out[6])

    def sample(self, K, n, seed=0, first=0, labels=True):
        """Draw events first .. first + n - 1 of the sample `seed` from the current K-cluster mixture (gmm_sample).
        Returns (events float32 [n][D], labels int32 [n] or None)."""
        n = int(n)
        ev = np.empty((max(n, 0), self.D), np.float32)
        lab = np.empty(max(n, 0), np.int32) if labels else None
        _check(self.lib.gmm_sample(self.h, K, n, C.c_ulonglong(seed & 0xFFFFFFFFFFFFFFFF), first,
                                   ev.ctypes.data if ev.size else None, lab.ctypes.data if lab is not None and lab.size else None))
        return ev, lab

    def sample_profile(self, reset=False):
        out = (C.c_double * 2)()
        _check(self.lib.gmm_get_sample_profile(self.h, out, int(reset)))
        return dict(kernel_ms=out[0], wall_ms=out[1])

    def condition(self, K, obs_dims, events_obs, labels=True, max_resp=True, logp=True, mean=True, var=False):
        """Score events measured on the dimensions obs_dims only and impute the others (gmm_condition) under the current
        K-cluster parameters.  events_obs is [n][len(obs_dims)].  Returns (labels int32, max_resp float32, logp float32,
        mean float32 [n][NM], var float32 [n][NM], loglik) with None for outputs not asked for; NM = D - len(obs_dims),
        and mean / var are None when NM = 0."""
        obs = np.ascontiguousarray(obs_dims, np.int32).reshape(-1)
        ev = np.ascontiguousarray(events_obs, np.float32)
        if ev.ndim != 2 or ev.shape[1] != obs.size:
            raise ValueError(f"events_obs must be [n][{obs.size}], got {ev.shape}")
        n, nm = ev.shape[0], self.D - obs.size
        lab = np.empty(n, np.int32) if labels else None
        mr = np.empty(n, np.float32) if max_resp else None
        lp = np.empty(n, np.float32) if logp else None
        cm = np.empty((n, nm), np.float32) if mean and nm > 0 else None
        cv = np.empty((n, nm), np.float32) if var and nm > 0 else None
        ptr = lambda a: a.ctypes.data if a is not None and a.size else None  # noqa: E731
        ll = C.c_double(0.0)
        _check(self.lib.gmm_condition(self.h, K, obs.ctypes.data if obs.size else None, int(obs.size), ptr(ev), n, ptr(lab),
                                      ptr(mr), ptr(lp), ptr(cm), ptr(cv), C.byref(ll)))
        return lab, mr, lp, cm, cv, ll.value

    def condition_profile(self, reset=False):
        out = (C.c_double * 2)()
        _check(self.lib.gmm_get_condition_profile(self.h, out, int(reset)))
        return dict(kernel_ms=out[0], wall_ms=out[1])

    def condition_stats(self, K, obs_dims, events_obs, stats=True, memberships=False):
        """M-step statistics of events measured on the dimensions obs_dims only (gmm_condition_stats): the expected full-D
        statistics under the current K-cluster parameters, and the posteriors under the marginal mixture of obs_dims.
        events_obs is [n][len(obs_dims)].  Returns (stats [K*F+1] float64 or None, shift [D] float64, memberships [K][n]
        float32 or None).  The statistics add to gmm_score_stats' and to other calls'; host_finalize turns their sum into
        one EM iteration."""
        obs = np.ascontiguousarray(obs_dims, np.int32).reshape(-1)
        ev = np.ascontiguousarray(events_obs, np.float32)
        if ev.ndim != 2 or ev.shape[1] != obs.size:
            raise ValueError(f"events_obs must be [n][{obs.size}], got {ev.shape}")
        n = ev.shape[0]
        st = np.empty(stats_len(K, self.D), np.float64) if stats else None
        sh = np.empty(self.D, np.float64)
        mb = np.empty((K, n), np.float32) if memberships else None
        ptr = lambda a: a.ctypes.data if a is not None else None  # noqa: E731
        _check(self.lib.gmm_condition_stats(self.h, K, obs.ctypes.data if obs.size else None, int(obs.size), ev.ctypes.data if n else None,
                                            n, ptr(st), ptr(sh), ptr(mb)))
        return st, sh, mb

    def condition_stats_profile(self, reset=False):
        out = (C.c_double * 4)()
        _check(self.lib.gmm_get_condition_stats_profile(self.h, out, int(reset)))
        return dict(kernel_ms=out[0], wall_ms=out[1], mstep_tensor_chunks=int(out[2]), mstep_simt_chunks=int(out[3]))

    def fit_profile(self):
        out = (C.c_double * 4)()
        _check(self.lib.gmm_get_fit_profile(self.h, out))
        return dict(reduce_order_ms=out[0], seed_ms=out[1], save_ms=out[2], device_finalize_launches=int(out[3]),
                    host_replays=int(round((out[3] - int(out[3])) * 1000)))

    def vb_em(self, K, min_iters=0, max_iters=100, tol=1e-3, prior_type=VB_DIRICHLET_PROCESS, weight_concentration=None,
              mean_precision=None, dof=None, mean=None, covariance=None, reg_covar=None, lower_bounds=False, out=None):
        """Variational Bayesian EM at K components from the current K-cluster parameters (gmm_vb_em; sklearn's
        BayesianGaussianMixture with covariance_type='full').  None selects the prior's default (sklearn's).
        Returns (clusters, posterior dict, lower bound, bounds per iteration or None, iterations, converged)."""
        out = out or self.new_clusters()
        p, keep = _vb_prior(self.D, prior_type, weight_concentration, mean_precision, dof, mean, covariance, reg_covar)
        post, ps = _vb_posterior(K, self.D, prior_type)
        lbs = np.full(max(int(max_iters), 1), np.nan) if lower_bounds else None
        lb, it, conv = C.c_double(), C.c_int(), C.c_int()
        s = out.struct()
        _check(self.lib.gmm_vb_em(self.h, K, C.byref(p), int(min_iters), int(max_iters), float(tol), C.byref(s), C.byref(ps), C.byref(lb),
                                  lbs.ctypes.data_as(_DP) if lbs is not None else None, C.byref(it), C.byref(conv)))
        del keep
        return out, post, lb.value, (lbs[:it.value] if lbs is not None else None), it.value, bool(conv.value)

    def vb_profile(self, reset=False):
        out = (C.c_double * 3)()
        _check(self.lib.gmm_get_vb_profile(self.h, out, int(reset)))
        return dict(entropy_ms=out[0], finalize_ms=out[1], wall_ms=out[2])

    def combine(self, K):
        """Entropy-criterion hierarchy of the K components over the memberships of the last E-step (gmm_combine).
        Returns dict(merges int32 [K-1][2], gain [K-1], entropy [K] (entropy[L-1] at L clusters), mass [K-1])."""
        merges = np.zeros((max(K - 1, 1), 2), np.int32)
        gain, mass = np.zeros(max(K - 1, 1)), np.zeros(max(K - 1, 1))
        ent = np.zeros(K)
        _check(self.lib.gmm_combine(self.h, K, merges.ctypes.data, gain.ctypes.data, ent.ctypes.data, mass.ctypes.data))
        return dict(merges=merges[:K - 1], gain=gain[:K - 1], entropy=ent, mass=mass[:K - 1])

    def combine_labels(self, K, group, G=None, max_sum=True):
        """Labels of this shard's events under a grouping of the K components (gmm_combine_labels): group int [K] with
        values in [0, G), G = max + 1 by default.  Returns (labels int32 [n], the group sum of the label float32 [n] or
        None)."""
        g = np.ascontiguousarray(group, np.int32).reshape(-1)
        if g.size != K:
            raise ValueError(f"group must have {K} values, got {g.size}")
        if G is None:
            G = int(g.max()) + 1 if g.size else 0
        lab = np.empty(max(self.n, 1), np.int32)
        mx = np.empty(max(self.n, 1), np.float32) if max_sum else None
        _check(self.lib.gmm_combine_labels(self.h, K, g.ctypes.data, G, lab.ctypes.data, mx.ctypes.data if mx is not None else None))
        return lab[:self.n], (mx[:self.n] if mx is not None else None)

    def combine_profile(self, reset=False):
        out = (C.c_double * 3)()
        _check(self.lib.gmm_get_combine_profile(self.h, out, int(reset)))
        return dict(kernel_ms=out[0], wall_ms=out[1], labels_wall_ms=out[2])

    def em_multisample(self, K, offsets, pi_init=None, min_iters=0, max_iters=100, epsilon=-1.0, logliks=False):
        """EM over S samples with shared components and per-sample mixing weights (gmm_em_multisample), from the current
        K-cluster parameters.  offsets: the S + 1 global event offsets of the samples; pi_init: [S][K] starting weights or
        None (the pooled pi).  Returns (pi [S][K] float64, n [S] float64, loglik, iters, logliks [iters + 1] or None)."""
        off = np.ascontiguousarray(offsets, np.int64).reshape(-1)
        S = off.size - 1
        if S < 1:
            raise ValueError("offsets must hold at least two values")
        p0 = None
        if pi_init is not None:
            p0 = np.ascontiguousarray(pi_init, np.float64)
            if p0.shape != (S, K):
                raise ValueError(f"pi_init must be [{S}][{K}], got {p0.shape}")
        pi = np.empty((S, K), np.float64)
        n = np.empty(S, np.float64)
        lls = np.full(max(int(max_iters), 0) + 1, np.nan, np.float32) if logliks else None
        ll, it = C.c_float(), C.c_int()
        _check(self.lib.gmm_em_multisample(self.h, K, S, off.ctypes.data, p0.ctypes.data if p0 is not None else None, int(min_iters),
                                           int(max_iters), float(epsilon), pi.ctypes.data, n.ctypes.data, C.byref(ll),
                                           lls.ctypes.data if lls is not None else None, C.byref(it)))
        return pi, n, ll.value, it.value, (lls[:it.value + 1] if lls is not None else None)

    def multisample_profile(self, reset=False):
        out = (C.c_double * 3)()
        _check(self.lib.gmm_get_multisample_profile(self.h, out, int(reset)))
        return dict(kernel_ms=out[0], host_ms=out[1], wall_ms=out[2])

    def modes(self, K, max_iter=500, tol=-1.0, merge_tol=-1.0):
        """The modes of the current K-component mixture reached from its means (gmm_modes).  Returns dict(modes [M][D]
        float64, logp [M], is_max bool [M], comp_mode int32 [K] (-1: pi = 0 or unconverged), iters int32 [K])."""
        modes = np.zeros((K, self.D), np.float64)
        lp = np.zeros(K, np.float64)
        cm, ismax, it = np.zeros(K, np.int32), np.zeros(K, np.int32), np.zeros(K, np.int32)
        nm = C.c_int()
        _check(self.lib.gmm_modes(self.h, K, int(max_iter), float(tol), float(merge_tol), C.byref(nm), modes.ctypes.data, lp.ctypes.data,
                                  cm.ctypes.data, ismax.ctypes.data, it.ctypes.data))
        m = nm.value
        return dict(modes=modes[:m], logp=lp[:m], is_max=ismax[:m].astype(bool), comp_mode=cm, iters=it)

    def mode_labels(self, K, modes, events=None, max_iter=500, tol=-1.0, merge_tol=-1.0, endpoints=False, logp=False, iters=False):
        """Each event's ascent (gmm_mode_labels) against the mode list modes [M][D]; events [n][D], or None for the
        context's own shard.  Returns dict(labels int32 [n] (-1 unconverged, -2 near no listed mode), endpoints [n][D]
        float32, logp [n] float32, iters int32 [n] (None when not asked for), unmatched, unconverged)."""
        md = np.ascontiguousarray(modes, np.float64).reshape(-1, self.D)
        if events is None:
            ev, n = None, self.n
        else:
            ev = np.ascontiguousarray(events, np.float32)
            if ev.ndim != 2 or ev.shape[1] != self.D:
                raise ValueError(f"events must be [n][{self.D}], got {ev.shape}")
            n = ev.shape[0]
        lab = np.empty(max(n, 1), np.int32)
        ep = np.empty((max(n, 1), self.D), np.float32) if endpoints else None
        lp = np.empty(max(n, 1), np.float32) if logp else None
        it = np.empty(max(n, 1), np.int32) if iters else None
        um, uc = C.c_longlong(), C.c_longlong()
        ptr = lambda a: a.ctypes.data if a is not None else None  # noqa: E731
        _check(self.lib.gmm_mode_labels(self.h, K, ptr(ev), n, md.ctypes.data if md.size else None, md.shape[0], int(max_iter),
                                        float(tol), float(merge_tol), lab.ctypes.data, ptr(ep), ptr(lp), ptr(it), C.byref(um),
                                        C.byref(uc)))
        cut = lambda a: a[:n] if a is not None else None  # noqa: E731
        return dict(labels=lab[:n], endpoints=cut(ep), logp=cut(lp), iters=cut(it), unmatched=um.value, unconverged=uc.value)

    def modes_profile(self, reset=False):
        out = (C.c_double * 4)()
        _check(self.lib.gmm_get_modes_profile(self.h, out, int(reset)))
        return dict(kernel_ms=out[0], modes_wall_ms=out[1], labels_wall_ms=out[2], event_iterations=int(out[3]))

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
