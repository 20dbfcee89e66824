"""GPU parity tests beyond one operator on one small input (run with -m gpu on an H100):

* gmm_em_iterations (the unit bench.py times) against the oracle's EM, from every state it can be entered in;
* the sharded path through the C ABI — one gmm_ctx per GPU driven from one host thread each, joined by the
  ncclAllReduce of the packed statistics (gaussian.cu:348-352 shard rule, :550-687 reductions) — against the
  single-GPU result and the oracle, at 2 / 4 / 8 GPUs (self-skipping below the needed GPU count);
* full-size parity: BASELINE config 2 for 50 iterations and one E-step + one M-step at config 3
  (N=10M, D=24, K=64) against the f64 oracle.
"""
import threading

import numpy as np
import pytest

from conftest import assert_params_close, gpu_count, RUN_RTOL_N, RUN_MEMB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def loaded(pkg):
    pkg.load_library()
    return pkg


def _oracle_em(pkg, oracle, ev, K, iters):
    ref = pkg.Clusters(K, ev.shape[1], ev.shape[0])
    oracle.seed(ev, K, ref)
    ll, _ = oracle.em(oracle.transpose(ev), ref, K, iters, iters)
    return ref, ll


@pytest.mark.parametrize("path", ["simt", "auto"])
def test_em_iterations_matches_oracle(loaded, oracle64, path):
    """estep + em_iterations(n) == oracle.em(n, n): on a fresh context, again after a finished gmm_em (whose last
    M-step left reduced statistics in the device buffer), and after gmm_upload_events of a different data set."""
    pkg = loaded
    N, D, K, n = 30_000, 8, 6, 5
    ev = pkg.synth.make_blobs(N, D, K, seed=41)
    ev2 = pkg.synth.make_blobs(N, D, K, seed=42)
    ref, ll_ref = _oracle_em(pkg, oracle64, ev, K, n)
    ref2, ll_ref2 = _oracle_em(pkg, oracle64, ev2, K, n)
    p = {"simt": pkg.PATH_SIMT, "auto": pkg.PATH_AUTO}[path]

    def check(eng, r, llr):
        got = eng.get_clusters(K, with_memberships=True)
        assert_params_close(got, r, K, rtol_N=RUN_RTOL_N)
        np.testing.assert_allclose(got.memberships, r.memberships, **RUN_MEMB)
        return got

    with pkg.Engine(ev, K) as eng:
        eng.set_option("path", p)
        seeded = eng.seed(K)
        eng.estep(K)
        ll = eng.em_iterations(K, n)
        assert abs(ll - ll_ref) <= 1e-5 * abs(ll_ref)
        check(eng, ref, ll_ref)
        # a finished gmm_em leaves the statistics of its last M-step behind; start over from the seed
        eng.em(K, 2, 2)
        eng.set_clusters(K, seeded)
        eng.estep(K)
        ll = eng.em_iterations(K, n)
        assert abs(ll - ll_ref) <= 1e-5 * abs(ll_ref)
        check(eng, ref, ll_ref)
        # new events in the same context: moments, shift and the E-step operand are rebuilt
        eng.upload_events(ev2)
        with pytest.raises(pkg.GmmError):
            eng.estep(K)                       # parameters have to be set again after an upload
        eng.seed(K)
        eng.estep(K)
        ll = eng.em_iterations(K, n)
        assert abs(ll - ll_ref2) <= 1e-5 * abs(ll_ref2)
        check(eng, ref2, ll_ref2)


def _run_sharded(pkg, ev, K, G, iters, path, allreduce=1):
    """G contexts (one per GPU, one host thread each) through the C ABI; returns rank 0's clusters with the
    memberships of all shards gathered, the log-likelihood and every rank's parameters."""
    N, D = ev.shape
    uid = pkg.nccl_unique_id() if G > 1 else None
    out, errs = [None] * G, [None] * G

    def worker(g):
        try:
            b, n = pkg.shard_range(N, G, g)
            with pkg.Engine(np.ascontiguousarray(ev[b:b + n]), K, device=g, n_global=N, offset=b) as eng:
                eng.set_option("path", path)
                eng.set_option("allreduce", allreduce)
                eng.comm_init(G, g, uid)
                eng.seed(K)
                ll, it = eng.em(K, iters, iters)
                out[g] = (eng.get_clusters(K, with_memberships=True), ll, it, b, n)
        except Exception as ex:  # noqa: BLE001
            errs[g] = ex

    ts = [threading.Thread(target=worker, args=(g,)) for g in range(G)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=600)
    for g in range(G):
        assert errs[g] is None, f"rank {g}: {errs[g]}"
        assert out[g] is not None, f"rank {g} did not finish"
    merged = out[0][0].copy()
    merged.memberships = np.zeros((K, N), np.float32)
    merged.n_events = N
    for cl, _, _, b, n in out:
        merged.memberships[:, b:b + n] = cl.memberships[:K]
    return merged, out[0][1], [o[0] for o in out]


@pytest.mark.parametrize("G", [2, 4, 8])
@pytest.mark.parametrize("path", ["simt", "auto"])
def test_sharded_c_abi_equals_single_gpu_and_oracle(loaded, oracle64, G, path):
    """gaussian.cu:348-352 (shards) + :550-687 (reductions) at the C-ABI level: G GPUs == 1 GPU == oracle (run-level
    bar); all ranks bit-identical."""
    if gpu_count() < G:
        pytest.skip(f"needs >= {G} GPUs")
    pkg = loaded
    N, D, K, iters = 120_003, 16, 12, 8          # odd N: remainder on the last shard
    ev = pkg.synth.make_blobs(N, D, K, seed=71)
    p = {"simt": pkg.PATH_SIMT, "auto": pkg.PATH_AUTO}[path]
    one, ll1, _ = _run_sharded(pkg, ev, K, 1, iters, p)
    many, llg, per_rank = _run_sharded(pkg, ev, K, G, iters, p)
    for f in ("N", "pi", "constant", "means", "R", "Rinv"):
        for r in per_rank[1:]:
            np.testing.assert_array_equal(getattr(r, f)[:K], getattr(per_rank[0], f)[:K], err_msg=f"rank-divergent {f}")
    assert abs(llg - ll1) <= 2e-6 * abs(ll1)
    # SIMT path: the statistics are FP64 sums, only their order differs.  Tensor path: each CTA keeps FP32 partial sums over
    # ITS event range, and the ranges change with the shard size: rounding noise of ~1e-7 per call, grown over 8 iterations.
    assert_params_close(many, one, K, rtol=2e-6 if path == "simt" else 5e-5)
    if path == "simt":
        np.testing.assert_allclose(many.memberships, one.memberships, rtol=1e-4, atol=2e-6)
    else:
        np.testing.assert_allclose(many.memberships, one.memberships, **RUN_MEMB)
    ref, ll_ref = _oracle_em(pkg, oracle64, ev, K, iters)
    assert abs(llg - ll_ref) <= 1e-5 * abs(ll_ref)
    assert_params_close(many, ref, K, rtol_N=RUN_RTOL_N)
    np.testing.assert_allclose(many.memberships, ref.memberships, **RUN_MEMB)


@pytest.mark.parametrize("G", [2, 8])
def test_peer_memory_allreduce_equals_nccl(loaded, G):
    """The statistics all-reduce of this library (one kernel over NVLink peer memory, rank-ordered sums) against
    ncclAllReduce on the same run: the packed statistics are doubles, only the summation order differs."""
    if gpu_count() < G:
        pytest.skip(f"needs >= {G} GPUs")
    pkg = loaded
    N, D, K, iters = 90_001, 24, 20, 6
    ev = pkg.synth.make_blobs(N, D, K, seed=72)
    a, lla, ranks_a = _run_sharded(pkg, ev, K, G, iters, pkg.PATH_AUTO, allreduce=1)
    b, llb, _ = _run_sharded(pkg, ev, K, G, iters, pkg.PATH_AUTO, allreduce=0)
    for f in ("N", "pi", "constant", "means", "R", "Rinv"):
        for r in ranks_a[1:]:
            np.testing.assert_array_equal(getattr(r, f)[:K], getattr(ranks_a[0], f)[:K], err_msg=f"rank-divergent {f}")
    assert abs(lla - llb) <= 1e-6 * abs(llb)
    assert_params_close(a, b, K, rtol=1e-6)
    np.testing.assert_allclose(a.memberships, b.memberships, rtol=1e-5, atol=1e-7)


@pytest.mark.parametrize("path", ["simt", "auto"])
def test_full_size_config2_50_iterations(loaded, oracle64, path):
    """BASELINE config 2 at full size (N=1M, D=16, K=32), the 50 iterations the config names, against the f64 oracle."""
    pkg = loaded
    cfg = pkg.synth.CONFIGS["c2"]
    N, D, K = cfg["N"], cfg["D"], cfg["K"]
    ev = pkg.synth.make_blobs(N, D, K)
    ref, ll_ref = _oracle_em(pkg, oracle64, ev, K, 50)
    with pkg.Engine(ev, K) as eng:
        eng.set_option("path", {"simt": pkg.PATH_SIMT, "auto": pkg.PATH_AUTO}[path])
        eng.seed(K)
        ll, it = eng.em(K, 50, 50)
        got = eng.get_clusters(K, with_memberships=True)
    assert it == 50
    assert abs(ll - ll_ref) <= 1e-5 * abs(ll_ref)
    assert_params_close(got, ref, K, rtol_N=RUN_RTOL_N)
    np.testing.assert_allclose(got.memberships, ref.memberships, **RUN_MEMB)


def test_full_size_config3_one_estep_one_mstep(loaded, oracle64):
    """BASELINE config 3 at full size (N=10M, D=24, K=64) on the default (tensor) path: one E-step and one M-step +
    constants from identical inputs against the f64 oracle, at the per-operator 1e-4 bar."""
    pkg = loaded
    cfg = pkg.synth.CONFIGS["c3"]
    N, D, K = cfg["N"], cfg["D"], cfg["K"]
    ev = pkg.synth.make_blobs(N, D, K)
    # realistic parameters: the oracle's EM on a 200k slice (seconds), then evaluated on all 10M events
    sl = np.ascontiguousarray(ev[:200_000])
    start = pkg.Clusters(K, D, sl.shape[0])
    oracle64.seed(sl, K, start)
    oracle64.em(oracle64.transpose(sl), start, K, 3, 3)
    ref = pkg.Clusters(K, D, N)
    for f in pkg.Clusters.FIELDS:
        getattr(ref, f)[...] = getattr(start, f)
    del start
    soa = oracle64.transpose(ev)
    with pkg.Engine(ev, K) as eng:
        eng.seed(K)
        eng.set_clusters(K, ref)
        ll = eng.estep(K)
        got = eng.get_clusters(K, with_memberships=True)
        ll_ref = oracle64.estep(soa, ref, K)
        np.testing.assert_allclose(got.memberships, ref.memberships, rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(got.memberships.sum(0), 1.0, atol=1e-5)
        assert abs(ll - ll_ref) <= 1e-5 * abs(ll_ref)
        del got
        eng.mstep(K)
        eng.constants(K)
        got = eng.get_clusters(K)
    oracle64.mstep(soa, ref, K)
    oracle64.constants(ref, K)
    assert_params_close(got, ref, K)


def test_upload_events_file_equals_array(loaded, tmp_path):
    """gmm_upload_events_file streams this shard's rows of a .bin file (readData.cpp:35-47 format) to the device through
    pinned staging buffers: bit-identical results to a context created from the host array, for a shard in the middle of
    the file; a header that does not match the context is refused."""
    pkg = loaded
    N, D, K = 50_001, 16, 5
    ev = pkg.synth.make_blobs(N, D, K, seed=91)
    path = str(tmp_path / "ev.bin")
    pkg.synth.write_bin(path, ev)
    b, n = 10_007, 30_000
    with pkg.Engine(np.ascontiguousarray(ev[b:b + n]), K, n_global=N, offset=b) as eng:
        eng.seed(K)
        ll_a, _ = eng.em(K, 3, 3)
        a = eng.get_clusters(K, with_memberships=True)
    with pkg.Engine(None, K, n_global=N, offset=b, n_local=n, D=D) as eng:
        eng.upload_events_file(path)
        eng.seed(K)
        ll_b, _ = eng.em(K, 3, 3)
        c = eng.get_clusters(K, with_memberships=True)
    assert ll_a == ll_b
    for f in ("N", "means", "R", "Rinv", "constant", "pi", "memberships"):
        np.testing.assert_array_equal(getattr(a, f), getattr(c, f))
    with pkg.Engine(None, K, n_global=N + 1, offset=0, n_local=n, D=D) as eng:
        with pytest.raises(pkg.GmmError):
            eng.upload_events_file(path)


def _run_iterations(pkg, ev, K, n, finalize, fault=None, em=False):
    with pkg.Engine(ev, K) as eng:
        eng.set_option("finalize", finalize)
        if fault is not None:
            eng.set_option("finalize_fault_iter", fault)
        eng.seed(K)
        if em:
            ll, iters = eng.em(K, n, n)
            assert iters == n
        else:
            eng.estep(K)
            ll = eng.em_iterations(K, n)
        got = eng.get_clusters(K, with_memberships=True)
        fp = eng.fit_profile()
        # a second batch in the same context (after a replay the context stays on the host path)
        ll2 = eng.em_iterations(K, 2)
        got2 = eng.get_clusters(K, with_memberships=True)
        fp2 = eng.fit_profile()
    return got, ll, fp, got2, ll2, fp2


@pytest.mark.parametrize("shape", [(30_000, 8, 6), (20_000, 16, 20), (25_000, 24, 64), (9_000, 24, 100)])
def test_device_finalisation_equals_host_finalisation(loaded, shape):
    """Option "finalize": the one-kernel device-side step between the reduced statistics and the next E-step (N, means, R,
    inverse, constants, pi, E-step operand) against the host finalisation of the same library — same arithmetic, so the
    two runs agree far inside the run-level tolerance — through gmm_em_iterations and through gmm_em (K > 64 included:
    two operand passes)."""
    pkg = loaded
    N, D, K = shape
    n = 6
    ev = pkg.synth.make_blobs(N, D, K, seed=77)
    for em in (False, True):
        host, ll_h, fp_h, host2, ll2_h, _ = _run_iterations(pkg, ev, K, n, 0, em=em)
        dev, ll_d, fp_d, dev2, ll2_d, fp2_d = _run_iterations(pkg, ev, K, n, 1, em=em)
        assert fp_h["device_finalize_launches"] == 0
        assert fp_d["device_finalize_launches"] == n and fp_d["host_replays"] == 0
        assert fp2_d["device_finalize_launches"] == n + 2
        for a, b, la, lb in ((dev, host, ll_d, ll_h), (dev2, host2, ll2_d, ll2_h)):
            assert abs(la - lb) <= 2e-6 * abs(lb)
            assert_params_close(a, b, K, rtol_N=2e-5)
            np.testing.assert_allclose(a.memberships, b.memberships, rtol=0, atol=2e-5)


@pytest.mark.parametrize("fault", [0, 3, 5])
def test_device_finalisation_replay_on_the_host(loaded, fault):
    """A finalisation that reports a cluster for the host path (forced by the test hook at iteration `fault` of 6): the
    work queued after it is discarded, the library replays from the last good parameter set through the host path, the
    result equals the all-host run, and the context stays on the host path afterwards."""
    pkg = loaded
    N, D, K, n = 25_000, 24, 32, 6
    ev = pkg.synth.make_blobs(N, D, K, seed=78)
    for em in (False, True):
        host, ll_h, _, host2, ll2_h, _ = _run_iterations(pkg, ev, K, n, 0, em=em)
        rep, ll_r, fp, rep2, ll2_r, fp2 = _run_iterations(pkg, ev, K, n, 1, fault=fault, em=em)
        assert fp["host_replays"] == 1 and fp["device_finalize_launches"] == n
        assert fp2["device_finalize_launches"] == n and fp2["host_replays"] == 1     # second batch: host path
        for a, b, la, lb in ((rep, host, ll_r, ll_h), (rep2, host2, ll2_r, ll2_h)):
            assert abs(la - lb) <= 2e-6 * abs(lb)
            assert_params_close(a, b, K, rtol_N=2e-5)
            np.testing.assert_allclose(a.memberships, b.memberships, rtol=0, atol=2e-5)
