"""The error models behind tests/test_gpu_cluster_cap.py at the cluster cap, on the CPU: the tensor E-step and scoring
emulations of tests/test_estep_error_model.py at K = 257, 449 and 512 (5, 8 and 8 passes of 64 clusters, 449 with a
last pass of one cluster), and the tensor M-step error model of tests/test_mstep_error_model.py at K = 512 (8 grid rows,
16 column blocks).  The faithful FP32 emulations stay within a quarter of the bars and every fault of those modules still
exceeds them at one of these K, so the bars the GPU file holds the kernels to are valid at 8 passes.

Parameter sets: "mixture" puts every mean on one of the emulated events (tests/test_gpu_score.py's mixture: random SPD
covariances, Dirichlet weights), so that each of the 512 clusters carries responsibility somewhere; "spd" is
tests/test_estep_error_model.py's random SPD set (Mahalanobis distances of several hundred)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as entry  # noqa: E402
from test_estep_error_model import (FAULTS, SCORE_FAULTS, VARIANTS, Emulation, blobs, fp32_gamma, fp32_logits,  # noqa: E402
                                    fp32_score, fp32_y, param_set, standardise, variant_gamma)
from test_gpu_score import mixture  # noqa: E402
from test_mstep_error_model import VARIANTS as M_VARIANTS, model_errors, np_gamma  # noqa: E402

CAP_K = (257, 449, 512)
CAP_D = (8, 16, 24)
N_EMU = 600
KINDS = ("mixture", "spd")

_sets = {}


def cap_set(kind, D, K):
    """(parameter set, events, shift, scale) of a shape, made once."""
    key = (kind, D, K)
    if key not in _sets:
        pkg = entry.load_package()
        ev = blobs(D)
        x = np.ascontiguousarray(ev[:N_EMU])
        if kind == "mixture":
            cl = mixture(pkg, x, K, seed=D * 1000 + K)
        else:
            cl = param_set(pkg, entry.load_oracle("f64"), "spd", D, K, ev)
        shift, scale = standardise(ev)[:2]
        _sets[key] = (cl, x, shift, scale)
    return _sets[key]


_estep = {}


def estep_result(kind, D, K):
    key = (kind, D, K)
    if key not in _estep:
        cl, x, shift, scale = cap_set(kind, D, K)
        em = Emulation(cl, K, x, shift, scale)
        _estep[key] = {v: em.ratio(variant_gamma(em, v)) for v in VARIANTS}
    return _estep[key]


SHAPES = [(kind, D, K) for kind in KINDS for D in CAP_D for K in CAP_K]


@pytest.mark.parametrize("kind,D,K", SHAPES)
def test_estep_faithful_within_quarter_bar_at_the_cap(kind, D, K):
    r = estep_result(kind, D, K)
    print(f"\n{kind} D={D} K={K}: " + "  ".join(f"{v} {r[v]:.3g}" for v in VARIANTS))
    assert r["faithful_rn"] <= 0.25 and r["faithful_trunc"] <= 0.25, r


def test_each_estep_fault_exceeds_the_bar_at_the_cap():
    res = {s: estep_result(*s) for s in SHAPES}
    for v in FAULTS:
        caught = {s[2] for s, r in res.items() if r[v] > 1.0}
        print(f"\n  {v}: exceeds the bar at K in {sorted(caught)}")
        assert caught, v


_score = {}


def score_result(kind, D, K):
    """gmm_score's faithful FP32 emulation and each scoring fault against the bars, on the mixture set; "dup" is that set
    with the last pass a copy of the first (cluster 448 + k = cluster k), so that exact ties span 7 passes."""
    key = (kind, D, K)
    if key not in _score:
        cl, x, shift, scale = cap_set("mixture", D, K)
        if kind == "dup":
            cl = mixture(entry.load_package(), x, K, seed=D * 1000 + K)
            for f in ("means", "R", "Rinv", "constant", "pi", "N"):
                getattr(cl, f)[448:K] = getattr(cl, f)[0:K - 448]
        em = Emulation(cl, K, x, shift, scale)
        l32 = fp32_logits(em.op, fp32_y(em.op, em.zh, em.zl, trunc=False))
        lab, mr, lp = fp32_score(l32, K)
        g = fp32_gamma(l32, K)[0]
        res = {"faithful": em.score_check(lab, mr, lp), "identity": bool(np.array_equal(mr, g[np.arange(len(lab)), lab]))}
        for v in SCORE_FAULTS:
            res[v] = em.score_check(*fp32_score(l32, K, fault=v))
        _score[key] = res
    return _score[key]


SCORE_SHAPES = [("mixture", D, K) for D in CAP_D for K in CAP_K] + [("dup", D, K) for D in CAP_D for K in (449, 512)]


@pytest.mark.parametrize("kind,D,K", SCORE_SHAPES)
def test_score_faithful_within_quarter_bar_at_the_cap(kind, D, K):
    r = score_result(kind, D, K)
    print(f"\nscore {kind} D={D} K={K}: " + "  ".join(f"{v} {r[v][0]:.3g}/{r[v][1]:.3g}/{r[v][2]}" for v in ("faithful",) + SCORE_FAULTS))
    assert r["faithful"][0] <= 0.25 and r["faithful"][1] <= 0.25 and r["faithful"][2] == 0, r["faithful"]
    assert r["identity"]


def test_each_scoring_fault_fails_at_the_cap():
    res = {s: score_result(*s) for s in SCORE_SHAPES}
    for v in SCORE_FAULTS:
        caught = [s for s, r in res.items() if r[v][0] > 1.0 or r[v][1] > 1.0 or r[v][2] > 0]
        print(f"\n  {v}: caught at {len(caught)} of {len(res)} shapes")
        assert caught, v


@pytest.mark.parametrize("D", [8, 24])
def test_mstep_error_model_at_the_cap(D):
    """K = 512 on 20 000 events: every fault above MSTEP_TOL, the faithful scheme within half of it.  With about 40 events
    per cluster the per-cluster relative bar has less margin than at K <= 100: the faithful scheme reaches 0.48 of it at
    D = 8 (a quarter at the shapes of tests/test_mstep_error_model.py), as the kernel does on the H100 (0.42 - 0.49 at
    D = 4 and 8, K = 449 and 512)."""
    K = 512
    x = entry.load_package().synth.make_blobs(20_000, D, 16, seed=600 + D)
    errs, zb = model_errors(x, np_gamma(x, K, iters=1))
    print(f"\nD={D} K={K} zb={zb:g}: " + "  ".join(f"{v} {errs[v]['worst']:.3g}" for v in M_VARIANTS))
    assert errs["faithful"]["worst"] <= 0.5, errs["faithful"]
    for v in M_VARIANTS[1:]:
        assert errs[v]["worst"] > 1.0, (v, errs[v])


def test_mstep_error_model_at_the_full_plus_one_shard():
    """The shard of tests/test_gpu_cluster_cap.py's full+1 case (4 225 events: 66 CTAs of 64 and one of 1, K = 512, about
    8 events per cluster).  MSTEP_TOL does not hold for the kernel's own scheme there: the faithful emulation reaches 1.15
    of it on N at D = 12 (a cluster of mass ~1 made mostly of events with small g, where the FP16 rounding of g_l, relative
    2^-12, is not averaged out), against 0.49 on 20 000 events of the same mixture.  The GPU case therefore holds the
    kernel to this emulation rather than to MSTEP_TOL alone."""
    from scipy.special import softmax
    from test_gpu_score import ref_logits
    from test_mstep_error_model import cta_ranges
    D, K = 12, 512
    N = 64 * 66 + 1
    assert cta_ranges(N, 132) == (64, 67)
    pkg = entry.load_package()
    big = pkg.synth.make_blobs(20_000, D, 16, seed=840 + D)
    cl = mixture(pkg, big, K)
    worst = {}
    for n in (N, 20_000):
        x = np.ascontiguousarray(big[:n])
        g = softmax(ref_logits(cl, K, x), axis=1).T.astype(np.float32)
        worst[n] = model_errors(x, g, variants=("faithful",))[0]["faithful"]
    print(f"\nfull+1 shard: faithful {worst[N]['worst']:.3f} of MSTEP_TOL (N {worst[N]['N']:.3g}); 20 000 events "
          f"{worst[20_000]['worst']:.3f}")
    assert 1.0 < worst[N]["worst"] <= 1.25, worst[N]
    assert worst[20_000]["worst"] <= 0.5, worst[20_000]
