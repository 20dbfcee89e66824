"""Error model of the WEIGHTED tensor M-step (`mstep_tc_kernel<D, NCL, true>`, csrc/kernels_tc.cu), on the CPU, numpy only.

The weighted kernel multiplies each responsibility by the scaled weight w^ = f32(w / W) (W = the largest weight, so w^ is
at most 1) before the g_h / g_l / g_s split, and the finalisation multiplies the sums by W.
Its operand is therefore the unweighted kernel's operand for the responsibilities f32(w^ g), which lie in [0, 1] like g:
the emulator and the exact reference of tests/test_mstep_error_model.py apply unchanged (imported, not restated), and W
cancels in the relative errors they measure.

What changes is where the statistic sits in the operand.  Without weights most of it comes from events with g near 0 or 1,
which g_h (multiples of 2^-6) and g_s = fp16(1024 g) hold exactly; the FP16 rounding of g_l (relative 2^-12) only touches
the small-g tail.  A weight whose w^ is not 1 moves a whole group of confident events off those points together: their
g_s = fp16(1024 w^ g) share one rounding error, which multiplies the FP16 feature remainder p_l with one sign.  At the
widest legal data range (zb = 64, the largest p_l) two weight values 1 and 1.4 (R = 1.4) reach 0.32 of the per-cluster bar
(MSTEP_TOL), and a constant 0.7 scaled by a power of two (w^ = 0.7) twice the bar on R.  So the library admits the tensor
M-step for weighted data only when the dynamic range max w / min positive w is RANGE_TC = 1: one positive value, zeros
allowed (a constant factor, a subset of the rows, or both); the kernel divides by the largest weight, so w^ is exactly 0
or 1 and the operand is the unweighted one with rows removed.  Other weights run the FP64 SIMT M-step (gmm_api.cu
kWeightRangeTc).  This module pins the bound:
  * inside it (unit weights, a constant 0.7, and zero / one weights of value 3) the faithful scheme stays within a
    quarter of the bar at every M-step D and at zb = 64;
  * just outside it (values 1 and 1.4 at zb = 64) it does not.
Run it as a script (python tests/test_weights_error_model.py) for the worst errors per range R = 2^r (r = 0 .. 10, over
D = 4 .. 24 and K = 7, 33 at 20 000 events) of four weight laws: uniform in [0.5, 1] (R = 2 whatever is asked), integer
counts 1 .. R, log-uniform over [R^-1/2, R^1/2], and 1 % of the events at weight R among unit ones (which pushes the bulk
of every cluster down to w^ = 1 / R, below 2^-7 the statistic rides wholly in the FP16 remainder): the last reaches the
whole bar from R = 64.
"""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_mstep_error_model import emulate, exact_mstep_stats, mstep_errors, np_gamma, blobs, outlier_blobs  # noqa: E402

RANGE_TC = 1.0                         # largest max w / min positive w served by the tensor M-step (gmm_api.cu kWeightRangeTc)
LAWS = ("uniform", "counts", "loguniform", "heavy")         # weight laws of a given dynamic range R
INSIDE = ("unit", "constant", "zero_one")                    # weights inside RANGE_TC
M_STEP_D = (4, 8, 12, 16, 20, 24)


def weights(law, R, N, seed):
    rng = np.random.default_rng(seed)
    if law == "uniform":
        w = rng.uniform(0.5, 1.0, N)
    elif law == "counts":
        w = rng.integers(1, int(R) + 1, N).astype(np.float64)
        w[:2] = (1.0, R)                                # the range itself, whatever the draw
    elif law == "loguniform":
        w = np.sqrt(R) ** rng.uniform(-1.0, 1.0, N)
        w[:2] = (R ** -0.5, R ** 0.5)
    elif law == "unit":
        w = np.ones(N)
    elif law == "constant":
        w = np.full(N, 0.7)
    elif law == "zero_one":
        w = np.where(rng.uniform(size=N) < 0.7, 3.0, 0.0)
    elif law == "heavy":
        w = np.ones(N)
        w[rng.choice(N, max(1, N // 100), replace=False)] = R
    else:
        raise ValueError(law)
    return w.astype(np.float32)


def weighted_operand(g, w):
    """The responsibilities the weighted kernel feeds its split: f32(g * f32(w / W)), W = max w."""
    w = np.asarray(w, np.float32).astype(np.float64)
    wh = (w / w.max()).astype(np.float32)
    return (np.asarray(g, np.float32) * wh[None, :]).astype(np.float32)


def weighted_errors(x, g, w):
    gw = weighted_operand(g, w)
    emu, shift, zb = emulate(x, gw, variants=("faithful",))
    return mstep_errors(emu["faithful"], exact_mstep_stats(x, gw, shift), shift, g.shape[0]), zb


_data = {}


def shape_data(D, K, N=20_000):
    if (D, K) not in _data:
        x = blobs(N, D, min(K, 16), seed=700 + D)
        _data[(D, K)] = (x, np_gamma(x, K))
    return _data[(D, K)]


@pytest.mark.parametrize("law", INSIDE)
@pytest.mark.parametrize("K", (7, 33))
@pytest.mark.parametrize("D", M_STEP_D)
def test_weighted_scheme_within_quarter_bar_inside_range(D, K, law):
    x, g = shape_data(D, K)
    e, _ = weighted_errors(x, g, weights(law, RANGE_TC, len(x), seed=D * 100 + K))
    print(f"\nD={D} K={K} {law} R={RANGE_TC:g}: N {e['N']:.2e} mean {e['mean']:.2e} R {e['R']:.2e} (x bar {e['worst']:.3f})")
    assert e["worst"] <= 0.25, e


@pytest.mark.parametrize("law", INSIDE)
def test_weighted_scheme_at_zb64_within_quarter_bar(law):
    x = outlier_blobs(200_000, 12, 63.0, seed=711)
    g = np_gamma(x, 8)
    e, zb = weighted_errors(x, g, weights(law, RANGE_TC, len(x), seed=712))
    print(f"\nzb={zb:g} {law}: x bar {e['worst']:.3f}")
    assert zb == 64.0
    assert e["worst"] <= 0.25, e


def test_first_range_outside_exceeds_quarter_bar():
    """Any range above 1 admits a weight whose w^ is not 1 for a whole group of confident events: two values 1 and 1.4
    (R = 1.4) at the widest legal data range (zb = 64) leave the quarter of the bar."""
    x = outlier_blobs(200_000, 12, 63.0, seed=711)
    g = np_gamma(x, 8)
    w = np.where(np.arange(len(x)) % 2 == 0, 1.0, 1.4).astype(np.float32)
    e, zb = weighted_errors(x, g, w)
    print(f"\nzb={zb:g} two values 1, 1.4: N {e['N']:.2e} mean {e['mean']:.2e} R {e['R']:.2e} (x bar {e['worst']:.3f})")
    assert zb == 64.0
    assert e["worst"] > 0.25, e


if __name__ == "__main__":
    for r in range(0, 11):
        R = 2.0 ** r
        row = []
        for law in LAWS:
            row.append(max(weighted_errors(*shape_data(D, K), weights(law, R, 20_000, seed=D * 100 + K))[0]["worst"]
                           for D in M_STEP_D for K in (7, 33)))
        print(f"R = 2^{r:2d}: " + "  ".join(f"{law} {v:.3f}" for law, v in zip(LAWS, row)), flush=True)
