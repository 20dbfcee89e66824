"""The restatement of gmm_modes / gmm_mode_labels (tests/_modes_ref.py) against analytic facts (no GPU needed)."""
import numpy as np
import pytest

import _modes_ref as mr


def _iso(means, s=1.0, pi=None):
    means = np.asarray(means, np.float64)
    K, D = means.shape
    pi = np.full(K, 1.0 / K) if pi is None else np.asarray(pi, np.float64)
    R = np.tile(np.eye(D) * s * s, (K, 1, 1))
    Rinv = np.tile(np.eye(D) / (s * s), (K, 1, 1))
    const = np.full(K, -0.5 * D * np.log(2 * np.pi * s * s))
    return mr.params(means, Rinv, R, const, pi)


def _modes_from_means(p, merge_tol=1e-2):
    ends, _, st = mr.climb(p, p["mu"])
    return mr.dedup(p, ends, st, merge_tol)


def test_one_component_reaches_the_mean_in_one_step():
    rng = np.random.default_rng(1)
    D = 5
    L = rng.normal(size=(D, D)) + 3 * np.eye(D)
    R = L @ L.T
    p = mr.params(rng.normal(size=(1, D)) * 100, np.linalg.inv(R)[None], R[None], [-3.0], [1.0])
    x0 = rng.normal(size=(4, D)) * 5
    x1 = x0 + mr.step(p, x0)[0]
    np.testing.assert_allclose(x1, np.repeat(p["mu"], 4, 0), atol=1e-9)
    _, it, st = mr.climb(p, x0)
    assert np.all(st == mr.CONVERGED) and np.all(it == 2)


@pytest.mark.parametrize("sep, want", [(1.9, 1), (2.1, 2)])
def test_two_equal_components_bimodal_beyond_two_sigma(sep, want):
    p = _iso([[0.0, 0.0], [sep, 0.0]])
    modes, cm = _modes_from_means(p)
    assert len(modes) == want
    assert np.all(mr.is_max(p, modes))


def _triangle(s):
    a = np.array([[np.cos(t), np.sin(t)] for t in (np.pi / 2, np.pi / 2 + 2 * np.pi / 3, np.pi / 2 + 4 * np.pi / 3)])
    return _iso(a, s)


def triangle_sigma():
    """The middle of the spreads (a grid in float64) for which the centroid of three vertices at unit distance from it is a
    strict local maximum while the means still climb to three vertex modes."""
    ok = []
    for s in np.linspace(0.60, 0.80, 201):
        p = _triangle(s)
        centroid = -p["c"][None]
        g, _ = mr.grad_hess(p, centroid)
        if np.max(np.abs(g)) < 1e-12 and mr.is_max(p, centroid)[0]:
            modes, _ = _modes_from_means(p)
            if len(modes) == 3 and np.all(mr.is_max(p, modes)):
                ok.append(float(s))
    return ok[len(ok) // 2] if ok else None


def test_triangle_has_a_mode_no_mean_reaches():
    s = triangle_sigma()
    assert s is not None
    p = _triangle(s)
    modes, cm = _modes_from_means(p)
    centroid = -p["c"]
    assert len(modes) == 3 and np.all(cm == [0, 1, 2])
    assert np.min(mr.rho(p, centroid[None], modes)) > 0.1
    ends, _, st = mr.climb(p, centroid[None] + 1e-3)
    assert st[0] == mr.CONVERGED and mr.rho(p, ends[0], centroid) < 1e-3
    assert mr.labels(p, ends, st, modes, 1e-2)[0] == -2


def test_logp_never_decreases():
    rng = np.random.default_rng(3)
    K, D = 12, 4
    means = rng.normal(size=(K, D)) * 3
    Ls = rng.normal(size=(K, D, D)) * 0.3 + np.eye(D)
    R = Ls @ np.swapaxes(Ls, 1, 2)
    p = mr.params(means, np.linalg.inv(R), R, -0.5 * np.log(np.linalg.det(R)), rng.dirichlet(np.ones(K)))
    _, _, st, hist = mr.climb(p, rng.normal(size=(500, D)) * 4, trace=True)
    h = np.array(hist)
    assert np.all(np.diff(h, axis=0) >= -1e-10 * np.abs(h[1:]))
    assert np.all(st == mr.CONVERGED)


def test_gradient_zero_and_hessian_negative_at_the_maxima():
    rng = np.random.default_rng(4)
    p = _iso(rng.normal(size=(6, 3)) * 4, 1.0, rng.dirichlet(np.ones(6)))
    modes, _ = _modes_from_means(p)
    g, _ = mr.grad_hess(p, modes)
    assert np.max(np.abs(g)) < 1e-6
    assert np.all(mr.is_max(p, modes))


def test_dedup_and_label_rules_with_ties():
    p = dict(inv_sigma=np.array([1.0, 2.0]), c=np.zeros(2))
    ends = np.array([[0.0, 0.0], [0.005, 0.0], [1.0, 0.0], [0.0, 0.006], [0.5, 0.5], [9.0, 9.0]])
    st = np.array([1, 1, 1, 1, 1, 2])
    modes, cm = mr.dedup(p, ends, st, 1e-2)
    # [0, 0.006]: rho = 0.012 from the first mode (sigma_1 = 0.5) -> a new mode
    assert len(modes) == 4 and list(cm) == [0, 0, 1, 2, 3, -1]
    two = np.array([[0.0, 0.0], [0.02, 0.0]])
    e = np.array([[0.01, 0.0], [0.012, 0.0], [0.5, 0.0], [0.0, 0.0]])
    lab = mr.labels(p, e, np.array([1, 1, 1, 2]), two, 1e-2)
    assert list(lab) == [0, 1, -2, -1]                            # an exact tie goes to the lower index
