"""CPU emulation of the tensor M-step's operand arithmetic (exact accumulation): which part of the per-call
covariance error comes from the FP16 hi/lo operand split (truncating vs round-to-nearest, 3 vs 4 products)?
Test infrastructure (uses the oracle); not part of the product.  The scheme the kernel runs now, with its CTA ranges,
chains and drains, is emulated by tests/test_mstep_error_model.py (python tests/test_mstep_error_model.py prints its table)."""
import sys, os
import numpy as np
sys.path.insert(0, os.getcwd())
import __graft_entry__ as e
pkg = e.load_package(); o64 = e.load_oracle("f64")

def split_trunc(v):
    v = v.astype(np.float32)
    hi = (v.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    lo = (v - hi).astype(np.float16).astype(np.float32)
    return hi.astype(np.float64), lo.astype(np.float64)

def split_rn(v):
    v = v.astype(np.float32)
    hi = v.astype(np.float16).astype(np.float32)
    lo = (v - hi).astype(np.float16).astype(np.float32)
    return hi.astype(np.float64), lo.astype(np.float64)

def cov_from_stats(S0, S1, S2):
    m = S1 / S0[:, None]
    return S2 / S0[:, None, None] - m[:, :, None] * m[:, None, :], m

def run(N, D, K, iters, seed=None):
    ev = pkg.synth.make_blobs(N, D, K) if seed is None else pkg.synth.make_blobs(N, D, K, seed=seed)
    ref = pkg.Clusters(K, D, N); o64.seed(ev, K, ref); o64.em(o64.transpose(ev), ref, K, iters, iters)
    g = ref.memberships.astype(np.float32)            # [K][N]
    x = ev.astype(np.float64)
    mean = x.mean(0); sd = x.std(0)
    sf = mean.astype(np.float32); isf = (1.0 / sd).astype(np.float32)
    z32 = ((ev - sf) * isf).astype(np.float32)
    # exact statistics from the float z (double) -> reference cov in z units
    zz = z32.astype(np.float64)
    gd = g.astype(np.float64)
    S0 = gd.sum(1); S1 = gd @ zz; S2 = np.einsum('kn,ni,nj->kij', gd, zz, zz)
    cov_ref, m_ref = cov_from_stats(S0, S1, S2)
    amp = (m_ref ** 2).max(1) / np.array([np.diag(cov_ref[k]).min() for k in range(K)])
    print(f"N={N} D={D} K={K}: cancellation factor max m^2/min var: median {np.median(amp):.0f} max {amp.max():.0f}")
    prod32 = (z32[:, :, None] * z32[:, None, :]).astype(np.float32)   # fl32 products as the builders form them
    for name, split, nprod in (("trunc3", split_trunc, 3), ("trunc4", split_trunc, 4), ("rn3", split_rn, 3), ("rn4", split_rn, 4)):
        gh, gl = split(g * np.float32(1024.0))
        oh, ol = split(np.ones(N, np.float32))
        zh, zl = split(z32)
        ph, pl = split(prod32.reshape(N, D * D)); ph = ph.reshape(N, D, D); pl = pl.reshape(N, D, D)
        def contract(fh, fl):
            r = gh @ fh + gh @ fl + gl @ fh
            if nprod == 4: r = r + gl @ fl
            return r / 1024.0
        s0 = contract(oh, ol)
        s1 = contract(zh, zl)
        s2 = contract(ph.reshape(N, D * D), pl.reshape(N, D * D)).reshape(K, D, D)
        cov, m = cov_from_stats(s0, s1, s2)
        dR = max(np.abs(cov[k] - cov_ref[k]).max() / np.abs(cov_ref[k]).max() for k in range(K))
        dS2 = np.abs(s2 / S2 - 1)[np.abs(S2) > 1e-3 * np.abs(S2).max()].max()
        print(f"  {name}: max rel cov err {dR:.2e}  dN {np.abs(s0 / S0 - 1).max():.2e}  dmean {np.abs(m - m_ref).max():.2e}  dS2(rel) {dS2:.2e}  bias S2 {np.mean((s2 / S2 - 1)[np.abs(S2) > 1e-2 * np.abs(S2).max()]):+.2e}")

run(10000, 4, 8, 20)
run(100000, 16, 32, 5)


PHI_BITS, G_BITS = 11, 6


def run_fixed(N, D, K, iters):
    """The round-2 operand scheme: fixed-point leading parts (exact accumulation) + FP16 remainders."""
    ev = pkg.synth.make_blobs(N, D, K)
    ref = pkg.Clusters(K, D, N); o64.seed(ev, K, ref); o64.em(o64.transpose(ev), ref, K, iters, iters)
    g = ref.memberships.astype(np.float32)
    x = ev.astype(np.float64)
    sf = x.mean(0).astype(np.float32); isf = (1.0 / x.std(0)).astype(np.float32)
    z32 = ((ev - sf) * isf).astype(np.float32)
    zz = z32.astype(np.float64); gd = g.astype(np.float64)
    S0 = gd.sum(1); S1 = gd @ zz; S2 = np.einsum('kn,ni,nj->kij', gd, zz, zz)
    cov_ref, m_ref = cov_from_stats(S0, S1, S2)
    zmax = 2.0 ** (np.floor(np.log2(np.abs(zz).max(0) * (1 + 1e-6))) + 1)
    f16 = lambda a: a.astype(np.float32).astype(np.float16).astype(np.float64)
    def fsplit(v, bound):
        q = bound / float(1 << PHI_BITS)
        h = np.round(v / q) * q
        return h, f16(v - h)
    gh = np.round(gd * float(1 << G_BITS)) / float(1 << G_BITS)
    gl = f16((gd - gh) * 1024.0) / 1024.0
    gs = f16(gd * 1024.0) / 1024.0
    zh, zl = fsplit(zz, zmax[None, :])
    prod = zz[:, :, None] * zz[:, None, :]
    ph, pl = fsplit(prod.reshape(N, D * D), (zmax[:, None] * zmax[None, :]).reshape(1, D * D))
    one = np.ones((N, 1))
    for name, rem in (("pl*gh (call B build)", gh), ("pl*gs", gs)):
        def contract(fh, fl):
            return gh @ fh + gl @ fh + rem @ fl
        s0 = contract(one, 0 * one)[:, 0]
        s1 = contract(zh, zl)
        s2 = contract(ph, pl).reshape(K, D, D)
        cov, m = cov_from_stats(s0, s1, s2)
        dR = max(np.abs(cov[k] - cov_ref[k]).max() / np.abs(cov_ref[k]).max() for k in range(K))
        print(f"  fixed-point, remainder product {name}: max rel cov err {dR:.2e}  dN {np.abs(s0 / S0 - 1).max():.2e}  dmean {np.abs(m - m_ref).max():.2e}")


print("fixed-point scheme (exact accumulation emulated)")
run_fixed(10000, 4, 8, 20)
run_fixed(100000, 16, 32, 5)
