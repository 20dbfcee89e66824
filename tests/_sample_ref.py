"""numpy restatement of gmm_sample (include/gmm.h): Philox4x32-10, the component draw, Box-Muller and the reverse Cholesky
factor, so that the GPU's labels can be checked bit for bit and its events against float64 arithmetic."""
import numpy as np

_MASK = np.uint64(0xFFFFFFFF)
_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)


def philox4x32_10(ctr, key):
    """Random123's philox4x32 with 10 rounds.  ctr: uint32 [..., 4]; key: (k0, k1).  Returns uint32 [..., 4]."""
    ctr = np.asarray(ctr, np.uint32).astype(np.uint64)
    c0, c1, c2, c3 = (ctr[..., i] for i in range(4))
    k0, k1 = np.uint64(int(key[0]) & 0xFFFFFFFF), np.uint64(int(key[1]) & 0xFFFFFFFF)
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
        p0, p1 = c0 * _M0, c2 * _M1                       # 32 x 32 -> 64 bits, exact in uint64
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _MASK
    return np.stack([c0, c1, c2, c3], -1).astype(np.uint32)


def words(seed, g, D):
    """The word stream of events g (int array): uint32 [len(g)][4 * blocks], blocks = ceil((2 + 2 ceil(D/2)) / 4)."""
    g = np.asarray(g, np.uint64)
    nblk = (2 + 2 * ((D + 1) // 2) + 3) // 4
    out = np.empty((g.size, 4 * nblk), np.uint32)
    key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    for j in range(nblk):
        ctr = np.zeros((g.size, 4), np.uint32)
        ctr[:, 0] = (g & _MASK).astype(np.uint32)
        ctr[:, 1] = (g >> np.uint64(32)).astype(np.uint32)
        ctr[:, 2] = j
        out[:, 4 * j:4 * j + 4] = philox4x32_10(ctr, key)
    return out


def uniform53(w0, w1):
    """u = ((w0 >> 5) 2^26 + (w1 >> 6)) 2^-53, exactly, in float64."""
    w0, w1 = np.asarray(w0, np.uint64), np.asarray(w1, np.uint64)
    return ((w0 >> np.uint64(5)) * np.uint64(1 << 26) + (w1 >> np.uint64(6))).astype(np.float64) * 2.0 ** -53


def box_muller_args(a, b):
    """The float inputs of the transform: u1 = ((float)a + 0.5f) 2^-32 and x = (float)b 2^-31, both float32."""
    u1 = (np.asarray(a, np.uint32).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -32)
    x = np.asarray(b, np.uint32).astype(np.float32) * np.float32(2.0 ** -31)
    return u1, x


def normals(W, D):
    """float64 z [n][D] from the float inputs of Box-Muller (words 2 + 2p and 3 + 2p)."""
    z = np.empty((W.shape[0], 2 * ((D + 1) // 2)))
    for p in range((D + 1) // 2):
        u1, x = box_muller_args(W[:, 2 + 2 * p], W[:, 3 + 2 * p])
        r = np.sqrt(-2.0 * np.log(u1.astype(np.float64)))
        z[:, 2 * p] = r * np.cos(np.pi * x.astype(np.float64))
        z[:, 2 * p + 1] = r * np.sin(np.pi * x.astype(np.float64))
    return z[:, :D]


def cumulative(pi):
    """C_k: the running sum in double of the float pi, in cluster order."""
    C = np.empty(len(pi))
    s = 0.0
    for k, p in enumerate(np.asarray(pi, np.float32)):
        s += float(p)
        C[k] = s
    return C


def labels_of(pi, W):
    C = cumulative(pi)
    t = uniform53(W[:, 0], W[:, 1]) * C[-1]
    lab = np.searchsorted(C, t, side="right")               # the first k with t < C_k
    klast = int(np.nonzero(np.asarray(pi) > 0)[0][-1])
    return np.where(lab < len(C), lab, klast).astype(np.int32)


def reverse_cholesky(R):
    """R = U U^T, U upper triangular, by host_math.cpp's loop: double from the float R, off-diagonal pairs averaged, pivots
    from the last one up.  Returns float64 U (the device rounds it to float)."""
    R = np.asarray(R, np.float32)
    D = R.shape[0]
    U = np.zeros((D, D))
    for j in range(D - 1, -1, -1):
        d = float(R[j, j])
        for m in range(j + 1, D):
            d -= U[j, m] * U[j, m]
        piv = np.sqrt(d)
        rp = 1.0 / piv
        U[j, j] = piv
        for i in range(j):
            v = 0.5 * (float(R[i, j]) + float(R[j, i]))
            for m in range(j + 1, D):
                v -= U[i, m] * U[j, m]
            U[i, j] = v * rp
    return U


def sample(cl, K, seed, first, n):
    """(x float64 [n][D], labels int32 [n], scale [n][D]) with scale_d = |mu_d| + sum_j |U_dj z_j| (the error bar's unit)."""
    D = cl.D
    W = words(seed, np.arange(first, first + n, dtype=np.uint64), D)
    lab = labels_of(cl.pi[:K], W)
    z = normals(W, D)
    x = np.empty((n, D))
    scale = np.empty((n, D))
    for k in np.unique(lab):
        sel = lab == k
        U = reverse_cholesky(cl.R[k]).astype(np.float32).astype(np.float64)
        mu = cl.means[k].astype(np.float64)
        x[sel] = mu + z[sel] @ U.T
        scale[sel] = np.abs(mu) + np.abs(z[sel]) @ np.abs(U).T
    return x, lab, scale
