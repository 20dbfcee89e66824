"""The split tensor E-step (`estep_tc_kernel`, D = 16 and 24) deep in its ring of logit slots (run with -m gpu on an H100).

launch_estep_d() runs grid = min(SMs, ceil(n / 128)) CTAs over 64-event tiles; tile i of a CTA is grid tile
2 b + i % 2 + (i / 2) 2 grid, and it goes through slot i % 3, use u = i / 3, barrier 2 s + (u & 1), wait parity
(u >> 1) & 1 (ring_depth below restates this and every case asserts the depth it claims).  A slot-ring fault shows only
where slots are reused at both wait parities, i.e. at several hundred thousand events, so the deep cases run 48+ tiles
on every CTA, with the last partial tile placed on each slot and each warpgroup, at every resident supergroup count and
at 2 and 3 passes of 64 clusters (modes 1, 2, 3).  D = 8 (the fused schedule) is a control.

Identities (exact unless stated):
  1. position invariance: gmm_score_stats' memberships of the rolled and the sliced events, in one chunk, are the rolled
     and sliced memberships of the resident E-step (same engine, so the same centre and scale);
  2. the shallow ring: chunks of 128 SMs events (at most 2 tiles per CTA, no slot reused), and chunks of one tile, give
     the deep run's memberships;
  3. gmm_score's max_resp is the top membership bit for bit at every K, its label the arg-max
     wherever the top two differ;
  4. the log-likelihood of gmm_estep (float32) is within 1 float32 ulp of float32(sum_e float64(logp_e)), logp from
     gmm_score (the same denominators);
  5. weighted events: memberships bit-identical to the unweighted run, log-likelihood sum_e w_e logp_e as in 4.
And every responsibility of the deep D = 16 / 24 shapes (first and last tiles of every CTA and a random 10 % of the
events), and every gmm_score logp, is held to the bar of tests/test_estep_error_model.py against its exact emulation
of the kernel's operands."""
import numpy as np
import pytest

from test_estep_error_model import ERR_K, KINDS, N_DATA, Emulation, blobs, param_set, standardise
from test_gpu_mstep_tc import n_sms
from test_gpu_score import check_shard, mixture

pytestmark = pytest.mark.gpu

TILE = 64


# ---- launch arithmetic -------------------------------------------------------------------------------------------------
def ring_depth(n, sms):
    """launch_estep_d()'s grid and tiles: per CTA the tiles it runs, the (slot, use parity, wait parity) triples that
    occur, and the (slot, warpgroup) of the last tile when it is partial."""
    grid = max(1, min(sms, -(-n // 128)))
    ntiles = -(-n // TILE)
    stride = 2 * grid
    counts, triples = [], set()
    for b in range(grid):
        c = 0
        for h in range(2):
            q = 0
            while 2 * b + h + q * stride < ntiles:
                i = 2 * q + h
                u = i // 3
                triples.add((i % 3, u & 1, (u >> 1) & 1))
                c += 1
                q += 1
        counts.append(c)
    last = None
    if n % TILE:
        T = ntiles - 1
        h, q = T % 2, T // stride
        last = ((2 * q + h) % 3, h)
    return dict(grid=grid, ntiles=ntiles, min_tiles=min(counts), max_tiles=max(counts), triples=triples, last=last)


ALL_TRIPLES = {(s, up, wp) for s in range(3) for up in range(2) for wp in range(2)}


def deep_n(sms, slot, wg, rem=37):
    """At least 48 tiles on every CTA, and a last partial tile (rem events) on the given slot and warpgroup."""
    nt = 48 * sms
    while True:
        n = TILE * (nt - 1) + rem
        if ring_depth(n, sms)["last"] == (slot, wg):
            return n
        nt += 1


def check_deep(n, sms, slot, wg):
    rd = ring_depth(n, sms)
    assert rd["grid"] == sms and rd["min_tiles"] >= 24 and rd["triples"] == ALL_TRIPLES and rd["last"] == (slot, wg), rd
    return rd


# ---- helpers -----------------------------------------------------------------------------------------------------------
def engine(pkg, ev, Kmax):
    eng = pkg.Engine(ev, Kmax)
    eng.set_option("estep_path", pkg.PATH_TENSOR)
    return eng


def resident(eng, K, cl):
    eng.set_clusters(K, cl)
    ll = eng.estep(K)
    return ll, eng.get_clusters(K, with_memberships=True).memberships[:K].copy()


def score_memberships(eng, K, x, chunk):
    eng.set_option("score_chunk", chunk)
    return eng.score_stats(K, x, stats=False, memberships=True)[2]


def assert_ll_ulp(ll, terms, what):
    """gmm_estep's float32 log-likelihood within 1 ulp of float32(sum of the float64 terms)."""
    ref = np.float32(np.sum(np.asarray(terms, np.float64)))
    assert abs(np.float64(np.float32(ll)) - np.float64(ref)) <= np.spacing(np.abs(ref)), (what, ll, float(ref))


def data(D, n):
    return np.ascontiguousarray(blobs(D)[:n])


SUPERGROUP_K = (1, 16, 17, 33, 49, 64)
PASS_K = (65, 128, 129, 209)
LANDINGS = [(s, w) for s in range(3) for w in range(2)]
DEEP = [(D, K) for D in (16, 24) for K in SUPERGROUP_K + PASS_K] + [(8, 17), (8, 129)]


# ---- A. identities deep in the ring -------------------------------------------------------------------------------------
@pytest.mark.parametrize("D,K", DEEP)
def test_deep_ring_identities(pkg, D, K):
    sms = n_sms()
    slot, wg = LANDINGS[DEEP.index((D, K)) % len(LANDINGS)]
    n = deep_n(sms, slot, wg)
    rd = check_deep(n, sms, slot, wg)
    print(f"\n[estep-tc] D={D} K={K} n={n}: grid {rd['grid']}, {rd['min_tiles']}..{rd['max_tiles']} tiles per CTA, "
          f"{len(rd['triples'])} (slot, use parity, wait parity) triples, last tile on slot {slot} warpgroup {wg}")
    ev = data(D, n)
    with engine(pkg, ev, K) as eng:
        ll, memb = resident(eng, K, mixture(pkg, ev, K))
        # 3. cross-kernel, 4. log-likelihood accounting
        lab, mr, lp = check_shard(eng, K, ev, ll)
        assert_ll_ulp(ll, lp, "estep vs score")
        # 1. position invariance, one chunk
        eng.score_stats_profile(reset=True)
        shifts = (1, 8, 37, 64, 3 * 64, 2 * 64 * sms + 5)
        for r in shifts:
            got = score_memberships(eng, K, np.roll(ev, r, axis=0), n)
            np.testing.assert_array_equal(got, np.roll(memb, r, axis=1), err_msg=f"roll {r}")
            got = score_memberships(eng, K, ev[r:], n)
            np.testing.assert_array_equal(got, memb[:, r:], err_msg=f"slice {r}")
        prof = eng.score_stats_profile()
        assert prof["estep_tensor_chunks"] == 2 * len(shifts) and prof["estep_simt_chunks"] == 0, prof
        # 2. the shallow ring: at most 2 tiles per CTA and launch
        chunk = 128 * sms
        assert ring_depth(chunk, sms)["max_tiles"] == 2
        np.testing.assert_array_equal(score_memberships(eng, K, ev, chunk), memb, err_msg="chunks of 128 SMs events")


@pytest.mark.parametrize("D", [8, 16, 24])
@pytest.mark.parametrize("K", [17, 129])
def test_small_shapes_and_one_tile_launches(pkg, D, K):
    """Fewer CTAs than SMs, a last CTA whose second warpgroup pair gets no tile, single events and partial tiles: the
    resident E-step equals chunks of one tile per launch, the rolled events and gmm_score."""
    sms = n_sms()
    cases = {"1": 1, "63": 63, "65": 65, "lone-wg0": 128 * 49 + 30, "grid<sms": 128 * (sms - 9) - 5}
    ev_all = data(D, 20_000)
    cl = mixture(pkg, ev_all, K)
    for name, n in cases.items():
        rd = ring_depth(n, sms)
        if name == "lone-wg0":
            assert rd["ntiles"] % 2 == 1 and rd["grid"] == rd["ntiles"] // 2 + 1 < sms, rd
        if name == "grid<sms":
            assert rd["grid"] < sms and rd["max_tiles"] == 2, rd
        ev = np.ascontiguousarray(ev_all[:n])
        with engine(pkg, ev, K) as eng:
            ll, memb = resident(eng, K, cl)
            lab, mr, lp = check_shard(eng, K, ev, ll)
            assert_ll_ulp(ll, lp, name)
            np.testing.assert_array_equal(score_memberships(eng, K, ev, TILE), memb, err_msg=f"{name}: one tile per launch")
            r = min(37, n - 1)
            np.testing.assert_array_equal(score_memberships(eng, K, np.roll(ev, r, axis=0), max(n, 1)), np.roll(memb, r, axis=1),
                                          err_msg=f"{name}: roll")


@pytest.mark.parametrize("D,K", [(16, 64), (24, 17), (24, 129)])
def test_one_tile_launches_deep_ring_reference(pkg, D, K):
    """Chunks of one tile (a single MMA warpgroup, slot 0, use 0) against the resident run on 40 000 events (5 tiles
    per CTA: slots reused at wait parity 0)."""
    sms = n_sms()
    n = 40_001
    rd = ring_depth(n, sms)
    assert rd["max_tiles"] >= 4
    ev = data(D, n)
    with engine(pkg, ev, K) as eng:
        ll, memb = resident(eng, K, mixture(pkg, ev, K))
        np.testing.assert_array_equal(score_memberships(eng, K, ev, TILE), memb)


@pytest.mark.parametrize("D,K", [(16, 17), (16, 64), (24, 64), (24, 129)])
def test_weighted_deep(pkg, D, K):
    """estep_tc_kernel<D, NSG, true>: non-constant weights with exact zeros change the log-likelihood only."""
    sms = n_sms()
    slot, wg = LANDINGS[(D + K) % len(LANDINGS)]
    n = deep_n(sms, slot, wg)
    check_deep(n, sms, slot, wg)
    ev = data(D, n)
    rng = np.random.default_rng(D * 1000 + K)
    w = rng.uniform(0.0, 3.0, n).astype(np.float32)
    w[rng.random(n) < 0.05] = 0.0
    with engine(pkg, ev, K) as eng:
        cl = mixture(pkg, ev, K)
        ll, memb = resident(eng, K, cl)
        lp = eng.score(K, ev)[2]
        eng.set_weights(w)
        llw, membw = resident(eng, K, cl)
        np.testing.assert_array_equal(membw, memb)
        assert_ll_ulp(llw, w.astype(np.float64) * lp.astype(np.float64), "weighted")
        assert_ll_ulp(ll, lp, "unweighted")


# ---- B. every responsibility against the exact emulation of the operands -------------------------------------------------
def emulated_events(n, sms, rng):
    """The first and last tile of each warpgroup of every CTA, and a random 10 % of the events."""
    rd = ring_depth(n, sms)
    g, nt = rd["grid"], rd["ntiles"]
    tiles = set()
    for b in range(g):
        for h in range(2):
            ts = list(range(2 * b + h, nt, 2 * g))
            if ts:
                tiles.update((ts[0], ts[-1]))
    idx = np.concatenate([np.arange(t * TILE, min(n, t * TILE + TILE)) for t in sorted(tiles)] + [rng.choice(n, n // 10, replace=False)])
    return np.unique(idx)


@pytest.mark.parametrize("K", ERR_K)
@pytest.mark.parametrize("D", [16, 24])
@pytest.mark.parametrize("kind", KINDS)
def test_deep_against_emulation(pkg, oracle64, kind, D, K):
    sms = n_sms()
    slot, wg = LANDINGS[(KINDS.index(kind) + D + K) % len(LANDINGS)]
    n = deep_n(sms, slot, wg)
    check_deep(n, sms, slot, wg)
    ev_all = blobs(D)
    assert n <= N_DATA
    ev = np.ascontiguousarray(ev_all[:n])
    cl = param_set(pkg, oracle64, kind, D, K, ev_all)
    with engine(pkg, ev, K) as eng:
        ll, memb = resident(eng, K, cl)
        held = eng.get_clusters(K)
        lp = eng.score(K, ev)[2]
        shift = eng.score_stats(K, ev[:1], stats=False, memberships=True)[1]
    assert_ll_ulp(ll, lp, "estep vs score")
    scale = standardise(ev)[1]
    idx = emulated_events(n, sms, np.random.default_rng(D + K))
    worst = worst_lp = 0.0
    for s in range(0, len(idx), 4096):
        sel = idx[s:s + 4096]
        em = Emulation(held, K, ev[sel], shift, scale)
        worst = max(worst, em.ratio(memb[:, sel]))
        worst_lp = max(worst_lp, em.lse_ratio(lp[sel]))
    print(f"\n[estep-tc emulation] {kind} D={D} K={K} n={n}, {len(idx)} events: responsibilities worst/bar {worst:.3g}, "
          f"logp worst/bar {worst_lp:.3g}")
    assert worst <= 1.0 and worst_lp <= 1.0, (worst, worst_lp)
