"""The numpy restatement of gmm_sample's random stream (tests/_sample_ref.py, no GPU needed): Philox4x32-10 against the
Random123 known-answer vectors, and the 53-bit and Box-Muller mappings on the edge words 0 and 2^32 - 1."""
import numpy as np
import pytest

import _sample_ref as ref

KAT = [  # (counter, key, result), Random123's kat_vectors for philox4x32 with 10 rounds
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,want", KAT)
def test_philox_known_answers(ctr, key, want):
    got = ref.philox4x32_10(np.array([ctr], np.uint32), key)[0]
    assert [int(v) for v in got] == list(want), [hex(int(v)) for v in got]


def test_word_stream_layout():
    # block j of event g is the counter (lo32(g), hi32(g), j, 0) under the key (lo32(seed), hi32(seed))
    seed, g, D = 0x0123456789ABCDEF, (1 << 32) + 5, 32
    W = ref.words(seed, np.array([g], np.uint64), D)
    assert W.shape == (1, 36)                                   # 2 + 2 * 16 words: 9 blocks
    for j in range(9):
        blk = ref.philox4x32_10(np.array([[5, 1, j, 0]], np.uint32), (0x89ABCDEF, 0x01234567))[0]
        np.testing.assert_array_equal(W[0, 4 * j:4 * j + 4], blk)
    assert ref.words(1, np.arange(3, dtype=np.uint64), 1).shape == (3, 4)   # D = 1: words 0 .. 3, one block


def test_uniform53_edges():
    top = np.uint32(0xFFFFFFFF)
    assert ref.uniform53(0, 0) == 0.0
    assert ref.uniform53(top, top) == 1.0 - 2.0 ** -53         # the largest value, below 1
    assert ref.uniform53(top, 0) == (2.0 ** 27 - 1) * 2.0 ** -27
    assert ref.uniform53(0, top) == (2.0 ** 26 - 1) * 2.0 ** -53


def test_box_muller_edges():
    u1, x = ref.box_muller_args(np.array([0, 0xFFFFFFFF], np.uint32), np.array([0, 0xFFFFFFFF], np.uint32))
    assert u1.dtype == np.float32 and x.dtype == np.float32
    assert u1[0] == np.float32(2.0 ** -33)                     # a = 0: the smallest u1, radius sqrt(66 ln 2) ~ 6.77
    assert u1[1] == np.float32(1.0)                            # a = 2^32 - 1 rounds to 2^32 in float: u1 = 1, radius 0
    assert x[0] == 0.0 and x[1] == np.float32(2.0)             # b = 2^32 - 1 rounds to 2^32: angle 2 pi
    W = np.zeros((2, 4), np.uint32)
    W[1, 2:] = 0xFFFFFFFF
    z = ref.normals(W, 2)
    np.testing.assert_allclose(z[0], [np.sqrt(66 * np.log(2.0)), 0.0], rtol=1e-15)
    np.testing.assert_allclose(z[1], [0.0, 0.0], atol=1e-300)


def test_labels_rules():
    # cumulative weights in double, first k with u T < C_k; a pi = 0 cluster is never drawn
    pi = np.array([0.0, 0.25, 0.0, 0.75, 0.0], np.float32)
    W = np.zeros((4, 4), np.uint32)
    W[1, :2] = 0x20000000, 0                                    # u = 0.125
    W[2, :2] = 0x40000000, 0                                    # u = 0.25 (on the boundary: the next cluster)
    W[3, :2] = 0xFFFFFFFF, 0xFFFFFFFF                           # u just below 1
    lab = ref.labels_of(pi, W)
    np.testing.assert_array_equal(lab, [1, 1, 3, 3])
    assert ref.uniform53(W[2, 0], W[2, 1]) == 0.25
