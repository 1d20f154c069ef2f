"""CPU side of the ABI-limit tests (test_abi_limits_gpu.py): oracle/philox.py against a pure-Python-int restatement of
Philox4x32-10 at counters whose high word hi32(n) is not 0, so that the oracle's uint64 handling of the high word is
right before the GPU masks are compared to it.  The row0 values are those of the GPU module's dropout cases."""
import numpy as np
import pytest

from oracle import guidance as CG
from oracle import philox as X

M32 = 0xFFFFFFFF


def philox_int(c, k0, k1):
    """Philox4x32-10 (Salmon et al., SC'11) on Python ints: counter words c[0..3], key (k0, k1)."""
    c0, c1, c2, c3 = c
    for r in range(10):
        if r:
            k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & M32, (p0 >> 32) ^ c3 ^ k1, p0 & M32
    return c0, c1, c2, c3


def keep_int(rate, seed, step, site, e):
    """Keep decision of element e (block e >> 2, word e & 3) of a site, from philox_int."""
    words = philox_int((e >> 2 & M32, e >> 2 >> 32, site & M32, step & M32), seed & M32, seed >> 32 & M32)
    return words[e & 3] >= int(rate * 4294967296.0)


def test_philox_int_matches_the_known_answer_vectors():
    assert philox_int((0, 0, 0, 0), 0, 0) == (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)
    assert philox_int((M32,) * 4, M32, M32) == (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)


@pytest.mark.parametrize("n", [2 ** 32 - 1, 2 ** 32, 2 ** 32 + 1, 2 ** 33 + 12345, 2 ** 40 + 7, 2 ** 62 + 3,
                               2 ** 64 - 1])
def test_oracle_philox_equals_the_int_restatement_above_2_32(n):
    for site, step, seed in ((4, 3, 9), (X.site_attn(5), 2 ** 31 + 1, 2 ** 40 + 3), (CG.SITE_CAPTION, 17, 2 ** 64 - 1)):
        want = philox_int((n & M32, n >> 32, site, step), seed & M32, seed >> 32)
        got = X.philox4x32_10(np.uint64(n & M32), np.uint64(n >> 32), site, step, seed & M32, seed >> 32)
        assert tuple(int(w) for w in got) == want, (n, site)


def test_elementwise_mask_across_hi32_equals_the_int_restatement():
    """cols = 512, row0 = 2^25 - 3, 8 rows: n = e >> 2 crosses 2^32 at local row 3."""
    rows, cols, row0 = 8, 512, 2 ** 25 - 3
    got = X.keep_elementwise(0.1, 9, 4, X.site_mlp_out(0), rows, cols, row0)
    e0 = row0 * cols
    assert (e0 >> 2) < 2 ** 32 <= (e0 + rows * cols - 1) >> 2
    want = np.array([[keep_int(0.1, 9, 4, X.site_mlp_out(0), e0 + r * cols + c) for c in range(cols)]
                     for r in range(rows)])
    assert np.array_equal(got, want)


def test_attention_mask_across_hi32_equals_the_int_restatement():
    """H = 32, S = 1280, row0 = 327: n crosses 2^32 inside head 21 of sequence 327.  The whole of head 21 and the first
    and last key blocks of heads 20 and 22 are restated."""
    H, S, row0, rate, seed, step, site = 32, 1280, 327, 0.1, 5, 11, X.site_attn(0)
    S2 = (S + 1) // 2
    n = lambda h, i, j: ((row0 * H + h) * S2 + i // 2) * S2 + j // 2
    assert n(21, 0, 0) < 2 ** 32 <= n(21, S - 1, S - 1) and n(20, S - 1, S - 1) < 2 ** 32 <= n(22, 0, 0)
    got = X.keep_attention(rate, seed, step, site, 1, H, S, row0)[0]
    thr = int(rate * 4294967296.0)
    for h, qs in ((21, range(S)), (20, (0, 1, S - 2, S - 1)), (22, (0, 1, S - 2, S - 1))):
        for i in qs:
            words = [philox_int((n(h, i, j) & M32, n(h, i, j) >> 32, site, step), seed, 0) for j in range(0, S, 2)]
            want = np.array([words[j // 2][2 * (i & 1) + (j & 1)] >= thr for j in range(S)])
            assert np.array_equal(got[h, i], want), (h, i)


def test_caption_decisions_across_hi32_equal_the_int_restatement():
    """row0 = 2^34 - 5, B = 10: the block index e >> 2 crosses 2^32 at sequence 5."""
    rate, seed, step, row0, B = 0.5, 2 ** 40 + 3, 17, 2 ** 34 - 5, 10
    got = CG.caption_dropped(rate, seed, step, B, row0)
    want = np.array([not keep_int(rate, seed, step, CG.SITE_CAPTION, row0 + b) for b in range(B)])
    assert np.array_equal(got, want)
    assert 0 < int(got.sum()) < B
