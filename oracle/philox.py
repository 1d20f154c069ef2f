"""ORACLE (test infrastructure, NOT product code) — numpy restatement of the dropout masks of the DALL-E step.

The reference draws its dropout masks from the TPU's stateful RNG, which cannot be reproduced; parity therefore means
"the reference's math under these masks".  The masks are those of include/dalle_b200.h (D0), restated here from the
published Philox4x32-10 algorithm (Salmon et al., SC'11; Random123):
  key = (lo32(seed), hi32(seed)), counter = (lo32(n), hi32(n), site, step), element reads word w;
  elementwise [rows][cols], row 0 = global row row0:  e = (row0 + r) * cols + c, n = e >> 2, w = e & 3;
  attention (b, h, i, j), b global, S2 = ceil(S / 2):  n = ((b H + h) S2 + i/2) S2 + j/2, w = 2 (i & 1) + (j & 1);
  keep iff word >= floor(rate * 2^32); kept values are scaled by float32(1 / (1 - rate)).
"""
import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)
_SH = np.uint64(32)

SITE_WTE, SITE_WPE = 0, 1


def site_attn(layer):
    return 2 + 3 * layer


def site_attn_out(layer):
    return 3 + 3 * layer


def site_mlp_out(layer):
    return 4 + 3 * layer


def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 of counter words c0..c3 (arrays, broadcast) under key (k0, k1): four uint32 arrays."""
    c = [np.asarray(x, dtype=np.uint64) & _LO for x in (c0, c1, c2, c3)]
    c = list(np.broadcast_arrays(*c))
    k0, k1 = int(k0) & 0xFFFFFFFF, int(k1) & 0xFFFFFFFF
    for r in range(10):
        if r:
            k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
        p0, p1 = _M0 * c[0], _M1 * c[2]
        c = [(p1 >> _SH) ^ c[1] ^ np.uint64(k0), p1 & _LO, (p0 >> _SH) ^ c[3] ^ np.uint64(k1), p0 & _LO]
    return [x.astype(np.uint32) for x in c]


def threshold_scale(rate):
    rate = float(rate)
    if not 0.0 <= rate < 1.0:
        raise ValueError(f"dropout rate {rate} outside [0, 1)")
    return int(rate * 4294967296.0), float(np.float32(1.0 / (1.0 - rate)))


def _words(seed, step, site, n, w):
    seed = int(seed) & (2 ** 64 - 1)
    n = np.asarray(n, dtype=np.uint64)
    out = philox4x32_10(n & _LO, n >> _SH, site, step, seed & 0xFFFFFFFF, seed >> 32)
    return np.choose(np.asarray(w), out)


def keep_elementwise(rate, seed, step, site, rows, cols, row0=0):
    """bool [rows, cols]: keep decisions of an elementwise site whose row 0 is global row row0."""
    thr, _ = threshold_scale(rate)
    e = (np.arange(rows, dtype=np.uint64)[:, None] + np.uint64(row0)) * np.uint64(cols) + \
        np.arange(cols, dtype=np.uint64)[None, :]
    return _words(seed, step, site, e >> np.uint64(2), (e & np.uint64(3)).astype(np.int64)) >= thr


def keep_attention(rate, seed, step, site, B, H, S, row0=0):
    """bool [B, H, S, S]: keep decisions of the attention weights (b, h, query i, key j), b = row0 + local index."""
    thr, _ = threshold_scale(rate)
    S2 = np.uint64((S + 1) // 2)
    b = np.arange(B, dtype=np.uint64)[:, None, None, None] + np.uint64(row0)
    h = np.arange(H, dtype=np.uint64)[None, :, None, None]
    i = np.arange(S, dtype=np.uint64)[None, None, :, None]
    j = np.arange(S, dtype=np.uint64)[None, None, None, :]
    one = np.uint64(1)
    n = ((b * np.uint64(H) + h) * S2 + (i >> one)) * S2 + (j >> one)
    w = (np.uint64(2) * (i & one) + (j & one)).astype(np.int64)
    return _words(seed, step, site, n, np.broadcast_to(w, n.shape)) >= thr
