"""numpy restatement of the per-edge dropout mask of GatedMessagePassingLayer (ptgnn_b200/csrc/edge_dropout.cuh).

Element (e, k) of the [E, K] mask: u = word k % 4 of Philox4x32-10(counter = (e, k // 4, 0, 0), key = (key0, key1)); kept iff
u >= round(p 2^32); a kept element is scaled by 1 / (1 - p).
"""
import numpy as np

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
_LOW = np.uint64(0xFFFFFFFF)


def philox4x32_10(counter, key):
    """counter: uint32 [..., 4], key: uint32 [2] (or [..., 2]) -> uint32 [..., 4] (Random123's philox4x32 with 10 rounds)."""
    c = np.array(counter, dtype=np.uint32)
    k = np.array(key, dtype=np.uint32)
    c0, c1, c2, c3 = (c[..., i].astype(np.uint64) for i in range(4))
    k0, k1 = k[..., 0].astype(np.uint64), k[..., 1].astype(np.uint64)
    for r in range(10):
        if r > 0:
            k0 = (k0 + _W0) & _LOW
            k1 = (k1 + _W1) & _LOW
        p0, p1 = _M0 * c0, _M1 * c2
        hi0, lo0 = p0 >> np.uint64(32), p0 & _LOW
        hi1, lo1 = p1 >> np.uint64(32), p1 & _LOW
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def threshold(p: float) -> int:
    """round(p 2^32); 2^32 (nothing kept) for p = 1."""
    if p <= 0:
        return 0
    if p >= 1:
        return 1 << 32
    return int(round(p * 2.0 ** 32))


def keep_mask(key, num_edges: int, K: int, p: float) -> np.ndarray:
    """bool [num_edges, K]: element (e, k) kept."""
    e = np.repeat(np.arange(num_edges, dtype=np.uint32), K // 4)
    q = np.tile(np.arange(K // 4, dtype=np.uint32), num_edges)
    ctr = np.stack([e, q, np.zeros_like(e), np.zeros_like(e)], axis=-1)
    u = philox4x32_10(ctr, np.asarray(key, dtype=np.uint32)).reshape(num_edges, K)
    return u.astype(np.uint64) >= np.uint64(threshold(p))


def keep_bits(mask: np.ndarray) -> np.ndarray:
    """bool [E, K] -> int32 [E, K / 32] words, bit k % 32 of word k / 32 set for a kept element."""
    E, K = mask.shape
    w = mask.reshape(E, K // 32, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)
    return w.sum(axis=-1).astype(np.uint32).view(np.int32)


def scale(p: float) -> float:
    return 1.0 / (1.0 - p) if p < 1 else 0.0
