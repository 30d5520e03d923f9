"""numpy forms of the two hashes the reference keys groups by (MurmurHash3 x86_32 for HashReduce, the low word
of x64_128 for Sort / Reduce; public-domain algorithm), vectorised over many short keys.  TEST INFRASTRUCTURE:
used to CONSTRUCT colliding dimension rows and to predict which groups merge; pinned against the oracle's
byte-wise C implementation in tests/test_hash_collisions.py."""
from __future__ import annotations

import numpy as np

M32 = np.uint64(0xFFFFFFFF)


def _rotl32(x, r):
    return ((x << np.uint64(r)) | (x >> np.uint64(32 - r))) & M32


def murmur3_32(rows: np.ndarray, seed: int = 0) -> np.ndarray:
    """rows: uint8[n, len] -> uint32[n]."""
    n, ln = rows.shape
    rows = np.ascontiguousarray(rows)
    words = np.ascontiguousarray(rows[:, :ln // 4 * 4]).view("<u4").reshape(n, ln // 4).astype(np.uint64)
    h = np.full(n, seed & 0xFFFFFFFF, np.uint64)
    for i in range(ln // 4):
        k = (words[:, i] * np.uint64(0xcc9e2d51)) & M32
        k = _rotl32(k, 15)
        k = (k * np.uint64(0x1b873593)) & M32
        h ^= k
        h = _rotl32(h, 13)
        h = (h * np.uint64(5) + np.uint64(0xe6546b64)) & M32
    if ln % 4:   # the 1-3 tail bytes, little-endian, without the block's final rotate-multiply-add
        k = np.zeros(n, np.uint64)
        for j in range(ln % 4):
            k |= rows[:, ln // 4 * 4 + j].astype(np.uint64) << np.uint64(8 * j)
        k = (k * np.uint64(0xcc9e2d51)) & M32
        k = _rotl32(k, 15)
        k = (k * np.uint64(0x1b873593)) & M32
        h ^= k
    h ^= np.uint64(ln)
    h ^= h >> np.uint64(16)
    h = (h * np.uint64(0x85ebca6b)) & M32
    h ^= h >> np.uint64(13)
    h = (h * np.uint64(0xc2b2ae35)) & M32
    h ^= h >> np.uint64(16)
    return h.astype(np.uint32)


def _rotl64(x, r):
    return (x << np.uint64(r)) | (x >> np.uint64(64 - r))


def _fmix64(k):
    k = k ^ (k >> np.uint64(33))
    k = k * np.uint64(0xff51afd7ed558ccd)
    k = k ^ (k >> np.uint64(33))
    k = k * np.uint64(0xc4ceb9fe1a85ec53)
    return k ^ (k >> np.uint64(33))


def murmur3_128_lo(rows: np.ndarray) -> np.ndarray:
    """rows: uint8[n, len], 0 < len <= 32 (the largest packed dimension row) -> low 64 bits of
    murmur3_x64_128(seed 0).  16-byte body blocks, then the tail of len % 16 bytes."""
    n, ln = rows.shape
    assert 0 < ln <= 32
    blocks, tail = divmod(ln, 16)
    pad = np.zeros((n, 32), np.uint8)
    pad[:, :ln] = rows
    w = pad.view("<u8").reshape(n, 4)
    c1, c2 = np.uint64(0x87c37b91114253d5), np.uint64(0x4cf5ad432745937f)
    with np.errstate(over="ignore"):
        h1 = np.zeros(n, np.uint64)
        h2 = np.zeros(n, np.uint64)
        for b in range(blocks):
            k1 = _rotl64(w[:, 2 * b] * c1, 31) * c2
            h1 ^= k1
            h1 = _rotl64(h1, 27) + h2
            h1 = h1 * np.uint64(5) + np.uint64(0x52dce729)
            k2 = _rotl64(w[:, 2 * b + 1] * c2, 33) * c1
            h2 ^= k2
            h2 = _rotl64(h2, 31) + h1
            h2 = h2 * np.uint64(5) + np.uint64(0x38495ab5)
        if tail > 8:
            k2 = w[:, 2 * blocks + 1] * c2
            k2 = _rotl64(k2, 33) * c1
            h2 ^= k2
        if tail > 0:
            k1 = w[:, 2 * blocks] * c1
            k1 = _rotl64(k1, 31) * c2
            h1 ^= k1
        h1 ^= np.uint64(ln)
        h2 ^= np.uint64(ln)
        h1 = h1 + h2
        h2 = h2 + h1
        h1 = _fmix64(h1)
        h2 = _fmix64(h2)
        return h1 + h2
