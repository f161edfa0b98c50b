"""TEST INFRASTRUCTURE — numpy restatement of the in-kernel noise of pn_sampler_step (panacea_b200/csrc/sampler.cu):
Philox4x32-10 (Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC'11) keyed by a 64-bit
seed, counter (e / 4 as 64 bits, draw as 64 bits), and Box-Muller in fp64 rounded once to fp32."""
from __future__ import annotations

import numpy as np

M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
W0, W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: uint32 [..., 4]; key: uint32 [..., 2] (broadcast) -> uint32 [..., 4]."""
    c = [np.asarray(ctr[..., i], dtype=np.uint32) for i in range(4)]
    k0 = np.asarray(key[..., 0], dtype=np.uint32)
    k1 = np.asarray(key[..., 1], dtype=np.uint32)
    with np.errstate(over="ignore"):
        for _ in range(10):
            p0 = M0 * c[0].astype(np.uint64)
            p1 = M1 * c[2].astype(np.uint64)
            hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & MASK).astype(np.uint32)
            hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & MASK).astype(np.uint32)
            c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
            k0 = k0 + W0
            k1 = k1 + W1
    return np.stack(c, axis=-1)


def philox_normal(seed: int, draw: int, n: int) -> np.ndarray:
    """The standard normals pn_sampler_step adds for elements 0 .. n-1 of draw `draw` under `seed` (fp32)."""
    e = np.arange(n, dtype=np.uint64)
    blk = e >> np.uint64(2)
    ctr = np.stack([(blk & MASK).astype(np.uint32), (blk >> np.uint64(32)).astype(np.uint32),
                    np.full(n, draw & 0xFFFFFFFF, np.uint32), np.full(n, (draw >> 32) & 0xFFFFFFFF, np.uint32)], -1)
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], dtype=np.uint32)
    w = philox4x32_10(ctr, key)
    pair = ((e >> np.uint64(1)) & np.uint64(1)).astype(bool)
    a = np.where(pair, w[:, 2], w[:, 0]).astype(np.float64)
    b = np.where(pair, w[:, 3], w[:, 1]).astype(np.float64)
    u1 = (a + 1.0) * 2.3283064365386963e-10
    u2 = b * 2.3283064365386963e-10
    r = np.sqrt(-2.0 * np.log(u1))
    th = 6.283185307179586 * u2
    odd = (e & np.uint64(1)).astype(bool)
    return np.where(odd, r * np.sin(th), r * np.cos(th)).astype(np.float32)
