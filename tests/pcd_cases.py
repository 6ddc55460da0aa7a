"""Crafted PointXYZRGBICT clouds and float bit patterns for the PCD writer's tests (DESIGN.md f13).

cloud(name) -> (n, 8) uint32 array of 32-byte records (word 3 = w, never written; word 4 = the bgra colour).
The bit-pattern sets of the formatter's structured check: every exponent's first and last mantissas, every exact tie at
the 9th significant digit, decade and %g style boundaries, and the special values."""
from __future__ import annotations

import numpy as np

F32_MAX = 0x7F7FFFFF


def f2u(x):
    return np.asarray(x, np.float32).view(np.uint32)


def specials():
    """+-0, +-inf, NaNs of both signs (quiet, signalling, every payload class), subnormals, FLT_MAX, FLT_MIN"""
    s = [0x00000000, 0x80000000, 0x7F800000, 0xFF800000,
         0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001, 0x7FBFFFFF, 0xFFFFFFFF, 0x7FC00001, 0x7FFFFFFF, 0xFFA5A5A5,
         0x00000001, 0x80000001, 0x00000002, 0x007FFFFF, 0x807FFFFF, 0x00400000, 0x00000100, 0x000F4240,
         F32_MAX, F32_MAX | 0x80000000, 0x00800000, 0x80800000, 0x3F800000, 0xBF800000]
    return np.array(s, np.uint32)


def exponent_edges(k=16):
    """every biased exponent with its first and last k mantissas, both signs"""
    man = np.concatenate([np.arange(k), 0x7FFFFF - np.arange(k)]).astype(np.uint32)
    ex = np.arange(256, dtype=np.uint32)
    b = (ex[:, None] << 23 | man[None, :]).ravel()
    return np.concatenate([b, b | 0x80000000]).astype(np.uint32)


def ties():
    """every float whose exact decimal value has 9 significant digits ending in 5 (a round-half-even tie at 8 digits).
    Such a value is N 10^q with N = 10 d + 5 < 10^9.  For q >= 0 it is an odd multiple of 2^q above 2^24, never a float;
    for q < 0 it is M 2^q with M = N / 5^-q, so 5^-q divides N, q >= -12, and M is odd and below 2^24.  Positive only
    (the sign does not take part in the rounding); the structured check adds a sample of negatives."""
    out = []
    for q in range(-12, 0):
        p5 = 5 ** (-q)
        lo, hi = -(-10 ** 8 // p5), (10 ** 9 - 1) // p5
        hi = min(hi, (1 << 24) - 1)
        if lo > hi:
            continue
        M = np.arange(lo | 1, hi + 1, 2, dtype=np.int64)
        out.append(np.ldexp(M.astype(np.float64), q).astype(np.float32).view(np.uint32))
    return np.concatenate(out).astype(np.uint32)


def boundaries(k=4):
    """the k floats on either side of each power of ten, of each value that rounds up into the next decade at 8 digits
    (9.99999995 10^j), and of 10^-4 / 10^8 (where %g switches style), both signs"""
    centres = []
    for j in range(-46, 40):
        centres += [10.0 ** j, 9.99999995 * 10.0 ** (j - 1), 9.9999999 * 10.0 ** (j - 1)]
    c = np.array(centres, np.float64)
    c = c[(c < 3.5e38) & (c > 1e-46)]
    base = c.astype(np.float32).view(np.uint32).astype(np.int64)
    off = np.arange(-k, k + 1)
    b = (base[:, None] + off[None, :]).ravel()
    b = b[(b >= 0) & (b <= F32_MAX)].astype(np.uint32)
    return np.concatenate([b, b | 0x80000000]).astype(np.uint32)


def records(words):
    """records with the given bit patterns in the seven written words (row-major), w = 0x3F800000"""
    w = np.asarray(words, np.uint32).ravel()
    n = -(-w.size // 7)
    flat = np.zeros(n * 7, np.uint32)
    flat[:w.size] = w
    flat = flat.reshape(n, 7)
    r = np.zeros((n, 8), np.uint32)
    r[:, [0, 1, 2, 4, 6, 5, 7]] = flat
    r[:, 3] = 0x3F800000
    return r


def harvest_like(n, seed=0):
    """records like the map's harvests: positions of a 0.1 m grid tens of metres out, heights, variances, colours with
    a = 0xff, intensities, traversabilities, and a few empty-cell sentinels"""
    rng = np.random.default_rng(seed)
    r = np.zeros((n, 8), np.float32)
    r[:, 0] = (rng.integers(-600, 600, n) * 0.1 + 0.05).astype(np.float32)
    r[:, 1] = (rng.integers(-600, 600, n) * 0.1 + 0.05).astype(np.float32)
    r[:, 2] = rng.normal(0.0, 0.8, n).astype(np.float32)
    r[:, 3] = 1.0
    col = rng.integers(0, 1 << 24, n, dtype=np.uint32) | np.uint32(0xFF000000)
    u = r.view(np.uint32)
    u[:, 4] = col
    r[:, 5] = rng.uniform(0.0, 0.05, n).astype(np.float32)
    r[:, 6] = rng.uniform(0.0, 255.0, n).astype(np.float32)
    r[:, 7] = rng.uniform(0.0, 1.0, n).astype(np.float32)
    r[rng.random(n) < 0.01, 7] = -10.0
    return u.copy()


CASES = {
    "one": lambda: harvest_like(1, 1),
    "specials": lambda: records(specials()),
    "exponent_edges": lambda: records(exponent_edges(4)),
    "boundaries": lambda: records(boundaries(2)),
    "ties": lambda: records(ties()[::997]),
    "colours": lambda: records(np.stack([np.arange(0, 1 << 24, 4099, dtype=np.uint32) | 0xFF000000] * 7, axis=1).ravel()),
    "random_bits": lambda: records(np.random.default_rng(5).integers(0, 1 << 32, 7 * 3001, dtype=np.uint64).astype(np.uint32)),
    "harvest_like": lambda: harvest_like(5000, 2),
    "odd_tail": lambda: harvest_like(257, 3),
}


def case_names():
    return list(CASES)


def cloud(name):
    return CASES[name]()
