"""A structured corpus of binary64 bit patterns for the shortest-digits float writer (arrow_to_json's Ryu).

Random bit patterns almost never reach the branches of Ryu that are hard to get right, so the corpus is built from
the cases that do:
  * every biased exponent 0 … 2046 with the mantissas 0, 1, 2, 3, 2^51, 2^52 - 2, 2^52 - 1 and one fixed pattern, in
    both signs: exact powers of two (mantissa 0, where the interval below the value is half as wide: mm_shift == 0),
    the smallest and largest mantissas and every table index and shift of d2d;
  * subnormals of 1 … 5000 ulp (few mantissa bits, the q <= 1 / vr_tz branches);
  * m * 10^e for m in 1 … 999 and e in -330 … 308 with their ±1-ulp neighbours: values whose shortest digits end in
    zeros (vm_tz / vr_tz) and the round-up cases right next to them;
  * the edges of the positional window (scientific exponent -6 / -5 and 9 / 10) and their neighbours;
  * ±0.0, ±inf and NaNs with several payloads in both signs.
"""
from __future__ import annotations

import math
import struct

import numpy as np

MANTISSAS = (0, 1, 2, 3, 1 << 51, (1 << 52) - 2, (1 << 52) - 1, 0x5555555555555)
SIGN = 1 << 63
# the first and last doubles whose scientific exponent is -5 and 9, the doubles just outside, and round numbers there
WINDOW_EDGES = (1e-5, 9.999999999999999e-6, 1e-6, 0.00001000000000000001, 999999999.9999999, 999999999.9999998, 1e9,
                1e10, 9999999999.999998, 9999999999.0, 123456789.0, 1234567890.0, 0.0001234, 0.000012345, 1.5e-5)
NAN_BITS = (0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x7FF4000000000000, 0xFFFFFFFFFFFFFFFF,
            0x7FFFFFFFFFFFFFFF, 0xFFF0000000000001)
SPECIAL_BITS = (0, SIGN, 0x7FF0000000000000, 0xFFF0000000000000) + NAN_BITS


def bits_of(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def f64(bits: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def corpus_bits() -> np.ndarray:
    """The corpus as uint64 bit patterns, each once, in ascending bit order (about 1.7 million values)."""
    out = []
    for e in range(2047):
        for m in MANTISSAS:
            b = (e << 52) | m
            out += [b, b | SIGN]
    out += list(range(1, 5001))
    out += [b | SIGN for b in range(1, 5001, 7)]
    for e in range(-330, 309):
        for m in range(1, 1000):
            x = float(f"{m}e{e}")
            if x == 0.0 or math.isinf(x):
                continue
            b = bits_of(x)
            out += [b - 1, b, b + 1]
    for x in WINDOW_EDGES:
        b = bits_of(x)
        for d in (-2, -1, 0, 1, 2):
            out += [b + d, (b + d) | SIGN]
    out += SPECIAL_BITS
    a = np.unique(np.array(out, np.uint64))
    # b + 1 of the largest finite value is +inf and b - 1 of a tiny value can cross zero: every pattern is still a
    # valid double, so they stay in
    return a


def sample(bits: np.ndarray, n: int, seed: int) -> np.ndarray:
    """A seeded subset of n patterns, the named edges always included."""
    rng = np.random.default_rng(seed)
    pick = rng.choice(len(bits), size=min(n, len(bits)), replace=False)
    must = np.array([bits_of(x) for x in WINDOW_EDGES] + [(e << 52) for e in range(0, 2047, 64)] + [1, 2, 3], np.uint64)
    return np.unique(np.concatenate([bits[np.sort(pick)], must]))
