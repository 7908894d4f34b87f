"""Seeded decimal strings for the number-parsing tests, grouped by the way decimal→double conversion goes wrong.

Every string is a valid JSON number and a valid CSV float.  The reference value of a string is Python's float(),
which is correctly rounded (round to nearest, ties to even).
"""
from __future__ import annotations

import random
import struct

# Named hard cases: the smallest normal, the two sides of the rounding of the smallest subnormal, the overflow
# threshold, 2^53 + 1, signed zeros and exponents far outside the range.
HARD = [
    "2.2250738585072011e-308", "2.2250738585072014e-308", "2.2250738585072009e-308",
    "2.4703282292062327e-324", "2.4703282292062328e-324", "4.9406564584124654e-324", "5e-324",
    "1.7976931348623157e308", "1.7976931348623158e308", "1.7976931348623159e308",
    "9007199254740993", "9007199254740992.5", "9007199254740993.0000000000000000001",
    "-0", "-0.0e5", "0e999999", "-0e-999999", "1e-99999", "1e99999", "-1e99999",
    "0.1", "0.3", "3.246986519402559e+185", "5.400430985016779e-303", "9.40971839401457964e-270",
    "1e23", "8.988465674311579e307", "8.98846567431158e307", "2.2250738585072012e-308",
    "4.4501477170144023e-308", "1.00000000000000011102230246251565404236316680908203125",
    "1.00000000000000011102230246251565404236316680908203124",
    "1.00000000000000011102230246251565404236316680908203126",
    "7.2057594037927933e16", "9223372036854775808", "18446744073709551615", "18446744073709551616",
    "123456789012345678901234567890", "0.30000000000000004", "1e-324", "1e-323", "1e308", "1e309",
]


def f64(bits: int) -> float:
    return struct.unpack("<d", struct.pack("<Q", bits))[0]


def bits_of(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


def _random_bits(rng: random.Random) -> int:
    """A finite, positive binary64 bit pattern: mostly uniform, 5 % subnormal, 5 % near the subnormal boundary."""
    while True:
        r = rng.random()
        if r < 0.05:
            b = rng.getrandbits(52)
        elif r < 0.10:
            b = rng.getrandbits(52) | (rng.randrange(1, 40) << 52)
        else:
            b = rng.getrandbits(63)
        if (b >> 52) != 0x7FF:
            return b


def random_doubles(rng: random.Random, n: int) -> list[float]:
    return [f64(_random_bits(rng) | (rng.getrandbits(1) << 63)) for _ in range(n)]


def _sci(digits: str, e10: int) -> str:
    """int(digits) · 10^e10 in scientific notation."""
    e = e10 + len(digits) - 1
    return (digits[0] + "." + digits[1:] if len(digits) > 1 else digits) + "e" + str(e)


def halfway(bits: int) -> tuple[int, int]:
    """The point halfway between the positive finite double `bits` and the next one up, exactly, as (N, e10) with
    value N · 10^e10.  It has at most 767 significant digits."""
    if bits >> 52:
        m, e = (bits & ((1 << 52) - 1)) | (1 << 52), (bits >> 52) - 1075
    else:
        m, e = bits, -1074
    if e - 1 >= 0:
        return (2 * m + 1) << (e - 1), 0
    return (2 * m + 1) * 5 ** (1 - e), e - 1


def halfway_strings(bits: int) -> list[str]:
    """The exact halfway point, its truncations to 19, 20, 25 and 40 digits, and it nudged one unit up and down in its
    last digit."""
    n, e10 = halfway(bits)
    ds = str(n)
    out = [_sci(ds, e10), _sci(str(n + 1), e10), _sci(str(n - 1), e10)]
    for t in (19, 20, 25, 40):
        if len(ds) > t:
            out.append(_sci(ds[:t], e10 + len(ds) - t))
    return out


def corpus(seed: int = 20240611, per_class: int = 100_000) -> dict[str, list[str]]:
    """{class name: strings}."""
    rng = random.Random(seed)
    c: dict[str, list[str]] = {}
    xs = random_doubles(rng, per_class)
    c["repr"] = [repr(x) for x in xs]
    c["%.17e"] = ["%.17e" % x for x in xs]
    c["%.25e"] = ["%.25e" % x for x in xs]
    c["%.40e"] = ["%.40e" % x for x in xs]
    # integers from 2^53 to past 2^64, written as floats (and as integer literals in a Float64 column)
    ints = [rng.getrandbits(rng.randrange(53, 80)) | (1 << 52) for _ in range(per_class)]
    c["integers"] = [("%d" if i % 2 else "%d.0") % v if i % 3 else "-%d" % v for i, v in enumerate(ints)]
    # <1-19 digits>e<q> over the whole exponent range and past it
    c["digits_e_q"] = ["%de%d" % (rng.randrange(1, 10 ** rng.randrange(1, 20)) , rng.randrange(-360, 330)) for _ in range(per_class)]
    # leading and trailing zeros that the exponent cancels: 0.000…0123e330, 12300000…e-340
    lz = []
    for _ in range(per_class // 5):
        d = str(rng.randrange(1, 10 ** rng.randrange(1, 18)))
        z = rng.randrange(0, 400)
        q = rng.randrange(-330, 300)
        lz.append("0." + "0" * z + d + "e" + str(q + z + 1))
        lz.append(d + "0" * z + "e" + str(q - z))
        lz.append(d + "0" * z + "." + "0" * rng.randrange(1, 30) + "e" + str(q - z))
        lz.append("0." + "0" * z + d + "0" * rng.randrange(0, 400) + "e" + str(q + z + 1))
        lz.append("-0." + "0" * z + d + "e" + str(q + z + 1))
    c["zeros"] = lz
    # exact halfway points: random normals, subnormals, the normal/subnormal boundary, and the exponents whose ties
    # have ≤ 19 digits (2^52 … 2^63, where a tie is an integer or has 1-4 fraction digits)
    hw = []
    for k in range(per_class // 7):
        r = k % 5
        if r == 0:
            b = rng.getrandbits(52)                                       # subnormal
        elif r == 1:
            b = (1 << 52) + rng.randrange(-2000, 2000)                    # around the smallest normal
        elif r == 2:
            b = (rng.randrange(1072, 1087) << 52) | rng.getrandbits(52)   # short ties
        else:
            b = _random_bits(rng)
        b = max(b, 1)
        hw += halfway_strings(b)
        if k % 2:
            hw[-1] = "-" + hw[-1]
    hw += halfway_strings(0x7FEFFFFFFFFFFFFF)  # halfway to 2^1024: the overflow threshold
    hw += halfway_strings(0)[:1]               # 2^-1075: rounds to zero
    c["halfway"] = hw
    c["hard"] = HARD
    return c
