"""CPU checks behind the number-parsing tests: the power-of-ten table the device conversion reads, and the reference
those tests compare with (Python's float(), pinned here to exact rational arithmetic)."""
import math
import os
import random
import re
from fractions import Fraction

import number_corpus as NC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _table():
    text = open(os.path.join(ROOT, "arkflow_b200", "csrc", "pow10_table.h")).read()
    k0 = int(re.search(r"#define ARK_POW10_MIN \((-?\d+)\)", text).group(1))
    k1 = int(re.search(r"#define ARK_POW10_MAX \((-?\d+)\)", text).group(1))

    def array(name):
        body = re.search(name + r"\[\] = \{(.*?)\};", text, re.S).group(1)
        return [int(v.rstrip("ul"), 0) for v in re.findall(r"-?0x[0-9A-Fa-f]+ull|-?\d+", body)]

    return k0, k1, array("kPow10Mant"), array("kPow10Lo"), array("kPow10Exp2")


def test_pow10_table_is_the_truncated_128_bit_mantissa():
    k0, k1, hi, lo, e2 = _table()
    assert (k0, k1) == (-343, 308)
    assert len(hi) == len(lo) == len(e2) == k1 - k0 + 1
    for k in range(k0, k1 + 1):
        i = k - k0
        m = (hi[i] << 64) | lo[i]
        assert 1 << 127 <= m < 1 << 128, k
        scaled = Fraction(10) ** k / Fraction(2) ** (e2[i] - 64)  # 10^k = (m + d) · 2^(e2 − 64), 0 ≤ d < 1
        assert m <= scaled < m + 1, k
        assert (scaled == m) == (0 <= k <= 55), k  # decimal.cuh treats exactly these products as exact


def _exact(s: str) -> float:
    """The correctly rounded double of decimal s, from exact rational arithmetic."""
    f = Fraction(s)
    try:
        v = float(f)
    except OverflowError:
        v = math.inf
    return math.copysign(v, -1.0 if s.lstrip().startswith("-") else 1.0)


def test_named_hard_cases_pin_the_reference():
    for s in NC.HARD:
        assert NC.bits_of(float(s)) == NC.bits_of(_exact(s)), s
    assert float("2.4703282292062327e-324") == 0.0 and float("2.4703282292062328e-324") == 5e-324
    assert float("1.7976931348623158e308") == 1.7976931348623157e308 and float("1.7976931348623159e308") == math.inf
    assert NC.bits_of(float("-0.0e5")) == 1 << 63


def test_halfway_strings_are_exact_and_round_to_even():
    rng = random.Random(3)
    for k in range(3000):
        b = [rng.getrandbits(52), (1 << 52) + rng.randrange(-50, 50), rng.getrandbits(63) % (0x7FF << 52)][k % 3]
        n, e10 = NC.halfway(b)
        x, y = NC.f64(b), NC.f64(b + 1)
        assert Fraction(n) * Fraction(10) ** e10 == (Fraction(x) + Fraction(y)) / 2
        full, up, down = NC.halfway_strings(b)[:3]
        even = x if b % 2 == 0 else y
        assert float(full) == _exact(full) == even
        assert float(up) == _exact(up) == y and float(down) == _exact(down) == x
