"""The Float64 text of arrow_to_json, on the CPU: the oracle's `_lexical_f64` (built on Python's repr) and
`scripts/gen_ryu_tables.fmt_lexical` (the line-by-line Python model of the device's Ryu) agree on the structured corpus
of tests/f64_corpus.py, and an independent check with exact rational arithmetic pins both to correctly rounded
shortest output: the text parses back to the same double, no text with one digit fewer does, and the digits are the
closest to the value among the texts of their length that parse back to it."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle.json_oracle import _lexical_f64
from scripts import gen_ryu_tables as ryu
from f64_corpus import WINDOW_EDGES, corpus_bits, f64, sample


@pytest.fixture(scope="module")
def corpus():
    return corpus_bits()


def _digits(text: str) -> tuple[int, int]:
    """(digits, e10) of a finite `_lexical_f64` text with the sign dropped: value = digits * 10^e10, digits without
    trailing zeros."""
    t = text.lstrip("-")
    mant, _, ex = t.partition("e")
    ip, _, fp = mant.partition(".")
    ds = (ip + fp).lstrip("0") or "0"
    e10 = (int(ex) if ex else 0) - len(fp)
    stripped = ds.rstrip("0")
    return int(stripped), e10 + len(ds) - len(stripped)


def _reads_as(q: Fraction, x: float) -> bool:
    try:
        return float(q) == x
    except OverflowError:  # past the largest double: reads as inf
        return False


def test_corpus_reaches_the_hard_branches(corpus):
    # exact powers of two in every binade, subnormals down to one ulp, and the corpus size the GPU test relies on
    assert len(corpus) > 1_500_000
    have = set(corpus.tolist())
    assert all((e << 52) in have for e in range(1, 2047))
    assert all(b in have for b in range(1, 5001))
    assert all(np.uint64(int(np.float64(x).view(np.uint64))) in corpus for x in WINDOW_EDGES)


def test_oracle_and_ryu_model_agree_on_the_corpus(corpus):
    bad = []
    for b in corpus.tolist():
        x = f64(b)
        want = _lexical_f64(x)
        if math.isnan(x) or math.isinf(x):
            assert want == "null"
            continue
        got = ryu.fmt_lexical(x)
        if got != want:
            bad.append((hex(b), got, want))
    assert not bad, bad[:10]


def test_positional_window_edges():
    # scientific exponent -5 and 9 are positional, -6 and 10 are not
    assert _lexical_f64(1e-5) == "0.00001"
    assert _lexical_f64(9.999999999999999e-6) == "9.999999999999999e-6"
    assert _lexical_f64(999999999.9999999) == "999999999.9999999"
    assert _lexical_f64(1e9) == "1000000000.0"
    assert _lexical_f64(1e10) == "1.0e10"
    assert _lexical_f64(-0.0) == "-0.0" and _lexical_f64(5e-324) == "5.0e-324"
    for x in (1e-5, 9.999999999999999e-6, 999999999.9999999, 1e9, 1e10, 5e-324, 2.0 ** -1074 * 3, 2.0 ** 1023):
        assert ryu.fmt_lexical(x) == _lexical_f64(x)


def test_shortest_and_correctly_rounded_by_exact_arithmetic(corpus):
    subset = sample(corpus, 100_000, seed=20261017)
    checked = 0
    for b in subset.tolist():
        x = f64(b)
        if math.isnan(x) or math.isinf(x) or x == 0.0:
            continue
        text = _lexical_f64(x)
        assert float(text) == x, (hex(b), text)
        d, e10 = _digits(text)
        nd = len(str(d))
        fx = Fraction(abs(x))
        unit = Fraction(10) ** e10
        # the closest text of nd digits that reads back as x: the grid point nearest x is d, or (below an exact power of
        # two, where the interval under x is half as wide) it does not read back as x and d is the next one over
        near = round(fx / unit)
        if near != d:
            assert abs(near - d) == 1 and not _reads_as(near * unit, abs(x)), (hex(b), text)
        if nd > 1:
            # no text of nd - 1 digits reads back as x: neither neighbour of x on the grid 10^(e10 + 1), nor the largest
            # (nd - 1)-digit number below 10^sci
            coarse = unit * 10
            lo = math.floor(fx / coarse)
            sci = e10 + nd - 1
            for cand in (lo * coarse, (lo + 1) * coarse, (10 ** (nd - 1) - 1) * Fraction(10) ** (sci - nd + 1)):
                assert not _reads_as(cand, abs(x)), (hex(b), text, cand)
        checked += 1
    assert checked > 95_000
