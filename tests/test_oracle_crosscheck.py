"""The oracle against a second, independent CPU implementation — Arrow C++ (pyarrow.compute / Acero) — on the part of
the SQL subset where DataFusion's and Arrow C++'s semantics coincide (Int64 arithmetic without overflow, Int64 /
Utf8 comparisons, inner equi-join, SUM / COUNT / MIN / MAX / AVG over Int64).  This does not pin the oracle to the
reference (only the reference's own assertions do, tests/golden/), but it catches slips in the restatement."""
import math

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from oracle.sql_oracle import sql_join, sql_process


def batch(seed, n=5000, keys=37, nulls=True):
    rng = np.random.default_rng(seed)
    v = rng.integers(-50, 50, n)
    w = rng.integers(0, 1000, n)
    k = rng.integers(0, keys, n)
    vm = rng.random(n) < 0.07 if nulls else np.zeros(n, bool)
    km = rng.random(n) < 0.03 if nulls else np.zeros(n, bool)
    return pa.record_batch({"v": pa.array(v, pa.int64(), mask=vm), "w": pa.array(w, pa.int64()),
                            "k": pa.array([f"key_{i:03d}" for i in k], pa.utf8(), mask=km)})


@pytest.mark.parametrize("seed", range(4))
def test_filter_project_matches_arrow_compute(seed):
    rb = batch(seed)
    t = pa.Table.from_batches([rb])
    cases = [
        ("SELECT v, w FROM flow WHERE v >= 10", pc.greater_equal(t["v"], 10)),
        ("SELECT v, w FROM flow WHERE v < 0 AND w > 500", pc.and_kleene(pc.less(t["v"], 0), pc.greater(t["w"], 500))),
        ("SELECT v, w FROM flow WHERE v = 7 OR k = 'key_003'", pc.or_kleene(pc.equal(t["v"], 7), pc.equal(t["k"], "key_003"))),
        ("SELECT v, w FROM flow WHERE k > 'key_020' AND v IS NOT NULL", pc.and_kleene(pc.greater(t["k"], "key_020"), pc.is_valid(t["v"]))),
        ("SELECT v, w FROM flow WHERE NOT (v > 3)", pc.invert(pc.greater(t["v"], 3))),
    ]
    for q, mask in cases:
        want = t.filter(mask).select(["v", "w"]).combine_chunks()  # filter drops NULL predicates, like SQL WHERE
        got = sql_process(rb, q)
        assert got.num_rows == want.num_rows, q
        assert got.column("v").equals(want["v"].combine_chunks() if want.num_rows else pa.array([], pa.int64())), q
        assert got.column("w").to_pylist() == want["w"].to_pylist(), q
    got = sql_process(rb, "SELECT v + w AS s, v * 3 - 1 AS m FROM flow")
    assert got.column("s").to_pylist() == pc.add(t["v"], t["w"]).to_pylist()
    assert got.column("m").to_pylist() == pc.subtract(pc.multiply(t["v"], 3), 1).to_pylist()


@pytest.mark.parametrize("seed", range(4))
def test_group_by_matches_acero(seed):
    rb = batch(10 + seed)
    t = pa.Table.from_batches([rb])
    want = t.group_by("k").aggregate([("v", "sum"), ("v", "count"), ("v", "min"), ("v", "max"), ("v", "mean"), ([], "count_all")])
    got = sql_process(rb, "SELECT k, SUM(v), COUNT(v), MIN(v), MAX(v), AVG(v), COUNT(*) FROM flow GROUP BY k")
    assert got.num_rows == want.num_rows

    def rows(tbl, names):
        return {r[names[0]]: tuple(r[n] for n in names[1:]) for r in tbl.to_pylist()}

    g = rows(got, ["k", "sum(flow.v)", "count(flow.v)", "min(flow.v)", "max(flow.v)", "avg(flow.v)", "count(*)"])
    w = rows(want, ["k", "v_sum", "v_count", "v_min", "v_max", "v_mean", "count_all"])
    assert g.keys() == w.keys()  # includes the NULL key: both keep it as a group
    for key in w:
        gs, gc, gmin, gmax, gavg, gn = g[key]
        ws, wc, wmin, wmax, wavg, wn = w[key]
        assert (gs, gc, gmin, gmax, gn) == (ws, wc, wmin, wmax, wn), key
        assert (gavg is None and wavg is None) or abs(gavg - wavg) <= 1e-12 * max(1.0, abs(wavg)), key


def test_inner_join_matches_acero():
    left = batch(31, n=3000, keys=50)
    rng = np.random.default_rng(32)
    right = pa.record_batch({"k": pa.array([f"key_{i:03d}" for i in range(0, 60, 2)] + [None]), "z": pa.array(rng.integers(0, 9, 31), pa.int64())})
    got = sql_join({"a": left, "b": right}, "SELECT a.k, v, z FROM a JOIN b ON a.k = b.k")
    want = pa.Table.from_batches([left]).join(pa.Table.from_batches([right]), keys="k", join_type="inner").select(["k", "v", "z"])
    key = lambda tbl: sorted(map(repr, zip(*[tbl.column(i).to_pylist() for i in range(3)])))
    assert key(got) == key(want)  # NULL keys never match, on either side


@pytest.mark.parametrize("kind,acero", [("LEFT", "left outer"), ("RIGHT", "right outer"), ("LEFT OUTER", "left outer")])
def test_outer_joins_match_acero(kind, acero):
    """LEFT / RIGHT [OUTER] JOIN of the oracle against Acero: unmatched rows of the preserved side come out once with NULLs
    on the other side, NULL keys never match (but are preserved), duplicate build keys multiply rows."""
    left = batch(41, n=2000, keys=40)
    rng = np.random.default_rng(42)
    rk = [f"key_{i:03d}" for i in range(10, 70, 3)] + [None, "key_013", "key_013"]
    right = pa.record_batch({"k": pa.array(rk), "z": pa.array(rng.integers(0, 9, len(rk)), pa.int64())})
    got = sql_join({"a": left, "b": right}, f"SELECT a.k, v, z FROM a {kind} JOIN b ON a.k = b.k")
    lt, rt = pa.Table.from_batches([left]), pa.Table.from_batches([right])
    want = lt.join(rt, keys="k", join_type=acero, coalesce_keys=False, right_suffix="_r").select(["k", "v", "z"])  # a.k as it is on the left side
    key = lambda tbl: sorted(map(repr, zip(*[tbl.column(i).to_pylist() for i in range(3)])))
    assert key(got) == key(want)


def test_nested_json_matches_arrow_json_reader():
    """List<scalar> and Struct columns of the oracle's optional nested decoding against Arrow C++'s JSON reader on records whose
    every row has the first record's shape (where first-record inference and whole-file inference agree)."""
    import io
    import json

    import pyarrow.json as pj

    import oracle.json_oracle as jo
    from arkflow_b200.processor import MessageBatch

    rng = np.random.default_rng(9)
    recs = [{"id": i, "tags": ["t%d" % int(x) for x in rng.integers(0, 5, int(rng.integers(1, 4)))], "nums": [int(x) for x in rng.integers(-9, 9, 3)],
             "pos": {"x": float(i) / 4, "y": int(i % 7), "label": "p%d" % i}} for i in range(300)]
    payloads = [json.dumps(r).encode() for r in recs]
    prev = jo.NESTED
    jo.NESTED = True
    try:
        got = jo.json_to_arrow(MessageBatch.new_binary(payloads).record_batch)
    finally:
        jo.NESTED = prev
    want = pj.read_json(io.BytesIO(b"\n".join(payloads)))
    assert got.schema.names == want.schema.names
    for name in want.schema.names:
        assert got.column(name).to_pylist() == want[name].to_pylist(), name


def test_json_decode_matches_arrow_json_reader():
    # uniform scalar records: arrow-json (first-record inference) and Arrow C++'s reader must decode the same values
    import io
    import json

    import pyarrow.json as pj

    from arkflow_b200.processor import MessageBatch
    from oracle.json_oracle import json_to_arrow

    rng = np.random.default_rng(5)
    NOTE = 'caf\u00e9 "q" \\ \n'  # non-ASCII, a quote, a backslash, a newline: all escaped by json.dumps
    recs = [{"timestamp": int(1625000000000 + i), "value": int(rng.integers(-10**12, 10**12)), "x": float(rng.normal() * 10.0 ** int(rng.integers(-8, 9))),
             "flag": bool(i % 3 == 0), "sensor": f"temp_{int(rng.integers(0, 50))}", "note": NOTE if i % 7 == 0 else "plain"} for i in range(500)]
    payloads = [json.dumps(r).encode() for r in recs]
    got = json_to_arrow(MessageBatch.new_binary(payloads).record_batch)
    want = pj.read_json(io.BytesIO(b"\n".join(payloads)))
    assert got.schema.names == want.schema.names
    for name in want.schema.names:
        assert got.column(name).to_pylist() == want[name].to_pylist(), name


# ---- non-finite float sums: group_sum_exact is total (NaN / ±inf where math.fsum raises) -----------------------------
INF, NAN = float("inf"), float("nan")


@pytest.mark.parametrize("xs, want", [
    ([INF, -INF], NAN),                   # fsum: ValueError (-inf + inf)
    ([1.0, INF, 2.0, -INF], NAN),
    ([NAN, 1.0], NAN),
    ([-NAN, INF], NAN),
    ([INF, 1e300, INF], INF),
    ([-INF, -5e-324, 3.0], -INF),
    ([1.7e308, 1.7e308], INF),            # fsum: OverflowError (the exact sum is out of range)
    ([-1.7e308, -1.7e308, 1.0], -INF),
    ([1.7e308, 1.7e308, -1.7e308], 1.7e308),   # a partial sum leaves the range, the exact sum does not
    ([1e300, 5e-324, -1e300], 5e-324),
    ([-0.0], -0.0),
    ([], 0.0),
])
def test_group_sum_exact_non_finite(xs, want):
    from fractions import Fraction

    from oracle.sql_oracle import group_sum_exact

    got = group_sum_exact(np.array(xs, np.float64), np.zeros(len(xs), np.int64), 1)[0]
    if math.isnan(want):
        assert math.isnan(got)
    else:
        assert got == want, (xs, got)
        if math.isfinite(want) and xs:
            assert Fraction(got) == Fraction(want)


def test_sql_sum_avg_over_non_finite_groups():
    """SUM / AVG over groups holding both infinities, NaN or an out-of-range exact sum: the oracle answers where it used to
    raise, and groups of finite values keep the correctly rounded sum."""
    k = ["both", "both", "nan", "nan", "pinf", "pinf", "big", "big", "fin", "fin", "null"]
    v = [INF, -INF, NAN, 2.0, INF, 1e300, 1.7e308, 1.7e308, 0.1, 0.2, None]
    rb = pa.record_batch({"k": pa.array(k), "v": pa.array(v, pa.float64())})
    got = sql_process(rb, "SELECT k, SUM(v), AVG(v), COUNT(v) FROM flow GROUP BY k")
    d = {r["k"]: (r["sum(flow.v)"], r["avg(flow.v)"], r["count(flow.v)"]) for r in got.to_pylist()}
    assert math.isnan(d["both"][0]) and math.isnan(d["both"][1])
    assert math.isnan(d["nan"][0]) and math.isnan(d["nan"][1])
    assert d["pinf"][:2] == (INF, INF)
    assert d["big"][:2] == (INF, INF)
    assert d["fin"] == (0.30000000000000004, 0.15000000000000002, 2)
    assert d["null"] == (None, None, 0)
