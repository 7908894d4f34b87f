"""Parity of the CUDA GROUP BY hash-aggregate (through the C ABI) against the oracle.

GROUP BY output order is unspecified in DataFusion, so results are compared as multisets keyed by the
group key.  Integer SUM / COUNT / MIN / MAX are bit-exact; Float64 SUM / AVG are checked against the
correctly-rounded sum with the tolerance of SURVEY.md §8(d):
    |got − exact| ≤ 2·(n_g − 1)·2⁻⁵³ · Σ|x_i|      (any summation order satisfies it).
"""
import math

import numpy as np
import pyarrow as pa
import pyarrow.compute  # noqa: F401
import pytest

from agg_util import float_sum_bound, float_sum_mismatches
from arkflow_b200.arrow_ffi import DeviceBatch
from arkflow_b200.processor import ArkError, MessageBatch, SqlProcessor
from oracle.sql_oracle import sql_process
from oracle.synth import synth_batch

pytestmark = pytest.mark.gpu


def run(rb, query, device=False):
    p = SqlProcessor({"query": query})
    if device:
        out = p.process_device(DeviceBatch.from_arrow(rb))
        return None if out is None else out.to_arrow()
    r = p.process(MessageBatch.new_arrow(rb))
    return None if r.is_none() else r.batches[0].record_batch


def rows_as_dict(rb, key_cols):
    cols = {n: rb.column(i).to_pylist() for i, n in enumerate(rb.schema.names)}
    out = {}
    for i in range(rb.num_rows):
        k = tuple(cols[c][i] for c in key_cols)
        assert k not in out, f"duplicate group {k}"
        out[k] = {n: cols[n][i] for n in cols}
    return out


def check_agg(rb, query, key_cols, float_cols=(), abs_sums=None, counts=None):
    want = sql_process(rb, query)
    for device in (False, True):
        got = run(rb, query, device=device)
        assert got.schema.names == want.schema.names, (got.schema, want.schema)
        assert [f.type for f in got.schema] == [f.type for f in want.schema], (got.schema, want.schema)
        assert got.num_rows == want.num_rows, (query, got.num_rows, want.num_rows)
        if not key_cols:  # global aggregate or key not projected: compare sorted rows
            g = sorted(map(tuple, zip(*[c.to_pylist() for c in got.columns])), key=repr)
            w = sorted(map(tuple, zip(*[c.to_pylist() for c in want.columns])), key=repr)
            if not float_cols:
                assert g == w
            else:  # float aggregates without a projected key: every row's floats within the §8(d) bound over the whole batch
                assert len(g) == len(w)
                n_rows = rb.num_rows
                s_abs = abs_sums[()] if abs_sums and () in abs_sums else None
                if s_abs is None and "value" in rb.schema.names:
                    s_abs = float(sum(abs(v) for v in rb.column("value").to_pylist() if v is not None))
                fidx = [i for i, nm in enumerate(want.schema.names) if nm in float_cols]
                key_of = lambda row: tuple(v for i, v in enumerate(row) if i not in fidx)  # noqa: E731
                g2, w2 = sorted(g, key=lambda r: repr(key_of(r))), sorted(w, key=lambda r: repr(key_of(r)))
                for gr, wr in zip(g2, w2):
                    assert key_of(gr) == key_of(wr)
                    for i in fidx:
                        gv, wv = gr[i], wr[i]
                        assert (gv is None) == (wv is None)
                        if wv is None:
                            continue
                        # the bound over the whole batch, not divided by the row count for AVG
                        bound = float_sum_bound(n_rows, s_abs if s_abs is not None else abs(wv) * n_rows, wv) + \
                            (abs(wv) * 2.0 ** -52 if want.schema.names[i].startswith("avg") else 0.0)
                        assert abs(gv - wv) <= bound, (want.schema.names[i], gv, wv, bound)
            continue
        gd, wd = rows_as_dict(got, key_cols), rows_as_dict(want, key_cols)
        assert gd.keys() == wd.keys()
        for k in wd:
            for n in want.schema.names:
                gv, wv = gd[k][n], wd[k][n]
                if n in float_cols and wv is not None and gv is not None:
                    ng = counts[k] if counts else 1
                    bad = float_sum_mismatches([gv], [wv], ng, abs_sums[k] if abs_sums else abs(wv), avg=n.startswith("avg"))
                    assert len(bad) == 0, (k, n, gv, wv)
                else:
                    assert gv == wv, (k, n, gv, wv)
    return want


def test_config3_group_by_sensor_int(gpu):
    rb = synth_batch(200_000, key_space=1000)
    out = check_agg(rb, "SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor", ["sensor"])
    assert out.num_rows == 1000
    assert out.schema.names == ["sensor", "sum(flow.value)", "count(*)"]


def test_config1a_generate_example_query(gpu):
    # examples/generate_example.yaml:26 — key not projected, literal column
    rb = pa.record_batch({"timestamp": pa.array([1625000000000], pa.int64()), "value": pa.array([10], pa.int64()),
                          "sensor": pa.array(["temp_1"])})
    out = check_agg(rb, "SELECT sum(value),avg(value) ,111 as x FROM flow  group by sensor", [])
    assert out.to_pydict() == {"sum(flow.value)": [10], "avg(flow.value)": [10.0], "x": [111]}


def test_drop_output_example_query(gpu):
    # examples/drop_output_example.yaml:18
    rb = synth_batch(50_000, key_space=13)
    check_agg(rb, "SELECT count(*) FROM flow WHERE value >= 10 group by sensor", [])
    check_agg(rb, "SELECT sensor, count(*) FROM flow WHERE value >= 10 group by sensor", ["sensor"])


def test_stream_data_fixture(gpu):
    import json, os
    p = os.path.join(os.path.dirname(__file__), "golden", "stream_data.json")
    rows = [json.loads(l) for l in open(p)]
    rb = pa.record_batch({"timestamp": pa.array([r["timestamp"] for r in rows], pa.int64()),
                          "value": pa.array([r["value"] for r in rows], pa.int64()),
                          "sensor": pa.array([r["sensor"] for r in rows])})
    out = check_agg(rb, "SELECT sensor, SUM(value), COUNT(*), AVG(value), MIN(value), MAX(value) FROM flow GROUP BY sensor", ["sensor"],
                    float_cols=["avg(flow.value)"])
    d = rows_as_dict(out, ["sensor"])
    assert d[("temp_1",)]["sum(flow.value)"] == 223 and d[("temp_1",)]["count(*)"] == 11
    assert d[("temp_2",)]["sum(flow.value)"] == 288 and d[("temp_2",)]["count(*)"] == 10


@pytest.mark.parametrize("k", [1, 2, 37, 5000, 100_000])
def test_cardinalities(gpu, k):
    rb = synth_batch(300_000, key_space=k, seed=7 + k)
    check_agg(rb, "SELECT sensor, SUM(value), COUNT(*), MIN(value), MAX(value) FROM flow GROUP BY sensor", ["sensor"])


def test_float_sum_avg_tolerance(gpu):
    rb = synth_batch(400_000, value_kind=1, key_space=500)
    keys = rb.column("sensor").to_pylist()
    vals = np.asarray(rb.column("value"))
    abs_sums, counts = {}, {}
    for kx, v in zip(keys, vals):
        abs_sums[(kx,)] = abs_sums.get((kx,), 0.0) + abs(v)
        counts[(kx,)] = counts.get((kx,), 0) + 1
    check_agg(rb, "SELECT sensor, SUM(value), AVG(value), COUNT(value), MIN(value), MAX(value) FROM flow GROUP BY sensor", ["sensor"],
              float_cols=["sum(flow.value)", "avg(flow.value)"], abs_sums=abs_sums, counts=counts)


def test_int64_key_and_wrapping_sum(gpu):
    rng = np.random.default_rng(5)
    n = 100_000
    big = rng.integers(-2**62, 2**62, n)
    rb = pa.record_batch({"id": pa.array(rng.integers(-50, 50, n), pa.int64()), "v": pa.array(big, pa.int64())})
    check_agg(rb, "SELECT id, SUM(v), COUNT(*), MIN(v), MAX(v) FROM flow GROUP BY id", ["id"])


def test_global_aggregates(gpu):
    rb = synth_batch(100_000, key_space=100)
    check_agg(rb, "SELECT COUNT(*), SUM(value), MIN(value), MAX(value) FROM flow", [])
    check_agg(rb, "SELECT COUNT(*) FROM flow WHERE value >= 10", [])
    out = check_agg(rb, "SELECT COUNT(*), SUM(value) FROM flow WHERE value > 1000", [])
    assert out.to_pydict() == {"count(*)": [0], "sum(flow.value)": [None]}


def test_count_star_pins_reference_value(gpu):
    # crates/arkflow-core/src/lib.rs:1811-1858: COUNT(*) over 5 rows is Int64 5
    rb = pa.record_batch({"id": pa.array([1, 2, 3, 4, 5], pa.int64())})
    out = run(rb, "SELECT COUNT(*) as cnt FROM flow")
    assert out.schema.field(0).type == pa.int64() and out.column(0).to_pylist() == [5]


def test_nulls_in_keys_and_values(gpu):
    rng = np.random.default_rng(11)
    n = 50_000
    keys = [None if rng.random() < 0.1 else "k%d" % int(rng.integers(0, 40)) for _ in range(n)]
    v = rng.integers(0, 100, n)
    rb = pa.record_batch({"sensor": pa.array(keys), "value": pa.array(v, pa.int64(), mask=rng.random(n) < 0.3),
                          "g": pa.array([None if rng.random() < 0.2 else int(x) % 7 for x in v], pa.int64()),
                          "b": pa.array([None if rng.random() < 0.2 else bool(x & 1) for x in v], pa.bool_())})
    check_agg(rb, "SELECT sensor, SUM(value), COUNT(value), COUNT(*), AVG(value), MIN(value), MAX(value) FROM flow GROUP BY sensor", ["sensor"],
              float_cols=["avg(flow.value)"])
    check_agg(rb, "SELECT g, COUNT(*), SUM(value) FROM flow GROUP BY g", ["g"])
    check_agg(rb, "SELECT b, COUNT(*), SUM(value) FROM flow GROUP BY b", ["b"])
    check_agg(rb, "SELECT sensor, SUM(value) FROM flow WHERE value IS NULL GROUP BY sensor", ["sensor"])


def test_long_and_ragged_string_keys(gpu):
    rng = np.random.default_rng(2)
    base = ["", "a", "ab", "exactly12chr", "thirteen chrs", "x" * 40, "x" * 40 + "y", "prefix_same_" + "a" * 30, "prefix_same_" + "b" * 30]
    base += ["key-%d-%s" % (i, "z" * int(rng.integers(0, 60))) for i in range(300)]
    n = 60_000
    keys = [base[int(i)] for i in rng.integers(0, len(base), n)]
    rb = pa.record_batch({"sensor": pa.array(keys), "value": pa.array(rng.integers(0, 1000, n), pa.int64())})
    check_agg(rb, "SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor", ["sensor"])
    rbb = pa.record_batch({"sensor": pa.array([k.encode() for k in keys], pa.binary()), "value": rb.column("value")})
    check_agg(rbb, "SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor", ["sensor"])


def test_low_cardinality_key_lengths_change_by_region(gpu):
    """ADVICE r1 (high): the per-CTA-table kernel stages a tile's key bytes only when they fit its window, and its mbarrier
    phase must advance only for staged tiles.  > 1M rows so that every CTA takes several tiles; short keys, then a region of
    ~48-byte keys that exceed the window sized from the batch average, then short keys again; also an all-empty-key region."""
    n = 1_400_000
    idx = np.arange(n)
    region = (idx // 100_000) % 7
    keys = np.where(region == 2, np.char.add("k" * 47, (idx % 5).astype(str)),
           np.where(region == 4, "", np.where(region == 5, np.char.add("a_key_of_25_bytes_exactly_", (idx % 3).astype(str)), np.char.add("s", (idx % 6).astype(str)))))
    rng = np.random.default_rng(5)
    rb = pa.record_batch({"sensor": pa.array(keys.tolist()), "value": pa.array(rng.integers(-50, 50, n), pa.int64())})
    for _ in range(2):  # the second call reuses the hints of the first (table size, window)
        check_agg(rb, "SELECT sensor, SUM(value), COUNT(*), MIN(value) FROM flow GROUP BY sensor", ["sensor"])


def test_computed_aggregate_arguments(gpu):
    rb = synth_batch(100_000, key_space=50)
    check_agg(rb, "SELECT sensor, SUM(value * 2 + 1), AVG(value + 0.5), COUNT(*) FROM flow WHERE value >= 3 GROUP BY sensor", ["sensor"],
              float_cols=["avg(flow.value + Float64(0.5))"])


def test_table_growth_from_small_hint(gpu):
    # first a tiny-cardinality batch (hint shrinks), then a high-cardinality one (forces the retry path)
    check_agg(synth_batch(10_000, key_space=2), "SELECT sensor, COUNT(*) FROM flow GROUP BY sensor", ["sensor"])
    check_agg(synth_batch(400_000, key_space=300_000, seed=9), "SELECT sensor, COUNT(*), SUM(value) FROM flow GROUP BY sensor", ["sensor"])


def test_table_larger_than_l2(gpu):
    # ~1.1 M groups: the table ends at 2^21 slots or more (>= 64 MB), more than the L2 of an H100 holds, which selects the
    # register-prefetch kernel of hash_agg_stream.cu instead of the TMA-staged one
    check_agg(synth_batch(2_000_000, key_space=1_500_000, seed=13), "SELECT sensor, COUNT(*), SUM(value) FROM flow GROUP BY sensor", ["sensor"])


def test_aggregate_planning_errors(gpu):
    rb = synth_batch(10)
    with pytest.raises(ArkError) as e:
        run(rb, "SELECT timestamp, COUNT(*) FROM flow GROUP BY sensor")
    assert e.value.kind == "Process"
    with pytest.raises(ArkError):
        run(rb, "SELECT SUM(sensor) FROM flow")


# ---- many groups: string, Int64, long and NULL keys, float values, one hot key --------------------------
def check_agg_sorted(rb, query, key, float_cols=()):
    """check_agg for many groups: both results sorted by the key column, columns compared as arrays."""
    want = sql_process(rb, query)
    for device in (False, True):
        got = run(rb, query, device=device)
        assert got.schema.names == want.schema.names
        assert [f.type for f in got.schema] == [f.type for f in want.schema]
        assert got.num_rows == want.num_rows
        g = pa.Table.from_batches([got]).sort_by(key)
        w = pa.Table.from_batches([want]).sort_by(key)
        for name in want.schema.names:
            a, b = g.column(name).combine_chunks(), w.column(name).combine_chunks()
            if name in float_cols:
                x, y = a.to_numpy(zero_copy_only=False), b.to_numpy(zero_copy_only=False)
                assert np.allclose(x, y, rtol=1e-12, atol=0.0), name  # ≤ a few hundred addends per group here
            else:
                assert a.equals(b), name
    return want


def test_many_groups_string_keys(gpu):
    rb = synth_batch(400_000, key_space=150_000, seed=21)
    q = "SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor"
    check_agg_sorted(rb, q, "sensor")  # first call may still be growing the capacity hint
    check_agg_sorted(rb, q, "sensor")
    check_agg_sorted(rb, "SELECT sensor, SUM(value), COUNT(*), MIN(value), MAX(value), AVG(value) FROM flow WHERE value >= 4 GROUP BY sensor",
                     "sensor", float_cols=["avg(flow.value)"])


def test_many_groups_float_values_and_int_keys(gpu):
    rb = synth_batch(300_000, value_kind=1, key_space=120_000, seed=22)
    check_agg_sorted(rb, "SELECT sensor, SUM(value), AVG(value), COUNT(*) FROM flow GROUP BY sensor", "sensor",
                     float_cols=["sum(flow.value)", "avg(flow.value)"])
    rng = np.random.default_rng(23)
    n = 300_000
    rb2 = pa.record_batch({"id": pa.array(rng.integers(-2**40, 2**40, n) // 2**23, pa.int64()), "v": pa.array(rng.integers(-2**62, 2**62, n), pa.int64())})
    check_agg_sorted(rb2, "SELECT id, SUM(v), COUNT(*), MIN(v), MAX(v) FROM flow GROUP BY id", "id")


def test_many_groups_long_keys_and_null_keys(gpu):
    rng = np.random.default_rng(24)
    n = 200_000
    ids = rng.integers(0, 90_000, n)
    keys = [None if i % 997 == 0 else (f"k{i}" if i % 3 else f"a-rather-long-sensor-name-{i:09d}") for i in ids.tolist()]
    rb = pa.record_batch({"sensor": pa.array(keys, pa.utf8()), "value": pa.array(rng.integers(0, 1000, n), pa.int64())})
    want = check_agg_sorted(rb, "SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor", "sensor")
    assert want.column("sensor").null_count == 1


def test_many_groups_one_hot_key(gpu):
    # half of the rows carry one key: its slot takes every other row's atomics
    rb = synth_batch(400_000, key_space=150_000, seed=25)
    hot = pa.array(["hot_sensor_0"] * 400_000)
    idx = np.arange(400_000)
    sensor = pa.compute.if_else(pa.array(idx % 2 == 0), hot, rb.column("sensor"))
    rb = pa.record_batch({"timestamp": rb.column("timestamp"), "value": rb.column("value"), "sensor": sensor})
    q = "SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor"
    check_agg_sorted(rb, q, "sensor")
    check_agg_sorted(rb, q, "sensor")


def test_protobuf_example_query_cast_of_aggregate_and_order_by(gpu):
    # examples/protobuf_example.yaml: a global aggregate with CAST(count(..) AS STRING) and an ORDER BY over its one row
    rb = synth_batch(50_000, key_space=11)
    q = ("SELECT count(timestamp) as timestamp, sum(value) as value, cast(count(sensor) as string) as  sensor "
         "FROM flow WHERE value >= 10 order by sensor")
    want = sql_process(rb, q)
    for device in (False, True):
        got = run(rb, q, device=device)
        assert got.schema.names == want.schema.names == ["timestamp", "value", "sensor"]
        assert [f.type for f in got.schema] == [pa.int64(), pa.int64(), pa.utf8()]
        assert got.to_pydict() == want.to_pydict()
    check_agg(rb, "SELECT sensor, cast(count(*) as string) AS c, cast(sum(value) as string), cast(min(value) as string) AS lo FROM flow GROUP BY sensor", ["sensor"])
    nulls = pa.record_batch({"k": pa.array(["a", "a", "b"]), "v": pa.array([None, None, 4], pa.int64())})
    out = check_agg(nulls, "SELECT k, cast(sum(v) as string) AS s, cast(count(v) as string) AS c FROM flow GROUP BY k", ["k"])
    assert sorted(zip(out.column("k").to_pylist(), out.column("s").to_pylist(), out.column("c").to_pylist())) == [("a", None, "0"), ("b", "4", "1")]
    with pytest.raises(ArkError) as e:
        SqlProcessor({"query": "SELECT sensor, count(*) FROM flow GROUP BY sensor ORDER BY sensor"})
    assert e.value.kind == "Unsupported"
    with pytest.raises(ArkError) as e:
        run(rb, "SELECT cast(avg(value) as string) FROM flow")
    assert e.value.kind == "Unsupported"


def test_two_group_by_keys(gpu):
    """Composite keys (KEY_PAIR): every combination of key types, NULLs in either key, the keys projected in any order."""
    rng = np.random.default_rng(21)
    n = 60_000
    rb = pa.record_batch({
        "a": pa.array([None if rng.random() < 0.05 else int(x) for x in rng.integers(0, 40, n)], pa.int64()),
        "s": pa.array([None if rng.random() < 0.05 else "k%d" % int(x) for x in rng.integers(0, 25, n)]),
        "long": pa.array(["a_long_key_value_%02d" % int(x) for x in rng.integers(0, 30, n)]),
        "b": pa.array([bool(x) for x in rng.integers(0, 2, n)], pa.bool_()),
        "v": pa.array(rng.integers(-100, 100, n), pa.int64()),
        "f": pa.array(rng.random(n), pa.float64()),
    })
    check_agg(rb, "SELECT a, s, SUM(v), COUNT(*) FROM flow GROUP BY a, s", ["a", "s"])
    check_agg(rb, "SELECT s, a, MIN(v), MAX(v), COUNT(v) FROM flow WHERE v <> 0 GROUP BY a, s", ["a", "s"])
    check_agg(rb, "SELECT long, b, COUNT(*), SUM(v) FROM flow GROUP BY long, b", ["long", "b"])
    check_agg(rb, "SELECT s, long, COUNT(*) FROM flow GROUP BY s, long", ["s", "long"])
    check_agg(rb, "SELECT b, a, COUNT(*) FROM flow GROUP BY b, a", ["b", "a"])
    check_agg(rb, "SELECT a, COUNT(*) FROM flow GROUP BY a, b", [])  # second key not projected: duplicate `a` rows
    sums = {}
    for a, s_, f in zip(rb.column("a").to_pylist(), rb.column("s").to_pylist(), rb.column("f").to_pylist()):
        sums[(a, s_)] = sums.get((a, s_), 0.0) + abs(f)
    counts = {}
    for a, s_ in zip(rb.column("a").to_pylist(), rb.column("s").to_pylist()):
        counts[(a, s_)] = counts.get((a, s_), 0) + 1
    check_agg(rb, "SELECT a, s, SUM(f), AVG(f) FROM flow GROUP BY a, s", ["a", "s"], float_cols=("sum(flow.f)", "avg(flow.f)"), abs_sums=sums, counts=counts)


def test_two_keys_high_cardinality(gpu):
    rb = synth_batch(400_000, key_space=50_000)
    check_agg(rb, "SELECT sensor, value, COUNT(*), SUM(timestamp) FROM flow GROUP BY sensor, value", ["sensor", "value"])


def test_key_dictionary_is_reused_across_batches(gpu):
    """The processor keeps a plan's table (its KEYS) from batch to batch (AggHints::CachedTable) and resets only the
    accumulators: keys of an earlier batch that are absent from the current one must not appear, new keys must, every
    aggregate must be the batch's own — for string and integer keys, MIN/MAX identities included."""
    for query, keys in (("SELECT sensor, SUM(value), COUNT(*), MIN(value), MAX(timestamp) FROM flow GROUP BY sensor", ["sensor"]),
                        ("SELECT value, COUNT(*), AVG(timestamp) FROM flow WHERE timestamp > 0 GROUP BY value", ["value"])):
        p = SqlProcessor({"query": query})
        rng = np.random.default_rng(9)
        for step in range(6):
            n = 60_000
            # key ranges drift: [0,3000) → [1500,4500) → … so that old keys disappear and new ones arrive
            lo = 1500 * (step % 4)
            k = rng.integers(lo, lo + 3000, n)
            rb = pa.record_batch({"timestamp": pa.array(rng.integers(1, 10**9, n), pa.int64()),
                                  "value": pa.array(k if "GROUP BY value" in query else rng.integers(-50, 50, n), pa.int64()),
                                  "sensor": pa.array(["s%05d" % x for x in k])})
            want = sql_process(rb, query)
            for device in (False, True):
                if device:
                    got = p.process_device(DeviceBatch.from_arrow(rb)).to_arrow()
                else:
                    got = p.process(MessageBatch.new_arrow(rb)).batches[0].record_batch
                assert got.num_rows == want.num_rows, (step, got.num_rows, want.num_rows)
                gd, wd = rows_as_dict(got, keys), rows_as_dict(want, keys)
                assert gd.keys() == wd.keys()
                for kk in wd:
                    for nm in want.schema.names:
                        gv, wv = gd[kk][nm], wd[kk][nm]
                        assert gv == wv or (isinstance(wv, float) and abs(gv - wv) <= 1e-9 * abs(wv)), (step, kk, nm, gv, wv)
