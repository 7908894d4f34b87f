"""Parity of the CUDA filter/project path (through the C ABI) against the oracle.

Mirrors the reference's in-file tests of the sql processor
(crates/arkflow-plugin/src/processor/sql.rs:257-425) and widens them with value checks:
integer / byte / index work must be bit-exact.
"""
import os

import numpy as np
import pyarrow as pa
import pytest

from arkflow_b200.arrow_ffi import DeviceBatch
from arkflow_b200.processor import ArkError, MessageBatch, SqlProcessor
from oracle.sql_oracle import OracleError, sql_process
from oracle.synth import synth_batch

pytestmark = pytest.mark.gpu


def run(rb, query, device=False, table_name=None):
    cfg = {"query": query}
    if table_name:
        cfg["table_name"] = table_name
    p = SqlProcessor(cfg)
    if device:
        out = p.process_device(DeviceBatch.from_arrow(rb))
        return None if out is None else out.to_arrow()
    r = p.process(MessageBatch.new_arrow(rb))
    return None if r.is_none() else r.batches[0].record_batch


def check(rb, query, **kw):
    want = sql_process(rb, query, kw.get("table_name") or "flow")
    for device in (False, True):
        got = run(rb, query, device=device, **kw)
        if want is None:
            assert got is None
            continue
        assert got.schema.names == want.schema.names, (got.schema, want.schema)
        assert [f.type for f in got.schema] == [f.type for f in want.schema], (got.schema, want.schema)
        assert got.num_rows == want.num_rows, (query, device, got.num_rows, want.num_rows)
        for name, g, w in zip(got.schema.names, got.columns, want.columns):
            assert g.equals(w), f"column {name} differs (device={device}) for {query}"
    return want


def test_basic_query(gpu):
    # sql.rs:257-297
    rb = pa.record_batch({"id": pa.array([1, 2, 3], pa.int64()), "name": pa.array(["a", "b", "c"])})
    out = check(rb, "SELECT * FROM flow")
    assert out.num_rows == 3


def test_empty_batch_is_none(gpu):
    # sql.rs:299-322
    rb = pa.record_batch({"id": pa.array([], pa.int64()), "name": pa.array([], pa.utf8())})
    assert run(rb, "SELECT * FROM flow") is None
    assert run(rb, "SELECT * FROM flow", device=True) is None


def test_invalid_query_fails_at_construction(gpu):
    # sql.rs:324-339
    with pytest.raises(ArkError) as e:
        SqlProcessor({"query": "INVALID SQL QUERY"})
    assert e.value.kind == "Process" and e.value.message.startswith("SQL query error")


def test_custom_table_name(gpu):
    # sql.rs:341-375
    rb = pa.record_batch({"id": pa.array([1], pa.int64())})
    out = check(rb, "SELECT * FROM custom_table", table_name="custom_table")
    assert out.num_rows == 1


def test_pool_performance_query(gpu):
    # sql.rs:377-425: WHERE id > 0 ×10 on a 5-row batch
    rb = pa.record_batch({"id": pa.array([1, 2, 3, 4, 5], pa.int64()), "value": pa.array([10, 20, 30, 40, 50], pa.int64())})
    p = SqlProcessor({"query": "SELECT * FROM flow WHERE id > 0"})
    for _ in range(10):
        r = p.process(rb)
        assert r.batches[0].num_rows == 5


@pytest.mark.parametrize("n", [1, 2, 31, 511, 512, 513, 2047, 2048, 2049, 4097, 100_003])
@pytest.mark.parametrize("value_kind", [0, 1])
def test_config2_filter_project_sizes(gpu, n, value_kind):
    rb = synth_batch(n, seed=42 + n, value_kind=value_kind, key_space=1000)
    check(rb, "SELECT sensor, value FROM flow WHERE value >= 10")


def test_config2_one_million(gpu):
    rb = synth_batch(1 << 20, key_space=1_000_000)
    out = check(rb, "SELECT sensor, value FROM flow WHERE value >= 10")
    assert abs(out.num_rows / rb.num_rows - 0.5) < 0.01


def test_readme_quickstart_select_star_where(gpu):
    rb = synth_batch(10_000, key_space=7)
    check(rb, "SELECT * FROM flow WHERE value >= 10")


def test_all_filtered_is_zero_row_batch_not_none(gpu):
    rb = synth_batch(5000)
    out = check(rb, "SELECT sensor, value FROM flow WHERE value >= 1000")
    assert out is not None and out.num_rows == 0


def test_none_filtered(gpu):
    rb = synth_batch(5000)
    out = check(rb, "SELECT timestamp, sensor, value FROM flow WHERE value >= 0")
    assert out.num_rows == 5000


@pytest.mark.parametrize("op", ["=", "!=", "<", "<=", ">", ">="])
def test_comparison_ops_int_and_float(gpu, op):
    rb = synth_batch(10_000, key_space=50)
    check(rb, f"SELECT value FROM flow WHERE value {op} 7")
    check(rb, f"SELECT value FROM flow WHERE 7 {op} value")
    rbf = synth_batch(10_000, value_kind=1, key_space=50)
    check(rbf, f"SELECT value FROM flow WHERE value {op} 7")
    check(rbf, f"SELECT value FROM flow WHERE value {op} 7.25")


def test_float_total_order(gpu):
    vals = [float("nan"), -float("nan"), float("inf"), -float("inf"), 0.0, -0.0, 10.0, 9.999999, 1e308, -1e308]
    rb = pa.record_batch({"value": pa.array(vals, pa.float64()), "i": pa.array(range(len(vals)), pa.int64())})
    out = check(rb, "SELECT i FROM flow WHERE value >= 10")
    assert 0 in out.column(0).to_pylist()  # NaN >= 10 is TRUE under totalOrder
    check(rb, "SELECT i FROM flow WHERE value < 0")   # -0.0 < 0.0 … no: -0.0 < +0.0 only vs the literal +0.0
    check(rb, "SELECT i FROM flow WHERE value = 0")
    check(rb, "SELECT i FROM flow WHERE value <= 0.0 AND value >= -0.0")


def test_vm_predicates(gpu):
    rb = synth_batch(20_000, key_space=10)
    check(rb, "SELECT sensor, value FROM flow WHERE value >= 5 AND value < 15")
    check(rb, "SELECT sensor FROM flow WHERE value < 3 OR value > 17 OR timestamp = 1625000005000")
    check(rb, "SELECT value FROM flow WHERE NOT (value >= 10)")
    check(rb, "SELECT value FROM flow WHERE value * 2 + 1 > 20")
    check(rb, "SELECT value FROM flow WHERE value % 3 = 0")
    check(rb, "SELECT value FROM flow WHERE sensor = 'temp_0000003'")
    check(rb, "SELECT value, sensor FROM flow WHERE sensor >= 'temp_0000005' AND value >= 10")
    check(rb, "SELECT value FROM flow WHERE 'temp_0000003' != sensor")


def test_computed_projections(gpu):
    rb = synth_batch(10_000, key_space=10)
    check(rb, "SELECT value * 2 + 1, value / 3, value - timestamp, value >= 10 FROM flow")
    check(rb, "SELECT value + 0.5 AS v, cast(value as double) AS d, 111 AS x, 2.5 AS y FROM flow WHERE value >= 10")
    check(rb, "SELECT -value AS neg, value % 7 AS m FROM flow WHERE value > 3")
    rbf = synth_batch(10_000, value_kind=1, key_space=10)
    check(rbf, "SELECT value * 2, cast(value as bigint) AS t, value / 0 AS inf FROM flow WHERE value < 10")


def test_divide_by_zero_is_a_process_error(gpu):
    rb = synth_batch(1000)
    with pytest.raises(ArkError) as e:
        run(rb, "SELECT 10 / value FROM flow")
    assert e.value.kind == "Process" and "Divide by zero" in e.value.message
    # rows removed by the filter are not evaluated (FilterExec runs before ProjectionExec)
    check(rb, "SELECT 10 / value FROM flow WHERE value > 0")


@pytest.mark.parametrize("env", [{}, {"ARK_FP_DEBUG": "4"}], ids=["default", "helping"])
def test_fast_path_in_subprocess(gpu, env):
    """The fast path's tile kernel as built and with forced helping — forward progress without in-order dispatch: with
    ARK_FP_DEBUG=4 some tiles publish their aggregate late and the look-back of their successors gives up spinning after 2
    polls and computes the missing aggregates itself (help_publish_aggregate, csrc/filter_project_tma.cu).  Both give the
    oracle's results, ragged last tiles, long strings (the unstaged path) and an empty result included.  Subprocess: the
    knob is read once per process."""
    import os
    import subprocess
    import sys

    code = '''
import sys
sys.path.insert(0, %r)
import pyarrow as pa
from arkflow_b200 import _lib as L
from arkflow_b200.processor import SqlProcessor, MessageBatch, _check
from oracle.sql_oracle import sql_process
from oracle.synth import synth_batch
_check(L.lib().ark_b200_init(0))
cases = [(300_000, "SELECT sensor, value FROM flow WHERE value >= 10"), (257_123, "SELECT timestamp, value, sensor FROM flow WHERE value < 7"),
         (99_999, "SELECT sensor FROM flow WHERE value <> 3"), (1, "SELECT sensor, value FROM flow WHERE value >= 0"),
         (5_000, "SELECT sensor, value FROM flow WHERE value > 1000"), (1_000_003, "SELECT sensor, timestamp FROM flow WHERE value >= 19"),
         (257_123, "SELECT timestamp, value FROM flow WHERE value < 7")]
for n, q in cases:
    rb = synth_batch(n, key_space=1000)
    got = SqlProcessor({"query": q}).process(MessageBatch.new_arrow(rb)).batches[0].record_batch
    assert got.equals(sql_process(rb, q)), q
long_rb = pa.record_batch({"value": pa.array([i %% 20 for i in range(40_000)], pa.int64()),
                           "sensor": pa.array([("x" * (300 if 20_000 <= i < 21_500 else i %% 9)) + str(i) for i in range(40_000)])})  # a few tiles exceed the staging window
q = "SELECT sensor, value FROM flow WHERE value >= 10"
got = SqlProcessor({"query": q}).process(MessageBatch.new_arrow(long_rb)).batches[0].record_batch
assert got.equals(sql_process(long_rb, q)), "long strings"
print("FAST_OK")
''' % os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300, env=dict(os.environ, **env))
    assert r.returncode == 0 and "FAST_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-1500:]


def test_min_over_minus_one_overflows_for_div_and_mod(gpu):
    """arrow-arith div_checked / mod_checked: i64::MIN / -1 and i64::MIN % -1 are ArithmeticOverflow errors, with arrow's text."""
    rb = pa.record_batch({"a": pa.array([5, -(2 ** 63), 7], pa.int64()), "b": pa.array([1, -1, 2], pa.int64())})
    for op in ("/", "%"):
        q = f"SELECT a {op} b FROM flow"
        with pytest.raises(ArkError) as e:
            run(rb, q)
        assert e.value.kind == "Process" and f"Overflow happened on: -9223372036854775808 {op} -1" in e.value.message
        with pytest.raises(OracleError) as oe:
            sql_process(rb, q)
        assert f"-9223372036854775808 {op} -1" in str(oe.value)
        check(rb, f"SELECT a {op} b FROM flow WHERE a > 0")


def test_nulls(gpu):
    rng = np.random.default_rng(7)
    n = 10_000
    v = rng.integers(0, 20, n)
    vm = rng.random(n) < 0.2
    s = [None if rng.random() < 0.3 else f"s{int(x)}" * int(rng.integers(0, 4)) for x in v]
    rb = pa.record_batch({
        "value": pa.array(v, pa.int64(), mask=vm),
        "sensor": pa.array(s, pa.utf8()),
        "flag": pa.array([None if rng.random() < 0.1 else bool(x & 1) for x in v], pa.bool_()),
        "f": pa.array(rng.random(n), pa.float64(), mask=rng.random(n) < 0.5),
    })
    check(rb, "SELECT * FROM flow WHERE value >= 10")
    check(rb, "SELECT sensor, f FROM flow WHERE value IS NULL")
    check(rb, "SELECT value, flag FROM flow WHERE sensor IS NOT NULL AND f < 0.5")
    check(rb, "SELECT value + 1, f * 2 FROM flow WHERE flag")
    check(rb, "SELECT value FROM flow WHERE value > 5 OR f > 0.9")
    check(rb, "SELECT flag, NOT flag, flag AND value > 3 FROM flow")


def test_sliced_input_arrays(gpu):
    rb = synth_batch(10_000, key_space=33).slice(1237, 5001)
    check(rb, "SELECT sensor, value FROM flow WHERE value >= 10")
    check(rb, "SELECT * FROM flow")


_DEVICE_SLICES = '''
import sys
sys.path.insert(0, %r)
import os

import numpy as np
import pyarrow as pa
from arkflow_b200 import _lib as L
from arkflow_b200.arrow_ffi import DeviceBatch
from arkflow_b200.processor import SqlProcessor, _check
from oracle.sql_oracle import sql_process
_check(L.lib().ark_b200_init(0))
rng = np.random.default_rng(17)
n = 70_000
v = rng.integers(0, 20, n + 1237)
rb = pa.record_batch({
    "value": pa.array(v, pa.int64(), mask=rng.random(n + 1237) < 0.1),
    "sensor": pa.array(["s%%d" %% x * int(x %% 4) for x in v], pa.utf8(), mask=rng.random(n + 1237) < 0.2),
    "blob": pa.array([b"\\x00b%%d" %% x for x in v], pa.binary()),
    "flag": pa.array(v %% 3 == 0, pa.bool_(), mask=rng.random(n + 1237) < 0.15),
    "f": pa.array(rng.uniform(-1, 1, n + 1237), pa.float64()),
})
queries = ["SELECT sensor, value FROM flow WHERE value >= 10", "SELECT * FROM flow WHERE f < 0.25", "SELECT * FROM flow",
           "SELECT value + 1, blob, flag FROM flow WHERE flag", "SELECT sensor, f FROM flow WHERE value IS NULL OR f > 0.5"]
for off in (1, 3, 7, 1237):
    for m in (1, 1000, n):
        sl = rb.slice(off, m)
        want_rb = pa.RecordBatch.from_arrays([pa.concat_arrays([c]) for c in sl.columns], schema=sl.schema)
        for q in queries:
            got = SqlProcessor({"query": q}).process_device(DeviceBatch.from_arrow(sl, keep_offsets=True)).to_arrow()
            assert got.equals(sql_process(want_rb, q)), (off, m, q)
print("SLICES_OK")
''' % os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("env", [{}, {"ARK_FP_DEBUG": "4"}])
def test_device_sliced_inputs(gpu, env):
    """Device batches whose columns are Arrow slices, as a producer that slices device batches hands them over: Int64 data
    8 bytes past a 16-byte boundary, offsets 4-aligned with offsets[0] != 0, validity and Boolean bits that start inside a
    byte.  The fast path as built and with forced helping (ARK_FP_DEBUG=4), whose look-back then reads the sliced predicate
    column and offsets itself.  Subprocess: the knob is read once per process."""
    import subprocess
    import sys

    r = subprocess.run([sys.executable, "-c", _DEVICE_SLICES], capture_output=True, text=True, timeout=300, env=dict(os.environ, **env))
    assert r.returncode == 0 and "SLICES_OK" in r.stdout, r.stdout[-1500:] + r.stderr[-1500:]


def test_ragged_and_long_strings(gpu):
    rng = np.random.default_rng(3)
    n = 6000
    strs = []
    for i in range(n):
        r = rng.random()
        if r < 0.1:
            strs.append("")
        elif r < 0.97:
            strs.append("x" * int(rng.integers(1, 40)) + str(i))
        else:
            strs.append(("long%d-" % i) * int(rng.integers(500, 3000)))  # forces the global-copy fallback
    rb = pa.record_batch({"value": pa.array(rng.integers(0, 20, n), pa.int64()), "sensor": pa.array(strs),
                          "payload": pa.array([s.encode()[::-1] for s in strs], pa.binary())})
    check(rb, "SELECT sensor, payload, value FROM flow WHERE value >= 10")
    check(rb, "SELECT payload FROM flow WHERE value < 2")


def test_many_output_columns(gpu):
    rb = synth_batch(5000, key_space=9)
    q = "SELECT sensor, sensor AS s2, sensor AS s3, value, value+1, value+2, value+3, value+4, timestamp, sensor AS s4 FROM flow WHERE value >= 10"
    check(rb, q)


def test_limit(gpu):
    rb = synth_batch(5000, key_space=9)
    check(rb, "SELECT sensor, value FROM flow WHERE value >= 10 LIMIT 17")
    check(rb, "SELECT * FROM flow LIMIT 3")


def test_unknown_column_and_unsupported(gpu):
    rb = synth_batch(10)
    with pytest.raises(ArkError) as e:
        run(rb, "SELECT nope FROM flow")
    assert e.value.kind == "Process" and "No field named nope" in e.value.message
    with pytest.raises(ArkError) as e:
        SqlProcessor({"query": "SELECT value FROM flow ORDER BY value"})
    assert e.value.kind == "Unsupported"


def test_missing_config(gpu):
    with pytest.raises(ArkError) as e:
        SqlProcessor(None)
    assert e.value.kind == "Config"


def test_cast_binary_to_string_validates_utf8(gpu):
    # examples/generate_example.yaml:30 — second sql of the shipped pipeline
    rb = pa.record_batch({"__value__": pa.array([b'{"sum(flow.value)":10}', "héllo 漢".encode(), b""], pa.binary()),
                          "x": pa.array([1, 2, 3], pa.int64())})
    out = check(rb, "SELECT *,cast( __value__  as string) as y FROM flow ")
    assert out.schema.names == ["__value__", "x", "y"] and out.schema.field("y").type == pa.utf8()
    bad = pa.record_batch({"__value__": pa.array([b"ok", b"\xff\xfe", b"\xed\xa0\x80", b"\xc0\xaf", b"\xe2\x82"], pa.binary()),
                           "i": pa.array(range(5), pa.int64())})
    for q in ("SELECT cast(__value__ as string) AS y FROM flow", "SELECT cast(__value__ as string) AS y FROM flow WHERE i >= 2"):
        with pytest.raises(ArkError) as e:
            run(bad, q)
        assert e.value.kind == "Process" and "utf-8" in e.value.message.lower()
    # rows removed by the filter are not validated (FilterExec runs before the projection)
    check(bad, "SELECT cast(__value__ as string) AS y FROM flow WHERE i < 1")
