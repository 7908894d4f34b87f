"""HAVING, expressions over aggregates and LIMIT in aggregate queries on the GPU, against tests/having_oracle.py.

Every case goes through the host entry and the device entry.  Group order is unspecified, so rows are matched by key.
Values are integer-valued, so every Float64 SUM and AVG is exact and every Float64 is compared by bit pattern.  A LIMIT
result must hold min(n, G′) distinct groups, each equal to the unlimited result's row for its key.
"""
import ctypes as C
import math
import struct

import numpy as np
import pyarrow as pa
import pytest

from arkflow_b200.arrow_ffi import DeviceBatch
from arkflow_b200.dist import NativeEngine
from arkflow_b200.input import FileInput
from arkflow_b200.processor import ArkError, MessageBatch, SqlProcessor
from having_oracle import sql_process_having
from oracle.sql_oracle import OracleError
from oracle.synth import synth_batch

pytestmark = pytest.mark.gpu


def run(rb, query, device=False):
    p = SqlProcessor({"query": query})
    if device:
        out = p.process_device(DeviceBatch.from_arrow(rb))
        return None if out is None else out.to_arrow()
    r = p.process(MessageBatch.new_arrow(rb))
    return None if r.is_none() else r.batches[0].record_batch


def canon(v):
    return ("f64", struct.pack("<d", v)) if isinstance(v, float) else v


def keyed(rb, keys):
    rows = {}
    for i, row in enumerate(rb.to_pylist()):
        k = tuple(canon(row[c]) for c in keys) if keys else i
        assert k not in rows, f"duplicate group {k}"
        rows[k] = {n: canon(v) for n, v in row.items()}
    return rows


def same_result(got, want, keys, limit=None):
    assert got.schema.names == want.schema.names, (got.schema, want.schema)
    assert [f.type for f in got.schema] == [f.type for f in want.schema], (got.schema, want.schema)
    assert [f.nullable for f in got.schema] == [f.nullable for f in want.schema], (got.schema, want.schema)
    got.validate(full=True)
    g, w = keyed(got, keys), keyed(want, keys)
    if limit is None:
        assert got.num_rows == want.num_rows
        if not keys:
            assert sorted(map(repr, g.values())) == sorted(map(repr, w.values()))
        else:
            assert g == w
    else:
        assert got.num_rows == min(limit, want.num_rows)
        for k, row in g.items():
            assert row == w[k], (k, row, w[k])


def check(rb, query, keys, limit=None):
    """`limit`: the query ends in LIMIT n, and `query` without it gives the full result to compare with."""
    full = query if limit is None else query[: query.rindex(" LIMIT ")]
    want = sql_process_having(rb, full)
    if limit is not None:
        assert sql_process_having(rb, query).num_rows == min(limit, want.num_rows)
    for device in (False, True):
        same_result(run(rb, query, device), want, keys, limit)
    return want


def check_error(rb, query, kind="Process"):
    with pytest.raises(OracleError) as w:
        sql_process_having(rb, query)
    for device in (False, True):
        with pytest.raises(ArkError) as g:
            run(rb, query, device)
        assert g.value.kind == w.value.kind == kind
        if kind == "Process":
            assert g.value.message == w.value.message


def table(n=4000, seed=7, n_keys=37):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, n_keys, n)
    value = rng.integers(-50, 100, n)
    nv = pa.array(value, pa.int64(), mask=(k % 5 == 0) | (rng.random(n) < 0.1))  # all NULL in every fifth group
    return pa.record_batch({
        "sensor": pa.array([None if x == 3 else f"s{x:02d}" for x in k], pa.utf8()),
        "long_key": pa.array([f"a_sensor_name_longer_than_twelve_{x}" for x in k], pa.utf8()),
        "bin": pa.array([b"\x00\xff" + bytes([x]) for x in k], pa.binary()),
        "flag": pa.array([bool(x % 3) for x in k], pa.bool_()),
        "ikey": pa.array(k * 1000 - 7, pa.int64()),
        "value": pa.array(value, pa.int64()),
        "fvalue": pa.array(value.astype(np.float64) / 4, pa.float64()),
        "nv": nv,
    })


@pytest.mark.parametrize("query,keys", [
    ("SELECT sensor, count(*) FROM flow GROUP BY sensor HAVING count(*) > 110", ["sensor"]),
    ("SELECT sensor, count(value) FROM flow GROUP BY sensor HAVING count(nv) < 80", ["sensor"]),
    ("SELECT sensor, sum(value) FROM flow GROUP BY sensor HAVING sum(value) > 2600", ["sensor"]),
    ("SELECT sensor, avg(fvalue) FROM flow GROUP BY sensor HAVING avg(fvalue) < 6.0", ["sensor"]),
    ("SELECT sensor, min(value) FROM flow GROUP BY sensor HAVING min(value) > -50 OR max(fvalue) < 24.75", ["sensor"]),
    ("SELECT sensor FROM flow GROUP BY sensor HAVING max(value) - min(value) < 149 AND sum(fvalue) > 0", ["sensor"]),
    ("SELECT sensor, sum(nv) FROM flow GROUP BY sensor HAVING sum(nv) IS NULL", ["sensor"]),
    ("SELECT sensor, sum(nv) FROM flow GROUP BY sensor HAVING NOT (sum(nv) > 2400)", ["sensor"]),
    ("SELECT sensor, sum(value) FROM flow GROUP BY sensor HAVING sensor > 's20' OR sensor IS NULL", ["sensor"]),
    ("SELECT sensor, count(*) AS c FROM flow GROUP BY sensor HAVING c > 110", ["sensor"]),
    ("SELECT flow.sensor AS s, count(*) AS value FROM flow GROUP BY sensor HAVING value > 110 AND flow.sensor != 's01'", ["s"]),
    ("SELECT long_key, max(value) FROM flow GROUP BY long_key HAVING count(*) % 2 = 0", ["long_key"]),
    ("SELECT bin, sum(value) FROM flow GROUP BY bin HAVING sum(value) > 2500", ["bin"]),
    ("SELECT flag, count(*) FROM flow GROUP BY flag HAVING flag", ["flag"]),
    ("SELECT ikey, avg(value) FROM flow GROUP BY ikey HAVING ikey < 20000 AND avg(value) > 24", ["ikey"]),
    ("SELECT sensor, flag, count(*) FROM flow GROUP BY sensor, flag HAVING count(*) > 100 OR NOT flag", ["sensor", "flag"]),
    ("SELECT f.sensor, count(*) FROM flow AS f WHERE value > 0 GROUP BY f.sensor HAVING sum(f.value) > 3500", ["sensor"]),
])
def test_having(gpu, query, keys):
    rb = table()
    want = check(rb, query, keys)
    groups = len(set(rb.column({"s": "sensor"}.get(keys[0], keys[0])).to_pylist()))
    assert 0 < want.num_rows < groups, "HAVING should keep some groups and drop others"


def test_computed_items(gpu):
    rb = table()
    check(rb, "SELECT sensor, max(value) - min(value) AS spread, sum(value) / count(*), avg(fvalue) * 2, count(*) > 110 AS hot, "
              "-sum(fvalue), CAST(count(*) AS STRING), concat(sensor, ':', count(*)), concat(sensor, '/', flag) "
              "FROM flow GROUP BY sensor, flag", ["sensor"])  # flag is a function of sensor in table()
    check(rb, "SELECT sensor, sum(nv) + 1, max(nv) IS NULL AS empty, CAST(max(nv) - min(nv) AS DOUBLE) FROM flow GROUP BY sensor", ["sensor"])
    check(rb, "SELECT count(*) * 2, avg(value) + 1, sum(value) / count(*) FROM flow", [])


@pytest.mark.parametrize("query", [
    "SELECT value FROM flow HAVING value > 1",
    "SELECT sensor, value + 1 FROM flow GROUP BY sensor",
    "SELECT sensor FROM flow GROUP BY sensor HAVING value > 1",
    "SELECT sum(count(*)) + 1 FROM flow",
    "SELECT sensor FROM flow GROUP BY sensor HAVING max(sum(value)) > 1",
])
def test_planning_errors(gpu, query):
    check_error(table(), query)


def test_division_by_zero_in_a_computed_item(gpu):
    check_error(table(), "SELECT sensor, sum(value) / (count(*) - count(*)) FROM flow GROUP BY sensor")


def test_float_special_values(gpu):
    f = [math.nan, 1.0, -0.0, 0.0, math.inf, -2.0, -math.inf, 3.0, -0.0, math.nan, 5.0, 0.0]
    k = ["nan", "nan", "z", "z", "inf", "inf", "ninf", "ninf", "nz", "nz2", "nz2", "zero"]
    rb = pa.record_batch({"sensor": pa.array(k), "f": pa.array(f, pa.float64())})
    for h in ("max(f) > 4.0", "min(f) < -1.0", "max(f) = 0.0", "min(f) = -0.0", "avg(f) >= 0.0", "max(f) > min(f)",
              "max(f) IS NOT NULL AND avg(f) < 100.0"):
        check(rb, f"SELECT sensor, min(f), max(f), avg(f) FROM flow GROUP BY sensor HAVING {h}", ["sensor"])


def test_json_aggregates_in_having(gpu):
    docs = [f'{{"k": "d{i % 9}", "n": {i % 13}}}' for i in range(900)]
    rb = pa.record_batch({"doc": pa.array(docs)})
    check(rb, "SELECT json_get_str(doc, 'k') AS k, sum(json_get_int(doc, 'n')) FROM flow GROUP BY json_get_str(doc, 'k') "
              "HAVING sum(json_get_int(doc, 'n')) > 600", ["k"])
    check(rb, "SELECT json_get_str(doc, 'k'), count(*) FROM flow GROUP BY json_get_str(doc, 'k') "
              "HAVING json_get_str(doc, 'k') < 'd5' AND max(json_get_int(doc, 'n')) = 12", ["json_get_str(flow.doc,Utf8(\"k\"))"])


@pytest.mark.parametrize("query,rows", [
    ("SELECT count(*), sum(value) FROM flow HAVING count(*) > 0", 1),
    ("SELECT count(*), sum(value) FROM flow HAVING count(*) > 1000000", 0),
    ("SELECT count(*), sum(value) FROM flow WHERE value > 1000 HAVING count(*) = 0", 1),
    ("SELECT count(*), sum(value) FROM flow WHERE value > 1000 HAVING sum(value) IS NOT NULL", 0),
    ("SELECT sum(value) FROM flow WHERE value > 1000 HAVING sum(value) IS NULL", 1),
    ("SELECT sensor, count(*) FROM flow WHERE value > 1000 GROUP BY sensor HAVING count(*) > 0", 0),
    ("SELECT sensor, max(value) - min(value), concat(sensor, 'x') FROM flow WHERE value > 1000 GROUP BY sensor LIMIT 3", 0),
])
def test_global_and_empty(gpu, query, rows):
    rb = table()
    want = sql_process_having(rb, query)
    assert want.num_rows == rows
    for device in (False, True):
        same_result(run(rb, query, device), want, [])


@pytest.mark.parametrize("n", [0, 1, 5, 36, 37, 1000])
@pytest.mark.parametrize("having", ["", " HAVING count(*) > 100"])
def test_limit(gpu, n, having):
    rb = table()
    check(rb, f"SELECT sensor, count(*), max(value) - min(value) FROM flow GROUP BY sensor{having} LIMIT {n}", ["sensor"], limit=n)
    check(rb, f"SELECT sensor, flag, sum(value) FROM flow GROUP BY sensor, flag{having} LIMIT {n}", ["sensor", "flag"], limit=n)
    check(rb, f"SELECT count(*) FROM flow{having} LIMIT {n}", [], limit=n)


def test_million_groups_keep_one_percent(gpu):
    rng = np.random.default_rng(11)
    n = 3_000_000
    key = rng.integers(0, 1_000_000, n)
    rb = pa.record_batch({"sensor": pa.array(key, pa.int64()), "value": pa.array(rng.integers(0, 1000, n), pa.int64())})
    want = check(rb, "SELECT sensor, count(*), sum(value), max(value) - min(value) FROM flow GROUP BY sensor HAVING count(*) > 7", ["sensor"])
    assert 5_000 < want.num_rows < 20_000


def test_file_input_having_query(gpu, tmp_path):
    rb = table(n=600)
    sensors = [s or "none" for s in rb.column("sensor").to_pylist()]
    p = tmp_path / "t.csv"
    p.write_text("\n".join(["sensor,value"] + [f"{s},{v}" for s, v in zip(sensors, rb.column("value").to_pylist())]) + "\n")
    q = "SELECT sensor, count(*), max(value) - min(value) AS spread FROM flow GROUP BY sensor HAVING count(*) > 16"
    inp = FileInput({"input_type": {"type": "csv", "path": str(p)}, "query": {"query": q}})
    inp.connect()
    got = inp.read()[0].record_batch
    with pytest.raises(ArkError) as e:
        inp.read()
    assert e.value.kind == "EOF"
    csv_rb = pa.record_batch({"sensor": pa.array(sensors, pa.utf8()), "value": rb.column("value")})
    want = sql_process_having(csv_rb, q)
    assert 0 < want.num_rows
    assert keyed(got, ["sensor"]) == keyed(want, ["sensor"])


MULTI = [
    ("SELECT sensor, count(*), sum(value) FROM flow GROUP BY sensor HAVING count(*) > 28", ["sensor"]),
    ("SELECT sensor, max(value) - min(value) AS spread, sum(value) / count(*) FROM flow GROUP BY sensor HAVING avg(value) > 0", ["sensor"]),
    ("SELECT count(*) * 2, sum(value) FROM flow HAVING count(*) > 0", []),
]


def _rows(outs, keys):
    """Every rank's rows, canonical and sorted; no group on two ranks."""
    rows, seen = [], set()
    for rb in outs:
        for row in rb.to_pylist():
            k = tuple(canon(row[c]) for c in keys)
            assert k not in seen, f"group {k} on two ranks"
            seen.add(k)
            rows.append(repr({n: canon(v) for n, v in row.items()}))
    return sorted(rows)


@pytest.mark.parametrize("query,keys", MULTI)
def test_partial_final_ranks(gpu, query, keys):
    ranks, n = 3, 20_000
    shards = [synth_batch(n, row0=r * n, seed=5, key_space=1531) for r in range(ranks)]
    eng = NativeEngine(query)
    parts = []
    for r in range(ranks):
        pb, rows = eng.partial_aggregate(DeviceBatch.from_arrow(shards[r]), ranks)
        rb = pb.to_arrow()
        starts = np.concatenate([[0], np.cumsum(rows)]).tolist()
        parts.append([rb.slice(starts[i], starts[i + 1] - starts[i]) for i in range(ranks)])
    owners = [[parts[src][owner] for src in range(ranks)] for owner in range(ranks)]
    if not keys:  # a global aggregate: one final merge over every partial state
        owners = [[b for o in owners for b in o]]
    outs = []
    for received in owners:
        received = pa.Table.from_batches(received).combine_chunks()
        if received.num_rows:
            outs.append(eng.final_aggregate(DeviceBatch.from_arrow(received.to_batches()[0])).to_arrow())
    full = pa.Table.from_batches(shards).combine_chunks().to_batches()[0]
    want = sql_process_having(full, query)
    assert all(o.schema.names == want.schema.names for o in outs)
    assert _rows(outs, keys) == _rows([want], keys)


@pytest.mark.parametrize("query,keys", MULTI)
def test_push_merge_ranks(gpu, query, keys):
    from arkflow_b200.dist import ExchangeContext

    ranks, n = 3, 20_000
    ctxs = [ExchangeContext(r, ranks, 1 << 20) for r in range(ranks)]
    handles = [c.handle() for c in ctxs]
    for c in ctxs:
        c.connect(handles)
    engines = [NativeEngine(query) for _ in range(ranks)]
    shards = [synth_batch(n, row0=r * n, seed=9, key_space=1531) for r in range(ranks)]
    for r in range(ranks):
        engines[r].group_by_push(DeviceBatch.from_arrow(shards[r]), ctxs[r])
    outs = [engines[r].group_by_merge(ctxs[r]).to_arrow() for r in range(ranks)]
    for c in ctxs:
        c.close()
    full = pa.Table.from_batches(shards).combine_chunks().to_batches()[0]
    want = sql_process_having(full, query)
    assert all(o.schema.names == want.schema.names for o in outs)
    assert _rows(outs, keys) == _rows([want], keys)


def test_limit_is_refused_on_every_rank(gpu):
    from arkflow_b200.dist import ExchangeContext

    q = "SELECT sensor, count(*) FROM flow GROUP BY sensor LIMIT 5"
    shard = DeviceBatch.from_arrow(synth_batch(1000, seed=3, key_space=100))
    ranks = 2
    for r in range(ranks):
        with pytest.raises(ArkError) as e:
            NativeEngine(q).partial_aggregate(shard, ranks)
        assert e.value.kind == "Unsupported" and "LIMIT" in e.value.message
    ctxs = [ExchangeContext(r, ranks, 1 << 18) for r in range(ranks)]
    handles = [c.handle() for c in ctxs]
    for c in ctxs:
        c.connect(handles)
    for r in range(ranks):
        with pytest.raises(ArkError) as e:
            NativeEngine(q).group_by_push(shard, ctxs[r])
        assert e.value.kind == "Unsupported" and "LIMIT" in e.value.message
    for c in ctxs:
        c.close()


def launches(lib, name):
    ms, n = C.c_double(), C.c_int64()
    lib.ark_kernel_timing_get(name.encode(), C.byref(ms), C.byref(n))
    return n.value


def test_launches(gpu):
    rb = synth_batch(200_000, seed=42, key_space=10_000)
    filters = ("filter_project_kernel", "filter_project_tma_kernel")
    gpu.ark_kernel_timing_enable(1)
    try:
        for query, per_call in (("SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor", 0),
                                ("SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor HAVING count(*) > 1", 1)):
            p = SqlProcessor({"query": query})
            p.process_device(DeviceBatch.from_arrow(rb))  # binds the plan
            before = sum(launches(gpu, k) for k in filters)
            for _ in range(3):
                p.process_device(DeviceBatch.from_arrow(rb))
            assert sum(launches(gpu, k) for k in filters) - before == 3 * per_call, query
    finally:
        gpu.ark_kernel_timing_enable(0)
