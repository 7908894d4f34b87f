"""The JSON path functions on the device (csrc/json_path.cu) against the oracle (tests/json_path_oracle.py): whole
batches, through process and process_device, floats compared bit for bit."""
import ctypes as C
import json
import random

import numpy as np
import pyarrow as pa
import pyarrow.ipc as ipc
import pytest

from arkflow_b200.arrow_ffi import DeviceBatch
from arkflow_b200.input import FileInput, GenerateInput
from arkflow_b200.processor import DEFAULT_BINARY_VALUE_FIELD, ArkError, MessageBatch, SqlProcessor
from json_path_oracle import sql_process_json

pytestmark = pytest.mark.gpu

FUNCS = ["json_get_str", "json_get_int", "json_get_float", "json_get_bool", "json_get_json", "json_as_text",
         "json_contains", "json_length"]

# every value kind, escapes, surrogate pairs, whitespace, duplicate keys, brackets and quotes inside strings, deep
# paths, integer limits, float bit patterns, truncated and malformed documents
DOCS = [
    '{"a":"x","b":1,"c":1.5,"d":true,"e":null,"f":[1,"two",{"g":3}],"h":{"i":{"j":"k"}}}',
    '{"a":"esc\\"aped\\\\ \\u00e9 \\ud83d\\ude00 \\n","b":-9223372036854775808,"c":-0,"d":false}',
    '{"a":7,"b":9223372036854775807,"c":9223372036854775808,"d":"true"}',
    '{"b":9223372036854775808,"c":1e400,"a":[],"f":{}}',
    ' \t\r\n{ "a" : "]}\\"[{" ,\n "b" : [ 1 , [ 2 , 3 ] ] , "c" : -0.0 } ',
    '{"a":1,"a":2,"b":{"x":1},"b":{"y":2}}',
    '{"k\\u0065y":"v","a":"\\ud83d"}',
    '{"a":"unterminated',
    '{"a":1,"b":',
    '{"a":1}trailing',
    '{"a":12x,"b":2}',
    '{"b":[1,],"a":1}',
    '{"b":01,"a":1}',
    '[10,20,{"a":[30,31]}]',
    '"just a string"',
    '4.9406564584124654e-324',
    '0.1',
    '123456789012345678901234567890',
    '2.2250738585072011e-308',
    '1.7976931348623157e308',
    '-1.5e-7',
    '{"a":{"b":{"c":{"d":{"e":{"f":{"g":{"h":[1,2,3]}}}}}}}}',
    '',
    '{}',
    '[]',
    'nul',
    '{"a":tru}',
]
PATHS = [[], ["a"], ["b"], ["c"], ["d"], ["f", 2, "g"], ["h", "i", "j"], ["key"], [1], [2, "a", 1], ["b", 1, 0],
         list("abcdefgh"), [5]]


def _lit(p):
    return f"'{p}'" if isinstance(p, str) else str(p)


def call(fn, path, doc="doc"):
    return f"{fn}({', '.join([doc] + [_lit(p) for p in path])})"


def run(rb, query, device):
    p = SqlProcessor({"query": query})
    if device:
        out = p.process_device(DeviceBatch.from_arrow(rb))
        return None if out is None else out.to_arrow()
    r = p.process(MessageBatch.new_arrow(rb))
    return None if r.is_none() else r.batches[0].record_batch


def same(g: pa.Array, w: pa.Array) -> bool:
    if pa.types.is_floating(w.type):
        if not g.is_valid().equals(w.is_valid()):
            return False
        gb, wb = (x.fill_null(0.0).to_numpy(zero_copy_only=False).view(np.uint64) for x in (g, w))
        return np.array_equal(gb, wb)
    return g.equals(w)


def check(rb, query, unordered=False):
    want = sql_process_json(rb, query)
    for device in (False, True):
        got = run(rb, query, device)
        if want is None:
            assert got is None
            continue
        assert got.schema.names == want.schema.names, (got.schema, want.schema)
        assert [f.type for f in got.schema] == [f.type for f in want.schema], (got.schema, want.schema)
        assert got.num_rows == want.num_rows, (query, device)
        if unordered:
            key = lambda b: sorted(zip(*[c.to_pylist() for c in b.columns]), key=repr)
            assert key(got) == key(want), (query, device)
            continue
        for name, g, w in zip(got.schema.names, got.columns, want.columns):
            assert same(g, w), f"column {name} differs (device={device}) for {query}"
    return want


def launches(lib, name):
    ms, n = C.c_double(), C.c_int64()
    lib.ark_kernel_timing_get(name.encode(), C.byref(ms), C.byref(n))
    return n.value


@pytest.fixture
def timing(gpu):
    gpu.ark_kernel_timing_enable(1)
    gpu.ark_kernel_timing_reset()
    yield gpu
    gpu.ark_kernel_timing_enable(0)


@pytest.mark.parametrize("fn", FUNCS)
def test_each_function_over_every_kind(gpu, fn):
    rb = pa.record_batch({"doc": pa.array(DOCS + [None])})
    for k in range(0, len(PATHS), 8):  # eight calls per query: one launch each
        check(rb, "SELECT " + ", ".join(call(fn, p) for p in PATHS[k:k + 8]) + " FROM flow")


def test_many_calls_on_one_column_share_one_scan(timing):
    rb = pa.record_batch({"doc": pa.array(DOCS * 10), "n": pa.array(range(len(DOCS) * 10))})
    q = "SELECT n, json_get_str(doc,'a'), json_get_int(doc,'b'), json_get_float(doc,'c') FROM flow"
    check(rb, q)
    assert launches(timing, "json_path_kernel") == 2  # one per route
    timing.ark_kernel_timing_reset()
    q = "SELECT " + ", ".join(call(f, p) for f in FUNCS[:5] for p in PATHS[:2]) + " FROM flow"  # 10 calls: 8 + 2
    check(rb, q)
    assert launches(timing, "json_path_kernel") == 2 * 2


def test_null_documents_at_warp_and_cta_edges_and_sliced_inputs(gpu):
    rng = random.Random(5)
    docs = [None if i in (0, 31, 32, 127, 128, 255, 256, 511) or rng.random() < 0.1 else rng.choice(DOCS) for i in range(700)]
    rb = pa.record_batch({"doc": pa.array(docs), "n": pa.array(range(700))})
    q = "SELECT n, json_get_str(doc,'a'), json_get_int(doc,'b'), json_length(doc), json_contains(doc,'c') FROM flow"
    check(rb, q)
    for off in (1, 3, 33, 130):  # a non-zero validity bit offset and offsets that do not start at 0
        check(rb.slice(off, 500), q)


def test_empty_batch_is_none(gpu):
    rb = pa.record_batch({"doc": pa.array([], pa.string())})
    assert run(rb, "SELECT json_get_int(doc,'a') FROM flow", False) is None
    assert run(rb, "SELECT json_get_int(doc,'a') FROM flow", True) is None


def test_documents_from_two_bytes_to_over_64_kib(gpu):
    big = {"pad": "x" * 70000, "arr": list(range(5000)), "a": "end \\u00e9"}
    docs = ["{}", "[]", '{"a":"short"}', json.dumps(big), json.dumps({"arr": [big] * 2, "a": 1}), json.dumps(big)[:-5]]
    rb = pa.record_batch({"doc": pa.array(docs)})
    assert len(docs[3]) > 65536
    check(rb, "SELECT json_get_str(doc,'a'), json_length(doc,'arr'), json_get_int(doc,'arr',4999), json_get_json(doc,'a'), "
              "json_as_text(doc,'arr',1,'a') FROM flow")


def test_expressions_where_limit_and_cast(gpu):
    rng = random.Random(7)
    docs = [json.dumps({"t": rng.randrange(-1000, 1000), "v": rng.uniform(-5, 5), "s": rng.choice("abc")}) for _ in range(3000)]
    rb = pa.record_batch({"doc": pa.array(docs), "n": pa.array(range(3000))})
    check(rb, "SELECT n, json_get_int(doc,'t') * 2 + 1 AS t2, json_get_float(doc,'v') > 0.5, json_get_int(doc,'x') IS NULL, "
              "CAST(json_get_int(doc,'t') AS DOUBLE) FROM flow")
    check(rb, "SELECT n, json_get_str(doc,'s') FROM flow WHERE json_get_int(doc,'t') > 100 LIMIT 17")
    check(rb, "SELECT json_get_float(doc,'v') FROM flow WHERE json_get_str(doc,'s') = 'b' AND json_get_int(doc,'t') < 0")


def test_group_by_a_json_key_with_aggregates_of_json_values(gpu):
    rng = random.Random(11)
    docs = [None if rng.random() < 0.02 else json.dumps({"sensor": f"s{rng.randrange(50)}", "value": rng.randrange(-100, 100) / 4,
                                                          "n": rng.randrange(10)}) for _ in range(20000)]
    rb = pa.record_batch({"doc": pa.array(docs)})
    check(rb, "SELECT json_get_str(doc,'sensor'), count(*), avg(json_get_float(doc,'value')), sum(json_get_int(doc,'n')), "
              "max(json_get_int(doc,'n')) FROM flow GROUP BY json_get_str(doc,'sensor')", unordered=True)
    check(rb, "SELECT count(*), sum(json_get_float(doc,'value')) FROM flow WHERE json_contains(doc,'sensor')", unordered=True)


def test_generate_value_cast_to_string(gpu):
    inp = GenerateInput({"context": '{"timestamp": 1625000000000, "value": 10, "sensor": "temp_1"}', "interval": "1ms",
                         "batch_size": 1000})
    inp.connect()
    msg, _ = inp.read()
    inp.close()
    rb = msg.record_batch
    q = (f"SELECT json_get_str(cast({DEFAULT_BINARY_VALUE_FIELD} as string), 'sensor') AS sensor, "
         f"json_get_float(cast({DEFAULT_BINARY_VALUE_FIELD} as string), 'value') FROM flow")
    out = check(rb, q)
    assert out.column(0).to_pylist() == ["temp_1"] * 1000


def test_cast_of_invalid_utf8_fails_as_the_cast_does(gpu):
    rb = pa.record_batch({"b": pa.array([b'{"a":1}', b'{"a":"\xff"}'])})
    with pytest.raises(ArkError) as e:
        run(rb, "SELECT json_get_int(cast(b as string), 'a') FROM flow", False)
    assert e.value.kind == "Process" and "Cannot cast binary to string" in e.value.message


def test_file_input_query_over_arrow_ipc(gpu, tmp_path):
    docs = [json.dumps({"id": i, "tag": f"t{i % 3}"}) if i % 7 else None for i in range(500)]
    rb = pa.record_batch({"doc": pa.array(docs), "k": pa.array(range(500))})
    p = tmp_path / "j.arrow"
    with ipc.new_file(str(p), rb.schema) as w:
        w.write_batch(rb)
    q = "SELECT k, json_get_int(doc,'id'), json_get_str(doc,'tag') FROM flow WHERE json_get_int(doc,'id') % 2 = 0"
    inp = FileInput({"input_type": {"type": "arrow", "path": str(p)}, "query": {"query": q}})
    inp.connect()
    got = []
    try:
        while True:
            got.append(inp.read()[0].record_batch)
    except ArkError as e:
        assert e.kind == "EOF", e.message
    want = sql_process_json(rb, q)
    got = pa.Table.from_batches(got).combine_chunks().to_batches()[0]
    assert got.schema.names == want.schema.names and got.equals(want)


def test_large_batch(gpu):
    # 2^22 generate-style documents; the expected columns come straight from the values the documents were printed from
    n = 1 << 22
    rng = np.random.default_rng(1)
    ts, vals = rng.integers(0, 10**12, n).tolist(), rng.integers(0, 10000, n).tolist()
    rb = pa.record_batch({"doc": pa.array([f'{{"timestamp":{t},"value":{v / 100},"sensor":"s{v % 97}"}}' for t, v in zip(ts, vals)])})
    keep = [k for k in range(n) if ts[k] > 500000000000]
    sensor, value = 'json_get_str(flow.doc,Utf8("sensor"))', 'json_get_float(flow.doc,Utf8("value"))'
    want = pa.record_batch({sensor: pa.array([f"s{vals[k] % 97}" for k in keep]), value: pa.array([vals[k] / 100 for k in keep], pa.float64())})
    q = "SELECT json_get_str(doc,'sensor'), json_get_float(doc,'value') FROM flow WHERE json_get_int(doc,'timestamp') > 500000000000"
    for device in (False, True):
        got = run(rb, q, device)
        assert got.schema.names == want.schema.names and got.num_rows == want.num_rows
        assert got.column(0).equals(want.column(0)) and same(got.column(1), want.column(1)), device


def test_join_queries_keep_todays_errors(gpu):
    rb = pa.record_batch({"doc": pa.array(['{"a":1}']), "k": pa.array([1])})
    p = SqlProcessor({"query": "SELECT json_get_int(doc, 'a') FROM flow"})
    with pytest.raises(ArkError) as e:
        p.process_tables({"flow": rb, "other": rb})
    assert e.value.kind == "Unsupported" and "scalar function json_get_int()" in e.value.message
    p = SqlProcessor({"query": "SELECT json_get_int(a.doc, 'a') FROM flow a JOIN other b ON a.k = b.k"})
    with pytest.raises(ArkError) as e:
        p.process_tables({"flow": rb, "other": rb})
    assert e.value.kind == "Unsupported"
