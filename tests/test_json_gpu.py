"""`json_to_arrow` on the device vs the oracle (tests mirror crates/arkflow-plugin/src/processor/json.rs:160-343)."""
import json

import numpy as np
import pyarrow as pa
import pytest

from arkflow_b200.arrow_ffi import DeviceBatch
from arkflow_b200.processor import ArkError, JsonToArrowProcessor, MessageBatch, Pipeline, SqlProcessor
from oracle.json_oracle import json_to_arrow
from oracle.sql_oracle import OracleError, sql_process

pytestmark = pytest.mark.gpu


def run(mb, cfg=None, device=False):
    p = JsonToArrowProcessor(cfg or {})
    if device:
        out = p.process_device(DeviceBatch.from_arrow(mb.record_batch))
        return out.to_arrow()
    return p.process(mb).batches[0].record_batch


def check(payloads, cfg=None):
    mb = MessageBatch.new_binary(payloads)
    inc = set(cfg["fields_to_include"]) if cfg and "fields_to_include" in cfg else None
    want = json_to_arrow(mb.record_batch, (cfg or {}).get("value_field", "__value__"), inc)
    for device in (False, True):
        got = run(mb, cfg, device)
        assert sorted(got.schema.names) == sorted(want.schema.names), (got.schema, want.schema)
        assert got.num_rows == want.num_rows
        for name in want.schema.names:
            g, w = got.column(name), want.column(name)
            assert g.type == w.type, (name, g.type, w.type)
            assert g.to_pylist() == w.to_pylist(), name
            if g.type == pa.float64():  # and the bits: -0.0 == 0.0 in Python
                assert g.fill_null(0.0).to_numpy().view(np.uint64).tolist() == w.fill_null(0.0).to_numpy().view(np.uint64).tolist(), name
    return want


def test_generate_example_payloads(gpu):
    # examples/generate_example.yaml:6
    out = check([b'{ "timestamp": 1625000000000, "value": 10, "sensor": "temp_1" }'] * 10)
    assert out.schema.names == ["timestamp", "value", "sensor"]
    assert [str(t) for t in out.schema.types] == ["int64", "int64", "string"]


def test_basic_types_scalar_fields(gpu):
    # json.rs:170-207, scalar fields (the full record: test_reference_basic_types_record_with_array_and_object)
    rec = {"null_field": None, "bool_field": True, "int_field": 42, "uint_field": 18446744073709551615, "float_field": 3.14, "string_field": "hello"}
    out = check([json.dumps(rec).encode()])
    assert out.num_rows == 1 and out.num_columns == 6
    assert [str(t) for t in out.schema.types] == ["null", "bool", "int64", "double", "double", "string"]


def test_field_filtering(gpu):
    # json.rs:209-243
    rec = {"a": 1, "b": "x", "c": 2.5, "d": [1, 2], "e": {"k": 1}}
    out = check([json.dumps(rec).encode()], {"fields_to_include": ["a", "c"]})
    assert sorted(out.schema.names) == ["a", "c"]


def test_invalid_input_is_error(gpu):
    # json.rs:245-266
    with pytest.raises(ArkError) as e:
        run(MessageBatch.new_binary([b"not a json object"]))
    assert e.value.kind == "Process"
    with pytest.raises(OracleError):
        json_to_arrow(MessageBatch.new_binary([b"not a json object"]).record_batch)


def test_missing_config_and_wrong_column(gpu):
    with pytest.raises(ArkError) as e:
        JsonToArrowProcessor(None)
    assert e.value.kind == "Config"
    with pytest.raises(ArkError) as e:
        run(MessageBatch.new_arrow(pa.record_batch({"x": pa.array([1], pa.int64())})))
    assert e.value.message == "not found column"
    with pytest.raises(ArkError) as e:
        run(MessageBatch.new_arrow(pa.record_batch({"__value__": pa.array(["{}"])})))
    assert e.value.message == "not support data type"


def check_nested(payloads, cfg=None, monkeypatch=None):
    """Host entry point only (the Python DeviceBatch mirror materialises flat columns); oracle in NESTED mode."""
    import oracle.json_oracle as jo

    monkeypatch.setattr(jo, "NESTED", True)
    mb = MessageBatch.new_binary(payloads)
    want = jo.json_to_arrow(mb.record_batch)
    got = run(mb, cfg, False)
    assert got.schema.names == want.schema.names
    assert got.num_rows == want.num_rows
    for name in want.schema.names:
        g, w = got.column(name), want.column(name)
        assert g.type == w.type, (name, g.type, w.type)
        assert g.to_pylist() == w.to_pylist(), name
    return got


def test_reference_basic_types_record_with_array_and_object(gpu, monkeypatch):
    # crates/arkflow-plugin/src/processor/json.rs:170-207, the record as the reference's own test builds it
    rec = {"null_field": None, "bool_field": True, "int_field": 42, "uint_field": 18446744073709551615, "float_field": 3.14,
           "string_field": "hello", "array_field": [1, 2, 3], "object_field": {"key": "value"}}
    import oracle.json_oracle as jo

    monkeypatch.setattr(jo, "NESTED", True)
    mb = MessageBatch.new_binary([json.dumps(rec).encode()])
    got = run(mb)
    assert got.num_rows == 1  # what the reference asserts
    assert got.column("array_field").to_pylist() == [[1, 2, 3]] and got.column("object_field").to_pylist() == [{"key": "value"}]
    assert str(got.schema.field("array_field").type) == "list<item: int64>" and str(got.schema.field("object_field").type) == "struct<key: string>"


def test_nested_lists_and_structs_vs_oracle(gpu, monkeypatch):
    rng = np.random.default_rng(3)
    payloads = []
    for i in range(3000):
        rec = {"id": i, "tags": ["t%d" % int(x) for x in rng.integers(0, 9, int(rng.integers(0, 5)))],
               "nums": [int(x) for x in rng.integers(-5, 5, int(rng.integers(0, 4)))],
               "ratios": [float(x) / 4 for x in rng.integers(0, 99, int(rng.integers(1, 3)))],
               "pos": {"x": float(i) / 8, "y": int(rng.integers(0, 100)), "label": "p\"%d" % i, "ok": bool(i & 1)},
               "flags": [bool(x) for x in rng.integers(0, 2, 2)]}
        if i % 7 == 3:
            rec["tags"] = None
        if i % 11 == 5:
            del rec["pos"]
        if i % 13 == 6:
            rec["pos"] = {"y": "17", "extra": [1, {"deep": 2}]}  # missing children → NULL, quoted number, ignored key
        if i % 17 == 8:
            rec["nums"] = [1, None, "3"]
        if i == 0:
            rec["ratios"] = [1, 2.5]  # Int64 + Float64 in the first record → List<Float64>
        payloads.append(json.dumps(rec).encode())
    got = check_nested(payloads, monkeypatch=monkeypatch)
    assert str(got.schema.field("ratios").type) == "list<item: double>"


def test_nested_edge_cases(gpu, monkeypatch):
    got = check_nested([b'{"a": [], "s": {}, "n": 1}', b'{"a": [null, null], "s": {}, "n": 2}', b'{"n": 3}'], monkeypatch=monkeypatch)
    assert str(got.schema.field("a").type) == "list<item: null>"
    # a scalar where the first record had an array / object is a type error, as in arrow-json
    for bad in (b'{"a": 5}', b'{"s": "x"}'):
        with pytest.raises(ArkError) as e:
            run(MessageBatch.new_binary([b'{"a": [1], "s": {"k": 1}}', bad]))
        assert e.value.kind == "Process"
    # two levels of nesting stay outside the subset
    for deep in (b'{"a": [[1]]}', b'{"a": [{"k": 1}]}', b'{"s": {"t": {"u": 1}}}', b'{"s": {"t": [1]}}', b'{"a": [1, "x"]}'):
        with pytest.raises(ArkError) as e:
            run(MessageBatch.new_binary([deep]))
        assert e.value.kind == "Unsupported"


def test_wide_records_and_long_field_names(gpu):
    """More than 16 top-level keys and names longer than 48 bytes (the r1 limits of the parameter-block field table)."""
    long_name = "a_field_name_that_is_considerably_longer_than_forty_eight_bytes_in_total"
    recs = []
    for i in range(500):
        r = {"k%02d" % c: i * c for c in range(40)}
        r[long_name] = "v%d" % i
        r["\u00e9t\u00e9"] = i  # a key that needs no escape once serialised as UTF-8
        recs.append(r)
    out = check([json.dumps(r, ensure_ascii=False).encode() for r in recs])
    assert out.num_columns == 42 and out.column(long_name)[499].as_py() == "v499"
    with pytest.raises(ArkError) as e:
        run(MessageBatch.new_binary([json.dumps({"c%d" % c: c for c in range(65)}).encode()]))
    assert e.value.kind == "Unsupported"


def test_keys_written_with_escapes(gpu):
    """A record may spell a key with escapes ("val\\u0075e", "sens\\/or" …): arrow-json's tape decoder compares decoded names, so
    such a key fills its column like any other (ADVICE r1: they used to be treated as unknown keys and dropped)."""
    payloads = [
        b'{"value": 1, "sensor": "a", "t/s": 5, "\\u00e9t\\u00e9": 7}',
        b'{"val\\u0075e": 2, "sens\\u006fr": "b", "t\\/s": 6, "\\u00e9t\\u00E9": 8}',
        b'{"\\u0076alue": 3, "sensor": "c", "val\\u0075": 99, "\\ud83d\\ude00": 1}',   # unknown escaped keys are skipped
        b'{"valu\\u0065": "4", "t\\u002fs": null}',
    ]
    out = check(payloads)
    assert out.column("value").to_pylist() == [1, 2, 3, 4]
    assert out.column("sensor").to_pylist() == ["a", "b", "c", None]
    assert out.column("t/s").to_pylist() == [5, 6, None, None]
    assert out.column("\u00e9t\u00e9").to_pylist() == [7, 8, None, None]


def test_non_strict_decoding(gpu):
    payloads = [
        b'{"timestamp": 1, "value": 10, "sensor": "a", "flag": true}',
        b'{"value": 11.9, "sensor": "b", "extra": {"deep": [1, {"x": "}"}]}, "timestamp": 2}',  # reordered, extra nested key, float into Int64
        b'{"timestamp": "3", "value": "12", "sensor": null}',                                     # quoted numbers, null, missing flag
        b'  {"sensor":"c" , "value":-7e2,"timestamp":4.0e0, "flag": false, "unknown": "x\\"y"}  ',
        b'{}',
    ]
    out = check(payloads)
    assert out.column("value").to_pylist() == [10, 11, 12, -700, None]


def test_string_escapes_and_unicode(gpu):
    strs = ["plain", "", 'quote"inside', "back\\slash", "nl\nnl\ttab", "unicode é ü 漢字 \U0001F600", "ctrl", "/slash"]
    payloads = [json.dumps({"s": s, "i": i}).encode() for i, s in enumerate(strs)]          # ensure_ascii: \uXXXX escapes + surrogate pairs
    payloads += [json.dumps({"s": s, "i": i}, ensure_ascii=False).encode() for i, s in enumerate(strs)]  # raw UTF-8
    out = check(payloads)
    assert out.column("s").to_pylist() == strs + strs


def test_numbers(gpu):
    ints = [0, -1, 1, 9223372036854775807, -9223372036854775808, 1234567890123, 10]
    floats = ["0.5", "-0.0", "3.14", "1e3", "2.5E-3", "123456789.125", "1e22", "9007199254740991", "0.1", "100"]
    payloads = [json.dumps({"i": 1, "f": 1.5}).encode()]
    payloads += [b'{"i": %d, "f": %s}' % (i, f.encode()) for i, f in zip(ints + ints, floats + floats)]
    check(payloads)
    # beyond Clinger's fast path: still correctly rounded (tests/test_number_parse_gpu.py covers the whole range)
    hard = [b'{"f": 1.5}', b'{"f": 1.7976931348623157e308}', b'{"f": 123456789012345678901234567890}', b'{"f": 4.9e-324}', b'{"f": 0.30000000000000004}',
            b'{"f": 3.246986519402559e+185}', b'{"f": 2.2250738585072011e-308}', b'{"f": -0.0}']
    check(hard)


def test_int_column_errors(gpu):
    with pytest.raises(ArkError):
        run(MessageBatch.new_binary([b'{"i": 1}', b'{"i": true}']))
    with pytest.raises(ArkError):
        run(MessageBatch.new_binary([b'{"i": 1}', b'{"i": 1e30}']))
    with pytest.raises(ArkError):
        run(MessageBatch.new_binary([b'{"s": "x"}', b'{"s": 5}']))
    with pytest.raises(ArkError):
        run(MessageBatch.new_binary([b'{"i": 1}', b'{"i": 1']))
    with pytest.raises(ArkError):
        run(MessageBatch.new_binary([b'{"i": 1}', b'[1,2]']))


def test_multiple_records_per_payload_and_null_payloads(gpu):
    rb = pa.record_batch([pa.array([b'{"a":1}\n{"a":2} {"a":3}', None, b"", b'{"a":4}', b"  \n "], pa.binary())], names=["__value__"])
    mb = MessageBatch.new_arrow(rb)
    want = json_to_arrow(rb)
    assert want.column("a").to_pylist() == [1, 2, 3, 4]
    for device in (False, True):
        got = run(mb, None, device)
        assert got.column("a").to_pylist() == [1, 2, 3, 4]


def test_empty_inputs(gpu):
    rb = pa.record_batch([pa.array([], pa.binary())], names=["__value__"])
    out = run(MessageBatch.new_arrow(rb))
    assert out.num_rows == 0 and out.num_columns == 0
    assert json_to_arrow(rb).num_columns == 0


def test_custom_value_field(gpu):
    rb = pa.record_batch({"payload": pa.array([b'{"x": 1}', b'{"x": 2}'], pa.binary()), "other": pa.array([1, 2], pa.int64())})
    out = JsonToArrowProcessor({"value_field": "payload"}).process(MessageBatch.new_arrow(rb)).batches[0].record_batch
    assert out.column("x").to_pylist() == [1, 2]


def test_large_batch_and_pipeline_into_sql(gpu):
    rng = np.random.default_rng(0)
    n = 200_000
    vals = rng.integers(0, 20, n)
    keys = rng.integers(0, 100, n)
    payloads = [b'{ "timestamp": %d, "value": %d, "sensor": "temp_%d" }' % (1625000000000 + 1000 * i, v, k) for i, (v, k) in enumerate(zip(vals, keys))]
    mb = MessageBatch.new_binary(payloads)
    want = check(payloads)
    # README quick-start pipeline: json_to_arrow -> sql (README.md:58-79)
    pipe = Pipeline([JsonToArrowProcessor({}), SqlProcessor({"query": "SELECT * FROM flow WHERE value >= 10"})])
    got = pipe.process(mb).batches[0].record_batch
    assert got.equals(sql_process(want, "SELECT * FROM flow WHERE value >= 10"))
