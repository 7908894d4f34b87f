"""`generate` and `file` inputs on the device (csrc/inputs.cu) — the reference's own generate tests
(crates/arkflow-plugin/src/input/generate.rs:127-263) mirrored, NDJSON / CSV scans compared with the oracle and pyarrow."""
import json
import time

import numpy as np
import pyarrow as pa
import pyarrow.csv as pacsv
import pytest

from arkflow_b200.input import FileInput, GenerateInput, build_input
from arkflow_b200.processor import DEFAULT_BINARY_VALUE_FIELD, ArkError, JsonToArrowProcessor, MessageBatch
from oracle.json_oracle import json_to_arrow
from oracle.sql_oracle import sql_process

pytestmark = pytest.mark.gpu


def test_generate_basic_functionality(gpu):  # generate.rs:133-156
    inp = GenerateInput({"context": "test message", "interval": "100ms"})
    inp.connect()
    msg, _ = inp.read()
    assert len(msg) == 1 and msg.to_binary(DEFAULT_BINARY_VALUE_FIELD) == [b"test message"]
    assert not msg.record_batch.schema.field(DEFAULT_BINARY_VALUE_FIELD).nullable
    inp.close()


def test_generate_batch_size(gpu):  # generate.rs:158-179
    inp = GenerateInput({"context": "test", "interval": "100ms", "batch_size": 3})
    msg, _ = inp.read()
    assert len(msg) == 3 and msg.to_binary(DEFAULT_BINARY_VALUE_FIELD) == [b"test"] * 3


def test_generate_count_limit(gpu):  # generate.rs:181-198
    inp = GenerateInput({"context": "test", "interval": "1ms", "count": 2, "batch_size": 1})
    inp.read()
    inp.read()
    with pytest.raises(ArkError) as e:
        inp.read()
    assert e.value.kind == "EOF"


def test_generate_count_with_batch_size(gpu):  # generate.rs:200-216: the next batch would exceed count → EOF
    inp = GenerateInput({"context": "test", "interval": "1ms", "count": 3, "batch_size": 2})
    msg, _ = inp.read()
    assert len(msg) == 2
    with pytest.raises(ArkError) as e:
        inp.read()
    assert e.value.kind == "EOF"


def test_generate_interval_delay(gpu):  # generate.rs:218-238
    inp = GenerateInput({"context": "test", "interval": "100ms"})
    t0 = time.perf_counter()
    inp.read()
    assert time.perf_counter() - t0 < 0.05
    t0 = time.perf_counter()
    inp.read()
    assert time.perf_counter() - t0 >= 0.1


def test_generate_builder(gpu):  # generate.rs:240-284
    inp = build_input({"type": "generate", "context": "test", "interval": "100ms", "count": 1, "batch_size": 1})
    inp.connect()
    inp.read()
    with pytest.raises(ArkError) as e:
        inp.read()
    assert e.value.kind == "EOF"
    with pytest.raises(ArkError) as e:
        GenerateInput(None)
    assert e.value.kind == "Config" and "Generate input configuration is missing" in e.value.message
    with pytest.raises(ArkError) as e:
        GenerateInput({"context": "x"})
    assert e.value.kind == "Serialization"


def test_generate_feeds_the_decoder_on_the_device(gpu):
    """examples/generate_example.yaml's input → json_to_arrow, device-resident: 100000 clones of the 63-byte payload."""
    ctx = '{ "timestamp": 1625000000000, "value": 10, "sensor": "temp_1" }'
    inp = GenerateInput({"context": ctx, "interval": "1ns", "batch_size": 100_000, "count": 300_000})
    dec = JsonToArrowProcessor({})
    total = 0
    for _ in range(3):
        b = inp.read_device()
        out = dec.process_device(b).to_arrow()
        assert out.num_rows == 100_000 and out.schema.names == ["timestamp", "value", "sensor"]
        assert out.column("value").to_pylist()[:3] == [10, 10, 10] and out.column("sensor")[99_999].as_py() == "temp_1"
        total += out.num_rows
    with pytest.raises(ArkError):
        inp.read_device()
    assert total == 300_000


def _write_ndjson(path, n, seed=0):
    rng = np.random.default_rng(seed)
    rows = []
    with open(path, "w") as f:
        for i in range(n):
            r = {"timestamp": 1625000000000 + i, "value": int(rng.integers(0, 20)), "sensor": "temp_%d" % int(rng.integers(0, 50)),
                 "ratio": float(rng.integers(0, 1000)) / 8.0, "ok": bool(i % 3)}
            if i % 17 == 5:
                del r["ratio"]
            rows.append(r)
            f.write(json.dumps(r) + "\n")
            if i % 101 == 0:
                f.write("\n")  # blank lines are skipped
    return rows


def test_file_ndjson_scan_matches_the_json_decoder(gpu, tmp_path):
    p = str(tmp_path / "data.json")
    _write_ndjson(p, 25_000)
    inp = FileInput({"input_type": {"type": "json", "path": p}, "batch_size": 10_000})
    inp.connect()
    got = []
    while True:
        try:
            msg, _ = inp.read()
        except ArkError as e:
            assert e.kind == "EOF"
            break
        got.append(msg.record_batch)
    table = pa.Table.from_batches(got)
    assert table.num_rows == 25_000
    payloads = [ln for ln in open(p, "rb").read().split(b"\n") if ln.strip()]
    want = json_to_arrow(pa.record_batch({"__value__": pa.array(payloads, pa.binary())}))
    assert table.schema.names == want.schema.names
    for name in want.schema.names:
        assert table.column(name).combine_chunks().equals(want.column(name)), name


def test_file_ndjson_schema_is_merged_over_the_first_records(gpu, tmp_path):
    """DataFusion infers a file's schema once, over its first 1000 records: a field missing from the first record still
    becomes a column, Int64 then Float64 coerces to Float64 (checked against Arrow C++'s reader, which merges the same way)."""
    import pyarrow.json as pajson

    p = str(tmp_path / "merge.json")
    with open(p, "w") as f:
        f.write('{"a": 1, "n": 5}\n{"a": 2, "b": "x", "n": 2.5}\n{"b": "y", "c": true, "n": 7}\n')
    inp = FileInput({"input_type": {"type": "json", "path": p}})
    inp.connect()
    got = inp.read()[0].record_batch
    want = pajson.read_json(p)
    assert got.schema.names == want.schema.names == ["a", "n", "b", "c"]
    assert [str(t) for t in got.schema.types] == ["int64", "double", "string", "bool"]
    assert got.to_pylist() == want.to_pylist()


def test_file_ndjson_with_query(gpu, tmp_path):
    p = str(tmp_path / "data.json")
    _write_ndjson(p, 8_000, seed=3)
    q = "SELECT sensor, value FROM flow WHERE value >= 10"
    inp = build_input({"type": "file", "name": "f1", "input_type": {"type": "json", "path": p}, "query": {"query": q}})
    inp.connect()
    msg, _ = inp.read()
    assert msg.input_name == "f1"
    payloads = [ln for ln in open(p, "rb").read().split(b"\n") if ln.strip()]
    want = sql_process(json_to_arrow(pa.record_batch({"__value__": pa.array(payloads, pa.binary())})), q)
    assert msg.record_batch.equals(want)


def test_file_csv_scan_matches_arrow_csv(gpu, tmp_path):
    rng = np.random.default_rng(5)
    n = 30_000
    p = str(tmp_path / "data.csv")
    with open(p, "w") as f:
        f.write("id,value,score,flag,name\n")
        for i in range(n):
            name = ['plain%d' % (i % 91), '"quoted, with comma %d"' % i, '"say ""hi"" %d"' % i, ""][i % 4]
            score = "" if i % 13 == 0 else ("%.3f" % (rng.random() * 100) if i % 5 else "%de-2" % int(rng.integers(1, 999)))
            f.write("%d,%d,%s,%s,%s\n" % (i, int(rng.integers(-50, 50)), score, "true" if i % 2 else "FALSE", name))
    inp = FileInput({"input_type": {"type": "csv", "path": p}, "batch_size": 7_000})
    inp.connect()
    got = []
    while True:
        try:
            got.append(inp.read()[0].record_batch)
        except ArkError as e:
            assert e.kind == "EOF"
            break
    table = pa.Table.from_batches(got).combine_chunks()
    want = pacsv.read_csv(p, convert_options=pacsv.ConvertOptions(strings_can_be_null=True, quoted_strings_can_be_null=True))
    assert table.num_rows == n and table.schema.names == want.schema.names
    assert [str(t) for t in table.schema.types] == ["int64", "int64", "double", "bool", "string"]
    for name in ("id", "value", "flag", "name"):
        assert table.column(name).to_pylist() == want.column(name).to_pylist(), name
    g, w = table.column("score"), want.column("score")
    assert [x is None for x in g.to_pylist()] == [x is None for x in w.to_pylist()]
    assert g.fill_null(0.0).to_numpy().view(np.uint64).tolist() == w.fill_null(0.0).to_numpy().view(np.uint64).tolist()  # correctly rounded


def test_file_errors(gpu, tmp_path):
    with pytest.raises(ArkError) as e:
        FileInput(None)
    assert e.value.kind == "Config"
    with pytest.raises(ArkError) as e:
        FileInput({"input_type": {"type": "parquet", "path": "x.parquet"}})
    assert e.value.kind == "Unsupported"
    inp = FileInput({"input_type": {"type": "json", "path": str(tmp_path / "missing.json")}})
    with pytest.raises(ArkError) as e:
        inp.connect()
    assert e.value.kind == "Process" and "Read input failed" in e.value.message
    with pytest.raises(ArkError) as e:
        FileInput({"input_type": {"type": "json", "path": "x"}}).read()
    assert "Stream is None" in e.value.message  # file.rs:433-435
    bad = str(tmp_path / "bad.csv")
    open(bad, "w").write("a,b\n1,2\n3\n")
    inp = FileInput({"input_type": {"type": "csv", "path": bad}})
    inp.connect()
    with pytest.raises(ArkError) as e:
        inp.read()
    assert e.value.kind == "Process"
