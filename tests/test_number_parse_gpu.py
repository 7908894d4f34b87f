"""Decimal → double on the device, bit for bit against correctly rounded conversion (Python's float()).

Every decoder that reads a Float64 from text goes through csrc/decimal.cuh: json_to_arrow (one and several records per
payload, host and device entry points), List<Float64> elements, and the NDJSON and CSV `file` inputs.  Each sees the
whole corpus of tests/number_corpus.py, with no tolerance.  Int64 columns are checked at the edges of the i64 range.
"""
import numpy as np
import pyarrow as pa
import pyarrow.csv as pacsv
import pytest

import number_corpus as NC
from arkflow_b200.arrow_ffi import DeviceBatch
from arkflow_b200.input import FileInput
from arkflow_b200.processor import ArkError, ArrowToJsonProcessor, JsonToArrowProcessor, MessageBatch
from oracle.json_oracle import json_to_arrow
from oracle.sql_oracle import OracleError

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def corpus():
    c = NC.corpus()
    flat = [s for strs in c.values() for s in strs]
    cls = np.array([k for k, strs in c.items() for _ in strs])
    want = np.array([float(s) for s in flat], np.float64)
    return flat, cls, want


def assert_bits(got, want, strs, cls):
    got = np.asarray(got, np.float64)
    assert got.shape == want.shape
    wrong = np.nonzero(got.view(np.uint64) != want.view(np.uint64))[0]
    if len(wrong):
        per = {str(k): int(n) for k, n in zip(*np.unique(cls[wrong], return_counts=True))}
        ex = [(strs[i][:80], float(got[i]).hex(), float(want[i]).hex()) for i in wrong[:5]]
        pytest.fail(f"{len(wrong)} of {len(want)} values differ in their bits; by class {per}; e.g. {ex}")


def values(col):
    assert col.null_count == 0 and col.type == pa.float64(), col.type
    return col.to_numpy(zero_copy_only=False)


def read_all(inp):
    inp.connect()
    out = []
    while True:
        try:
            out.append(inp.read()[0].record_batch)
        except ArkError as e:
            assert e.kind == "EOF"
            return pa.Table.from_batches(out)


@pytest.mark.parametrize("per_payload", [1, 7])
@pytest.mark.parametrize("device", [False, True])
def test_json_to_arrow_float64(gpu, corpus, per_payload, device):
    """MODE 2 (one record per payload) and MODE 1 (several); 0.5 first so that the column is Float64."""
    strs, cls, want = corpus
    recs = [b'{"f": 0.5}'] + [b'{"f": %s}' % s.encode() for s in strs]
    payloads = [b"\n".join(recs[i:i + per_payload]) for i in range(0, len(recs), per_payload)]
    mb = MessageBatch.new_binary(payloads)
    p = JsonToArrowProcessor({})
    rb = p.process_device(DeviceBatch.from_arrow(mb.record_batch)).to_arrow() if device else p.process(mb).batches[0].record_batch
    assert rb.schema.names == ["f"] and rb.num_rows == len(recs)
    assert_bits(values(rb.column("f"))[1:], want, strs, cls)


def test_json_list_float64_elements(gpu, corpus):
    strs, cls, want = corpus
    payloads = [b'{"l": [0.5]}'] + [b'{"l": [%s]}' % ", ".join(strs[i:i + 16]).encode() for i in range(0, len(strs), 16)]
    rb = JsonToArrowProcessor({}).process(MessageBatch.new_binary(payloads)).batches[0].record_batch
    col = rb.column("l")
    assert col.type == pa.list_(pa.float64())
    assert_bits(values(col.flatten())[1:], want, strs, cls)


def test_file_ndjson(gpu, corpus, tmp_path):
    strs, cls, want = corpus
    p = tmp_path / "numbers.json"
    p.write_text('{"f": 0.5}\n' + "".join('{"f": %s}\n' % s for s in strs))
    t = read_all(FileInput({"input_type": {"type": "json", "path": str(p)}, "batch_size": 300_000}))
    assert t.schema.names == ["f"]
    assert_bits(values(t.column("f").combine_chunks())[1:], want, strs, cls)


def test_file_csv(gpu, corpus, tmp_path):
    strs, cls, want = corpus
    p = tmp_path / "numbers.csv"
    p.write_text("f,g\n0.5,0.5\n" + "".join("%s,%s\n" % (s, t) for s, t in zip(strs, reversed(strs))))
    t = read_all(FileInput({"input_type": {"type": "csv", "path": str(p)}, "batch_size": 300_000}))
    assert t.schema.names == ["f", "g"]
    assert_bits(values(t.column("f").combine_chunks())[1:], want, strs, cls)
    assert_bits(values(t.column("g").combine_chunks())[1:], want[::-1], strs[::-1], cls[::-1])


@pytest.fixture(scope="module")
def round_trip_batch():
    import random

    rng = random.Random(7)
    xs = [0.5, 0.0, -0.0, 5e-324, -5e-324, 2.2250738585072014e-308, 2.225073858507201e-308, 1.7976931348623157e308, -1.7976931348623157e308]
    xs += NC.random_doubles(rng, 1_000_000)
    return pa.record_batch({"f": pa.array(xs, pa.float64())})


def test_round_trip_through_arrow_to_json_host(gpu, round_trip_batch):
    rb = round_trip_batch
    lines = ArrowToJsonProcessor({}).process(MessageBatch.new_arrow(rb)).batches[0].record_batch
    back = JsonToArrowProcessor({}).process(MessageBatch.new_arrow(lines)).batches[0].record_batch
    want = values(rb.column("f"))
    assert_bits(values(back.column("f")), want, [str(x) for x in want], np.array(["round trip"] * len(want)))


def test_round_trip_through_arrow_to_json_device(gpu, round_trip_batch):
    rb = round_trip_batch
    cur = DeviceBatch.from_arrow(rb)
    for st in (ArrowToJsonProcessor({}), JsonToArrowProcessor({})):
        cur = st.process_device(cur)
    want = values(rb.column("f"))
    assert_bits(values(cur.to_arrow().column("f")), want, [str(x) for x in want], np.array(["round trip"] * len(want)))


INT64_LITERALS = [
    "9223372036854775807", "-9223372036854775807", "-9223372036854775808", "9223372036854775808", "-9223372036854775809",
    "18446744073709551615", "18446744073709551616", "-18446744073709551616",
    "1234567890123456789", "-1234567890123456789", "12345678901234567890", "-12345678901234567890",
    "1234567890123456789012345", "-1234567890123456789012345", "0", "-0",
    "1e18", "-1e18", "1e19", "1.5", "-1.5", "0.999999999999999999999", "-0.5", "1E3", "2.5e-3", "1e-400", "-0.0",
    "9.2233720368547748e18", "-9.2233720368547748e18", "9.223372036854775807e18", "9.2233720368547758e18",
    "-9.223372036854775808e18", "-9.2233720368547758e18", "-9.223372036854776e18", "-9.2233720368547778e18",
    "-9.223372036854777856e18", "-9.2233720368547778559e18", "123456789012345678.9", "9007199254740993.5",
    "1.8446744073709551615e19", "1e400", "-1e400",
]


@pytest.mark.parametrize("lit", INT64_LITERALS)
def test_json_int64_edges_match_the_oracle(gpu, lit):
    for text in (lit, '"%s"' % lit):  # a quoted number is accepted for numeric columns
        rb = MessageBatch.new_binary([b'{"i": 1}', b'{"i": %s}' % text.encode()]).record_batch
        try:
            want, err = json_to_arrow(rb).column("i").to_pylist(), None
        except OracleError as e:
            want, err = None, e.kind
        for device in (False, True):
            p = JsonToArrowProcessor({})
            try:
                got = (p.process_device(DeviceBatch.from_arrow(rb)).to_arrow() if device else p.process(MessageBatch.new_arrow(rb)).batches[0].record_batch)
                got, gerr = got.column("i").to_pylist(), None
            except ArkError as e:
                got, gerr = None, e.kind
            assert (got, gerr) == (want, err), (text, device)


def test_csv_int64_edges_match_pyarrow(gpu, tmp_path):
    p = tmp_path / "ints.csv"
    p.write_text("a,b\n1,-9223372036854775808\n9223372036854775807,-9223372036854775808\n-9223372036854775807,-9223372036854775808\n"
                 "-9223372036854775808,-9223372036854775808\n")
    got = read_all(FileInput({"input_type": {"type": "csv", "path": str(p)}}))
    want = pacsv.read_csv(str(p))
    assert [str(t) for t in got.schema.types] == [str(t) for t in want.schema.types] == ["int64", "int64"]
    assert got.to_pylist() == want.to_pylist()


# spelling → the type the CSV input infers for a column holding only it
CSV_SPELLINGS = {
    "-9223372036854775808": "int64", "+9223372036854775807": "int64", "0005": "int64", "9223372036854775808": "double",
    "-9223372036854775809": "double", "100000000000000000000000": "double",
    "1.": "double", ".5": "double", "-.5e-3": "double", "+1.5E+3": "double", "1e400": "double", "0e999999": "double",
    "inf": "double", "-Inf": "double", "+INF": "double", "infinity": "double", "-Infinity": "double", "nan": "double", "-NaN": "double",
    "0x1p3": "string", "0x10": "string", "1e": "string", "1e+": "string", "1_0": "string", "infinit": "string", "nan0": "string",
    ".": "string", "-": "string", "+": "string", "e5": "string", "1.5.": "string", " 1": "string", "1d5": "string",
}


def test_csv_inference_follows_the_kernel_grammar(gpu, tmp_path):
    """Int64 is decided by value, not by length; Float64 only for what csv_parse_kernel accepts, so no column inferred
    numeric fails to parse."""
    names = list(CSV_SPELLINGS)
    for start in range(0, len(names), 16):
        chunk = names[start:start + 16]
        p = tmp_path / ("spell%d.csv" % start)
        p.write_text(",".join("c%d" % i for i in range(len(chunk))) + "\n" + ",".join('"%s"' % s if s.startswith(" ") else s for s in chunk) + "\n")
        t = read_all(FileInput({"input_type": {"type": "csv", "path": str(p)}}))
        for i, s in enumerate(chunk):
            col = t.column("c%d" % i)
            assert str(col.type) == CSV_SPELLINGS[s], s
            v = col.to_pylist()[0]
            if col.type == pa.float64():
                w = float(s)
                assert NC.bits_of(v) == NC.bits_of(w) or (w != w and v != v), s
            elif col.type == pa.int64():
                assert v == int(s), s
            else:
                assert v == s, s
    # the ones Arrow C++'s reader also reads this way (it turns "nan" into NULL and reads "+5" as a double)
    for s in ("-9223372036854775808", "9223372036854775808", "0x1p3", "infinity", "-Infinity", "1e", "1.", ".5"):
        p = tmp_path / "one.csv"
        p.write_text("c\n%s\n" % s)
        assert str(pacsv.read_csv(str(p)).schema.types[0]) == CSV_SPELLINGS[s], s
