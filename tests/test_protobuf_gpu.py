"""`protobuf_to_arrow` / `arrow_to_protobuf` on the device vs oracle/protobuf_oracle.py: the reference's four tests
(crates/arkflow-plugin/src/processor/protobuf.rs:292-468), every scalar kind over 10^6 messages, round trips, NULL and
zero-length payloads, every error class, both entry points, the examples/protobuf_example.yaml pipeline and concurrent
callers."""
import json
import struct
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pyarrow as pa
import pytest

from arkflow_b200.arrow_ffi import DeviceBatch
from arkflow_b200.processor import (ArkError, ArrowToProtobufProcessor, JsonToArrowProcessor, MessageBatch, Pipeline,
                                    ProtobufToArrowProcessor, SqlProcessor)
from oracle import protobuf_oracle as O
from oracle.json_oracle import json_to_arrow
from oracle.protobuf_oracle import PbField
from oracle.sql_oracle import sql_process

pytestmark = pytest.mark.gpu

TEST_PROTO = 'syntax = "proto3";\n\npackage test;\n\nmessage TestMessage {\n  int64 timestamp = 1;\n  double value = 2;\n  string sensor = 3;\n}\n'
S_FIELDS = [PbField("timestamp", 1, "int64"), PbField("value", 2, "double"), PbField("sensor", 3, "string")]

KINDS = ["int32", "int64", "uint32", "uint64", "sint32", "sint64", "fixed32", "fixed64", "sfixed32", "sfixed64",
         "bool", "float", "double", "string", "bytes", "enum"]
ALL3 = [PbField(f"f_{k}", i + 1, k) for i, k in enumerate(KINDS)]
ALL2 = [PbField(f"f_{k}", i + 1, k, presence=True, default=d) for i, (k, d) in enumerate(zip(KINDS, [
    -7, 1 << 40, 7, 1 << 60, -3, -(1 << 50), 9, 11, -13, -17, True, 1.5, -2.25, "dé", b"\x00\xff", 1]))]


def proto_dir(tmp_path, text, name="m"):
    d = tmp_path / name
    d.mkdir(parents=True, exist_ok=True)
    (d / f"{name}.proto").write_text(text)
    return str(d)


def processors(tmp_path, fields, syntax="proto3", **kw):
    d = proto_dir(tmp_path, O.proto_text("t", "M", fields, syntax), syntax)
    cfg = {"proto_inputs": [d], "message_type": "t.M"}
    return ProtobufToArrowProcessor(dict(cfg, **kw.get("dec", {}))), ArrowToProtobufProcessor(dict(cfg, **kw.get("enc", {})))


def decode(proc, payloads, device=False):
    mb = MessageBatch.new_binary(payloads) if isinstance(payloads, list) else MessageBatch.new_arrow(payloads)
    if device:
        out = proc.process_device(DeviceBatch.from_arrow(mb.record_batch))
        return None if out is None else out.to_arrow()
    r = proc.process(mb)
    return None if r.is_none() else r.batches[0].record_batch


def encode(proc, rb, device=False):
    if device:
        out = proc.process_device(DeviceBatch.from_arrow(rb))
        return None if out is None else out.to_arrow()
    r = proc.process(MessageBatch.new_arrow(rb))
    return None if r.is_none() else r.batches[0].record_batch


def assert_same_batch(got, want):
    assert got.schema == want.schema, (got.schema, want.schema)
    for i, f in enumerate(want.schema):
        a, b = got.column(i), want.column(i)
        if pa.types.is_floating(f.type):  # NaN != NaN for Array.equals: compare the bits
            w = np.uint32 if f.type == pa.float32() else np.uint64
            assert np.array_equal(a.to_numpy(zero_copy_only=False).view(w), b.to_numpy(zero_copy_only=False).view(w)), f.name
        else:
            assert a.equals(b), f.name


# ---- the reference's tests (processor/protobuf.rs:292-468) -----------------------------------------------------------
def test_protobuf_to_arrow_conversion(gpu, tmp_path):
    d = proto_dir(tmp_path, TEST_PROTO, "proto")
    p = ProtobufToArrowProcessor({"proto_inputs": [d], "proto_includes": None, "message_type": "test.TestMessage", "value_field": "__value__"})
    encoded = O.encode_message(S_FIELDS, {"timestamp": 1634567890, "value": 42.5, "sensor": "temperature"})
    r = p.process(MessageBatch.new_binary([encoded]))
    assert len(r) == 1
    b = r.batches[0].record_batch
    assert b.num_columns == 3 and set(b.schema.names) == {"timestamp", "value", "sensor"}
    assert b.to_pydict() == {"timestamp": [1634567890], "value": [42.5], "sensor": ["temperature"]}


def test_arrow_to_protobuf_conversion(gpu, tmp_path):
    d = proto_dir(tmp_path, TEST_PROTO, "proto")
    p = ArrowToProtobufProcessor({"proto_inputs": [d], "proto_includes": None, "message_type": "test.TestMessage"})
    rb = pa.RecordBatch.from_arrays([pa.array([1634567890], pa.int64()), pa.array([42.5]), pa.array(["temperature"])],
                                    schema=pa.schema([pa.field("timestamp", pa.int64(), False), pa.field("value", pa.float64(), False),
                                                      pa.field("sensor", pa.utf8(), False)]))
    r = p.process(MessageBatch.new_arrow(rb))
    assert len(r) == 1
    binary = r.batches[0].to_binary("__value__")
    assert len(binary) == 1
    assert O.decode_message(S_FIELDS, binary[0]) == {"timestamp": 1634567890, "value": 42.5, "sensor": "temperature"}


def test_protobuf_processor_empty_batch(gpu, tmp_path):
    d = proto_dir(tmp_path, TEST_PROTO, "proto")
    p = ProtobufToArrowProcessor({"proto_inputs": [d], "message_type": "test.TestMessage"})
    assert len(p.process(MessageBatch.new_binary([]))) == 0
    e = ArrowToProtobufProcessor({"proto_inputs": [d], "message_type": "test.TestMessage"})
    assert len(e.process(MessageBatch.new_arrow(pa.record_batch({"timestamp": pa.array([], pa.int64())})))) == 0
    assert p.process_device(DeviceBatch.from_arrow(MessageBatch.new_binary([]).record_batch)) is None


def test_processor_builder(gpu, tmp_path):
    for cls in (ProtobufToArrowProcessor, ArrowToProtobufProcessor):
        with pytest.raises(ArkError):
            cls(None)
    d = proto_dir(tmp_path, TEST_PROTO, "proto")
    ProtobufToArrowProcessor({"proto_inputs": [d], "proto_includes": None, "message_type": "test.TestMessage", "value_field": None})


# ---- every scalar kind, 10^6 messages --------------------------------------------------------------------------------
STR_POOL = ["", "a", "temp_1", "é", "漢字", "😀x", "line\nbreak", "z" * 40]
BYTES_POOL = [b"", b"\x00", b"\xff\xfe", b"abc", bytes(range(20))]


def random_columns(rng, n, neg_zero=False):
    """Arrow columns of every kind (ARROW_TYPE), special values included; floats from random bit patterns."""
    def pick(vals, size):
        return np.where(rng.random(size) < 0.15, rng.choice(vals, size), rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, size, dtype=np.int64))

    i64 = pick([0, 1, -1, 2**63 - 1, -2**63], n)
    cols = {
        "int32": i64.astype(np.int32), "sint32": pick([0, -1, 2**31 - 1, -2**31], n).astype(np.int32),
        "sfixed32": i64[::-1].astype(np.int32), "enum": rng.integers(-3, 6, n).astype(np.int32),
        "int64": i64, "sint64": pick([0, -1, 2**63 - 1, -2**63], n), "sfixed64": i64[::-1].copy(),
        "uint32": i64.view(np.uint64).astype(np.uint32), "fixed32": (i64 >> 7).view(np.uint64).astype(np.uint32),
        "uint64": i64.view(np.uint64), "fixed64": np.roll(i64, 1).view(np.uint64),
        "bool": rng.random(n) < 0.5,
    }
    # zeros, -0.0 (proto3 without presence leaves it out, so it decodes as +0.0: only with neg_zero), NaN, ±inf, denormals
    f32 = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    sp = rng.random(n) < 0.1
    f32[sp] = np.array([0, 0x80000000 if neg_zero else 0, 0x7FC00000, 0x7F800000, 0xFF800000, 1], np.uint32)[rng.integers(0, 6, int(sp.sum()))]
    f64 = rng.integers(0, 2**64, n, dtype=np.uint64)
    sp = rng.random(n) < 0.1
    f64[sp] = np.array([0, 1 << 63 if neg_zero else 0, 0x7FF8000000000000, 0x7FF0000000000000, 0xFFF0000000000000, 1], np.uint64)[rng.integers(0, 6, int(sp.sum()))]
    cols["float"] = f32.view(np.float32)
    cols["double"] = f64.view(np.float64)
    arrays = {k: pa.array(v) for k, v in cols.items()}
    arrays["int32"], arrays["sint32"], arrays["sfixed32"], arrays["enum"] = (pa.array(cols[k], pa.int32()) for k in ("int32", "sint32", "sfixed32", "enum"))
    si = rng.integers(0, len(STR_POOL), n)
    bi = rng.integers(0, len(BYTES_POOL), n)
    arrays["string"] = pa.array(np.array(STR_POOL, dtype=object)[si], pa.utf8())
    arrays["bytes"] = pa.array(np.array(BYTES_POOL, dtype=object)[bi], pa.binary())
    return arrays


def _varints(u):
    """(n, 10) byte matrix and byte counts of the varints of uint64 `u`."""
    n = len(u)
    m = np.zeros((n, 10), np.uint8)
    lens = np.ones(n, np.int64)
    v = u.astype(np.uint64)
    for j in range(10):
        rest = v >> np.uint64(7)
        m[:, j] = (v & np.uint64(0x7F)).astype(np.uint8) | np.where(rest != 0, 0x80, 0).astype(np.uint8)
        if j < 9:
            lens += rest != 0
        v = rest
    return m, lens


def encode_vectorized(fields, arrays, skip_zeros):
    """Canonical encoding of whole columns with numpy (every field in ascending number order; `skip_zeros`: proto3
    implicit presence).  Checked against O.encode_message on a sample below."""
    n = len(next(iter(arrays.values())))
    blocks = []
    for f in sorted(fields, key=lambda f: f.number):
        a = arrays[f.kind]
        k = f.kind
        if k in ("string", "bytes"):
            offs = np.frombuffer(a.buffers()[1], np.int32)[: n + 1]
            data = np.frombuffer(a.buffers()[2], np.uint8) if a.buffers()[2] is not None else np.zeros(1, np.uint8)
            ln = np.diff(offs).astype(np.int64)
            lm, ll = _varints(ln.astype(np.uint64))
            w = int(ln.max()) if n else 0
            body = np.zeros((n, max(w, 1)), np.uint8)
            idx = offs[:-1, None] + np.arange(max(w, 1))[None, :]
            valid = np.arange(max(w, 1))[None, :] < ln[:, None]
            body[valid] = data[np.minimum(idx, len(data) - 1)][valid]
            vals = [(lm, ll), (body, ln)]
            zero = ln == 0
        else:
            raw = a.to_numpy(zero_copy_only=False)
            if k in ("int32", "enum"):
                u = raw.astype(np.int64).view(np.uint64)
            elif k == "sint32":
                s = raw.astype(np.int32)
                u = ((s.astype(np.uint32) << np.uint32(1)) ^ (s >> 31).astype(np.uint32)).astype(np.uint64)
            elif k == "sint64":
                s = raw.astype(np.int64)
                u = (s.view(np.uint64) << np.uint64(1)) ^ (s >> 63).view(np.uint64)
            elif k == "bool":
                u = raw.astype(np.uint64)
            elif k in ("float", "double"):
                u = None  # written as their bits
            else:
                u = raw.view(np.uint64) if raw.dtype.itemsize == 8 else raw.astype(np.uint64)
            wire = O.WIRE.get(k, O.VARINT)
            if wire == O.VARINT:
                vals = [_varints(u)]
            else:
                w = 4 if wire == O.I32 else 8
                vals = [(raw.view(np.uint8).reshape(n, w), np.full(n, w, np.int64))]
            zero = (raw == 0) if k in ("float", "double") else (u == 0)
        key = bytearray()
        O.put_varint(key, (f.number << 3) | O.WIRE.get(k, O.VARINT))
        km = np.tile(np.frombuffer(bytes(key), np.uint8), (n, 1))
        keep = ~zero if (skip_zeros and not f.presence) else np.ones(n, bool)
        blocks.append((km, np.where(keep, len(key), 0)))
        for m, ln in vals:
            blocks.append((m, np.where(keep, ln, 0)))
    mat = np.hstack([m for m, _ in blocks])
    mask = np.hstack([np.arange(m.shape[1])[None, :] < ln[:, None] for m, ln in blocks])
    sizes = mask.sum(axis=1)
    offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    return pa.Array.from_buffers(pa.binary(), n, [None, pa.py_buffer(offsets.tobytes()), pa.py_buffer(mat[mask].tobytes())])


@pytest.mark.parametrize("syntax", ["proto3", "proto2"])
def test_all_kinds_million_messages_decode_and_encode(gpu, tmp_path, syntax):
    fields = ALL3 if syntax == "proto3" else ALL2
    dec, enc = processors(tmp_path, fields, syntax)
    rng = np.random.default_rng(17)
    batches = 4
    n = (1 << 20) // batches if syntax == "proto3" else 50_000
    for b in range(batches):
        arrays = random_columns(rng, n, neg_zero=syntax == "proto2")
        payloads = encode_vectorized(fields, arrays, skip_zeros=syntax == "proto3")
        sample = rng.choice(n, 500, replace=False)
        for i in sample:  # the vectorised encoder is the oracle's encoding
            vals = {f.name: O._column_values(arrays[f.kind].slice(int(i), 1))[0] for f in fields}
            assert payloads[int(i)].as_py() == O.encode_message(fields, vals)
        rb = pa.RecordBatch.from_arrays([payloads], names=["__value__"])
        got = decode(dec, rb, device=b % 2 == 1)
        want = pa.RecordBatch.from_arrays([arrays[f.kind] for f in fields],
                                          schema=pa.schema([pa.field(f.name, O.ARROW_TYPE[f.kind], nullable=False) for f in fields]))
        assert_same_batch(got, want)
        small = rb.slice(int(sample[0]) // 2, 3000)
        assert_same_batch(decode(dec, small), O.protobuf_to_arrow(fields, small))
        # encode: the decoded batch back to bytes, equal to the canonical encoding byte for byte
        out = encode(enc, got, device=b % 2 == 0)
        assert out.schema.names == [f.name for f in fields] + ["__value__"]
        assert out.column("__value__").equals(payloads)
        part = got.slice(0, 2000)
        assert encode(enc, part).column("__value__").to_pylist() == O.arrow_to_protobuf_values(fields, part)


def test_round_trip_and_unknown_fields_and_repeats(gpu, tmp_path):
    dec, enc = processors(tmp_path, ALL3)
    rng = np.random.default_rng(3)
    n = 20_000
    arrays = random_columns(rng, n)
    rb = pa.RecordBatch.from_arrays([arrays[f.kind] for f in ALL3], names=[f.name for f in ALL3])
    encoded = encode(enc, rb)
    back = decode(dec, pa.RecordBatch.from_arrays([encoded.column("__value__")], names=["__value__"]))
    assert_same_batch(back, pa.RecordBatch.from_arrays(rb.columns, schema=back.schema))
    # unknown fields, groups, repeated occurrences: the last one wins
    payloads = []
    for i in range(3000):
        a = {f.name: v for f in ALL3 for v in [O._column_values(arrays[f.kind].slice(i, 1))[0]] if rng.random() < 0.5}
        c = {f.name: v for f in ALL3 for v in [O._column_values(arrays[f.kind].slice(n - 1 - i, 1))[0]] if rng.random() < 0.5}
        junk = bytearray()
        for num, wire, body in ((100, 0, b"\x96\x01"), (101, 1, b"\x00" * 8), (102, 2, b"\x03abc"), (103, 5, b"\x01\x02\x03\x04"),
                                (2**29 - 1, 0, b"\x01")):
            O.put_varint(junk, (num << 3) | wire)
            junk += body
        O.put_varint(junk, (104 << 3) | 3)
        O.put_varint(junk, (5 << 3) | 3); O.put_varint(junk, (1 << 3) | 0); junk += b"\x05"; O.put_varint(junk, (5 << 3) | 4)
        O.put_varint(junk, (104 << 3) | 4)
        payloads.append(O.encode_message(ALL3, a) + bytes(junk) + O.encode_message(ALL3, c))
    mb = MessageBatch.new_binary(payloads).record_batch
    assert_same_batch(decode(dec, mb), O.protobuf_to_arrow(ALL3, mb))
    assert_same_batch(decode(dec, mb, device=True), O.protobuf_to_arrow(ALL3, mb))


def test_null_and_zero_length_payloads_and_defaults(gpu, tmp_path):
    for fields, syntax in ((ALL3, "proto3"), (ALL2, "proto2")):
        dec, _ = processors(tmp_path, fields, syntax)
        one = O.encode_message(fields, {fields[0].name: 5, "f_string": "x"})
        arr = pa.array([one, None, b"", None, one, b""] * 500, pa.binary())
        rb = pa.RecordBatch.from_arrays([arr, pa.array(range(len(arr)))], names=["__value__", "other"])
        want = O.protobuf_to_arrow(fields, rb)
        assert want.num_rows == 2000
        assert_same_batch(decode(dec, rb), want)
        assert_same_batch(decode(dec, rb, device=True), want)
        allnull = pa.RecordBatch.from_arrays([pa.array([None, None], pa.binary())], names=["__value__"])
        got = decode(dec, allnull)
        assert got.num_rows == 0 and got.schema.names == [f.name for f in fields]
    # a custom value_field; the other columns and the input name are not carried over
    dec, _ = processors(tmp_path, S_FIELDS, dec={"value_field": "payload"})
    rb = pa.RecordBatch.from_arrays([pa.array([1, 2]), pa.array([O.encode_message(S_FIELDS, {"sensor": "s"}), b""], pa.binary())], names=["k", "payload"])
    r = dec.process(MessageBatch(rb, "input1")).batches[0]
    assert r.input_name is None and r.record_batch.to_pydict() == {"timestamp": [0, 0], "value": [0.0, 0.0], "sensor": ["s", ""]}
    for bad, text in ((pa.RecordBatch.from_arrays([pa.array([1])], names=["k"]), "not found column"),
                      (pa.RecordBatch.from_arrays([pa.array(["x"])], names=["payload"]), "not support data type")):
        with pytest.raises(ArkError) as e:
            dec.process(MessageBatch.new_arrow(bad))
        assert e.value.kind == "Process" and e.value.message == text


MALFORMED = [b"\x08", b"\x08\x80", b"\x12\x05ab", b"\x00\x01", b"\x08" + b"\xff" * 10 + b"\x01", b"\x08" + b"\xff" * 9 + b"\x02",
             b"\x0d\x00\x00\x00\x00", b"\x14", b"\x0b\x14", b"\x1a\x02\xc3\x28", b"\x1e", b"\x0f", b"\xf8\xff\xff\xff\x7f\x00",
             b"\x83\x01" * 101, b"\x83\x01\x08\x01"]


@pytest.mark.parametrize("bad", MALFORMED)
def test_decode_errors(gpu, tmp_path, bad):
    fields = [PbField("i", 1, "int32"), PbField("s", 3, "string"), PbField("b", 4, "bytes")]
    dec, _ = processors(tmp_path, fields)
    with pytest.raises(O.ProtobufError):
        O.decode_message(fields, bad)
    good = O.encode_message(fields, {"i": 3, "s": "ok"})
    for device in (False, True):
        with pytest.raises(ArkError) as e:
            decode(dec, [good] * 300 + [bad] + [good] * 5, device=device)
        assert e.value.kind == "Process" and e.value.message.startswith("Protobuf message parsing failed: "), e.value.message
        assert "(payload 300)" in e.value.message
    assert O.decode_message(fields, b"\x22\x02\xc3\x28") == {"i": 0, "s": "", "b": b"\xc3\x28"}  # bytes need not be UTF-8
    assert decode(dec, [b"\x22\x02\xc3\x28"]).column("b").to_pylist() == [b"\xc3\x28"]


def test_repeated_map_and_message_fields(gpu, tmp_path):
    d = proto_dir(tmp_path, 'syntax = "proto3";\npackage r;\nmessage Sub { int32 x = 1; }\n'
                            'message M { int32 a = 1; repeated int32 r = 2; map<string, int32> m = 3; Sub s = 4; }\n'
                            'message N { int32 a = 1; Sub s = 2; repeated int32 r = 3; }\n', "r")
    for mt, first in (("r.M", "r"), ("r.N", "s")):
        dec = ProtobufToArrowProcessor({"proto_inputs": [d], "message_type": mt})
        for payloads in ([b""], [b"\x08\x01", None]):
            with pytest.raises(ArkError) as e:
                decode(dec, pa.RecordBatch.from_arrays([pa.array(payloads, pa.binary())], names=["__value__"]))
            assert e.value.kind == "Process" and e.value.message == f"Unsupported field type: {first}"
        assert decode(dec, []) is None
    enc = ArrowToProtobufProcessor({"proto_inputs": [d], "message_type": "r.M"})
    ok = encode(enc, pa.record_batch({"a": pa.array([1, 0], pa.int32()), "r": pa.array([1, 2], pa.int64())}))  # r: Int64 ≠ Int32, skipped
    assert ok.column("__value__").to_pylist() == [b"\x08\x01", b""]
    for col, kind in (({"s": pa.array([1])}, "Process"), ({"m": pa.array(["x"])}, "Process"), ({"r": pa.array([1], pa.int32())}, "Unsupported")):
        with pytest.raises(ArkError) as e:
            encode(enc, pa.record_batch(col))
        assert e.value.kind == kind, e.value.message
        if kind == "Process":
            assert e.value.message.startswith("Unsupported Protobuf type: ")


def test_encode_selection_rules(gpu, tmp_path):
    fields = [PbField("a", 3, "int32"), PbField("b", 1, "string"), PbField("x", 5, "int64", oneof=0), PbField("y", 4, "string", oneof=0),
              PbField("f", 2, "float"), PbField("o", 6, "double", presence=True)]
    _, enc = processors(tmp_path, fields)
    rb = pa.RecordBatch.from_arrays(
        [pa.array([1, None, -1], pa.int32()), pa.array(["s", "", None]), pa.array([0, 7, 8]), pa.array(["u", "v", ""]),
         pa.array([-0.0, float("nan"), 0.0], pa.float32()), pa.array([0.0, -0.0, 1.0]), pa.array([9, 9, 9], pa.int64()),
         pa.array([1.0, 2.0, 3.0]), pa.array([True, False, True])],
        names=["a", "b", "x", "y", "f", "o", "a", "extra", "flag"])  # second `a` is Int64: skipped
    for cfg_inc in (None, ["a", "y", "o"], ["b", "x"]):
        _, enc = processors(tmp_path, fields, enc={} if cfg_inc is None else {"fields_to_include": cfg_inc})
        got = encode(enc, rb)
        want = O.arrow_to_protobuf(fields, rb, None if cfg_inc is None else set(cfg_inc))
        assert got.schema.names == want.schema.names and got.column("__value__").equals(want.column("__value__"))
        no_dup = rb.select([0, 1, 2, 3, 4, 5, 7, 8])  # (DeviceBatch.from_arrow needs distinct names)
        dev = encode(enc, no_dup, device=True)
        assert_same_batch(dev.select(range(no_dup.num_columns)), no_dup)
        assert dev.column("__value__").equals(O.arrow_to_protobuf(fields, no_dup, None if cfg_inc is None else set(cfg_inc)).column("__value__"))
    # y (oneof member, column after x) wins over x; -0.0 without presence is left out; `o` has presence
    assert O.decode_message(fields, encode(processors(tmp_path, fields)[1], rb).column("__value__")[0].as_py())["y"] == "u"
    _, enc = processors(tmp_path, fields, enc={"fields_to_include": ["nothing"]})
    with pytest.raises(ArkError) as e:
        encode(enc, rb)
    assert e.value.kind == "Process" and e.value.message.startswith("Creating an Arrow record batch failed")


def test_protobuf_example_pipeline_on_device(gpu, tmp_path):
    """examples/protobuf_example.yaml: generate → json_to_arrow → sql → arrow_to_protobuf → protobuf_to_arrow, device-resident."""
    from arkflow_b200.input import GenerateInput

    d = proto_dir(tmp_path, 'syntax = "proto3";\n\npackage message;\n\n\nmessage Message{\n  int64 timestamp = 1;\n  double value = 2;\n  string sensor = 3;\n}',
                  "examples")
    q = "SELECT count(timestamp) as timestamp, sum(value) as value, cast(count(sensor) as string) as  sensor FROM flow WHERE value >= 10 order by sensor"
    context = '{ "timestamp": 1625000000000, "value": 10.0, "sensor": "temp_1" }'
    inp = GenerateInput({"context": context, "interval": "1ms", "batch_size": 1000})
    inp.connect()
    stages = [JsonToArrowProcessor({}), SqlProcessor({"query": q}),
              ArrowToProtobufProcessor({"proto_inputs": [d], "message_type": "message.Message"}),
              ProtobufToArrowProcessor({"proto_inputs": [d], "message_type": "message.Message"})]
    cur = inp.read_device()
    host = cur.to_arrow()
    inp.close()
    for st in stages:
        cur = st.process_device(cur)
    got = cur.to_arrow()
    fields = [PbField("timestamp", 1, "int64"), PbField("value", 2, "double"), PbField("sensor", 3, "string")]
    aggregated = sql_process(json_to_arrow(host), q)
    want = O.protobuf_to_arrow(fields, O.arrow_to_protobuf(fields, aggregated).select(["__value__"]))
    assert_same_batch(got, want)
    assert got.to_pydict() == {"timestamp": [1000], "value": [10000.0], "sensor": ["1000"]}
    # the same pipeline through the host entry points
    out = Pipeline(stages).process(MessageBatch.new_binary([context.encode()] * 10)).batches[0].record_batch
    assert out.to_pydict() == {"timestamp": [10], "value": [100.0], "sensor": ["10"]}


def test_concurrent_callers_share_processors(gpu, tmp_path):
    dec, enc = processors(tmp_path, ALL3)
    rng = np.random.default_rng(8)
    work = []
    for i in range(6):
        arrays = random_columns(rng, 20_000 + 1000 * i)
        rb = pa.RecordBatch.from_arrays([arrays[f.kind] for f in ALL3], names=[f.name for f in ALL3])
        payloads = encode_vectorized(ALL3, arrays, skip_zeros=True)
        work.append((rb, payloads, pa.RecordBatch.from_arrays([payloads], names=["__value__"])))

    def run(t):
        for rep in range(5):
            rb, payloads, prb = work[(t + rep) % len(work)]
            assert encode(enc, rb, device=rep % 2 == 0).column("__value__").equals(payloads)
            assert_same_batch(decode(dec, prb, device=rep % 2 == 1),
                              pa.RecordBatch.from_arrays(rb.columns, schema=pa.schema([pa.field(f.name, O.ARROW_TYPE[f.kind], False) for f in ALL3])))
        return True

    with ThreadPoolExecutor(max_workers=6) as pool:
        assert all(pool.map(run, range(6)))


def test_example_message_decodes_like_json(gpu, tmp_path):
    # the generate context of examples/protobuf_example.yaml as one protobuf payload per row
    d = proto_dir(tmp_path, TEST_PROTO, "proto")
    dec = ProtobufToArrowProcessor({"proto_inputs": [d], "message_type": "test.TestMessage"})
    rec = json.loads('{ "timestamp": 1625000000000, "value": 10.0, "sensor": "temp_1" }')
    payload = O.encode_message(S_FIELDS, rec)
    assert payload == b"\x08\x80\xf4\xb0\xcc\xa5/\x11" + struct.pack("<d", 10.0) + b"\x1a\x06temp_1"
    assert decode(dec, [payload] * 3).to_pydict() == {k: [v] * 3 for k, v in rec.items()}


def test_oneof_decode_keeps_the_last_member(gpu, tmp_path):
    # merging a oneof member clears the others: of x (5) then y ("hi") on the wire only y keeps its value
    pair = [PbField("x", 1, "int32", oneof=0), PbField("y", 2, "string", oneof=0), PbField("k", 3, "int64")]
    dec, _ = processors(tmp_path, pair)
    payload = O.encode_message(pair, {"x": 5}) + O.encode_message(pair, {"k": 7, "y": "hi"})
    for device in (False, True):
        assert decode(dec, [payload], device=device).to_pydict() == {"x": [0], "y": ["hi"], "k": [7]}
    fields = [PbField("a", 1, "int32"), PbField("x", 2, "int32", oneof=0), PbField("y", 3, "string", oneof=0),
              PbField("z", 4, "double", oneof=0), PbField("p", 5, "bool", oneof=1), PbField("q", 6, "bytes", oneof=1)]
    dec, _ = processors(tmp_path / "two", fields)
    rng = np.random.default_rng(21)
    payloads = []
    for _ in range(20_000):
        b = b""
        for _ in range(int(rng.integers(0, 6))):  # single-field messages concatenated, as merged messages arrive
            f = fields[int(rng.integers(0, len(fields)))]
            v = {"int32": int(rng.integers(-2**31, 2**31)), "string": "s%d" % rng.integers(0, 99), "double": float(rng.normal()),
                 "bool": bool(rng.integers(0, 2)), "bytes": bytes(rng.integers(0, 256, int(rng.integers(0, 4))).tolist())}[f.kind]
            b += O.encode_message(fields, {f.name: v})
        payloads.append(b)
    rb = MessageBatch.new_binary(payloads).record_batch
    want = O.protobuf_to_arrow(fields, rb)
    assert_same_batch(decode(dec, rb), want)
    assert_same_batch(decode(dec, rb, device=True), want)


@pytest.mark.parametrize("rows", [40_000, 66_000])
def test_string_column_beyond_int32_offsets_is_an_error(gpu, tmp_path, rows):
    # a 64 KiB proto2 string default taken by every empty payload: 2.6 GB (int32 scan negative) and 4.3 GB (the scan wraps
    # past 2^32 back to a small positive total); both must fail before any string byte is copied
    big = "ab" * 32768
    fields = [PbField("s", 1, "string", presence=True, default=big), PbField("i", 2, "int32", presence=True)]
    dec, _ = processors(tmp_path, fields, "proto2")
    assert decode(dec, [b"\x10\x07"] * 3).to_pydict() == {"s": [big] * 3, "i": [7] * 3}
    with pytest.raises(ArkError) as e:
        decode(dec, [b""] * rows)
    assert e.value.kind == "Process" and "2 GiB" in e.value.message, e.value.message
