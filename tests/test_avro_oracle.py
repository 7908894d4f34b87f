"""oracle/avro_oracle.py against the Avro specification's own encodings, hand-assembled snappy streams and round trips;
and the schema / codec / header errors the `file` input's `avro` type decides at connect() from the header alone,
before the device is touched (so they run without a GPU)."""
import json
import struct
import zlib

import pyarrow as pa
import pytest

from arkflow_b200.input import FileInput
from arkflow_b200.processor import ArkError
from oracle.avro_oracle import (DEFAULT_SYNC, PFX, SnappyError, block_bytes, encode_record, header, put_long, put_string, put_varint,
                                read_avro, record_schema, snappy_compress, snappy_decompress, write_avro)

ALL = [("n", "null"), ("b", "boolean"), ("i", "int"), ("l", "long"), ("f", "float"), ("d", "double"), ("y", "bytes"), ("s", "string"),
       ("ni", ["null", "int"]), ("sn", ["string", "null"])]


def test_spec_encodings():
    # specification 1.11, "Binary Encoding": zig-zag longs, the string "foo", and the union example
    for v, enc in ((0, "00"), (-1, "01"), (1, "02"), (-2, "03"), (2, "04"), (-64, "7f"), (64, "8001")):
        assert put_long(v) == bytes.fromhex(enc), v
    assert put_string("foo") == bytes.fromhex("06666f6f")
    sc = record_schema([("u", ["null", "string"])])
    assert encode_record(sc, [None]) == bytes.fromhex("00")
    assert encode_record(sc, ["a"]) == bytes.fromhex("020261")
    assert put_varint(0, width=3) == b"\x80\x80\x00"  # overlong encodings (assumption A3)


def test_snappy_hand_assembled():
    # literal with 0..4 extra length bytes
    for extra in range(5):
        tag = bytes([2 << 2]) if extra == 0 else bytes([(59 + extra) << 2]) + (2).to_bytes(extra, "little")
        assert snappy_decompress(put_varint(3) + tag + b"abc") == b"abc"
    # copy-1 (length 4..11, 11-bit offset), copy-2, copy-4; offset 1 < length: a run
    ab = put_varint(2) + bytes([1 << 2]) + b"ab"
    assert snappy_decompress(put_varint(9) + bytes([1 << 2]) + b"ab" + bytes([1 | (2 << 2), 2]) + bytes([0]) + b"c") == b"ababababc"
    assert snappy_decompress(put_varint(10) + bytes([0]) + b"x" + bytes([2 | (8 << 2), 1, 0])) == b"x" * 10
    assert snappy_decompress(put_varint(7) + ab[1:] + bytes([3 | (4 << 2), 2, 0, 0, 0])) == b"abababa"
    for bad, msg in ((put_varint(2) + bytes([2 << 2]) + b"abc", "overruns"), (put_varint(5) + bytes([1 << 2]) + b"ab", "underfills"),
                     (put_varint(6) + bytes([0]) + b"x" + bytes([2 | (4 << 2), 2, 0]), "malformed"),  # offset beyond the output
                     (put_varint(6) + bytes([0]) + b"x" + bytes([2 | (4 << 2), 0, 0]), "malformed"),  # offset 0
                     (put_varint(3) + bytes([61 << 2]), "malformed")):  # literal length bytes missing
        with pytest.raises(SnappyError) as e:
            snappy_decompress(bad)
        assert msg in str(e.value)


@pytest.mark.parametrize("opts", [{}, {"copy_form": 1}, {"copy_form": 2}, {"copy_form": 4}, {"literal_extra": 0}, {"literal_extra": 4},
                                  {"matches": False}])
def test_snappy_round_trip(opts):
    data = b"".join(b"rec%05d|" % (i % 37) + b"z" * (i % 70) for i in range(300))
    s = snappy_compress(data, **opts)
    assert snappy_decompress(s) == data
    if opts.get("matches", True):
        assert len(s) < len(data)


def rows_all(n):
    return [(None, i % 3 == 0, i - 50, (i - 50) * 10**12, float(i) / 4, -float(i) / 3, bytes([i % 256]) * (i % 5), "é" * (i % 4),
             None if i % 4 == 1 else i, None if i % 6 == 2 else "s%d" % i) for i in range(n)]


@pytest.mark.parametrize("codec", ["null", "snappy"])
def test_writer_reader_round_trip(codec):
    sc = record_schema(ALL)
    rows = rows_all(300)
    data = write_avro(sc, rows, block_rows=[1, 0, 120, 179], codec=codec)
    got, err = read_avro(data, batch_rows=128)
    assert err is None and [b.num_rows for b in got] == [128, 128, 44]
    t = pa.Table.from_batches(got)
    assert [str(x) for x in t.schema.types] == ["null", "bool", "int32", "int64", "float", "double", "binary", "string", "int32", "string"]
    assert [f.nullable for f in t.schema] == [True, False, False, False, False, False, False, False, True, True]
    for k, (name, _) in enumerate(ALL):
        want = [r[k] for r in rows]
        if name == "f":
            want = [struct.unpack("<f", struct.pack("<f", v))[0] for v in want]
        assert t.column(name).to_pylist() == want, name


def test_reader_errors():
    sc = record_schema([("i", "int"), ("s", ["null", "string"])])
    good = write_avro(sc, [(1, "a"), (2, None)], block_rows=1)
    assert read_avro(good)[1] is None
    assert read_avro(b"Obj\x02" + good[4:])[1].message == PFX + "not an Avro object container file (bad magic)"
    h = header(sc)
    rec = encode_record(sc, (1, "a"))
    b1 = block_bytes(1, rec)
    assert read_avro(h + b1 + block_bytes(1, rec, sync=b"\0" * 16))[1].message == PFX + "sync marker mismatch (block at offset %d)" % (len(h) + len(b1))
    assert read_avro(h + b1[:-3])[1].message == PFX + "truncated block (block at offset %d)" % len(h)
    assert read_avro(h + put_long(-1) + put_long(0) + DEFAULT_SYNC)[1].message == PFX + "negative block count (block at offset %d)" % len(h)
    bad_int = put_long(2**31) + put_long(0)
    got, err = read_avro(h + b1 + block_bytes(2, rec + bad_int), batch_rows=1)
    assert [b.num_rows for b in got] == [1, 1] and err.message == PFX + "int value out of the i32 range in record 2 (block at offset %d)" % (len(h) + len(b1))
    for codec in ("deflate", "zstandard", "bzip2", "xz"):
        assert read_avro(header(sc, codec))[1].kind == "Unsupported"
    snap = header(sc, "snappy")
    raw = rec * 3
    blk = snappy_compress(raw) + struct.pack(">I", zlib.crc32(raw) ^ 1)
    assert read_avro(snap + block_bytes(3, blk))[1].message == PFX + "snappy block CRC-32 mismatch in record 0 (block at offset %d)" % len(snap)


# ---- connect() without a GPU ------------------------------------------------------------------------------------------
UNSUPPORTED_SCHEMAS = [
    ({"type": "array", "items": "int"}, "avro input: the top-level schema is array, not a record"),
    ('"long"', "avro input: the top-level schema is long, not a record"),
    (record_schema([("a", "int"), ("r", {"type": "record", "name": "in", "fields": []})]), "avro input: field 'r' has type record, which is not decoded on the GPU"),
    (record_schema([("x", {"type": "array", "items": "int"})]), "avro input: field 'x' has type array, which is not decoded on the GPU"),
    (record_schema([("x", {"type": "map", "values": "int"})]), "avro input: field 'x' has type map, which is not decoded on the GPU"),
    (record_schema([("x", {"type": "enum", "name": "e", "symbols": ["A"]})]), "avro input: field 'x' has type enum, which is not decoded on the GPU"),
    (record_schema([("x", {"type": "fixed", "name": "f", "size": 4})]), "avro input: field 'x' has type fixed, which is not decoded on the GPU"),
    (record_schema([("x", {"type": "long", "logicalType": "timestamp-millis"})]), "avro input: field 'x' has type logicalType timestamp-millis, which is not decoded on the GPU"),
    (record_schema([("x", ["null", "int", "string"])]), "avro input: field 'x' has type union, which is not decoded on the GPU"),
    (record_schema([("x", ["int", "string"])]), "avro input: field 'x' has type union, which is not decoded on the GPU"),
    (record_schema([("x", ["null", "null"])]), "avro input: field 'x' has type union, which is not decoded on the GPU"),
    (record_schema([("x", "Named")]), "avro input: field 'x' has type Named, which is not decoded on the GPU"),
    (record_schema([("f%d" % i, "int") for i in range(65)]), "avro input: more than 64 fields in a record"),
]


def connect_error(path):
    inp = FileInput({"input_type": {"type": "avro", "path": str(path)}})
    with pytest.raises(ArkError) as e:
        inp.connect()
    return e.value


@pytest.mark.parametrize("k", range(len(UNSUPPORTED_SCHEMAS)))
def test_connect_unsupported_schema(tmp_path, k):
    schema, message = UNSUPPORTED_SCHEMAS[k]
    p = tmp_path / "u.avro"
    p.write_bytes(header(schema))
    e = connect_error(p)
    want = read_avro(p.read_bytes())[1]
    assert (e.kind, e.message) == (want.kind, want.message) == ("Unsupported", message)


@pytest.mark.parametrize("codec", ["deflate", "zstandard", "bzip2", "xz"])
def test_connect_unsupported_codec(tmp_path, codec):
    p = tmp_path / "c.avro"
    p.write_bytes(header(record_schema([("a", "long")]), codec))
    e = connect_error(p)
    assert (e.kind, e.message) == ("Unsupported", "avro input: codec '%s' is not decoded on the GPU (null and snappy are)" % codec)


def test_connect_header_errors(tmp_path):
    sc = record_schema([("a", "long")])
    h = header(sc)
    meta_only = b"Obj\x01" + put_long(1) + put_string("avro.codec") + put_string("null") + put_long(0) + DEFAULT_SYNC
    for data, msg in ((b"", "not an Avro object container file (bad magic)"), (b"PAR1" + h[4:], "not an Avro object container file (bad magic)"),
                      (h[:-5], "truncated header"), (meta_only, "the header has no avro.schema"),
                      (b"Obj\x01" + b"\xff" * 11, "varint longer than 10 bytes in the header")):
        p = tmp_path / "h.avro"
        p.write_bytes(data)
        e = connect_error(p)
        want = read_avro(data)[1]
        assert (e.kind, e.message) == (want.kind, want.message) == ("Process", PFX + msg), msg


def test_header_in_several_map_blocks(tmp_path):
    # a metadata map written in two blocks, the first with a negative count and its byte size (assumption A8)
    sc = json.dumps(record_schema([("a", "long")])).encode()
    e1 = put_string("avro.schema") + put_long(len(sc)) + sc
    e2 = put_string("avro.codec") + put_string("xz")
    data = b"Obj\x01" + put_long(-1) + put_long(len(e1)) + e1 + put_long(1) + e2 + put_long(0) + DEFAULT_SYNC
    p = tmp_path / "m.avro"
    p.write_bytes(data)
    e = connect_error(p)
    assert (e.kind, e.message) == ("Unsupported", "avro input: codec 'xz' is not decoded on the GPU (null and snappy are)")
    assert read_avro(data)[1].message == e.message
