"""oracle/arrow_ipc_oracle.py against pyarrow (its IPC writer and reader, its LZ4 codec) and the xxHash32 test vector; and
the errors the `file` input's `arrow` type decides at connect() from metadata alone, before the device is touched (so
they run without a GPU)."""
import io
import struct

import pyarrow as pa
import pytest

from arkflow_b200.input import FileInput
from arkflow_b200.processor import ArkError
from oracle.arrow_ipc_oracle import (PFX, Lz4Error, Stored, compress_buffer, lz4_decode, lz4_frame, read_ipc, stored_from_arrow,
                                     write_ipc, xxh32)


def sample(n, seed=0):
    r = range(seed, seed + n)
    return pa.record_batch({
        "n": pa.nulls(n),
        "b": pa.array([None if i % 7 == 0 else i % 3 == 0 for i in r], pa.bool_()),
        "i": pa.array([None if i % 5 == 0 else i * 7919 - 50000 for i in r], pa.int32()),
        "l": pa.array([i * 10**11 - 7 for i in r], pa.int64()),
        "ui": pa.array([i * 3 for i in r], pa.uint32()),
        "ul": pa.array([None if i % 4 == 1 else 2**63 + i for i in r], pa.uint64()),
        "f": pa.array([i / 8 for i in r], pa.float32()),
        "d": pa.array([None if i % 6 == 2 else -i / 3 for i in r], pa.float64()),
        "s": pa.array([None if i % 9 == 4 else "é漢"[: i % 3] + "x" * (i % 11) for i in r], pa.utf8()),
        "y": pa.array([bytes([i % 256]) * (i % 5) for i in r], pa.binary()),
    })


def fields_of(rb):
    return [(f.name, f.type, f.nullable) for f in rb.schema]


def pyarrow_file(batches, compression=None, legacy=False):
    sink = io.BytesIO()
    opts = pa.ipc.IpcWriteOptions(compression=compression, use_legacy_format=legacy)
    with pa.ipc.new_file(sink, batches[0].schema, options=opts) as w:
        for b in batches:
            w.write(b)
    return sink.getvalue()


def test_xxh32_vectors():
    assert xxh32(b"") == 0x02CC5D05
    # the header-checksum byte of pyarrow's frames: (xxh32 of FLG..descriptor end) >> 8 & 0xFF
    f = pa.compress(b"abc" * 1000, codec="lz4", asbytes=True)
    desc_len = 2 + (8 if f[4] & 0x08 else 0)
    assert (xxh32(f[4:4 + desc_len]) >> 8) & 0xFF == f[4 + desc_len]


@pytest.mark.parametrize("kw", [{}, {"independent": True}, {"block_checksum": True}, {"content_checksum": True}, {"content_size": True},
                                {"stored": True}, {"stored": (1,)}, {"block_code": 5}, {"block_code": 7}, {"matches": False},
                                {"independent": True, "block_checksum": True, "content_checksum": True, "content_size": True}])
def test_lz4_round_trip(kw):
    data = b"".join(b"rec%05d|" % (i % 37) + b"z" * (i % 70) for i in range(3000))
    f = lz4_frame(data, **kw)
    assert lz4_decode(f, len(data)) == data
    assert pa.decompress(f, len(data), codec="lz4", asbytes=True) == data
    assert lz4_decode(pa.compress(data, codec="lz4", asbytes=True), len(data)) == data


def test_lz4_errors():
    data = b"abcdefgh" * 100
    f = lz4_frame(data)
    cases = [(f[:5], "truncated"), (b"\0" + f[1:], "malformed"), (f[:-4], "truncated"), (f + b"\0", "bytes after"),
             (lz4_frame(data, content_size=True), None)]
    for bad, msg in cases:
        if msg is None:
            assert lz4_decode(bad, len(data)) == data
            continue
        with pytest.raises(Lz4Error) as e:
            lz4_decode(bad, len(data))
        assert msg in str(e.value)
    for ulen, msg in ((len(data) - 1, "overruns"), (len(data) + 1, "underfills")):
        with pytest.raises(Lz4Error) as e:
            lz4_decode(f, ulen)
        assert msg in str(e.value)
    with pytest.raises(Lz4Error) as e:
        lz4_decode(lz4_frame(data, content_size=True), len(data) + 1)
    assert "content size" in str(e.value)
    ck = bytearray(lz4_frame(data, content_checksum=True))
    ck[-1] ^= 1
    with pytest.raises(Lz4Error) as e:
        lz4_decode(bytes(ck), len(data))
    assert "checksum" in str(e.value)


@pytest.mark.parametrize("legacy", [False, True])
@pytest.mark.parametrize("lz4", [None, True])
def test_oracle_writer_read_by_pyarrow(legacy, lz4):
    rbs = [sample(100), sample(0), sample(37, 5)]
    data = write_ipc(fields_of(rbs[0]), [stored_from_arrow(rb, lz4=lz4) for rb in rbs], legacy=legacy)
    got = pa.ipc.open_file(pa.BufferReader(data))
    assert got.num_record_batches == 3
    for k, rb in enumerate(rbs):
        assert got.get_batch(k).equals(rb)


@pytest.mark.parametrize("frame", [{"independent": True}, {"block_checksum": True, "content_checksum": True}, {"stored": True}, {"raw": True}])
def test_oracle_frames_read_by_pyarrow(frame):
    rb = sample(500)
    data = write_ipc(fields_of(rb), [stored_from_arrow(rb, lz4=True, **frame)])
    assert pa.ipc.open_file(pa.BufferReader(data)).get_batch(0).equals(rb)
    got, err = read_ipc(data)
    assert err is None and got[0].equals(rb)


@pytest.mark.parametrize("legacy", [False, True])
@pytest.mark.parametrize("compression", [None, "lz4"])
@pytest.mark.parametrize("shape", [(1000,), (1, 2, 3), (0, 64, 0, 7), (300, 300)])
@pytest.mark.parametrize("batch_rows", [None, 1, 7, 300])
def test_pyarrow_files_read_by_oracle(legacy, compression, shape, batch_rows):
    rbs = [sample(n, 11 * k) for k, n in enumerate(shape)]
    data = pyarrow_file(rbs, compression, legacy)
    got, err = read_ipc(data, batch_rows)
    assert err is None
    want = pa.ipc.open_file(pa.BufferReader(data)).read_all().combine_chunks()
    step = batch_rows or 1 << 22
    assert [b.num_rows for b in got] == [min(step, len(want) - r) for r in range(0, len(want), step)]
    if got:
        assert pa.Table.from_batches(got).equals(pa.Table.from_batches(want.to_batches()))


def test_pyarrow_sliced_arrays():
    rb = sample(200).slice(13, 101)
    data = pyarrow_file([rb])
    got, err = read_ipc(data)
    assert err is None and got[0].equals(rb)


# ---- connect() without a GPU ------------------------------------------------------------------------------------------
def connect_error(tmp_path, data):
    p = tmp_path / "t.arrow"
    p.write_bytes(data)
    want = read_ipc(data)[1]
    inp = FileInput({"input_type": {"type": "arrow", "path": str(p)}})
    with pytest.raises(ArkError) as e:
        inp.connect()
    assert want is not None and (e.value.kind, e.value.message) == (want.kind, want.message)
    return e.value


UNSUPPORTED = [pa.int8(), pa.int16(), pa.uint8(), pa.float16(), pa.large_utf8(), pa.large_binary(), pa.date32(), pa.string_view()]


@pytest.mark.parametrize("t", UNSUPPORTED, ids=str)
def test_connect_unsupported_type(tmp_path, t):
    data = write_ipc([("ok", pa.int64(), True), ("bad", t, True)], [])
    e = connect_error(tmp_path, data)
    assert e.kind == "Unsupported" and "field 'bad'" in e.message


def test_connect_unsupported_pyarrow_types(tmp_path):
    for arr in (pa.array([[1]]), pa.array([{"a": 1}]), pa.array(["a"]).dictionary_encode(),
                pa.array([1], pa.timestamp("us")), pa.array([1], pa.decimal128(5, 2))):
        data = pyarrow_file([pa.record_batch({"x": arr})])
        e = connect_error(tmp_path, data)
        assert e.kind == "Unsupported" and "field 'x'" in e.message


def test_connect_big_endian_and_zstd(tmp_path):
    e = connect_error(tmp_path, write_ipc([("a", pa.int64(), True)], [], big_endian=True))
    assert e.kind == "Unsupported" and "big-endian" in e.message
    e = connect_error(tmp_path, pyarrow_file([sample(10)], "zstd"))
    assert e.kind == "Unsupported" and "ZSTD" in e.message
    e = connect_error(tmp_path, write_ipc([("a", pa.int8(), True, "dict")], []))
    assert e.kind == "Unsupported" and "dictionary-encoded" in e.message


def good():
    rb = pa.record_batch({"i": pa.array([1, 2, 3], pa.int64()), "s": pa.array(["a", None, "c"])})
    return fields_of(rb), rb


def test_connect_structural_errors(tmp_path):
    f, rb = good()
    data = write_ipc(f, [stored_from_arrow(rb)])
    stream = io.BytesIO()
    with pa.ipc.new_stream(stream, rb.schema) as w:
        w.write(rb)
    foot_len = struct.unpack_from("<i", data, len(data) - 10)[0]
    cases = {
        b"": "bad magic", data[:-1]: "bad magic", b"X" + data[1:]: "bad magic", stream.getvalue(): "bad magic",
        data[:-10] + struct.pack("<i", len(data)) + b"ARROW1": "footer out of range",
        data[:-10] + struct.pack("<i", 0) + b"ARROW1": "footer out of range",
        data[:-10 - foot_len] + bytes(foot_len) + data[-10:]: "malformed footer",
    }
    for bad, msg in cases.items():
        e = connect_error(tmp_path, bad)
        assert e.kind == "Process" and e.message.startswith(PFX) and msg in e.message, (msg, e.message)


def edited(mut, lz4=None, fields=None):
    f, rb = good()
    s = stored_from_arrow(rb, lz4=lz4)
    s2 = stored_from_arrow(rb, lz4=lz4)
    mut(s2)
    return write_ipc(fields or f, [s, s2])


@pytest.mark.parametrize("mut,msg", [
    (lambda s: setattr(s, "nodes", s.nodes[:1]), "field node count differs from the schema (record batch 1)"),
    (lambda s: setattr(s, "buffers", s.buffers[:4]), "buffer count differs from the schema (record batch 1)"),
    (lambda s: setattr(s, "nodes", [(2, 0), s.nodes[1]]), "node length differs from the batch length (record batch 1, column 'i')"),
    (lambda s: setattr(s, "nodes", [s.nodes[0], (3, 4)]), "invalid null count (record batch 1, column 's')"),
    (lambda s: setattr(s, "nodes", [s.nodes[0], (3, -1)]), "invalid null count (record batch 1, column 's')"),
    (lambda s: setattr(s, "buffers", [s.buffers[0], s.buffers[1][:16]] + s.buffers[2:]), "buffer too short for its node (record batch 1, column 'i')"),
    (lambda s: setattr(s, "buffers", s.buffers[:2] + [b"", s.buffers[3][:12]] + s.buffers[4:]), "buffer too short for its node (record batch 1, column 's')"),
    (lambda s: setattr(s, "gaps", [0, 4, 0, 0, 0]), "buffer not 8-byte aligned (record batch 1, column 'i')"),
])
def test_connect_batch_errors(tmp_path, mut, msg):
    e = connect_error(tmp_path, edited(mut))
    assert e.kind == "Process" and e.message == PFX + msg


def test_connect_non_nullable_with_nulls(tmp_path):
    _, rb = good()
    f = [("i", pa.int64(), True), ("s", pa.utf8(), False)]
    e = connect_error(tmp_path, write_ipc(f, [stored_from_arrow(rb)]))
    assert e.message == PFX + "null values in a non-nullable field (record batch 0, column 's')"


def test_connect_prefix_errors(tmp_path):
    def short_prefix(s):
        s.buffers[1] = b"\1\2\3"
    def bad_len(s):
        s.buffers[1] = struct.pack("<q", -2) + s.buffers[1][8:]
    def small(s):
        s.buffers[1] = compress_buffer(b"\0" * 16)
    for mut, msg in ((short_prefix, "buffer shorter than its length prefix"), (bad_len, "invalid uncompressed length"),
                     (small, "buffer too short for its node")):
        e = connect_error(tmp_path, edited(mut, lz4=True))
        assert e.message == PFX + msg + " (record batch 1, column 'i')"


def test_connect_block_outside_file(tmp_path):
    # cutting the bytes between the first 200 and the footer keeps the footer but leaves its block outside the file
    f, rb = good()
    s = stored_from_arrow(rb)
    s.buffers[1] = s.buffers[1] + bytes(1 << 20)
    big = write_ipc(f, [s])
    fl = struct.unpack_from("<i", big, len(big) - 10)[0]
    e = connect_error(tmp_path, big[:200] + big[len(big) - 10 - fl:])
    assert e.message == PFX + "block outside the file (record batch 0)"
