"""The `file` input's `avro` type (csrc/avro.cu) against oracle/avro_oracle.py, whole batches at a time.

Every file is written from an index or a seed into tmp_path.  Batches are compared by the rules of
tests/test_inputs_edges_gpu.py (schema names, types and nullability, Array.equals per column, floats by bit pattern,
validate(full=True)), through both read() and read_device().to_arrow(); errors by kind and full message.  Each case
asserts the launch counts of the Avro kernels (ark_kernel_timing_get), so it shows which kernels ran.
"""
import struct

import numpy as np
import pyarrow as pa
import pytest

from arkflow_b200.input import FileInput
from arkflow_b200.processor import ArkError
from oracle.avro_oracle import (DEFAULT_SYNC, PFX, block_bytes, crc32_be, encode_record, header, put_long, put_varint, read_avro,
                                record_schema, snappy_block_data, snappy_compress, write_avro)
from oracle.sql_oracle import sql_process
from test_avro_oracle import UNSUPPORTED_SCHEMAS
from test_inputs_edges_gpu import CHUNK, launches, same_batches

pytestmark = pytest.mark.gpu

KERNELS = ("avro_snappy_kernel", "avro_index_kernel", "avro_decode_kernel")
ALL = [("n", "null"), ("b", "boolean"), ("i", "int"), ("l", "long"), ("f", "float"), ("d", "double"), ("y", "bytes"), ("s", "string"),
       ("ni", ["null", "int"]), ("sn", ["string", "null"]), ("nd", ["null", "double"]), ("bn", ["boolean", "null"])]


@pytest.fixture(scope="module", autouse=True)
def timing(gpu):
    gpu.ark_kernel_timing_enable(1)
    yield gpu
    gpu.ark_kernel_timing_enable(0)


def scan(path, device=False, **cfg):
    out = []
    try:
        inp = FileInput(dict(cfg, input_type={"type": "avro", "path": str(path)}))
        inp.connect()
        while True:
            out.append(inp.read_device().to_arrow() if device else inp.read()[0].record_batch)
    except ArkError as e:
        return out, (None if e.kind == "EOF" else e)


def check(lib, tmp_path, data, batch_size=None, query=None, snappy=None, name="t.avro"):
    """Scans `data` both ways, compares with the oracle and returns it; asserts which kernels ran: per batch read (and
    per failing read) one index and one decode launch, and one snappy launch when the codec is snappy."""
    p = tmp_path / name
    p.write_bytes(data)
    want, werr = read_avro(data, batch_size)
    if query:
        want = [b for b in (sql_process(rb, query) for rb in want) if b is not None]
    cfg = {} if batch_size is None else {"batch_size": batch_size}
    if query:
        cfg["query"] = {"query": query}
    for device in (False, True):
        lib.ark_kernel_timing_reset()
        got, err = scan(p, device, **cfg)
        if werr is not None:
            assert err is not None, ("no error", werr.message)
            assert (err.kind, err.message) == (werr.kind, werr.message)
        else:
            assert err is None, err.message
        same_batches(got, want, "device" if device else "host")
        reads = len(read_avro(data, batch_size)[0]) + (1 if werr is not None and werr.message.find(" in record ") > 0 else 0)
        assert launches(lib, "avro_decode_kernel") == reads and launches(lib, "avro_index_kernel") == reads
        if snappy is not None:
            assert launches(lib, "avro_snappy_kernel") == (reads if snappy else 0)
    return want, werr


def tile_rows(n):
    """Values of every ALL field; NULLs at the 128-record CTA edges and elsewhere."""
    rows = []
    for i in range(n):
        edge = i % 128 in (0, 127)
        rows.append((None, i % 3 == 0, (i * 7919) % 100000 - 50000, i * 10**11 - 7, float(i) / 8, -float(i) / 3,
                     bytes([i % 256]) * (i % 6), "é漢\U0001F600"[: i % 4] + "x" * (i % 9),
                     None if edge or i % 5 == 1 else -i, None if edge or i % 7 == 2 else "s%d" % i,
                     None if edge or i % 4 == 3 else i * 0.5, None if i % 128 == 64 else i % 2 == 1))
    return rows


@pytest.mark.parametrize("codec", ["null", "snappy"])
@pytest.mark.parametrize("batch_size", [None, 300])
def test_every_type(timing, tmp_path, codec, batch_size):
    sc = record_schema(ALL)
    data = write_avro(sc, tile_rows(1000), block_rows=[1, 127, 0, 256, 616], codec=codec)
    want, err = check(timing, tmp_path, data, batch_size, snappy=codec == "snappy")
    assert err is None and sum(b.num_rows for b in want) == 1000


def test_int_limits_and_varints(timing, tmp_path):
    sc = record_schema([("i", "int"), ("l", "long"), ("u", ["null", "long"])])
    recs = []
    for v in (0, 1, -1, 2**31 - 1, -2**31, 63, -64, 64):
        recs.append(put_long(v) + put_long(v) + put_long(1) + put_long(v))
    for v in (2**63 - 1, -2**63, 2**62, -2**62 - 1):
        recs.append(put_long(0) + put_long(v) + put_long(0))
    for w in range(1, 11):  # 1- to 10-byte varints, overlong ones included (assumption A3)
        recs.append(put_long(5, w) + put_long(-3, w) + put_long(1, w) + put_long(2**40, max(w, 6)))
    data = header(sc) + block_bytes(len(recs), b"".join(recs))
    want, err = check(timing, tmp_path, data)
    assert err is None and want[0].column("l").to_pylist()[8:12] == [2**63 - 1, -2**63, 2**62, -2**62 - 1]


def test_float_bits(timing, tmp_path):
    sc = record_schema([("f", "float"), ("d", "double"), ("nf", ["null", "float"])])
    f32 = [0x7FC00001, 0xFFC12345, 0x7F800001, 0x80000000, 0x00000001, 0x007FFFFF, 0x7F800000, 0xFF800000]
    f64 = [0x7FF8000000000001, 0xFFF123456789ABCD, 0x7FF0000000000001, 0x8000000000000000, 1, 0x000FFFFFFFFFFFFF, 0x7FF0000000000000, 3]
    rows = [(struct.pack("<I", a), struct.pack("<Q", b), None if k % 3 == 0 else struct.pack("<I", a)) for k, (a, b) in enumerate(zip(f32, f64))]
    check(timing, tmp_path, write_avro(sc, rows, block_rows=3))


@pytest.mark.parametrize("codec", ["null", "snappy"])
def test_strings(timing, tmp_path, codec):
    sc = record_schema([("s", "string"), ("y", "bytes"), ("ns", ["null", "string"])])
    big = "€" * 25000  # 75 000 bytes
    rows = [("", b"", ""), (big, bytes(range(256)) * 300, None), ("a", b"\x00", "ß"), ("\U0010FFFF漢", b"", big), ("", b"\xff" * 70000, "")]
    check(timing, tmp_path, write_avro(sc, rows * 3, block_rows=[2, 4, 9], codec=codec), snappy=codec == "snappy")


def test_block_sizes(timing, tmp_path):
    sc = record_schema([("l", "long"), ("s", ["null", "string"])])
    rows = [(i, None if i % 11 == 0 else "r%d" % (i % 1000)) for i in range(100_010)]
    check(timing, tmp_path, write_avro(sc, rows, block_rows=[1] * 5 + [100_000] + [1] * 5), batch_size=40_000)


def straddling_file(codec):
    """A file of three upload chunks: a block header straddles the first chunk boundary (inside its size varint) and a
    sync marker the second.  Returns (bytes, records)."""
    sc = record_schema([("y", "bytes"), ("k", "long")])
    out = bytearray(header(sc, codec))
    k = 0

    def blk(n):
        raw = encode_record(sc, (bytes([k % 251]) * n, k))
        return block_bytes(1, snappy_block_data(raw, matches=False) if codec == "snappy" else raw)

    targets = [(CHUNK, "header"), (2 * CHUNK, "sync")]
    for b, what in targets:
        while True:
            gap = b - len(out)
            # the block that ends right before b: header straddle → next block starts at b - 2; sync straddle → this
            # block's sync covers b
            want_end = b - 2 if what == "header" else b + 8
            if gap > 3000:
                out += blk(1000); k += 1
                continue
            for n in range(0, 3000):
                if len(out) + len(blk(n)) == want_end:
                    out += blk(n); k += 1
                    break
            else:
                raise AssertionError("no payload size fits")
            break
    while len(out) < 2 * CHUNK + 200_000:
        out += blk(777); k += 1
    return bytes(out), k


@pytest.mark.parametrize("codec", ["null", "snappy"])
def test_three_chunks(timing, tmp_path, codec):
    data, n = straddling_file(codec)
    assert len(data) > 2 * CHUNK
    want, err = check(timing, tmp_path, data, batch_size=5000, snappy=codec == "snappy")
    assert err is None and sum(b.num_rows for b in want) == n


def test_batch_splits(timing, tmp_path):
    sc = record_schema([("l", "long"), ("s", "string"), ("d", ["double", "null"])])
    rows = [(i, "v%d" % i, None if i % 3 else i / 7) for i in range(503)]
    data = write_avro(sc, rows, block_rows=10)
    whole = pa.Table.from_batches(check(timing, tmp_path, data)[0])
    for bs in (1, 7, 10, 128, 502):
        got = pa.Table.from_batches(check(timing, tmp_path, data, batch_size=bs)[0])
        assert got.equals(whole), bs


def test_header_only(timing, tmp_path):
    p = tmp_path / "h.avro"
    p.write_bytes(header(record_schema([("l", "long")])))
    timing.ark_kernel_timing_reset()
    got, err = scan(p)
    assert got == [] and err is None and all(launches(timing, k) == 0 for k in KERNELS)


def test_query(timing, tmp_path):
    sc = record_schema([("l", "long"), ("d", "double"), ("s", "string"), ("b", "boolean"), ("nl", ["null", "long"])])
    rows = [(i, i / 4, "k%d" % (i % 13), i % 2 == 0, None if i % 5 == 0 else i * 3) for i in range(2000)]
    data = write_avro(sc, rows, block_rows=300, codec="snappy")
    check(timing, tmp_path, data, batch_size=700, query="SELECT l, s, nl FROM flow WHERE l > 100 AND b", snappy=True)
    check(timing, tmp_path, data, query="SELECT d, s FROM flow WHERE d >= 100.0")


@pytest.mark.parametrize("k", range(len(UNSUPPORTED_SCHEMAS)))
def test_unsupported_schema(timing, tmp_path, k):
    schema, message = UNSUPPORTED_SCHEMAS[k]
    want, err = check(timing, tmp_path, header(schema) + block_bytes(0, b""))
    assert (err.kind, err.message) == ("Unsupported", message)


@pytest.mark.parametrize("codec", ["deflate", "zstandard", "bzip2", "xz"])
def test_unsupported_codec(timing, tmp_path, codec):
    want, err = check(timing, tmp_path, header(record_schema([("l", "long")]), codec))
    assert err.kind == "Unsupported" and codec in err.message


# ---- malformed data ---------------------------------------------------------------------------------------------------
MSC = record_schema([("i", "int"), ("b", "boolean"), ("u", ["null", "long"]), ("s", "string"), ("y", "bytes")])


def good(i):
    return encode_record(MSC, (i, i % 2 == 1, None if i % 3 == 0 else i, "s%d" % i, b"y" * (i % 4)))


BAD_RECORDS = {
    "varint": put_long(1) + b"\x01" + put_long(1) + b"\xff" * 10 + b"\x01",
    "int_range": put_long(2**31) + b"\x00" + put_long(0) + put_long(0) + put_long(0),
    "int_range_neg": put_long(-2**31 - 1) + b"\x00" + put_long(0) + put_long(0) + put_long(0),
    "bool": put_long(1) + b"\x02" + put_long(0) + put_long(0) + put_long(0),
    "union": put_long(1) + b"\x00" + put_long(2) + put_long(0) + put_long(0),
    "union_neg": put_long(1) + b"\x00" + put_long(-1) + put_long(0) + put_long(0),
    "neg_len": put_long(1) + b"\x00" + put_long(0) + put_long(-1) + put_long(0),
    "overrun_len": put_long(1) + b"\x00" + put_long(0) + put_long(0) + put_long(10**6),
    "utf8": put_long(1) + b"\x00" + put_long(0) + put_long(2) + b"\xc0\xaf" + put_long(0),
    "surrogate": put_long(1) + b"\x00" + put_long(0) + put_long(3) + b"\xed\xa0\x80" + put_long(0),
}


def blocks_with(bad_block, bad, codec="null", n_blocks=5, per=6):
    out, r = bytearray(header(MSC, codec)), 0
    for k in range(n_blocks):
        recs = [good(r + j) for j in range(per)]
        if k == bad_block:
            recs[2] = bad
        raw = b"".join(recs)
        out += block_bytes(per, snappy_block_data(raw) if codec == "snappy" else raw)
        r += per
    return bytes(out)


@pytest.mark.parametrize("where", [0, 2, 4])
@pytest.mark.parametrize("kind", sorted(BAD_RECORDS))
def test_bad_record(timing, tmp_path, kind, where):
    want, err = check(timing, tmp_path, blocks_with(where, BAD_RECORDS[kind]), batch_size=4)
    assert err is not None and err.kind == "Process" and (" in record %d " % (where * 6 + 2)) in err.message
    # each good read before it copies its `s` and `y` bytes; the failing read copies nothing
    assert launches(timing, "protobuf_strings_kernel") == 2 * ((where * 6 + 2) // 4)


@pytest.mark.parametrize("where", [0, 2, 4])
def test_record_past_block_end(timing, tmp_path, where):
    out, r = bytearray(header(MSC)), 0
    for k in range(5):
        raw = b"".join(good(r + j) for j in range(6))
        out += block_bytes(7 if k == where else 6, raw)  # one record more than the block holds
        r += 6
    want, err = check(timing, tmp_path, bytes(out), batch_size=5)
    assert err.message.startswith(PFX + "record runs past the end of its block in record %d " % (where * 6 + 6))


def structure_variants(where):
    """(name, bytes): the block at index `where` of 4 made malformed in its structure."""
    h = header(MSC)
    blocks = [block_bytes(3, b"".join(good(3 * k + j) for j in range(3))) for k in range(4)]

    def with_block(b):
        bl = list(blocks)
        bl[where] = b
        return h + b"".join(bl)
    raw = b"".join(good(j) for j in range(3))
    yield "sync", with_block(put_long(3) + put_long(len(raw)) + raw + bytes(16))
    yield "neg_count", with_block(put_long(-3) + put_long(len(raw)) + raw + DEFAULT_SYNC)
    yield "neg_size", with_block(put_long(3) + put_long(-5) + raw + DEFAULT_SYNC)
    yield "varint", with_block(b"\x86" * 10 + b"\x00" + put_long(len(raw)) + raw + DEFAULT_SYNC)
    yield "truncated", h + b"".join(blocks[:where]) + blocks[where][:-20]
    yield "bad_magic", b"Obj\x00" + (h + b"".join(blocks))[4:]


@pytest.mark.parametrize("where", [0, 1, 3])
def test_bad_structure(timing, tmp_path, where):
    for name, data in structure_variants(where):
        want, err = check(timing, tmp_path, data, batch_size=2, name=name + ".avro")
        assert err is not None and err.kind == "Process" and want == [], name


# ---- snappy -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opts", [{"copy_form": 1}, {"copy_form": 2}, {"copy_form": 4}, {"literal_extra": 0}, {"literal_extra": 1},
                                  {"literal_extra": 2}, {"literal_extra": 3}, {"literal_extra": 4}, {"matches": False}])
def test_snappy_forms(timing, tmp_path, opts):
    sc = record_schema([("s", "string"), ("l", "long"), ("r", "bytes")])
    rows = [("key%03d" % (i % 50), i, b"ab" * (i % 40) + b"\x00" * (i % 100)) for i in range(3000)]
    check(timing, tmp_path, write_avro(sc, rows, block_rows=[1, 999, 2000], codec="snappy", snappy=opts), batch_size=1024, snappy=True)


def snappy_bad_block(kind):
    raw = b"".join(good(j) for j in range(6))
    body = snappy_compress(raw)[len(put_varint(len(raw))):]
    if kind == "crc":
        return put_varint(len(raw)) + body + bytes(a ^ b for a, b in zip(crc32_be(raw), b"\x00\x00\x00\x01"))
    if kind == "underfill":
        return put_varint(len(raw) + 1) + body + crc32_be(raw)
    if kind == "overrun":
        return put_varint(len(raw) - 1) + body + crc32_be(raw)
    return put_varint(len(raw)) + b"\x02\x05\x00" + body + crc32_be(raw)  # a copy before any output: offset past the start


@pytest.mark.parametrize("where", [0, 2, 4])
@pytest.mark.parametrize("kind", ["crc", "underfill", "overrun", "offset"])
def test_snappy_bad_block(timing, tmp_path, kind, where):
    out = bytearray(header(MSC, "snappy"))
    for k in range(5):
        raw = b"".join(good(6 * k + j) for j in range(6))
        out += block_bytes(6, snappy_bad_block(kind) if k == where else snappy_block_data(raw))
    want, err = check(timing, tmp_path, bytes(out), batch_size=4, snappy=True)
    assert err is not None and (" in record %d " % (where * 6)) in err.message


# ---- a batch of 2^22 records ------------------------------------------------------------------------------------------
def test_four_million_rows(timing, tmp_path):
    n, per = 1 << 22, 1 << 16
    idx = np.arange(n, dtype=np.int64)
    rec = np.zeros(n, dtype=[("d", "<f8"), ("f", "<f4"), ("b", "u1")])
    rec["d"] = idx * 0.25 - 3.0
    rec["f"] = (idx % 1000).astype(np.float32) / 3
    rec["b"] = idx % 2
    raw = rec.tobytes()
    sc = record_schema([("d", "double"), ("f", "float"), ("b", "boolean")])
    out = bytearray(header(sc))
    w = rec.dtype.itemsize
    for k in range(n // per):
        out += block_bytes(per, raw[k * per * w:(k + 1) * per * w])
    p = tmp_path / "big.avro"
    p.write_bytes(bytes(out))
    for device in (False, True):
        timing.ark_kernel_timing_reset()
        got, err = scan(p, device)
        assert err is None and [b.num_rows for b in got] == [n]
        assert launches(timing, "avro_index_kernel") == 1 and launches(timing, "avro_decode_kernel") == 1
        b = got[0]
        b.validate(full=True)
        assert np.array_equal(b.column("d").to_numpy().view(np.uint64), rec["d"].view(np.uint64))
        assert np.array_equal(b.column("f").to_numpy().view(np.uint32), rec["f"].view(np.uint32))
        assert np.array_equal(b.column("b").to_numpy(zero_copy_only=False).astype(np.uint8), rec["b"])
