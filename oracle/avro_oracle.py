"""CPU oracle for the `file` input's `avro` type (csrc/avro.cu) — TEST INFRASTRUCTURE (see oracle/__init__.py).

A pure-Python restatement of Avro object container files (specification 1.11) and of how the input reads them: no Avro
library is needed, so GPU tests can import it.  tests/test_avro_oracle.py checks it against the specification's own
encodings, hand-assembled snappy streams and round trips.

Writer: `write_avro` (schema JSON, any block sizes and sync marker, codecs null / snappy), built from the pieces
`header`, `encode_record` and `block_bytes`, so a test can put deliberately malformed bytes anywhere.
`snappy_compress` can be told which element forms to emit; `snappy_decompress` reads any stream.

Reader: `read_avro(data, batch_rows)` → (batches, error), the batches the input yields before its first error:
  * schema: a record of null / boolean / int / long / float / double / bytes / string fields, or two-branch unions of
    null and one of these in either order → Null, Boolean, Int32, Int64, Float32, Float64, Binary, Utf8 (DataFusion's
    Avro reader's mapping); a plain field is non-nullable, a union field nullable (a `null` field is a nullable Null);
  * anything else, and any codec but null / snappy, is Unsupported from connect(), the codec decided before the schema;
  * the container's structure (magic, header, block count / size, sync markers, the snappy length preamble) is checked
    at connect(): an error there yields no batch;
  * every batch but the last holds exactly `batch_rows` records, cutting through blocks where it must;
  * a data error fails the batch holding the first failing record in file order; a snappy block that does not
    decompress to its declared length, or whose CRC-32 (big-endian, of the uncompressed data, after the stream)
    mismatches, is the failure of the block's first record.

ASSUMPTIONS (apache-avro's sources were not available to check them):
  A1. bytes left in a block after its `count` records are ignored (the reader takes `count` records from the block);
  A2. a block of 0 records is legal and holds no rows; its data is not decoded (nor, with snappy, decompressed);
  A3. a varint may be overlong (e.g. 0 written as 80 00) as long as it ends within 10 bytes; bits of the 10th byte past
      bit 63 are dropped (decode_variable);
  A4. an `int` is a long that must fit i32 (zag_i32's try_from);
  A5. a union's index is a zig-zag long like any other (`[null, T]`: 0 is null, 1 is T);
  A6. a boolean is one byte that must be 0 or 1;
  A7. a snappy element that copies from offset 0 or from before the start of the output is malformed;
  A8. the header's metadata map may come in several blocks, and a negative block count is followed by its byte size.
"""
from __future__ import annotations

import json
import struct
import zlib
from typing import Any, Optional, Sequence

import numpy as np
import pyarrow as pa

from .sql_oracle import OracleError

MAGIC = b"Obj\x01"
PRIMS = ("null", "boolean", "int", "long", "float", "double", "bytes", "string")
ARROW = {"null": pa.null(), "boolean": pa.bool_(), "int": pa.int32(), "long": pa.int64(), "float": pa.float32(),
         "double": pa.float64(), "bytes": pa.binary(), "string": pa.utf8()}
PFX = "Read input failed: Avro error: "
DEFAULT_SYNC = bytes(range(0x10, 0x20))

# data errors, in the decoder's words
E_VARINT, E_TRUNCATED, E_INT, E_BOOL, E_UNION, E_LEN, E_UTF8 = (
    "varint longer than 10 bytes", "record runs past the end of its block", "int value out of the i32 range",
    "boolean byte other than 0 or 1", "union index out of range", "negative or overrunning length", "string is not valid UTF-8")
E_OVERRUN, E_UNDERFILL, E_SNAPPY, E_CRC = ("snappy stream overruns its declared length", "snappy stream underfills its declared length",
                                           "malformed snappy stream", "snappy block CRC-32 mismatch")


# ---- encoding ---------------------------------------------------------------------------------------------------------
def zigzag(v: int) -> int:
    return ((v << 1) ^ (v >> 63)) & 0xFFFFFFFFFFFFFFFF


def put_varint(u: int, width: Optional[int] = None) -> bytes:
    """Unsigned LEB128; `width` pads it with zero continuation groups to that many bytes (an overlong encoding)."""
    out = bytearray()
    while True:
        b = u & 0x7F
        u >>= 7
        if u == 0 and (width is None or len(out) + 1 >= width):
            out.append(b)
            return bytes(out)
        out.append(b | 0x80)


def put_long(v: int, width: Optional[int] = None) -> bytes:
    return put_varint(zigzag(v), width)


def put_bytes(b: bytes) -> bytes:
    return put_long(len(b)) + b


def put_string(s: str) -> bytes:
    return put_bytes(s.encode())


def field_type(t: Any) -> tuple[str, int]:
    """(primitive, index of the null branch or -1), or raises Unsupported via the caller."""
    if isinstance(t, str) and t in PRIMS:
        return t, -1
    if isinstance(t, dict) and "logicalType" not in t and isinstance(t.get("type"), str) and t["type"] in PRIMS:
        return t["type"], -1
    if isinstance(t, list) and len(t) == 2:
        a, b = (field_type(x)[0] if _prim(x) else None for x in t)
        if a == "null" and b not in (None, "null"):
            return b, 0
        if b == "null" and a not in (None, "null"):
            return a, 1
    raise ValueError(t)


def _prim(t) -> bool:
    try:
        return field_type(t)[1] == -1
    except ValueError:
        return False


def type_desc(t: Any) -> str:
    if isinstance(t, str):
        return t
    if isinstance(t, list):
        return "union"
    if isinstance(t, dict):
        if "logicalType" in t:
            return "logicalType " + (t["logicalType"] if isinstance(t["logicalType"], str) else "?")
        if isinstance(t.get("type"), str):
            return t["type"]
    return "?"


def record_schema(fields: Sequence[tuple[str, Any]], name: str = "r") -> dict:
    return {"type": "record", "name": name, "fields": [{"name": n, "type": t} for n, t in fields]}


def encode_value(kind: str, v: Any) -> bytes:
    """`v` may be raw bytes for float / double (a bit pattern, NaN payloads included)."""
    if kind == "null":
        return b""
    if kind == "boolean":
        return bytes([1 if v else 0])
    if kind in ("int", "long"):
        return put_long(v)
    if kind in ("float", "double"):
        if isinstance(v, (bytes, bytearray)):
            return bytes(v)
        return struct.pack("<f" if kind == "float" else "<d", v)
    if kind == "bytes":
        return put_bytes(bytes(v))
    return put_string(v)


def encode_record(schema: dict, row: Sequence[Any]) -> bytes:
    out = bytearray()
    for f, v in zip(schema["fields"], row):
        kind, nb = field_type(f["type"])
        if nb >= 0:
            out += put_long(nb if v is None else 1 - nb)
            if v is None:
                continue
        out += encode_value(kind, v)
    return bytes(out)


# ---- snappy -----------------------------------------------------------------------------------------------------------
def _literal(chunk: bytes, extra: Optional[int]) -> bytes:
    n = len(chunk) - 1
    if extra is None:
        extra = 0 if n < 60 else (1 if n < 1 << 8 else 2 if n < 1 << 16 else 3 if n < 1 << 24 else 4)
    if extra == 0:
        assert n < 60
        return bytes([n << 2]) + chunk
    return bytes([(59 + extra) << 2]) + n.to_bytes(extra, "little") + chunk


def _copy(off: int, length: int, form: int) -> bytes:
    if form == 1:
        assert 4 <= length <= 11 and off < 2048
        return bytes([1 | ((length - 4) << 2) | ((off >> 8) << 5), off & 0xFF])
    assert 1 <= length <= 64
    if form == 2:
        assert off < 1 << 16
        return bytes([2 | ((length - 1) << 2)]) + off.to_bytes(2, "little")
    return bytes([3 | ((length - 1) << 2)]) + off.to_bytes(4, "little")


def snappy_compress(data: bytes, copy_form: Optional[int] = None, literal_extra: Optional[int] = None, matches: bool = True,
                    window: int = 1 << 15) -> bytes:
    """Greedy snappy stream (preamble + elements).  `copy_form` 1 / 2 / 4 forces the copy element form (copy-1 where
    its length and offset allow, else copy-2); `literal_extra` 0..4 forces a literal's length-byte count (0 needs a
    literal of at most 60 bytes: longer ones are split); `matches=False` emits literals only.  Matches may overlap
    their own output (offset < length), as runs do."""
    out = bytearray(put_varint(len(data)))
    n, i, lit0 = len(data), 0, 0
    last: dict[bytes, int] = {}
    max_lit = 60 if literal_extra == 0 else (1 << 32)

    def flush(upto):
        nonlocal lit0
        while lit0 < upto:
            k = min(upto - lit0, max_lit)
            out.extend(_literal(data[lit0:lit0 + k], literal_extra))
            lit0 += k

    while matches and i + 4 <= n:
        key = data[i:i + 4]
        j = last.get(key)
        last[key] = i
        if j is None or i - j > window:
            i += 1
            continue
        length = 4
        while i + length < n and data[j + length] == data[i + length]:
            length += 1
        flush(i)
        off = i - j
        left = length
        while left >= 4:
            if copy_form == 1 and off < 2048:
                k = min(left, 11)
                form = 1
            else:
                k = min(left, 64)
                form = 4 if copy_form == 4 else 2 if off < 1 << 16 else 4
            if 0 < left - k < 4:
                k = left - 4
            out.extend(_copy(off, k, form))
            left -= k
        i += length - left
        lit0 = i
    flush(n)
    return bytes(out)


class SnappyError(Exception):
    pass


def snappy_decompress(buf: bytes) -> bytes:
    """Reads a stream with its preamble; raises SnappyError(message) in the decoder's words and order."""
    ulen, p = 0, 0
    for k in range(5):
        if p >= len(buf):
            raise SnappyError(E_SNAPPY)
        c = buf[p]
        p += 1
        ulen |= (c & 0x7F) << (7 * k)
        if c < 0x80:
            break
    else:
        raise SnappyError(E_SNAPPY)
    return _snappy_body(buf, p, len(buf), ulen)


def _snappy_body(buf: bytes, p: int, end: int, ulen: int) -> bytes:
    out = bytearray()
    while p < end:
        t = buf[p]
        p += 1
        if t & 3 == 0:
            n = t >> 2
            if n >= 60:
                nx = n - 59
                if end - p < nx:
                    raise SnappyError(E_SNAPPY)
                n = int.from_bytes(buf[p:p + nx], "little")
                p += nx
            n += 1
            if end - p < n:
                raise SnappyError(E_SNAPPY)
            if n > ulen - len(out):
                raise SnappyError(E_OVERRUN)
            out += buf[p:p + n]
            p += n
            continue
        need = {1: 1, 2: 2, 3: 4}[t & 3]
        if end - p < need:
            raise SnappyError(E_SNAPPY)
        if t & 3 == 1:
            n, off = 4 + ((t >> 2) & 7), ((t >> 5) << 8) | buf[p]
        else:
            n, off = (t >> 2) + 1, int.from_bytes(buf[p:p + need], "little")
        p += need
        if off == 0 or off > len(out):
            raise SnappyError(E_SNAPPY)
        if n > ulen - len(out):
            raise SnappyError(E_OVERRUN)
        for _ in range(n):
            out.append(out[-off])
    if len(out) != ulen:
        raise SnappyError(E_UNDERFILL)
    return bytes(out)


def crc32_be(data: bytes) -> bytes:
    return zlib.crc32(data).to_bytes(4, "big")


# ---- container --------------------------------------------------------------------------------------------------------
def header(schema: Any, codec: Optional[str] = "null", sync: bytes = DEFAULT_SYNC, meta: Optional[dict] = None) -> bytes:
    m = {"avro.schema": (schema if isinstance(schema, str) else json.dumps(schema)).encode()}
    if codec is not None:
        m["avro.codec"] = codec.encode()
    m.update(meta or {})
    out = bytearray(MAGIC)
    if m:
        out += put_long(len(m))
        for k, v in m.items():
            out += put_string(k) + put_bytes(v)
    out += put_long(0) + sync
    return bytes(out)


def block_bytes(count: int, data: bytes, sync: bytes = DEFAULT_SYNC, size: Optional[int] = None) -> bytes:
    return put_long(count) + put_long(len(data) if size is None else size) + data + sync


def snappy_block_data(raw: bytes, **opts) -> bytes:
    return snappy_compress(raw, **opts) + crc32_be(raw)


def write_avro(schema: dict, rows: Sequence[Sequence[Any]], block_rows: Any = 1000, codec: str = "null",
               sync: bytes = DEFAULT_SYNC, snappy: Optional[dict] = None) -> bytes:
    """`block_rows`: records per block (an int), or the list of block sizes (they must add up to len(rows))."""
    sizes = block_rows if isinstance(block_rows, (list, tuple)) else \
        [min(block_rows, len(rows) - i) for i in range(0, len(rows), block_rows)]
    assert sum(sizes) == len(rows)
    out, r = bytearray(header(schema, codec, sync)), 0
    for k in sizes:
        raw = b"".join(encode_record(schema, rows[i]) for i in range(r, r + k))
        r += k
        data = snappy_block_data(raw, **(snappy or {})) if codec == "snappy" else raw
        out += block_bytes(k, data, sync)
    return bytes(out)


# ---- reader -----------------------------------------------------------------------------------------------------------
def _varint(data: bytes, p: int, end: int):
    """(value, next) of a zig-zag long; None when `end` comes first; raises on more than 10 bytes."""
    u = 0
    for k in range(10):
        if p + k >= end:
            return None
        c = data[p + k]
        u |= (c & 0x7F) << (7 * k)
        if c < 0x80:
            u &= 0xFFFFFFFFFFFFFFFF
            return ((u >> 1) ^ -(u & 1)), p + k + 1
    raise ValueError("varint")


def _fail(msg):
    raise OracleError("Process", PFX + msg)


def _schema_fields(text: bytes):
    try:
        s = json.loads(text.decode())
    except Exception as e:  # the decoder names its own JSON parser's complaint
        _fail("invalid schema: %s" % e)
    ty = s.get("type") if isinstance(s, dict) else None
    if ty != "record":
        raise OracleError("Unsupported", "avro input: the top-level schema is %s, not a record" % type_desc(s))
    fs = s.get("fields")
    if not isinstance(fs, list):
        _fail("invalid schema: a record without `fields`")
    out = []
    for f in fs:
        if not isinstance(f, dict) or not isinstance(f.get("name"), str) or "type" not in f:
            _fail("invalid schema: a field without `name` or `type`")
        try:
            kind, nb = field_type(f["type"])
        except ValueError:
            raise OracleError("Unsupported", "avro input: field '%s' has type %s, which is not decoded on the GPU" % (f["name"], type_desc(f["type"])))
        out.append((f["name"], kind, nb))
    if len(out) > 64:
        raise OracleError("Unsupported", "avro input: more than 64 fields in a record")
    return out


def parse_container(data: bytes):
    """connect(): (fields, snappy, blocks) with blocks = [(offset, data_off, size, count, preamble_len, ulen)]."""
    n = len(data)
    if n < 4 or data[:4] != MAGIC:
        _fail("not an Avro object container file (bad magic)")
    p, meta = 4, {}

    def hv(p):
        try:
            r = _varint(data, p, n)
        except ValueError:
            _fail("varint longer than 10 bytes in the header")
        if r is None:
            _fail("truncated header")
        return r
    while True:
        cnt, p = hv(p)
        if cnt == 0:
            break
        if cnt < 0:
            cnt = -cnt
            _, p = hv(p)
        for _ in range(cnt):
            kv = []
            for _ in range(2):
                ln, p = hv(p)
                if ln < 0:
                    _fail("negative length in the header")
                if ln > n - p:
                    _fail("truncated header")
                kv.append(data[p:p + ln])
                p += ln
            meta[kv[0].decode("utf-8", "replace")] = kv[1]
    if n - p < 16:
        _fail("truncated header")
    sync = data[p:p + 16]
    p += 16
    if "avro.schema" not in meta:
        _fail("the header has no avro.schema")
    codec = meta.get("avro.codec", b"null").decode("utf-8", "replace")
    if codec not in ("null", "snappy", ""):
        raise OracleError("Unsupported", "avro input: codec '%s' is not decoded on the GPU (null and snappy are)" % codec)
    fields = _schema_fields(meta["avro.schema"])
    snappy = codec == "snappy"
    blocks = []
    while p < n:
        at = " (block at offset %d)" % p
        try:
            r1 = _varint(data, p, n)
            r2 = None if r1 is None else _varint(data, r1[1], n)
        except ValueError:
            _fail("varint longer than 10 bytes" + at)
        if r1 is None or r2 is None:
            _fail("truncated block" + at)
        (count, q), (size, d) = r1, r2
        if count < 0:
            _fail("negative block count" + at)
        if size < 0:
            _fail("negative block size" + at)
        pre, ulen = 0, size
        if snappy:
            avail, v = min(n - d, size), 0
            for i in range(6):
                if i == 5 or i >= size - 4:
                    _fail("snappy block without a valid length preamble" + at)
                if i >= avail:
                    _fail("truncated block" + at)
                c = data[d + i]
                v |= (c & 0x7F) << (7 * i)
                if c < 0x80:
                    pre = i + 1
                    break
            if v > 0xFFFFFFFF:
                _fail("snappy block without a valid length preamble" + at)
            ulen = v
        if d + size + 16 > n:
            _fail("truncated block" + at)
        if data[d + size:d + size + 16] != sync:
            _fail("sync marker mismatch" + at)
        blocks.append((p, d, size, count, pre, ulen))
        p = d + size + 16
    return fields, snappy, blocks


def _decode_record(fields, buf: bytes, p: int, end: int, cols):
    """Appends one record's values to `cols`; returns the next position or raises ValueError(message)."""
    vals = []
    for name, kind, nb in fields:
        present = kind != "null"
        if nb >= 0:
            try:
                r = _varint(buf, p, end)
            except ValueError:
                raise ValueError(E_VARINT)
            if r is None:
                raise ValueError(E_TRUNCATED)
            b, p = r
            if b not in (0, 1):
                raise ValueError(E_UNION)
            if b == nb:
                present = False
        if not present:
            vals.append(None)
            continue
        if kind == "boolean":
            if p >= end:
                raise ValueError(E_TRUNCATED)
            if buf[p] > 1:
                raise ValueError(E_BOOL)
            vals.append(buf[p] == 1)
            p += 1
        elif kind in ("int", "long"):
            try:
                r = _varint(buf, p, end)
            except ValueError:
                raise ValueError(E_VARINT)
            if r is None:
                raise ValueError(E_TRUNCATED)
            v, p = r
            if kind == "int" and not -2**31 <= v < 2**31:
                raise ValueError(E_INT)
            vals.append(v)
        elif kind in ("float", "double"):
            w = 4 if kind == "float" else 8
            if end - p < w:
                raise ValueError(E_TRUNCATED)
            vals.append(int.from_bytes(buf[p:p + w], "little"))
            p += w
        else:
            try:
                r = _varint(buf, p, end)
            except ValueError:
                raise ValueError(E_VARINT)
            if r is None:
                raise ValueError(E_TRUNCATED)
            ln, p = r
            if ln < 0 or ln > end - p:
                raise ValueError(E_LEN)
            s = bytes(buf[p:p + ln])
            if kind == "string":
                try:
                    s = s.decode("utf-8")
                except UnicodeDecodeError:
                    raise ValueError(E_UTF8)
            vals.append(s)
            p += ln
    for c, v in zip(cols, vals):
        c.append(v)
    return p


def _column(kind, nb, vals):
    n = len(vals)
    if kind == "null":
        return pa.nulls(n)
    if kind in ("float", "double"):
        dt = np.uint32 if kind == "float" else np.uint64
        bits = np.array([0 if v is None else v for v in vals], dtype=dt)
        mask = np.array([v is None for v in vals], dtype=bool)
        arr = pa.array(bits.view(np.float32 if kind == "float" else np.float64), type=ARROW[kind], mask=mask if mask.any() else None)
        return arr
    return pa.array(vals, type=ARROW[kind])


def read_avro(data: bytes, batch_rows: Optional[int] = None):
    """(batches, error): what the input yields up to EOF (error None) or up to its first other error."""
    try:
        fields, snappy, blocks = parse_container(data)
    except OracleError as e:
        return [], e
    batch_rows = batch_rows or (1 << 22)
    cols = [[] for _ in fields]
    fail = None  # (row, message, block offset)
    row = 0
    for off, d, size, count, pre, ulen in blocks:
        if count == 0:  # A2: no rows, nothing decoded
            continue
        if snappy:
            try:
                buf = _snappy_body(data, d + pre, d + size - 4, ulen)
                if crc32_be(buf) != data[d + size - 4:d + size]:
                    raise SnappyError(E_CRC)
            except SnappyError as e:
                fail = (row, str(e), off)
                break
            p, end = 0, len(buf)
        else:
            buf, p, end = data, d, d + size
        for j in range(count):
            try:
                p = _decode_record(fields, buf, p, end, cols)
            except ValueError as e:
                fail = (row + j, str(e), off)
                break
        if fail:
            break
        row += count
    total = fail[0] if fail else row
    schema = pa.schema([pa.field(nm, ARROW[k], nullable=(nb >= 0 or k == "null")) for nm, k, nb in fields])
    batches = []
    for r0 in range(0, total, batch_rows):
        if fail and r0 + batch_rows > fail[0]:
            break
        n = min(batch_rows, total - r0)
        batches.append(pa.RecordBatch.from_arrays([_column(k, nb, c[r0:r0 + n]) for (nm, k, nb), c in zip(fields, cols)], schema=schema))
    if fail:
        return batches, OracleError("Process", PFX + "%s in record %d (block at offset %d)" % (fail[1], fail[0], fail[2]))
    return batches, None
