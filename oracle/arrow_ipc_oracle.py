"""CPU oracle for the `file` input's `arrow` type (csrc/arrow_ipc.cu) — TEST INFRASTRUCTURE (see oracle/__init__.py).

A Python restatement of the Arrow IPC file format and of how the input reads it.  tests/test_arrow_ipc_oracle.py checks
it against pyarrow's writer, reader and LZ4 codec.

Writer: `write_ipc(fields, batches, legacy=False)` writes schema, record batches and footer with the continuation-marker
or the legacy (pre-0.15) message prefix.  A batch is a `Stored`: its row count, its field nodes and the body bytes of
every buffer, so a test can place any frame form, `-1` prefix or broken frame in any buffer (`stored_from_arrow` builds
one from a pyarrow RecordBatch).  `lz4_frame` encodes an LZ4 frame with knobs for every form the format allows,
`lz4_decode` decodes one in the input's words, and `xxh32` is the frame format's checksum.  The flatbuffers are written
and read by the small builder and reader below; no flatbuffers library is needed.

Reader: `read_ipc(data, batch_rows)` → (batches, error), what the input yields before its first error.  The values are
decoded by pyarrow (an independent implementation); on top of it this module applies the input's rules:
  * field types Null, Boolean, Int32, Int64, UInt32, UInt64, Float32, Float64, Utf8, Binary; any other type (dictionary-
    encoded ones too), a big-endian schema and a ZSTD body are Unsupported from connect(), the first in file order;
  * checks that need only metadata and the 8-byte length prefixes of compressed buffers fail connect(): magic, footer,
    block and buffer ranges, 8-byte buffer alignment, node lengths and null counts, NULLs in a non-nullable field, and
    every buffer's (uncompressed) size against what its type and length need;
  * checks that need body bytes fail the read that first touches the stored batch: its LZ4 frames, its offsets (non-
    negative, non-decreasing, inside the data buffer), UTF-8 of every Utf8 slot, and, when a node's null_count > 0, the
    bitmap's zero bits over [0, length).  The first failure in (batch, column, row) order wins; within a column a frame
    failure comes first and a null-count mismatch last;
  * every batch but the last holds exactly `batch_rows` rows (default 2^22), cutting through stored batches in footer
    order; a stored batch of 0 rows yields nothing and its body is not read.
Messages are "Read input failed: Arrow IPC error: <what> (record batch k[, column 'c'][, row r])".

ASSUMPTIONS (the arrow-rs and lz4_flex sources were not available to check them):
  A1. arrow-rs's validate_nulls rejects a node whose null_count differs from its bitmap's zero bits;
  A2. a node with null_count == 0 has no validity: its bitmap is ignored;
  A3. no end-of-block LZ4 restrictions (last five bytes literals, MFLIMIT) are enforced by the decoder;
  A4. one frame per buffer: bytes after the frame's end mark (and content checksum) are an error;
  A5. an uncompressed-length prefix of 0 is an empty buffer whose frame is not read; a prefix below -1 is an error;
  A6. every slot of a Utf8 column, NULL ones included, must be valid UTF-8 (arrow-rs validates each offset window);
  A7. IPC body buffers start 8-byte aligned (the format's rule); a misaligned buffer fails connect();
  A8. a frame with a dictionary id is malformed; a block larger than the frame's maximum block size is malformed;
  A9. a stored batch of 0 rows is never decoded, so its body bytes are not checked.
"""
from __future__ import annotations

import struct
from dataclasses import dataclass, field as dfield
from typing import List, Optional

import pyarrow as pa

from .sql_oracle import OracleError

PFX = "Read input failed: Arrow IPC error: "
MAGIC = b"ARROW1"
ROW_LAST = (1 << 31) - 1

# ---------------------------------------------------------------------------------------------------------------------
# xxHash32 and LZ4 frames

P1, P2, P3, P4, P5 = 2654435761, 2246822519, 3266489917, 668265263, 374761393
M32 = 0xFFFFFFFF


def _rotl(x, r):
    return ((x << r) | (x >> (32 - r))) & M32


def xxh32(data: bytes, seed: int = 0) -> int:
    n, p = len(data), 0
    if n >= 16:
        v = [(seed + P1 + P2) & M32, (seed + P2) & M32, seed & M32, (seed - P1) & M32]
        while n - p >= 16:
            for k in range(4):
                v[k] = (_rotl((v[k] + struct.unpack_from("<I", data, p + 4 * k)[0] * P2) & M32, 13) * P1) & M32
            p += 16
        h = (_rotl(v[0], 1) + _rotl(v[1], 7) + _rotl(v[2], 12) + _rotl(v[3], 18)) & M32
    else:
        h = (seed + P5) & M32
    h = (h + n) & M32
    while n - p >= 4:
        h = (_rotl((h + struct.unpack_from("<I", data, p)[0] * P3) & M32, 17) * P4) & M32
        p += 4
    while p < n:
        h = (_rotl((h + data[p] * P5) & M32, 11) * P1) & M32
        p += 1
    h ^= h >> 15
    h = (h * P2) & M32
    h ^= h >> 13
    h = (h * P3) & M32
    h ^= h >> 16
    return h


def _lz4_len(n):
    out = bytearray()
    while n >= 255:
        out.append(255)
        n -= 255
    out.append(n)
    return bytes(out)


def lz4_block(data: bytes, start: int, end: int, window0: int, matches: bool = True) -> bytes:
    """LZ4 block of data[start:end]; matches may reach back to window0 (start: independent block).  Greedy, and within
    the format's end-of-block rules (the last match starts 12 bytes or more before the end, the last 5 bytes are
    literals)."""
    out = bytearray()
    table = {data[j:j + 4]: j for j in range(window0, start)}  # linked blocks: matches may reach into earlier blocks
    i = lit0 = start
    limit = end - 12
    while matches and i < limit:
        key = data[i:i + 4]
        cand = table.get(key)
        table[key] = i
        if cand is None or cand < window0 or i - cand > 65535:
            i += 1
            continue
        ml = 4
        while i + ml < end - 5 and data[cand + ml] == data[i + ml]:
            ml += 1
        lit = i - lit0
        tok = (min(lit, 15) << 4) | min(ml - 4, 15)
        out.append(tok)
        if lit >= 15:
            out += _lz4_len(lit - 15)
        out += data[lit0:i]
        out += struct.pack("<H", i - cand)
        if ml - 4 >= 15:
            out += _lz4_len(ml - 4 - 15)
        i += ml
        lit0 = i
    lit = end - lit0
    out.append(min(lit, 15) << 4)
    if lit >= 15:
        out += _lz4_len(lit - 15)
    out += data[lit0:end]
    return bytes(out)


def lz4_frame(data: bytes, block_code: int = 4, independent: bool = False, block_checksum: bool = False,
              content_checksum: bool = False, content_size: bool = False, stored=(), matches: bool = True) -> bytes:
    """An LZ4 frame of `data`: max block size code 4..7 (64 KiB .. 4 MiB), linked or independent blocks, optional block
    and content checksums and content size; the blocks whose indexes are in `stored` (or all, stored=True) are stored
    uncompressed (high bit of the block size)."""
    flg = 0x40 | (0x20 if independent else 0) | (0x10 if block_checksum else 0) | (0x08 if content_size else 0) | (
        0x04 if content_checksum else 0)
    desc = bytes([flg, block_code << 4]) + (struct.pack("<Q", len(data)) if content_size else b"")
    out = bytearray(struct.pack("<I", 0x184D2204) + desc + bytes([(xxh32(desc) >> 8) & 0xFF]))
    bs = 1 << (8 + 2 * block_code)
    for k, s in enumerate(range(0, len(data), bs)):
        e = min(s + bs, len(data))
        if stored is True or k in stored:
            body, word = data[s:e], (e - s) | 0x80000000
        else:
            body = lz4_block(data, s, e, s if independent else max(0, s - 65535), matches)
            word = len(body)
            if word >= e - s:  # incompressible: stored, as an encoder must when the block would outgrow its maximum
                body, word = data[s:e], (e - s) | 0x80000000
        out += struct.pack("<I", word) + body
        if block_checksum:
            out += struct.pack("<I", xxh32(body))
    out += struct.pack("<I", 0)
    if content_checksum:
        out += struct.pack("<I", xxh32(data))
    return bytes(out)


# frame errors, in the decoder's words and in their order of precedence
E_BAD, E_CSIZE, E_TRUNC, E_ZERO, E_OFFSET, E_OVERRUN, E_UNDERFILL, E_CHECKSUM, E_TRAIL = (
    "malformed LZ4 frame header", "LZ4 frame content size differs from the buffer's uncompressed length", "truncated LZ4 frame",
    "LZ4 match with offset 0", "LZ4 match reaches before the start of its output", "LZ4 frame overruns the buffer's uncompressed length",
    "LZ4 frame underfills the buffer's uncompressed length", "LZ4 frame checksum mismatch", "bytes after the end of the LZ4 frame")
E_OFFSETS, E_UTF8, E_NULLS = ("offsets are negative, decreasing or past the end of the data buffer", "invalid UTF-8 in a Utf8 value",
                              "null count differs from the validity bitmap")
CODES = [None, E_BAD, E_CSIZE, E_TRUNC, E_ZERO, E_OFFSET, E_OVERRUN, E_UNDERFILL, E_CHECKSUM, E_TRAIL, E_OFFSETS, E_UTF8, E_NULLS]


class Lz4Error(Exception):
    pass


def lz4_decode(f: bytes, ulen: int) -> bytes:
    """One frame that must decode to exactly `ulen` bytes (A3, A4, A8)."""
    n = len(f)
    if n < 7:
        raise Lz4Error(E_TRUNC)
    flg, bd = f[4], f[5]
    if struct.unpack_from("<I", f)[0] != 0x184D2204 or flg >> 6 != 1 or flg & 3 or bd & 0x8F or (bd >> 4) & 7 < 4:
        raise Lz4Error(E_BAD)
    indep, bsum, csize, csum = flg & 0x20, flg & 0x10, flg & 0x08, flg & 0x04
    max_block = 1 << (8 + 2 * ((bd >> 4) & 7))
    desc = 2 + (8 if csize else 0)
    if n < 4 + desc + 1:
        raise Lz4Error(E_TRUNC)
    if (xxh32(f[4:4 + desc]) >> 8) & 0xFF != f[4 + desc]:
        raise Lz4Error(E_CHECKSUM)
    if csize and struct.unpack_from("<Q", f, 6)[0] != ulen:
        raise Lz4Error(E_CSIZE)
    p = 4 + desc + 1
    out = bytearray()
    while True:
        if n - p < 4:
            raise Lz4Error(E_TRUNC)
        word = struct.unpack_from("<I", f, p)[0]
        p += 4
        if word == 0:
            break
        bsz = word & 0x7FFFFFFF
        if bsz > max_block:
            raise Lz4Error(E_BAD)
        if n - p < bsz + (4 if bsum else 0):
            raise Lz4Error(E_TRUNC)
        bend = p + bsz
        if bsum and xxh32(f[p:bend]) != struct.unpack_from("<I", f, bend)[0]:
            raise Lz4Error(E_CHECKSUM)
        block0 = len(out)
        if word >> 31:
            if bsz > ulen - len(out):
                raise Lz4Error(E_OVERRUN)
            out += f[p:bend]
        else:
            q = p
            while True:
                if q >= bend:
                    raise Lz4Error(E_TRUNC)
                tok = f[q]
                q += 1
                lit = tok >> 4
                if lit == 15:
                    while True:
                        if q >= bend:
                            raise Lz4Error(E_TRUNC)
                        b = f[q]
                        q += 1
                        lit += b
                        if b != 255:
                            break
                if lit > bend - q:
                    raise Lz4Error(E_TRUNC)
                if lit > ulen - len(out):
                    raise Lz4Error(E_OVERRUN)
                out += f[q:q + lit]
                q += lit
                if q == bend:
                    break
                if bend - q < 2:
                    raise Lz4Error(E_TRUNC)
                off = f[q] | (f[q + 1] << 8)
                q += 2
                if off == 0:
                    raise Lz4Error(E_ZERO)
                if off > len(out) - (block0 if indep else 0):
                    raise Lz4Error(E_OFFSET)
                ml = tok & 15
                if ml == 15:
                    while True:
                        if q >= bend:
                            raise Lz4Error(E_TRUNC)
                        b = f[q]
                        q += 1
                        ml += b
                        if b != 255:
                            break
                ml += 4
                if ml > ulen - len(out):
                    raise Lz4Error(E_OVERRUN)
                s = len(out) - off
                out += (out[s:] * (ml // off + 1))[:ml]  # a match longer than its offset repeats the offset's period
        p = bend + (4 if bsum else 0)
    if len(out) != ulen:
        raise Lz4Error(E_UNDERFILL)
    if csum:
        if n - p < 4:
            raise Lz4Error(E_TRUNC)
        if xxh32(bytes(out)) != struct.unpack_from("<I", f, p)[0]:
            raise Lz4Error(E_CHECKSUM)
        p += 4
    if p != n:
        raise Lz4Error(E_TRAIL)
    return bytes(out)


# ---------------------------------------------------------------------------------------------------------------------
# flatbuffers: a builder that lays every object out after the one that refers to it, and a bounds-checked reader

class T:
    """A table: `fields[i]` is None (absent), (fmt, value) for a scalar, or an object (T, Vec, Str, Structs)."""

    def __init__(self, *fields):
        self.fields = list(fields)


class Vec:  # a vector of tables
    def __init__(self, items):
        self.items = list(items)


class Str:
    def __init__(self, s):
        self.b = s.encode() if isinstance(s, str) else bytes(s)


class Structs:  # a vector of structs: `count` elements of raw bytes, 8-byte aligned
    def __init__(self, raw, count):
        self.raw, self.count = bytes(raw), count


def fb_build(root: T) -> bytes:
    buf = bytearray(4)
    todo = []

    def align(a, extra=0):
        while (len(buf) + extra) % a:
            buf.append(0)

    def place(obj):
        if isinstance(obj, T):
            layout, size = [], 4
            for i, f in enumerate(obj.fields):
                if f is None:
                    continue
                w = 4 if not isinstance(f, tuple) else struct.calcsize("<" + f[0])
                size = (size + w - 1) // w * w
                layout.append((i, size, f))
                size += w
            nslots = max([i for i, _, _ in layout], default=-1) + 1
            vt = struct.pack("<HH", 4 + 2 * nslots, size) + b"".join(
                struct.pack("<H", next((o for i, o, _ in layout if i == k), 0)) for k in range(nslots))
            align(8)
            vpos = len(buf)
            buf.extend(vt)
            align(8)
            tpos = len(buf)
            buf.extend(bytes(size))
            struct.pack_into("<i", buf, tpos, tpos - vpos)
            for i, o, f in layout:
                if isinstance(f, tuple):
                    struct.pack_into("<" + f[0], buf, tpos + o, f[1])
                else:
                    todo.append((tpos + o, f))
            return tpos
        if isinstance(obj, Vec):
            align(4)
            pos = len(buf)
            buf.extend(struct.pack("<I", len(obj.items)) + bytes(4 * len(obj.items)))
            for k, it in enumerate(obj.items):
                todo.append((pos + 4 + 4 * k, it))
            return pos
        if isinstance(obj, Structs):
            align(8, 4)
            pos = len(buf)
            buf.extend(struct.pack("<I", obj.count) + obj.raw)
            return pos
        align(4)
        pos = len(buf)
        buf.extend(struct.pack("<I", len(obj.b)) + obj.b + b"\0")
        return pos

    struct.pack_into("<I", buf, 0, place(root))
    while todo:
        at, obj = todo.pop(0)
        struct.pack_into("<I", buf, at, place(obj) - at)
    align(8)
    return bytes(buf)


class FbError(Exception):
    pass


class FbT:
    def __init__(self, b: bytes, pos: int):
        self.b, self.pos = b, pos
        soff = self._rd("<i", pos)
        self.vt = pos - soff
        if self.vt < 0 or self.vt >= len(b):
            raise FbError()
        self.vlen = self._rd("<H", self.vt)
        if self.vlen < 4 or self.vlen & 1:
            raise FbError()

    def _rd(self, fmt, at):
        if at < 0 or at + struct.calcsize(fmt) > len(self.b):
            raise FbError()
        return struct.unpack_from(fmt, self.b, at)[0]

    def field(self, i):
        if 4 + 2 * i + 2 > self.vlen:
            return 0
        o = self._rd("<H", self.vt + 4 + 2 * i)
        return self.pos + o if o else 0

    def scalar(self, i, fmt, dflt=0):
        f = self.field(i)
        return self._rd(fmt, f) if f else dflt

    def table(self, i):
        f = self.field(i)
        return FbT(self.b, f + self._rd("<I", f)) if f else None

    def vec(self, i, elem):
        f = self.field(i)
        if not f:
            return 0, 0
        v = f + self._rd("<I", f)
        cnt = self._rd("<I", v)
        if v + 4 > len(self.b) or cnt > (len(self.b) - v - 4) // elem:
            raise FbError()
        return v + 4, cnt

    def elem_table(self, v, k):
        e = v[0] + 4 * k
        return FbT(self.b, e + self._rd("<I", e))

    def string(self, i):
        v = self.vec(i, 1)
        return self.b[v[0]:v[0] + v[1]].decode("utf-8", "replace") if v[1] else ""


def fb_root(b: bytes) -> FbT:
    if len(b) < 4:
        raise FbError()
    return FbT(b, struct.unpack_from("<I", b)[0])


# ---------------------------------------------------------------------------------------------------------------------
# types

TYPE_NAMES = ["NONE", "Null", "Int", "FloatingPoint", "Binary", "Utf8", "Bool", "Decimal", "Date", "Time", "Timestamp", "Interval", "List",
              "Struct", "Union", "FixedSizeBinary", "FixedSizeList", "Map", "Duration", "LargeBinary", "LargeUtf8", "LargeList",
              "RunEndEncoded", "BinaryView", "Utf8View", "ListView", "LargeListView"]
WIDTH = {pa.int32(): 4, pa.uint32(): 4, pa.float32(): 4, pa.int64(): 8, pa.uint64(): 8, pa.float64(): 8}


def _nbuf(t):
    return 0 if t == pa.null() else 3 if t in (pa.utf8(), pa.binary()) else 2


def _type_of(fl: FbT):
    """(pyarrow type or None, description)"""
    tt = fl.scalar(2, "<B")
    t = fl.table(3)
    desc, r = TYPE_NAMES[tt] if tt < len(TYPE_NAMES) else "unknown", None
    if tt == 1:
        r = pa.null()
    elif tt == 2:
        bits = t.scalar(0, "<i") if t else 0
        sig = bool(t.scalar(1, "<B")) if t else False
        desc = ("Int" if sig else "UInt") + str(bits)
        r = {(32, True): pa.int32(), (32, False): pa.uint32(), (64, True): pa.int64(), (64, False): pa.uint64()}.get((bits, sig))
    elif tt == 3:
        prec = t.scalar(0, "<h") if t else 0
        desc = ("Float16", "Float32", "Float64")[prec] if 0 <= prec <= 2 else "Float64"
        r = {1: pa.float32(), 2: pa.float64()}.get(prec)
    elif tt in (4, 5, 6):
        r = {4: pa.binary(), 5: pa.utf8(), 6: pa.bool_()}[tt]
    if fl.table(4) is not None:
        return None, "dictionary-encoded " + desc
    return r, desc


def _type_table(t):
    """(union tag, type table) for writing a supported pyarrow type (Int8 etc. for the Unsupported tests too)."""
    if pa.types.is_integer(t):
        return 2, T(("i", t.bit_width), ("B", int(pa.types.is_signed_integer(t))))
    if pa.types.is_floating(t):
        return 3, T(("h", {16: 0, 32: 1, 64: 2}[t.bit_width]))
    tags = {pa.null(): 1, pa.binary(): 4, pa.utf8(): 5, pa.bool_(): 6, pa.large_binary(): 19, pa.large_utf8(): 20,
            pa.date32(): 8, pa.binary_view(): 23, pa.string_view(): 24}
    return tags[t], T()


# ---------------------------------------------------------------------------------------------------------------------
# writer

@dataclass
class Stored:
    """One record batch as written: `nodes` [(length, null_count)] per field, `buffers` the body bytes of each buffer
    (for a compressed body: prefix and frame), `compression` None, 0 (LZ4_FRAME) or 1 (ZSTD)."""
    rows: int
    nodes: List[tuple]
    buffers: List[bytes]
    compression: Optional[int] = None
    gaps: List[int] = dfield(default_factory=list)  # extra padding before each buffer (multiples of 8 keep alignment)


def _arrow_buffers(a: pa.Array):
    """The IPC body buffers of an unsliced array: validity (empty when it has no NULLs), then values or offsets + data."""
    n = len(a)
    t = a.type
    if t == pa.null():
        return []
    bufs = a.buffers()
    nb = (n + 7) // 8
    val = bufs[0].to_pybytes()[:nb] if (a.null_count and bufs[0] is not None) else b""
    if t in (pa.utf8(), pa.binary()):
        offs = bufs[1].to_pybytes()[:4 * (n + 1)] if n else b""
        end = struct.unpack_from("<i", offs, 4 * n)[0] if n else 0
        return [val, offs, bufs[2].to_pybytes()[:end] if bufs[2] is not None else b""]
    if t == pa.bool_():
        return [val, bufs[1].to_pybytes()[:nb]]
    return [val, bufs[1].to_pybytes()[:n * WIDTH[t]]]


def compress_buffer(buf: bytes, raw: bool = False, **frame) -> bytes:
    """prefix + LZ4 frame; raw=True stores the buffer raw behind a -1 prefix; an empty buffer stays empty."""
    if not buf:
        return b""
    if raw:
        return struct.pack("<q", -1) + buf
    return struct.pack("<q", len(buf)) + lz4_frame(buf, **frame)


def stored_from_arrow(rb: pa.RecordBatch, lz4=None, **frame) -> Stored:
    """`lz4`: None (uncompressed body) or True; `frame`: lz4_frame's knobs (or raw=True) for every buffer."""
    assert all(c.offset == 0 for c in rb.columns), "stored_from_arrow takes unsliced arrays"
    nodes, bufs = [], []
    for a in rb.columns:
        nodes.append((len(a), a.null_count))
        for b in _arrow_buffers(a):
            bufs.append(compress_buffer(b, **dict(frame)) if lz4 else b)
    return Stored(rb.num_rows, nodes, bufs, 0 if lz4 else None)


def _pad8(b: bytes) -> bytes:
    return b + bytes(-len(b) % 8)


def _message(header_type, header, body_len, legacy):
    fb = fb_build(T(("h", 4), ("B", header_type), header, ("q", body_len)))
    if legacy:
        fb = fb + bytes(-(len(fb) + 4) % 8)
        return struct.pack("<i", len(fb)) + fb
    fb = fb + bytes(-(len(fb) + 8) % 8)
    return struct.pack("<Ii", 0xFFFFFFFF, len(fb)) + fb


def _schema_table(fields, big_endian=False):
    """fields: [(name, pyarrow type, nullable)] or (name, type, nullable, 'dict') for a dictionary-encoded field."""
    fts = []
    for f in fields:
        tag, tt = _type_table(f[1])
        dict_enc = T(("q", 0), T(("i", 32), ("B", 1))) if len(f) > 3 and f[3] == "dict" else None
        fts.append(T(Str(f[0]), ("B", int(f[2])), ("B", tag), tt, dict_enc, Vec([])))
    return T(("h", int(big_endian)), Vec(fts))


def write_ipc(fields, batches: List[Stored], legacy=False, big_endian=False) -> bytes:
    """An IPC file: magic, schema message, the batches' messages and bodies, footer, footer length, magic."""
    out = bytearray(MAGIC + b"\0\0")
    out += _message(1, _schema_table(fields, big_endian), 0, legacy)
    blocks = []
    for s in batches:
        body, bspec = bytearray(), bytearray()
        for b, g in zip(s.buffers, s.gaps or [0] * len(s.buffers)):
            body += bytes(g)
            bspec += struct.pack("<qq", len(body), len(b))
            body += _pad8(b)
        nodes = b"".join(struct.pack("<qq", *nd) for nd in s.nodes)
        comp = None if s.compression is None else T(("b", s.compression), ("b", 0))
        meta = _message(3, T(("q", s.rows), Structs(nodes, len(s.nodes)), Structs(bspec, len(s.buffers)), comp), len(body), legacy)
        blocks.append(struct.pack("<qiiq", len(out), len(meta), 0, len(body)))
        out += meta + body
    footer = fb_build(T(("h", 4), _schema_table(fields, big_endian), Structs(b"", 0), Structs(b"".join(blocks), len(blocks))))
    out += footer + struct.pack("<i", len(footer)) + MAGIC
    return bytes(out)


# ---------------------------------------------------------------------------------------------------------------------
# reader

def _e(what, k=None, col=None, row=None):
    where = []
    if k is not None:
        where.append("record batch %d" % k)
    if col is not None:
        where.append("column '%s'" % col)
    if row is not None:
        where.append("row %d" % row)
    return OracleError("Process", PFX + what + (" (" + ", ".join(where) + ")" if where else ""))


def _unsupported(msg):
    return OracleError("Unsupported", "arrow input: " + msg)


@dataclass
class _Batch:
    k: int
    rows: int
    first_row: int
    nodes: list
    bufs: list  # per field: [(src, len, size, lz4)] * n_buffers


def parse_file(data: bytes):
    """connect(): (fields [(name, type, nullable)], stored batches); raises OracleError."""
    n = len(data)
    if n < 18 or data[:6] != MAGIC or data[-6:] != MAGIC:
        raise _e("not an Arrow IPC file (bad magic)")
    flen = struct.unpack_from("<i", data, n - 10)[0]
    if flen <= 0 or flen > n - 18:
        raise _e("footer out of range")
    foot = n - 10 - flen
    fb = data[foot:foot + flen]
    fields, blocks = [], []
    try:
        footer = fb_root(fb)
        schema = footer.table(1)
        if schema is None:
            raise _e("the footer has no schema")
        if schema.scalar(0, "<h") != 0:
            raise _unsupported("the schema is big-endian, which is not decoded on the GPU")
        fv = schema.vec(1, 4)
        if fv[1] > 1024:
            raise _unsupported("more than 1024 fields in a schema")
        for i in range(fv[1]):
            fl = schema.elem_table(fv, i)
            name = fl.string(0)
            t, desc = _type_of(fl)
            if t is None:
                raise _unsupported("field '%s' has type %s, which is not decoded on the GPU" % (name, desc))
            fields.append((name, t, bool(fl.scalar(1, "<B"))))
        rv = footer.vec(3, 24)
        for k in range(rv[1]):
            blocks.append(struct.unpack_from("<qi4xq", fb, rv[0] + 24 * k))
    except FbError:
        raise _e("malformed footer")
    out, rows = [], 0
    for k, (off, meta_len, body_len) in enumerate(blocks):
        b = _read_batch(data, fields, k, off, meta_len, body_len, foot)
        b.first_row = rows
        rows += b.rows
        out.append(b)
    return fields, out


def _read_batch(data, fields, k, off, meta_len, body_len, end):
    if off < 8 or meta_len < 8 or body_len < 0 or meta_len > end - off or body_len > end - off - meta_len:
        raise _e("block outside the file", k)
    meta = data[off:off + meta_len]
    fb0, ln = 4, struct.unpack_from("<i", meta)[0]
    if ln == -1:
        fb0, ln = 8, struct.unpack_from("<i", meta, 4)[0]
    if ln <= 0 or ln > meta_len - fb0:
        raise _e("malformed message", k)
    fb = meta[fb0:fb0 + ln]
    body = off + meta_len
    nbuf = sum(_nbuf(t) for _, t, _ in fields)
    lz4 = False
    try:
        msg = fb_root(fb)
        if msg.scalar(1, "<B") != 3:
            raise _e("message is not a record batch", k)
        rb = msg.table(2)
        if rb is None:
            raise FbError()
        rows = rb.scalar(0, "<q")
        if rows < 0:
            raise _e("negative row count", k)
        if rows > ROW_LAST:
            raise _unsupported("record batch %d holds more than 2^31 - 1 rows" % k)
        nv, bv = rb.vec(1, 16), rb.vec(2, 16)
        if nv[1] != len(fields):
            raise _e("field node count differs from the schema", k)
        if bv[1] != nbuf:
            raise _e("buffer count differs from the schema", k)
        nodes = [struct.unpack_from("<qq", fb, nv[0] + 16 * c) for c in range(nv[1])]
        specs = [struct.unpack_from("<qq", fb, bv[0] + 16 * j) for j in range(bv[1])]
        comp = rb.table(3)
        if comp is not None:
            codec = comp.scalar(0, "<b")
            if codec == 1:
                raise _unsupported("record batch %d has a ZSTD body, which is not decoded on the GPU (uncompressed and LZ4_FRAME are)" % k)
            if codec != 0 or comp.scalar(1, "<b") != 0:
                raise _e("unknown body compression", k)
            lz4 = True
    except FbError:
        raise _e("malformed message", k)
    j, bufs = 0, []
    for (name, t, nullable), (length, nulls) in zip(fields, nodes):
        if length != rows:
            raise _e("node length differs from the batch length", k, name)
        if nulls < 0 or nulls > length:
            raise _e("invalid null count", k, name)
        if not nullable and nulls > 0 and t != pa.null():
            raise _e("null values in a non-nullable field", k, name)
        cb = []
        for _ in range(_nbuf(t)):
            o, ln = specs[j]
            j += 1
            if o < 0 or ln < 0 or o > body_len or ln > body_len - o:
                raise _e("buffer outside the body", k, name)
            if (body + o) % 8:
                raise _e("buffer not 8-byte aligned", k, name)
            src, size, is_lz4 = body + o, ln, False
            if lz4 and ln > 0:
                if ln < 8:
                    raise _e("buffer shorter than its length prefix", k, name)
                u = struct.unpack_from("<q", data, body + o)[0]
                src, ln = src + 8, ln - 8
                if u == -1:
                    size = ln
                elif u == 0:
                    size = ln = 0
                elif u < 0:
                    raise _e("invalid uncompressed length", k, name)
                else:
                    size, is_lz4 = u, True
            cb.append((src, ln, size, is_lz4))
        nb = (length + 7) // 8
        short = nulls > 0 and t != pa.null() and cb[0][2] < nb
        if t in WIDTH:
            short = short or cb[1][2] < length * WIDTH[t]
        if t == pa.bool_():
            short = short or cb[1][2] < nb
        if t in (pa.utf8(), pa.binary()) and length > 0:
            short = short or cb[1][2] < 4 * (length + 1)
        if short:
            raise _e("buffer too short for its node", k, name)
        bufs.append(cb)
    return _Batch(k, rows, 0, nodes, bufs)


def _check_batch(data, fields, b: _Batch):
    """The read-time checks of one stored batch: the first failure, or None."""
    for (name, t, _), (length, nulls), cb in zip(fields, b.nodes, b.bufs):
        raw, codes = [], []
        for src, ln, size, is_lz4 in cb:
            if is_lz4:
                try:
                    raw.append(lz4_decode(data[src:src + ln], size))
                except Lz4Error as e:
                    codes.append(CODES.index(str(e)))
                    raw.append(b"")
            else:
                raw.append(data[src:src + size])
        if codes:
            return _e(CODES[min(codes)], b.k, name)
        if t in (pa.utf8(), pa.binary()) and length > 0:
            offs = struct.unpack_from("<%di" % (length + 1), raw[1])
            for r in range(length):
                a, e = offs[r], offs[r + 1]
                if a < 0 or e < a or e > len(raw[2]):
                    return _e(E_OFFSETS, b.k, name, r)
                if t == pa.utf8():
                    try:
                        raw[2][a:e].decode("utf-8")
                    except UnicodeDecodeError:
                        return _e(E_UTF8, b.k, name, r)
        if nulls > 0 and t != pa.null():
            zeros = sum(1 for r in range(length) if not (raw[0][r >> 3] >> (r & 7)) & 1)
            if zeros != nulls:
                return _e(E_NULLS, b.k, name)
    return None


def read_ipc(data: bytes, batch_rows: Optional[int] = None):
    """(batches, error): what the input yields up to EOF (error None) or up to its first other error."""
    try:
        fields, stored = parse_file(data)
    except OracleError as e:
        return [], e
    batch_rows = batch_rows or (1 << 22)
    schema = pa.schema([pa.field(nm, t, nullable=nl) for nm, t, nl in fields])
    total = sum(b.rows for b in stored)
    reader = None
    checked = set()
    out = []
    for r0 in range(0, total, batch_rows):
        n = min(batch_rows, total - r0)
        touched = [b for b in stored if b.rows and b.first_row < r0 + n and b.first_row + b.rows > r0]
        for b in touched:
            if b.k not in checked:
                err = _check_batch(data, fields, b)
                if err is not None:
                    return out, err
                checked.add(b.k)
        if reader is None:
            reader = pa.ipc.open_file(pa.BufferReader(data))
        pieces = []
        for b in touched:
            a = max(r0, b.first_row) - b.first_row
            e = min(r0 + n, b.first_row + b.rows) - b.first_row
            got = reader.get_batch(b.k)
            pieces.append(pa.record_batch(got.slice(a, e - a).columns, schema=schema))
        out.append(pa.concat_batches(pieces) if len(pieces) > 1 else pieces[0])
    return out, None
