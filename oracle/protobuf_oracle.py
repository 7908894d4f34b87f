"""CPU oracle for `protobuf_to_arrow` / `arrow_to_protobuf` — TEST INFRASTRUCTURE (see oracle/__init__.py).

A pure-Python restatement of the protobuf wire format and of the conversions in
crates/arkflow-plugin/src/component/protobuf.rs:115-339 (prost-reflect 0.16's DynamicMessage, third-party, not
vendored).  It does not use google.protobuf, so GPU tests can import it; tests/test_protobuf_oracle.py checks it
against google.protobuf (upb).

A message schema is a list of `PbField`s in declaration order (what the `.proto` file declares).

protobuf_to_arrow (MessageBatch::to_binary + DynamicMessage::decode + one column per field):
  * NULL payloads are dropped; every other payload, a zero-length one included, is one row;
  * one non-nullable column per field, in declaration order, typed by ARROW_TYPE;
  * an absent field takes its default: the proto2 [default = …] value, else 0 / 0.0 / false / "" / b"" / the enum's
    first value;
  * of the members of one oneof only the last one on the wire keeps its value, the others take their defaults (merging a
    oneof member clears the others);
  * unknown fields are skipped (groups up to their matching end-group);
  * errors ("Protobuf message parsing failed"): truncated buffer, varint longer than 10 bytes (or a 10th byte > 1),
    key beyond 32 bits, field number 0, wire type 6 or 7, a known field with the wrong wire type, an end-group that
    closes no open group, a `string` value that is not UTF-8;
  * a repeated / map / message field: "Unsupported field type: <name>" for every non-empty batch.
arrow_to_protobuf (DynamicMessage::set_field_by_name per column + encode):
  * columns in schema order; a column whose name is a field and whose Arrow type is ARROW_TYPE[kind] sets that field
    for every row (NULL slots: the value buffer's contents), other columns are ignored; setting a oneof member clears
    the others;
  * fields are written in ascending field-number order;
  * a field without explicit presence is left out when it holds its zero value (0, false, "", b"", and for float /
    double any value == 0.0, so -0.0 too);
  * the output is the input batch plus a non-null Binary `__value__` column.

ASSUMPTIONS (prost-reflect's sources were not available to check them; each is the prost / protobuf-spec behaviour):
  A1. a proto3 float / double field without presence counts as default when `value == 0.0` (prost's `!= 0.0`), so
      -0.0 is left out; upb compares bits and writes it;
  A2. protobuf_to_arrow's columns follow declaration order (MessageDescriptor::fields());
  A3. when a field occurs more than once in a payload, the last occurrence wins (scalars are merged by replacement);
  A4. unknown groups nest at most 100 deep (prost's recursion limit); a deeper nesting is a parse error;
  A5. a missing proto2 `required` field is not an error (DynamicMessage::decode does not check required fields).
"""
from __future__ import annotations

import struct
from dataclasses import dataclass
from typing import Any, Optional

import numpy as np
import pyarrow as pa

DEFAULT_BINARY_VALUE_FIELD = "__value__"

VARINT, I64, LEN, SGROUP, EGROUP, I32 = 0, 1, 2, 3, 4, 5

SCALAR_KINDS = ("double", "float", "int64", "uint64", "int32", "fixed64", "fixed32", "bool", "string", "bytes",
                "uint32", "sfixed32", "sfixed64", "sint32", "sint64", "enum")

WIRE = {"double": I64, "fixed64": I64, "sfixed64": I64, "float": I32, "fixed32": I32, "sfixed32": I32,
        "string": LEN, "bytes": LEN}  # every other scalar kind: VARINT

ARROW_TYPE = {"bool": pa.bool_(), "int32": pa.int32(), "sint32": pa.int32(), "sfixed32": pa.int32(), "enum": pa.int32(),
              "int64": pa.int64(), "sint64": pa.int64(), "sfixed64": pa.int64(), "uint32": pa.uint32(),
              "fixed32": pa.uint32(), "uint64": pa.uint64(), "fixed64": pa.uint64(), "float": pa.float32(),
              "double": pa.float64(), "string": pa.utf8(), "bytes": pa.binary()}

_NP = {pa.int32(): np.int32, pa.int64(): np.int64, pa.uint32(): np.uint32, pa.uint64(): np.uint64,
       pa.float32(): np.uint32, pa.float64(): np.uint64}  # floats are handled as their IEEE bits


class ProtobufError(Exception):
    """`kind` / `message` as the processor raises them (arkflow_core::Error)."""

    def __init__(self, kind: str, message: str):
        super().__init__(message)
        self.kind, self.message = kind, message


@dataclass
class PbField:
    name: str
    number: int
    kind: str                     # a SCALAR_KINDS entry, or "message"
    presence: bool = False        # proto2 optional / required, proto3 `optional`, oneof members
    default: Any = None           # the value of an absent field; None: the kind's zero (enum: give the first value)
    repeated: bool = False        # repeated and map fields
    oneof: Optional[int] = None

    def zero(self):
        if self.default is not None:
            return self.default
        return {"string": "", "bytes": b"", "bool": False, "float": 0.0, "double": 0.0}.get(self.kind, 0)


# ---- wire primitives ---------------------------------------------------------------------------------------------
def put_varint(out: bytearray, v: int) -> None:
    v &= (1 << 64) - 1
    while v >= 0x80:
        out.append((v & 0x7F) | 0x80)
        v >>= 7
    out.append(v)


def zigzag32(n: int) -> int:
    return ((n << 1) ^ (n >> 31)) & 0xFFFFFFFF


def zigzag64(n: int) -> int:
    return ((n << 1) ^ (n >> 63)) & 0xFFFFFFFFFFFFFFFF


def unzigzag(v: int) -> int:
    return (v >> 1) ^ -(v & 1)


def _signed(v: int, bits: int) -> int:
    v &= (1 << bits) - 1
    return v - (1 << bits) if v >> (bits - 1) else v


def f32_bits(x: float) -> int:
    return struct.unpack("<I", struct.pack("<f", x))[0]


def f64_bits(x: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", x))[0]


class _Reader:
    __slots__ = ("b", "p", "end")

    def __init__(self, b: bytes):
        self.b, self.p, self.end = b, 0, len(b)

    def fail(self, why: str):
        raise ProtobufError("Process", "Protobuf message parsing failed: " + why)

    def varint(self) -> int:
        v = 0
        for s in range(10):
            if self.p >= self.end:
                self.fail("buffer underflow")
            b = self.b[self.p]
            self.p += 1
            if s == 9 and b > 1:
                self.fail("invalid varint")
            v |= (b & 0x7F) << (7 * s)
            if b < 0x80:
                return v
        self.fail("invalid varint")

    def key(self):
        k = self.varint()
        if k > 0xFFFFFFFF:
            self.fail("invalid key value")
        wire = k & 7
        if wire > 5:
            self.fail("invalid wire type value")
        num = k >> 3
        if num == 0:
            self.fail("invalid tag value: 0")
        return num, wire

    def take(self, n: int) -> bytes:
        if n > self.end - self.p:
            self.fail("buffer underflow")
        v = self.b[self.p:self.p + n]
        self.p += n
        return v

    def skip(self, num: int, wire: int) -> None:
        open_groups = []
        while True:
            if wire == VARINT:
                self.varint()
            elif wire == I64:
                self.take(8)
            elif wire == I32:
                self.take(4)
            elif wire == LEN:
                self.take(self.varint())
            elif wire == SGROUP:
                if len(open_groups) == 100:  # A4
                    self.fail("recursion limit reached")
                open_groups.append(num)
            else:  # EGROUP
                if not open_groups or open_groups[-1] != num:
                    self.fail("unexpected end group tag")
                open_groups.pop()
            if not open_groups:
                return
            num, wire = self.key()


# ---- one message ---------------------------------------------------------------------------------------------------
def decode_message_raw(fields: list[PbField], data: bytes) -> dict:
    """field name → value; float / double values as their IEEE bits (int), absent fields at their default."""
    by_num = {f.number: f for f in fields}
    r = _Reader(bytes(data))
    got = {}
    while r.p < r.end:
        num, wire = r.key()
        f = by_num.get(num)
        if f is None or f.kind == "message" or f.repeated:
            r.skip(num, wire)  # (a batch with such fields never gets here: protobuf_to_arrow rejects it first)
            continue
        if wire != WIRE.get(f.kind, VARINT):
            r.fail("invalid wire type")
        k = f.kind
        if wire == VARINT:
            v = r.varint()
            if k in ("int32", "enum"):
                v = _signed(v, 32)
            elif k == "int64":
                v = _signed(v, 64)
            elif k == "uint32":
                v &= 0xFFFFFFFF
            elif k == "sint32":
                v = unzigzag(v & 0xFFFFFFFF)
            elif k == "sint64":
                v = unzigzag(v)
            elif k == "bool":
                v = v != 0
        elif wire == I32:
            v = int.from_bytes(r.take(4), "little")
            if k == "sfixed32":
                v = _signed(v, 32)
        elif wire == I64:
            v = int.from_bytes(r.take(8), "little")
            if k == "sfixed64":
                v = _signed(v, 64)
        else:
            raw = r.take(r.varint())
            if k == "string":
                try:
                    v = raw.decode("utf-8")
                except UnicodeDecodeError:
                    r.fail("invalid string value: data is not UTF-8 encoded")
            else:
                v = bytes(raw)
        if f.oneof is not None:  # a oneof keeps only its last member read: the others take their defaults
            for g in fields:
                if g.oneof == f.oneof:
                    got.pop(g.name, None)
        got[f.name] = v  # A3: the last occurrence wins
    out = {}
    for f in fields:
        if f.name in got:
            out[f.name] = got[f.name]
        else:
            z = f.zero()
            out[f.name] = f32_bits(z) if f.kind == "float" else f64_bits(z) if f.kind == "double" else z
    return out


def decode_message(fields: list[PbField], data: bytes) -> dict:
    """field name → Python value (floats as floats)."""
    raw = decode_message_raw(fields, data)
    for f in fields:
        if f.kind == "float":
            raw[f.name] = struct.unpack("<f", struct.pack("<I", raw[f.name]))[0]
        elif f.kind == "double":
            raw[f.name] = struct.unpack("<d", struct.pack("<Q", raw[f.name]))[0]
    return raw


def encode_message(fields: list[PbField], values: dict) -> bytes:
    """Canonical encoding of the fields present in `values` (floats may be given as floats, or as IEEE bits ints when
    `values` comes from an Arrow column: see _column_values)."""
    out = bytearray()
    for f in sorted(fields, key=lambda f: f.number):
        if f.name not in values:
            continue
        v, k = values[f.name], f.kind
        if k == "float" and isinstance(v, float):
            v = f32_bits(v)
        elif k == "double" and isinstance(v, float):
            v = f64_bits(v)
        if not f.presence and f.oneof is None:  # implicit presence: zero values are not written (A1 for floats)
            if k == "float":
                if struct.unpack("<f", struct.pack("<I", v))[0] == 0.0:
                    continue
            elif k == "double":
                if struct.unpack("<d", struct.pack("<Q", v))[0] == 0.0:
                    continue
            elif not v:
                continue
        wire = WIRE.get(k, VARINT)
        put_varint(out, (f.number << 3) | wire)
        if k in ("int32", "enum", "int64", "uint32", "uint64"):
            put_varint(out, int(v))  # negative int32 / enum: sign-extended to 64 bits, 10 bytes
        elif k == "bool":
            put_varint(out, 1 if v else 0)
        elif k == "sint32":
            put_varint(out, zigzag32(int(v)))
        elif k == "sint64":
            put_varint(out, zigzag64(int(v)))
        elif wire == I32:
            out += (int(v) & 0xFFFFFFFF).to_bytes(4, "little")
        elif wire == I64:
            out += (int(v) & 0xFFFFFFFFFFFFFFFF).to_bytes(8, "little")
        else:
            b = v.encode("utf-8") if isinstance(v, str) else bytes(v)
            put_varint(out, len(b))
            out += b
    return bytes(out)


# ---- batches -------------------------------------------------------------------------------------------------------
def _unsupported(fields: list[PbField]) -> Optional[PbField]:
    return next((f for f in fields if f.repeated or f.kind == "message"), None)


def protobuf_to_arrow(fields: list[PbField], rb: pa.RecordBatch, value_field: str = DEFAULT_BINARY_VALUE_FIELD) -> Optional[pa.RecordBatch]:
    """None for an empty batch (ProcessResult::None)."""
    if rb.num_rows == 0:
        return None
    if value_field not in rb.schema.names:
        raise ProtobufError("Process", "not found column")
    col = rb.column(value_field)
    if col.type != pa.binary():
        raise ProtobufError("Process", "not support data type")
    bad = _unsupported(fields)
    if bad is not None:
        raise ProtobufError("Process", f"Unsupported field type: {bad.name}")
    msgs = [decode_message_raw(fields, v.as_py()) for v in col if v.is_valid]
    if not fields and msgs:
        raise ProtobufError("Process", "Creating an Arrow record batch failed: Invalid argument error: must either specify a row count or at least one column")
    arrays = []
    for f in fields:
        t = ARROW_TYPE[f.kind]
        vals = [m[f.name] for m in msgs]
        if f.kind == "float":
            arrays.append(pa.array(np.array(vals, dtype=np.uint32).view(np.float32), t))
        elif f.kind == "double":
            arrays.append(pa.array(np.array(vals, dtype=np.uint64).view(np.float64), t))
        else:
            arrays.append(pa.array(vals, t))
    return pa.RecordBatch.from_arrays(arrays, schema=pa.schema([pa.field(f.name, ARROW_TYPE[f.kind], nullable=False) for f in fields]))


def _column_values(arr: pa.Array) -> list:
    """Every slot's value read from the value buffer, NULL slots included; floats as IEEE bits."""
    n, off = len(arr), arr.offset
    bufs = arr.buffers()
    if arr.type == pa.bool_():
        bits = np.frombuffer(bufs[1], dtype=np.uint8)
        idx = np.arange(off, off + n)
        return [bool(b) for b in (bits[idx >> 3] >> (idx & 7)) & 1]
    if arr.type in (pa.utf8(), pa.binary()):
        offs = np.frombuffer(bufs[1], dtype=np.int32)[off:off + n + 1]
        data = bufs[2].to_pybytes() if bufs[2] is not None else b""
        return [data[offs[i]:offs[i + 1]] for i in range(n)]
    return np.frombuffer(bufs[1], dtype=_NP[arr.type])[off:off + n].tolist()


def arrow_to_protobuf_values(fields: list[PbField], rb: pa.RecordBatch, fields_to_include=None) -> Optional[list[bytes]]:
    """The `__value__` payloads; None for an empty batch."""
    if rb.num_rows == 0:
        return None
    names = rb.schema.names
    kept = [i for i, nm in enumerate(names) if fields_to_include is None or nm in fields_to_include]
    if fields_to_include is not None and not kept:
        raise ProtobufError("Process", "Creating an Arrow record batch failed: Invalid argument error: all columns in a record batch must have the same length")
    by_name = {f.name: f for f in fields}
    setters = {}  # field name → column values
    for i in kept:
        f = by_name.get(names[i])
        if f is None:
            continue
        if f.kind == "message":
            raise ProtobufError("Process", f"Unsupported Protobuf type: Message({f.name})")
        if rb.column(i).type != ARROW_TYPE[f.kind]:
            continue
        if f.repeated:
            raise ProtobufError("Unsupported", f"arrow_to_protobuf: column '{names[i]}' sets repeated field '{f.name}'")
        if f.oneof is not None:
            for g in fields:
                if g.oneof == f.oneof:
                    setters.pop(g.name, None)
        setters[f.name] = _column_values(rb.column(i))
    return [encode_message(fields, {k: v[r] for k, v in setters.items()}) for r in range(rb.num_rows)]


def arrow_to_protobuf(fields: list[PbField], rb: pa.RecordBatch, fields_to_include=None) -> Optional[pa.RecordBatch]:
    vals = arrow_to_protobuf_values(fields, rb, fields_to_include)
    if vals is None:
        return None
    return pa.RecordBatch.from_arrays(list(rb.columns) + [pa.array(vals, pa.binary())],
                                      schema=pa.schema(list(rb.schema) + [pa.field(DEFAULT_BINARY_VALUE_FIELD, pa.binary(), nullable=False)]))


def proto_text(package: str, message: str, fields: list[PbField], syntax: str = "proto3", enum_values=(("E0", 0), ("E1", 1))) -> str:
    """The `.proto` source declaring `fields` (scalar kinds; `enum` fields use one enum `Kind` with `enum_values`)."""
    lines = [f'syntax = "{syntax}";', f"package {package};", f"enum Kind {{ {' '.join(f'{n} = {v};' for n, v in enum_values)} }}",
             f"message {message} {{"]
    oneofs: dict[int, list[str]] = {}
    order: list = []  # a oneof block stands where its first member is declared
    for f in fields:
        t = "Kind" if f.kind == "enum" else f.kind
        if f.repeated:
            label = "repeated "
        elif f.oneof is None and (syntax == "proto2" or f.presence):
            label = "optional "
        else:
            label = ""
        opt = ""
        if f.default is not None and syntax == "proto2":
            d = f.default
            if f.kind == "enum":
                d = next(n for n, v in enum_values if v == d)
            elif f.kind == "bool":
                d = "true" if d else "false"
            elif f.kind in ("string", "bytes"):
                b = d.encode() if isinstance(d, str) else d
                d = '"' + "".join(f"\\{c:03o}" for c in b) + '"'
            elif f.kind in ("float", "double"):
                d = "inf" if d == float("inf") else "-inf" if d == float("-inf") else "nan" if d != d else repr(float(d))
            opt = f" [default = {d}]"
        decl = f"{label}{t} {f.name} = {f.number}{opt};"
        if f.oneof is not None:
            if f.oneof not in oneofs:
                order.append(f.oneof)
            oneofs.setdefault(f.oneof, []).append(decl)
        else:
            order.append(decl)
    for item in order:
        lines.append(f"  oneof choice{item} {{ " + " ".join(oneofs[item]) + " }" if isinstance(item, int) else "  " + item)
    lines.append("}")
    return "\n".join(lines) + "\n"
