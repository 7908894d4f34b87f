"""oracle/protobuf_oracle.py against google.protobuf (upb) on randomized messages of every scalar kind.

The descriptors are built with descriptor_pb2 (no protoc).  Where prost and upb differ the oracle follows prost and the
case is left out of the comparison: a proto3 float / double holding -0.0 (prost compares `!= 0.0` and leaves it out, upb
compares bits and writes it), a known field arriving with the wrong wire type (upb keeps it as an unknown field), a
10-byte varint whose last byte is above 1 (upb drops the excess bits), a proto2 enum value outside the enum (upb keeps
it as an unknown field)."""
import math
import struct

import numpy as np
import pytest

from oracle.protobuf_oracle import (PbField, ProtobufError, decode_message, encode_message, f32_bits, f64_bits, put_varint,
                                    zigzag32, zigzag64)

descriptor_pb2 = pytest.importorskip("google.protobuf.descriptor_pb2")
from google.protobuf import descriptor_pool, message_factory  # noqa: E402

_T = descriptor_pb2.FieldDescriptorProto
TYPE = {"double": _T.TYPE_DOUBLE, "float": _T.TYPE_FLOAT, "int64": _T.TYPE_INT64, "uint64": _T.TYPE_UINT64, "int32": _T.TYPE_INT32,
        "fixed64": _T.TYPE_FIXED64, "fixed32": _T.TYPE_FIXED32, "bool": _T.TYPE_BOOL, "string": _T.TYPE_STRING, "bytes": _T.TYPE_BYTES,
        "uint32": _T.TYPE_UINT32, "sfixed32": _T.TYPE_SFIXED32, "sfixed64": _T.TYPE_SFIXED64, "sint32": _T.TYPE_SINT32,
        "sint64": _T.TYPE_SINT64, "enum": _T.TYPE_ENUM}
KINDS = list(TYPE)


def all_kinds(presence=False, first=1):
    return [PbField(f"f_{k}", first + i, k, presence=presence) for i, k in enumerate(KINDS)]


_n_files = [0]


def upb_class(fields, syntax="proto3"):
    _n_files[0] += 1
    name = f"x{_n_files[0]}"
    fdp = descriptor_pb2.FileDescriptorProto(name=f"{name}.proto", package=name, syntax=syntax)
    e = fdp.enum_type.add(name="Kind")
    e.value.add(name="E0", number=0)
    e.value.add(name="E1", number=1)
    m = fdp.message_type.add(name="M")
    oneofs = sorted({f.oneof for f in fields if f.oneof is not None})  # declared oneofs come before proto3 `optional`'s
    for k in oneofs:
        m.oneof_decl.add(name=f"choice{k}")
    for f in fields:
        fd = m.field.add(name=f.name, number=f.number, type=TYPE[f.kind], label=_T.LABEL_OPTIONAL)
        if f.kind == "enum":
            fd.type_name = f".{name}.Kind"
        if f.oneof is not None:
            fd.oneof_index = oneofs.index(f.oneof)
        elif syntax == "proto3" and f.presence:
            fd.proto3_optional = True
            fd.oneof_index = len(m.oneof_decl)
            m.oneof_decl.add(name="_" + f.name)
        if syntax == "proto2" and f.default is not None:
            d = f.default
            fd.default_value = ("true" if d else "false") if f.kind == "bool" else ("E1" if d == 1 else "E0") if f.kind == "enum" else \
                d if isinstance(d, str) else d.decode() if isinstance(d, bytes) else repr(d) if isinstance(d, float) else str(d)
    pool = descriptor_pool.DescriptorPool()
    pool.Add(fdp)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName(f"{name}.M"))


def rand_value(rng, kind, proto3=True):
    r = rng.random()
    if kind in ("int32", "sfixed32", "sint32"):
        return int(rng.choice([0, 1, -1, 2**31 - 1, -2**31])) if r < 0.3 else int(rng.integers(-2**31, 2**31))
    if kind == "enum":
        return int(rng.integers(-5, 5)) if proto3 else int(rng.integers(0, 2))
    if kind in ("int64", "sfixed64", "sint64"):
        return int(rng.choice([0, 1, -1, 2**63 - 1, -2**63])) if r < 0.3 else int(rng.integers(-2**63, 2**63))
    if kind in ("uint32", "fixed32"):
        return int(rng.integers(0, 2**32))
    if kind in ("uint64", "fixed64"):
        return int(rng.integers(0, 2**64, dtype=np.uint64))
    if kind == "bool":
        return bool(rng.integers(0, 2))
    if kind in ("float", "double"):
        special = [0.0, 1.5, float("nan"), float("inf"), -float("inf"), 1e-45 if kind == "float" else 5e-324]
        v = float(rng.choice(special)) if r < 0.3 else float(rng.normal(0, 1e6))
        return float(np.float32(v)) if kind == "float" else v
    if kind == "string":
        alphabet = ["a", "Z", " ", "é", "漢", "😀", "\x00", "\n"]
        return "".join(alphabet[int(i)] for i in rng.integers(0, len(alphabet), int(rng.integers(0, 12))))
    return bytes(rng.integers(0, 256, int(rng.integers(0, 12))).tolist())


def same(kind, a, b):
    if kind == "float":
        return f32_bits(a) == f32_bits(b)
    if kind == "double":
        return f64_bits(a) == f64_bits(b) or (math.isnan(a) and math.isnan(b))
    return a == b


def fill(cls, fields, values):
    msg = cls()
    for f in fields:
        if f.name in values:
            setattr(msg, f.name, values[f.name])
    return msg


@pytest.mark.parametrize("syntax,presence", [("proto3", False), ("proto3", True), ("proto2", True)])
def test_encode_and_decode_match_upb(syntax, presence):
    rng = np.random.default_rng(5 if presence else 4)
    fields = all_kinds(presence=presence)
    cls = upb_class(fields, syntax)
    for _ in range(400):
        values = {f.name: rand_value(rng, f.kind, syntax == "proto3") for f in fields if rng.random() < 0.8}
        for f in fields:  # A1: -0.0 is where prost and upb disagree
            if f.kind in ("float", "double") and f.name in values and values[f.name] == 0.0 and math.copysign(1, values[f.name]) < 0:
                values[f.name] = 0.0
        want = fill(cls, fields, values).SerializeToString(deterministic=True)
        got = encode_message(fields, values)
        assert got == want, values
        back = cls.FromString(got)
        dec = decode_message(fields, got)
        for f in fields:
            assert same(f.kind, dec[f.name], getattr(back, f.name)), (f.name, dec[f.name], getattr(back, f.name))


def test_negative_int32_and_enum_take_ten_bytes_and_zigzag_edges():
    fields = [PbField("i", 1, "int32"), PbField("e", 2, "enum"), PbField("s", 3, "sint32"), PbField("t", 4, "sint64")]
    cls = upb_class(fields)
    for vals in ({"i": -1}, {"e": -3}, {"i": -2**31}, {"s": -2**31}, {"s": 2**31 - 1}, {"t": -2**63}, {"t": 2**63 - 1}, {"s": -1, "t": 1}):
        got = encode_message(fields, vals)
        assert got == fill(cls, fields, vals).SerializeToString()
        assert decode_message(fields, got) == {**{"i": 0, "e": 0, "s": 0, "t": 0}, **vals}
    assert len(encode_message(fields, {"i": -1})) == 1 + 10
    assert zigzag32(-1) == 1 and zigzag32(2**31 - 1) == 2**32 - 2 and zigzag32(-2**31) == 2**32 - 1
    assert zigzag64(-2**63) == 2**64 - 1


def test_unknown_fields_repeated_occurrences_and_multibyte_utf8():
    fields = all_kinds()
    cls = upb_class(fields)
    rng = np.random.default_rng(9)
    known = all_kinds(first=1)
    for _ in range(200):
        a = {f.name: rand_value(rng, f.kind) for f in known if rng.random() < 0.5}
        b = {f.name: rand_value(rng, f.kind) for f in known if rng.random() < 0.5}
        unknown = bytearray()
        for num, wire in ((100, 0), (101, 1), (102, 2), (103, 5), (2**29 - 1, 0)):
            put_varint(unknown, (num << 3) | wire)
            unknown += {0: b"\x96\x01", 1: b"\x00" * 8, 2: b"\x03abc", 5: b"\x01\x02\x03\x04"}[wire]
        put_varint(unknown, (104 << 3) | 3)  # a group holding a field and a nested group
        put_varint(unknown, (1 << 3) | 0); unknown += b"\x05"
        put_varint(unknown, (2 << 3) | 3); put_varint(unknown, (2 << 3) | 4)
        put_varint(unknown, (104 << 3) | 4)
        payload = encode_message(fields, a) + bytes(unknown) + encode_message(fields, b)  # b's occurrences come last
        dec = decode_message(fields, payload)
        up = cls.FromString(payload)
        for f in fields:
            assert same(f.kind, dec[f.name], getattr(up, f.name)), f.name
    s = "añ漢😀"
    assert decode_message([PbField("s", 1, "string")], encode_message([PbField("s", 1, "string")], {"s": s}))["s"] == s


def test_proto2_defaults_and_proto3_optional():
    fields = [PbField("a", 1, "int32", presence=True, default=-7), PbField("b", 2, "string", presence=True, default="hé"),
              PbField("c", 3, "bool", presence=True, default=True), PbField("d", 4, "double", presence=True, default=2.5),
              PbField("e", 5, "enum", presence=True, default=1), PbField("f", 6, "float", presence=True, default=float("inf")),
              PbField("g", 7, "bytes", presence=True, default=b"xy")]
    cls = upb_class(fields, "proto2")
    empty = decode_message(fields, b"")
    up = cls.FromString(b"")
    for f in fields:
        assert same(f.kind, empty[f.name], getattr(up, f.name)), f.name
    # explicit presence: the zero value is written
    zeros = {"a": 0, "b": "", "c": False, "d": 0.0}
    assert encode_message(fields, zeros) == fill(cls, fields, zeros).SerializeToString()
    p3 = [PbField("o", 1, "int64", presence=True), PbField("p", 2, "int64")]
    cls3 = upb_class(p3)
    assert encode_message(p3, {"o": 0, "p": 0}) == fill(cls3, p3, {"o": 0, "p": 0}).SerializeToString() == b"\x08\x00"


def test_minus_zero_is_left_out_without_presence():
    # A1: prost's `!= 0.0` — not compared with upb, which writes -0.0
    fields = [PbField("f", 1, "float"), PbField("d", 2, "double")]
    assert encode_message(fields, {"f": -0.0, "d": -0.0}) == b""
    assert encode_message([PbField("d", 2, "double", presence=True)], {"d": -0.0}) == b"\x11" + struct.pack("<d", -0.0)


@pytest.mark.parametrize("payload", [b"\x08", b"\x08\x80", b"\x12\x05ab", b"\x00\x01", b"\x08" + b"\xff" * 10 + b"\x01",
                                     b"\x1a\x02\xc3\x28"])
def test_malformed_payloads_fail_in_both(payload):
    fields = [PbField("i", 1, "int32"), PbField("s", 2, "string"), PbField("t", 3, "string")]
    cls = upb_class(fields)
    with pytest.raises(ProtobufError) as e:
        decode_message(fields, payload)
    assert e.value.kind == "Process" and e.value.message.startswith("Protobuf message parsing failed: ")
    with pytest.raises(Exception):
        cls.FromString(payload)


def test_prost_only_rules():
    fields = [PbField("i", 1, "int32")]
    for payload in (b"\x0d\x00\x00\x00\x00",  # known field, wrong wire type (upb: unknown field)
                    b"\x14",                   # end-group that closes nothing
                    b"\x0b\x14",               # group 1 closed by end-group 2
                    b"\x08" + b"\xff" * 9 + b"\x02"):  # 10th varint byte > 1: bits beyond 64 (upb drops them)
        with pytest.raises(ProtobufError):
            decode_message(fields, payload)
    deep = bytearray()
    for _ in range(101):
        put_varint(deep, (7 << 3) | 3)
    with pytest.raises(ProtobufError) as e:  # A4
        decode_message(fields, bytes(deep))
    assert "recursion" in e.value.message


def test_oneof_keeps_the_last_member_on_the_wire():
    fields = [PbField("a", 1, "int32"), PbField("x", 2, "int32", oneof=0), PbField("y", 3, "string", oneof=0),
              PbField("z", 4, "double", oneof=0), PbField("p", 5, "bool", oneof=1), PbField("q", 6, "bytes", oneof=1)]
    cls = upb_class(fields)
    one = upb_class([PbField("x", 1, "int32", oneof=0), PbField("y", 2, "string", oneof=0)])
    pair = [PbField("x", 1, "int32", oneof=0), PbField("y", 2, "string", oneof=0)]
    payload = encode_message(pair, {"x": 5}) + encode_message(pair, {"y": "hi"})
    assert decode_message(pair, payload) == {"x": 0, "y": "hi"}
    up = one.FromString(payload)
    assert (up.x, up.y, up.WhichOneof("choice0")) == (0, "hi", "y")
    rng = np.random.default_rng(12)
    for _ in range(300):
        payload = b""
        for _ in range(int(rng.integers(1, 6))):  # single-field messages, concatenated: a merge of several messages
            f = fields[int(rng.integers(0, len(fields)))]
            payload += encode_message(fields, {f.name: rand_value(rng, f.kind)})
        dec = decode_message(fields, payload)
        up = cls.FromString(payload)
        for f in fields:
            assert same(f.kind, dec[f.name], getattr(up, f.name)), (f.name, payload)
