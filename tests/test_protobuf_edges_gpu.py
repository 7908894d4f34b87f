"""protobuf_to_arrow / arrow_to_protobuf (csrc/protobuf.cu) against oracle/protobuf_oracle.py at the branches random
data over a small schema does not reach.

Decoder: known field numbers on both sides of the 128-entry lookup table, with keys of 1 to 5 bytes; 64-field messages
(bit 63 of the `seen` mask, oneofs past bit 32) and the 65-field limit; every varint form of every varint kind; the UTF-8
edges of `string` fields; the staged / in-place choice of each CTA, restated on the host (`stage_bytes`, `cta_staged`)
and asserted for every case built for it; sliced payload columns with NULLs at warp and CTA edges; proto2 defaults of
every kind.  Encoder: length varints of 1 to 4 bytes; the write kernel's staged / direct choice per CTA (`stage_window`,
`write_plan`) with every output misalignment; input columns sliced inside a byte; 5-byte keys; 64 / 65 fields; rows that
set no field; float special values.  Every schema also round-trips through both entries.

Integers and bytes compare exactly, floats by bit pattern, errors by kind, message prefix and payload index.  Each case
runs through the host entry (`process`), the device entry (`process_device`) and, for sliced inputs, a device batch that
keeps the parent's buffers and Arrow offset."""
import dataclasses

import numpy as np
import pyarrow as pa
import pytest

from arkflow_b200.arrow_ffi import DeviceBatch
from arkflow_b200.processor import ArkError, ArrowToProtobufProcessor, ProtobufToArrowProcessor
from oracle import protobuf_oracle as O
from oracle.protobuf_oracle import PbField
from test_protobuf_gpu import ALL2, ALL3, KINDS, assert_same_batch, decode, encode, processors

pytestmark = pytest.mark.gpu

CTA = 128              # PB_THREADS: payloads per decode CTA, rows per encode CTA
STAGE_MAX = 44 * 1024  # stage_window's cap
PREFIX = "Protobuf message parsing failed: "


# ---- wire pieces ---------------------------------------------------------------------------------------------------------
def varint(v):
    out = bytearray()
    O.put_varint(out, v)
    return bytes(out)


def key(num, wire):
    return varint((num << 3) | wire)


def varint_form(v, length):
    """`v` as a varint of exactly `length` bytes: overlong when longer than the canonical form."""
    assert 0 <= v < 1 << (7 * length) and 1 <= length <= 10
    return bytes(((v >> (7 * i)) & 0x7F) | (0x80 if i < length - 1 else 0) for i in range(length))


def one_field(f, v):
    """One occurrence of `f` holding `v`, written even when `v` is the zero value."""
    return O.encode_message([dataclasses.replace(f, presence=True, oneof=None)], {f.name: v})


def wrong_wire(f):
    return O.I32 if O.WIRE.get(f.kind, O.VARINT) != O.I32 else O.VARINT


def wire_body(wire, rng):
    if wire == O.VARINT:
        return varint(int(rng.integers(0, 2**63)))
    if wire == O.I64:
        return bytes(rng.integers(0, 256, 8).tolist())
    if wire == O.I32:
        return bytes(rng.integers(0, 256, 4).tolist())
    body = bytes(rng.integers(0, 256, int(rng.integers(0, 20))).tolist())
    return varint(len(body)) + body


def unknown_field(rng, num):
    wire = int(rng.choice([O.VARINT, O.I64, O.LEN, O.I32]))
    return key(num, wire) + wire_body(wire, rng)


def unknown_group(rng, num, known):
    """Group `num` (unknown) holding known field numbers with the wrong wire type and a nested group numbered like a
    known field: all of it is skipped."""
    out = key(num, O.SGROUP)
    for f in known:
        w = wrong_wire(f)
        out += key(f.number, w) + wire_body(w, rng)
    g = known[0].number
    out += key(g, O.SGROUP) + key(known[-1].number, O.VARINT) + b"\x01" + key(g, O.EGROUP)
    return out + key(num, O.EGROUP)


# ---- values and batches --------------------------------------------------------------------------------------------------
F32_SPECIAL = [0, 0x80000000, 0x7FC00000, 0x7FC00001, 0xFFBFFFFF, 0x7F800001, 0x7F800000, 0xFF800000, 1, 0x80000001,
               0x00800000, 0x7F7FFFFF]
F64_SPECIAL = [0, 1 << 63, 0x7FF8000000000000, 0x7FF8000000000001, 0xFFF7FFFFFFFFFFFF, 0x7FF0000000000001,
               0x7FF0000000000000, 0xFFF0000000000000, 1, (1 << 63) | 1, 0x0010000000000000, 0x7FEFFFFFFFFFFFFF]
STRS = ["", "a", "é", "漢字", "😀", "a\x00b", "z" * 130]
NONZERO = {"int32": -5, "int64": 6, "uint32": 7, "uint64": 8, "sint32": -9, "sint64": 10, "fixed32": 11, "fixed64": 12,
           "sfixed32": -77, "sfixed64": 2**40, "bool": True, "float": 0x3FC00000, "double": 0x3FF8000000000000, "string": "v",
           "bytes": b"\x01z", "enum": 1}


def pick(rng, seq):
    return seq[int(rng.integers(0, len(seq)))]  # (rng.choice would turn integers past 2^63 into floats)


def rand_value(rng, kind):
    """A value of `kind` as the oracle holds it (floats as their IEEE bits), an edge value about a third of the time."""
    edge = rng.random() < 0.35
    if kind in ("int32", "sint32", "sfixed32", "enum"):
        return pick(rng, [0, 1, -1, 2**31 - 1, -2**31]) if edge else int(rng.integers(-2**31, 2**31))
    if kind in ("int64", "sint64", "sfixed64"):
        return pick(rng, [0, 1, -1, 2**63 - 1, -2**63]) if edge else int(rng.integers(-2**63, 2**63))
    if kind in ("uint32", "fixed32"):
        return pick(rng, [0, 1, 2**32 - 1]) if edge else int(rng.integers(0, 2**32))
    if kind in ("uint64", "fixed64"):
        return pick(rng, [0, 1, 2**64 - 1]) if edge else int(rng.integers(0, 2**64, dtype=np.uint64))
    if kind == "bool":
        return bool(rng.integers(0, 2))
    if kind == "float":
        return pick(rng, F32_SPECIAL) if edge else int(rng.integers(0, 2**32))
    if kind == "double":
        return pick(rng, F64_SPECIAL) if edge else int(rng.integers(0, 2**64, dtype=np.uint64))
    if kind == "string":
        return STRS[int(rng.integers(0, len(STRS)))] + "x" * int(rng.integers(0, 3))
    return bytes(rng.integers(0, 256, int(rng.integers(0, 140))).tolist())


def schema_of(fields):
    return pa.schema([pa.field(f.name, O.ARROW_TYPE[f.kind], nullable=False) for f in fields])


def value_batch(fields, rows):
    """One non-nullable column per field from row dicts (floats given as their bits)."""
    arrays = []
    for f in fields:
        vals = [r[f.name] for r in rows]
        t = O.ARROW_TYPE[f.kind]
        if f.kind == "float":
            arrays.append(pa.array(np.array(vals, np.uint32).view(np.float32), t))
        elif f.kind == "double":
            arrays.append(pa.array(np.array(vals, np.uint64).view(np.float64), t))
        else:
            arrays.append(pa.array(vals, t))
    return pa.RecordBatch.from_arrays(arrays, schema=schema_of(fields))


def payload_batch(payloads):
    return pa.record_batch([pa.array(payloads, pa.binary())], names=["__value__"])


def normalised(rb):
    return pa.RecordBatch.from_arrays([pa.concat_arrays([c]) for c in rb.columns], schema=rb.schema)


def enum_processors(tmp_path, fields, syntax, enum_values):
    d = tmp_path / "enum"
    d.mkdir(parents=True, exist_ok=True)
    (d / "m.proto").write_text(O.proto_text("t", "M", fields, syntax, enum_values))
    cfg = {"proto_inputs": [str(d)], "message_type": "t.M"}
    return ProtobufToArrowProcessor(cfg), ArrowToProtobufProcessor(cfg)


# ---- running a case ------------------------------------------------------------------------------------------------------
def _sliced_device(proc, rb):
    out = proc.process_device(DeviceBatch.from_arrow(rb, keep_offsets=True))
    return None if out is None else out.to_arrow()


def _routes(rb):
    """(route, callable(proc) -> RecordBatch, input the route hands over): the host entry, the device entry (sliced
    columns normalised to offset 0) and, for sliced inputs, a device batch holding the parent's buffers."""
    yield "host", lambda p: decode(p, rb) if isinstance(p, ProtobufToArrowProcessor) else encode(p, rb), rb
    yield "device", lambda p: (decode if isinstance(p, ProtobufToArrowProcessor) else encode)(p, rb, device=True), normalised(rb)
    if any(c.offset for c in rb.columns):
        yield "device, parent buffers", lambda p: _sliced_device(p, rb), rb


def check_decode(dec, fields, rb):
    if isinstance(rb, list):
        rb = payload_batch(rb)
    want = O.protobuf_to_arrow(fields, rb)
    for route, run, _ in _routes(rb):
        got = run(dec)
        try:
            assert_same_batch(got, want)
        except AssertionError as e:
            raise AssertionError(f"{route}: {e}") from None
    return want


def check_decode_error(dec, fields, payloads, text=None):
    """The oracle's first failing payload must be the one the library names, through both entries."""
    bad = None
    for i, p in enumerate(payloads):
        if p is None:
            continue
        try:
            O.decode_message_raw(fields, p)
        except O.ProtobufError as e:
            bad, why = i, e.message
            break
    assert bad is not None, "the oracle accepts every payload"
    if text:
        assert text in why, why
    rb = payload_batch(payloads)
    for device in (False, True):
        with pytest.raises(ArkError) as e:
            decode(dec, rb, device=device)
        msg = e.value.message
        assert e.value.kind == "Process" and msg.startswith(PREFIX) and msg.endswith(f" (payload {bad})"), (device, msg)
        if text:
            assert text in msg, (device, msg)


def check_encode(enc, fields, rb, include=None):
    for route, run, given in _routes(rb):
        want = O.arrow_to_protobuf(fields, given, include)
        got = run(enc)
        assert got.schema.names == want.schema.names, route
        g, w = got.column(got.num_columns - 1), want.column(want.num_columns - 1)
        assert g.type == pa.binary() and g.null_count == 0, route
        if not g.equals(w):
            gl, wl = g.to_pylist(), w.to_pylist()
            bad = next(i for i in range(len(wl)) if gl[i] != wl[i])
            raise AssertionError((route, bad, gl[bad][:64], wl[bad][:64]))
    return O.arrow_to_protobuf(fields, rb, include)


def check_round_trip(dec, enc, fields, rb, want=None):
    """decode(encode(rb)) through both entries equals `want`; by default rb itself as the oracle round-trips it (a float
    or double -0.0 without presence is left out, so it comes back as +0.0)."""
    if want is None:
        want = O.protobuf_to_arrow(fields, O.arrow_to_protobuf(fields, rb).select(["__value__"]))
    for device in (False, True):
        out = encode(enc, rb, device=device)
        back = decode(dec, out.select(["__value__"]), device=device)
        try:
            assert_same_batch(back, want)
        except AssertionError as e:
            raise AssertionError(f"device={device}: {e}") from None


# ---- the decode kernel's staging rule ------------------------------------------------------------------------------------
def stage_bytes(data_bytes, n):
    """record_stage_window: round_up((int64)(avg * 128 * 1.25) + 256, 1024) when payloads average at most 256 bytes, else
    0 (every CTA parses in place)."""
    avg = data_bytes / n
    return 0 if avg > 256.0 else -(-(int(avg * CTA * 1.25) + 256) // 1024) * 1024


def cta_windows(offsets):
    """Per CTA: its payload bytes and its 16-byte-aligned window [a0 & ~15, (a1 + 15) & ~15).  The payload buffer is
    16-byte aligned and its offsets start at 0, so byte o sits at o (mod 16)."""
    offs = np.asarray(offsets, np.int64)
    n = len(offs) - 1
    i0 = np.arange(0, n, CTA)
    o0, o1 = offs[i0], offs[np.minimum(i0 + CTA, n)]
    return o1 - o0, ((o1 + 15) & ~15) - (o0 & ~15)


def cta_staged(offsets, stage):
    nbytes, window = cta_windows(offsets)
    return (stage > 0) & (nbytes > 0) & (window <= stage)


def offsets_of(lens):
    return np.concatenate([[0], np.cumsum(np.asarray(lens, np.int64))])


# ---- the write kernel's staging rule -------------------------------------------------------------------------------------
def stage_window(total, n):
    """The encode write kernel's window: the average CTA's bytes + 50 % + 256, rounded up to 1 KiB, at most 44 KiB."""
    return min(STAGE_MAX, -(-(int(total / n * CTA * 1.5) + 256) // 1024) * 1024)


def write_plan(msg_lens):
    """(stage, [(CTA output start, CTA bytes, staged)]): a CTA writes through shared memory iff its bytes ≤ stage - 16."""
    lens = np.asarray(msg_lens, np.int64)
    n, total = len(lens), int(lens.sum())
    stage = stage_window(total, n)
    starts = offsets_of(lens)
    ctas = []
    for c in range(0, n, CTA):
        b0, b1 = int(starts[c]), int(starts[min(c + CTA, n)])
        ctas.append((b0, b1 - b0, b1 - b0 <= stage - 16))
    return stage, ctas


# ==== decoder ==============================================================================================================
# keys of 1 to 5 bytes on both sides of the table; the first and the last declared fields are both found by the linear
# search (numbers ≥ 128)
FN = [PbField(f"n{num}", num, kind) for num, kind in (
    (2048, "sint64"), (1, "int32"), (15, "string"), (16, "fixed32"), (127, "bool"), (128, "double"), (129, "bytes"),
    (2047, "uint64"), (262143, "float"), (262144, "enum"), (33554431, "sfixed64"), (33554432, "string"),
    (536870911, "sint32"))]
FN_UNKNOWN = [2, 14, 17, 126, 130, 2046, 2049, 262142, 262145, 33554430, 33554433, 536870910]


def field_number_payloads(rng, n):
    out = []
    for _ in range(n):
        parts = []
        for f in FN:
            for _ in range(int(rng.choice([0, 1, 1, 2]))):  # absent, once, or twice (the last occurrence wins)
                parts.append(one_field(f, rand_value(rng, f.kind)))
        for num in FN_UNKNOWN:
            if rng.random() < 0.25:
                parts.append(unknown_field(rng, num))
        if rng.random() < 0.3:
            picks = [FN[int(j)] for j in rng.choice(len(FN), 3, replace=False)]
            parts.append(unknown_group(rng, int(rng.choice(FN_UNKNOWN)), picks))
        rng.shuffle(parts)
        out.append(b"".join(parts))
    return out


def test_field_numbers_and_key_lengths(gpu, tmp_path):
    assert [len(key(f.number, 0)) for f in FN] == [3, 1, 1, 2, 2, 2, 2, 2, 3, 4, 4, 5, 5]
    dec, enc = processors(tmp_path, FN)
    rng = np.random.default_rng(101)
    payloads = field_number_payloads(rng, 1500)
    # every known field alone, first and last declared included
    payloads += [one_field(f, rand_value(np.random.default_rng(f.number), f.kind)) for f in FN]
    want = check_decode(dec, FN, payloads)
    assert all(len(set(want.column(f.name).to_pylist())) > 2 for f in FN if f.kind != "bool")
    # a known field number inside an unknown group with the right wire type is skipped as well
    inner = unknown_group(rng, 130, FN[:2])[:-len(key(130, O.EGROUP))] + one_field(FN[0], 5) + key(130, O.EGROUP)
    got = check_decode(dec, FN, [inner + one_field(FN[-1], -3)])
    assert got.column("n2048").to_pylist() == [0] and got.column("n536870911").to_pylist() == [-3]
    # encode: 5-byte keys, fields in number order
    rows = [{f.name: rand_value(rng, f.kind) for f in FN} for _ in range(700)]
    rb = value_batch(FN, rows)
    want = check_encode(enc, FN, rb)
    top = key(536870911, O.VARINT)
    assert len(top) == 5 and sum(v.as_py().find(top) >= 0 for v in want.column("__value__")) > 500
    check_round_trip(dec, enc, FN, rb)


def wide_fields(n, oneofs=False):
    """n fields cycling through every kind; numbers below and above 128 (index 63 takes number 2, through the table);
    with `oneofs`, oneofs over declaration indices 31-32, 40-42 and 62-63."""
    groups = {31: 0, 32: 0, 40: 1, 41: 1, 42: 1, 62: 2, 63: 2} if oneofs else {}
    return [PbField(f"w{j}", 65 - j if j % 3 != 2 else 300 + j, KINDS[j % len(KINDS)], presence=j % 5 == 4 and j not in groups,
                    oneof=groups.get(j)) for j in range(n)]


def test_sixty_four_fields(gpu, tmp_path):
    fields = wide_fields(64)
    assert fields[63].number < 128 and len({f.number for f in fields}) == 64
    dec, enc = processors(tmp_path, fields)
    rng = np.random.default_rng(64)
    payloads = []
    for i in range(1200):
        subset = {f.name: rand_value(rng, f.kind) for f in fields if rng.random() < 0.5}
        payloads.append(O.encode_message([dataclasses.replace(f, presence=True) for f in fields], subset))
    assert (fields[0].kind, fields[63].kind) == ("int32", "enum")
    payloads += [one_field(fields[63], 7), one_field(fields[0], 7), b""]
    want = check_decode(dec, fields, payloads)
    assert want.column("w63").to_pylist()[-3:] == [7, 0, 0] and want.column("w0").to_pylist()[-3:] == [0, 7, 0]
    rows = [{f.name: rand_value(rng, f.kind) for f in fields} for _ in range(600)]
    rb = value_batch(fields, rows)
    check_encode(enc, fields, rb)
    check_round_trip(dec, enc, fields, rb)


def test_oneof_members_past_bit_32(gpu, tmp_path):
    fields = wide_fields(64, oneofs=True)
    dec, _ = processors(tmp_path, fields)
    w = {j: fields[j] for j in (8, 9, 10, 30, 31, 32, 33, 40, 41, 42, 62, 63)}
    v = {j: NONZERO[f.kind] for j, f in w.items()}
    # read 40 then 41: only 41 keeps its value; 8, 9 and 10 (bits 40-42 mod 32) keep theirs
    pay = b"".join(one_field(w[j], v[j]) for j in (8, 9, 10, 40, 41))
    got = check_decode(dec, fields, [pay, b"".join(one_field(w[j], v[j]) for j in (33, 32, 31, 30, 62, 63, 42))])
    assert got.column("w40").to_pylist()[0] == O.decode_message_raw(fields, b"")["w40"]
    assert [got.column(f"w{j}").to_pylist()[0] for j in (8, 9, 10, 41)] == [v[8], v[9], v[10], v[41]]
    rng = np.random.default_rng(40)
    members = [fields[j] for j in (31, 32, 40, 41, 42, 62, 63)]
    others = [fields[j] for j in (0, 8, 9, 10, 30, 33, 61)]
    payloads = []
    for _ in range(3000):
        parts = []
        for _ in range(int(rng.integers(0, 7))):  # single-field messages concatenated, as merged messages arrive
            f = members[int(rng.integers(0, len(members)))] if rng.random() < 0.75 else others[int(rng.integers(0, len(others)))]
            parts.append(one_field(f, rand_value(rng, f.kind)))
        payloads.append(b"".join(parts))
    check_decode(dec, fields, payloads)


def test_sixty_five_fields_are_unsupported(gpu, tmp_path):
    fields = wide_fields(65)
    dec, enc = processors(tmp_path, fields)
    for payloads in ([b""], [None, b"\x08\x01"]):
        for device in (False, True):
            with pytest.raises(ArkError) as e:
                decode(dec, payload_batch(payloads), device=device)
            assert e.value.kind == "Unsupported", e.value.message
    assert decode(dec, []) is None
    rng = np.random.default_rng(65)
    rb = value_batch(fields, [{f.name: rand_value(rng, f.kind) for f in fields} for _ in range(50)])
    for device in (False, True):
        with pytest.raises(ArkError) as e:
            encode(enc, rb, device=device)
        assert e.value.kind == "Unsupported", e.value.message
    check_encode(enc, fields, rb.select(range(1, 65)))  # 64 of them are encoded


VARINT_FIELDS = [PbField("i32", 1, "int32"), PbField("i64", 2, "int64"), PbField("u32", 3, "uint32"), PbField("u64", 4, "uint64"),
                 PbField("s32", 5, "sint32"), PbField("s64", 6, "sint64"), PbField("b", 7, "bool"), PbField("e", 8, "enum")]
# (value, lengths): overlong 0 / 1 / -1, the largest legal 10th byte (2^63 needs 0x01 there), values past 2^32 that
# int32 / uint32 / enum truncate and sint32 must truncate before unzigzagging, 2 and 2^63 for bool
VARINT_VALUES = [(0, range(1, 11)), (1, range(1, 11)), (2**64 - 1, [10]), (2**63, [10]), (2**63 + 7, [10]),
                 (2**32 + 2, [5, 10]), (2**32 + 5, [5, 7]), (2**33 - 1, [5]), (0xFFFFFFFF80000000, [10]), (0xFFFFFFFF, [5, 6]),
                 (2, [1, 4]), (2**40 + 3, [6, 10]), (O.zigzag64(-2**40), [6, 10]), (O.zigzag64(2**62 + 1), [10])]


def test_varint_forms_of_every_kind(gpu, tmp_path):
    dec, _ = processors(tmp_path, VARINT_FIELDS)
    payloads = []
    for f in VARINT_FIELDS:
        for v, lengths in VARINT_VALUES:
            for n in lengths:
                payloads.append(key(f.number, O.VARINT) + varint_form(v, n))
        # an overlong key in front of a value
        payloads.append(varint_form((f.number << 3) | O.VARINT, 3) + varint_form(1, 2))
    rng = np.random.default_rng(7)
    for _ in range(400):  # several forms in one payload, the last one of each field wins
        parts = []
        for _ in range(int(rng.integers(1, 9))):
            f = VARINT_FIELDS[int(rng.integers(0, len(VARINT_FIELDS)))]
            v, lengths = pick(rng, VARINT_VALUES)
            parts.append(key(f.number, O.VARINT) + varint_form(v, pick(rng, list(lengths))))
        payloads.append(b"".join(parts))
    want = check_decode(dec, VARINT_FIELDS, payloads)
    got = dict(zip(want.schema.names, (c.to_pylist() for c in want.columns)))
    # the rules the oracle states, on single payloads (row = field index * forms + form index)
    forms = sum(len(list(ls)) for _, ls in VARINT_VALUES) + 1
    row = lambda f, v, n: VARINT_FIELDS.index(f) * forms + [(a, m) for a, ls in VARINT_VALUES for m in ls].index((v, n))
    i32, u32, s32, b = (VARINT_FIELDS[k] for k in (0, 2, 4, 6))
    assert got["i32"][row(i32, 2**32 + 5, 7)] == 5 and got["i32"][row(i32, 0xFFFFFFFF80000000, 10)] == -2**31
    assert got["u32"][row(u32, 2**33 - 1, 5)] == 2**32 - 1 and got["s32"][row(s32, 2**32 + 2, 5)] == 1
    assert got["b"][row(b, 2, 4)] is True and got["b"][row(b, 2**63, 10)] is True and got["b"][row(b, 0, 10)] is False
    # the smallest illegal 10th byte, and an 11-byte varint, in every kind
    good = b"".join(key(f.number, O.VARINT) + b"\x01" for f in VARINT_FIELDS)
    for f in VARINT_FIELDS:
        for bad in (b"\xff" * 9 + b"\x02", b"\x80" * 9 + b"\x02", b"\x80" * 10 + b"\x00"):
            check_decode_error(dec, VARINT_FIELDS, [good] * 131 + [key(f.number, O.VARINT) + bad] + [good] * 3, "invalid varint")


UTF8_FIELDS = [PbField("s", 1, "string"), PbField("b", 2, "bytes"), PbField("t", 3, "string")]
UTF8_BAD = [b"\xc0\x80", b"\xc1\xbf", b"\xe0\x80\x80", b"\xe0\x9f\xbf", b"\xf0\x80\x80\x80", b"\xf0\x8f\xbf\xbf",
            b"\xed\xa0\x80", b"\xed\xbf\xbf", b"\xf4\x90\x80\x80", b"\xf5\x80\x80\x80", b"\xff", b"\x80", b"a\xbfb",
            b"ab\xc3", b"ab\xe6\xbc", b"ab\xf0\x9f\x98", b"\xc3\x28"]
UTF8_GOOD = [b"\xc2\x80", b"\xdf\xbf", b"\xe0\xa0\x80", b"\xed\x9f\xbf", b"\xee\x80\x80", b"\xef\xbf\xbf", b"\xf0\x90\x80\x80",
             b"\xf4\x8f\xbf\xbf", "ab😀".encode(), "\U0010ffff".encode()]
# key 0x98 0x01 (field 19, varint: unknown), then 0x01: its first byte is a continuation byte, so a check that read past
# the end of a field or of a payload would complete a character cut short there
TRAP = b"\x98\x01\x01"


def test_utf8_edges_of_string_fields(gpu, tmp_path):
    dec, _ = processors(tmp_path, UTF8_FIELDS)
    s, b, t = UTF8_FIELDS

    def at_field_end(x):
        return key(1, O.LEN) + varint(len(x)) + x + TRAP + one_field(t, "ok")

    def at_payload_end(x):
        return one_field(t, "ok") + TRAP + key(1, O.LEN) + varint(len(x)) + x

    good = [f(x) for x in UTF8_GOOD for f in (at_field_end, at_payload_end)]
    want = check_decode(dec, UTF8_FIELDS, good + [TRAP] * 3)
    assert want.column("s").to_pylist()[:len(good)] == [x.decode() for x in UTF8_GOOD for _ in range(2)]
    for x in UTF8_BAD:
        for f in (at_field_end, at_payload_end):
            # the next payload starts with a continuation byte too
            check_decode_error(dec, UTF8_FIELDS, (good * 7)[:130] + [f(x)] + [TRAP] * 4, "not UTF-8")
    # the same bytes in a `bytes` field pass through unchanged
    raw = [key(2, O.LEN) + varint(len(x)) + x + (TRAP if i % 2 else b"") for i, x in enumerate(UTF8_BAD + UTF8_GOOD)]
    want = check_decode(dec, UTF8_FIELDS, raw + [TRAP])
    assert want.column("b").to_pylist()[:-1] == UTF8_BAD + UTF8_GOOD


# ---- staging ------------------------------------------------------------------------------------------------------------
ST = [PbField("i", 1, "int64", presence=True, default=-9), PbField("s", 2, "string", presence=True, default="dé漢"),
      PbField("b", 3, "bytes", presence=True, default=b"\x00d"), PbField("t", 4, "string", presence=True, default="té")]


def sized_payload(i, length):
    """A payload of exactly `length` (≥ 16) bytes.  Even i fills `s` (its string comes from the payload); odd i fills `b`
    and leaves `s` to its default, and `t` from the payload or its default in turn."""
    head = O.encode_message(ST, {"i": i - 5000} if i % 2 == 0 else {"i": i, **({"t": "é" * (i % 3)} if i % 4 == 1 else {})})
    tag = key(2 if i % 2 == 0 else 3, O.LEN)
    for pad in (b"", key(9, O.VARINT) + b"\x00"):  # field 9 is unknown: two bytes that bridge the lengths a LEN field skips
        rest = length - len(head) - len(pad)
        for vl in (1, 2):
            k = rest - 1 - vl
            if k >= 0 and len(varint(k)) == vl:
                fill = ("é" * (k // 2) + "a" * (k % 2)).encode() if i % 4 == 0 else bytes(97 + (i + j) % 26 for j in range(k))
                out = head + tag + varint(k) + fill + pad
                assert len(out) == length
                return out
    raise AssertionError(length)


def set_cta(lens, c, total):
    lens[c * CTA:(c + 1) * CTA] = total // CTA
    lens[c * CTA:c * CTA + total % CTA] += 1


def mixed_lengths():
    """24 CTAs and a partial one of 48-byte payloads, but: CTA 5 holds exactly the staging size from an aligned start
    (staged, window == stage), CTA 9 16 bytes more (in place), CTA 12 starts at 7 (mod 16) and its window is exactly
    the staging size (staged), CTA 14 starts at 7 and holds one byte more than that (window stage + 16, in place)."""
    n_cta, base = 24, 48
    lens = np.full(n_cta * CTA + 37, base, np.int64)
    s = stage_bytes(lens.sum(), len(lens))
    for _ in range(10):
        lens[:] = base
        for c, total in ((5, s), (9, s + 16), (11, CTA * base + 7), (12, s - 7), (13, CTA * base + 7), (14, s - 6)):
            set_cta(lens, c, total)
        new = stage_bytes(lens.sum(), len(lens))
        if new == s:
            break
        s = new
    assert stage_bytes(lens.sum(), len(lens)) == s
    return lens


def staging_cases():
    rng = np.random.default_rng(256)
    yield "staged", rng.integers(16, 81, 20 * CTA + 5), "staged"
    yield "in place", rng.integers(200, 421, 5 * CTA + 3), "inplace"
    yield "mixed", mixed_lengths(), "mixed"
    yield "average 256", np.tile([192, 320], 3 * CTA // 2), "staged"
    yield "average 257", np.tile([193, 321], 3 * CTA // 2), "inplace"


@pytest.mark.parametrize("case", [c[0] for c in staging_cases()])
def test_decode_staging_mix(gpu, tmp_path, case):
    _, lens, mix = next(c for c in staging_cases() if c[0] == case)
    offs = offsets_of(lens)
    stage = stage_bytes(int(offs[-1]), len(lens))
    staged = cta_staged(offs, stage)
    assert ("staged" if staged.all() else "inplace" if not staged.any() else "mixed") == mix, (stage, staged)
    if case.startswith("average"):
        assert offs[-1] == len(lens) * int(case.split()[1]) and (stage > 0) == (case == "average 256")
    if case == "mixed":
        nbytes, window = cta_windows(offs)
        assert [int(window[c]) for c in (5, 12, 9, 14)] == [stage, stage, stage + 16, stage + 16]
        assert [int(offs[c * CTA]) % 16 for c in (5, 9, 12, 14)] == [0, 0, 7, 7]
        assert [c for c in range(len(staged)) if not staged[c]] == [9, 14]
    dec, _ = processors(tmp_path, ST, "proto2")
    payloads = [sized_payload(i, int(n)) for i, n in enumerate(lens)]
    want = check_decode(dec, ST, payloads)
    s = want.column("s").to_pylist()
    assert s[1] == "dé漢" and s[0] != "dé漢" and want.column("t").to_pylist()[1:3] == ["é", "té"]


@pytest.mark.parametrize("off", [1, 3, 33, 130])
def test_sliced_payload_columns_with_nulls(gpu, tmp_path, off):
    dec, _ = processors(tmp_path, ST, "proto2")
    m, nulls = 300, {0, 31, 32, 127, 128, 255, 256}
    parent = []
    for j in range(off + m + 9):
        r = j - off
        parent.append(None if r in nulls else b"" if r % 7 == 3 else sized_payload(j, 16 + (j * 13) % 50))
    rb = payload_batch(parent).slice(off, m)
    assert rb.column(0).offset == off and rb.column(0).null_count == len(nulls)
    want = check_decode(dec, ST, rb)
    assert want.num_rows == m - len(nulls)
    empty = payload_batch([b"\x08\x01"] * off + [None] * 200 + [b"\x08\x02"]).slice(off, 200)
    want = check_decode(dec, ST, empty)
    assert want.num_rows == 0 and want.schema == schema_of(ST)


DEFAULTS = {"int32": -2**31, "int64": -2**63, "uint32": 2**32 - 1, "uint64": 2**64 - 1, "sint32": -1, "sint64": 2**63 - 1,
            "fixed32": 2**31, "fixed64": 2**63, "sfixed32": -7, "sfixed64": -(2**40), "bool": True, "float": float("-inf"),
            "double": 5e-324, "string": "dé漢😀", "bytes": b"\x00a\x00\xff", "enum": -5}
ENUM_VALUES = (("EN", -5), ("E0", 0), ("E1", 1))


def test_proto2_defaults_of_every_kind(gpu, tmp_path):
    fields = [PbField(f"d_{k}", i + 1, k, presence=True, default=DEFAULTS[k]) for i, k in enumerate(KINDS)]
    dec, enc = enum_processors(tmp_path, fields, "proto2", ENUM_VALUES)
    rng = np.random.default_rng(2)
    payloads = []
    for r in range(1000):  # field k present on rows r with r + k even: absent and present alternate row by row
        vals = {f.name: (int(rng.choice([-5, 0, 1])) if f.kind == "enum" else rand_value(rng, f.kind))
                for k, f in enumerate(fields) if (r + k) % 2 == 0}
        payloads.append(O.encode_message(fields, vals))
    want = check_decode(dec, fields, payloads)
    assert want.column("d_string").to_pylist()[0] == "dé漢😀" and want.column("d_bytes").to_pylist()[1] == b"\x00a\x00\xff"
    assert want.column("d_enum").to_pylist()[0] == -5 and want.column("d_int64").to_pylist()[0] == -2**63
    check_round_trip(dec, enc, fields, want)


# ==== encoder ==============================================================================================================
def test_encode_length_varints(gpu, tmp_path):
    fields = [PbField("s", 1, "string"), PbField("b", 2, "bytes"), PbField("k", 3, "int32")]
    dec, enc = processors(tmp_path, fields)
    rng = np.random.default_rng(16)
    rows = []
    for n in (0, 127, 128, 16383, 16384, 2097151, 2097152):
        rows.append({"s": ("é" * (n // 2) + "a" * (n % 2)), "b": bytes(range(256)) * (n // 256) + bytes(n % 256), "k": n})
        rows += [{"s": STRS[j % len(STRS)], "b": bytes([j % 256]) * (j % 5), "k": int(rng.integers(-9, 9))} for j in range(40)]
    rb = value_batch(fields, rows)
    want = check_encode(enc, fields, rb)
    v = want.column("__value__").to_pylist()
    assert v[41 * 6].startswith(b"\x0a\x80\x80\x80\x01") and v[41 * 5].startswith(b"\x0a\xff\xff\x7f")
    check_round_trip(dec, enc, fields, rb)


def message_value(length):
    """The `bytes` value whose message (key, length varint, value) is exactly `length` bytes, or None."""
    if length == 0:
        return b""
    for vl in (1, 2, 3):
        k = length - 1 - vl
        if k >= 0 and len(varint(k)) == vl:
            return bytes(97 + i % 26 for i in range(k))
    return None


def split_cta(total, rows):
    lens = [total // rows + (1 if r < total % rows else 0) for r in range(rows)]
    for _ in range(4 * rows):
        bad = [r for r in range(rows) if message_value(lens[r]) is None]
        if not bad:
            return lens
        lens[bad[0]] -= 1
        lens[(bad[0] + 1) % rows] += 1
    raise AssertionError(total)


def write_case(case):
    """Message lengths for the write kernel.  `boundary`: CTAs 0-15 start at every misalignment mod 16, CTA 16 holds
    exactly stage - 16 bytes (staged), CTA 17 stage - 15 (direct), CTA 19 a 100 000-byte row (direct) between staged
    CTAs, and a partial last CTA.  `capped`: the same boundary with the window at its 44 KiB cap."""
    if case == "boundary":
        plan = [5121] * 16 + ["s-16", "s-15", 5121, "long", 5121]
        tail, base = 50, 5121
    else:
        plan = [40000, "s-16", "s-15", 40001, 40000]
        tail, base = 30, 40000
    stage = STAGE_MAX
    for _ in range(10):
        lens = []
        for p in plan:
            if p == "long":
                lens += split_cta(5000, CTA - 1) + [100000]
            else:
                lens += split_cta(stage - int(p[2:]) if isinstance(p, str) else p, CTA)
        lens += split_cta(base * tail // CTA, tail)
        new, _ = write_plan(lens)
        if new == stage:
            break
        stage = new
    return lens


@pytest.mark.parametrize("case", ["boundary", "capped"])
def test_encode_write_staging(gpu, tmp_path, case):
    lens = write_case(case)
    stage, ctas = write_plan(lens)
    flags = [s for _, _, s in ctas]
    if case == "boundary":
        assert stage < STAGE_MAX and flags == [True] * 17 + [False, True, False, True, True]
        assert sorted(b0 % 16 for b0, _, _ in ctas[:16]) == list(range(16))
        assert (ctas[16][1], ctas[17][1]) == (stage - 16, stage - 15)
    else:
        assert stage == STAGE_MAX and flags == [True, True, False, True, True, True]
        assert (ctas[1][1], ctas[2][1]) == (stage - 16, stage - 15) and ctas[3][0] % 16 != 0
    fields = [PbField("b", 1, "bytes")]
    dec, enc = processors(tmp_path, fields)
    rb = pa.RecordBatch.from_arrays([pa.array([message_value(n) for n in lens], pa.binary())], schema=schema_of(fields))
    want = check_encode(enc, fields, rb)
    assert [len(v) for v in want.column("__value__").to_pylist()] == lens
    check_round_trip(dec, enc, fields, rb)


def parent_column(rng, kind, n):
    """A nullable column with known contents under its NULL slots (which the encoder writes)."""
    t = O.ARROW_TYPE[kind]
    valid = rng.random(n) < 0.7
    vbuf = pa.py_buffer(np.packbits(valid, bitorder="little").tobytes())
    nulls = int((~valid).sum())
    if kind == "bool":
        data = pa.py_buffer(np.packbits(rng.random(n) < 0.5, bitorder="little").tobytes())
        return pa.Array.from_buffers(t, n, [vbuf, data], null_count=nulls)
    if kind in ("string", "bytes"):
        vals = [rand_value(rng, kind) for _ in range(n)]
        raw = [v.encode() if isinstance(v, str) else v for v in vals]
        offs = offsets_of([len(x) for x in raw]).astype(np.int32)
        return pa.Array.from_buffers(t, n, [vbuf, pa.py_buffer(offs.tobytes()), pa.py_buffer(b"".join(raw))], null_count=nulls)
    width = 4 if kind in ("int32", "sint32", "sfixed32", "enum", "uint32", "fixed32", "float") else 8
    vals = rng.integers(0, 2**64, n, dtype=np.uint64)
    vals[rng.random(n) < 0.2] = 0
    data = vals.astype(np.uint32) if width == 4 else vals
    return pa.Array.from_buffers(t, n, [vbuf, pa.py_buffer(data.tobytes())], null_count=nulls)


@pytest.mark.parametrize("syntax", ["proto3", "proto2"])
def test_encode_sliced_columns_of_every_kind(gpu, tmp_path, syntax):
    fields = ALL3 if syntax == "proto3" else ALL2
    _, enc = processors(tmp_path, fields, syntax)
    rng = np.random.default_rng(9)
    parent = pa.RecordBatch.from_arrays([parent_column(rng, f.kind, 200) for f in fields], names=[f.name for f in fields])
    for off in (1, 7, 9, 63):
        rb = parent.slice(off, 100)
        flag = rb.column("f_bool")
        assert flag.offset % 8 != 0 and all(c.null_count for c in rb.columns)
        check_encode(enc, fields, rb)


def test_encode_field_numbers_width_and_empty_rows(gpu, tmp_path):
    # no column sets a field: other names, a type that is not the field's, proto3 zero values
    _, enc = processors(tmp_path, ALL3)
    n = 300
    rb = pa.RecordBatch.from_arrays(
        [pa.array(range(n), pa.int64()), pa.array(range(n), pa.int64()), pa.array([""] * n), pa.array([False] * n),
         pa.array([0.0] * n, pa.float32())],
        names=["other", "f_int32", "f_string", "f_bool", "f_float"])
    want = check_encode(enc, ALL3, rb)
    assert want.column("__value__").to_pylist() == [b""] * n
    _, enc = processors(tmp_path, ALL3, enc={"fields_to_include": ["other", "f_uint32"]})
    rb2 = pa.RecordBatch.from_arrays([pa.array(range(n), pa.int64()), pa.array(range(1, n + 1), pa.uint64())], names=["other", "f_uint64"])
    assert check_encode(enc, ALL3, rb2, {"other", "f_uint32"}).column("__value__").to_pylist() == [b""] * n


def test_encode_float_special_values(gpu, tmp_path):
    fields = [PbField("f", 1, "float"), PbField("d", 2, "double"), PbField("fp", 3, "float", presence=True),
              PbField("dp", 4, "double", presence=True)]
    dec, enc = processors(tmp_path, fields)
    k = len(F32_SPECIAL)
    rows = [{"f": F32_SPECIAL[i % k], "d": F64_SPECIAL[(i // k) % k], "fp": F32_SPECIAL[(i + 3) % k], "dp": F64_SPECIAL[(i * 5) % k]}
            for i in range(k * k)]
    rb = value_batch(fields, rows)
    want = check_encode(enc, fields, rb)
    v = want.column("__value__").to_pylist()
    assert v[1].startswith(b"\x1d") and v[8].startswith(b"\x0d\x01\x00\x00\x00")  # A1: -0.0 left out; a denormal is not
    # without presence -0.0 comes back as +0.0; every NaN payload and the denormals keep their bits
    back = [{**r, "f": 0 if r["f"] == 0x80000000 else r["f"], "d": 0 if r["d"] == 1 << 63 else r["d"]} for r in rows]
    check_round_trip(dec, enc, fields, rb, value_batch(fields, back))
