"""concat_batches on the device (csrc/concat.cu) and the buffer stage that calls it, against oracle/buffer_oracle.py.

The oracle restates arrow-rs `concat_batches(schema, batches)`: columns matched by position, names, types and
nullability from the schema batch each call site picks, a Process error for differing types and for NULLs under a
non-nullable field.  Every input is built from a seed.  Results are compared as whole batches: validate(full=True),
schema names, types and nullability, null counts, Array.equals per column, Float32 / Float64 by bit pattern (NaN
payloads, -0.0).  Every concat runs through the host entry point and the device one, whose members are sliced device
batches (DeviceBatch.from_arrow(keep_offsets=True)): data pointers off alignment, offsets[0] != 0, bitmaps that start
inside a byte.  The launch counts (ark_kernel_timing_get) show which kernels ran: one concat_copy_kernel per call that
moves bytes, one concat_offsets_kernel per Utf8/Binary column, one concat_bits_kernel per Boolean column and per column
where a member has NULLs; a one-batch call launches none.
"""
import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from arkflow_b200.arrow_ffi import DeviceBatch, DeviceColumn
from arkflow_b200.buffer import MemoryBuffer, SessionWindow, SlidingWindow, TumblingWindow, concat_batches, concat_batches_device
from arkflow_b200.input import FileInput
from arkflow_b200.processor import ArkError, BatchProcessor, MessageBatch
from oracle import protobuf_oracle as PO
from oracle.avro_oracle import record_schema, write_avro
from oracle.buffer_oracle import batch_processor, concat, memory_drain, sliding_windows, window_drain
from oracle.protobuf_oracle import PbField
from oracle.sql_oracle import OracleError
from test_inputs_edges_gpu import launches
from test_protobuf_gpu import _pattern_bytes, decode, processors

pytestmark = pytest.mark.gpu

KINDS = ["int64", "float64", "bool", "utf8", "binary", "int32", "uint32", "uint64", "float32", "null"]
COPY, OFFS, BITS = "concat_copy_kernel", "concat_offsets_kernel", "concat_bits_kernel"
F64_SPECIAL = np.array([0x7FF8000000000001, 0xFFF123456789ABCD, 0x7FF0000000000001, 0x8000000000000000, 1,
                        0x7FF0000000000000, 0xFFF0000000000000], np.uint64)
F32_SPECIAL = np.array([0x7FC00001, 0xFFC12345, 0x7F800001, 0x80000000, 1, 0x7F800000, 0xFF800000], np.uint32)
UTF8_POOL = pa.array(["", "a", "é", "漢字", "\U0001F600x", "ab\x00c", "ÿ€" * 5, "z" * 40])
BIN_POOL = pa.array([b"", b"\x00", bytes(range(256)), b"\xff\xfe", b"\x00" * 17, b"json{}", bytes(range(255, -1, -1))[:33]],
                    pa.binary())


@pytest.fixture(scope="module", autouse=True)
def timing(gpu):
    gpu.ark_kernel_timing_enable(1)
    yield gpu
    gpu.ark_kernel_timing_enable(0)


def column(kind, n, rng, nulls):
    mask = (rng.random(n) < 0.25) if nulls else None
    if kind == "null":
        return pa.nulls(n)
    if kind in ("int64", "int32", "uint32", "uint64"):
        info = np.iinfo(kind)
        v = rng.integers(info.min, info.max, n, dtype=kind, endpoint=True)
        return pa.array(v, mask=mask)
    if kind in ("float64", "float32"):
        u, sp = (np.uint64, F64_SPECIAL) if kind == "float64" else (np.uint32, F32_SPECIAL)
        bits = rng.integers(0, np.iinfo(u).max, n, dtype=u, endpoint=True)
        k = rng.random(n) < 0.2
        bits[k] = sp[rng.integers(0, len(sp), int(k.sum()))]
        return pa.array(bits.view(np.float64 if kind == "float64" else np.float32), mask=mask)
    if kind == "bool":
        return pa.array(rng.random(n) < 0.5, mask=mask)
    pool = UTF8_POOL if kind == "utf8" else BIN_POOL
    v = pool.take(pa.array(rng.integers(0, len(pool), n)))
    return v if mask is None else pc.if_else(pa.array(~mask), v, pa.nulls(n, v.type))


def mixed_batch(n, seed, nulls=True, kinds=KINDS):
    rng = np.random.default_rng(seed)
    return pa.record_batch([column(k, n, rng, nulls and k != "null") for k in kinds], names=list(kinds))


def same_batch(got, want, what=""):
    got.validate(full=True)
    assert got.schema.names == want.schema.names, what
    assert [str(t) for t in got.schema.types] == [str(t) for t in want.schema.types], what
    assert [f.nullable for f in got.schema] == [f.nullable for f in want.schema], what
    assert got.num_rows == want.num_rows, what
    for i, (g, w) in enumerate(zip(got.columns, want.columns)):
        assert g.null_count == w.null_count, (what, i)
        if pa.types.is_floating(w.type):
            u = np.uint32 if w.type == pa.float32() else np.uint64
            assert g.is_valid().equals(w.is_valid()), (what, i)
            gb, wb = (x.fill_null(0).to_numpy(zero_copy_only=False).view(u) for x in (g, w))
            assert np.array_equal(gb, wb), (what, i, np.flatnonzero(gb != wb)[:5])
        else:
            assert g.equals(w), (what, i)


def offsets_of(c):
    """The int32 offsets of a (sliced) Utf8/Binary array: len(c) + 1 values, the first one offsets[0]."""
    return np.frombuffer(c.buffers()[1], np.int32)[c.offset:c.offset + len(c) + 1]


def expected_launches(members):
    """{kernel: launches} of one concat of these members."""
    if len(members) == 1:
        return {COPY: 0, OFFS: 0, BITS: 0}
    rows = sum(m.num_rows for m in members)
    moved, offs, bits = 0, 0, 0
    for i, t in enumerate(members[0].schema.types):
        cols = [m.column(i) for m in members]
        if pa.types.is_string(t) or pa.types.is_binary(t):
            moved += sum(int(offsets_of(c)[-1] - offsets_of(c)[0]) for c in cols if len(c))
            offs += rows > 0
        elif t != pa.null() and t != pa.bool_():
            moved += rows * t.bit_width // 8
        bits += rows > 0 and (t == pa.bool_()) + (t != pa.null() and any(c.null_count for c in cols))
    return {COPY: int(moved > 0), OFFS: offs, BITS: bits}


def run_concat(lib, members, device):
    lib.ark_kernel_timing_reset()
    if device:
        out = concat_batches_device([DeviceBatch.from_arrow(m, keep_offsets=True) for m in members])
        got = out.to_arrow()
        out.close()
    else:
        got = concat_batches(members)
    return got, {k: launches(lib, k) for k in (COPY, OFFS, BITS)}


def check(lib, members, what=""):
    """Both entry points against the oracle; the launch counts when the concat succeeds."""
    try:
        want = concat(members)
    except OracleError as e:
        want = e
    for device in (False, True):
        w = (what, "device" if device else "host")
        if isinstance(want, OracleError):
            with pytest.raises(ArkError) as e:
                run_concat(lib, members, device)
            assert e.value.kind == want.kind, (w, e.value.message)
            continue
        got, n = run_concat(lib, members, device)
        same_batch(got, want, w)
        assert n == expected_launches(members), (w, n)
    return want


# ---- types and bit edges ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_every_type_one_and_many_members(timing, kind):
    rng = np.random.default_rng(KINDS.index(kind))
    parts = []
    for k, n in enumerate([5, 0, 1, 300, 8, 0, 17]):
        c = column(kind, n + 3, rng, nulls=kind != "null" and k % 2 == 0)  # members with and without NULLs
        parts.append(pa.record_batch([c], names=[kind]).slice(k % 3, n))
    check(timing, parts[:1], (kind, "one"))
    check(timing, parts[3:4], (kind, "one, sliced"))
    check(timing, parts, (kind, "many"))


@pytest.mark.parametrize("nulls", [False, True])
def test_members_sharing_output_bytes(timing, nulls):
    # members of 0-17 rows: several members land in one output byte, and every member starts at bit 1-7 of its bitmaps
    sizes = [0, 1, 2, 7, 8, 9, 17, 0, 1, 0, 2, 7, 9, 17, 8, 1]
    members = []
    for k, n in enumerate(sizes):
        off = 1 + k % 7
        members.append(mixed_batch(n + off + 2, 100 + k, nulls=nulls and k % 3 != 1).slice(off, n))
    check(timing, members, "shared bytes")
    check(timing, members[::-1], "shared bytes, reversed")
    check(timing, [m for m in members if m.num_rows == 0], "all empty")


def test_3000_one_row_members(timing):
    members = [mixed_batch(1 + i % 3, 1000 + i, nulls=i % 2 == 0).slice(i % 3, 1) for i in range(3000)]
    assert check(timing, members, "3000 members").num_rows == 3000


# ---- copy edges ---------------------------------------------------------------------------------------------------------
def binary_member(fo, lengths, rng, kind="binary"):
    """A one-column member whose offsets[0] is `fo` (a slice of a parent with an fo-byte first value)."""
    vals = [bytes(rng.integers(0, 256, n, dtype=np.uint8)) for n in lengths]
    if kind == "utf8":
        vals = [("é" * (n // 2) + "x" * (n % 2)).encode() for n in lengths]
    arr = pa.array([b"\x01" * fo] + vals, pa.binary()).slice(1)
    if kind == "utf8":
        arr = arr.cast(pa.utf8())
    return pa.record_batch([arr], names=["v"])


@pytest.mark.parametrize("kind", ["binary", "utf8"])
def test_span_alignment_classes_and_chunk_edges(timing, kind):
    rng = np.random.default_rng(11)
    members, base, classes, short = [], 0, set(), False
    plan = [(fo, [int(x) for x in rng.integers(0, 9, int(rng.integers(1, 4)))]) for fo in range(0, 33)]
    plan += [(3, [65536]), (0, [65535]), (5, [65537]), (16, [65536, 1]), (7, [2 * 65536 + 3]), (0, [0, 0]), (9, [1])]
    for fo, lengths in plan:
        m = binary_member(fo, lengths, rng, kind)
        nb = int(offsets_of(m.column(0))[-1]) - fo
        x = (fo ^ base) & 15  # the device path's source / destination misalignment
        classes.add(16 if x == 0 else 8 if x & 7 == 0 else 4 if x & 3 == 0 else 1)
        short = short or 0 < nb < (16 - fo % 16) % 16
        members.append(m)
        base += nb
    assert classes == {16, 8, 4, 1} and short
    check(timing, members, kind)


@pytest.mark.parametrize("kind", ["int32", "uint32", "float32", "int64", "float64", "uint64"])
def test_fixed_width_at_odd_row_offsets(timing, kind):
    rng = np.random.default_rng(3)
    members = [pa.record_batch([column(kind, n + 9, rng, nulls=True)], names=["x"]).slice(off, n)
               for n, off in [(1, 1), (3, 3), (16384, 5), (16383, 7), (5, 1), (70000, 3)]]
    check(timing, members, kind)


# ---- scale --------------------------------------------------------------------------------------------------------------
def test_config5_shape_through_tumbling_window(timing):
    # 125 writes of 100 000 63-byte JSON payloads (bench config 5), each row numbered, drained newest write first
    rows, writes = 100_000, 125
    tpl = np.frombuffer(b'{ "timestamp": 1625000000000, "value": 10, "sensor": "temp_0000000" }'[:63], np.uint8)
    assert len(tpl) == 63
    batches = []
    for w in range(writes):
        m = np.tile(tpl, (rows, 1))
        idx = np.arange(w * rows, (w + 1) * rows)
        for d in range(8):  # the row number, 8 decimal digits, over the tail of the payload
            m[:, 54 - d] = ord("0") + (idx // 10 ** d) % 10
        arr = pa.Array.from_buffers(pa.binary(), rows, [None, pa.py_buffer(np.arange(0, 63 * rows + 1, 63, dtype=np.int32)),
                                                        pa.py_buffer(m.tobytes())])
        batches.append(pa.record_batch([arr], schema=pa.schema([pa.field("__value__", pa.binary(), nullable=False)])))
    buf = TumblingWindow({"interval": "1h"})
    for b in batches:
        buf.write(MessageBatch.new_arrow(b))
    timing.ark_kernel_timing_reset()
    got = buf.read()[0].record_batch
    # per input one concat of the 125 writes, then the concat across inputs of that one batch
    assert (launches(timing, COPY), launches(timing, OFFS), launches(timing, BITS)) == (1, 1, 0)
    want = window_drain([(None, b) for b in batches])
    assert got.num_rows == rows * writes
    same_batch(got, want, "config 5")
    buf.close()


def test_mixed_types_ten_million_rows(timing):
    members = [mixed_batch(n, 50 + k) for k, n in enumerate([4_000_001, 3, 2_999_999, 0, 3_000_000])]
    members[2] = members[2].slice(1)
    check(timing, members, "1e7 rows")


# ---- the 2 GiB guard ----------------------------------------------------------------------------------------------------
def bytes_member(data, lo, hi):
    import torch

    off = torch.tensor([lo, hi], dtype=torch.int32, device="cuda")
    return DeviceBatch([DeviceColumn("v", "binary", 1, data, off, None, 0, False)], 1)


def test_binary_total_of_2gib_minus_one(timing):
    import torch

    total = 2 ** 31 - 1
    data = _pattern_bytes(total)
    half = 2 ** 30 + 3
    timing.ark_kernel_timing_reset()
    out = concat_batches_device([bytes_member(data, 0, half), bytes_member(data, half, total)])
    assert (launches(timing, COPY), launches(timing, OFFS), launches(timing, BITS)) == (1, 1, 0)
    c = out.columns[0]
    assert c.offsets.cpu().tolist() == [0, half, total]
    got = c.data.tensor()
    assert got.numel() == total
    step = 1 << 28
    for i0 in range(0, total, step):
        assert torch.equal(got[i0:i0 + step], data[i0:i0 + step]), i0
    del got
    out.close()


@pytest.mark.parametrize("sizes", [[2 ** 30, 2 ** 30], [3 << 29] * 3])
def test_binary_total_beyond_2gib_is_an_error(timing, sizes):
    # 2^31 bytes; three 1.5 GiB members, whose total wraps an int32 back to 0.5 GiB
    import torch

    data = torch.zeros(max(sizes), dtype=torch.uint8, device="cuda")
    with pytest.raises(ArkError) as e:
        concat_batches_device([bytes_member(data, 0, n) for n in sizes])
    assert e.value.kind == "Process" and e.value.message.startswith("Merge batches failed: "), e.value.message


# ---- schema rules at every call site ------------------------------------------------------------------------------------
def one_col(name, values, t=pa.int64(), nullable=True):
    return pa.record_batch([pa.array(values, t)], schema=pa.schema([pa.field(name, t, nullable=nullable)]))


def drain_all(kind, writes, device=False):
    """Every write through one buffer kind (or `batch`), then one read; ('ok', batch) or ('err', ArkError)."""
    try:
        if kind == "batch":
            p = BatchProcessor({"count": len(writes), "timeout_ms": 3_600_000})
            out = [p.process(MessageBatch.new_arrow(rb)) for _, rb in writes]
            assert all(r.is_empty() for r in out[:-1])
            return "ok", out[-1].batches[0].record_batch
        buf = {"memory": lambda: MemoryBuffer({"capacity": 1 << 30, "timeout": "1h"}),
               "tumbling_window": lambda: TumblingWindow({"interval": "1h"}),
               "session_window": lambda: SessionWindow({"gap": "1ms"}),
               "sliding_window": lambda: SlidingWindow({"window_size": len(writes), "interval": "1h", "slide_size": 1})}[kind]()
        for k, (name, rb) in enumerate(writes):
            if device and k % 2:
                buf.write_device(DeviceBatch.from_arrow(rb, keep_offsets=True), input_name=name)
            else:
                buf.write(MessageBatch(rb, name))
        if kind == "memory":
            buf.flush()
        if device:
            r = buf.read_device()
            got = r[0].to_arrow()
        else:
            got = buf.read()[0].record_batch
        buf.close()
        return "ok", got
    except ArkError as e:
        return "err", e


def oracle_drain(kind, writes):
    rbs = [rb for _, rb in writes]
    try:
        if kind == "memory":
            return "ok", memory_drain(rbs)
        if kind == "batch":
            return "ok", batch_processor(rbs, len(rbs))[0]
        if kind == "sliding_window":
            return "ok", sliding_windows(rbs, len(rbs), 1)[0]
        return "ok", window_drain(writes)
    except OracleError as e:
        return "err", e


BUFFER_KINDS = ["memory", "tumbling_window", "session_window", "sliding_window", "batch"]


def check_drain(kind, writes, what, devices=(False, True)):
    want = oracle_drain(kind, writes)
    for device in devices:
        if device and kind == "batch":
            continue  # the batch processor takes host batches
        got = drain_all(kind, writes, device)
        w = (what, kind, "device" if device else "host")
        assert got[0] == want[0], (w, got[1] if got[0] == "err" else got[1].schema)
        if want[0] == "ok":
            same_batch(got[1], want[1], w)
        else:
            assert got[1].kind == want[1].kind == "Process", (w, got[1].message)
            assert got[1].message.startswith("Merge batches failed: "), (w, got[1].message)
            if "non-nullable" in want[1].message:
                assert got[1].message == want[1].message, w
    return want


@pytest.mark.parametrize("kind", BUFFER_KINDS)
def test_names_come_from_the_call_sites_schema_batch(timing, kind):
    writes = [("p", one_col("old", [1, 2])), ("q", one_col("mid", [3])), ("p", one_col("new", [4, None]))]
    want = check_drain(kind, writes, "names")
    assert want[1].schema.names == {"memory": ["old"], "batch": ["old"], "sliding_window": ["old"]}.get(kind, ["new"])


@pytest.mark.parametrize("kind", BUFFER_KINDS)
def test_differing_types_are_a_process_error(timing, kind):
    for other in (one_col("x", [1], pa.int32()), one_col("x", ["1"], pa.utf8()), one_col("x", [None], pa.null())):
        want = check_drain(kind, [("p", one_col("x", [5])), ("p", other)], ("types", str(other.schema.types[0])))
        assert want[0] == "err"


@pytest.mark.parametrize("kind", BUFFER_KINDS)
def test_non_nullable_schema_field_with_nulls(timing, kind):
    strict = pa.record_batch([pa.array([1, 2], pa.int32()), pa.array(["a", "b"])],
                             schema=pa.schema([pa.field("a", pa.int32(), nullable=False), pa.field("s", pa.utf8(), nullable=False)]))
    loose = pa.record_batch([pa.array([3, 4], pa.int32()), pa.array([None, "d"])], names=["a", "s"])
    clean = pa.record_batch([pa.array([None, 5], pa.int32()).slice(1), pa.array(["e"])], names=["a", "s"])
    # memory / batch / sliding take the oldest batch's schema (strict): NULLs there fail; the windows take the newest
    out = check_drain(kind, [("p", strict), ("p", loose)], "strict first")
    assert out[0] == ("err" if kind in ("memory", "batch", "sliding_window") else "ok")
    out = check_drain(kind, [("p", loose), ("p", strict)], "strict last")
    assert out[0] == ("ok" if kind in ("memory", "batch", "sliding_window") else "err")
    assert out[0] == "ok" or out[1].message.endswith("Column 's' is declared as non-nullable but contains null values")
    assert check_drain(kind, [("p", strict), ("p", clean)], "no nulls")[0] == "ok"
    # two inputs: the first input's merged batch gives the schema across inputs
    if kind in ("tumbling_window", "session_window"):
        assert check_drain(kind, [("p", strict), ("q", loose)], "inputs")[0] == "err"
        assert check_drain(kind, [("q", loose), ("p", strict)], "inputs")[0] == "ok"


@pytest.mark.parametrize("with_null", [False, True])
def test_unknown_null_counts_under_a_non_nullable_field(timing, with_null):
    # a validity bitmap whose null count its producer left unknown (-1), as exchanged IPC slices carry it: the bits
    # kernel counts the NULLs, also for one batch, which then does not take the one-batch return
    import torch

    vals = [None if with_null else 4, 5, 6]

    def unknown(nullable):
        data = torch.tensor([v or 0 for v in vals], dtype=torch.int64, device="cuda")
        bits = torch.tensor([0b110 if with_null else 0b111], dtype=torch.uint8, device="cuda")
        return DeviceBatch([DeviceColumn("a", "int64", 3, data, None, bits, -1, nullable)], 3)

    strict = one_col("a", [1, 2], nullable=False)
    for members, head in (([unknown(False)], []), ([DeviceBatch.from_arrow(strict), unknown(True)], [1, 2])):
        timing.ark_kernel_timing_reset()
        if with_null:
            with pytest.raises(ArkError) as e:
                concat_batches_device(members)
            assert (e.value.kind, e.value.message) == ("Process", "Merge batches failed: Invalid argument error: Column 'a' is "
                                                                  "declared as non-nullable but contains null values")
        else:
            got = concat_batches_device(members).to_arrow()
            got.validate(full=True)
            assert got.column(0).to_pylist() == head + vals and not got.schema.field(0).nullable
        assert (launches(timing, COPY), launches(timing, BITS)) == (1, 1)


def test_non_nullable_rule_on_the_concat_entry_points(timing):
    strict = one_col("a", [1, 2], nullable=False)
    check(timing, [strict, one_col("b", [None, 3])], "nulls")
    check(timing, [strict, one_col("b", [None, 3]).slice(1)], "no nulls left")
    check(timing, [one_col("b", [None, 3]), strict], "nullable schema")


# ---- buffers end to end -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", BUFFER_KINDS)
def test_buffers_mixed_writes_every_type(timing, kind):
    writes = [(None, mixed_batch(n + 3, 200 + k, nulls=k % 2 == 0).slice(k % 4, n)) for k, n in enumerate([100, 0, 9, 1000, 17])]
    check_drain(kind, writes, "mixed")


@pytest.mark.parametrize("kind", BUFFER_KINDS)
@pytest.mark.parametrize("col", KINDS)
def test_one_batch_reads_keep_every_type(timing, kind, col):
    rb = mixed_batch(40, KINDS.index(col), kinds=[col, "int64"]).slice(3, 30)
    check_drain(kind, [("p", rb)], ("one batch", col))


def test_avro_file_into_memory_buffer(timing, tmp_path):
    sc = record_schema([("i", "int"), ("f", "float"), ("n", "null"), ("u", ["null", "int"]), ("s", ["string", "null"]),
                        ("d", "double")])
    rows = [(i * 7919 - 40000, float(i) / 8, None, None if i % 3 == 0 else -i, None if i % 5 == 1 else "é%d" % i, i * 0.25)
            for i in range(1000)]
    p = tmp_path / "t.avro"
    p.write_bytes(write_avro(sc, rows, block_rows=[300, 700]))
    for batch_size in (None, 256):
        inp = FileInput(dict({"input_type": {"type": "avro", "path": str(p)}}, **({"batch_size": batch_size} if batch_size else {})))
        inp.connect()
        read = []
        while True:
            try:
                read.append(inp.read()[0].record_batch)
            except ArkError as e:
                assert e.kind == "EOF"
                break
        assert [str(t) for t in read[0].schema.types] == ["int32", "float", "null", "int32", "string", "double"]
        check_drain("memory", [(None, b) for b in read], ("avro", batch_size))
        check_drain("memory", [(None, read[0])], ("avro one batch", batch_size))


def test_protobuf_to_arrow_into_batch(timing, tmp_path):
    fields = [PbField("i", 1, "int32"), PbField("u", 2, "uint32"), PbField("w", 3, "uint64"), PbField("f", 4, "float"),
              PbField("s", 5, "string")]
    dec, _ = processors(tmp_path, fields)
    msgs = [PO.encode_message(fields, {"i": -k, "u": 2 ** 32 - 1 - k, "w": 2 ** 64 - 1 - k, "f": k / 3, "s": "é" * (k % 4)})
            for k in range(50)]
    decoded = [decode(dec, msgs[a:b]) for a, b in [(0, 10), (10, 11), (11, 50)]]
    assert [str(t) for t in decoded[0].schema.types] == ["int32", "uint32", "uint64", "float", "string"]
    check_drain("batch", [(None, d) for d in decoded], "protobuf")
    check_drain("batch", [(None, decoded[2])], "protobuf one batch")


# ---- unsupported types --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arr", [pa.array([[1], [], None], pa.list_(pa.int64())), pa.array([1, None, 3], pa.date32())],
                         ids=["list", "date32"])
def test_unsupported_types_fail_at_every_batch_count(timing, arr):
    rb = pa.record_batch([pa.array([1, 2, 3], pa.int64()), arr], names=["k", "x"])
    for members in ([rb], [rb, rb.slice(1)]):
        with pytest.raises(ArkError) as e:
            concat_batches(members)
        assert e.value.kind == "Unsupported", e.value.message
        for kind in BUFFER_KINDS:
            got = drain_all(kind, [(None, m) for m in members])
            assert got[0] == "err" and got[1].kind == "Unsupported", (kind, len(members), got)
