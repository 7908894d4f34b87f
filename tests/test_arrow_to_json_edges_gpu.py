"""`arrow_to_json` (csrc/arrow_to_json.cu) against the oracle (oracle/json_oracle.py arrow_to_json), at its edges.

Every case runs through the host entry point (process) and the device one (process_device), the latter both with
DeviceBatch.from_arrow(...) and with keep_offsets=True slices (offsets[0] != 0, validity and Boolean bits starting
inside a byte).  The whole `__value__` column must equal the oracle's byte for byte, the passed-through columns must
come back unchanged (Float64 by bit pattern), the output must pass validate(full=True), and the launch counts
(ark_kernel_timing_*) must show one measure and one write launch, and protobuf_sum64_kernel (the exact 64-bit sum of the
row lengths) only when the host's bound on the output passes 2^31 - 1.

Covered: the Float64 writer on a structured corpus of about 1.7 million doubles (tests/f64_corpus.py: every binade's
powers of two and extreme mantissas, subnormals, m * 10^e and their neighbours, the positional window's edges, zeros,
infinities and NaNs), Int64 extremes and powers of ten, every byte of Utf8 and Binary, keys that need escaping and the
72-byte key and 16-column limits, the unsupported types, batch sizes around the 128-row CTA, all-NULL rows at CTA edges,
bit offsets 1 … 7, and the shared-memory staging of the write kernel (a model of the launcher predicts which CTAs are
staged; CTAs at exactly stage - 16 and stage - 15 bytes, staged CTAs at every output address residue mod 16).

The 2 GiB limit of a Binary column: 2^31 - 1 output bytes in one row and over many CTAs must be written correctly
(checked on the device, chunk by chunk), and 2^31 bytes, a total that an int32 wraps back to a positive value, a row that
is negative in int32 and a row that an int32 wraps back to a positive length must all be Process errors raised before
the write kernel launches.
"""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

from arkflow_b200.arrow_ffi import DeviceBatch, DeviceColumn
from arkflow_b200.processor import ArkError, ArrowToJsonProcessor, MessageBatch
from f64_corpus import corpus_bits
from oracle.json_oracle import arrow_to_json

pytestmark = pytest.mark.gpu

KERNELS = ("arrow_to_json_measure_kernel", "arrow_to_json_write_kernel", "protobuf_sum64_kernel")
I32_MAX = 2 ** 31 - 1
CTA, STAGE_MAX = 128, 44 * 1024
MIB = 1 << 20


# ---- launch counts -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def timing(gpu):
    gpu.ark_kernel_timing_enable(1)
    yield gpu
    gpu.ark_kernel_timing_enable(0)


def _launches(lib):
    out = {}
    for name in KERNELS:
        ms, n = C.c_double(), C.c_int64()
        lib.ark_kernel_timing_get(name.encode(), C.byref(ms), C.byref(n))
        out[name] = n.value
    return out


def _escaped_key_len(name: str) -> int:
    """Bytes of `"name":` as the encoder writes it (serde_json escapes, \\u00xx for other control characters)."""
    n = 3
    for ch in name.encode():
        n += 2 if ch in b'"\\\b\f\n\r\t' else 6 if ch < 0x20 else 1
    return n


def output_bound(rb: pa.RecordBatch, include=None) -> int:
    """The launcher's bound on the output bytes: per row 2 + each emitted column's key, comma and widest value (Int64
    20, Float64 24, Bool 5, string quotes 2), plus 6 bytes per Utf8 byte and 2 per Binary byte."""
    row, var = 2, 0
    for f, col in zip(rb.schema, rb.columns):
        if f.type == pa.null() or (include is not None and f.name not in include):
            continue
        row += _escaped_key_len(f.name) + 1 + {pa.int64(): 20, pa.float64(): 24, pa.bool_(): 5}.get(f.type, 2)
        if f.type in (pa.utf8(), pa.binary()):
            offs = np.frombuffer(col.buffers()[1], np.int32)[col.offset:col.offset + len(col) + 1]
            var += (6 if f.type == pa.utf8() else 2) * (int(offs[-1]) - int(offs[0]) if len(col) else 0)
    return var + rb.num_rows * row


def want_launches(n: int, bound: int) -> dict:
    return {"arrow_to_json_measure_kernel": int(n > 0), "arrow_to_json_write_kernel": int(n > 0),
            "protobuf_sum64_kernel": int(n > 0 and bound > I32_MAX)}


# ---- the staging model -------------------------------------------------------------------------------------------------
def stage_of(total: int, n: int) -> int:
    """The write kernel's shared-memory window: the average CTA's bytes + 50 % + 256, rounded up to 1 KiB, at most
    44 KiB."""
    return min(STAGE_MAX, -(-(int(total / n * CTA * 1.5) + 256) // 1024) * 1024)


def stage_plan(line_lens):
    """(stage bytes, [(CTA output start, CTA bytes, staged)]) as arrow_to_json_device launches the write kernel: a CTA
    is staged iff its bytes fit the window less 16 (the misalignment slack)."""
    lens = np.asarray(line_lens, np.int64)
    n, total = len(lens), int(lens.sum())
    if n == 0:
        return 0, []
    stage = stage_of(total, n)
    starts = np.concatenate([[0], np.cumsum(lens)])
    ctas = []
    for c in range(0, n, CTA):
        b0, b1 = int(starts[c]), int(starts[min(c + CTA, n)])
        ctas.append((b0, b1 - b0, b1 - b0 <= stage - 16))
    return stage, ctas


# ---- running one case --------------------------------------------------------------------------------------------------
def to_device(rb, keep_offsets=False):
    """DeviceBatch.from_arrow, with Null-typed columns (which it does not upload) put back in their places."""
    keep = [i for i, f in enumerate(rb.schema) if f.type != pa.null()]
    sub = pa.RecordBatch.from_arrays([rb.column(i) for i in keep], schema=pa.schema([rb.schema.field(i) for i in keep]))
    up = iter(DeviceBatch.from_arrow(sub, keep_offsets=keep_offsets).columns)
    cols = [next(up) if f.type != pa.null() else DeviceColumn(f.name, "null", rb.num_rows, None, null_count=rb.num_rows)
            for f in rb.schema]
    return DeviceBatch(cols, rb.num_rows)


def _routes(rb):
    """(name, callable(proc) -> RecordBatch) for the host entry, the device entry and device slices."""
    yield "host", lambda p: p.process(MessageBatch.new_arrow(rb)).batches[0].record_batch
    yield "device", lambda p: p.process_device(to_device(rb)).to_arrow()
    if any(c.offset for c in rb.columns):
        yield "device-slices", lambda p: p.process_device(to_device(rb, keep_offsets=True)).to_arrow()


def _same_column(a: pa.Array, b: pa.Array) -> bool:
    if b.type == pa.float64():
        if a.null_count != b.null_count or not a.is_null().equals(b.is_null()):
            return False
        fa = a.to_numpy(zero_copy_only=False) if a.null_count == 0 else a.fill_null(0.0).to_numpy(zero_copy_only=False)
        fb = b.to_numpy(zero_copy_only=False) if b.null_count == 0 else b.fill_null(0.0).to_numpy(zero_copy_only=False)
        return np.array_equal(fa.view(np.uint64), fb.view(np.uint64))
    return a.equals(b)


def check(timing, rb, cfg=None, want=None, staging=None):
    """Run rb through every route and compare with the oracle.  staging = (n staged CTAs, n direct CTAs) asserts the
    mix the case was built for, from the oracle's line lengths."""
    inc = set(cfg["fields_to_include"]) if cfg and "fields_to_include" in cfg else None
    want = arrow_to_json(rb, inc) if want is None else want
    wv = want.column(want.num_columns - 1)
    bound = output_bound(rb, inc)
    if staging is not None:
        lens = np.diff(np.frombuffer(wv.buffers()[1], np.int32)[: rb.num_rows + 1])
        _, ctas = stage_plan(lens)
        assert (sum(s for _, _, s in ctas), sum(not s for _, _, s in ctas)) == staging
    proc = ArrowToJsonProcessor(cfg or {})
    for route, run in _routes(rb):
        timing.ark_kernel_timing_reset()
        got = run(proc)
        launched = _launches(timing)
        assert launched == want_launches(rb.num_rows, bound), (route, launched, bound)
        got.validate(full=True)
        assert got.schema.names == want.schema.names, route
        assert got.num_rows == want.num_rows, route
        gv = got.column(got.num_columns - 1)
        assert gv.type == pa.binary() and gv.null_count == 0, route
        if not gv.equals(wv):
            g, w = gv.to_pylist(), wv.to_pylist()
            bad = next(i for i in range(len(w)) if g[i] != w[i])
            raise AssertionError((route, bad, g[bad], w[bad]))
        for i in range(rb.num_columns):
            assert _same_column(got.column(i), rb.column(i)), (route, rb.schema.names[i])
    return want


# ---- Float64 -----------------------------------------------------------------------------------------------------------
def test_float64_structured_corpus_bit_for_bit(timing):
    bits = corpus_bits()
    rb = pa.record_batch({"f": pa.array(bits.view(np.float64), pa.float64())})
    check(timing, rb)
    # the same values behind NULLs, as a slice starting inside a validity byte
    rng = np.random.default_rng(1)
    sub = bits[rng.choice(len(bits), 200_003, replace=False)]
    rb = pa.record_batch({"f": pa.array(sub.view(np.float64), pa.float64(), mask=rng.random(len(sub)) < 0.1),
                          "i": pa.array(np.arange(len(sub)), pa.int64())}).slice(5, 200_000)
    check(timing, rb)


# ---- Int64 -------------------------------------------------------------------------------------------------------------
def test_int64_extremes_and_powers_of_ten(timing):
    vals = [-2 ** 63, 2 ** 63 - 1, 0, -1, 1]
    for k in range(19):
        vals += [10 ** k, -10 ** k, 10 ** k - 1, -(10 ** k - 1), 10 ** k + 1, -(10 ** k + 1)]
    vals += [2 ** 63 - 2, -2 ** 63 + 1, 2 ** 62, -2 ** 62, 2 ** 32, -2 ** 32, 2 ** 31 - 1, -2 ** 31]
    rb = pa.record_batch({"i": pa.array(vals, pa.int64())})
    check(timing, rb)
    rng = np.random.default_rng(2)
    big = np.array(vals * 40, np.int64)
    rb = pa.record_batch({"i": pa.array(big, pa.int64(), mask=rng.random(len(big)) < 0.2),
                          "j": pa.array(big[::-1].copy(), pa.int64())}).slice(3, len(big) - 7)
    check(timing, rb)


# ---- strings -----------------------------------------------------------------------------------------------------------
# 1- to 4-byte UTF-8 at the ends of each length, U+2028 / U+2029 (verbatim in JSON), quotes and backslashes
UTF8_SEQS = [chr(c) for c in (0x80, 0xE9, 0x7FF, 0x800, 0x6F22, 0xD7FF, 0xE000, 0xFFFF, 0x10000, 0x1F600, 0x10FFFF, 0x2028, 0x2029)]
UTF8_SEQS += ["a\u2028b\u2029c", '"', "\\", "", '"\\"', '\\"', "\x7f", "/", "</script>"]


def test_utf8_every_ascii_byte_and_multibyte_sequences(timing):
    strs = [chr(b) for b in range(0x80)] + UTF8_SEQS + ["".join(chr(b) for b in range(0x80)) * 3]
    rb = pa.record_batch({"s": pa.array(strs, pa.utf8())})
    want = check(timing, rb)
    lines = want.column(1).to_pylist()
    # the seven short escapes, \u00xx in lowercase and DEL verbatim
    assert lines[0x08] == b'{"s":"\\b"}' and lines[0x0C] == b'{"s":"\\f"}' and lines[0x0A] == b'{"s":"\\n"}'
    assert lines[0x0D] == b'{"s":"\\r"}' and lines[0x09] == b'{"s":"\\t"}'
    assert lines[0x22] == b'{"s":"\\""}' and lines[0x5C] == b'{"s":"\\\\"}'
    assert lines[0x1F] == b'{"s":"\\u001f"}' and lines[0x7F] == b'{"s":"\x7f"}'
    # with NULLs and as a slice whose first offset is not 0
    rng = np.random.default_rng(3)
    many = [strs[int(k)] for k in rng.integers(0, len(strs), 5000)]
    rb = pa.record_batch({"s": pa.array(many, pa.utf8(), mask=rng.random(5000) < 0.1)}).slice(77, 4000)
    check(timing, rb)


def test_binary_every_byte_value(timing):
    vals = [bytes([b]) for b in range(256)] + [bytes(range(256)), b"", bytes(range(255, -1, -1)) * 4]
    rb = pa.record_batch({"z": pa.array(vals, pa.binary())})
    want = check(timing, rb)
    assert want.column(1)[0xAB].as_py() == b'{"z":"ab"}'
    rng = np.random.default_rng(4)
    many = [bytes(rng.integers(0, 256, int(k)).tolist()) for k in rng.integers(0, 40, 3000)]
    rb = pa.record_batch({"z": pa.array(many, pa.binary(), mask=rng.random(3000) < 0.1),
                          "s": pa.array([m.hex() for m in many], pa.utf8())}).slice(129, 2500)
    check(timing, rb)


def test_long_rows_take_the_direct_path(timing):
    """A CTA of escaped control characters (6 output bytes each) among short rows: its bytes pass the window and it
    formats straight into global memory; every other CTA is staged."""
    n = 128 * 6
    strs = ["r%d" % i for i in range(n)]
    for r in range(256, 384):
        strs[r] = "\x01\n\"" * (40 + r) if r % 3 else "\x1f" * 600
    rb = pa.record_batch({"s": pa.array(strs, pa.utf8()), "z": pa.array([s.encode()[:5] for s in strs], pa.binary())})
    check(timing, rb, staging=(5, 1))
    check(timing, rb.slice(1, n - 2), staging=(5, 1))


# ---- keys and columns --------------------------------------------------------------------------------------------------
def test_keys_that_need_escaping(timing):
    names = ['q"uote', "back\\slash", "tab\tnl\nret\r", "ctl\x01\x1f\x7f", "é漢😀", "\b\f", "", "/", " "]
    rng = np.random.default_rng(5)
    rb = pa.record_batch({nm: pa.array(rng.integers(-5, 5, 300), pa.int64(), mask=rng.random(300) < 0.3) for nm in names})
    want = check(timing, rb)
    assert b'"ctl\\u0001\\u001f\x7f":' in b"".join(want.column(len(names)).to_pylist())


def test_key_of_72_bytes_is_accepted_73_unsupported(timing):
    ok = "k" * 69  # `"` + 69 + `":` = 72 bytes
    assert _escaped_key_len(ok) == 72
    check(timing, pa.record_batch({ok: pa.array([1, None, 3], pa.int64())}))
    esc = "\x01" * 11 + "abc"  # 11 * 6 + 3 + 3 = 72 bytes once escaped
    assert _escaped_key_len(esc) == 72
    check(timing, pa.record_batch({esc: pa.array([True, False], pa.bool_())}))
    for name in ("k" * 70, "\x01" * 11 + "abcd", "é" * 35):
        assert _escaped_key_len(name) == 73
        rb = pa.record_batch({"a": pa.array([1], pa.int64()), name: pa.array([1], pa.int64())})
        for route, run in _routes(rb):
            with pytest.raises(ArkError) as e:
                run(ArrowToJsonProcessor({}))
            assert e.value.kind == "Unsupported" and "too long" in e.value.message, (route, e.value.message)


def test_sixteen_columns_accepted_seventeenth_unsupported(timing):
    rng = np.random.default_rng(6)
    n = 300
    cols = {}
    for k in range(16):
        t = k % 5
        arr = [pa.array(rng.integers(-10 ** 6, 10 ** 6, n), pa.int64()), pa.array(rng.normal(0, 1e4, n), pa.float64()),
               pa.array(rng.random(n) < 0.5, pa.bool_()), pa.array(["v%d" % v for v in rng.integers(0, 99, n)], pa.utf8()),
               pa.array([bytes([v]) for v in rng.integers(0, 256, n)], pa.binary())][t]
        cols["c%02d" % k] = pa.array(arr.to_pylist(), arr.type, mask=rng.random(n) < 0.1)
    cols["nul"] = pa.nulls(n)  # a Null column is never emitted and does not count
    check(timing, pa.record_batch(cols))
    cols17 = dict(cols, extra=pa.array(np.arange(n), pa.int64()))
    rb17 = pa.record_batch(cols17)
    for route, run in _routes(rb17):
        with pytest.raises(ArkError) as e:
            run(ArrowToJsonProcessor({}))
        assert e.value.kind == "Unsupported" and "16 columns" in e.value.message, (route, e.value.message)
    # a column left out by fields_to_include does not count either
    keep = [nm for nm in cols17 if nm != "c03"]
    check(timing, rb17, {"fields_to_include": keep})


def test_fields_to_include_naming_no_column_is_a_process_error(timing):
    rb = pa.record_batch({"a": pa.array([1, 2], pa.int64()), "b": pa.array(["x", None])})
    for route, run in _routes(rb):
        with pytest.raises(ArkError) as e:
            run(ArrowToJsonProcessor({"fields_to_include": ["zz"]}))
        assert e.value.kind == "Process" and "same length" in e.value.message, (route, e.value.message)
    check(timing, rb, {"fields_to_include": ["b"]})


@pytest.mark.parametrize("arr", [pa.array([1, 2], pa.int32()), pa.array([[1], []], pa.list_(pa.int64())),
                                 pa.array([1, 2], pa.date32())], ids=["int32", "list", "date32"])
def test_unsupported_types_name_the_column(gpu, arr):
    rb = pa.record_batch({"ok": pa.array([1, 2], pa.int64()), "bad col": arr})
    runs = [("host", lambda p: p.process(MessageBatch.new_arrow(rb)))]
    if arr.type == pa.int32():
        runs.append(("device", lambda p: p.process_device(to_device(rb))))
    for route, run in runs:
        with pytest.raises(ArkError) as e:
            run(ArrowToJsonProcessor({}))
        assert e.value.kind == "Unsupported" and "'bad col'" in e.value.message, (route, e.value.message)


# ---- shapes, NULLs and bits --------------------------------------------------------------------------------------------
def mixed(n, rng, null_rows=()):
    """Int64, Float64, Bool, Utf8, Binary and Null columns with NULLs; every field of the rows in null_rows is NULL."""
    allnull = np.zeros(n, bool)
    allnull[[r for r in null_rows if 0 <= r < n]] = True
    m = lambda p: (rng.random(n) < p) | allnull  # noqa: E731
    pool = ["", "a", 'q"', "t\tn\n", "é漢", "\x00\x1f", "x" * 50]
    return pa.record_batch({
        "i": pa.array(rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64), pa.int64(), mask=m(0.1)),
        "f": pa.array(rng.normal(0, 1e6, n), pa.float64(), mask=m(0.1)),
        "b": pa.array(rng.random(n) < 0.5, pa.bool_(), mask=m(0.2)),
        "s": pa.array([pool[int(k)] for k in rng.integers(0, len(pool), n)], pa.utf8(), mask=m(0.1)),
        "z": pa.array([bytes(rng.integers(0, 256, int(k)).tolist()) for k in rng.integers(0, 6, n)], pa.binary(), mask=m(0.1)),
        "n": pa.nulls(n),
    })


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 255, 256, 257])
def test_batch_sizes_and_all_null_rows_at_cta_edges(timing, n):
    rng = np.random.default_rng(100 + n)
    edges = (0, 126, 127, 128, 129, 254, 255, 256, n - 1)
    rb = mixed(n, rng, null_rows=edges)
    want = check(timing, rb)
    lines = want.column(want.num_columns - 1).to_pylist()
    assert all(lines[r] == b"{}" for r in edges if 0 <= r < n)


def test_batch_of_2_20_plus_3_rows(timing):
    n = 2 ** 20 + 3
    rng = np.random.default_rng(7)
    allnull = np.zeros(n, bool)
    allnull[np.arange(127, n, 128)] = True
    rb = pa.record_batch({
        "i": pa.array(rng.integers(-2 ** 63, 2 ** 63 - 1, n, dtype=np.int64), pa.int64(), mask=allnull | (rng.random(n) < 0.1)),
        "b": pa.array(rng.random(n) < 0.5, pa.bool_(), mask=allnull),
    })
    want = check(timing, rb)
    lines = want.column(2)
    assert all(lines[int(r)].as_py() == b"{}" for r in np.arange(127, n, 128))


@pytest.mark.parametrize("bit", range(1, 8))
def test_bool_data_and_validity_at_bit_offsets(timing, bit):
    rng = np.random.default_rng(200 + bit)
    n = 1000
    base = pa.record_batch({
        "b": pa.array(rng.random(n) < 0.5, pa.bool_(), mask=rng.random(n) < 0.25),
        "t": pa.array(rng.random(n) < 0.5, pa.bool_()),  # no validity: data bits only
        "s": pa.array(["s%d" % k for k in rng.integers(0, 10 ** bit, n)], pa.utf8(), mask=rng.random(n) < 0.25),
        "z": pa.array([bytes([k]) * (k % 4) for k in rng.integers(0, 256, n)], pa.binary()),
    })
    for start, length in ((bit, 700), (8 + bit, 129), (16 * bit + bit, 1)):
        rb = base.slice(start, length)
        assert all(c.offset == start for c in rb.columns)
        check(timing, rb)


# ---- staging -----------------------------------------------------------------------------------------------------------
def _fill_cta(tb, key="s"):
    """128 Utf8 values of plain letters whose lines `{"s":"…"}` add up to exactly tb bytes."""
    fixed = len('{"%s":""}' % key)
    body = tb - CTA * fixed
    assert body >= 0
    q, r = divmod(body, CTA)
    return ["abcdefghijklmnopqrstuvwxyz"[i % 26] * (q + (i < r)) for i in range(CTA)]


def _cta_batch(tbs):
    vals = [v for tb in tbs for v in _fill_cta(tb)]
    return pa.record_batch({"s": pa.array(vals, pa.utf8())})


def test_staging_window_boundary(timing):
    """Two CTAs at exactly stage - 16 (staged) and stage - 15 (direct) bytes, among fillers that set the window."""
    S = 8192
    filler = next(f for f in range(CTA * 8, S) if stage_of(2 * S - 31 + 6 * f, 8 * CTA) == S)
    tbs = [filler, S - 16, filler, S - 15, filler, filler, filler, filler]
    rb = _cta_batch(tbs)
    want = arrow_to_json(rb)
    lens = np.diff(np.frombuffer(want.column(1).buffers()[1], np.int32)[: rb.num_rows + 1])
    stage, ctas = stage_plan(lens)
    assert stage == S and [tb for _, tb, _ in ctas] == tbs
    assert [s for _, _, s in ctas] == [True, True, True, False, True, True, True, True]
    check(timing, rb, want=want, staging=(7, 1))


def test_staged_ctas_at_every_output_residue(timing):
    """17 staged CTAs of 128 * 9 + 1 bytes: their output starts cover every residue mod 16, so the 16-byte stores of
    the staged image start at every misalignment."""
    tb = CTA * 9 + 1
    rb = _cta_batch([tb] * 17)
    want = arrow_to_json(rb)
    lens = np.diff(np.frombuffer(want.column(1).buffers()[1], np.int32)[: rb.num_rows + 1])
    _, ctas = stage_plan(lens)
    assert all(s for _, _, s in ctas) and {b0 % 16 for b0, _, _ in ctas} == set(range(16))
    check(timing, rb, want=want, staging=(17, 0))
    # the same rows behind a leading row of 1..15 extra bytes, and a partial last CTA
    for pad in (1, 7, 15):
        rb2 = pa.record_batch({"s": pa.array(["p" * pad] + rb.column(0).to_pylist()[:-5], pa.utf8())})
        check(timing, rb2)


# ---- 2 GiB (inputs built on the device) --------------------------------------------------------------------------------
HEX = b"0123456789abcdef"


def _torch():
    import torch

    return torch


def _dev_int64(name, vals, validity=None, null_count=0):
    torch = _torch()
    return DeviceColumn(name, "int64", len(vals), torch.tensor(vals, dtype=torch.int64, device="cuda"), None, validity,
                        null_count, validity is not None)


def _dev_var(name, dtype, data, offsets):
    torch = _torch()
    offs = torch.tensor(offsets, dtype=torch.int32, device="cuda") if not hasattr(offsets, "device") else offsets
    return DeviceColumn(name, dtype, offs.numel() - 1, data, offs, None, 0, False)


def _run_device(timing, cols, n):
    timing.ark_kernel_timing_reset()
    try:
        out = ArrowToJsonProcessor({}).process_device(DeviceBatch(cols, n))
    finally:
        launched = _launches(timing)
    return out, launched


def _value_column(out):
    v = out.columns[-1]
    assert v.name == "__value__" and v.dtype == "binary"
    return v


@pytest.fixture(scope="module")
def ones(gpu):
    """768 MiB of 0x01 bytes: the Utf8 data of every control-character case."""
    torch = _torch()
    t = torch.ones(768 * MIB, dtype=torch.uint8, device="cuda")
    yield t
    del t
    torch.cuda.empty_cache()


def test_2gib_minus_one_bytes_in_one_row(timing):
    """{"i":10,"z":"<hex of 2^30 - 8 bytes>"}: 15 + 2^31 - 16 = 2^31 - 1 bytes, all in one CTA, which takes the direct
    path (the staging test tb > stage - 16 holds; tb + 16 would overflow int32)."""
    torch = _torch()
    L = 2 ** 30 - 8
    assert 13 + 2 * L + 2 == I32_MAX
    z = torch.empty(L, dtype=torch.uint8, device="cuda")
    for j0 in range(0, L, 256 * MIB):  # byte j = j % 251
        z[j0:j0 + 256 * MIB] = (torch.arange(j0, min(j0 + 256 * MIB, L), device="cuda") % 251).to(torch.uint8)
    out, launched = _run_device(timing, [_dev_int64("i", [10]), _dev_var("z", "binary", z, [0, L])], 1)
    bound = 2 + (4 + 1 + 20) + (4 + 1 + 2) + 2 * L
    assert launched == want_launches(1, bound), launched
    v = _value_column(out)
    offs = v.offsets.cpu().numpy()
    assert offs.tolist() == [0, I32_MAX]
    data = v.data.tensor()
    assert data.numel() == I32_MAX
    assert bytes(data[:13].cpu().numpy()) == b'{"i":10,"z":"' and bytes(data[-2:].cpu().numpy()) == b'"}'
    lut = torch.tensor(list(HEX), dtype=torch.uint8, device="cuda")
    step = 256 * MIB
    for j0 in range(0, L, step):
        zz = z[j0:j0 + step].to(torch.int64)
        want = torch.stack([lut[zz >> 4], lut[zz & 15]], dim=1).reshape(-1)
        got = data[13 + 2 * j0: 13 + 2 * j0 + want.numel()]
        assert torch.equal(got, want), j0
    del data, z
    out.close()


def test_2gib_minus_one_bytes_over_many_ctas(timing, ones):
    """3 * 2^15 rows {"i":D,"s":"\\u0001…"}: 14 + 6 L bytes each, one row with i = 10 adds 1: 2^31 - 1 bytes in all.
    Even CTAs hold empty strings (staged), odd CTAs the long ones (direct)."""
    torch = _torch()
    n = 3 * 2 ** 15
    body = (I32_MAX - 1 - 14 * n)
    assert body % 6 == 0
    long_rows = np.arange(n)[(np.arange(n) // CTA) % 2 == 1]
    lens = np.zeros(n, np.int64)
    q, r = divmod(body // 6, len(long_rows))
    lens[long_rows] = q
    lens[long_rows[:r]] += 1
    offsets = np.concatenate([[0], np.cumsum(lens)])
    assert offsets[-1] <= ones.numel()
    ivals = [1] * n
    ivals[n // 2 + 5] = 10
    line = 14 + 6 * lens + (np.array(ivals) == 10)
    assert int(line.sum()) == I32_MAX
    stage, ctas = stage_plan(line)
    assert stage == STAGE_MAX and sum(s for _, _, s in ctas) == len(ctas) // 2
    cols = [_dev_int64("i", ivals), _dev_var("s", "utf8", ones[:int(offsets[-1])], offsets.astype(np.int32).tolist())]
    out, launched = _run_device(timing, cols, n)
    bound = n * (2 + (4 + 1 + 20) + (4 + 1 + 2)) + 6 * int(offsets[-1])
    assert launched == want_launches(n, bound), launched
    v = _value_column(out)
    want_offs = np.concatenate([[0], np.cumsum(line)])
    assert np.array_equal(v.offsets.cpu().numpy().astype(np.int64), want_offs)
    data = v.data.tensor()
    assert data.numel() == I32_MAX
    # every line as the device expects it, built in torch from the line offsets, 128 Mi output bytes at a time
    offs_t = torch.tensor(want_offs, dtype=torch.int64, device="cuda")
    ten = torch.tensor(np.array(ivals) == 10, device="cuda")
    pre1, pre2 = (torch.tensor(list(p), dtype=torch.uint8, device="cuda") for p in (b'{"i":1,"s":"', b'{"i":10,"s":"'))
    esc = torch.tensor(list(b"\\u0001"), dtype=torch.uint8, device="cuda")
    step = 128 * MIB
    for p0 in range(0, I32_MAX, step):
        pos = torch.arange(p0, min(p0 + step, I32_MAX), device="cuda", dtype=torch.int64)
        row = torch.searchsorted(offs_t, pos, right=True) - 1
        k = pos - offs_t[row]
        end = offs_t[row + 1] - pos  # 1 = the closing brace, 2 = the closing quote
        is10 = ten[row]
        plen = torch.where(is10, 13, 12)
        want = esc[((k - plen).clamp(min=0)) % 6]
        want = torch.where(k < plen, torch.where(is10, pre2[k.clamp(max=12)], pre1[k.clamp(max=11)]), want)
        want = torch.where(end == 2, torch.tensor(ord('"'), dtype=torch.uint8, device="cuda"), want)
        want = torch.where(end == 1, torch.tensor(ord("}"), dtype=torch.uint8, device="cuda"), want)
        assert torch.equal(data[p0:p0 + pos.numel()], want), p0
    del data
    out.close()


def test_2gib_exactly_is_a_process_error(timing):
    """{"i":100,"z":"<hex of 2^30 - 8 bytes>"}: 2^31 bytes, one past the int32 offsets."""
    torch = _torch()
    L = 2 ** 30 - 8
    z = torch.zeros(L, dtype=torch.uint8, device="cuda")
    with pytest.raises(ArkError) as e:
        _run_device(timing, [_dev_int64("i", [100]), _dev_var("z", "binary", z, [0, L])], 1)
    assert e.value.kind == "Process" and "arrow_to_json" in e.value.message and "2 GiB" in e.value.message, e.value.message
    assert _launches(timing) == {"arrow_to_json_measure_kernel": 1, "arrow_to_json_write_kernel": 0, "protobuf_sum64_kernel": 1}


@pytest.mark.parametrize("case", ["8x96MiB", "400MiB", "768MiB"])
def test_2gib_control_characters_past_the_limit_are_process_errors(timing, ones, case):
    """Utf8 rows of 0x01 bytes, 6 output bytes each (\\u0001), line = 8 + 6 L:
    8 x 96 MiB: 4.5 GiB in all, which an int32 scan wraps to +0.5 GiB (each row fits int32);
    400 MiB: one row of 2.3 GiB, negative as an int32;
    768 MiB: one row of 4.5 GiB, which an int32 row length wraps back to a positive 0.5 GiB."""
    rows, L = {"8x96MiB": (8, 96 * MIB), "400MiB": (1, 400 * MIB), "768MiB": (1, 768 * MIB)}[case]
    line = 8 + 6 * L
    total = rows * line
    wrapped = (total + 2 ** 31) % 2 ** 32 - 2 ** 31  # the total as an int32 scan leaves it
    if case == "8x96MiB":
        assert line <= I32_MAX and 2 ** 32 < total < 2 ** 32 + 2 ** 31 and 0 < wrapped == total - 2 ** 32
    elif case == "400MiB":
        assert 2 ** 31 < line < 2 ** 32 and wrapped < 0
    else:
        row_wrapped = (line + 2 ** 31) % 2 ** 32 - 2 ** 31
        assert 2 ** 32 < line and 0 < row_wrapped < 2 ** 31
    offsets = [k * L for k in range(rows + 1)]
    with pytest.raises(ArkError) as e:
        _run_device(timing, [_dev_var("s", "utf8", ones[:rows * L], offsets)], rows)
    assert e.value.kind == "Process" and "arrow_to_json" in e.value.message and "2 GiB" in e.value.message, e.value.message
    assert _launches(timing) == {"arrow_to_json_measure_kernel": 1, "arrow_to_json_write_kernel": 0, "protobuf_sum64_kernel": 1}
