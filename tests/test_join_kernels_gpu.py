"""The hash join, its gathers and the hash repartition (csrc/hash_join.cu) against the oracle, at their edges.

Every join case runs through the host entry point (process_tables) and the device one (process_tables_device), and,
where a case says so, through device slices (DeviceBatch.from_arrow(keep_offsets=True): data pointers off 16-byte
alignment, offsets[0] != 0, validity and Boolean bits starting inside a byte).  Each input carries an Int64 row id;
both the engine's output and the oracle's (oracle/sql_oracle.py sql_join) are sorted by (left id, right id), NULLs
last.  Schema names, types and nullability must be equal; every result is validated in full; non-float columns are
compared with Array.equals and Float64 columns through their uint64 view (NaN payloads and -0.0 bit for bit).

Each run also checks which gather kernels launched (ark_kernel_timing_*): take_columns hands up to 8 plain fixed-width
and 4 plain string columns to take_multi_kernel and everything else to take_column (take_fixed8 / take_bits /
take_lengths + take_bytes_tile, take_bits or take_matched for the validity).  The launch counts are predicted per
column, so a column that silently takes the other path fails.  For string columns the test also predicts, with the
launcher's staging formula, which 1024-row tiles of take_bytes_tile_kernel take the per-row branch.

The output-size guard (a string column of more than 2^31 - 1 bytes is a Process error) is checked at 2^31 - 1,
2^31, inside (2^31, 2^32) and past 2^32, where an int32 total wraps back to a positive value.
"""
import ctypes as C

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from arkflow_b200.arrow_ffi import DeviceBatch, DeviceColumn
from arkflow_b200.dist import NativeEngine
from arkflow_b200.processor import ArkError, SqlProcessor
from oracle.sql_oracle import sql_join

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
GATHERS = ("take_multi_kernel", "take_fixed8_kernel", "take_bits_kernel", "take_matched_kernel", "take_lengths_kernel",
           "take_bytes_tile_kernel")
TAKE_TILE, TAKE_STAGE_MAX, TAKE_MAX_FIXED, TAKE_MAX_STR = 1024, 44 * 1024, 8, 4
NAN_BITS = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFFFFFFFFFFFFFFF, 0x8000000000000000,
                     0x0000000000000001, 0x7FF0000000000000], np.uint64)


# ---- launch counts -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def timing(gpu):
    gpu.ark_kernel_timing_enable(1)
    yield gpu
    gpu.ark_kernel_timing_enable(0)


def _launches(lib):
    out = {}
    for name in GATHERS:
        ms, n = C.c_double(), C.c_int64()
        lib.ark_kernel_timing_get(name.encode(), C.byref(ms), C.byref(n))
        out[name] = n.value
    return out


def predict_gathers(srcs, n_out):
    """Launch counts of the gathers of one output batch: srcs = [(source array, may_miss)] in output order."""
    want = dict.fromkeys(GATHERS, 0)
    if n_out == 0:  # nothing to gather: no launch at all
        return want
    n_fixed = n_str = 0
    for arr, may_miss in srcs:
        t = arr.type
        has_validity = arr.null_count > 0
        plain = not has_validity and not may_miss
        fixed = t in (pa.int64(), pa.float64())
        var = t in (pa.utf8(), pa.binary())
        if plain and fixed and n_fixed < TAKE_MAX_FIXED:
            n_fixed += 1
            continue
        if plain and var and n_str < TAKE_MAX_STR:
            n_str += 1
            continue
        if fixed:
            want["take_fixed8_kernel"] += 1
        elif t == pa.bool_():
            want["take_bits_kernel"] += 1
        elif var:
            want["take_lengths_kernel"] += 1
            want["take_bytes_tile_kernel"] += 1
        if has_validity:
            want["take_bits_kernel"] += 1
        elif may_miss:
            want["take_matched_kernel"] += 1
    if n_fixed or n_str:
        want["take_multi_kernel"] = 1
        want["take_bytes_tile_kernel"] += n_str
    return want


def tile_branches(arr):
    """(staged tiles, per-row tiles) of take_bytes_tile_kernel for the string column `arr` as the engine emitted it: the
    launcher sizes staging as min(44 KiB, round_up(total / n * 1024 * 1.5 + 256, 1024)), and a tile whose bytes tb
    satisfy tb + 16 > stage is copied row by row."""
    n = len(arr)
    if n == 0:
        return 0, 0
    off = np.frombuffer(arr.buffers()[1], np.int32)[arr.offset:arr.offset + n + 1].astype(np.int64)
    total = int(off[-1] - off[0])
    stage = min(TAKE_STAGE_MAX, -(-(int(total / n * TAKE_TILE * 1.5) + 256) // 1024) * 1024)
    ends = np.minimum(np.arange(0, n, TAKE_TILE) + TAKE_TILE, n)
    tb = off[ends] - off[np.arange(0, n, TAKE_TILE)]
    per_row = int((tb + 16 > stage).sum())
    return len(tb) - per_row, per_row


# ---- inputs ------------------------------------------------------------------------------------------------------------
def varlen(lengths, binary=False, salt=0):
    """Strings of the given lengths: ASCII letters (Utf8) or every byte value, NUL included (Binary)."""
    lengths = np.asarray(lengths, np.int64)
    offsets = np.zeros(len(lengths) + 1, np.int64)
    np.cumsum(lengths, out=offsets[1:])
    pos = np.arange(offsets[-1], dtype=np.int64) * 131 + salt
    data = (pos % 256 if binary else pos % 26 + 97).astype(np.uint8)
    return pa.Array.from_buffers(pa.binary() if binary else pa.utf8(), len(lengths),
                                 [None, pa.py_buffer(offsets.astype(np.int32)), pa.py_buffer(data)])


def with_nulls(arr, mask):
    return pc.if_else(pa.array(mask), pa.nulls(len(arr), arr.type), arr)


def payload(n, rng, wide=False, nullable=True):
    """Payload columns: Float64 with NaN payloads / ±0.0 / ±inf, Utf8 with lengths of every residue mod 4, Binary with
    every byte value, a Boolean (wide: 10 Int64/Float64 and 6 Utf8/Binary columns besides the id)."""
    f = rng.normal(0, 1e3, n)
    k = rng.random(n) < 0.1
    f[k] = rng.choice(NAN_BITS, int(k.sum())).view(np.float64)
    cols = {"f": pa.array(f, pa.float64())}
    cols["s"] = varlen(rng.integers(0, 41, n), False, int(rng.integers(0, 99)))
    cols["b"] = varlen(rng.integers(0, 23, n), True, int(rng.integers(0, 99)))
    cols["t"] = pa.array(rng.random(n) < 0.5, pa.bool_())
    if nullable:
        cols["fn"] = pa.array(f[::-1].copy(), pa.float64(), mask=rng.random(n) < 0.2)
        cols["sn"] = with_nulls(varlen(rng.integers(0, 19, n), False, 3), rng.random(n) < 0.2)
        cols["tn"] = pa.array(rng.random(n) < 0.5, pa.bool_(), mask=rng.random(n) < 0.3)
        cols["in"] = pa.array(rng.integers(I64_MIN, I64_MAX, n, endpoint=True), pa.int64(), mask=rng.random(n) < 0.25)
    if wide:
        for j in range(9):
            cols[f"w{j}"] = pa.array(rng.integers(I64_MIN, I64_MAX, n, endpoint=True), pa.int64()) if j % 2 else \
                pa.array(rng.normal(0, 1, n), pa.float64())
        for j in range(5):
            cols[f"ws{j}"] = varlen(rng.integers(0, 30, n), j % 2 == 1, j)
    return cols


def table(keys, rng, id0=0, wide=False, nullable=True, extra=True, non_null=("id", "f", "s")):
    """id (0..n-1 + id0, non-nullable), k = keys, payload columns.  Fields in `non_null` are declared non-nullable."""
    keys = keys if isinstance(keys, pa.Array) else pa.array(keys, pa.int64())
    n = len(keys)
    cols = {"id": pa.array(np.arange(n, dtype=np.int64) + id0, pa.int64()), "k": keys}
    if extra:
        cols.update(payload(n, rng, wide, nullable))
    fields = [pa.field(name, a.type, nullable=not (name in non_null and a.null_count == 0)) for name, a in cols.items()]
    return pa.RecordBatch.from_arrays(list(cols.values()), schema=pa.schema(fields))


def normalised(rb):
    return pa.RecordBatch.from_arrays([pa.concat_arrays([c]) for c in rb.columns], schema=rb.schema)


def to_device(rb, keep_offsets=False):
    """DeviceBatch.from_arrow, plus Null-typed columns (no buffers)."""
    nulls = [i for i, f in enumerate(rb.schema) if f.type == pa.null()]
    keep = [i for i in range(rb.num_columns) if i not in nulls]
    db = DeviceBatch.from_arrow(pa.RecordBatch.from_arrays([rb.column(i) for i in keep], schema=pa.schema([rb.schema.field(i) for i in keep])),
                                keep_offsets=keep_offsets)
    if not nulls:
        return db
    cols = list(db.columns)
    for i in nulls:
        cols.insert(i, DeviceColumn(rb.schema.field(i).name, "null", rb.num_rows, None, null_count=rb.num_rows, nullable=True))
    return DeviceBatch(cols, rb.num_rows)


# ---- comparison --------------------------------------------------------------------------------------------------------
def sort_by_ids(rb, i, j):
    t = pa.table({"a": rb.column(i), "b": rb.column(j)})
    return rb.take(pc.sort_indices(t, sort_keys=[("a", "ascending"), ("b", "ascending")], null_placement="at_end"))


def compare(got, want, what, ids=None):
    assert got.schema.names == want.schema.names, (what, got.schema, want.schema)
    assert [f.type for f in got.schema] == [f.type for f in want.schema], (what, got.schema, want.schema)
    assert [f.nullable for f in got.schema] == [f.nullable for f in want.schema], (what, got.schema, want.schema)
    assert got.num_rows == want.num_rows, (what, got.num_rows, want.num_rows)
    for c in got.columns:
        c.validate(full=True)
    if ids is not None:
        got, want = sort_by_ids(got, *ids), sort_by_ids(want, *ids)
    for k, (g, w) in enumerate(zip(got.columns, want.columns)):
        g, w = pa.concat_arrays([g]), pa.concat_arrays([w])
        if w.type == pa.float64():
            assert g.is_null().equals(w.is_null()), (what, k, "validity")
            gv = pc.fill_null(g, 0.0).to_numpy(zero_copy_only=False).view(np.uint64)
            wv = pc.fill_null(w, 0.0).to_numpy(zero_copy_only=False).view(np.uint64)
            bad = np.flatnonzero(gv != wv)
            assert len(bad) == 0, (what, k, [(int(i), hex(gv[i]), hex(wv[i])) for i in bad[:5]])
        else:
            assert g.equals(w), (what, k, got.schema.names[k])


def _query(a, b, jt, on="k", alias=None):
    x, y = alias or (a, b)
    frm = f"{a} {x} " if alias else f"{a} "
    to = f"{b} {y}" if alias else b
    return f"SELECT * FROM {frm}{jt}JOIN {to} ON {x}.{on} = {y}.{on}"


JOIN_TYPES = {"inner": "", "left": "LEFT ", "right": "RIGHT "}


def check_join(timing, tables, jt="inner", slices=False, alias=None, branches=None):
    """Runs `SELECT * FROM a <jt> JOIN b ON a.k = b.k` (tables = {"a": …, "b": …}, or {"a": …} for a self-join through
    aliases) through every entry point and compares each result with the oracle.  branches = "per_row" / "staged" /
    "both": the string gathers must take that take_bytes_tile_kernel branch in some tile.  Returns the oracle's result."""
    names = list(tables)
    a, b = (names[0], names[0]) if len(names) == 1 else names
    q = _query(a, b, JOIN_TYPES[jt], alias=alias)
    L, R = tables[a], tables[b]
    want = sql_join(tables, q)
    ids = (0, L.num_columns)
    srcs = [(c, jt == "right") for c in L.columns] + [(c, jt == "left") for c in R.columns]
    for c, _ in srcs:
        c.null_count  # noqa: B018 (computed once, so the host export carries the exact count)
    p = SqlProcessor({"query": q})
    runs = [("host", lambda: p.process_tables(tables)),
            ("device", lambda: p.process_tables_device({k: to_device(v) for k, v in tables.items()}).to_arrow())]
    if slices:
        runs.append(("slices", lambda: p.process_tables_device({k: to_device(v, keep_offsets=True) for k, v in tables.items()}).to_arrow()))
    seen = [0, 0]
    for name, run in runs:
        timing.ark_kernel_timing_reset()
        got = run()
        what = (q, jt, name, {k: v.num_rows for k, v in tables.items()})
        assert got is not None, what
        compare(got, want, what, ids)
        launched = _launches(timing)
        assert launched == predict_gathers(srcs, want.num_rows), (what, launched, predict_gathers(srcs, want.num_rows))
        for k, c in enumerate(got.columns):
            if c.type in (pa.utf8(), pa.binary()):
                st, pr = tile_branches(c)
                seen[0] += st
                seen[1] += pr
    if branches in ("per_row", "both"):
        assert seen[1] > 0, (q, "no tile took the per-row branch", seen)
    if branches in ("staged", "both"):
        assert seen[0] > 0, (q, "no tile took the staged branch", seen)
    return want


def check_all_types(timing, tables, **kw):
    return [check_join(timing, tables, jt, **kw) for jt in JOIN_TYPES]


# ---- key encoding ------------------------------------------------------------------------------------------------------
def test_int64_edge_keys(timing):
    rng = np.random.default_rng(1)
    k0 = 0x1234_5678
    # pairs k / k + 2^32 (equal low words) and k / k ^ 2^63 (k - 2^63 for k >= 0: equal but for the sign bit)
    edges = [I64_MIN, I64_MIN + 1, I64_MAX, I64_MAX - 1, -1, 0, 1, k0, k0 + 2 ** 32, k0 - 2 ** 63, 7, 7 + 2 ** 32, 7 - 2 ** 63,
             -(2 ** 32), 2 ** 32, -5, -5 + 2 ** 32]
    # the probe side holds every edge; the build side holds one member of some pairs only
    lk = [edges[int(i)] if i < len(edges) else None for i in rng.integers(0, len(edges) + 2, 3000)]
    bset = [I64_MIN, I64_MAX, -1, 0, k0 + 2 ** 32, 7 - 2 ** 63, -(2 ** 32), -5 + 2 ** 32, 1, 5 + 2 ** 32]
    rk = [bset[int(i)] if i < len(bset) else None for i in rng.integers(0, len(bset) + 1, 700)]
    check_all_types(timing, {"a": table(lk, rng), "b": table(rk, rng, id0=10_000)}, slices=True)


def hash32_int64(v):
    """numpy copy of hash32_key16 (csrc/hashkey.cuh) of an Int64 key: lo = the value, hi = KEYTAG_INT << 32."""
    M = np.uint64(0xFFFFFFFF)
    u = v.astype(np.uint64)
    lo, hi = u & M, u >> np.uint64(32)

    def mul(a, c):
        return (a * np.uint64(c)) & M

    def rotl(a, r):
        return ((a << np.uint64(r)) | (a >> np.uint64(32 - r))) & M

    h = mul(lo, 0x85EBCA6B) ^ rotl(mul(hi, 0xC2B2AE35), 13) ^ np.uint64((0x40000000 * 0x165667B1) & 0xFFFFFFFF)
    h ^= h >> np.uint64(16)
    h = mul(h, 0x85EBCA6B)
    h ^= h >> np.uint64(13)
    h = mul(h, 0xC2B2AE35)
    h ^= h >> np.uint64(16)
    return h


def colliding_keys(count, target):
    """`count` distinct Int64 keys whose hash32_key16 is equal: before the final mix the hash is
    lo32 * C1 ^ rotl(hi32 * C2, 13) ^ const, and C1 is odd, so each high word gets the low word that lands on `target`."""
    C1_INV = pow(0x85EBCA6B, -1, 2 ** 32)
    const = (0x40000000 * 0x165667B1) & 0xFFFFFFFF
    out = []
    for hi in range(1, count + 1):
        hi_w = (hi * 0x9E3779B1) & 0xFFFFFFFF
        m = (hi_w * 0xC2B2AE35) & 0xFFFFFFFF
        r = ((m << 13) | (m >> 19)) & 0xFFFFFFFF
        lo = ((target ^ r ^ const) * C1_INV) & 0xFFFFFFFF
        u = (hi_w << 32) | lo
        out.append(u - 2 ** 64 if u >= 2 ** 63 else u)
    return np.array(out, np.int64)


def test_colliding_int64_keys_wrap_the_table(timing):
    """~2000 distinct keys with one table hash.  The table has max(1024, next_pow2(2 * build rows)) slots and the join
    spreads the 32-bit hash as h * 0x9E3779B1 before masking; the shared value is chosen (through the numpy copy of the
    whole hash) so that the home slot is among the table's last 16, and the probe chain wraps past its last slot.  The
    keys collide by construction of the pre-mix value alone: were the numpy copy of the final mix wrong, they would still
    collide, only the wrap-around would be lost."""
    rng = np.random.default_rng(2)
    n_build = 2100  # 2000 members, 100 of them twice
    cap = 1024
    while cap < 2 * n_build:
        cap *= 2
    best = None
    for target in range(1, 1 << 20):
        keys = colliding_keys(1, target)
        h = int(hash32_int64(keys)[0])
        slot = (h * 0x9E3779B1) & (cap - 1)
        if slot >= cap - 16:
            best = target
            break
    assert best is not None
    keys = colliding_keys(4000, best)
    h = hash32_int64(keys)
    assert (h == h[0]).all()
    members, others = keys[:2000], keys[2000:]
    bk = np.concatenate([members, members[:100]])
    rng.shuffle(bk)
    pk = np.concatenate([rng.choice(members, 3000), rng.choice(others, 2000), rng.integers(-10 ** 9, 10 ** 9, 500)])
    rng.shuffle(pk)
    pk = pa.array(pk, pa.int64(), mask=rng.random(len(pk)) < 0.05)
    a, b = table(pk, rng), table(pa.array(bk, pa.int64()), rng, id0=100_000)
    assert b.num_rows == n_build
    check_all_types(timing, {"a": a, "b": b})


def utf8_keys():
    """Lengths 0, 1, 11, 12, 13 and 4096; "a" and "a\\0"; long keys with one 4-byte prefix and one length that differ
    only in the last byte or only in byte 12; multi-byte UTF-8 (12 and 13 bytes long, and past the inline limit)."""
    base = "abcdefghijklmnopqrstuvwxyz"
    keys = ["", "a", "a\0", "\0", "b", base[:11], base[:12], base[:13], "x" * 4096, "x" * 4095 + "y", "x" * 4095 + "z"]
    for n in (13, 14, 40):
        keys += ["PREF" + base[:n - 5] + c for c in "012"]  # equal prefix and length, differ in the last byte
    keys += ["PREFabcdefgh" + c + "tail" for c in "xyz"]  # … only in byte 12
    keys += ["PREFabcdefg" + c for c in "xyz"]  # 12 bytes: inline
    keys += ["ÿé€", "ÿé€𝄞", "ß" * 6, "ß" * 6 + "a", "€" * 4, "€" * 4 + "ü", "日本語のキー" * 3, "日本語のキー" * 3 + "!"]
    return keys


def test_utf8_keys(timing):
    rng = np.random.default_rng(3)
    keys = utf8_keys()
    lk = [keys[int(i)] if i < len(keys) else None for i in rng.integers(0, len(keys) + 3, 4000)]
    sub = keys[::2] + ["a\0", "x" * 4095 + "z", "not on the left at all", "PREFabcdefghxtaiL"]
    rk = [sub[int(i)] if i < len(sub) else None for i in rng.integers(0, len(sub) + 1, 900)]
    a = table(pa.array(lk, pa.utf8()), rng)
    b = table(pa.array(rk, pa.utf8()), rng, id0=10_000)
    check_all_types(timing, {"a": a, "b": b}, slices=True)
    # families of long keys with one prefix and one length that differ only in the last byte, or only in byte 12: at
    # ~0.4 load a probe meets its siblings on the way to its own slot, and only the byte comparison tells them apart
    fam = [("PREFIXED-KEY-" + chr(33 + i)) for i in range(90)] + [("x" * 39 + chr(33 + i)) for i in range(90)] + \
          [("PREFabcdefgh" + chr(33 + i) + "tail-of-the-key") for i in range(90)]
    bk = fam[::2] + ["filler-key-%06d" % i for i in range(285)]  # 420 distinct keys in 1024 slots
    pk = [fam[int(i)] for i in rng.integers(0, len(fam), 3000)]
    check_all_types(timing, {"a": table(pa.array(pk, pa.utf8()), rng), "b": table(pa.array(bk, pa.utf8()), rng, id0=10_000)})
    # "" against NULL: neither matches a NULL, "" matches ""
    a = table(pa.array(["", None, "", None, "a"], pa.utf8()), rng)
    b = table(pa.array([None, "", None], pa.utf8()), rng, id0=100)
    out = check_all_types(timing, {"a": a, "b": b})
    assert out[0].num_rows == 2


def test_self_join_through_aliases(timing):
    """FROM a x JOIN a y: both sides are one column, so equal long keys of the same row compare by row reference."""
    rng = np.random.default_rng(4)
    keys = utf8_keys()
    k = pa.array([keys[int(i)] if i < len(keys) else None for i in rng.integers(0, len(keys) + 2, 1500)], pa.utf8())
    a = table(k, rng)
    for jt in JOIN_TYPES:
        check_join(timing, {"a": a}, jt, alias=("x", "y"))
    ik = table(pa.array(rng.integers(-50, 50, 3000), pa.int64(), mask=rng.random(3000) < 0.1), rng)
    check_join(timing, {"a": ik}, "inner", alias=("x", "y"))


# ---- shapes ------------------------------------------------------------------------------------------------------------
def test_empty_and_null_sides(timing):
    rng = np.random.default_rng(5)
    full = table(rng.integers(0, 50, 700), rng)
    empty = table(np.zeros(0, np.int64), rng, id0=10_000)
    for tables in ({"a": full, "b": empty}, {"a": empty, "b": full}, {"a": empty, "b": empty}):
        out = check_all_types(timing, tables)
        assert out[0].num_rows == 0
    nulls = table(pa.nulls(300, pa.int64()), rng, id0=10_000)
    for tables in ({"a": full, "b": nulls}, {"a": nulls, "b": full}):
        out = check_all_types(timing, tables)
        assert out[0].num_rows == 0
    far = table(rng.integers(1000, 2000, 400), rng, id0=10_000)
    out = check_all_types(timing, {"a": full, "b": far})
    assert out[0].num_rows == 0 and out[1].num_rows == 700 and out[2].num_rows == 400


def test_build_side_choice_keeps_column_order(timing):
    """Inner joins build on the smaller side (the left one when sizes are equal); the output is left columns then right
    columns either way."""
    rng = np.random.default_rng(6)
    for nl, nr in ((300, 2000), (2000, 300), (1000, 1000)):
        a = table(rng.integers(0, 200, nl), rng)
        b = table(rng.integers(100, 300, nr), rng, id0=10_000, nullable=False)
        check_all_types(timing, {"a": a, "b": b})


@pytest.mark.parametrize("nb", [511, 512, 513])
def test_build_sizes_at_table_doubling(timing, nb):
    rng = np.random.default_rng(nb)
    b = table(rng.permutation(nb).astype(np.int64) * 3, rng, id0=10_000)  # distinct keys: load factor nb / slots
    a = table(rng.integers(-10, 3 * nb + 10, 5000), rng)
    check_all_types(timing, {"a": a, "b": b})


def test_large_build_and_probe(timing):
    """2^20 distinct build keys (2 * 2^20 slots: the fullest table the sizing allows), then 2^22 probe rows against 2^20
    build rows with duplicates."""
    rng = np.random.default_rng(7)
    n = 1 << 20
    b = table(rng.permutation(n).astype(np.int64), rng, id0=1 << 30, extra=False)
    a = table(rng.integers(-1000, n + 1000, n), rng, extra=False)
    check_join(timing, {"a": a, "b": b}, "inner")
    b = table(rng.integers(0, n // 2, n), rng, id0=1 << 30, extra=False)
    b = pa.RecordBatch.from_arrays(list(b.columns) + [varlen(rng.integers(0, 20, n))], names=b.schema.names + ["s"])
    a = table(rng.integers(0, n, 1 << 22), rng, extra=False)
    check_join(timing, {"a": a, "b": b}, "inner")


def test_skewed_key(timing):
    """One key with 5000 build rows against 4000 probe rows: 2 * 10^7 pairs from 5000-long next[] chains."""
    rng = np.random.default_rng(8)
    b = table(np.concatenate([np.full(5000, 42), rng.integers(0, 1000, 500)]), rng, id0=1 << 20, extra=False)
    a = table(np.concatenate([np.full(4000, 42), rng.integers(500, 1500, 500)]), rng, extra=False)
    out = check_join(timing, {"a": a, "b": b}, "inner")
    assert out.num_rows >= 2 * 10 ** 7


def test_pair_limit_is_unsupported(gpu):
    """65 536 x 32 768 equal keys make exactly 2^31 pairs: an Unsupported error, not a crash."""
    a = pa.record_batch({"k": pa.array(np.full(65536, 5), pa.int64())})
    b = pa.record_batch({"k": pa.array(np.full(32768, 5), pa.int64()), "y": pa.array(np.arange(32768), pa.int64())})
    p = SqlProcessor({"query": "SELECT * FROM a JOIN b ON a.k = b.k"})
    for run in (lambda: p.process_tables({"a": a, "b": b}),
                lambda: p.process_tables_device({"a": DeviceBatch.from_arrow(a), "b": DeviceBatch.from_arrow(b)})):
        with pytest.raises(ArkError) as e:
            run()
        assert e.value.kind == "Unsupported" and "2^31" in e.value.message, e.value.message


# ---- gathers -----------------------------------------------------------------------------------------------------------
def test_wide_select_star(timing):
    """10 Int64/Float64 and 6 Utf8/Binary plain columns a side, plus nullable ones: take_multi_kernel is full (8 + 4) and
    the rest take take_column."""
    rng = np.random.default_rng(9)
    a = table(rng.integers(0, 300, 3000), rng, wide=True)
    b = table(rng.integers(100, 400, 2000), rng, id0=10_000, wide=True)
    check_all_types(timing, {"a": a, "b": b}, slices=True)


@pytest.mark.parametrize("off", range(1, 8))
def test_sliced_boolean_and_validity_bits(timing, off):
    """Booleans and validity bitmaps sliced at bit offsets 1 to 7 (host slices and device slices)."""
    rng = np.random.default_rng(10 + off)
    a = table(rng.integers(0, 100, 2000 + off), rng)
    b = table(rng.integers(50, 150, 900 + off), rng, id0=10_000)
    check_all_types(timing, {"a": a.slice(off, 2000 - off), "b": b.slice(off, 900)}, slices=True)


def test_null_typed_columns_are_unsupported(gpu):
    """A Null-typed column on either side cannot be gathered: the join says so (Unsupported) on both entry points, and a
    projection that leaves it out still matches the oracle."""
    rng = np.random.default_rng(11)
    a = pa.record_batch({"id": pa.array(np.arange(500), pa.int64()), "k": pa.array(rng.integers(0, 40, 500), pa.int64()), "z": pa.nulls(500)})
    b = pa.record_batch({"id": pa.array(np.arange(80) + 1000, pa.int64()), "k": pa.array(rng.integers(0, 40, 80), pa.int64()), "z": pa.nulls(80)})
    for jt in JOIN_TYPES.values():
        q = f"SELECT * FROM a {jt}JOIN b ON a.k = b.k"
        p = SqlProcessor({"query": q})
        for run in (lambda: p.process_tables({"a": a, "b": b}), lambda: p.process_tables_device({"a": to_device(a), "b": to_device(b)})):
            with pytest.raises(ArkError) as e:
                run()
            assert e.value.kind == "Unsupported" and "'n'" in e.value.message, e.value.message
        q = f"SELECT a.id, b.id AS bid, a.k, b.k AS bk FROM a {jt}JOIN b ON a.k = b.k"
        want = sql_join({"a": a, "b": b}, q)
        got = SqlProcessor({"query": q}).process_tables_device({"a": to_device(a), "b": to_device(b)}).to_arrow()
        compare(got, want, q, ids=(0, 1))


def test_string_tiles_take_both_branches(timing):
    """Short strings with a run of 300-byte ones: the staging buffer is sized to the average row, so the tiles of the
    run are copied row by row, the others are staged; on the plain path and through take_column (outer-join misses)."""
    rng = np.random.default_rng(12)
    n = 60_000
    lens = rng.integers(0, 13, n)
    lens[20_000:26_000] = 300
    a = pa.record_batch({"id": pa.array(np.arange(n), pa.int64()), "k": pa.array(np.arange(n), pa.int64()),
                         "s": varlen(lens), "b": varlen(lens[::-1].copy(), True)})
    b = pa.record_batch({"id": pa.array(np.arange(n) + n, pa.int64()), "k": pa.array(np.arange(n), pa.int64()),
                         "s": varlen(lens, salt=5)})
    for jt in JOIN_TYPES:
        check_join(timing, {"a": a, "b": b}, jt, slices=True, branches="both")


def test_every_byte_value_in_binary_columns(timing):
    rng = np.random.default_rng(13)
    n = 4096
    vals = [bytes([(i + j) % 256 for j in range(i % 37)]) for i in range(n)]
    a = pa.record_batch({"id": pa.array(np.arange(n), pa.int64()), "k": pa.array(np.arange(n) % 300, pa.int64()), "x": pa.array(vals, pa.binary())})
    b = pa.record_batch({"id": pa.array(np.arange(500) + n, pa.int64()), "k": pa.array(rng.integers(0, 400, 500), pa.int64()),
                         "y": pa.array([bytes(range(256))[i % 256:] for i in range(500)], pa.binary())})
    check_all_types(timing, {"a": a, "b": b}, slices=True)


# ---- the 2 GiB output guard --------------------------------------------------------------------------------------------
GUARD_SQL = {"plain": "SELECT * FROM p JOIN b ON p.pk = b.bk", "nullable": "SELECT * FROM p JOIN b ON p.pk = b.bk",
             "left": "SELECT * FROM p LEFT JOIN b ON p.pk = b.bk"}


def _guard_tables(case, variant):
    """b holds the long strings (key 1, and key 2 for the exact case), p repeats their keys.  The total of the gathered
    string column: 'exact' 1023 * 2^21 + (2^21 - 1) = 2^31 - 1 (one 1024-row tile), 'pow31' 1024 * 2^21 = 2^31,
    'mid' 1500 * 2^21, 'wrap' 4200 * 2^20 = 4 404 019 200, which an int32 wraps to +109 051 904 (b has 4096 rows, 4095 of
    them empty, so the source's average string is 256 bytes)."""
    if case == "wrap":
        lens = np.zeros(4096, np.int64)
        lens[0] = 1 << 20
        bk = np.arange(1, 4097)
        pk = np.ones(4200, np.int64)
    else:
        lens = np.array([1 << 21, (1 << 21) - 1, 0], np.int64)
        bk = np.array([1, 2, 3])
        reps = {"exact": 1023, "pow31": 1024, "mid": 1500}[case]
        pk = np.array([1] * reps + ([2] if case == "exact" else []), np.int64)
    s = varlen(lens, salt=7)
    if variant == "nullable":
        s = with_nulls(s, np.arange(len(lens)) == len(lens) - 1)  # the last row is NULL and matches nothing
    b = pa.record_batch({"bid": pa.array(np.arange(len(bk)), pa.int64()), "bk": pa.array(bk, pa.int64()), "s": s})
    p = pa.record_batch({"pid": pa.array(np.arange(len(pk)), pa.int64()), "pk": pa.array(pk, pa.int64())})
    return p, b, lens


@pytest.mark.parametrize("variant", ["plain", "nullable", "left"])
def test_output_of_2gib_minus_one_bytes(timing, variant):
    """2^31 - 1 output bytes fit the int32 offsets: offsets and bytes checked against numpy (one download)."""
    p, b, lens = _guard_tables("exact", variant)
    proc = SqlProcessor({"query": GUARD_SQL[variant]})
    timing.ark_kernel_timing_reset()
    out = proc.process_tables_device({"p": DeviceBatch.from_arrow(p), "b": DeviceBatch.from_arrow(b)})
    launched = _launches(timing)
    srcs = [(c, False) for c in p.columns] + [(c, variant == "left") for c in b.columns]
    assert launched == predict_gathers(srcs, 1024), launched
    assert launched["take_lengths_kernel"] == (variant != "plain"), launched  # the string column takes take_column
    cols = {c.name: c for c in out.columns}
    assert out.num_rows == 1024
    bid = cols["bid"].data.cpu().numpy()
    offs = cols["s"].offsets.cpu().numpy().astype(np.int64)
    want_offs = np.concatenate([[0], np.cumsum(lens[bid])])
    assert offs[-1] == 2 ** 31 - 1 and np.array_equal(offs, want_offs)
    assert cols["s"].validity is None or bool((cols["s"].validity.cpu().numpy()[:128] == 255).all())
    data = cols["s"].data.cpu().numpy()
    src = np.frombuffer(b.column("s").buffers()[2], np.uint8)
    src_off = np.frombuffer(b.column("s").buffers()[1], np.int32)
    for r in range(len(bid)):
        k = int(bid[r])
        assert np.array_equal(data[offs[r]:offs[r + 1]], src[src_off[k]:src_off[k + 1]]), r
    del data
    out.close()


@pytest.mark.parametrize("case", ["pow31", "mid", "wrap"])
@pytest.mark.parametrize("variant", ["plain", "nullable", "left"])
def test_output_past_2gib_is_a_process_error(gpu, case, variant):
    p, b, lens = _guard_tables(case, variant)
    total = int(lens[0]) * p.num_rows
    assert total > 2 ** 31 - 1
    if case == "wrap":
        assert 2 ** 32 < total < 2 ** 32 + 2 ** 31 and 0 < (total % 2 ** 32) < 2 ** 31
    proc = SqlProcessor({"query": GUARD_SQL[variant]})
    for run in (lambda: proc.process_tables({"p": p, "b": b}),
                lambda: proc.process_tables_device({"p": DeviceBatch.from_arrow(p), "b": DeviceBatch.from_arrow(b)})):
        with pytest.raises(ArkError) as e:
            run()
        assert e.value.kind == "Process" and "offset overflow" in e.value.message, e.value.message


def test_concat_past_2gib_is_a_process_error(gpu):
    """concat(s, <64 KiB literal>) over 70 000 rows: 70 000 * (65 536 + |s|) bytes, past 2^32, an int32 total that wraps
    back to a positive value."""
    n = 70_000
    rb = pa.record_batch({"s": pa.array(["r%d" % i for i in range(n)])})
    total = n * 65536 + sum(len("r%d" % i) for i in range(n))
    assert 2 ** 32 < total and 0 < total % 2 ** 32 < 2 ** 31
    proc = SqlProcessor({"query": "SELECT concat(s, '" + "L" * 65536 + "') AS c FROM flow"})
    with pytest.raises(ArkError) as e:
        proc.process(rb)
    assert e.value.kind == "Process" and "offset overflow" in e.value.message, e.value.message


# ---- hash repartition --------------------------------------------------------------------------------------------------
def part_table(kind, n, rng, wide=False):
    if kind == "int64":
        k = pa.array(rng.choice(np.array([I64_MIN, I64_MAX, -1, 0, 1, 2 ** 32, -(2 ** 32)]), n) if n else np.zeros(0, np.int64), pa.int64())
        k = pc.if_else(pa.array(rng.random(n) < 0.5), pa.array(rng.integers(-10 ** 6, 10 ** 6, n), pa.int64()), k)
    elif kind == "bool":
        k = pa.array(rng.random(n) < 0.5, pa.bool_())
    else:
        keys = utf8_keys() + ["k%d" % i for i in range(300)]
        k = pa.array([keys[int(i)] for i in rng.integers(0, len(keys), n)], pa.utf8())
        if kind == "binary":
            k = k.cast(pa.binary())
    k = with_nulls(k, rng.random(n) < 0.05)
    return table(k, rng, wide=wide)


def check_partition(timing, rb, n_parts, owners, keep_offsets=False):
    """One hash_partition call: the output is a permutation of rb with the same schema, counts sum to n, each key lies in
    one partition, and that partition is the one `owners` saw for the key before (other batches, slices, row orders)."""
    for c in rb.columns:
        c.null_count  # noqa: B018
    eng = NativeEngine("SELECT * FROM flow")
    timing.ark_kernel_timing_reset()
    out, counts = eng.hash_partition(to_device(rb, keep_offsets), "k", n_parts)
    launched = _launches(timing)
    got = out.to_arrow()
    what = (rb.num_rows, n_parts, rb.schema.field("k").type, keep_offsets)
    assert len(counts) == n_parts and sum(counts) == rb.num_rows and min(counts) >= 0, (what, counts)
    assert launched == predict_gathers([(c, False) for c in rb.columns], rb.num_rows), (what, launched)
    compare(got, normalised(rb), what + ("permutation",), ids=(0, 0))
    part = np.repeat(np.arange(n_parts), counts)
    keys = got.column("k")
    for key, p in zip(keys.to_pylist(), part.tolist()):
        assert owners.setdefault(key, p) == p, (what, key, owners[key], p)
    return got


@pytest.mark.parametrize("kind", ["int64", "bool", "utf8", "binary"])
def test_partition_edges(timing, kind):
    rng = np.random.default_rng(20)
    for n_parts in (1, 2, 3, 31, 32):
        owners = {}
        for n in (0, 1, 2047, 2048, 2049):
            check_partition(timing, part_table(kind, n, rng), n_parts, owners)
        # the same keys in other compositions: another batch, reversed, a device slice at a bit offset
        rb = part_table(kind, 5003, rng)
        check_partition(timing, rb, n_parts, owners)
        check_partition(timing, rb.take(pa.array(np.arange(rb.num_rows)[::-1].copy())), n_parts, owners)
        check_partition(timing, rb.slice(3, 4000), n_parts, owners, keep_offsets=True)
        check_partition(timing, rb.slice(13, 2049), n_parts, owners)
        if n_parts == 1:
            assert set(owners.values()) <= {0}


def test_partition_wide_schema_and_large_batch(timing):
    rng = np.random.default_rng(21)
    owners = {}
    for n_parts in (3, 32):
        check_partition(timing, part_table("utf8", 4099, rng, wide=True), n_parts, owners if n_parts == 32 else {})
    rb = part_table("int64", (1 << 22) + 5, rng)
    eng = NativeEngine("SELECT * FROM flow")
    out, counts = eng.hash_partition(to_device(rb), "k", 32)
    got = out.to_arrow()
    assert sum(counts) == rb.num_rows
    compare(got, rb, "large partition", ids=(0, 0))
    t = pa.table({"k": got.column("k"), "p": pa.array(np.repeat(np.arange(32), counts))})
    per_key = t.group_by("k").aggregate([("p", "count_distinct")])
    assert pc.max(per_key.column("p_count_distinct")).as_py() == 1


@pytest.mark.parametrize("n_parts", [0, 33])
def test_partition_count_out_of_range(gpu, n_parts):
    rb = part_table("int64", 100, np.random.default_rng(22))
    with pytest.raises(ArkError):
        NativeEngine("SELECT * FROM flow").hash_partition(DeviceBatch.from_arrow(rb), "k", n_parts)
