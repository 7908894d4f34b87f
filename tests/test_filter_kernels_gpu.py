"""Every filter + project kernel against the oracle (oracle/sql_oracle.py), at the shapes and values where kernels go wrong.

The fast path `SELECT <≤ 2 Int64/Float64 columns> [, <one Utf8/Binary column>] WHERE <col> <cmp> <literal>` has several
kernels, each with its own copy of the predicate, ranking, look-back and string staging (DESIGN.md §4.1): the default
tile kernel (filter_project_tile_kernel), the persistent ring kernel (ARK_FP_IMPL=3), the persistent pipelined kernel
(ARK_FP_IMPL=0) and the round-1 kernel (ARK_FP_IMPL=1); every other query runs the general filter_project_kernel<PRED, NV>.
The knobs that pick a kernel are read once per process, so each path runs in a child process: this process builds the
inputs and the oracle's answers, the child runs the library and writes its results as Arrow IPC together with the kernels
each call launched.  Every case asserts that the intended kernel ran, or that the path declines the case by design (the
ring kernel's (NF, NFX) set and shared-memory budget, 512-row tiles without a string output): a silent fallback fails.

Survival is decided by construction: the predicate column holds values on the right side of the literal exactly where a
selection pattern says so (all, none, alternating, one row per tile, runs of empty and full tiles and groups of 32
tiles, random at σ = 0.01 / 0.5 / 0.99).  Comparison: schema names and types equal the oracle's, every non-float column
passes Array.equals, Float64 columns are compared through their uint64 view (NaN payloads and -0.0 bit for bit).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
TILE, RING, PIPE, R1, GENERAL = ("filter_project_tile_kernel", "filter_project_ring_kernel", "filter_project_pipe_kernel",
                                 "filter_project_r1_kernel", "filter_project_kernel")
FAST = (TILE, RING, PIPE, R1)
KERNELS = ("filter_project_tma_kernel",) + FAST + (GENERAL,)
NAN_BITS = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFF0000000000001, 0x7FFFFFFFFFFFFFFF,
                     0xFFFFFFFFFFFFFFFF, 0x7FF4000000000123, 0xFFF400000000ABCD], dtype=np.uint64)

PATHS = {  # name → (environment, kernel it selects, rows per tile)
    "default": ({}, TILE, 1024),
    "tiles2048": ({"ARK_FP_THREADS": "512"}, TILE, 2048),
    "ticket": ({"ARK_FP_TICKET": "1"}, TILE, 1024),
    "lb_chain": ({"ARK_FP_LB": "1"}, TILE, 1024),
    "lb_narrow": ({"ARK_FP_LB_WINDOWS": "1"}, TILE, 1024),
    "maxr32": ({"ARK_FP_MAXR": "32"}, TILE, 1024),
    "maxr56": ({"ARK_FP_MAXR": "56"}, TILE, 1024),
    "desc_dense": ({"ARK_FP_DESC_STRIDE": "1"}, TILE, 1024),
    "small_staging": ({"ARK_FP_CAP_SLACK": "0.25"}, TILE, 1024),
    "helping": ({"ARK_FP_DEBUG": "4"}, TILE, 1024),
    "helping_narrow": ({"ARK_FP_DEBUG": "4", "ARK_FP_LB_WINDOWS": "1"}, TILE, 1024),
    "ring": ({"ARK_FP_IMPL": "3"}, RING, 1024),
    "ring512": ({"ARK_FP_IMPL": "3", "ARK_FP_THREADS": "128"}, RING, 512),
    "pipe_minb3": ({"ARK_FP_IMPL": "0", "ARK_FP_MINB": "3"}, PIPE, 1024),
    "pipe_minb4": ({"ARK_FP_IMPL": "0", "ARK_FP_MINB": "4"}, PIPE, 1024),
    "pipe_minb5": ({"ARK_FP_IMPL": "0", "ARK_FP_MINB": "5"}, PIPE, 1024),
    "r1_256": ({"ARK_FP_IMPL": "1"}, R1, 1024),
    "r1_512": ({"ARK_FP_IMPL": "1", "ARK_FP_THREADS": "512"}, R1, 2048),
}


# ---- staging size and ring budget, as launch_filter_project_tma computes them (csrc/filter_project_tma.cu) -------------
def str_cap(avg_len, tt, slack=1.0625):
    """Shared-memory bytes per string buffer: `cap = round_up((int64_t)(avg * TT * slack) + 64, 1024)`, clamped to
    [4096 (2048 for 512-row tiles), 24 KB per 1024 rows]; avg = referenced string bytes / rows of the batch."""
    cap = -(-(int(avg_len * tt * slack) + 64) // 1024) * 1024
    return max(4096 if tt >= 1024 else 2048, min(cap, max(tt // 1024, 1) * 24 * 1024))


def ring_takes(nf, nfx, cap, tt):
    """The ring kernel exists for (NF, NFX) ∈ {(0,0), (1,0), (1,1), (2,1)} and runs when two input and two output stages
    fit in 112 KB of shared memory."""
    if (nf, nfx) not in ((0, 0), (1, 0), (1, 1), (2, 1)):
        return False
    pred = tt * 8 + 32
    offs = ((tt + 1) * 4 + 32 + 15) // 16 * 16
    smem = 2 * (pred + offs + nfx * pred + cap + 32) + 2 * (nf * tt * 8 + tt * 4 + 16 + cap + 32)
    return smem <= 112 * 1024


# ---- inputs -----------------------------------------------------------------------------------------------------------
def _varlen(lengths, binary, salt=0):
    """Strings of the given lengths: ASCII letters (Utf8) or every byte value, NUL included (Binary)."""
    offsets = np.zeros(len(lengths) + 1, np.int64)
    np.cumsum(lengths, out=offsets[1:])
    assert offsets[-1] < 2 ** 31
    pos = np.arange(offsets[-1], dtype=np.int64) * 131 + salt
    data = (pos % 256 if binary else pos % 26 + 97).astype(np.uint8)
    t = pa.binary() if binary else pa.utf8()
    return pa.Array.from_buffers(t, len(lengths), [None, pa.py_buffer(offsets.astype(np.int32)), pa.py_buffer(data)])


def _lengths(kind, n, rng):
    if kind == "fixed":  # the benchmark's "temp_%07d": every warp takes the equal-length branch
        return np.full(n, 12, np.int64)
    if kind == "empty":  # zero string bytes: no bulk copy at all
        return np.zeros(n, np.int64)
    lens = rng.integers(0, 41, n)
    if kind == "long":  # a region of 300-byte strings: their tiles overflow the staging buffer
        lo = n // 3
        lens[lo:lo + max(1, min(n // 4, 20_000))] = 300
    return lens


def selection(pattern, n, tt, rng):
    r = np.arange(n)
    if pattern == "all":
        return np.ones(n, bool)
    if pattern == "none":
        return np.zeros(n, bool)
    if pattern == "alt":
        return r % 2 == 0
    if pattern == "first":  # a single survivor on row 0 of each tile
        return r % tt == 0
    if pattern == "last":  # … on the last row of each tile, and on the last row of the batch
        return (r % tt == tt - 1) | (r == n - 1)
    if pattern == "tiles":  # runs of three empty tiles, then three full tiles
        return (r // tt) // 3 % 2 == 1
    if pattern == "groups":  # whole groups of 32 tiles with no survivor, then full groups
        return (r // (32 * tt)) % 2 == 1
    if pattern == "groups64k":  # the same at 65 536 rows (32 tiles of 2048 rows), shared by every tile size
        return (r // 65536) % 2 == 1
    return rng.random(n) < float(pattern[1:])  # "s0.5"


def make_table(n, pattern="s0.5", tt=1024, strings="mixed", seed=0, binary=True):
    """`value` (Int64) ≥ 10 and `fv` (Float64) ≥ 0.5 exactly on the selected rows.  `fv` puts +NaN and +inf among the
    survivors and -NaN, -inf, ±0.0 among the others; `x` and `timestamp` are passed through: random bits (NaN payloads,
    subnormals) and the full Int64 range."""
    rng = np.random.default_rng(seed)
    m = selection(pattern, n, tt, rng)
    value = np.where(m, rng.integers(10, 2 ** 40, n), rng.integers(-2 ** 40, 10, n))
    fv = np.where(m, rng.uniform(0.5, 1e6, n), rng.uniform(-1e6, 0.5, n))
    k = rng.random(n) < 0.02
    fv[k & m] = rng.choice(np.array([np.nan, np.inf, 0.5]), int((k & m).sum()))
    lo = rng.choice(np.array([0x7FF8000000000000 ^ (1 << 63), 0xFFF0000000000000, 0x8000000000000000, 0, 0x3FDFFFFFFFFFFFFF],
                             np.uint64), int((k & ~m).sum())).view(np.float64)  # -NaN, -inf, -0.0, 0.0, 0.5 - ulp
    fv[k & ~m] = lo
    cols = {"value": pa.array(value, pa.int64()), "fv": pa.array(fv, pa.float64())}
    cols["timestamp"] = pa.array(rng.integers(I64_MIN, I64_MAX, n, endpoint=True), pa.int64())
    x = rng.integers(0, 2 ** 64, n, dtype=np.uint64)
    k = rng.random(n) < 0.05
    x[k] = rng.choice(np.concatenate([NAN_BITS, np.array([0x8000000000000000, 1, 0x8000000000000001], np.uint64)]), int(k.sum()))
    cols["x"] = pa.array(x.view(np.float64), pa.float64())
    lens = _lengths(strings, n, rng)
    cols["sensor"] = _varlen(lens, False, seed)
    if binary:
        cols["bsensor"] = _varlen(lens, True, seed)
    return pa.record_batch(cols)


def window_table(tt=1024):
    """Tiles of 12-byte strings, except one tile whose string bytes are exactly str_cap and one with str_cap + 16; every
    tile's bytes are a multiple of 16, so a tile's 16-byte-aligned window is its own bytes.  The first is staged through
    shared memory and fills it to the last byte, the second takes the unstaged path."""
    n_tiles = 30
    cap = str_cap(12, tt)
    for _ in range(10):  # the average length depends on the two wide tiles: iterate to the fixed point
        lens = np.full(n_tiles * tt, 12, np.int64)
        for t, extra in ((7, 0), (19, 16)):
            total = cap + extra
            lens[t * tt:(t + 1) * tt] = total // tt
            lens[t * tt:t * tt + total % tt] += 1
        new = str_cap(lens.sum() / len(lens), tt)
        if new == cap:
            break
        cap = new
    assert str_cap(lens.sum() / len(lens), tt) == cap and (12 * tt) % 16 == 0 and cap % 16 == 0
    rng = np.random.default_rng(77)
    n = len(lens)
    m = rng.random(n) < 0.9
    return pa.record_batch({"value": pa.array(np.where(m, 10 + np.arange(n), -np.arange(n)), pa.int64()),
                            "timestamp": pa.array(np.arange(n) * 3, pa.int64()), "sensor": _varlen(lens, False, 5),
                            "bsensor": _varlen(lens, True, 5)})


EDGE_I = np.array([I64_MIN, I64_MIN + 1, -1, 0, I64_MAX - 1, I64_MAX], np.int64)
EDGE_F = np.concatenate([NAN_BITS, np.array([0x7FF0000000000000, 0xFFF0000000000000, 0, 1 << 63, 1, (1 << 63) | 1],
                                            np.uint64), np.array([1e300, -1e300, -2.5, 2.5, 2.0 ** 53, 2.0 ** 53 + 2,
                                                                  2.0 ** 63, -2.0 ** 63]).view(np.uint64)])


def edge_table(n=5003, seed=21):
    """Int64 and Float64 columns where every row is an edge value or next to one."""
    rng = np.random.default_rng(seed)
    i = rng.choice(EDGE_I, n)
    k = rng.random(n) < 0.3
    i[k] = rng.integers(I64_MIN, I64_MAX, int(k.sum()), endpoint=True)
    f = rng.choice(EDGE_F, n)
    k = rng.random(n) < 0.3
    f[k] = rng.normal(0, 10, int(k.sum())).view(np.uint64)
    return pa.record_batch({"i": pa.array(i, pa.int64()), "f": pa.array(f.view(np.float64), pa.float64()),
                            "sensor": _varlen(rng.integers(0, 41, n), False, seed)})


def general_table(n, seed=31, long=False):
    """Nullable columns of every projected type (validity and Boolean bits are sliced at bit offsets by the cases)."""
    rng = np.random.default_rng(seed)
    m = rng.random(n) < 0.5
    cols = {
        "value": pa.array(np.where(m, rng.integers(10, 1000, n), rng.integers(-1000, 10, n)), pa.int64(), mask=rng.random(n) < 0.1),
        "fv": pa.array(rng.uniform(-100, 100, n), pa.float64(), mask=rng.random(n) < 0.1),
        "i": pa.array(rng.integers(-2 ** 40, 2 ** 40, n), pa.int64(), mask=rng.random(n) < 0.2),
        "t": pa.array(rng.random(n) < 0.5, pa.bool_(), mask=rng.random(n) < 0.2),
    }
    xb = rng.integers(0, 2 ** 64, n, dtype=np.uint64)
    k = rng.random(n) < 0.05
    xb[k] = rng.choice(NAN_BITS, int(k.sum()))
    cols["x"] = pa.array(xb.view(np.float64), pa.float64(), mask=rng.random(n) < 0.2)
    lens = _lengths("long" if long else "mixed", n, rng)
    s = _varlen(lens, False, seed)
    # b's strings are s's plus 0-8 bytes: every tile's bytes differ between the two var-len outputs of one launch
    cols["s"] = pa.Array.from_buffers(pa.utf8(), n, [pa.array(rng.random(n) >= 0.2).buffers()[1]] + s.buffers()[1:],
                                      null_count=-1)
    b = _varlen(lens + rng.integers(0, 9, n), True, seed + 1)
    cols["b"] = pa.Array.from_buffers(pa.binary(), n, [pa.array(rng.random(n) >= 0.3).buffers()[1]] + b.buffers()[1:],
                                      null_count=-1)
    cols["s2"] = _varlen(rng.integers(0, 41, n), False, seed + 2)
    return pa.record_batch(cols)


# ---- cases ------------------------------------------------------------------------------------------------------------
# (name, query, NF, NFX, string output)
W, WF = " WHERE value >= 10", " WHERE fv >= 0.5"
SHAPES = [
    ("nf1_pred", "SELECT sensor, value FROM flow" + W, 1, 0, True),
    ("nf2", "SELECT timestamp, value, sensor FROM flow" + W, 2, 1, True),
    ("nf1_other", "SELECT sensor, timestamp FROM flow" + W, 1, 1, True),
    ("nf0", "SELECT sensor FROM flow" + W, 0, 0, True),
    ("nf2_dup", "SELECT value, value AS v2, sensor FROM flow" + W, 2, 0, True),
    ("nfx2", "SELECT timestamp, x, sensor FROM flow" + W, 2, 2, True),
    ("fixed_i", "SELECT timestamp, value FROM flow" + W, 2, 1, False),
    ("fixed_f", "SELECT x, fv FROM flow" + WF, 2, 1, False),
    ("str_f", "SELECT sensor, fv FROM flow" + WF, 1, 0, True),
    ("bin_nf1", "SELECT bsensor, value FROM flow" + W, 1, 0, True),
    ("bin_nf2", "SELECT timestamp, value, bsensor FROM flow" + W, 2, 1, True),
    ("bin_nf0", "SELECT bsensor FROM flow" + W, 0, 0, True),
    ("bin_nfx2", "SELECT timestamp, x, bsensor FROM flow" + W, 2, 2, True),
    ("lit_left", "SELECT sensor, value FROM flow WHERE 10 <= value", 1, 0, True),
]
SHAPE = {s[0]: s for s in SHAPES}
PATTERNS = ["all", "none", "alt", "first", "last", "tiles", "groups", "s0.01", "s0.5", "s0.99"]
TINY_PATTERNS = ["all", "none", "alt", "last", "s0.5"]
BIG = (1 << 22) + 3
OPS = ["=", "!=", "<", "<=", ">", ">="]
I_LITS = ["9223372036854775807", "-9223372036854775807"]
F_LITS = ["-0.0", "0.0", "-2.5", "1e309", "-1e309", "5e-324"]
IF_LITS = ["9007199254740993", "9223372036854775807"]  # Int64 literals against Float64: rounded to the nearest double


def _sizes(tt):
    return [1, 31, 32, 33] + [tt - 1, tt, tt + 1, 32 * tt - 1, 32 * tt, 32 * tt + 1]


def _table_spec(name):
    """Parses the table names the cases use into make_table arguments."""
    kind, *rest = name.split(":")
    if kind == "p":  # p:<tt>:<n>:<pattern>
        tt, n, pattern = int(rest[0]), int(rest[1]), rest[2]
        strings = ("mixed", "fixed")[(PATTERNS.index(pattern) + n) % 2]
        return dict(fn="make", n=n, pattern=pattern, tt=tt, strings=strings, seed=n * 31 + PATTERNS.index(pattern))
    if kind == "big":  # big:<pattern>
        return dict(fn="make", n=BIG, pattern=rest[0], tt=1024, strings="fixed", seed=5, binary=False)
    if kind == "huge":  # huge:<pattern>: 2^24 + 1 rows
        return dict(fn="make", n=(1 << 24) + 1, pattern=rest[0], tt=1024, strings="fixed", seed=6, binary=False)
    if kind == "str":  # str:<strings>
        return dict(fn="make", n=3 * 1024 * 4 + 17, pattern="s0.5", tt=1024, strings=rest[0], seed=11)
    if kind == "slices":
        return dict(fn="make", n=60_000 + 1237, pattern="s0.5", tt=1024, strings="mixed", seed=13)
    if kind == "window":
        return dict(fn="window", tt=int(rest[0]))
    if kind == "edge":
        return dict(fn="edge")
    if kind == "gen":  # gen:<n>[:long]
        return dict(fn="general", n=int(rest[0]), long=len(rest) > 1)
    raise ValueError(name)


def _case(cases, path, table, query, nf=None, nfx=None, v=None, off=None, device=False, general=False):
    cases.append(dict(id=f"{path}-{len(cases)}", table=table, query=query, nf=nf, nfx=nfx, v=v, off=off, device=device,
                      general=general))


def _fast_cases(path):
    _, _, tt = PATHS[path]
    cases = []
    for n in _sizes(tt):
        for pattern in (TINY_PATTERNS if n < 64 else PATTERNS):
            for name, q, nf, nfx, v in SHAPES:
                _case(cases, path, f"p:{tt}:{n}:{pattern}", q, nf, nfx, v)
    for pattern in ("all", "groups64k", "s0.5"):  # 2^22 + 3 rows: a few shapes
        for name in ("nf1_pred", "nf2", "fixed_f"):
            _, q, nf, nfx, v = SHAPE[name]
            _case(cases, path, f"big:{pattern}", q, nf, nfx, v)
    for op in OPS:  # predicate edges
        for lit in I_LITS:
            _case(cases, path, "edge", f"SELECT sensor, i FROM flow WHERE i {op} {lit}", 1, 0, True)
        for lit in F_LITS + IF_LITS:
            _case(cases, path, "edge", f"SELECT sensor, f FROM flow WHERE f {op} {lit}", 1, 0, True)
        _case(cases, path, "edge", f"SELECT i, f FROM flow WHERE f {op} -2.5", 2, 1, False)
    for strings in ("empty", "mixed", "long"):  # string edges
        for name in ("nf1_pred", "nf2", "nf0", "bin_nfx2"):
            _, q, nf, nfx, v = SHAPE[name]
            _case(cases, path, f"str:{strings}", q, nf, nfx, v)
    if tt == 1024:
        for name in ("nf1_pred", "nf0", "bin_nf2"):
            _, q, nf, nfx, v = SHAPE[name]
            _case(cases, path, "window:1024", q, nf, nfx, v)
    if path in ("default", "ring", "pipe_minb4"):  # device slices: unaligned data pointers, offsets[0] != 0
        for off in (1, 3, 7, 1237):
            for name in ("nf1_pred", "nf2", "nf0", "nfx2", "str_f"):
                _, q, nf, nfx, v = SHAPE[name]
                _case(cases, path, "slices", q, nf, nfx, v, off=off, device=True)
    return cases


def _general_cases():
    cases = []
    queries = [
        "SELECT s, value FROM flow WHERE value >= 10",  # nullable predicate column: PRED=1 with validity
        "SELECT fv, x FROM flow WHERE fv < 12.5",
        "SELECT i, x, t, s, b FROM flow WHERE value >= 10 AND fv < 50.0",  # VM predicate
        "SELECT s FROM flow WHERE value > 0 OR t",
        "SELECT value + 1 AS a, fv * 2.0 AS b2, value > 100 AS c, x FROM flow WHERE value >= 10",  # computed outputs
        "SELECT s, b FROM flow WHERE value >= 10",  # two var-len outputs
        "SELECT s, b FROM flow WHERE value < 10 AND i > 0",
        # 13 outputs, 4 computed, 3 var-len: several launches
        "SELECT value, fv, i, t, x, s, b, s2, value + 1 AS c1, value * 2 AS c2, fv + 1.0 AS c3, i - 3 AS c4, s AS s3 FROM flow WHERE value >= 10",
    ]
    for n in (2047, 2048, 2049):
        for q in queries:
            for off in (None, 3):
                _case(cases, "general", f"gen:{n}", q, off=off, general=True)
                _case(cases, "general", f"gen:{n}", q, off=off, device=True, general=True)
    for q in (queries[0], queries[2], queries[5], queries[7]):
        _case(cases, "general", f"gen:{BIG}", q, general=True)
    for q in (queries[5], queries[7]):  # 300-byte strings: tiles beyond the shared-memory staging of both outputs
        _case(cases, "general", f"gen:{1 << 17}:long", q, general=True)
        _case(cases, "general", f"gen:{1 << 17}:long", q, off=5, device=True, general=True)
    return cases


def _limit_cases(counts):
    cases = []
    for fast, table, q in ((True, "p:1024:33792:s0.5", "SELECT sensor, value FROM flow WHERE value >= 10"),
                           (True, "p:1024:33792:s0.5", "SELECT timestamp, value FROM flow WHERE value >= 10"),
                           (False, "gen:2049", "SELECT s, b, value FROM flow WHERE value >= 10")):
        c = counts[(table, q)]
        for k in sorted({0, 1, max(c - 1, 0), c, c + 1}):
            if fast:
                v = "sensor" in q
                _case(cases, "default", table, f"{q} LIMIT {k}", 1 if v else 2, 0 if v else 1, v)
            else:
                _case(cases, "default", table, f"{q} LIMIT {k}", general=True)
    return cases


# ---- child: runs the library -----------------------------------------------------------------------------------------
def _child(spec_path):
    import ctypes as C

    sys.path.insert(0, ROOT)
    from arkflow_b200 import _lib as L
    from arkflow_b200.arrow_ffi import DeviceBatch
    from arkflow_b200.processor import MessageBatch, SqlProcessor, _check

    spec = json.load(open(spec_path))
    d, src = os.path.dirname(spec_path), spec["tables"]
    lib = L.lib()
    _check(lib.ark_b200_init(0))
    lib.ark_kernel_timing_enable(1)
    tables, report = {}, {}
    for c in spec["cases"]:
        if c["table"] not in tables:
            with pa.ipc.open_file(os.path.join(src, _fname(c["table"]))) as r:
                tables[c["table"]] = r.get_batch(0)
        rb = tables[c["table"]]
        if c["off"] is not None:
            rb = rb.slice(c["off"], rb.num_rows - 1237 if c["table"] == "slices" else rb.num_rows - c["off"] - 1)
        lib.ark_kernel_timing_reset()
        try:
            p = SqlProcessor({"query": c["query"]})
            if c["device"]:
                out = p.process_device(DeviceBatch.from_arrow(rb, keep_offsets=True))
                out = None if out is None else out.to_arrow()
            else:
                r = p.process(MessageBatch.new_arrow(rb))
                out = None if r.is_none() else r.batches[0].record_batch
        except Exception as e:  # reported, and failed, by the parent
            report[c["id"]] = {"error": repr(e)}
            continue
        counts = {}
        for name in KERNELS:
            ms, n = C.c_double(), C.c_int64()
            lib.ark_kernel_timing_get(name.encode(), C.byref(ms), C.byref(n))
            counts[name] = n.value
        if out is not None:
            with pa.ipc.new_file(os.path.join(d, f"{c['id']}.arrow"), out.schema) as w:
                w.write_batch(out)
        report[c["id"]] = {"counts": counts, "none": out is None}
    json.dump(report, open(os.path.join(d, "report.json"), "w"))
    print("CHILD_OK")


def _run_child(tmp, tables_dir, cases, env):
    spec = os.path.join(tmp, "spec.json")
    json.dump({"cases": cases, "tables": tables_dir}, open(spec, "w"))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), spec], capture_output=True, text=True, timeout=1200,
                       env=dict(os.environ, **env))
    assert r.returncode == 0 and "CHILD_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    return json.load(open(os.path.join(tmp, "report.json")))


# ---- parent: inputs, the oracle and the comparison --------------------------------------------------------------------
_INPUTS, _ORACLE = {}, {}


def _fname(table):
    return table.replace(":", "_") + ".arrow"


def _input(table):
    if table not in _INPUTS:
        s = _table_spec(table)
        fn = s.pop("fn")
        _INPUTS[table] = {"make": make_table, "window": window_table, "edge": edge_table, "general": general_table}[fn](**s)
    return _INPUTS[table]


def _sliced(table, off):
    rb = _input(table)
    if off is None:
        return rb
    rb = rb.slice(off, rb.num_rows - 1237 if table == "slices" else rb.num_rows - off - 1)
    return pa.RecordBatch.from_arrays([pa.concat_arrays([c]) for c in rb.columns], schema=rb.schema)


def _oracle(table, query, off):
    from oracle.sql_oracle import sql_process

    k = (table, query, off)
    if k not in _ORACLE:
        _ORACLE[k] = sql_process(_sliced(table, off), query)
    return _ORACLE[k]


@pytest.fixture(scope="module")
def tables_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("filter_tables"))


def _write_inputs(tables_dir, cases):
    for t in sorted({c["table"] for c in cases}):
        path = os.path.join(tables_dir, _fname(t))
        if not os.path.exists(path):
            rb = _input(t)
            with pa.ipc.new_file(path, rb.schema) as w:
                w.write_batch(rb)


def _f64_bits(col):
    """(valid mask, uint64 bits) of a Float64 column, read from its buffers: no conversion touches a NaN."""
    a = col.combine_chunks() if isinstance(col, pa.ChunkedArray) else col
    bits = np.frombuffer(a.buffers()[1], np.uint64)[a.offset:a.offset + len(a)] if len(a) else np.zeros(0, np.uint64)
    valid = a.is_valid().to_numpy(zero_copy_only=False) if a.null_count else np.ones(len(a), bool)
    return valid, bits


def read_result(path, what):
    """The child's result, fully validated: offsets that go backwards or past the data fail here, before anything
    prints or compares the batch (which would crash the process)."""
    with pa.ipc.open_file(path) as r:
        got = r.get_batch(0) if r.num_record_batches else r.schema.empty_table().to_batches()[0]
    try:
        got.validate(full=True)
    except pa.ArrowInvalid as e:
        raise AssertionError((what, "invalid result", str(e))) from None
    return got


def compare(got, want, what):
    assert got.schema.names == want.schema.names, (what, got.schema, want.schema)
    assert [f.type for f in got.schema] == [f.type for f in want.schema], (what, got.schema, want.schema)
    assert got.num_rows == want.num_rows, (what, got.num_rows, want.num_rows)
    for name, g, w in zip(want.schema.names, got.columns, want.columns):
        if pa.types.is_floating(w.type):
            gv, gb = _f64_bits(g)
            wv, wb = _f64_bits(w)
            assert np.array_equal(gv, wv), (what, name, "validity")
            bad = np.flatnonzero(wv & (gb != wb))
            assert len(bad) == 0, (what, name, len(bad), [(int(i), hex(gb[i]), hex(wb[i])) for i in bad[:5]])
        else:
            assert g.equals(w), (what, name, _first_diff(g, w))


def _first_diff(g, w):
    for i in range(min(len(g), len(w))):
        if g[i] != w[i]:
            return i, g[i], w[i]
    return None


def _string_bytes(col):
    offs = np.frombuffer(col.buffers()[1], np.int32)[col.offset:col.offset + len(col) + 1]
    return int(offs[-1]) - int(offs[0])


def _expected_kernel(path, c, avg_hint):
    """The kernel case `c` must run on `path`.  The staging size follows the batch's average string length; a device
    batch's string extent is not resolved for the fast path, which then sizes from the average selected length of the
    previous fast-path call in the process (`avg_hint`)."""
    if c["general"]:
        return GENERAL
    _, kernel, tt = PATHS[path]
    if kernel != RING:
        return kernel
    if c["v"]:
        rb = _sliced(c["table"], c["off"])
        col = rb.column("bsensor" if "bsensor" in c["query"] else "sensor")
        avg = avg_hint if c["device"] else _string_bytes(col) / len(col)
        if ring_takes(c["nf"], c["nfx"], str_cap(avg, tt), tt):
            return RING
    # declined by the ring kernel: the one-tile-per-CTA kernel takes it; with 512-row tiles nothing but the general kernel
    return TILE if tt == 1024 else GENERAL


def _run_path(path, tmp, tables_dir, cases, env=None):
    env = PATHS[path][0] if env is None else env
    _write_inputs(tables_dir, cases)
    report = _run_child(str(tmp), tables_dir, cases, env)
    seen = {}
    avg_hint = 12.8  # filter_project_tma.cu: g_avg_len_hint before the first call
    for c in cases:
        what = (path, c["table"], c["query"], c["off"], c["device"])
        run = report[c["id"]]
        assert "error" not in run, (what, run)
        want = _oracle(c["table"], c["query"], c["off"])
        assert want is not None and not run["none"], (what, want, run)
        got = read_result(os.path.join(str(tmp), f"{c['id']}.arrow"), what)
        compare(got, want, what)
        need = _expected_kernel(path, c, avg_hint)
        if need != GENERAL and c["v"] and got.num_rows > 0:
            avg_hint = _string_bytes(got.column([n for n in got.schema.names if "sensor" in n][0])) / got.num_rows
        counts = run["counts"]
        assert counts[need] >= 1, (what, need, counts)
        assert all(counts[k] == 0 for k in FAST + (GENERAL,) if k != need), (what, need, counts)
        # every fast-path launch is timed under filter_project_tma_kernel as well (the name bench.py reports)
        assert counts["filter_project_tma_kernel"] == (counts[need] if need != GENERAL else 0), (what, counts)
        seen[need] = seen.get(need, 0) + 1
    return seen


@pytest.mark.parametrize("path", list(PATHS))
def test_fast_path_kernel_matches_oracle(gpu, tmp_path, tables_dir, path):
    seen = _run_path(path, tmp_path, tables_dir, _fast_cases(path))
    assert seen.get(PATHS[path][1], 0) > 0, seen


def test_general_kernel_matches_oracle(gpu, tmp_path, tables_dir):
    """filter_project_kernel<PRED, NV>: NULLs, VM predicates, computed outputs, two var-len outputs and the multi-launch
    split, at 2047 / 2048 / 2049 rows (its tile is 2048 rows) and at 2^22 + 3."""
    _run_path("default", tmp_path, tables_dir, _general_cases())


def test_limit_matches_oracle(gpu, tmp_path, tables_dir):
    """LIMIT 0, 1, count - 1, count, count + 1 after the fast path (which re-resolves the var-len extents) and after the
    general kernel."""
    counts = {}
    for table, q in (("p:1024:33792:s0.5", "SELECT sensor, value FROM flow WHERE value >= 10"),
                     ("p:1024:33792:s0.5", "SELECT timestamp, value FROM flow WHERE value >= 10"),
                     ("gen:2049", "SELECT s, b, value FROM flow WHERE value >= 10")):
        counts[(table, q)] = _oracle(table, q, None).num_rows
    _run_path("default", tmp_path, tables_dir, _limit_cases(counts))


def test_config2_batch_of_2_24_rows(gpu, tmp_path, tables_dir):
    """One batch of 2^24 + 1 rows on the default path (16 385 tiles, 513 groups), every row and half of them surviving;
    compared with a numpy mask and pc.filter (test_oracle_crosscheck ties pc.filter to the oracle)."""
    cases = []
    for pattern in ("all", "s0.5"):
        table = f"huge:{pattern}"
        _case(cases, "default", table, "SELECT sensor, value FROM flow WHERE value >= 10", 1, 0, True)
    _write_inputs(tables_dir, cases)
    report = _run_child(str(tmp_path), tables_dir, cases, {})
    for c in cases:
        run = report[c["id"]]
        assert "error" not in run and not run["none"], (c, run)
        rb = _input(c["table"])
        m = pc.greater_equal(rb.column("value"), 10)
        want = pa.record_batch({"sensor": pc.filter(rb.column("sensor"), m), "value": pc.filter(rb.column("value"), m)})
        got = read_result(os.path.join(str(tmp_path), f"{c['id']}.arrow"), c["table"])
        compare(got, want, c["table"])
        assert run["counts"][TILE] == 1 and run["counts"][GENERAL] == 0, run
        _INPUTS.pop(c["table"])


if __name__ == "__main__":
    _child(sys.argv[1])
