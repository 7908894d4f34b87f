"""The `file` input's `arrow` type (csrc/arrow_ipc.cu) against oracle/arrow_ipc_oracle.py, whole batches at a time.

Every file is written from a seed into tmp_path, by pyarrow or by the oracle's writer (which can place any frame form
and any broken byte).  Batches are compared by the rules of tests/test_inputs_edges_gpu.py (schema names, types and
nullability, Array.equals per column, floats by bit pattern of their own width, validate(full=True)), through both read() and
read_device().to_arrow(); errors by kind and full message.  Each case asserts the launch counts (ark_kernel_timing_get):
a view runs neither the LZ4 kernel nor concat's copy.
"""
import io
import struct

import numpy as np
import pyarrow as pa
import pytest

from arkflow_b200.input import FileInput
from arkflow_b200.processor import ArkError, SqlProcessor
from oracle.arrow_ipc_oracle import PFX, lz4_frame, read_ipc, stored_from_arrow, write_ipc, xxh32
from oracle.sql_oracle import sql_process
from test_arrow_ipc_oracle import fields_of, pyarrow_file, sample
from test_inputs_edges_gpu import CHUNK, launches, same_batch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def timing(gpu):
    gpu.ark_kernel_timing_enable(1)
    yield gpu
    gpu.ark_kernel_timing_enable(0)


def scan(path, device=False, **cfg):
    out = []
    try:
        inp = FileInput(dict(cfg, input_type={"type": "arrow", "path": str(path)}))
        inp.connect()
        while True:
            out.append(inp.read_device().to_arrow() if device else inp.read()[0].record_batch)
    except ArkError as e:
        return out, (None if e.kind == "EOF" else e)


def same_batches(got, want, what=""):
    """test_inputs_edges_gpu.same_batches, with Float32 columns compared by their 32-bit patterns."""
    assert [b.num_rows for b in got] == [b.num_rows for b in want], what
    for k, (g, w) in enumerate(zip(got, want)):
        f32 = [i for i, f in enumerate(w.schema) if f.type == pa.float32()]
        for i in f32:
            gb, wb = (x.column(i).fill_null(0.0).to_numpy(zero_copy_only=False).view(np.uint32) for x in (g, w))
            assert g.column(i).is_valid().equals(w.column(i).is_valid()) and np.array_equal(gb, wb), (what, k, i)
        keep = [i for i in range(w.num_columns) if i not in f32]
        same_batch(pa.record_batch([g.column(i) for i in keep], names=[g.schema.names[i] for i in keep]).cast(pa.schema([g.schema.field(i) for i in keep])) if f32 else g,
                   pa.record_batch([w.column(i) for i in keep], names=[w.schema.names[i] for i in keep]).cast(pa.schema([w.schema.field(i) for i in keep])) if f32 else w,
                   (what, "batch", k))


def check(lib, tmp_path, data, batch_size=None, query=None, lz4=None, copy=None):
    """Scans `data` both ways and compares with the oracle; `lz4` / `copy`: whether the LZ4 kernel / concat's copy ran."""
    p = tmp_path / "t.arrow"
    p.write_bytes(data)
    want, werr = read_ipc(data, batch_size)
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
        if lz4 is not None:
            assert (launches(lib, "ipc_lz4_kernel") > 0) == lz4
        if copy is not None:
            assert (launches(lib, "concat_copy_kernel") > 0) == copy
    return want, werr


def nulls_at_edges(n, seed=0):
    """sample() with NULLs also at the 32-row word and 8192-row validation-CTA edges."""
    rb = sample(n, seed)
    edge = [i % 8192 in (0, 8191) or i % 32 in (0, 31) for i in range(n)]
    cols = [rb.column(k) if rb.schema.field(k).type == pa.null() else
            pa.array([None if e else v for e, v in zip(edge, rb.column(k).to_pylist())], rb.schema.field(k).type) for k in range(rb.num_columns)]
    return pa.record_batch(cols, schema=rb.schema)


@pytest.mark.parametrize("compression", [None, "lz4"])
@pytest.mark.parametrize("legacy", [False, True])
def test_every_type_view(gpu, tmp_path, compression, legacy):
    data = pyarrow_file([nulls_at_edges(20000)], compression, legacy)
    check(gpu, tmp_path, data, lz4=compression is not None, copy=False)


@pytest.mark.parametrize("batch_size", [None, 1, 7, 300, 301, 1000, 4096])
def test_batch_sizes(gpu, tmp_path, batch_size):
    rbs = [sample(n, 17 * k) for k, n in enumerate([300, 0, 1, 700, 0, 300])]
    check(gpu, tmp_path, pyarrow_file(rbs), batch_size=batch_size)
    check(gpu, tmp_path, pyarrow_file(rbs, "lz4"), batch_size=batch_size, lz4=True)


def test_view_and_concat_routes(gpu, tmp_path):
    rbs = [sample(300, 0), sample(300, 300)]
    check(gpu, tmp_path, pyarrow_file(rbs), batch_size=300, lz4=False, copy=False)
    check(gpu, tmp_path, pyarrow_file(rbs), batch_size=150, lz4=False, copy=False)
    check(gpu, tmp_path, pyarrow_file(rbs), batch_size=200, lz4=False, copy=True)


def test_sliced_and_empty(gpu, tmp_path):
    base = nulls_at_edges(1000)
    check(gpu, tmp_path, pyarrow_file([base.slice(13, 500), base.slice(0, 0), base.slice(999, 1)]))
    check(gpu, tmp_path, pyarrow_file([base.slice(13, 500), base.slice(3, 77)], "lz4"), batch_size=100)
    # a schema and no batches
    want, err = check(gpu, tmp_path, write_ipc(fields_of(base), []))
    assert want == [] and err is None


def test_large_file(gpu, tmp_path):
    rb = pa.record_batch({"l": pa.array(range(3 * CHUNK // 16), pa.int64()), "s": pa.array(["v%d" % (i % 1000) for i in range(3 * CHUNK // 16)])})
    data = pyarrow_file([rb.slice(0, len(rb) // 2), rb.slice(len(rb) // 2)])
    assert len(data) > 2 * CHUNK
    check(gpu, tmp_path, data, batch_size=1 << 20)


@pytest.mark.parametrize("frame", [{}, {"independent": True}, {"block_checksum": True, "content_checksum": True, "content_size": True},
                                   {"stored": True}, {"stored": (0,)}, {"block_code": 5}, {"matches": False}, {"raw": True}])
def test_lz4_frame_forms(gpu, tmp_path, frame):
    rb = nulls_at_edges(30000)
    data = write_ipc(fields_of(rb), [stored_from_arrow(rb, lz4=True, **frame), stored_from_arrow(sample(0), lz4=True, **frame)])
    check(gpu, tmp_path, data, lz4=not frame.get("raw", False))
    check(gpu, tmp_path, data, batch_size=7777)


def test_query(gpu, tmp_path):
    rbs = [sample(500, 0), sample(500, 500)]
    check(gpu, tmp_path, pyarrow_file(rbs), batch_size=400, query="SELECT l, s, d FROM flow WHERE l > 20000000000000")
    # SQL over an Int32 column is outside the GPU subset: the input reports what the sql processor reports
    p = tmp_path / "q.arrow"
    p.write_bytes(pyarrow_file(rbs))
    for q in ("SELECT i FROM flow", "SELECT i FROM flow WHERE i > 0", "SELECT * FROM flow"):
        got, err = scan(p, query={"query": q})
        with pytest.raises(ArkError) as want:
            SqlProcessor({"query": q}).process(rbs[0])
        assert got == [] and err is not None and (err.kind, err.message) == (want.value.kind, want.value.message) and err.kind == "Unsupported"


# ---- read-time errors ------------------------------------------------------------------------------------------------
def five(mutate_at, mut, lz4=None, frame=None):
    """Five stored batches of 100 rows; batch `mutate_at` is rewritten by `mut(stored)`."""
    rbs = [sample(100, 100 * k) for k in range(5)]
    st = [stored_from_arrow(rb, lz4=lz4, **(frame or {})) for rb in rbs]
    mut(st[mutate_at])
    return write_ipc(fields_of(rbs[0]), st)


def buf_index(name, which):
    """Index of buffer `which` (0 validity, 1 values / offsets, 2 data) of field `name` in a sample() batch."""
    j = 0
    for f in sample(1).schema:
        nb = 0 if f.type == pa.null() else 3 if f.type in (pa.utf8(), pa.binary()) else 2
        if f.name == name:
            return j + which
        j += nb
    raise KeyError(name)


def set_i32(b, at, v):
    b = bytearray(b)
    struct.pack_into("<i", b, at, v)
    return bytes(b)


MUTS = {
    "offsets": lambda s: s.buffers.__setitem__(buf_index("y", 1), set_i32(s.buffers[buf_index("y", 1)], 4 * 50, 10**6)),
    "decreasing": lambda s: s.buffers.__setitem__(buf_index("s", 1), set_i32(s.buffers[buf_index("s", 1)], 4 * 30, 0)),
    "utf8": lambda s: s.buffers.__setitem__(buf_index("s", 2), b"\xff" + s.buffers[buf_index("s", 2)][1:]),
    "nulls": lambda s: s.nodes.__setitem__(2, (100, s.nodes[2][1] + 1)),
}


@pytest.mark.parametrize("at", [0, 2, 4])
@pytest.mark.parametrize("what", sorted(MUTS))
def test_validation_errors(gpu, tmp_path, at, what):
    for bs in (None, 100, 150):
        want, err = check(gpu, tmp_path, five(at, MUTS[what]), batch_size=bs)
        assert err is not None and err.message.startswith(PFX) and "(record batch %d, column" % at in err.message


def frame_mut(kind):
    def mut(s):
        j = buf_index("l", 1)
        raw = bytes(range(256)) * 3 + bytes(800 - 768)
        if kind in ("zero", "before"):
            # the first block's first sequence: token at byte 11, its literals, then the match offset
            blk = bytearray(lz4_frame(b"ab" * 400))
            lit = blk[11] >> 4
            blk[12 + lit:14 + lit] = struct.pack("<H", 0 if kind == "zero" else 60000)
            s.buffers[j] = struct.pack("<q", 800) + bytes(blk)
        elif kind == "overrun":
            s.buffers[j] = struct.pack("<q", 800) + lz4_frame(raw + b"x")
        elif kind == "underfill":
            s.buffers[j] = struct.pack("<q", 800) + lz4_frame(raw[:-1])
        elif kind == "truncated":
            s.buffers[j] = struct.pack("<q", 800) + lz4_frame(raw)[:-6]
        elif kind == "checksum":
            f = bytearray(lz4_frame(raw, content_checksum=True))
            f[-1] ^= 0x10
            s.buffers[j] = struct.pack("<q", 800) + bytes(f)
        elif kind == "header":
            f = bytearray(lz4_frame(raw))
            f[6] ^= 1
            s.buffers[j] = struct.pack("<q", 800) + bytes(f)
    return mut


@pytest.mark.parametrize("at", [0, 2, 4])
@pytest.mark.parametrize("kind", ["zero", "before", "overrun", "underfill", "truncated", "checksum", "header"])
def test_lz4_errors(gpu, tmp_path, at, kind):
    want, err = check(gpu, tmp_path, five(at, frame_mut(kind), lz4=True), lz4=True)
    assert err is not None and "(record batch %d, column 'l')" % at in err.message


def test_independent_block_offset(gpu, tmp_path):
    # linked blocks whose FLG claims independence: the second block's matches reach into the first
    data = (bytes(range(200)) * 2000)[:200000]

    def mut(s):
        f = bytearray(lz4_frame(data))
        f[4] |= 0x20
        f[6] = (xxh32(bytes(f[4:6])) >> 8) & 0xFF
        s.buffers[buf_index("y", 2)] = struct.pack("<q", len(data)) + bytes(f)
        s.buffers[buf_index("y", 1)] = struct.pack("<q", -1) + struct.pack("<101i", *([0] * 100 + [len(data)]))
    want, err = check(gpu, tmp_path, five(1, mut, lz4=True), lz4=True)
    assert err is not None and "before the start" in err.message


def test_first_failure_in_file_order(gpu, tmp_path):
    rbs = [sample(100, 100 * k) for k in range(3)]
    st = [stored_from_arrow(rb) for rb in rbs]
    MUTS["utf8"](st[1])
    MUTS["nulls"](st[1])
    MUTS["offsets"](st[2])
    want, err = check(gpu, tmp_path, write_ipc(fields_of(rbs[0]), st), batch_size=1000)
    assert "(record batch 1, column 'i')" in err.message and len(want) == 0


def test_batch_of_2_22_rows(gpu, tmp_path):
    n = 1 << 22
    rb = pa.record_batch({"l": pa.array(range(n), pa.int64()), "b": pa.array([i % 3 == 0 for i in range(n)]),
                          "s": pa.array(["r%d" % (i % 97) if i % 5 else None for i in range(n)])})
    check(gpu, tmp_path, pyarrow_file([rb.slice(0, 3000000), rb.slice(3000000)]), lz4=False, copy=True)
    check(gpu, tmp_path, pyarrow_file([rb]), lz4=False, copy=False)
