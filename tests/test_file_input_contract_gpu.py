"""The `file` input's contract, the same for every format (csv, json, avro, arrow) over the same logical rows.

Each format is written from the same 23 rows (a: Int64, b: Float64, s: Utf8) and scanned through FileInput: a missing
path, read before connect(), connect() twice, read after close() and after EOF, an empty file, `batch_size` cuts around
the row count, a `query` that empties some batches, and the kernels each connect() and read() launches.  The rows joined
back together are compared with the plain rows; Avro and Arrow IPC files are also compared with their oracles.
"""
import io
import json

import pyarrow as pa
import pytest

from arkflow_b200.input import FileInput
from arkflow_b200.processor import ArkError, SqlProcessor
from oracle.arrow_ipc_oracle import read_ipc
from oracle.avro_oracle import header, read_avro, record_schema, write_avro
from oracle.csv_oracle import csv_read
from test_inputs_edges_gpu import launches

pytestmark = pytest.mark.gpu

FORMATS = ("csv", "json", "avro", "arrow")
ROWS = 23
AVRO_SCHEMA = record_schema([("a", "long"), ("b", "double"), ("s", "string")])
ARROW_SCHEMA = pa.schema([("a", pa.int64()), ("b", pa.float64()), ("s", pa.utf8())])
# every kernel timer a file read can reach: the inputs, the json decoder, the bitmap, varlen, concat and query kernels
TIMERS = ("line_start_flags_kernel", "rebase_offsets_kernel", "csv_parse_kernel", "csv_strings_kernel", "json_count_kernel",
          "json_parse_kernel", "json_strings_kernel", "json_quoted_numbers_kernel", "json_list_count_kernel",
          "json_list_fill_kernel", "avro_snappy_kernel", "avro_index_kernel", "avro_decode_kernel", "ipc_lz4_kernel",
          "ipc_validate_kernel", "count_zeros_kernel", "pack_bits_kernel", "realign_bits_kernel", "gather_extents_kernel",
          "utf8_validate_kernel", "concat_lengths_kernel", "concat_offsets_kernel", "concat_copy_kernel",
          "concat_write_kernel", "concat_bits_kernel", "filter_project_kernel", "filter_project_tma_kernel",
          "take_fixed8_kernel", "take_lengths_kernel", "take_bytes_tile_kernel", "take_bits_kernel", "take_multi_kernel")
QUERY = "SELECT a, s FROM flow WHERE a > 25"  # with batch_size 7 the first two batches keep no row


@pytest.fixture(scope="module", autouse=True)
def timing(gpu):
    gpu.ark_kernel_timing_enable(1)
    yield gpu
    gpu.ark_kernel_timing_enable(0)


def rows(n=ROWS):
    return [(3 * i - 20, i + 0.25, f"s{i}") for i in range(n)]


def file_bytes(fmt, n=ROWS):
    """The rows in format `fmt`; n == 0 gives the format's empty file (header-only CSV, zero-line NDJSON, an Avro file
    with no blocks, a schema-only IPC file).  Avro and IPC files hold several blocks / record batches."""
    rs = rows(n)
    if fmt == "csv":
        return ("a,b,s\n" + "".join("%d,%r,%s\n" % r for r in rs)).encode()
    if fmt == "json":
        return "".join(json.dumps({"a": a, "b": b, "s": s}) + "\n" for a, b, s in rs).encode()
    if fmt == "avro":
        return write_avro(AVRO_SCHEMA, rs, block_rows=5) if n else header(AVRO_SCHEMA)
    sink = io.BytesIO()
    with pa.ipc.new_file(sink, ARROW_SCHEMA) as w:
        for k in range(0, n, 5):
            w.write(pa.record_batch([pa.array(c) for c in zip(*rs[k:k + 5])], schema=ARROW_SCHEMA))
    return sink.getvalue()


def make(tmp_path, fmt, data=None, **cfg):
    p = tmp_path / f"t.{fmt}"
    p.write_bytes(file_bytes(fmt) if data is None else data)
    return FileInput(dict(cfg, input_type={"type": fmt, "path": str(p)}))


def read_all(inp):
    out = []
    while True:
        try:
            out.append(inp.read()[0].record_batch)
        except ArkError as e:
            assert e.kind == "EOF", (e.kind, e.message)
            return out


def joined(batches):
    return pa.Table.from_batches(batches).to_pydict() if batches else {}


def expect_eof(inp):
    with pytest.raises(ArkError) as e:
        inp.read()
    assert e.value.kind == "EOF"


@pytest.mark.parametrize("fmt", FORMATS)
def test_missing_path(gpu, tmp_path, fmt):
    p = tmp_path / "missing"
    inp = FileInput({"input_type": {"type": fmt, "path": str(p)}})
    with pytest.raises(ArkError) as e:
        inp.connect()
    assert (e.value.kind, e.value.message) == ("Process", f"Read input failed: Object at location {p} not found")
    with pytest.raises(ArkError) as e:  # a failed connect() leaves the input unconnected
        inp.read()
    assert (e.value.kind, e.value.message) == ("Process", "Stream is None")


@pytest.mark.parametrize("fmt", FORMATS)
def test_lifecycle(gpu, tmp_path, fmt):
    inp = make(tmp_path, fmt)
    with pytest.raises(ArkError) as e:
        inp.read()
    assert (e.value.kind, e.value.message) == ("Process", "Stream is None")
    inp.connect()
    inp.connect()  # idempotent: the file is not read again
    got = read_all(inp)
    assert [b.num_rows for b in got] == [ROWS]
    expect_eof(inp)  # after EOF, EOF again
    inp = make(tmp_path, fmt, batch_size=5)
    inp.connect()
    assert inp.read()[0].record_batch.num_rows == 5
    inp.close()
    expect_eof(inp)
    expect_eof(inp)


@pytest.mark.parametrize("fmt", FORMATS)
def test_empty_file(gpu, tmp_path, fmt):
    inp = make(tmp_path, fmt, data=file_bytes(fmt, 0))
    inp.connect()
    expect_eof(inp)


@pytest.mark.parametrize("batch_size", [1, 7, ROWS - 1, ROWS, ROWS + 1])
@pytest.mark.parametrize("fmt", FORMATS)
def test_batch_sizes(gpu, tmp_path, fmt, batch_size):
    inp = make(tmp_path, fmt, batch_size=batch_size)
    inp.connect()
    got = read_all(inp)
    sizes = [b.num_rows for b in got]
    assert sizes[:-1] == [batch_size] * (len(sizes) - 1) and 0 < sizes[-1] <= batch_size
    a, b, s = (list(c) for c in zip(*rows()))
    assert joined(got) == {"a": a, "b": b, "s": s}
    data = file_bytes(fmt)
    if fmt == "csv":
        want = csv_read(data, batch_rows=batch_size)
    elif fmt == "avro":
        want, err = read_avro(data, batch_size)
        assert err is None
    elif fmt == "arrow":
        want, err = read_ipc(data, batch_size)
        assert err is None
    else:
        return
    assert sizes == [w.num_rows for w in want]
    for g, w in zip(got, want):
        assert g.schema == w.schema and g.equals(w)


@pytest.mark.parametrize("fmt", FORMATS)
def test_query_that_empties_batches(gpu, tmp_path, fmt):
    inp = make(tmp_path, fmt, batch_size=7, query={"query": QUERY})
    inp.connect()
    got = read_all(inp)
    # a batch the filter empties comes back as a batch of 0 rows with the query's columns
    assert [b.num_rows for b in got] == [0, 0, 5, 2] and all(b.schema.names == ["a", "s"] for b in got)
    keep = [r for r in rows() if r[0] > 25]
    assert joined(got) == {"a": [r[0] for r in keep], "s": [r[2] for r in keep]}


AVRO_NARROW = record_schema([("i", "int"), ("f", "float"), ("l", "long")])


@pytest.mark.parametrize("q", ["SELECT i FROM flow", "SELECT i FROM flow WHERE i > 0", "SELECT f FROM flow",
                               "SELECT l FROM flow WHERE f > 0", "SELECT * FROM flow"])
def test_avro_int32_float32_query_is_unsupported(gpu, tmp_path, q):
    """Int32 and Float32 columns reach the query's planner as the sql processor's import presents them, for every
    format: a query that reads one is Unsupported with the sql processor's own message."""
    n = 10
    data = write_avro(AVRO_NARROW, [(i - 3, i / 4, i) for i in range(n)], block_rows=4)
    inp = make(tmp_path, "avro", data=data, query={"query": q})
    inp.connect()
    with pytest.raises(ArkError) as got:
        inp.read()
    rb = pa.record_batch({"i": pa.array(range(-3, n - 3), pa.int32()), "f": pa.array([i / 4 for i in range(n)], pa.float32()),
                          "l": pa.array(range(n), pa.int64())})
    with pytest.raises(ArkError) as want:
        SqlProcessor({"query": q}).process(rb)
    assert want.value.kind == "Unsupported"
    assert (got.value.kind, got.value.message) == (want.value.kind, want.value.message)


def test_avro_query_over_wide_columns_only(gpu, tmp_path):
    data = write_avro(AVRO_NARROW, [(i - 3, i / 4, i) for i in range(10)], block_rows=4)
    inp = make(tmp_path, "avro", data=data, query={"query": "SELECT l FROM flow WHERE l > 6"})
    inp.connect()
    assert joined(read_all(inp)) == {"l": [7, 8, 9]}


# ---- kernels per call: (launches, {timer: launches}) for connect() and then every read() up to and including EOF ------
def trace(lib, inp):
    out = []

    def step(call):
        lib.ark_kernel_timing_reset()
        n0 = lib.ark_kernel_launch_count()
        eof = False
        try:
            call()
        except ArkError as e:
            assert e.kind == "EOF", e.message
            eof = True
        n = lib.ark_kernel_launch_count() - n0
        out.append((n, {t: launches(lib, t) for t in TIMERS if launches(lib, t)}))
        return eof

    step(inp.connect)
    while not step(inp.read):
        pass
    return out


CONNECT_LINES = (2, {"line_start_flags_kernel": 1})  # the flags kernel and the flagged select
CSV_READ = (7, {"rebase_offsets_kernel": 1, "csv_parse_kernel": 1, "csv_strings_kernel": 1, "pack_bits_kernel": 3})
JSON_READ = (7, {"rebase_offsets_kernel": 1, "json_parse_kernel": 1, "json_strings_kernel": 1, "pack_bits_kernel": 3})
AVRO_READ = (4, {"avro_index_kernel": 1, "avro_decode_kernel": 1})
ARROW_SPAN = (4, {"ipc_validate_kernel": 1, "gather_extents_kernel": 1, "concat_offsets_kernel": 1, "concat_copy_kernel": 1})
ARROW_VIEW = (2, {"rebase_offsets_kernel": 1, "gather_extents_kernel": 1})
EOF_READ = (0, {})
EXPECTED_TRACE = {"csv": [CONNECT_LINES] + [CSV_READ] * 4 + [EOF_READ],
                  "json": [CONNECT_LINES] + [JSON_READ] * 4 + [EOF_READ],
                  "avro": [EOF_READ] + [AVRO_READ] * 4 + [EOF_READ],
                  "arrow": [EOF_READ] + [ARROW_SPAN] * 3 + [ARROW_VIEW] + [EOF_READ]}


def with_query(step, view=False):
    """`step` followed by the query's filter kernel (a view's Utf8 slice needs no rebase when the query reads it)."""
    n, t = step
    t = dict(t, filter_project_tma_kernel=1)
    if view:
        del t["rebase_offsets_kernel"]
    return (n + 1 - view, t)


EXPECTED_QUERY_TRACE = {"csv": [CONNECT_LINES] + [with_query(CSV_READ)] * 4 + [EOF_READ],
                        "json": [CONNECT_LINES] + [with_query(JSON_READ)] * 4 + [EOF_READ],
                        "avro": [EOF_READ] + [with_query(AVRO_READ)] * 4 + [EOF_READ],
                        "arrow": [EOF_READ] + [with_query(ARROW_SPAN)] * 3 + [with_query(ARROW_VIEW, view=True)] + [EOF_READ]}


@pytest.mark.parametrize("fmt", FORMATS)
def test_kernels_per_call(gpu, tmp_path, fmt):
    assert trace(gpu, make(tmp_path, fmt, batch_size=7)) == EXPECTED_TRACE[fmt]
    assert trace(gpu, make(tmp_path, fmt, batch_size=7, query={"query": QUERY})) == EXPECTED_QUERY_TRACE[fmt]
