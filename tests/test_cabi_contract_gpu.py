"""The C ABI's call contract on the device: every processor entry point, host and device, releases its moved-in input
exactly once on success and on ProcessResult::None (after the call returns, or when an output that aliases it is
released); an empty input is None for sql and protobuf in both directions; the device exports normalise what they
hand over (a sliced Utf8 column's offsets rebased, a validity bitmap that starts inside a byte realigned); and each call
launches a pinned number of kernels, so moving work between an entry point and its callees cannot add launches unseen."""
import ctypes as C
import json

import numpy as np
import pyarrow as pa
import pytest

from arkflow_b200 import _lib as L
from arkflow_b200.arrow_ffi import DeviceBatch, release_schema

pytestmark = pytest.mark.gpu

PROTO = 'syntax = "proto3";\npackage pkg;\nmessage M { int64 timestamp = 1; double value = 2; string sensor = 3; }\n'

# kernel launches of one call on the inputs below (host, device), measured on an H100
LAUNCHES = {
    "sql/host": 3,
    "sql/device": 2,
    "sql_filter/host": 3,
    "sql_filter/device": 3,
    "json_to_arrow/host": 6,
    "json_to_arrow/device": 7,
    "arrow_to_json/host": 6,
    "arrow_to_json/device": 7,
    "protobuf_to_arrow/host": 3,
    "protobuf_to_arrow/device": 4,
    "arrow_to_protobuf/host": 4,
    "arrow_to_protobuf/device": 5,
    "concat/device": 5,
    "buffer_read/host_write": 3,
    "buffer_read/device_write": 4,
    "input_read/device": 1,
    "ipc_concat_slices/device": 5,
    "expr[sensor]/host": 2,
    "expr[sensor]/device": 1,
    "expr[value + 1]/host": 2,
    "expr[value + 1]/device": 2,
}


def base_batch(nulls=True, n=40):
    rng = np.random.default_rng(7)
    ts = pa.array(1_700_000_000_000 + np.arange(n), pa.int64())
    vals = rng.integers(0, 20, n).astype(np.float64)
    value = pa.array([None if nulls and i % 3 == 0 else float(v) for i, v in enumerate(vals)], pa.float64())
    sensor = pa.array([None if nulls and i % 5 == 1 else f"temp_{i % 7}" + "x" * (i % 4) for i in range(n)], pa.string())
    return pa.record_batch([ts, value, sensor], names=["timestamp", "value", "sensor"])


class Counted:
    """Wraps an exported array's release callback so that its calls are counted."""

    def __init__(self, arr):
        self.calls = 0
        self._orig = L.RELEASE_ARRAY(arr.release)

        def rel(p):
            self.calls += 1
            self._orig(p)

        self._cb = L.RELEASE_ARRAY(rel)
        arr.release = C.cast(self._cb, C.c_void_p).value


class HostIn:
    def __init__(self, rb):
        self.arr, self.sch = L.ArrowArray(), L.ArrowSchema()
        rb._export_to_c(C.addressof(self.arr), C.addressof(self.sch))
        self.count = Counted(self.arr)

    def close(self):
        release_schema(self.sch)


class DevIn:
    def __init__(self, rb):
        self.batch = DeviceBatch.from_arrow(rb, keep_offsets=True)
        self.arr, self.sch = self.batch.export()
        self.count = Counted(self.arr.array)

    def close(self):
        pass


def result(out, osch, device):
    """The output as pyarrow (None for ProcessResult::None); a device output is released before returning."""
    if (out.array.release if device else out.release) is None:
        return None
    if not device:
        return pa.RecordBatch._import_from_c(C.addressof(out), C.addressof(osch))
    b = DeviceBatch.adopt(out, osch)
    rb = b.to_arrow()
    b._owner.close()
    return rb


def call(lib, fn, *args, device):
    out, osch = (L.ArrowDeviceArray() if device else L.ArrowArray()), L.ArrowSchema()
    n0 = lib.ark_kernel_launch_count()
    st = fn(*args, C.byref(out), C.byref(osch))
    launches = lib.ark_kernel_launch_count() - n0
    assert st == L.ARK_OK, lib.ark_last_error()
    return out, osch, launches


def check_launches(key, n):
    assert n == LAUNCHES[key], (key, n)


@pytest.fixture(scope="module")
def procs(gpu, tmp_path_factory):
    d = tmp_path_factory.mktemp("proto")
    (d / "m.proto").write_text(PROTO)
    pb = json.dumps({"proto_inputs": [str(d)], "message_type": "pkg.M"}).encode()
    configs = {"sql": b'{"query": "SELECT * FROM flow"}', "sql_filter": b'{"query": "SELECT sensor, value FROM flow WHERE value > 5"}',
               "json_to_arrow": b"{}", "arrow_to_json": b"{}", "protobuf_to_arrow": pb, "arrow_to_protobuf": pb}
    hs = {}
    for k, cfg in configs.items():
        h = C.c_void_p()
        kind = "sql" if k.startswith("sql") else k
        assert getattr(gpu, f"ark_{kind}_create")(cfg, C.byref(h)) == L.ARK_OK, gpu.ark_last_error()
        hs[k] = h
    yield hs
    for h in hs.values():
        gpu.ark_proc_destroy(h)


def encoded(lib, procs, kind):
    """A batch of JSON documents / protobuf messages in __value__, encoded on the host path."""
    h = procs["arrow_to_json" if kind == "json" else "arrow_to_protobuf"]
    inp = HostIn(base_batch(nulls=kind == "json"))
    fn = lib.ark_arrow_to_json_process if kind == "json" else lib.ark_arrow_to_protobuf_process
    out, osch, _ = call(lib, fn, h, C.byref(inp.arr), C.byref(inp.sch), device=False)
    inp.close()
    return result(out, osch, False)


def inputs(lib, procs, key):
    if key == "json_to_arrow":
        return encoded(lib, procs, "json")
    if key == "protobuf_to_arrow":
        return encoded(lib, procs, "protobuf")
    return base_batch(nulls=key != "arrow_to_protobuf")


def process_name(key, device):
    kind = "sql" if key.startswith("sql") else key
    return f"ark_{kind}_process_device" if device else f"ark_{kind}_process"


def run_process(lib, procs, key, rb, device):
    inp = (DevIn if device else HostIn)(rb)
    out, osch, launches = call(lib, getattr(lib, process_name(key, device)), procs[key], C.byref(inp.arr), C.byref(inp.sch), device=device)
    assert inp.count.calls <= 1
    got = result(out, osch, device)  # releases a device output, and with it an input it aliased
    assert inp.count.calls == 1, "the input's release ran %d times" % inp.count.calls
    inp.close()
    return got, launches


KEYS = ["sql", "sql_filter", "json_to_arrow", "arrow_to_json", "protobuf_to_arrow", "arrow_to_protobuf"]


@pytest.mark.parametrize("key", KEYS)
def test_processor_releases_its_input_once_and_devices_agree(gpu, procs, key):
    rb = inputs(gpu, procs, key).slice(5, 30)  # offsets[0] != 0 and bitmaps that start inside a byte
    host, nh = run_process(gpu, procs, key, rb, False)
    dev, nd = run_process(gpu, procs, key, rb, True)
    assert host is not None and dev is not None
    assert dev.equals(host), (dev, host)
    if key == "sql":
        assert host.equals(rb)
    check_launches(f"{key}/host", nh)
    check_launches(f"{key}/device", nd)


@pytest.mark.parametrize("key", KEYS)
def test_processor_on_an_empty_input(gpu, procs, key):
    rb = inputs(gpu, procs, key).slice(0, 0)
    host, _ = run_process(gpu, procs, key, rb, False)
    dev, _ = run_process(gpu, procs, key, rb, True)
    if key.startswith("sql") or "protobuf" in key:
        assert host is None and dev is None  # ProcessResult::None
    else:
        assert host is not None and dev is not None and dev.equals(host)


def test_concat_device_normalises_sliced_members(gpu):
    from arkflow_b200.buffer import concat_batches_device

    rb = base_batch()
    parts = [rb.slice(3, 11), rb.slice(17, 20)]
    n0 = gpu.ark_kernel_launch_count()
    got = concat_batches_device([DeviceBatch.from_arrow(p, keep_offsets=True) for p in parts]).to_arrow()
    check_launches("concat/device", gpu.ark_kernel_launch_count() - n0)
    assert got.equals(pa.concat_batches(parts))


@pytest.mark.parametrize("device_write", [False, True], ids=["host_write", "device_write"])
def test_buffer_read_device_normalises_sliced_batches(gpu, device_write):
    from arkflow_b200.buffer import MemoryBuffer

    rb = base_batch().slice(5, 30)
    buf = MemoryBuffer({"capacity": 1, "timeout": "10s"})
    if device_write:
        buf.write_device(DeviceBatch.from_arrow(rb, keep_offsets=True))
    else:
        buf.write(rb)
    n0 = gpu.ark_kernel_launch_count()
    got, _ack = buf.read_device()
    check_launches(f"buffer_read/{'device' if device_write else 'host'}_write", gpu.ark_kernel_launch_count() - n0)
    buf.close()
    assert got.to_arrow().equals(rb)


def test_input_read_device_matches_the_host_read(gpu):
    from arkflow_b200.input import GenerateInput

    cfg = {"context": '{"timestamp": 1625000000000, "value": 10, "sensor": "temp_1"}', "interval": "1ms", "count": 10, "batch_size": 5}
    a, b = GenerateInput(cfg), GenerateInput(cfg)
    a.connect(), b.connect()
    host, _ = a.read()
    n0 = gpu.ark_kernel_launch_count()
    dev = b.read_device()
    check_launches("input_read/device", gpu.ark_kernel_launch_count() - n0)
    assert dev.to_arrow().equals(host.record_batch)
    a.close(), b.close()


def test_ipc_concat_slices_device_normalises_a_sliced_batch(gpu):
    rb = base_batch().slice(5, 30)
    inp = DevIn(rb)
    blob, size = (C.c_uint8 * 65536)(), C.c_int64()
    assert gpu.ark_ipc_export_device(C.byref(inp.arr), C.byref(inp.sch), blob, 65536, C.byref(size)) == L.ARK_OK, gpu.ark_last_error()
    assert inp.count.calls == 1
    blobs = (C.POINTER(C.c_uint8) * 1)(C.cast(blob, C.POINTER(C.c_uint8)))
    sizes, row0, n_rows = (C.c_int64 * 1)(size.value), (C.c_int64 * 1)(4), (C.c_int64 * 1)(20)
    out, osch, n = call(gpu, gpu.ark_ipc_concat_slices_device, 1, blobs, sizes, row0, n_rows, device=True)
    check_launches("ipc_concat_slices/device", n)
    assert result(out, osch, True).equals(rb.slice(4, 20))


@pytest.mark.parametrize("expr", ["sensor", "value + 1"])
def test_expr_evaluate_device_matches_the_host(gpu, expr):
    rb = base_batch().slice(5, 30)
    got = {}
    for device in (False, True):
        inp = (DevIn if device else HostIn)(rb)
        fn = gpu.ark_expr_evaluate_device if device else gpu.ark_expr_evaluate
        scalar = C.c_int(-1)
        out, osch, n = call(gpu, lambda o, s: fn(expr.encode(), C.byref(inp.arr), C.byref(inp.sch), o, s, C.byref(scalar)), device=device)
        got[device] = result(out, osch, device)
        assert inp.count.calls == 1 and scalar.value == 0
        inp.close()
        check_launches(f"expr[{expr}]/{'device' if device else 'host'}", n)
    assert got[True].equals(got[False])
    assert got[False].column(0).to_pylist() == (rb.column(2) if expr == "sensor" else pa.compute.add(rb.column(1), 1)).to_pylist()
