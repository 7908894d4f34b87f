"""The C ABI's call contract on the paths that fail before any CUDA call: a processor handle of the wrong type (or NULL), a
NULL buffer / batch processor, an input that was already released and a count below one are rejected with ARK_ERR_PROCESS
and the exact message; the entry point fills no output; and a moved-in input is released exactly once, by the callee."""
import ctypes as C
import json

import pytest

from arkflow_b200 import _lib as L

PROTO = 'syntax = "proto3";\npackage pkg;\nmessage M { int64 timestamp = 1; double value = 2; string sensor = 3; }\n'
TYPES = ("sql", "json_to_arrow", "arrow_to_json", "protobuf_to_arrow", "arrow_to_protobuf")
HOST_PROCESS = {t: f"ark_{t}_process" for t in TYPES}
DEVICE_PROCESS = {t: f"ark_{t}_process_device" for t in TYPES}


def handle_message(t):
    return f"handle is not {'an' if t[0] in 'aeiou' else 'a'} {t} processor"


class Input:
    """A one-row struct array with no columns whose release callback counts its calls."""

    def __init__(self, device=False):
        self.calls = 0
        self._cb = L.RELEASE_ARRAY(self._release)
        self._bufs = (C.c_void_p * 1)(None)
        self.dev = L.ArrowDeviceArray()
        self.arr = self.dev.array if device else L.ArrowArray()
        for a in (self.dev.array, self.arr):
            a.length, a.n_buffers, a.buffers = 1, 1, self._bufs
            a.release = C.cast(self._cb, C.c_void_p).value
        self.dev.device_type = L.ARROW_DEVICE_CUDA
        self.device = device
        self.schema = L.ArrowSchema(format=b"+s", name=b"")

    def _release(self, ptr):
        self.calls += 1
        ptr.contents.release = None

    def released(self):
        """Marks the input released, as a consumer that had already taken it would leave it."""
        self.dev.array.release = None
        self.arr.release = None
        return self

    def ref(self):
        return C.byref(self.dev) if self.device else C.byref(self.arr)

    def moved(self):
        return (self.dev.array if self.device else self.arr).release is None


@pytest.fixture(scope="module")
def handles(lib, tmp_path_factory):
    d = tmp_path_factory.mktemp("proto")
    (d / "m.proto").write_text(PROTO)
    pb = json.dumps({"proto_inputs": [str(d)], "message_type": "pkg.M"}).encode()
    configs = {"sql": b'{"query": "SELECT * FROM flow"}', "json_to_arrow": b"{}", "arrow_to_json": b"{}",
               "protobuf_to_arrow": pb, "arrow_to_protobuf": pb}
    hs = {}
    for t in TYPES:
        h = C.c_void_p()
        assert getattr(lib, f"ark_{t}_create")(configs[t], C.byref(h)) == L.ARK_OK, lib.ark_last_error()
        hs[t] = h
    yield hs
    for h in hs.values():
        lib.ark_proc_destroy(h)


def expect(lib, status, message):
    assert status == L.ARK_ERR_PROCESS
    assert lib.ark_last_error().decode() == message


def outputs(device):
    return (L.ArrowDeviceArray() if device else L.ArrowArray()), L.ArrowSchema()


def out_release(out):
    return out.array.release if isinstance(out, L.ArrowDeviceArray) else out.release


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("want,given", [(w, g) for w in TYPES for g in TYPES + (None,) if g != w])
def test_processor_rejects_a_handle_of_another_type(lib, handles, want, given, device):
    inp = Input(device)
    out, out_schema = outputs(device)
    fn = getattr(lib, (DEVICE_PROCESS if device else HOST_PROCESS)[want])
    status = fn(handles[given] if given else None, inp.ref(), C.byref(inp.schema), C.byref(out), C.byref(out_schema))
    expect(lib, status, handle_message(want))
    assert out_release(out) is None and out_schema.release is None
    assert inp.moved() and inp.calls == 1


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("t", TYPES)
def test_processor_rejects_a_released_input(lib, handles, t, device):
    inp = Input(device).released()
    out, out_schema = outputs(device)
    fn = getattr(lib, (DEVICE_PROCESS if device else HOST_PROCESS)[t])
    expect(lib, fn(handles[t], inp.ref(), C.byref(inp.schema), C.byref(out), C.byref(out_schema)), "input array already released")
    assert out_release(out) is None and inp.calls == 0


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("given", [t for t in TYPES if t != "sql"] + [None])
def test_sql_tables_rejects_a_handle_of_another_type(lib, handles, given, device):
    ins = [Input(device), Input(device)]
    Arr = L.ArrowDeviceArray if device else L.ArrowArray
    arrs = (Arr * 2)(*[i.dev if device else i.arr for i in ins])
    schs = (L.ArrowSchema * 2)(ins[0].schema, ins[1].schema)
    names = (C.c_char_p * 2)(b"a", b"b")
    out, out_schema = outputs(device)
    fn = lib.ark_sql_process_tables_device if device else lib.ark_sql_process_tables
    status = fn(handles[given] if given else None, 2, names, arrs, schs, C.byref(out), C.byref(out_schema))
    expect(lib, status, handle_message("sql"))
    assert out_release(out) is None
    assert all(a.release is None for a in ((x.array for x in arrs) if device else arrs))
    assert [i.calls for i in ins] == [1, 1]


@pytest.mark.parametrize("given", [t for t in TYPES if t != "sql"] + [None])
def test_sql_device_entry_points_reject_a_handle_of_another_type(lib, handles, given):
    h = handles[given] if given else None
    parts = (C.c_int64 * 2)()
    inp = Input(True)
    out, out_schema = outputs(True)
    expect(lib, lib.ark_sql_partial_aggregate_device(h, inp.ref(), C.byref(inp.schema), 2, C.byref(out), C.byref(out_schema), parts),
           handle_message("sql"))
    assert inp.moved() and inp.calls == 1 and out.array.release is None
    inp = Input(True)
    expect(lib, lib.ark_sql_final_aggregate_device(h, inp.ref(), C.byref(inp.schema), C.byref(out), C.byref(out_schema)), handle_message("sql"))
    assert inp.moved() and inp.calls == 1 and out.array.release is None
    inp = Input(True)
    expect(lib, lib.ark_sql_group_by_push_device(h, None, inp.ref(), C.byref(inp.schema)), handle_message("sql"))
    assert inp.moved() and inp.calls == 1
    expect(lib, lib.ark_sql_group_by_merge_device(h, None, C.byref(out), C.byref(out_schema)), handle_message("sql"))
    assert out.array.release is None


@pytest.mark.parametrize("n_parts", [0, -1])
def test_partial_aggregate_rejects_fewer_than_one_part(lib, handles, n_parts):
    inp = Input(True)
    out, out_schema = outputs(True)
    parts = (C.c_int64 * 1)()
    status = lib.ark_sql_partial_aggregate_device(handles["sql"], inp.ref(), C.byref(inp.schema), n_parts, C.byref(out), C.byref(out_schema), parts)
    expect(lib, status, "n_parts must be >= 1")
    assert inp.moved() and inp.calls == 1 and out.array.release is None


def test_sql_device_entry_points_reject_a_released_input(lib, handles):
    h = handles["sql"]
    out, out_schema = outputs(True)
    parts = (C.c_int64 * 2)()
    inp = Input(True).released()
    expect(lib, lib.ark_sql_partial_aggregate_device(h, inp.ref(), C.byref(inp.schema), 2, C.byref(out), C.byref(out_schema), parts),
           "input array already released")
    expect(lib, lib.ark_sql_final_aggregate_device(h, inp.ref(), C.byref(inp.schema), C.byref(out), C.byref(out_schema)),
           "input array already released")
    expect(lib, lib.ark_hash_partition_device(inp.ref(), C.byref(inp.schema), b"k", 2, C.byref(out), C.byref(out_schema), parts),
           "input array already released")
    blob, size = (C.c_uint8 * 64)(), C.c_int64()
    expect(lib, lib.ark_ipc_export_device(inp.ref(), C.byref(inp.schema), blob, 64, C.byref(size)), "input array already released")
    assert out.array.release is None and inp.calls == 0


def test_group_by_push_needs_a_connected_exchange(lib, handles):
    inp = Input(True)
    expect(lib, lib.ark_sql_group_by_push_device(handles["sql"], None, inp.ref(), C.byref(inp.schema)), "exchange context is not connected")
    assert inp.moved() and inp.calls == 1


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_expr_evaluate_rejects_null_and_released_arguments(lib, device):
    fn = lib.ark_expr_evaluate_device if device else lib.ark_expr_evaluate
    out, out_schema = outputs(device)
    inp = Input(device)
    expect(lib, fn(None, inp.ref(), C.byref(inp.schema), C.byref(out), C.byref(out_schema), None), "null argument")
    assert inp.moved() and inp.calls == 1 and out_release(out) is None
    inp = Input(device)
    expect(lib, fn(b"value + 1", inp.ref(), C.byref(inp.schema), None, C.byref(out_schema), None), "null argument")
    assert inp.moved() and inp.calls == 1
    inp = Input(device).released()
    expect(lib, fn(b"value + 1", inp.ref(), C.byref(inp.schema), C.byref(out), C.byref(out_schema), None), "input array already released")
    assert out_release(out) is None and inp.calls == 0


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
@pytest.mark.parametrize("n", [0, -1])
def test_concat_needs_a_batch(lib, device, n):
    out, out_schema = outputs(device)
    fn = lib.ark_concat_batches_device if device else lib.ark_concat_batches
    expect(lib, fn(n, None, None, C.byref(out), C.byref(out_schema)), "Merge batches failed: no batches")
    assert out_release(out) is None


def test_buffer_and_batch_entry_points_reject_null_handles(lib):
    for device, fn in ((False, lib.ark_buffer_write), (True, lib.ark_buffer_write_device)):
        inp = Input(device)
        expect(lib, fn(None, inp.ref(), C.byref(inp.schema), b"in", 7), "null buffer")
        assert inp.moved() and inp.calls == 1
    acks, n_acks = (C.c_uint64 * 4)(), C.c_int64()
    for device, fn in ((False, lib.ark_buffer_read), (True, lib.ark_buffer_read_device)):
        out, out_schema = outputs(device)
        expect(lib, fn(None, C.byref(out), C.byref(out_schema), acks, 4, C.byref(n_acks)), "null buffer")
        assert out_release(out) is None
    inp = Input()
    out, out_schema = outputs(False)
    expect(lib, lib.ark_batch_process(None, inp.ref(), C.byref(inp.schema), C.byref(out), C.byref(out_schema)), "null batch processor")
    assert inp.moved() and inp.calls == 1 and out.release is None
    expect(lib, lib.ark_batch_flush(None, C.byref(out), C.byref(out_schema)), "null batch processor")
    assert out.release is None


def test_buffer_and_batch_entry_points_reject_a_released_input(lib):
    buf, bat = C.c_void_p(), C.c_void_p()
    assert lib.ark_buffer_create(b"memory", b'{"capacity": 4, "timeout": "1s"}', None, C.byref(buf)) == L.ARK_OK, lib.ark_last_error()
    assert lib.ark_batch_create(b'{"count": 4, "timeout_ms": 1000}', C.byref(bat)) == L.ARK_OK, lib.ark_last_error()
    try:
        for device, fn in ((False, lib.ark_buffer_write), (True, lib.ark_buffer_write_device)):
            inp = Input(device).released()
            expect(lib, fn(buf, inp.ref(), C.byref(inp.schema), b"in", 7), "input array already released")
        inp = Input().released()
        out, out_schema = outputs(False)
        expect(lib, lib.ark_batch_process(bat, inp.ref(), C.byref(inp.schema), C.byref(out), C.byref(out_schema)),
               "input array already released")
        assert out.release is None
    finally:
        lib.ark_buffer_close(buf)
        lib.ark_buffer_destroy(buf)
        lib.ark_batch_destroy(bat)


@pytest.mark.parametrize("device", [False, True], ids=["host", "device"])
def test_input_read_rejects_a_null_input(lib, device):
    out, out_schema = outputs(device)
    fn = lib.ark_input_read_device if device else lib.ark_input_read
    expect(lib, fn(None, C.byref(out), C.byref(out_schema)), "null argument")
    assert out_release(out) is None


def test_ipc_concat_slices_rejects_no_sources(lib):
    out, out_schema = outputs(True)
    one = (C.c_int64 * 1)()
    blobs = (C.POINTER(C.c_uint8) * 1)()
    expect(lib, lib.ark_ipc_concat_slices_device(0, blobs, one, one, one, C.byref(out), C.byref(out_schema)), "null argument")
    expect(lib, lib.ark_ipc_concat_slices_device(1, None, one, one, one, C.byref(out), C.byref(out_schema)), "null argument")
    assert out.array.release is None
