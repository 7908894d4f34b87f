"""Arrow C Data Interface glue between pyarrow / torch and the C ABI.

Host batches are `pyarrow.RecordBatch`es exported with `_export_to_c` (the same mechanism the
reference's python processor uses, crates/arkflow-plugin/src/processor/python.rs:52,67).
Device batches (`DeviceBatch`) are ArrowDeviceArray structs whose buffers are torch CUDA tensors;
torch is only the owner of device memory here.
"""
from __future__ import annotations

import ctypes as C
import itertools
from typing import Optional

import pyarrow as pa

from . import _lib as L

# ---------------------------------------------------------------------------------------------
# host
# ---------------------------------------------------------------------------------------------


def export_record_batch(rb: pa.RecordBatch):
    """pyarrow.RecordBatch → (ArrowArray, ArrowSchema) ctypes structs (ownership: the structs)."""
    arr, sch = L.ArrowArray(), L.ArrowSchema()
    rb._export_to_c(C.addressof(arr), C.addressof(sch))
    return arr, sch


def import_record_batch(arr: L.ArrowArray, sch: L.ArrowSchema) -> pa.RecordBatch:
    return pa.RecordBatch._import_from_c(C.addressof(arr), C.addressof(sch))


def release_schema(sch: L.ArrowSchema):
    if sch.release:
        L.RELEASE_SCHEMA(sch.release)(C.byref(sch))


def release_array(arr: L.ArrowArray):
    if arr.release:
        L.RELEASE_ARRAY(arr.release)(C.byref(arr))


# ---------------------------------------------------------------------------------------------
# device
# ---------------------------------------------------------------------------------------------

_FMT = {"int64": b"l", "float64": b"g", "utf8": b"u", "binary": b"z", "bool": b"b", "null": b"n",
        "int32": b"i", "uint32": b"I", "uint64": b"L", "float32": b"f"}
_FMT_INV = {v: k for k, v in _FMT.items()}
# fixed-width column types: (array-interface / numpy typestr, bytes per value, torch dtype name, pyarrow type factory).
# int32 / uint32 / uint64 / float32 columns come from protobuf_to_arrow and feed arrow_to_protobuf.
_FIXED = {"int64": ("<i8", 8, "int64", pa.int64), "float64": ("<f8", 8, "float64", pa.float64),
          "int32": ("<i4", 4, "int32", pa.int32), "uint32": ("<u4", 4, "uint32", pa.uint32),
          "uint64": ("<u8", 8, "uint64", pa.uint64), "float32": ("<f4", 4, "float32", pa.float32)}


class DeviceColumn:
    """One column resident in HBM.  `data`/`offsets`/`validity` are torch CUDA tensors (or None).  `offset` is the
    Arrow offset of a slice: the column's rows start at element / bit `offset` of those buffers."""

    def __init__(self, name: str, dtype: str, length: int, data, offsets=None, validity=None,
                 null_count: int = 0, nullable: bool = True, offset: int = 0):
        assert dtype in _FMT, dtype
        self.name, self.dtype, self.length = name, dtype, int(length)
        self.data, self.offsets, self.validity = data, offsets, validity
        self.null_count, self.nullable = null_count, nullable
        self.offset = int(offset)


class _LazyBytes:
    """The data buffer of a var-len column adopted from C: its size is offsets[n], which lives on the
    device; reading it costs a synchronising copy, so it is deferred until somebody touches the bytes."""

    def __init__(self, ptr, offsets, n, owner):
        self._ptr, self._offsets, self._n, self._owner, self._t = ptr, offsets, n, owner, None

    def tensor(self):
        import torch

        if self._t is None:
            nbytes = int(self._offsets[-1].item()) if self._n > 0 else 0
            if not self._ptr or nbytes <= 0:
                self._t = torch.empty(0, dtype=torch.uint8, device="cuda")
            else:
                self._t = torch.as_tensor(_CudaPtr(self._ptr, nbytes, "|u1", 1, self._owner), device="cuda")
        return self._t

    def data_ptr(self):
        return self._ptr or 0

    def numel(self):
        return self.tensor().numel()

    def cpu(self):
        return self.tensor().cpu()

    def __getitem__(self, item):
        return self.tensor()[item]

    @property
    def device(self):
        return self._offsets.device


class _CudaPtr:
    """Zero-copy view of foreign device memory for torch.as_tensor (via __cuda_array_interface__)."""

    def __init__(self, ptr: int, nbytes: int, typestr: str, itemsize: int, owner):
        self.__cuda_array_interface__ = {
            "shape": (nbytes // itemsize,), "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None,
        }
        self._owner = owner


_live_exports: dict[int, object] = {}


def _keepalive_release_array(ptr):
    arr = ptr.contents
    for i in range(arr.n_children):  # Arrow: a parent's release releases its children
        child = arr.children[i].contents
        if child.release:
            _live_exports.pop(child.private_data, None)
            child.release = None
    _live_exports.pop(arr.private_data, None)
    arr.release = None


def _keepalive_release_schema(ptr):
    sch = ptr.contents
    for i in range(sch.n_children):
        child = sch.children[i].contents
        if child.release:
            _live_exports.pop(child.private_data, None)
            child.release = None
    _live_exports.pop(sch.private_data, None)
    sch.release = None


_REL_ARR = L.RELEASE_ARRAY(_keepalive_release_array)
_REL_SCH = L.RELEASE_SCHEMA(_keepalive_release_schema)
_next_token = itertools.count(1)  # next() on a count is atomic under the GIL: worker threads never share a token


def _token(obj) -> int:
    t = next(_next_token)
    _live_exports[t] = obj
    return t


class DeviceBatch:
    """A RecordBatch resident in HBM (list of DeviceColumn)."""

    def __init__(self, columns: list[DeviceColumn], num_rows: int, owner=None):
        self._columns, self.num_rows, self._owner = columns, int(num_rows), owner

    # --- Python → C (we own the memory; the release callback just drops our references) ---
    def export(self):
        """(ArrowDeviceArray, ArrowSchema) for one C-ABI call.  The struct tree is built once per batch
        and re-armed on every export (the callee's release only drops our keep-alive tokens)."""
        import torch

        # the library runs on its own streams: whatever torch / NCCL queued on the current stream to
        # produce these tensors must have completed before the pointers are handed over.  A batch adopted
        # from the library itself was complete when the call that produced it returned.
        if not getattr(self, "_library_made", False):
            torch.cuda.current_stream().synchronize()
        cache = getattr(self, "_export_cache", None)
        if cache is None:
            n = len(self.columns)
            dev = L.ArrowDeviceArray()
            sch = L.ArrowSchema()
            child_arrs = (L.ArrowArray * max(n, 1))()
            child_ptrs = (C.POINTER(L.ArrowArray) * max(n, 1))()
            child_schs = (L.ArrowSchema * max(n, 1))()
            child_sptrs = (C.POINTER(L.ArrowSchema) * max(n, 1))()
            keep = [self]
            for i, c in enumerate(self.columns):
                if c.dtype == "null":
                    bufs = []
                else:
                    first = c.offsets if c.dtype in ("utf8", "binary") else c.data
                    bufs = [c.validity.data_ptr() if c.validity is not None else None,
                            first.data_ptr() if first is not None else None]
                    if c.dtype in ("utf8", "binary"):
                        bufs.append((c.data.data_ptr() or None) if c.data is not None else None)
                barr = (C.c_void_p * max(len(bufs), 1))(*bufs)
                a = child_arrs[i]
                a.length, a.null_count, a.offset = c.length, (c.null_count if c.validity is not None else 0), c.offset
                a.n_buffers, a.n_children = len(bufs), 0
                a.buffers = C.cast(barr, C.POINTER(C.c_void_p))
                child_ptrs[i] = C.pointer(a)
                s = child_schs[i]
                nm = c.name.encode()
                s.format, s.name, s.metadata = _FMT[c.dtype], nm, None
                s.flags = 2 if c.nullable else 0
                s.n_children = 0
                child_sptrs[i] = C.pointer(s)
                keep.append((barr, nm, c))
            top_bufs = (C.c_void_p * 1)(None)
            dev.array.length, dev.array.null_count, dev.array.offset = self.num_rows, 0, 0
            dev.array.n_buffers, dev.array.n_children = 1, n
            dev.array.buffers = C.cast(top_bufs, C.POINTER(C.c_void_p))
            dev.array.children = C.cast(child_ptrs, C.POINTER(C.POINTER(L.ArrowArray)))
            dev.device_id = torch.cuda.current_device()
            dev.device_type = L.ARROW_DEVICE_CUDA
            dev.sync_event = None
            sch.format, sch.name, sch.metadata, sch.flags = b"+s", b"", None, 0
            sch.n_children = n
            sch.children = C.cast(child_sptrs, C.POINTER(C.POINTER(L.ArrowSchema)))
            cache = (dev, sch, child_arrs, child_schs, (top_bufs, child_ptrs, child_sptrs, keep), n)
            self._export_cache = cache
        dev, sch, child_arrs, child_schs, keep, n = cache
        if dev.array.release or sch.release:
            # a previous export is still armed (concurrent use of one batch): build a private copy
            clone = DeviceBatch(self.columns, self.num_rows, self._owner)
            return clone.export()
        rel_a, rel_s = C.cast(_REL_ARR, C.c_void_p), C.cast(_REL_SCH, C.c_void_p)
        for i in range(n):
            child_arrs[i].release = rel_a
            child_arrs[i].private_data = None
            child_schs[i].release = rel_s
            child_schs[i].private_data = None
        dev.array.release = rel_a
        dev.array.private_data = _token(cache)
        sch.release = rel_s
        sch.private_data = _token(cache)
        return dev, sch

    # --- C → Python (the library owns the memory; we hold the struct and release it on close) ---
    @staticmethod
    def adopt(dev: L.ArrowDeviceArray, sch: L.ArrowSchema) -> "DeviceBatch":
        """Wrap a callee-allocated result.  Columns (torch views of the device buffers) are built lazily."""
        b = DeviceBatch.__new__(DeviceBatch)
        b.num_rows = dev.array.length
        b._owner = _CResult(dev, sch)
        b._columns = None
        b._library_made = True
        return b

    @property
    def columns(self):
        if self._columns is None:
            self._columns = self._materialise()
        return self._columns

    @columns.setter
    def columns(self, v):
        self._columns = v
        self._library_made = False  # torch may still be producing the new tensors: export() synchronises again
        self._export_cache = None

    def _materialise(self):
        import torch

        owner = self._owner
        dev, sch = owner.dev, owner.sch
        cols = []
        for i in range(dev.array.n_children):
            a = dev.array.children[i].contents
            s = sch.children[i].contents
            dtype = _FMT_INV[s.format]
            n = a.length

            def view(idx, nbytes, typestr, itemsize, tdtype):
                ptr = a.buffers[idx]
                if not ptr or nbytes <= 0:
                    return torch.empty(0, dtype=tdtype, device="cuda")
                return torch.as_tensor(_CudaPtr(ptr, nbytes, typestr, itemsize, owner), device="cuda")

            if dtype == "null":
                cols.append(DeviceColumn(s.name.decode(), dtype, n, None, None, None, null_count=n, nullable=True))
                continue
            validity = view(0, (n + 7) // 8, "|u1", 1, torch.uint8) if (a.n_buffers > 0 and a.buffers[0]) else None
            offsets = None
            if dtype in _FIXED:
                ts, w, tname, _ = _FIXED[dtype]
                data = view(1, n * w, ts, w, getattr(torch, tname))
            elif dtype == "bool":
                data = view(1, (n + 7) // 8, "|u1", 1, torch.uint8)
            else:
                offsets = view(1, (n + 1) * 4, "<i4", 4, torch.int32)
                ptr2 = a.buffers[2] if a.n_buffers > 2 else None
                data = _LazyBytes(ptr2, offsets, n, owner)  # resolved on first use (needs one device read)
            cols.append(DeviceColumn(s.name.decode(), dtype, n, data, offsets, validity,
                                     null_count=a.null_count, nullable=bool(s.flags & 2)))
        return cols

    def to_arrow(self) -> pa.RecordBatch:
        """Copy to host as a pyarrow RecordBatch (tests / debugging)."""
        arrays, fields = [], []
        for c in self.columns:
            n = c.length
            vbuf = pa.py_buffer(c.validity.cpu().numpy().tobytes()) if c.validity is not None and c.validity.numel() else None
            nulls = c.null_count if vbuf is not None else 0
            if c.dtype == "null":
                arrays.append(pa.nulls(n))
                fields.append(pa.field(c.name, pa.null(), nullable=True))
                continue
            off = getattr(c, "offset", 0)
            if c.dtype in _FIXED:
                t = _FIXED[c.dtype][3]()
                arr = pa.Array.from_buffers(t, n, [vbuf, pa.py_buffer(c.data.cpu().numpy().tobytes())], null_count=nulls, offset=off)
            elif c.dtype == "bool":
                arr = pa.Array.from_buffers(pa.bool_(), n, [vbuf, pa.py_buffer(c.data.cpu().numpy().tobytes())], null_count=nulls, offset=off)
            else:
                t = pa.utf8() if c.dtype == "utf8" else pa.binary()
                arr = pa.Array.from_buffers(t, n, [vbuf, pa.py_buffer(c.offsets.cpu().numpy().tobytes()),
                                                   pa.py_buffer(c.data.cpu().numpy().tobytes())], null_count=nulls, offset=off)
            arrays.append(arr)
            fields.append(pa.field(c.name, arr.type, nullable=c.nullable))
        return pa.RecordBatch.from_arrays(arrays, schema=pa.schema(fields))

    @staticmethod
    def from_arrow(rb: pa.RecordBatch, device="cuda", keep_offsets: bool = False) -> "DeviceBatch":
        """Upload a pyarrow RecordBatch with torch (test helper; the product H2D path is the C ABI).

        Sliced columns are normalised to offset 0, unless keep_offsets: then each sliced column's parent buffers are
        uploaded whole and exported with the slice's Arrow offset, as a producer that slices device batches (arrow-rs
        RecordBatch::slice) hands them over: data pointers not 16-byte aligned, offsets[0] != 0, validity and Boolean
        bits that start inside a byte."""
        import numpy as np
        import torch

        def up(buf, np_dtype, count=None, offset_bytes=0):
            if buf is None:
                return None
            a = np.frombuffer(buf, dtype=np.uint8)[offset_bytes:]
            a = a.view(np_dtype) if np_dtype != np.uint8 else a
            if count is not None:
                a = a[:count]
            return torch.from_numpy(a.copy()).to(device)

        cols = []
        for name, arr in zip(rb.schema.names, rb.columns):
            f = rb.schema.field(name)
            if arr.offset != 0 and not keep_offsets:
                arr = pa.concat_arrays([arr])  # normalise slices
            off = arr.offset
            bufs = arr.buffers()
            n = len(arr)
            validity = up(bufs[0], np.uint8) if (bufs[0] is not None and arr.null_count) else None
            fixed = [k for k, v in _FIXED.items() if arr.type == v[3]()]
            if fixed:
                dt = fixed[0]
                data = up(bufs[1], np.dtype(_FIXED[dt][0]), off + n)
                cols.append(DeviceColumn(name, dt, n, data, None, validity, arr.null_count, f.nullable, off))
            elif pa.types.is_boolean(arr.type):
                cols.append(DeviceColumn(name, "bool", n, up(bufs[1], np.uint8), None, validity, arr.null_count, f.nullable, off))
            elif pa.types.is_string(arr.type) or pa.types.is_binary(arr.type):
                dt = "utf8" if pa.types.is_string(arr.type) else "binary"
                offsets = up(bufs[1], np.int32, off + n + 1)
                data = up(bufs[2], np.uint8) if bufs[2] is not None else torch.empty(0, dtype=torch.uint8, device=device)
                cols.append(DeviceColumn(name, dt, n, data, offsets, validity, arr.null_count, f.nullable, off))
            else:
                raise TypeError(f"unsupported Arrow type for device upload: {arr.type}")
        return DeviceBatch(cols, rb.num_rows)

    def close(self):
        if self._owner is not None:
            self._owner.close()
            self._owner = None


class _CResult:
    """Owns a callee-allocated ArrowDeviceArray + ArrowSchema; releases them exactly once."""

    def __init__(self, dev, sch):
        self.dev, self.sch = dev, sch
        self._open = True

    def close(self):
        if self._open:
            self._open = False
            release_array(self.dev.array)
            release_schema(self.sch)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
