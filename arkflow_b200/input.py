"""Host-side mirror of the two reference inputs that produce their batches on the device (csrc/inputs.cu).

    trait Input { connect, read, close }   → class Input          (core/input/mod.rs)
    GenerateInput                          → class GenerateInput  (plugin/input/generate.rs:26-96)
    FileInput (json / csv / avro / arrow)  → class FileInput      (plugin/input/file.rs:395-455)
    InputConfig::build                     → build_input(cfg)

read() returns (MessageBatch, NoopAck) like the reference; read_device() leaves the batch in HBM.  End of input is
ArkError(kind "EOF"), as Error::EOF in the reference.  All work goes through the C ABI; there is no CPU path.
"""
from __future__ import annotations

import ctypes as C
import json
from typing import Optional

from . import _lib as L
from . import arrow_ffi as F
from .buffer import NoopAck
from .processor import ArkError, MessageBatch, _check


class Input:
    TYPE = ""

    def __init__(self, config: Optional[dict], name: Optional[str] = None):
        self.input_name = name
        h = C.c_void_p()
        cfg = None if config is None else json.dumps(config).encode()
        _check(L.lib().ark_input_create(self.TYPE.encode(), cfg, C.byref(h)))
        self._h = h

    def connect(self) -> None:
        _check(L.lib().ark_input_connect(self._h))

    def read(self):
        out_arr, out_sch = L.ArrowArray(), L.ArrowSchema()
        _check(L.lib().ark_input_read(self._h, C.byref(out_arr), C.byref(out_sch)))
        rb = F.import_record_batch(out_arr, out_sch)
        return MessageBatch(rb, self.input_name), NoopAck()  # generate.rs:92-93, file.rs:447-450

    def read_device(self):
        out_dev, out_sch = L.ArrowDeviceArray(), L.ArrowSchema()
        _check(L.lib().ark_input_read_device(self._h, C.byref(out_dev), C.byref(out_sch)))
        return F.DeviceBatch.adopt(out_dev, out_sch)

    def close(self) -> None:
        _check(L.lib().ark_input_close(self._h))

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                L.lib().ark_input_destroy(self._h)
                self._h = None
        except Exception:
            pass


class GenerateInput(Input):
    """`type: generate` {context, interval, count?, batch_size?}."""

    TYPE = "generate"


class FileInput(Input):
    """`type: file` {input_type: {type: json | csv | avro | arrow, path}, query?: {query, table?}, batch_size?}.

    `avro`: object container files with codec null or snappy, decoded on the GPU.  The top-level record's fields may be
    null, boolean, int, long, float, double, bytes or string, or a [null, T] / [T, null] union of one of these: Arrow
    Null, Boolean, Int32, Int64, Float32, Float64, Binary, Utf8, nullable only for unions.  Other schemas and codecs
    raise Unsupported from connect(); malformed data raises Process naming the first failing record and its block's
    file offset (structural damage already from connect()).  SQL `query` over Int32 / Float32 columns is Unsupported.

    `arrow`: Arrow IPC files (the footer-indexed file format, current or pre-0.15 message prefixes) with uncompressed or
    LZ4_FRAME bodies, read on the GPU.  Fields may be Null, Boolean, Int32, Int64, UInt32, UInt64, Float32, Float64,
    Utf8 or Binary, nullable or not; every other type (dictionary-encoded, nested, Large / View, Int8 / Int16, temporal,
    decimal), a big-endian schema and a ZSTD body raise Unsupported from connect(), which reads all metadata before the
    device is touched.  Structural damage (magic, footer, ranges, sizes, NULLs in a non-nullable field) raises Process
    from connect(); bad body bytes (LZ4 frames, offsets, UTF-8, a null count that differs from its bitmap) fail the
    read that first touches the record batch, naming the batch, column and row.  Batches cut through record batches;
    one that lies inside a single record batch is a view of the file in HBM.  A `query` that reads an Int32, UInt32,
    UInt64 or Float32 column raises Unsupported, as the sql processor does.  Parquet raises Unsupported.
    """

    TYPE = "file"


_INPUTS = {"generate": GenerateInput, "file": FileInput}


def build_input(config: dict) -> Input:
    """InputConfig::build: {"type": ..., "name"?: ..., <flattened config>}."""
    cfg = dict(config)
    kind = cfg.pop("type", None)
    name = cfg.pop("name", None)
    if kind not in _INPUTS:
        raise ArkError(L.ARK_ERR_CONFIG, f"Unknown input type: {kind}")
    return _INPUTS[kind](cfg if cfg else None, name)
