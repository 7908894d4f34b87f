"""Host-side mirror of the reference's Processor plugin surface for the hot path.

Same names, configuration keys and error behaviour as the reference so that the parity tests read
like the reference's own (crates/arkflow-plugin/src/processor/sql.rs:250-426, json.rs:160-343, protobuf.rs:246-468):

    trait Processor        → class Processor            (core/processor/mod.rs:32-79)
    ProcessResult          → class ProcessResult        (core/lib.rs:179-187)
    MessageBatch           → class MessageBatch         (core/lib.rs:236-377)
    ProcessorConfig.build  → build_processor(cfg)       (core/processor/mod.rs:93-104)
    register_processor_builder                          (core/processor/mod.rs:116-129)

All compute goes through the C ABI (libarkflow_b200.so → sm_90a kernels).  There is no CPU path.
"""
from __future__ import annotations

import ctypes as C
import json
from typing import Callable, Optional

import pyarrow as pa

from . import _lib as L
from . import arrow_ffi as F

DEFAULT_BINARY_VALUE_FIELD = "__value__"  # core/lib.rs:46
DEFAULT_RECORD_BATCH = 8192  # core/lib.rs:47


class ArkError(Exception):
    """Mirror of arkflow_core::Error (core/lib.rs:66-110); `kind` names the variant."""

    KINDS = {L.ARK_ERR_CONFIG: "Config", L.ARK_ERR_PROCESS: "Process", L.ARK_ERR_UNSUPPORTED: "Unsupported",
             L.ARK_ERR_SERIALIZATION: "Serialization", L.ARK_ERR_CUDA: "Process", L.ARK_ERR_EOF: "EOF"}

    def __init__(self, code: int, message: str):
        super().__init__(message)
        self.code, self.kind, self.message = code, self.KINDS.get(code, "Process"), message


def _check(status: int):
    if status != L.ARK_OK:
        raise ArkError(status, (L.lib().ark_last_error() or b"").decode("utf-8", "replace"))


class MessageBatch:
    """RecordBatch + optional input name (core/lib.rs:236-240)."""

    def __init__(self, record_batch: pa.RecordBatch, input_name: Optional[str] = None):
        self.record_batch, self.input_name = record_batch, input_name

    @staticmethod
    def new_arrow(rb: pa.RecordBatch) -> "MessageBatch":
        return MessageBatch(rb)

    @staticmethod
    def new_binary(content: list[bytes], field_name: Optional[str] = None) -> "MessageBatch":
        """core/lib.rs:243-270: one non-null Binary column named __value__."""
        name = field_name or DEFAULT_BINARY_VALUE_FIELD
        arr = pa.array(content, type=pa.binary())
        return MessageBatch(pa.RecordBatch.from_arrays([arr], schema=pa.schema([pa.field(name, pa.binary(), nullable=False)])))

    def new_binary_with_origin(self, content: list[bytes]) -> "MessageBatch":
        """core/lib.rs:280-302: original columns + a trailing non-null Binary __value__ column."""
        rb = self.record_batch
        fields = list(rb.schema) + [pa.field(DEFAULT_BINARY_VALUE_FIELD, pa.binary(), nullable=False)]
        cols = list(rb.columns) + [pa.array(content, type=pa.binary())]
        return MessageBatch(pa.RecordBatch.from_arrays(cols, schema=pa.schema(fields)))

    def to_binary(self, name: str) -> list[bytes]:
        """core/lib.rs:355-371."""
        if name not in self.record_batch.schema.names:
            raise ArkError(L.ARK_ERR_PROCESS, "not found column")
        col = self.record_batch.column(name)
        if col.type != pa.binary():
            raise ArkError(L.ARK_ERR_PROCESS, "not support data type")
        return [v.as_py() for v in col if v.is_valid]

    def is_empty(self) -> bool:
        return self.record_batch.num_rows == 0

    def __len__(self):
        return self.record_batch.num_rows

    @property
    def num_rows(self):
        return self.record_batch.num_rows

    @property
    def schema(self):
        return self.record_batch.schema


class ProcessResult:
    """core/lib.rs:179-187: Single(batch) | Multiple(batches) | None."""

    def __init__(self, kind: str, batches: list):
        self.kind, self.batches = kind, batches

    @staticmethod
    def single(b):
        return ProcessResult("Single", [b])

    @staticmethod
    def none():
        return ProcessResult("None", [])

    def is_none(self):
        return self.kind == "None"

    def is_empty(self):  # ProcessResult::is_empty, core/lib.rs
        return len(self.batches) == 0

    def into_vec(self):
        return list(self.batches)

    def __len__(self):
        return len(self.batches)


class Processor:
    """trait Processor (core/processor/mod.rs:32-79)."""

    def process(self, msg_batch) -> ProcessResult:  # pragma: no cover - interface
        raise NotImplementedError

    def close(self) -> None:
        pass


class _NativeProcessor(Processor):
    _create: str = ""
    _process: str = ""
    _process_device: str = ""

    def __init__(self, config: Optional[dict]):
        lib = L.lib()
        handle = C.c_void_p()
        cfg = None if config is None else json.dumps(config).encode()
        _check(getattr(lib, self._create)(cfg, C.byref(handle)))
        self._h = handle
        self.config = config

    def process(self, msg_batch) -> ProcessResult:
        if isinstance(msg_batch, F.DeviceBatch):
            out = self.process_device(msg_batch)
            return ProcessResult.none() if out is None else ProcessResult.single(out)
        mb = msg_batch if isinstance(msg_batch, MessageBatch) else MessageBatch(msg_batch)
        lib = L.lib()
        arr, sch = F.export_record_batch(mb.record_batch)
        out_arr, out_sch = L.ArrowArray(), L.ArrowSchema()
        try:
            status = getattr(lib, self._process)(self._h, C.byref(arr), C.byref(sch), C.byref(out_arr), C.byref(out_sch))
        finally:
            F.release_schema(sch)
            F.release_array(arr)  # no-op when the callee consumed it
        _check(status)
        if not out_arr.release:
            return ProcessResult.none()
        rb = F.import_record_batch(out_arr, out_sch)
        return ProcessResult.single(MessageBatch(rb, mb.input_name))

    def process_device(self, batch: F.DeviceBatch) -> Optional[F.DeviceBatch]:
        lib = L.lib()
        dev, sch = batch.export()
        out_dev, out_sch = L.ArrowDeviceArray(), L.ArrowSchema()
        try:
            status = getattr(lib, self._process_device)(self._h, C.byref(dev), C.byref(sch), C.byref(out_dev), C.byref(out_sch))
        finally:
            F.release_schema(sch)
            F.release_array(dev.array)
        _check(status)
        if not out_dev.array.release:
            return None
        return F.DeviceBatch.adopt(out_dev, out_sch)

    def close(self) -> None:
        if getattr(self, "_h", None):
            L.lib().ark_proc_close(self._h)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                L.lib().ark_proc_destroy(self._h)
                self._h = None
        except Exception:
            pass


class SqlProcessor(_NativeProcessor):
    """`type: sql` — crates/arkflow-plugin/src/processor/sql.rs:59-225.

    config: {"query": str, "table_name": str = "flow", "temporary_list": [...]?}
    """

    _create, _process, _process_device = "ark_sql_create", "ark_sql_process", "ark_sql_process_device"

    def __init__(self, config: Optional[dict], resource=None):
        # SqlProcessor::new (sql.rs:68-105): every configured temporary must exist in Resource
        self._temporaries = []
        if config and config.get("temporary_list"):
            from .expr import Expr

            known = getattr(resource, "temporary", None) or {}
            for t in config["temporary_list"]:
                for field in ("name", "table_name", "key"):
                    if field not in t:
                        raise ArkError(L.ARK_ERR_SERIALIZATION, f"missing field `{field}` (TemporaryConfig)")
                if t["name"] not in known:
                    raise ArkError(L.ARK_ERR_PROCESS, f"Temporary {t['name']} not found")
                self._temporaries.append((known[t["name"]], t["table_name"], Expr.from_config(t["key"])))
            config = dict(config, temporaries_resolved=True)
        super().__init__(config)

    def process(self, msg_batch) -> ProcessResult:
        if not self._temporaries or isinstance(msg_batch, F.DeviceBatch):
            return super().process(msg_batch)
        # execute_query with get_temporary_message_batch (sql.rs:108-186): evaluate each key on the batch,
        # ask the Temporary for its rows, register them next to the batch, run the query
        from .expr import ColumnarValue, evaluate_expr

        mb = msg_batch if isinstance(msg_batch, MessageBatch) else MessageBatch(msg_batch)
        if mb.num_rows == 0:
            return ProcessResult.none()  # sql.rs:211-213
        tables = {(self.config or {}).get("table_name") or "flow": mb.record_batch}
        for temporary, table_name, key in self._temporaries:
            if key.kind == "Value":
                cv = ColumnarValue.scalar_utf8(key.payload)
            else:
                try:
                    cv = evaluate_expr(key.payload, mb.record_batch)
                except ArkError as e:
                    raise ArkError(L.ARK_ERR_PROCESS, f"Evaluate expression failed: {e.message}")
            data = temporary.get([cv])
            if data is not None:
                tables[table_name] = data.record_batch if isinstance(data, MessageBatch) else data
        out = self.process_tables(tables)
        return ProcessResult.none() if out is None else ProcessResult.single(MessageBatch(out, mb.input_name))

    def process_tables(self, tables: dict[str, pa.RecordBatch]) -> Optional[pa.RecordBatch]:
        """JoinOperation's `ctx.sql(query)` over several registered tables (buffer/join.rs:92-118)."""
        lib = L.lib()
        n = len(tables)
        names = (C.c_char_p * n)(*[k.encode() for k in tables])
        arrs = (L.ArrowArray * n)()
        schs = (L.ArrowSchema * n)()
        for i, rb in enumerate(tables.values()):
            rb._export_to_c(C.addressof(arrs[i]), C.addressof(schs[i]))
        out_arr, out_sch = L.ArrowArray(), L.ArrowSchema()
        try:
            status = lib.ark_sql_process_tables(self._h, n, names, arrs, schs, C.byref(out_arr), C.byref(out_sch))
        finally:
            for i in range(n):
                F.release_schema(schs[i])
                F.release_array(arrs[i])
        _check(status)
        if not out_arr.release:
            return None
        return F.import_record_batch(out_arr, out_sch)


    def process_tables_device(self, tables: dict) -> Optional["F.DeviceBatch"]:
        lib = L.lib()
        n = len(tables)
        names = (C.c_char_p * n)(*[k.encode() for k in tables])
        devs = (L.ArrowDeviceArray * n)()
        schs = (L.ArrowSchema * n)()
        for i, b in enumerate(tables.values()):
            d, s = b.export()
            C.memmove(C.addressof(devs[i]), C.addressof(d), C.sizeof(L.ArrowDeviceArray))
            C.memmove(C.addressof(schs[i]), C.addressof(s), C.sizeof(L.ArrowSchema))
        out_dev, out_sch = L.ArrowDeviceArray(), L.ArrowSchema()
        try:
            status = lib.ark_sql_process_tables_device(self._h, n, names, devs, schs, C.byref(out_dev), C.byref(out_sch))
        finally:
            for i in range(n):
                F.release_schema(schs[i])
                F.release_array(devs[i].array)
        _check(status)
        if not out_dev.array.release:
            return None
        return F.DeviceBatch.adopt(out_dev, out_sch)


class JsonToArrowProcessor(_NativeProcessor):
    """`type: json_to_arrow` — crates/arkflow-plugin/src/processor/json.rs:42-72."""

    _create, _process, _process_device = ("ark_json_to_arrow_create", "ark_json_to_arrow_process",
                                          "ark_json_to_arrow_process_device")

    def __init__(self, config: Optional[dict]):
        if config is not None and isinstance(config.get("fields_to_include"), (set, frozenset)):
            config = dict(config, fields_to_include=sorted(config["fields_to_include"]))
        super().__init__(config)


class ArrowToJsonProcessor(_NativeProcessor):
    """`type: arrow_to_json` — crates/arkflow-plugin/src/processor/json.rs:74-113."""

    _create, _process, _process_device = "ark_arrow_to_json_create", "ark_arrow_to_json_process", "ark_arrow_to_json_process_device"

    def __init__(self, config: Optional[dict]):
        if config is not None and isinstance(config.get("fields_to_include"), (set, frozenset)):
            config = dict(config, fields_to_include=sorted(config["fields_to_include"]))
        super().__init__(config)


class _ProtobufProcessor(_NativeProcessor):
    def __init__(self, config: Optional[dict]):
        if isinstance(config, dict) and isinstance(config.get("fields_to_include"), (set, frozenset)):
            config = dict(config, fields_to_include=sorted(config["fields_to_include"]))
        super().__init__(config)

    def process(self, msg_batch) -> ProcessResult:
        # both directions build their output with MessageBatch::new_arrow: the input name is not carried over
        r = super().process(msg_batch)
        for b in r.batches:
            if isinstance(b, MessageBatch):
                b.input_name = None
        return r


class ProtobufToArrowProcessor(_ProtobufProcessor):
    """`type: protobuf_to_arrow` — crates/arkflow-plugin/src/processor/protobuf.rs:118-139, 197-214.

    config (flat): {"proto_inputs": [dir, ...], "proto_includes": [dir, ...]?, "message_type": "pkg.Msg",
    "value_field": "__value__"?}
    """

    _create, _process, _process_device = ("ark_protobuf_to_arrow_create", "ark_protobuf_to_arrow_process",
                                          "ark_protobuf_to_arrow_process_device")


class ArrowToProtobufProcessor(_ProtobufProcessor):
    """`type: arrow_to_protobuf` — crates/arkflow-plugin/src/processor/protobuf.rs:106-117, 215-232.

    config (flat): {"proto_inputs": [dir, ...], "proto_includes": [dir, ...]?, "message_type": "pkg.Msg",
    "fields_to_include": [name, ...]?}
    """

    _create, _process, _process_device = ("ark_arrow_to_protobuf_create", "ark_arrow_to_protobuf_process",
                                          "ark_arrow_to_protobuf_process_device")


class BatchProcessor(Processor):
    """`type: batch` {count, timeout_ms} — processor/batch.rs:37-124.  Holds the incoming batches in HBM and
    returns their concatenation once `count` of them are held or `timeout_ms` has passed since the last flush."""

    def __init__(self, config: Optional[dict]):
        handle = C.c_void_p()
        cfg = None if config is None else json.dumps(config).encode()
        _check(L.lib().ark_batch_create(cfg, C.byref(handle)))
        self._h = handle
        self.config = config

    def _result(self, out_arr, out_sch, input_name=None) -> ProcessResult:
        if not out_arr.release:
            return ProcessResult.none()
        return ProcessResult.single(MessageBatch(F.import_record_batch(out_arr, out_sch), input_name))

    def process(self, msg_batch) -> ProcessResult:
        mb = msg_batch if isinstance(msg_batch, MessageBatch) else MessageBatch(msg_batch)
        arr, sch = F.export_record_batch(mb.record_batch)
        out_arr, out_sch = L.ArrowArray(), L.ArrowSchema()
        try:
            status = L.lib().ark_batch_process(self._h, C.byref(arr), C.byref(sch), C.byref(out_arr), C.byref(out_sch))
        finally:
            F.release_schema(sch)
            F.release_array(arr)
        _check(status)
        return self._result(out_arr, out_sch)

    def flush(self) -> ProcessResult:
        """BatchProcessor::flush (batch.rs:72-92): Vec<MessageBatchRef> of zero or one batch."""
        out_arr, out_sch = L.ArrowArray(), L.ArrowSchema()
        _check(L.lib().ark_batch_flush(self._h, C.byref(out_arr), C.byref(out_sch)))
        return self._result(out_arr, out_sch)

    def close(self) -> None:
        if getattr(self, "_h", None):
            _check(L.lib().ark_batch_close(self._h))

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                L.lib().ark_batch_destroy(self._h)
                self._h = None
        except Exception:
            pass


# ---- registry (core/processor/mod.rs:107-129) --------------------------------------------------------
_PROCESSOR_BUILDERS: dict[str, Callable[[Optional[str], Optional[dict]], Processor]] = {}


def register_processor_builder(type_name: str, builder) -> None:
    if type_name in _PROCESSOR_BUILDERS:
        raise ArkError(L.ARK_ERR_CONFIG, f"Processor type already registered: {type_name}")
    _PROCESSOR_BUILDERS[type_name] = builder


def build_processor(config: dict) -> Processor:
    """ProcessorConfig::build: {"type": ..., "name": ...?, <flattened component config>}."""
    cfg = dict(config)
    type_name = cfg.pop("type", None)
    name = cfg.pop("name", None)
    builder = _PROCESSOR_BUILDERS.get(type_name)
    if builder is None:
        raise ArkError(L.ARK_ERR_CONFIG, f"Unknown processor type: {type_name}")
    return builder(name, cfg if cfg else None)


def init() -> None:
    """plugin::processor::init for the hot-path processors (processor/mod.rs:28-35)."""
    for t, cls in (("sql", SqlProcessor), ("json_to_arrow", JsonToArrowProcessor), ("arrow_to_json", ArrowToJsonProcessor),
                   ("protobuf_to_arrow", ProtobufToArrowProcessor), ("arrow_to_protobuf", ArrowToProtobufProcessor),
                   ("batch", BatchProcessor)):
        if t not in _PROCESSOR_BUILDERS:
            register_processor_builder(t, lambda name, cfg, _c=cls: _c(cfg))


class Pipeline:
    """core/pipeline/mod.rs:57-85: fold a batch through the processors; Multiple fans out, None stops."""

    def __init__(self, processors: list[Processor]):
        self.processors = processors

    def process(self, msg) -> ProcessResult:
        current = [msg]
        for p in self.processors:
            nxt = []
            for m in current:
                r = p.process(m)
                nxt.extend(r.into_vec())
            current = nxt
            if not current:
                return ProcessResult.none()
        if len(current) == 1:
            return ProcessResult.single(current[0])
        return ProcessResult("Multiple", current)


def split_batch(rb: pa.RecordBatch, size: int) -> list[pa.RecordBatch]:
    """core/lib.rs:432-458 (host logic, zero-copy slices)."""
    size = max(size, 1)
    total = rb.num_rows
    if total <= DEFAULT_RECORD_BATCH:
        return [rb]
    if size * DEFAULT_RECORD_BATCH < total:
        chunk = -(-total // size)
    else:
        chunk = DEFAULT_RECORD_BATCH
    out, off = [], 0
    while off < total:
        ln = min(chunk, total - off)
        out.append(rb.slice(off, ln))
        off += ln
    return out
