"""ctypes binding of libarkflow_b200.so (the C ABI in include/arkflow_b200.h).

The library is the product path: there is NO Python/CPU fallback.  Importing this module fails
loudly when the shared object has not been built (`python -c "import __graft_entry__ as g; g.build()"`
or `make`), and every compute entry point fails loudly when no CUDA device is present.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libarkflow_b200.so")


class ArrowSchema(C.Structure):
    pass


class ArrowArray(C.Structure):
    pass


ArrowSchema._fields_ = [
    ("format", C.c_char_p),
    ("name", C.c_char_p),
    ("metadata", C.c_char_p),
    ("flags", C.c_int64),
    ("n_children", C.c_int64),
    ("children", C.POINTER(C.POINTER(ArrowSchema))),
    ("dictionary", C.POINTER(ArrowSchema)),
    ("release", C.c_void_p),
    ("private_data", C.c_void_p),
]

ArrowArray._fields_ = [
    ("length", C.c_int64),
    ("null_count", C.c_int64),
    ("offset", C.c_int64),
    ("n_buffers", C.c_int64),
    ("n_children", C.c_int64),
    ("buffers", C.POINTER(C.c_void_p)),
    ("children", C.POINTER(C.POINTER(ArrowArray))),
    ("dictionary", C.POINTER(ArrowArray)),
    ("release", C.c_void_p),
    ("private_data", C.c_void_p),
]


class ArrowDeviceArray(C.Structure):
    _fields_ = [
        ("array", ArrowArray),
        ("device_id", C.c_int64),
        ("device_type", C.c_int32),
        ("sync_event", C.c_void_p),
        ("reserved", C.c_int64 * 3),
    ]


ARROW_DEVICE_CUDA = 2

ARK_OK, ARK_ERR_CONFIG, ARK_ERR_PROCESS, ARK_ERR_UNSUPPORTED, ARK_ERR_SERIALIZATION, ARK_ERR_CUDA, ARK_ERR_EOF = range(7)

RELEASE_SCHEMA = C.CFUNCTYPE(None, C.POINTER(ArrowSchema))
RELEASE_ARRAY = C.CFUNCTYPE(None, C.POINTER(ArrowArray))


def _declare(lib):
    P = C.POINTER
    vp = C.c_void_p
    sig = {
        "ark_b200_init": (C.c_int, [C.c_int]),
        "ark_b200_device_count": (C.c_int, [P(C.c_int)]),
        "ark_b200_version": (C.c_char_p, []),
        "ark_last_error": (C.c_char_p, []),
        "ark_sql_create": (C.c_int, [C.c_char_p, P(vp)]),
        "ark_sql_process": (C.c_int, [vp, P(ArrowArray), P(ArrowSchema), P(ArrowArray), P(ArrowSchema)]),
        "ark_sql_process_device": (C.c_int, [vp, P(ArrowDeviceArray), P(ArrowSchema), P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_sql_process_tables": (C.c_int, [vp, C.c_int, P(C.c_char_p), P(ArrowArray), P(ArrowSchema), P(ArrowArray), P(ArrowSchema)]),
        "ark_sql_process_tables_device": (C.c_int, [vp, C.c_int, P(C.c_char_p), P(ArrowDeviceArray), P(ArrowSchema), P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_json_to_arrow_create": (C.c_int, [C.c_char_p, P(vp)]),
        "ark_json_to_arrow_process": (C.c_int, [vp, P(ArrowArray), P(ArrowSchema), P(ArrowArray), P(ArrowSchema)]),
        "ark_json_to_arrow_process_device": (C.c_int, [vp, P(ArrowDeviceArray), P(ArrowSchema), P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_arrow_to_json_create": (C.c_int, [C.c_char_p, P(vp)]),
        "ark_arrow_to_json_process": (C.c_int, [vp, P(ArrowArray), P(ArrowSchema), P(ArrowArray), P(ArrowSchema)]),
        "ark_arrow_to_json_process_device": (C.c_int, [vp, P(ArrowDeviceArray), P(ArrowSchema), P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_protobuf_to_arrow_create": (C.c_int, [C.c_char_p, P(vp)]),
        "ark_protobuf_to_arrow_process": (C.c_int, [vp, P(ArrowArray), P(ArrowSchema), P(ArrowArray), P(ArrowSchema)]),
        "ark_protobuf_to_arrow_process_device": (C.c_int, [vp, P(ArrowDeviceArray), P(ArrowSchema), P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_arrow_to_protobuf_create": (C.c_int, [C.c_char_p, P(vp)]),
        "ark_arrow_to_protobuf_process": (C.c_int, [vp, P(ArrowArray), P(ArrowSchema), P(ArrowArray), P(ArrowSchema)]),
        "ark_arrow_to_protobuf_process_device": (C.c_int, [vp, P(ArrowDeviceArray), P(ArrowSchema), P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_expr_evaluate": (C.c_int, [C.c_char_p, P(ArrowArray), P(ArrowSchema), P(ArrowArray), P(ArrowSchema), P(C.c_int)]),
        "ark_expr_evaluate_device": (C.c_int, [C.c_char_p, P(ArrowDeviceArray), P(ArrowSchema), P(ArrowDeviceArray), P(ArrowSchema), P(C.c_int)]),
        "ark_proc_close": (C.c_int, [vp]),
        "ark_proc_destroy": (None, [vp]),
        "ark_concat_batches": (C.c_int, [C.c_int, P(ArrowArray), P(ArrowSchema), P(ArrowArray), P(ArrowSchema)]),
        "ark_concat_batches_device": (C.c_int, [C.c_int, P(ArrowDeviceArray), P(ArrowSchema), P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_buffer_create": (C.c_int, [C.c_char_p, C.c_char_p, C.c_char_p, P(vp)]),
        "ark_buffer_write": (C.c_int, [vp, P(ArrowArray), P(ArrowSchema), C.c_char_p, C.c_uint64]),
        "ark_buffer_read": (C.c_int, [vp, P(ArrowArray), P(ArrowSchema), P(C.c_uint64), C.c_int64, P(C.c_int64)]),
        "ark_buffer_write_device": (C.c_int, [vp, P(ArrowDeviceArray), P(ArrowSchema), C.c_char_p, C.c_uint64]),
        "ark_buffer_read_device": (C.c_int, [vp, P(ArrowDeviceArray), P(ArrowSchema), P(C.c_uint64), C.c_int64, P(C.c_int64)]),
        "ark_buffer_flush": (C.c_int, [vp]),
        "ark_input_create": (C.c_int, [C.c_char_p, C.c_char_p, P(vp)]),
        "ark_input_connect": (C.c_int, [vp]),
        "ark_input_read": (C.c_int, [vp, P(ArrowArray), P(ArrowSchema)]),
        "ark_input_read_device": (C.c_int, [vp, P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_input_close": (C.c_int, [vp]),
        "ark_input_destroy": (None, [vp]),
        "ark_buffer_close": (C.c_int, [vp]),
        "ark_buffer_destroy": (None, [vp]),
        "ark_batch_create": (C.c_int, [C.c_char_p, P(vp)]),
        "ark_batch_process": (C.c_int, [vp, P(ArrowArray), P(ArrowSchema), P(ArrowArray), P(ArrowSchema)]),
        "ark_batch_flush": (C.c_int, [vp, P(ArrowArray), P(ArrowSchema)]),
        "ark_batch_close": (C.c_int, [vp]),
        "ark_batch_destroy": (None, [vp]),
        "ark_sql_partial_aggregate_device": (C.c_int, [vp, P(ArrowDeviceArray), P(ArrowSchema), C.c_int, P(ArrowDeviceArray), P(ArrowSchema), P(C.c_int64)]),
        "ark_sql_final_aggregate_device": (C.c_int, [vp, P(ArrowDeviceArray), P(ArrowSchema), P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_hash_partition_device": (C.c_int, [P(ArrowDeviceArray), P(ArrowSchema), C.c_char_p, C.c_int, P(ArrowDeviceArray), P(ArrowSchema), P(C.c_int64)]),
        "ark_ipc_export_device": (C.c_int, [P(ArrowDeviceArray), P(ArrowSchema), P(C.c_uint8), C.c_int64, P(C.c_int64)]),
        "ark_ipc_concat_slices_device": (C.c_int, [C.c_int, P(P(C.c_uint8)), P(C.c_int64), P(C.c_int64), P(C.c_int64), P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_dist_create": (C.c_int, [C.c_int, C.c_int, C.c_int64, P(vp)]),
        "ark_dist_handle_bytes": (C.c_int64, []),
        "ark_dist_export": (C.c_int, [vp, P(C.c_uint8), C.c_int64, P(C.c_int64)]),
        "ark_dist_connect": (C.c_int, [vp, P(C.c_uint8), C.c_int64]),
        "ark_dist_stats": (C.c_int, [vp, P(C.c_int64)]),
        "ark_dist_destroy": (None, [vp]),
        "ark_sql_group_by_exchange_device": (C.c_int, [vp, vp, P(ArrowDeviceArray), P(ArrowSchema), P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_sql_group_by_push_device": (C.c_int, [vp, vp, P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_sql_group_by_merge_device": (C.c_int, [vp, vp, P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_synth_batch_device": (C.c_int, [C.c_int64, C.c_int64, C.c_uint64, C.c_int, C.c_int64, P(ArrowDeviceArray), P(ArrowSchema)]),
        "ark_kernel_launch_count": (C.c_int64, []),
        "ark_kernel_timing_enable": (None, [C.c_int]),
        "ark_kernel_timing_reset": (None, []),
        "ark_kernel_timing_get": (C.c_int, [C.c_char_p, P(C.c_double), P(C.c_int64)]),
        "ark_host_copy": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int64, C.c_int]),
    }
    missing = []
    for name, (res, args) in sig.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            missing.append(name)
            continue
        fn.restype = res
        fn.argtypes = args
    return sig, missing


EXPORTED_SYMBOLS: tuple = ()
_lib = None


def lib():
    """The loaded library.  Raises (never falls back) when it is missing or incomplete."""
    global _lib, EXPORTED_SYMBOLS
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is not built; run `make` (or __graft_entry__.build()). "
                "arkflow_b200 has no CPU fallback."
            )
        handle = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        sig, missing = _declare(handle)
        if missing:
            raise RuntimeError(f"{LIB_PATH} does not export: {', '.join(missing)}")
        EXPORTED_SYMBOLS = tuple(sig)
        _lib = handle
    return _lib


def declared_symbols() -> list[str]:
    """Every `ark_*` function declared in include/arkflow_b200.h (parsed from the header)."""
    import re

    hdr = os.path.join(os.path.dirname(_HERE), "include", "arkflow_b200.h")
    text = open(hdr).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(ark_[a-z0-9_]+)\s*\(", text)))
