#!/usr/bin/env python
"""Run one query repeatedly on device-resident synthetic batches (for ncu / quick timing).
Usage: python scripts/prof_query.py "<sql>" [rows] [keys] [reps] [value_kind]"""
import ctypes as C
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch

from arkflow_b200 import _lib as L
from arkflow_b200 import arrow_ffi as F
from arkflow_b200.processor import SqlProcessor, _check

q = sys.argv[1]
rows = int(sys.argv[2]) if len(sys.argv) > 2 else 1 << 24
keys = int(sys.argv[3]) if len(sys.argv) > 3 else 1_000_000
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 6
kind = int(sys.argv[5]) if len(sys.argv) > 5 else 0
nres = int(sys.argv[6]) if len(sys.argv) > 6 else 3
lib = L.lib()
_check(lib.ark_b200_init(0))
proc = SqlProcessor({"query": q})
bs = []
for b in range(nres):
    dev, sch = L.ArrowDeviceArray(), L.ArrowSchema()
    _check(lib.ark_synth_batch_device(rows, b * rows, 42, kind, keys, C.byref(dev), C.byref(sch)))
    bs.append(F.DeviceBatch.adopt(dev, sch))
for i in range(3):
    proc.process_device(bs[i % nres]).close()
lib.ark_kernel_timing_reset()
lib.ark_kernel_timing_enable(1)
for i in range(reps):
    proc.process_device(bs[i % nres]).close()
torch.cuda.synchronize()
import time
t0 = time.perf_counter()
for i in range(reps):
    proc.process_device(bs[i % nres]).close()
torch.cuda.synchronize()
print(f"call wall avg {(time.perf_counter() - t0) / reps * 1e3:.3f} ms")
for name in (b"hash_agg_staged_kernel", b"hash_agg_stream_kernel", b"hash_agg_kernel", b"hash_agg_tile_kernel", b"filter_project_tma_kernel", b"filter_project_kernel", b"agg_init_kernel", b"agg_compact_kernel", b"agg_emit_keys_kernel", b"agg_gather_acc_kernel", b"agg_finalize_kernel"):
    ms, n = C.c_double(), C.c_int64()
    lib.ark_kernel_timing_get(name, C.byref(ms), C.byref(n))
    if n.value:
        print(f"{name.decode():28s} avg {ms.value / n.value:.4f} ms over {n.value} launches")
