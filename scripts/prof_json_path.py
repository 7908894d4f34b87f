#!/usr/bin/env python
"""prof_json_path.py — the JSON path functions against today's route to the same result, on one device.

2^24 generate-style documents ({"timestamp":…,"value":…,"sensor":"…"}, ~60 bytes each) in one Utf8 column, and
    A  SELECT json_get_str(doc,'sensor'), json_get_float(doc,'value') FROM flow WHERE json_get_int(doc,'timestamp') > X
    B  json_to_arrow over the same bytes as Binary, then SELECT sensor, value FROM flow WHERE timestamp > X
Both run on device-resident batches (process_device).  After warm-up, each route is timed over --iters calls with CUDA
events (every call ends in a device synchronisation), and the kernels' own times come from ark_kernel_timing_*.
Prints one JSON line with the card's name and power limit; the two results are checked equal first.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import pyarrow as pa  # noqa: E402
import pyarrow.compute as pc  # noqa: E402


def docs(n: int, seed: int = 1) -> pa.Array:
    rng = np.random.default_rng(seed)
    ts = pa.array(rng.integers(1_600_000_000_000, 1_700_000_000_000, n))
    val = pa.array(rng.integers(0, 100_000, n) / 100.0 + 0.001)  # never integral: json_to_arrow infers Float64
    sensor = pa.array(rng.integers(0, 1000, n))
    parts = ['{"timestamp":', pc.cast(ts, pa.string()), ',"value":', pc.cast(val, pa.string()), ',"sensor":"temp_',
             pc.cast(sensor, pa.string()), '"}']
    return pc.binary_join_element_wise(*[p if isinstance(p, pa.Array) else pa.scalar(p) for p in parts], "")


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, check=True).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"gpu": name, "power_limit": power}
    except Exception as e:  # the numbers are still printed, marked with what is unknown
        return {"gpu": "unknown", "power_limit": "unknown", "why": str(e)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 24)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "prof_json_path.py measures on a CUDA device"
    from arkflow_b200 import _lib as L
    from arkflow_b200.arrow_ffi import DeviceBatch
    from arkflow_b200.processor import JsonToArrowProcessor, SqlProcessor

    lib = L.lib()
    d = docs(a.rows)
    x = 1_650_000_000_000
    doc_bytes = int(pc.sum(pc.binary_length(d)).as_py())
    dev_a = DeviceBatch.from_arrow(pa.record_batch({"doc": d}))
    dev_b = DeviceBatch.from_arrow(pa.record_batch({"__value__": d.cast(pa.binary())}))
    qa = SqlProcessor({"query": "SELECT json_get_str(doc,'sensor'), json_get_float(doc,'value') FROM flow "
                                f"WHERE json_get_int(doc,'timestamp') > {x}"})
    dec = JsonToArrowProcessor({})
    qb = SqlProcessor({"query": f"SELECT sensor, value FROM flow WHERE timestamp > {x}"})

    def route_a():
        return qa.process_device(dev_a)

    def route_b():
        return qb.process_device(dec.process_device(dev_b))

    ra, rb = route_a().to_arrow(), route_b().to_arrow()
    assert ra.num_rows == rb.num_rows and ra.column(0).equals(rb.column(0)) and ra.column(1).equals(rb.column(1)), "routes differ"
    res = {"rows": a.rows, "doc_bytes": doc_bytes, "rows_out": ra.num_rows, **card()}
    kernels = ["json_path_kernel", "json_parse_kernel", "json_strings_kernel", "protobuf_strings_kernel"]
    for name, fn in (("A_json_functions", route_a), ("B_json_to_arrow_then_sql", route_b)):
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        lib.ark_kernel_timing_enable(1)
        lib.ark_kernel_timing_reset()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.iters
        ks = {}
        for k in kernels:
            t, n = C.c_double(), C.c_int64()
            lib.ark_kernel_timing_get(k.encode(), C.byref(t), C.byref(n))
            if n.value:
                ks[k] = round(t.value / a.iters, 3)
        lib.ark_kernel_timing_enable(0)
        res[name] = {"call_ms": round(ms, 3), "doc_GB_per_s": round(doc_bytes / ms / 1e6, 2), "kernel_ms_per_call": ks}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
