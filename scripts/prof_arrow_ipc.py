"""Time the `file` input's `arrow` type over 2^24 rows of schema S (oracle.synth) stored four ways by pyarrow's IPC
writer: uncompressed in one record batch (every read a view of the uploaded file), uncompressed in 64 Ki-row batches
(reads joined by concat), LZ4_FRAME in 64 Ki-row batches, and LZ4_FRAME in one record batch (one warp per frame, so as
many warps as the batch has buffers).  For each: connect() plus every read_device() up to EOF, timed by the host clock
(each read ends in a device synchronise), the best of --repeats after one warm-up scan; then one more scan with kernel
timing on for per-kernel CUDA-event times.  Prints one JSON report: the card's name, power limit and SM clock (read in
the same call), file sizes, times and file GB/s.

    python scripts/prof_arrow_ipc.py [--rows N] [--batch-rows B] [--repeats R] [--out report.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import tempfile
import time

import pyarrow as pa

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from arkflow_b200 import _lib as L  # noqa: E402
from arkflow_b200.processor import _check  # noqa: E402
from oracle.synth import synth_batch  # noqa: E402
from prof_avro import card, scan  # noqa: E402

KERNELS = ["ipc_lz4_kernel", "ipc_validate_kernel", "count_zeros_kernel", "gather_extents_kernel", "concat_copy_kernel",
           "concat_offsets_kernel", "concat_bits_kernel"]


def write(path: str, rb: pa.RecordBatch, batch_rows: int, compression) -> int:
    opts = pa.ipc.IpcWriteOptions(compression=compression)
    with pa.OSFile(path, "wb") as f, pa.ipc.new_file(f, rb.schema, options=opts) as w:
        for r in range(0, rb.num_rows, batch_rows):
            w.write(rb.slice(r, batch_rows))
    return (rb.num_rows + batch_rows - 1) // batch_rows


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 24)
    ap.add_argument("--batch-rows", type=int, default=1 << 16)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "prof_arrow_ipc.py measures on a CUDA device"
    lib = L.lib()
    _check(lib.ark_b200_init(0))
    report = {"rows": a.rows, "batch_rows": a.batch_rows, "card_before": card(), "files": {}}
    rb = synth_batch(a.rows)
    with tempfile.TemporaryDirectory() as tmp:
        paths = {}
        for name, rows, comp in (("none_1batch", a.rows, None), ("none_batches", a.batch_rows, None),
                                 ("lz4_batches", a.batch_rows, "lz4"), ("lz4_1batch", a.rows, "lz4")):
            p = os.path.join(tmp, name + ".arrow")
            report["files"][name] = {"record_batches": write(p, rb, rows, comp)}
            paths[name] = p
        for name, p in paths.items():
            r = report["files"][name]
            r["bytes"] = os.path.getsize(p)
            assert scan(p, "arrow") == a.rows  # warm-up
            times = []
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                scan(p, "arrow")
                times.append(time.perf_counter() - t0)
            r["connect_and_reads_s"] = min(times)
            r["all_s"] = times
            r["file_GBps"] = r["bytes"] / min(times) / 1e9
            lib.ark_kernel_timing_enable(1)
            lib.ark_kernel_timing_reset()
            scan(p, "arrow")
            lib.ark_kernel_timing_enable(0)
            ks = {}
            for k in KERNELS:
                ms, n = C.c_double(), C.c_int64()
                lib.ark_kernel_timing_get(k.encode(), C.byref(ms), C.byref(n))
                if n.value:
                    ks[k] = {"ms": round(ms.value, 3), "launches": n.value}
            r["kernels"] = ks
    report["card_after"] = card()
    s = json.dumps(report, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
