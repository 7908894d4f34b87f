"""Time the `file` input over 2^24 rows of schema S (oracle.synth) stored three ways: Avro with codec null, Avro with
codec snappy, and NDJSON.  For each: connect() plus every read_device() up to EOF, timed by the host clock (each read
ends in a device synchronise), the best of --repeats after one warm-up scan; then one more scan with kernel timing on
for per-kernel CUDA-event times.  Prints one JSON report: the card's name, power limit and SM clock (read in the same
call), block counts, file sizes, times and file GB/s.

The snappy file's blocks are single literals (this script's Python writer has no fast match finder), so its
avro_snappy_kernel time is that of the literal-copy path and the CRC-32, not of match copies.

    python scripts/prof_avro.py [--rows N] [--block-rows B] [--repeats R] [--out report.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from arkflow_b200 import _lib as L  # noqa: E402
from arkflow_b200.input import FileInput  # noqa: E402
from arkflow_b200.processor import ArkError, _check  # noqa: E402
from oracle.avro_oracle import block_bytes, crc32_be, header, put_varint, record_schema  # noqa: E402
from oracle.synth import synth_columns  # noqa: E402

KERNELS = ["avro_snappy_kernel", "avro_index_kernel", "avro_decode_kernel", "protobuf_strings_kernel", "cub::DeviceScan::ExclusiveSum",
           "line_start_flags_kernel", "json_parse_kernel", "json_strings_kernel"]
SCHEMA = record_schema([("timestamp", "long"), ("value", "long"), ("sensor", "string")], "S")


def records(n: int) -> np.ndarray:
    """Schema S records, 20 bytes each: timestamp (zig-zag varint, 6 bytes for these values), value (1 byte), sensor
    (length byte + 12 bytes)."""
    ts, value, key = synth_columns(n)
    zz = (ts.astype(np.uint64) << np.uint64(1))
    assert (zz >= np.uint64(1 << 35)).all() and (zz < np.uint64(1 << 42)).all()
    out = np.zeros((n, 20), dtype=np.uint8)
    for k in range(6):
        b = (zz >> np.uint64(7 * k)) & np.uint64(0x7F)
        out[:, k] = (b | (np.uint64(0x80) if k < 5 else np.uint64(0))).astype(np.uint8)
    out[:, 6] = (value.astype(np.int64) * 2).astype(np.uint8)
    out[:, 7] = 24
    out[:, 8:13] = np.frombuffer(b"temp_", dtype=np.uint8)
    k = key.copy()
    for d in range(6, -1, -1):
        out[:, 13 + d] = (k % 10).astype(np.uint8) + ord("0")
        k //= 10
    return out


def write_avro_file(path: str, rec: np.ndarray, block_rows: int, codec: str) -> int:
    n = len(rec)
    blocks = 0
    with open(path, "wb") as f:
        f.write(header(SCHEMA, codec))
        for r in range(0, n, block_rows):
            raw = rec[r:r + block_rows].tobytes()
            if codec == "snappy":
                lit = len(raw) - 1
                data = put_varint(len(raw)) + bytes([63 << 2]) + lit.to_bytes(4, "little") + raw + crc32_be(raw)
            else:
                data = raw
            f.write(block_bytes(min(block_rows, n - r), data))
            blocks += 1
    return blocks


def write_ndjson(path: str, n: int) -> None:
    ts, value, key = synth_columns(n)
    with open(path, "w") as f:
        step = 1 << 20
        for r in range(0, n, step):
            f.write("".join('{"timestamp":%d,"value":%d,"sensor":"temp_%07d"}\n' % t
                            for t in zip(ts[r:r + step].tolist(), value[r:r + step].tolist(), key[r:r + step].tolist())))


def scan(path: str, kind: str) -> int:
    inp = FileInput({"input_type": {"type": kind, "path": path}})
    inp.connect()
    rows = 0
    try:
        while True:
            b = inp.read_device()
            rows += b.num_rows
            b.close()
    except ArkError as e:
        if e.kind != "EOF":
            raise
    return rows


def card() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
        return dict(zip(q.split(","), [x.strip() for x in line.splitlines()[0].split(",")]))
    except Exception as e:  # the report says what could not be read
        return {"error": str(e)}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 24)
    ap.add_argument("--block-rows", type=int, default=1 << 14)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "prof_avro.py measures on a CUDA device"
    lib = L.lib()
    _check(lib.ark_b200_init(0))
    report = {"rows": a.rows, "block_rows": a.block_rows, "card_before": card(), "files": {}}
    with tempfile.TemporaryDirectory() as tmp:
        rec = records(a.rows)
        paths = {}
        for codec in ("null", "snappy"):
            p = os.path.join(tmp, codec + ".avro")
            report["files"]["avro_" + codec] = {"blocks": write_avro_file(p, rec, a.block_rows, codec)}
            paths["avro_" + codec] = (p, "avro")
        p = os.path.join(tmp, "s.ndjson")
        write_ndjson(p, a.rows)
        paths["ndjson"] = (p, "json")
        for name, (p, kind) in paths.items():
            r = report["files"].setdefault(name, {})
            r["bytes"] = os.path.getsize(p)
            assert scan(p, kind) == a.rows  # warm-up
            times = []
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                scan(p, kind)
                times.append(time.perf_counter() - t0)
            r["connect_and_reads_s"] = min(times)
            r["all_s"] = times
            r["file_GBps"] = r["bytes"] / min(times) / 1e9
            lib.ark_kernel_timing_enable(1)
            lib.ark_kernel_timing_reset()
            scan(p, kind)
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
