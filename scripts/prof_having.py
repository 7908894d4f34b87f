#!/usr/bin/env python
"""prof_having.py — what the stage after the aggregate (HAVING, computed items, LIMIT) costs on bench.py's GROUP BY.

bench.py's GROUP BY workload: device-resident synthetic batches of 2^24 rows over 10^6 sensors (csrc/synth.cu), and
    plain     SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor
    keep p    the same query with HAVING count(*) > k, k chosen from the plain result so about p of the groups stay
              (1 %, 50 %, 100 %)
    computed  the same query with one more item, SUM(value) / COUNT(*)
Call time comes from CUDA events after warm-up with kernel timing off (every call ends in a device synchronisation).
The stage's kernel time comes from ark_kernel_timing_* in a second pass.  Before timing, every query is checked against
tests/having_oracle.py on a smaller batch.  Prints one JSON line with the card's name and power limit.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

PLAIN = "SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor"
STAGE_KERNELS = ("filter_project_tma_kernel", "filter_project_kernel")


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
    ap.add_argument("--keys", type=int, default=1_000_000)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    import torch

    assert torch.cuda.is_available(), "prof_having.py measures on a CUDA device"
    from arkflow_b200 import _lib as L
    from arkflow_b200.arrow_ffi import DeviceBatch
    from arkflow_b200.processor import SqlProcessor, _check
    from having_oracle import sql_process_having
    from oracle.synth import synth_batch

    lib = L.lib()
    _check(lib.ark_b200_init(0))

    def synth_device(n, key_space):
        dev, sch = L.ArrowDeviceArray(), L.ArrowSchema()
        _check(lib.ark_synth_batch_device(n, 0, 42, 0, key_space, C.byref(dev), C.byref(sch)))
        return DeviceBatch.adopt(dev, sch)

    batch = synth_device(a.rows, a.keys)
    plain = SqlProcessor({"query": PLAIN})
    counts = np.asarray(plain.process_device(batch).to_arrow().column("count(*)"))
    queries = {"plain": PLAIN}
    for p in (0.01, 0.5, 1.0):
        k = int(np.quantile(counts, 1.0 - p)) if p < 1.0 else 0
        queries[f"keep_{int(p * 100)}pct"] = f"{PLAIN} HAVING count(*) > {k}"
    queries["computed"] = "SELECT sensor, SUM(value), COUNT(*), SUM(value) / COUNT(*) FROM flow GROUP BY sensor"

    # outputs against the oracle, at a size the oracle handles quickly
    small = synth_batch(1 << 18, seed=42, key_space=10_000)
    for name, q in queries.items():
        want = sql_process_having(small, q)
        got = SqlProcessor({"query": q}).process_device(DeviceBatch.from_arrow(small)).to_arrow()
        key = lambda rb: sorted(map(repr, rb.to_pylist()))  # noqa: E731
        assert got.schema.names == want.schema.names and key(got) == key(want), name

    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    res = {"rows": a.rows, "keys": a.keys, "iters": a.iters, **card(), "workloads": {}}
    for name, q in queries.items():
        proc = SqlProcessor({"query": q})
        for _ in range(a.warmup):
            proc.process_device(batch).close()
        torch.cuda.synchronize()
        ev0.record()
        rows = 0
        for _ in range(a.iters):
            out = proc.process_device(batch)
            rows = out.num_rows
            out.close()
        ev1.record()
        ev1.synchronize()
        call_ms = ev0.elapsed_time(ev1) / a.iters
        lib.ark_kernel_timing_reset()
        lib.ark_kernel_timing_enable(1)
        for _ in range(a.iters):
            proc.process_device(batch).close()
        lib.ark_kernel_timing_enable(0)
        stage_ms, launches = 0.0, 0
        for kname in STAGE_KERNELS:
            ms, n = C.c_double(), C.c_int64()
            lib.ark_kernel_timing_get(kname.encode(), C.byref(ms), C.byref(n))
            stage_ms += ms.value
            launches += n.value
        stage_ms /= a.iters
        res["workloads"][name] = {"query": q, "groups_out": rows, "call_ms": round(call_ms, 4),
                                  "stage_kernel_ms": round(stage_ms, 4), "stage_launches_per_call": launches / a.iters,
                                  "stage_share_of_call": round(stage_ms / call_ms, 4)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
