"""Consecutive filter fast-path calls against the oracle (oracle/sql_oracle.py).

Every leased stream keeps two look-back descriptor buffers for the tile kernel: consecutive launches on a stream use them
in turn, each launch zeroes the other one for a launch with the same tile count, and a buffer in any other state is
cleared with one memset first.  These cases run many calls on one processor while the tile count changes from call to
call (2^24 rows, then 1, 2047, 2048 and 2049 rows: 8192, 1, 1, 1 and 2 tiles), repeat tile counts so that launches run on
buffers zeroed by the launch before, and check every output against the oracle:
  * one caller, as built and with the look-back forced to help (ARK_FP_DEBUG=4, read once per process: a child process);
  * several threads sharing one processor, each on a stream of its own;
  * sliced inputs (Arrow offsets, offsets[0] != 0), and SELECT * outputs, which alias their input, used after the input
    handle is gone.
Each case also asserts that the tile kernel ran once per call: a silent fallback to the general kernel fails.
"""
import ctypes as C
import gc
import os
import subprocess
import sys
import threading

import pyarrow as pa
import pyarrow.compute as pc
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

pytestmark = pytest.mark.gpu

QUERY = "SELECT sensor, value FROM flow WHERE value >= 10"
TILE = "filter_project_tile_kernel"
# rows per call: tile counts 8192, 8192, 1, 1, 1, 2, 2, 1, 33, 8192, 1
SEQUENCE = [1 << 24, 1 << 24, 1, 2047, 2048, 2049, 2049, 2048, 2048 * 32 + 1, 1 << 24, 1]


def _batch(n, row0):
    from oracle.synth import synth_batch

    return synth_batch(n, row0=row0, key_space=1000)


def _expected(rb, query=QUERY):
    if rb.num_rows > 1 << 20:  # pc.filter stands in for the oracle at 2^24 rows (test_oracle_crosscheck ties the two)
        m = pc.greater_equal(rb.column("value"), 10)
        return pa.record_batch({"sensor": pc.filter(rb.column("sensor"), m), "value": pc.filter(rb.column("value"), m)})
    from oracle.sql_oracle import sql_process

    return sql_process(pa.RecordBatch.from_arrays([pa.concat_arrays([c]) for c in rb.columns], schema=rb.schema), query)


def _tile_launches(lib):
    ms, n = C.c_double(), C.c_int64()
    lib.ark_kernel_timing_get(TILE.encode(), C.byref(ms), C.byref(n))
    return n.value


def _run_sequence(lib, proc, sizes, row0=0):
    """Every call's output compared with the oracle; returns the number of calls."""
    from arkflow_b200.arrow_ffi import DeviceBatch

    for k, n in enumerate(sizes):
        rb = _batch(n, row0 + 7919 * k)
        out = proc.process_device(DeviceBatch.from_arrow(rb))
        got = out.to_arrow()
        out.close()
        want = _expected(rb)
        assert got.schema.names == want.schema.names and got.equals(want), (k, n)
    return len(sizes)


def _single_caller():
    from arkflow_b200 import _lib as L
    from arkflow_b200.processor import SqlProcessor, _check

    lib = L.lib()
    _check(lib.ark_b200_init(0))
    lib.ark_kernel_timing_reset()
    lib.ark_kernel_timing_enable(1)
    proc = SqlProcessor({"query": QUERY})
    calls = _run_sequence(lib, proc, SEQUENCE) + _run_sequence(lib, proc, SEQUENCE[::-1], row0=1 << 30)
    assert _tile_launches(lib) == calls, (_tile_launches(lib), calls)
    lib.ark_kernel_timing_enable(0)


def test_consecutive_calls_changing_tile_count(gpu):
    _single_caller()


def test_consecutive_calls_with_helping():
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "single"], capture_output=True, text=True, timeout=1200,
                       env=dict(os.environ, ARK_FP_DEBUG="4"))
    assert r.returncode == 0 and "CHILD_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]


def test_threads_share_one_processor(gpu):
    from arkflow_b200.processor import SqlProcessor

    proc = SqlProcessor({"query": QUERY})
    sizes = [2049, 1, 2048 * 40 + 7, 1 << 20, 2047, 1 << 20, 2048, 2049]
    errors = []

    def worker(t):
        try:
            for rnd in range(3):
                _run_sequence(gpu, proc, sizes[t % 4:] + sizes[:t % 4], row0=(t * 3 + rnd) << 24)
        except Exception as e:  # noqa: BLE001 — reported by the main thread
            errors.append(f"thread {t}: {e!r}")

    gpu.ark_kernel_timing_reset()
    gpu.ark_kernel_timing_enable(1)
    threads = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert _tile_launches(gpu) == 4 * 3 * len(sizes)
    gpu.ark_kernel_timing_enable(0)


def test_sliced_inputs_and_select_star_outputs(gpu):
    from arkflow_b200.arrow_ffi import DeviceBatch
    from arkflow_b200.processor import SqlProcessor
    from oracle.sql_oracle import sql_process

    proc = SqlProcessor({"query": QUERY})
    star = SqlProcessor({"query": "SELECT * FROM flow"})
    kept = []
    gpu.ark_kernel_timing_reset()
    gpu.ark_kernel_timing_enable(1)
    calls = 0
    for k, (n, off) in enumerate([(2048 * 3 + 5, 1), (2049, 13), (70_001, 2047), (4097, 2048), (2048 * 33, 777)]):
        rb = _batch(n, 1000 * k)
        sl = rb.slice(off, n - off - (k % 3))
        out = proc.process_device(DeviceBatch.from_arrow(sl, keep_offsets=True))
        got = out.to_arrow()
        out.close()
        calls += 1
        assert got.equals(_expected(sl)), (n, off)
        # SELECT * hands back the input's own buffers: the output must stay valid after the input handle is dropped,
        # while fast-path calls on the same streams go on
        inp = DeviceBatch.from_arrow(sl, keep_offsets=True)
        kept.append((star.process_device(inp), sl))
        del inp
        gc.collect()
    assert _tile_launches(gpu) == calls
    gpu.ark_kernel_timing_enable(0)
    for out, sl in kept:
        want = sql_process(pa.RecordBatch.from_arrays([pa.concat_arrays([c]) for c in sl.columns], schema=sl.schema),
                           "SELECT * FROM flow")
        assert out.to_arrow().equals(want)
        out.close()


if __name__ == "__main__":
    if sys.argv[1] == "single":
        _single_caller()
        print("CHILD_OK")
