#!/usr/bin/env python
"""CSV `file` input scan throughput: 2^22 rows written to a temporary file, read through FileInput repeatedly.

    prof_csv.py [reps] [int | float]

`int` rows hold integers and 3-decimal scores (the shape of tests/test_inputs_gpu.py); `float` rows hold three
random doubles written shortest-round-trip (repr).  Reports the wall time per scan and csv_parse_kernel's time."""
import ctypes as C, os, random, sys, tempfile, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from arkflow_b200 import _lib as L
from arkflow_b200.input import FileInput
from arkflow_b200.processor import ArkError, _check
lib = L.lib(); _check(lib.ark_b200_init(0))
n = 1 << 22
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
kind = sys.argv[2] if len(sys.argv) > 2 else "int"
rng = random.Random(1)
with tempfile.TemporaryDirectory() as tmp:
    path = os.path.join(tmp, "scan.csv")
    with open(path, "w") as f:
        if kind == "int":
            f.write("id,value,score\n")
            f.writelines("%d,%d,%.3f\n" % (i, rng.randrange(-50, 50), rng.random() * 100) for i in range(n))
        else:
            f.write("x,y,z\n")
            f.writelines("%r,%r,%r\n" % (rng.uniform(-1e3, 1e3), rng.lognormvariate(0, 5), rng.gauss(0, 1)) for _ in range(n))
    size = os.path.getsize(path)

    def scan():
        inp = FileInput({"input_type": {"type": "csv", "path": path}})
        inp.connect()
        rows = 0
        while True:
            try:
                b = inp.read_device()
            except ArkError:
                return rows
            rows += b.num_rows
            b.close()

    for _ in range(2): scan()
    lib.ark_kernel_timing_reset(); lib.ark_kernel_timing_enable(1)
    torch.cuda.synchronize(); t0 = time.perf_counter()
    for _ in range(reps): assert scan() == n
    torch.cuda.synchronize(); dt = (time.perf_counter() - t0) / reps
    print(f"{kind} csv ({size / n:.1f} B/row, {size / 2**20:.0f} MiB): scan wall avg {dt * 1e3:.1f} ms ({size / dt / 1e9:.2f} GB/s)")
    ms, cnt = C.c_double(), C.c_int64()
    lib.ark_kernel_timing_get(b"csv_parse_kernel", C.byref(ms), C.byref(cnt))
    if cnt.value: print(f"csv_parse_kernel         avg {ms.value / cnt.value:.4f} ms over {cnt.value} launches")
