#!/usr/bin/env python
"""json_to_arrow on 2^22 device-resident messages, repeatedly (for ncu / quick timing).

    prof_json.py [reps] [int | float]

`int` (the default) is the 63-byte message of examples/generate_example.yaml, whose numbers are integers.  `float`
gives every message three random doubles written shortest-round-trip (repr), so that the Float64 columns go through
the full decimal conversion rather than Clinger's fast path."""
import ctypes as C, os, random, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from arkflow_b200 import _lib as L, arrow_ffi as F
from arkflow_b200.processor import JsonToArrowProcessor, _check
lib = L.lib(); _check(lib.ark_b200_init(0))
m = 1 << 22
reps = int(sys.argv[1]) if len(sys.argv) > 1 else 6
kind = sys.argv[2] if len(sys.argv) > 2 else "int"
if kind == "int":
    msg = b'{ "timestamp": 1625000000000, "value": 10, "sensor": "temp_1" }'
    blob, lens = msg * m, np.full(m, len(msg), np.int64)
else:
    rng = random.Random(1)
    msgs = [b'{"x": %r, "y": %r, "z": %r}' % (rng.uniform(-1e3, 1e3), rng.lognormvariate(0, 5), rng.gauss(0, 1)) for _ in range(m)]
    blob, lens = b"".join(msgs), np.array([len(x) for x in msgs], np.int64)
data = torch.from_numpy(np.frombuffer(blob, dtype=np.uint8).copy()).cuda()
offs = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int32)).cuda()
payload = F.DeviceBatch([F.DeviceColumn("__value__", "binary", m, data, offs, None, 0, False)], m)
proc = JsonToArrowProcessor({})
for _ in range(3): proc.process_device(payload).close()
lib.ark_kernel_timing_reset(); lib.ark_kernel_timing_enable(1)
torch.cuda.synchronize(); t0 = time.perf_counter()
for _ in range(reps): proc.process_device(payload).close()
torch.cuda.synchronize(); print(f"{kind} payload ({len(blob) / m:.1f} B/msg): call wall avg {(time.perf_counter()-t0)/reps*1e3:.3f} ms")
for name in (b"json_parse_kernel", b"json_count_kernel", b"json_strings_kernel", b"pack_bits_kernel"):
    ms, n = C.c_double(), C.c_int64()
    lib.ark_kernel_timing_get(name, C.byref(ms), C.byref(n))
    if n.value: print(f"{name.decode():24s} avg {ms.value/n.value:.4f} ms over {n.value} launches")
