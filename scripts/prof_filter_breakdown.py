#!/usr/bin/env python
"""Where the time of config 2's filter kernel goes: filter_project_tile_kernel on 2^24-row device-resident batches
(SELECT sensor, value FROM flow WHERE value >= 10), CUDA-event time per launch from ark_kernel_timing_get, for
  default         the kernel as built;
  stub_lookback   ARK_FP_DEBUG=1: the look-back is replaced by a made-up prefix (results are garbage; time only) —
                  the data path alone, the least time any look-back design can reach;
  lb_delay_0      ARK_FP_LB_DELAY=0: no sleep before the look-back's first poll;
  d2d_copy        reference line: a device-to-device torch copy of 302 MB (302 MB read + 302 MB written = the
                  kernel's 604 MB of algorithmic traffic).
The knobs are read once per process, so each variant runs in a child process of its own; the variants are alternated
--rounds times.  Prints the card's name, power limit and SM clock beside the numbers.
Usage: python scripts/prof_filter_breakdown.py [--rounds 2] [--launches 48] [--out DIR]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QUERY = "SELECT sensor, value FROM flow WHERE value >= 10"
ROWS, SEED, KEY_SPACE, N_RESIDENT, WARMUP = 1 << 24, 42, 1_000_000, 8, 4
COPY_BYTES = 302_000_000
VARIANTS = {
    "default": {},
    "stub_lookback": {"ARK_FP_DEBUG": "1"},
    "lb_delay_0": {"ARK_FP_LB_DELAY": "0"},
    "d2d_copy": {},
}


def smi(fields):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={fields}", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, timeout=30)
    return r.stdout.strip()


def child(name, launches):
    sys.path.insert(0, ROOT)
    import torch

    assert torch.cuda.is_available(), "this measurement needs a CUDA device"
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    if name == "d2d_copy":
        src = torch.empty(COPY_BYTES, dtype=torch.uint8, device="cuda")
        dst = torch.empty_like(src)
        for _ in range(WARMUP):
            dst.copy_(src)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(launches):
            dst.copy_(src)
        e1.record()
        e1.synchronize()
        ms, n = e0.elapsed_time(e1) / launches, launches
    else:
        from arkflow_b200 import _lib as L
        from arkflow_b200 import arrow_ffi as F
        from arkflow_b200.processor import SqlProcessor, _check

        lib = L.lib()
        _check(lib.ark_b200_init(0))
        proc = SqlProcessor({"query": QUERY})
        resident = []
        for b in range(N_RESIDENT):
            dev, sch = L.ArrowDeviceArray(), L.ArrowSchema()
            _check(lib.ark_synth_batch_device(ROWS, b * ROWS, SEED, 0, KEY_SPACE, C.byref(dev), C.byref(sch)))
            resident.append(F.DeviceBatch.adopt(dev, sch))
        for i in range(WARMUP):
            proc.process_device(resident[i % N_RESIDENT]).close()
        torch.cuda.synchronize()
        lib.ark_kernel_timing_reset()
        lib.ark_kernel_timing_enable(1)
        for i in range(launches):
            proc.process_device(resident[i % N_RESIDENT]).close()
        torch.cuda.synchronize()
        lib.ark_kernel_timing_enable(0)
        tot, cnt = C.c_double(), C.c_int64()
        lib.ark_kernel_timing_get(b"filter_project_tile_kernel", C.byref(tot), C.byref(cnt))
        assert cnt.value == launches, f"expected {launches} launches of filter_project_tile_kernel, got {cnt.value}"
        ms, n = tot.value / cnt.value, cnt.value
    print(json.dumps({"variant": name, "ms": ms, "launches": n, "sm_clock": smi("clocks.sm")}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--launches", type=int, default=48)
    ap.add_argument("--out", default=None, help="directory for breakdown.json")
    ap.add_argument("--variant", action="append", default=[], metavar="NAME:KEY=VALUE[,KEY=VALUE]",
                    help="an extra variant of the kernel under the given environment (e.g. lb_delay_300:ARK_FP_LB_DELAY=300)")
    ap.add_argument("--child", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        child(a.child, a.launches)
        return
    for v in a.variant:
        name, _, kv = v.partition(":")
        VARIANTS[name] = dict(x.split("=", 1) for x in kv.split(","))
    card = smi("name,power.limit,clocks.max.sm")
    print(f"card, power limit, max SM clock: {card}")
    runs = {k: [] for k in VARIANTS}
    for r in range(a.rounds):
        for name, env in VARIANTS.items():
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", name, "--launches", str(a.launches)],
                               env={**os.environ, **env}, capture_output=True, text=True, cwd=ROOT)
            if p.returncode != 0:
                sys.stderr.write(p.stdout + p.stderr)
                raise SystemExit(f"variant {name} failed (exit {p.returncode})")
            res = json.loads(p.stdout.strip().splitlines()[-1])
            runs[name].append(res)
            print(f"round {r}  {name:14s} {res['ms']:.4f} ms/launch over {res['launches']}  (SM clock {res['sm_clock']})", flush=True)
    best = {k: min(x["ms"] for x in v) for k, v in runs.items()}
    algo_bytes = 604e6
    print(f"\n{'variant':14s} {'ms per launch (each round)':32s} algorithmic TB/s (best)")
    for k, v in runs.items():
        print(f"{k:14s} {', '.join(f'{x['ms']:.4f}' for x in v):32s} {algo_bytes / best[k] / 1e9:.2f}")
    gap = best["default"] - best["stub_lookback"]
    print(f"\nlook-back share of the default kernel: {gap:.4f} ms = {gap / best['default']:.1%} (default - stubbed)")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "breakdown.json"), "w") as f:
            json.dump({"card": card, "runs": runs}, f, indent=1)


if __name__ == "__main__":
    main()
