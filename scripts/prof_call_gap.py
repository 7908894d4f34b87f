"""Where the time between consecutive config-2 filter calls goes: bench.py's single-caller loop (same 2^24-row resident
batches, `process_device` then `close`, kernel timing on), 64 steps after 4 warm-up steps.

Two child processes run the same loop:
  * plain: ARK_TRACE off — the step time as bench.py measures it (CUDA events around the loop) and the kernel time;
  * traced: ARK_TRACE=1 — the GPU idle time from one filter kernel's end event to the next one's start event
    (`filter_call_gap`), the host time of each native phase of ark_sql_process_device (its stderr lines), and the
    Python time per step: the step's wall time minus the native call's time.

    python scripts/prof_call_gap.py [--steps 64] [--warmup 4] [--out DIR]

Prints one table (medians over the steps, and means) and writes it as JSON to DIR/prof_call_gap.json (DIR defaults to a
directory under the system's temporary directory).
"""
import argparse
import ctypes as C
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRACE_RE = re.compile(r"\[ark trace\] sql_process_device: (.*)")
PHASES = [("plan", "plan"), ("import", "import"), ("to launch enqueued", "execute → launch enqueued"),
          ("outputs and scratch", "  of which: outputs and scratch"), ("launch", "  of which: launch (with its events)"),
          ("gpu wait", "launch enqueued → sync return (GPU)"), ("sync return to export done", "sync return → export done"),
          ("input release", "input release"), ("total", "native total")]


def child(args):
    sys.path.insert(0, ROOT)
    import torch

    import bench
    from arkflow_b200 import _lib as L
    from arkflow_b200 import arrow_ffi as F
    from arkflow_b200.processor import SqlProcessor, _check

    lib = L.lib()
    _check(lib.ark_b200_init(0))
    proc = SqlProcessor({"query": bench.QUERY})
    n_resident = min(bench.N_BATCHES, max(args.steps, 8))
    resident = []
    for b in range(n_resident):
        dev, sch = L.ArrowDeviceArray(), L.ArrowSchema()
        _check(lib.ark_synth_batch_device(bench.ROWS_PER_BATCH, b * bench.ROWS_PER_BATCH, bench.SEED, 0, bench.KEY_SPACE,
                                          C.byref(dev), C.byref(sch)))
        db = F.DeviceBatch.adopt(dev, sch)
        d, s_ = db.export()  # as bench.py: the Arrow struct tree of a resident input is built before the loop
        F.release_schema(s_)
        F.release_array(d.array)
        resident.append(db)

    def step(i):
        out = proc.process_device(resident[i % n_resident])
        rows = out.num_rows
        out.close()
        return rows

    for i in range(args.warmup):
        step(i)
    torch.cuda.synchronize()
    lib.ark_kernel_timing_reset()
    lib.ark_kernel_timing_enable(1)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    walls = []
    sys.stderr.flush()
    print("@@timed", file=sys.stderr, flush=True)
    ev0.record()
    for i in range(args.steps):
        t = time.perf_counter()
        step(i)
        walls.append((time.perf_counter() - t) * 1e6)
    torch.cuda.synchronize()
    ev1.record()
    ev1.synchronize()
    lib.ark_kernel_timing_enable(0)

    def timing(name):
        ms, n = C.c_double(), C.c_int64()
        lib.ark_kernel_timing_get(name.encode(), C.byref(ms), C.byref(n))
        return ms.value, int(n.value)

    k_ms, k_n = timing("filter_project_tma_kernel")
    g_ms, g_n = timing("filter_call_gap")
    print(json.dumps({"ms_per_step": ev0.elapsed_time(ev1) / args.steps, "kernel_ms": k_ms / max(k_n, 1), "kernels": k_n,
                      "gap_us_mean": g_ms * 1e3 / g_n if g_n else None, "gaps": g_n, "step_wall_us": walls}), flush=True)


def run_child(args, traced):
    env = dict(os.environ)
    env.pop("ARK_TRACE", None)
    if traced:
        env["ARK_TRACE"] = "1"
    cmd = [sys.executable, os.path.abspath(__file__), "--child", "--steps", str(args.steps), "--warmup", str(args.warmup)]
    p = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if p.returncode != 0:
        sys.stderr.write(p.stderr[-4000:])
        raise SystemExit(f"child ({'traced' if traced else 'plain'}) failed with exit code {p.returncode}")
    res = json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("{")][-1])
    phases = []
    if traced:
        timed = p.stderr.split("@@timed", 1)[1]
        for ln in timed.splitlines():
            m = TRACE_RE.search(ln)
            if m:
                phases.append({k.strip(): float(v) for k, v in re.findall(r"([a-z][a-z ]*?) ([0-9.]+) us", m.group(1))})
    res["phases"] = phases
    return res


def med(xs):
    return statistics.median(xs) if xs else float("nan")


def mean(xs):
    return statistics.fmean(xs) if xs else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        return child(args)

    plain = run_child(args, False)
    traced = run_child(args, True)
    ph = traced["phases"][-args.steps:]
    walls = traced["step_wall_us"]
    native = [p["total"] for p in ph]
    python = [w - n for w, n in zip(walls, native)]
    rows = [("step, CUDA events around the loop (plain)", plain["ms_per_step"] * 1e3, plain["ms_per_step"] * 1e3),
            ("filter kernel, CUDA events (plain)", plain["kernel_ms"] * 1e3, plain["kernel_ms"] * 1e3),
            ("step, CUDA events around the loop (traced)", traced["ms_per_step"] * 1e3, traced["ms_per_step"] * 1e3),
            ("GPU idle between consecutive filter kernels (traced)", traced["gap_us_mean"], traced["gap_us_mean"]),
            ("step wall time, host clock (traced)", med(walls), mean(walls))]
    for key, label in PHASES:
        vals = [p.get(key, float("nan")) for p in ph]
        rows.append((f"native: {label}", med(vals), mean(vals)))
    entry = [p["plan"] + p["import"] + p["to launch enqueued"] for p in ph]
    rows.append(("native: entry → launch enqueued", med(entry), mean(entry)))
    rows.append(("Python: step wall minus native total", med(python), mean(python)))
    print(f"{'per step (us)':<56} {'median':>9} {'mean':>9}")
    for name, m, a in rows:
        print(f"{name:<56} {m:>9.1f} {a:>9.1f}")
    out = args.out or os.path.join(tempfile.gettempdir(), "prof_call_gap")
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "prof_call_gap.json"), "w") as f:
        json.dump({"rows": [{"what": n, "median_us": m, "mean_us": a} for n, m, a in rows],
                   "plain": {k: v for k, v in plain.items() if k != "phases"}, "traced_phases": ph}, f)
    return 0


if __name__ == "__main__":
    sys.exit(main())
