#!/usr/bin/env python
"""Secondary measurements for the other BASELINE configs on ONE GPU (device-resident), each with its
algorithmic-bytes roofline fraction (SURVEY.md §8(d)).  bench.py stays the contract benchmark (config 2);
this script feeds DESIGN.md.

  config 3  GROUP BY sensor: SUM(value), COUNT(*)       24 B/row            hash_agg_kernel
  config 4  hash join probe 2^24 x build K unique keys   inputs + output     join_probe_kernel (+ gathers)
  config 5  window concat of k batches                   2 x bytes           concat_copy_kernel
  json      json_to_arrow of 63-byte messages            67 B in + 26 B out  json_parse_kernel
  protobuf  arrow_to_protobuf + protobuf_to_arrow of 2^22 schema-S rows, and the JSON pair on the same rows

Usage: python scripts/bench_configs.py [--rows 16777216] [--reps 5] [--out configs.json]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=1 << 24)
    ap.add_argument("--keys", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    ap.add_argument("--only", default="", help="comma-separated legs: groupby,join,concat,json,tojson,protobuf (default: all)")
    args = ap.parse_args()

    import numpy as np
    import pyarrow as pa
    import torch

    from arkflow_b200 import _lib as L
    from arkflow_b200 import arrow_ffi as F
    from arkflow_b200.buffer import concat_batches_device
    from arkflow_b200.processor import JsonToArrowProcessor, SqlProcessor, _check

    lib = L.lib()
    _check(lib.ark_b200_init(0))
    peak = 3350.0  # H100 SXM HBM3 data sheet, unless MEASURED_PEAKS.json says otherwise
    try:
        peak = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
    except Exception:
        pass

    def synth(n, row0=0, kind=0, keys=args.keys, seed=42):
        dev, sch = L.ArrowDeviceArray(), L.ArrowSchema()
        _check(lib.ark_synth_batch_device(n, row0, seed, kind, keys, C.byref(dev), C.byref(sch)))
        return F.DeviceBatch.adopt(dev, sch)

    def timed(fn, kernel_names):
        fn()  # warm-up (pools, plan cache, table-size hint)
        fn()
        lib.ark_kernel_timing_reset()
        lib.ark_kernel_timing_enable(1)
        torch.cuda.synchronize()
        per_call = []
        for _ in range(args.reps):  # every entry point synchronises its stream before returning
            t0 = time.perf_counter()
            fn()
            per_call.append(time.perf_counter() - t0)
        torch.cuda.synchronize()
        wall = sorted(per_call)[len(per_call) // 2]  # median: a one-off host hiccup (GC, allocator growth) is not the path's cost
        lib.ark_kernel_timing_enable(0)
        kern = {}
        for k in kernel_names:
            ms, n = C.c_double(), C.c_int64()
            lib.ark_kernel_timing_get(k.encode(), C.byref(ms), C.byref(n))
            kern[k] = {"avg_ms": ms.value / max(n.value, 1), "launches": n.value}
        return wall, kern

    results = {"peak_gbs": peak, "rows": args.rows, "keys": args.keys}
    n = args.rows
    legs = set(args.only.split(",")) if args.only else {"groupby", "join", "concat", "json", "tojson", "protobuf"}

    # ---- config 3: GROUP BY ----
    for kind, label in ((0, "int64"), (1, "float64")) if "groupby" in legs else ():
        batches = [synth(n, row0=i * n, kind=kind) for i in range(3)]
        proc = SqlProcessor({"query": "SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor"})
        state = {"i": 0}

        def step():
            out = proc.process_device(batches[state["i"] % 3])
            state["i"] += 1
            out.close()

        wall, kern = timed(step, ["hash_agg_kernel", "agg_init_kernel", "agg_compact_kernel"])
        alg = n * 24
        k = kern["hash_agg_kernel"]["avg_ms"]
        results[f"config3_group_by_{label}"] = {
            "rows_per_s_call": n / wall, "ms_per_call": wall * 1e3, "kernel_ms": k,
            "roofline": {"bound": "hbm", "achieved": alg / (k / 1e3) / 1e9 if k else None, "peak": peak,
                         "frac": (alg / (k / 1e3) / 1e9 / peak) if k else None, "algorithmic_bytes_per_launch": alg}, "kernels": kern}
        del batches

    # ---- config 4: join (probe n rows, build K unique keys) ----
    if "join" in legs:
        K = min(args.keys, 1_000_000)
        probe = synth(n, keys=K)
        bkeys = pa.array(["temp_%07d" % i for i in np.random.default_rng(0).permutation(K)])
        build = F.DeviceBatch.from_arrow(pa.record_batch({"sensor": bkeys, "w": pa.array(np.arange(K), pa.int64())}))
        jp = SqlProcessor({"query": "SELECT * FROM p JOIN b ON p.sensor = b.sensor"})

        def jstep():
            out = jp.process_tables_device({"p": probe, "b": build})
            out.close()

        wall, kern = timed(jstep, ["join_build_kernel", "join_probe_count_kernel", "join_probe_fill_kernel", "take_fixed8_kernel", "take_bytes_tile_kernel", "take_lengths_kernel"])
        alg = n * 32 + K * 24 + n * (32 + 24)
        results["config4_join"] = {"probe_rows_per_s_call": n / wall, "ms_per_call": wall * 1e3, "algorithmic_bytes": alg,
                                   "achieved_gbs_call": alg / wall / 1e9, "frac_call": alg / wall / 1e9 / peak, "kernels": kern}
        del probe, build

    # ---- config 5: concat of 16 batches of n/16 rows ----
    if "concat" in legs:
        parts = [synth(n // 16, row0=i * (n // 16)) for i in range(16)]

        def cstep():
            out = concat_batches_device(parts)
            out.close()

        wall, kern = timed(cstep, ["concat_copy_kernel", "concat_offsets_kernel"])
        alg = 2 * n * 32
        k = kern["concat_copy_kernel"]["avg_ms"]
        results["config5_concat"] = {"rows_per_s_call": n / wall, "ms_per_call": wall * 1e3, "kernel_ms": k,
                                     "roofline": {"bound": "hbm", "achieved": (2 * n * 28) / (k / 1e3) / 1e9 if k else None, "peak": peak,
                                                  "frac": ((2 * n * 28) / (k / 1e3) / 1e9 / peak) if k else None,
                                                  "note": "concat_copy_kernel moves the 28 B/row of values + string bytes; offsets (4 B/row) go through concat_offsets_kernel"},
                                     "kernels": kern}
        del parts

    # ---- json_to_arrow ----
    if "json" in legs:
        m = min(n, 1 << 22)
        msg = b'{ "timestamp": 1625000000000, "value": 10, "sensor": "temp_1" }'
        data = torch.from_numpy(np.frombuffer(msg * m, dtype=np.uint8).copy()).cuda()
        offs = torch.arange(0, (m + 1) * len(msg), len(msg), dtype=torch.int32, device="cuda")
        payload = F.DeviceBatch([F.DeviceColumn("__value__", "binary", m, data, offs, None, 0, False)], m)
        jproc = JsonToArrowProcessor({})

        def pstep():
            out = jproc.process_device(payload)
            out.close()

        wall, kern = timed(pstep, ["json_count_kernel", "json_parse_kernel", "json_strings_kernel"])
        alg = m * (len(msg) + 4) + m * 26
        k = kern["json_parse_kernel"]["avg_ms"]
        results["json_to_arrow"] = {"msgs_per_s_call": m / wall, "ms_per_call": wall * 1e3, "kernel_ms": k,
                                    "roofline": {"bound": "hbm", "achieved": alg / (k / 1e3) / 1e9 if k else None, "peak": peak,
                                                 "frac": (alg / (k / 1e3) / 1e9 / peak) if k else None, "algorithmic_bytes_per_launch": alg},
                                    "kernels": kern}
    if "tojson" in legs:
        # ---- arrow_to_json of schema S (host entry point only: the processor appends a Binary column) ----
        from arkflow_b200.processor import ArrowToJsonProcessor, MessageBatch
        from oracle.synth import synth_batch

        m = min(n, 1 << 22)
        rb = synth_batch(m, key_space=args.keys)
        aproc = ArrowToJsonProcessor({})
        mb = MessageBatch.new_arrow(rb)

        def astep():
            aproc.process(mb)

        wall, kern = timed(astep, ["arrow_to_json_measure_kernel", "arrow_to_json_write_kernel"])
        out_bytes = int(aproc.process(mb).batches[0].record_batch.column("__value__").nbytes)
        alg = m * 32 + out_bytes
        k = kern["arrow_to_json_measure_kernel"]["avg_ms"] + kern["arrow_to_json_write_kernel"]["avg_ms"]
        results["arrow_to_json"] = {"rows_per_s_call_host_to_host": m / wall, "ms_per_call": wall * 1e3, "kernel_ms": k,
                                    "roofline": {"bound": "hbm", "achieved": alg / (k / 1e3) / 1e9 if k else None, "peak": peak,
                                                 "frac": (alg / (k / 1e3) / 1e9 / peak) if k else None, "algorithmic_bytes_per_launch": alg},
                                    "kernels": kern}
    if "protobuf" in legs:
        # ---- protobuf_to_arrow / arrow_to_protobuf of schema S, and the JSON codec pair on the same records ----
        import shutil
        import tempfile

        from arkflow_b200.processor import ArrowToJsonProcessor, ArrowToProtobufProcessor, ProtobufToArrowProcessor
        from oracle.synth import synth_batch

        m = min(n, 1 << 22)
        pdir = tempfile.mkdtemp(prefix="ark_bench_proto_")  # nothing is written into the tree
        with open(os.path.join(pdir, "s.proto"), "w") as f:
            f.write('syntax = "proto3";\npackage bench;\nmessage S { int64 timestamp = 1; double value = 2; string sensor = 3; }\n')
        cfg = {"proto_inputs": [pdir], "message_type": "bench.S"}
        rows = F.DeviceBatch.from_arrow(synth_batch(m, value_kind=1, key_space=args.keys))
        codecs = {"protobuf": (ArrowToProtobufProcessor(cfg), ProtobufToArrowProcessor(cfg),
                               ["protobuf_encode_measure_kernel", "protobuf_encode_write_kernel"], ["protobuf_decode_kernel", "protobuf_strings_kernel"]),
                  "json": (ArrowToJsonProcessor({}), JsonToArrowProcessor({}),
                           ["arrow_to_json_measure_kernel", "arrow_to_json_write_kernel"], ["json_parse_kernel", "json_strings_kernel"])}
        res = {"messages": m, "schema": "timestamp Int64, value Float64, sensor Utf8 (12 B)"}
        for name, (enc, dec, enc_k, dec_k) in codecs.items():
            encoded = enc.process_device(rows)
            value = [c for c in encoded.columns if c.name == "__value__"][0]
            payload = F.DeviceBatch([value], m)
            payload_bytes = int(value.offsets[-1].item())

            def estep():
                enc.process_device(rows).close()

            def dstep():
                dec.process_device(payload).close()

            wall_e, kern_e = timed(estep, enc_k)
            wall_d, kern_d = timed(dstep, dec_k)
            k_e = sum(kern_e[k]["avg_ms"] for k in enc_k)
            k_d = kern_d[dec_k[0]]["avg_ms"]
            # encode: both passes read the 32 B/row of the columns (8 + 8 + 4 offset + 12 string bytes); the lengths (4 B/row)
            # are written and read back; the messages are written once.  decode (parse kernel): offsets + payload bytes in,
            # 8 + 8 B of values + the sensor span (8 B source, 4 B length) out per message.
            alg_e = 2 * m * 32 + 2 * m * 4 + payload_bytes
            alg_d = m * 4 + payload_bytes + m * (8 + 8 + 12)
            roof = lambda alg, k: {"bound": "hbm", "achieved": alg / (k / 1e3) / 1e9 if k else None, "peak": peak,
                                   "frac": (alg / (k / 1e3) / 1e9 / peak) if k else None, "algorithmic_bytes_per_launch": alg}
            res[name] = {"payload_bytes_per_msg": payload_bytes / m,
                         "encode": {"msgs_per_s_call": m / wall_e, "ms_per_call": wall_e * 1e3, "kernel_ms": k_e, "roofline": roof(alg_e, k_e), "kernels": kern_e},
                         "decode": {"msgs_per_s_call": m / wall_d, "ms_per_call": wall_d * 1e3, "kernel_ms": k_d, "roofline": roof(alg_d, k_d), "kernels": kern_d}}
            payload.close()
            encoded.close()
        results["protobuf_vs_json"] = res
        shutil.rmtree(pdir, ignore_errors=True)
    print(json.dumps(results, indent=1))
    if args.out:
        with open(os.path.join(ROOT, args.out), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
