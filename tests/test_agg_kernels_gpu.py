"""Every GROUP BY kernel against the oracle (oracle/sql_oracle.py), at the shapes and values where kernels go wrong.

Several implementations accumulate into the same table (DESIGN.md §4.2), each with its own accumulate, merge and
identity logic: the per-CTA shared-memory table (hash_agg_tile_kernel; ≤ 64 slots reduce in the warp first), the
TMA-staged kernel (hash_agg_staged_kernel), the register-prefetch kernel (hash_agg_stream_kernel), the general row
kernel (hash_agg_kernel) and a cached key dictionary whose accumulators agg_reset_acc_kernel resets.  ARK_AGG_KERNEL,
which forces a kernel, is read once per process, so each path runs in a child process: this process builds the inputs
and the oracle's answers, the child runs the library and writes its results as Arrow IPC together with the kernels
each call launched.  Every case asserts that the intended kernel ran, or that the path declines the case by design (VM
predicate, two keys, Boolean key, more than six accumulators for the tile kernel): a silent fallback fails.

Comparison: keys, integers and counts exactly; Float64 MIN / MAX bitwise (totalOrder separates -0.0 from +0.0 and NaN
payloads); Float64 SUM / AVG by tests/agg_util.py (NaN ↔ NaN, ±inf exact, else the §7 bound).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -2 ** 63, 2 ** 63 - 1
TABLE_KERNELS = ("hash_agg_tile_kernel", "hash_agg_staged_kernel", "hash_agg_stream_kernel", "hash_agg_kernel")
KERNELS = TABLE_KERNELS + ("agg_reset_acc_kernel",)
# quiet and signalling NaNs of both signs; 0x7FFF… and 0xFFFF… have the totalOrder keys INT64_MAX / INT64_MIN, the
# identities of the MIN / MAX accumulators
NAN_BITS = np.array([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x7FFFFFFFFFFFFFFF, 0xFFFFFFFFFFFFFFFF,
                     0x7FF4000000000123], dtype=np.uint64)
NANS = NAN_BITS.view(np.float64)


# ---- inputs -----------------------------------------------------------------------------------------------------------
def _utf8_key(x):
    """Key lengths 0, 1-5, 12, 13 and 40: the 13-byte keys share their first 12 bytes with a 12-byte key, the 40-byte
    keys share a 12-byte prefix among themselves (both are stored by row reference and compared past the prefix)."""
    if x == 0:
        return ""
    c = x % 4
    if c == 0:
        return f"{x:012d}"
    if c == 1:
        return "shared_pref_" + f"{x:028d}"
    if c == 2:
        return f"{x:013d}"
    return f"{x:x}"


def _key_values(kind, g):
    xs = range(g)
    if kind == "utf8":
        return pa.array([_utf8_key(x) for x in xs], pa.utf8())
    if kind == "short":  # ≤ 12 bytes: self-contained keys, so the table may be cached across batches
        return pa.array(["" if x == 0 else f"{x:x}" for x in xs], pa.utf8())
    if kind == "binary":  # NUL bytes inside keys
        return pa.array([_utf8_key(x).encode().replace(b"0", b"\x00") for x in xs], pa.binary())
    edges = [I64_MIN, I64_MAX, 0, -1]
    return pa.array(edges[:g] + [((x * 0x9E3779B97F4A7C15 + 2 ** 63) % 2 ** 64) - 2 ** 63 for x in range(4, g)], pa.int64())


def make_table(n, g, key="utf8", seed=0, code_lo=0, long_region=False):
    """n rows over group codes [code_lo, g).  Groups 1 / 2 hold only INT64_MAX / INT64_MIN in `i`; `f` takes, by group
    code mod 8: finite values, NaNs only, +inf only, -inf only, ±0.0 (some groups -0.0 only), every edge mixed with
    finite values, ±1e300 with finite values, ±5e-324 — finite magnitudes stay far from overflowing any partial sum."""
    rng = np.random.default_rng(seed)
    codes = rng.integers(code_lo, g, n)
    if long_region:  # a region of 40-byte keys only: its tiles overflow the staging window sized from the average
        lo, hi = n // 3, n // 3 + min(n // 4, 400_000)
        codes[lo:hi] = np.minimum((codes[lo:hi] // 4) * 4 + 1, g - 1 - (g - 2) % 4)
    cols = {}
    if key == "bool":
        cols["k"] = pa.array(rng.random(n) < 0.5, pa.bool_(), mask=rng.random(n) < 0.05)
    else:
        cols["k"] = _key_values("int64" if key == "pair" else key, g).take(pa.array(codes))
        cols["k"] = pc.if_else(pa.array(rng.random(n) < 0.02), pa.nulls(n, cols["k"].type), cols["k"])  # NULL keys
    cols["g2"] = pa.array(codes % 3, pa.int64())  # second key of two-key cases
    i = rng.integers(-2 ** 62, 2 ** 62, n)
    i[codes == 1] = I64_MAX
    i[codes == 2] = I64_MIN
    e3 = codes == 3
    i[e3] = rng.choice(np.array([I64_MIN, I64_MAX, 0, -1], np.int64), int(e3.sum()))
    cols["i"] = pa.array(i, pa.int64(), mask=rng.random(n) < 0.1)
    f = rng.uniform(-1e3, 1e3, n)
    mode = codes % 8
    edges = np.concatenate([NANS, [np.inf, -np.inf, 0.0, -0.0, 5e-324, -5e-324, 1e300, -1e300, 1.5, -2.25]])

    def put(m, choices):
        f[m] = rng.choice(np.asarray(choices, np.float64), int(m.sum()))

    put(mode == 1, NANS)
    f[mode == 2] = np.inf
    f[mode == 3] = -np.inf
    put(mode == 4, [0.0, -0.0])
    f[(codes % 16) == 12] = -0.0
    put(mode == 5, edges)
    put(mode == 6, [1e300, -1e300, 3.0, -7.5])
    put(mode == 7, [5e-324, -5e-324])
    cols["f"] = pa.array(f, pa.float64(), mask=rng.random(n) < 0.1)
    s = np.array(["", "a", "some text", "x" * 30], dtype=object)[rng.integers(0, 4, n)]
    cols["s"] = pa.array(s.tolist(), pa.utf8(), mask=rng.random(n) < 0.2)
    cols["b"] = pa.array([v.encode() for v in s.tolist()], pa.binary(), mask=rng.random(n) < 0.3)
    cols["t"] = pa.array(rng.random(n) < 0.5, pa.bool_(), mask=rng.random(n) < 0.25)
    cols["p"] = pa.array(rng.integers(-5, 6, n), pa.int64(), mask=rng.random(n) < 0.05)
    q = rng.uniform(-2, 2, n)
    q[rng.random(n) < 0.05] = np.nan
    q[rng.random(n) < 0.05] = -0.0
    q[rng.random(n) < 0.05] = 0.0
    cols["q"] = pa.array(q, pa.float64(), mask=rng.random(n) < 0.05)
    cols["j"] = pa.array(rng.integers(-10 ** 6, 10 ** 6, n), pa.int64())
    cols["m"] = pa.array(rng.integers(-2 ** 62, 2 ** 62, n), pa.int64())
    cols["h"] = pa.array(rng.uniform(-100, 100, n), pa.float64())
    return pa.record_batch(cols)


def _normalised(rb):
    return pa.RecordBatch.from_arrays([pa.concat_arrays([c]) for c in rb.columns], schema=rb.schema)


# ---- queries ----------------------------------------------------------------------------------------------------------
Q_INT = "SELECT {K}, SUM(i), AVG(i), MIN(i), MAX(i), COUNT(i) FROM flow{W} GROUP BY {K}"
Q_FLT = "SELECT {K}, SUM(f), AVG(f), MIN(f), MAX(f), COUNT(f) FROM flow{W} GROUP BY {K}"
Q_CNT = "SELECT {K}, COUNT(*), COUNT(i), COUNT(f), COUNT(s), COUNT(b), COUNT(t) FROM flow{W} GROUP BY {K}"
Q_WIDE = "SELECT {K}, SUM(j), AVG(j), MIN(i), MAX(f), COUNT(s), COUNT(*) FROM flow{W} GROUP BY {K}"  # 8 accumulators
Q_ARGS3 = "SELECT {K}, SUM(j), MAX(m), MIN(h), AVG(h) FROM flow{W} GROUP BY {K}"  # 3rd argument is loaded in place
Q_NONNULL = "SELECT {K}, COUNT(*), SUM(j), MIN(j), MAX(m), AVG(j) FROM flow{W} GROUP BY {K}"  # non-null, ≤ 2 arguments
Q_NONNULL_F = "SELECT {K}, SUM(h), MAX(h), MIN(h), COUNT(*) FROM flow{W} GROUP BY {K}"
Q_AUX = "SELECT {K}, COUNT(f), SUM(af), COUNT(i), SUM(ai), COUNT(j), SUM(aj), COUNT(h), SUM(ah) FROM flow{W} GROUP BY {K}"
W_INT, W_FLT, W_FLT2, W_VM = " WHERE p > 0", " WHERE q < 0.0", " WHERE q >= 1.5", " WHERE p > 0 AND q < 0.5"
FLOAT_SUMS = {"sum(flow.f)": "f", "avg(flow.f)": "f", "avg(flow.i)": "i", "avg(flow.j)": "j", "avg(flow.h)": "h",
              "sum(flow.h)": "h"}

ROWS_EDGES = (1, 255, 257, 1023, 1025, 2049)
TABLES = {f"u{n}": dict(n=n, g=12, seed=n) for n in ROWS_EDGES}
TABLES.update({
    "i_lo": dict(n=4099, g=10, key="int64", seed=1),
    "bool": dict(n=10_000, g=40, key="bool", seed=2),
    "u_mid": dict(n=100_003, g=300, seed=3),
    "b_mid": dict(n=50_000, g=300, key="binary", seed=4),
    "pair": dict(n=30_000, g=200, key="pair", seed=5),
    "u_hi": dict(n=300_000, g=100_000, seed=6),
    "b_hi": dict(n=120_000, g=40_000, key="binary", seed=7),
    "i_hi": dict(n=200_000, g=150_000, key="int64", seed=8),
    "u_big": dict(n=(1 << 21) + 3, g=60_000, seed=9, long_region=True),  # every persistent CTA reuses both ring stages
    "c_a": dict(n=60_000, g=3000, key="int64", seed=10),
    "c_b": dict(n=60_000, g=4500, key="int64", seed=11, code_lo=1500),
    "s_a": dict(n=60_000, g=3000, key="short", seed=12),
    "s_b": dict(n=60_000, g=4500, key="short", seed=13, code_lo=1500),
    "sl_lo": dict(n=5000 + 1237, g=12, seed=14),
    "sl_hi": dict(n=60_000 + 1237, g=20_000, seed=15),
    "sl_i": dict(n=60_000 + 1237, g=20_000, key="int64", seed=16),
})
LOW = [f"u{n}" for n in ROWS_EDGES] + ["i_lo", "bool"]
MID = ["u_mid", "b_mid", "pair"]
HIGH = ["u_hi", "b_hi", "i_hi"]
FULL = [Q_INT, Q_FLT, Q_CNT, Q_WIDE, Q_ARGS3]
PRED = [(Q_INT, W_INT), (Q_FLT, W_FLT), (Q_ARGS3, W_FLT2), (Q_CNT, W_VM)]

PATHS = {  # name → (environment, kernel it selects)
    "tile": ({}, "hash_agg_tile_kernel"),
    "staged": ({"ARK_AGG_KERNEL": "staged"}, "hash_agg_staged_kernel"),
    "stream": ({"ARK_AGG_KERNEL": "stream"}, "hash_agg_stream_kernel"),
    "general": ({"ARK_AGG_KERNEL": "general"}, "hash_agg_kernel"),
}


def _keys_of(table):
    return "k, g2" if TABLES[table].get("key") == "pair" else "k"


def _cases(path):
    """(case id, table, query, calls, slice offset or None, device) of one path."""
    out = []

    def add(table, q, w="", calls=1, off=None, device=False):
        query = q.format(K=_keys_of(table), W=w)
        out.append((f"{path}-{len(out)}", table, query, calls, off, device))

    # the tile kernel: ≤ 16 groups from the second call of a processor on (≤ 64 slots), a few hundred groups
    calls = 2 if path == "tile" else 1
    tables = LOW + MID + ([] if path == "tile" else HIGH)
    for t in tables:
        for q in (FULL if TABLES[t]["n"] >= 2049 else [Q_INT, Q_FLT, Q_CNT]):
            add(t, q, calls=calls)
        if TABLES[t]["n"] >= 4099:
            for q, w in PRED:
                add(t, q, w, calls=calls)
    if path != "tile":
        for q in (Q_INT, Q_ARGS3, Q_CNT):
            add("u_big", q)
        for t in HIGH + ["u_big"]:  # every argument non-null: the staged kernel stages both
            add(t, Q_NONNULL)
            add(t, Q_NONNULL_F, W_FLT)
    if path in ("tile", "staged", "stream"):  # device slices (and host slices) of the default, staged and prefetch paths
        for off in (1, 3, 7, 1237):
            for t in ("sl_lo", "sl_hi", "sl_i"):
                for device in (True, False):
                    add(t, Q_FLT if off % 2 else Q_CNT, off=off, device=device, calls=calls if t == "sl_lo" else 1)
                    add(t, Q_ARGS3, W_INT, off=off, device=device, calls=calls if t == "sl_lo" else 1)
    return out


def _expected(path, table, query, call):
    """(kernel that call number `call` of a case must have run, table kernels allowed to run)."""
    env, kernel = PATHS[path]
    key = TABLES[table].get("key", "utf8")
    if " AND " in query or key == "pair":  # VM predicate, two keys: only the general kernel takes them
        return "hash_agg_kernel", {"hash_agg_kernel"}
    if path == "tile":
        # A fresh processor starts from a 2^16-slot table, too large for the tile kernel: its first call runs the kernel
        # the default picks for a table that fits the L2, the staged one.  From the second call on the table is sized
        # from the groups seen.  Q_WIDE has 8 accumulators, the tile kernel keeps ≤ 6.
        if call > 0 and "AVG(j), MIN(i)" not in query:
            return kernel, {kernel}
        kernel = "hash_agg_staged_kernel"
    if key == "bool" and kernel != "hash_agg_tile_kernel":  # the staged and prefetch kernels take Utf8 / Binary / Int64 keys
        return "hash_agg_kernel", {"hash_agg_kernel"}
    return kernel, {kernel}


# ---- child: runs the library -----------------------------------------------------------------------------------------
def _child(spec_path):
    import ctypes as C

    sys.path.insert(0, ROOT)
    from arkflow_b200 import _lib as L
    from arkflow_b200.arrow_ffi import DeviceBatch
    from arkflow_b200.processor import MessageBatch, SqlProcessor, _check

    spec = json.load(open(spec_path))
    d = os.path.dirname(spec_path)
    lib = L.lib()
    _check(lib.ark_b200_init(0))
    lib.ark_kernel_timing_enable(1)
    tables, procs, report = {}, {}, {}
    for c in spec["cases"]:
        if c["table"] not in tables:
            with pa.ipc.open_file(os.path.join(d, c["table"] + ".arrow")) as r:
                tables[c["table"]] = r.get_batch(0)
        rb = tables[c["table"]]
        if c["off"] is not None:
            rb = rb.slice(c["off"], rb.num_rows - 1237)
        p = procs.setdefault(c["proc"], SqlProcessor({"query": c["query"]})) if c.get("proc") else SqlProcessor({"query": c["query"]})
        runs = []
        for k in range(c["calls"]):
            lib.ark_kernel_timing_reset()
            try:
                if c["device"]:
                    out = p.process_device(DeviceBatch.from_arrow(rb, keep_offsets=True)).to_arrow()
                else:
                    out = p.process(MessageBatch.new_arrow(rb)).batches[0].record_batch
            except Exception as e:  # reported, and failed, by the parent
                runs.append({"error": repr(e)})
                continue
            counts = {}
            for name in KERNELS:
                ms, n = C.c_double(), C.c_int64()
                lib.ark_kernel_timing_get(name.encode(), C.byref(ms), C.byref(n))
                counts[name] = n.value
            # the hash_agg_kernel timer counts the staged and register-prefetch launches too (the GROUP BY table kernel,
            # whichever ran): the general row kernel's own launches are the rest
            counts["hash_agg_kernel"] -= counts["hash_agg_staged_kernel"] + counts["hash_agg_stream_kernel"]
            with pa.ipc.new_file(os.path.join(d, f"{c['id']}.{k}.arrow"), out.schema) as w:
                w.write_batch(out)
            runs.append({"counts": counts})
        report[c["id"]] = runs
    json.dump(report, open(os.path.join(d, "report.json"), "w"))
    print("CHILD_OK")


def _run_child(tmp, cases, env):
    spec = os.path.join(tmp, "spec.json")
    json.dump({"cases": cases}, open(spec, "w"))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), spec], capture_output=True, text=True, timeout=900,
                       env=dict(os.environ, **env))
    assert r.returncode == 0 and "CHILD_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    return json.load(open(os.path.join(tmp, "report.json")))


# ---- parent: the oracle and the comparison -----------------------------------------------------------------------------
_ORACLE = {}
_INPUTS = {}


def _input(table):
    if table not in _INPUTS:
        _INPUTS[table] = make_table(**TABLES[table])
    return _INPUTS[table]


def _oracle(table, query, off):
    from oracle.sql_oracle import sql_process

    k = (table, query, off)
    if k not in _ORACLE:
        rb = _input(table)
        if off is not None:
            rb = _normalised(rb.slice(off, rb.num_rows - 1237))
        want = sql_process(rb, query)
        aux = None
        if any(n in FLOAT_SUMS for n in want.schema.names):
            w = query[query.index(" FROM flow") + len(" FROM flow"):query.index(" GROUP BY")]
            absd = {f"a{c}": pc.abs(pc.cast(rb.column(c), pa.float64(), safe=False)) for c in "fijh"}
            rba = pa.RecordBatch.from_arrays(list(rb.columns) + list(absd.values()), names=rb.schema.names + list(absd))
            aux = sql_process(rba, Q_AUX.format(K=_keys_of(table), W=w))
        _ORACLE[k] = (want, aux)
    return _ORACLE[k]


def _sorted(rb, keys):
    return pa.Table.from_batches([rb]).sort_by([(c, "ascending") for c in keys]).combine_chunks()


def _compare(got, want, aux, keys, what):
    assert got.schema.names == want.schema.names, (what, got.schema, want.schema)
    assert [f.type for f in got.schema] == [f.type for f in want.schema], (what, got.schema, want.schema)
    assert got.num_rows == want.num_rows, (what, got.num_rows, want.num_rows)
    from agg_util import float_sum_mismatches

    g, w = _sorted(got, keys), _sorted(want, keys)
    a = _sorted(aux, keys) if aux is not None else None
    for name in want.schema.names:
        gc, wc = g.column(name).combine_chunks(), w.column(name).combine_chunks()
        if name in keys or not pa.types.is_floating(wc.type):
            assert gc.equals(wc), (what, name)
            continue
        assert gc.is_null().equals(wc.is_null()), (what, name, "validity")
        gv = pc.fill_null(gc, 0.0).to_numpy(zero_copy_only=False)
        wv = pc.fill_null(wc, 0.0).to_numpy(zero_copy_only=False)
        if name in FLOAT_SUMS:
            c = FLOAT_SUMS[name]
            n_g = pc.fill_null(a.column(f"count(flow.{c})"), 0).to_numpy(zero_copy_only=False)
            s_abs = pc.fill_null(a.column(f"sum(flow.a{c})"), 0.0).to_numpy(zero_copy_only=False)
            bad = float_sum_mismatches(gv, wv, n_g, s_abs, avg=name.startswith("avg"))
            assert len(bad) == 0, (what, name, [(g.column(keys[0])[int(i)].as_py(), gv[i], wv[i]) for i in bad[:5]])
        else:  # MIN / MAX: bit for bit
            bad = np.flatnonzero(gv.view(np.uint64) != wv.view(np.uint64))
            assert len(bad) == 0, (what, name, [(hex(gv.view(np.uint64)[i]), hex(wv.view(np.uint64)[i])) for i in bad[:5]])


def _run_path(path, tmp, cases, check_kernels=True):
    env, _ = PATHS[path]
    for t in sorted({c[1] for c in cases}):
        rb = _input(t)
        with pa.ipc.new_file(os.path.join(tmp, t + ".arrow"), rb.schema) as wr:
            wr.write_batch(rb)
    spec = [dict(id=i, table=t, query=q, calls=n, off=off, device=dev, proc=proc) for i, t, q, n, off, dev, proc in cases]
    report = _run_child(str(tmp), spec, env)
    for i, t, q, n, off, dev, proc in cases:
        want, aux = _oracle(t, q, off)
        keys = [k.strip() for k in _keys_of(t).split(",")]
        for k, run in enumerate(report[i]):
            what = (path, t, q, off, dev, k)
            assert "error" not in run, (what, run)
            with pa.ipc.open_file(os.path.join(str(tmp), f"{i}.{k}.arrow")) as r:
                got = r.get_batch(0) if r.num_record_batches else r.schema.empty_table().to_batches()[0]
            _compare(got, want, aux, keys, what)
            if check_kernels:
                need, allowed = _expected(path, t, q, k)
                counts = run["counts"]
                assert counts[need] >= 1, (what, need, counts)
                assert all(counts[x] == 0 for x in TABLE_KERNELS if x not in allowed), (what, allowed, counts)
    return report


@pytest.mark.parametrize("path", list(PATHS))
def test_kernel_path_matches_oracle(gpu, tmp_path, path):
    cases = [c + (None,) for c in _cases(path)]
    _run_path(path, tmp_path, cases)


def test_cached_key_dictionary_resets_accumulators(gpu, tmp_path):
    """One processor, four batches: the first grows the table, the second builds it at its final size, the third (the
    same batch again) and the fourth (other keys and values) reuse its key dictionary and only reset the accumulators
    (agg_reset_acc_kernel).  Every batch's MIN / MAX, float ones included, must start from the identities again."""
    cases = []
    for name, (a, b), q in (("ci", ("c_a", "c_b"), Q_FLT), ("ci2", ("c_a", "c_b"), Q_INT), ("cs", ("s_a", "s_b"), Q_INT)):
        for step, t in enumerate((a, a, a, b)):
            cases.append((f"{name}-{step}", t, q.format(K="k", W=""), 1, None, step == 3, name))
    report = _run_path("tile", tmp_path, cases, check_kernels=False)
    for c in cases:
        counts = report[c[0]][0]["counts"]
        if int(c[0].rsplit("-", 1)[1]) >= 2:
            assert counts["agg_reset_acc_kernel"] >= 1 and counts["hash_agg_staged_kernel"] >= 1, (c, counts)
            assert counts["hash_agg_tile_kernel"] == 0, (c, counts)


if __name__ == "__main__":
    _child(sys.argv[1])
