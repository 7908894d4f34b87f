"""The json_to_arrow decoder (csrc/json.cu) against the oracle (oracle/json_oracle.py), at the shapes and bytes where
it can go wrong.

The decoder has two routes: the optimistic one-pass json_parse_kernel<2> (payload i → row i), and, when a payload is
NULL, blank or holds several records, or any error shows up, the count pass json_parse_kernel<0> (timed as
json_count_kernel) followed by json_parse_kernel<1>.  Each CTA parses its 128 payloads from a shared-memory copy when
their 16-byte-aligned window fits the staging size, else in place from global memory.  ARK_JSON_NO_STAGE turns the
staging off and ARK_JSON_TWO_PASS skips the optimistic pass; both are read once per process, so every path runs in a
child process: this process builds the inputs and the oracle's answers, the child runs the library (host entry and
process_device, plus device slices that keep their offsets) and writes its results as Arrow IPC with the kernels each
call launched.

Every case asserts the route it took (launch counts of the parse, count, string and list kernels) and, through a model
of the staging rule (`stage_bytes`, `cta_staged`), the mix of staged and in-place CTAs it claims.  Results must equal
the oracle's: names and types, Array.equals (Float64 bit for bit), Struct children as arrays (NULL under a NULL or
missing struct row), and every array must pass validate(full=True), which also rejects invalid UTF-8.
"""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

JS_THREADS = 128
PATHS = {
    "default": {},
    "no_stage": {"ARK_JSON_NO_STAGE": "1"},
    "two_pass": {"ARK_JSON_TWO_PASS": "1"},
    "no_stage_two_pass": {"ARK_JSON_NO_STAGE": "1", "ARK_JSON_TWO_PASS": "1"},
}
KERNELS = ("json_parse_kernel", "json_count_kernel", "json_strings_kernel", "json_list_count_kernel", "json_list_fill_kernel",
           "json_quoted_numbers_kernel")


# ---- the staging rule of json_to_arrow_device / json_parse_kernel ------------------------------------------------------
def stage_bytes(data_bytes, n, no_stage=False):
    """Shared-memory staging per CTA: round_up((int64)(avg * 128 * 1.25) + 256, 1024) when the payloads average at most
    256 bytes, else 0 (every CTA parses in place)."""
    avg = data_bytes / n
    if no_stage or avg > 256.0:
        return 0
    return -(-(int(avg * JS_THREADS * 1.25) + 256) // 1024) * 1024


def cta_staged(offsets, stage, keep_offsets):
    """Per CTA, whether its window [a0 & ~15, (a1 + 15) & ~15) fits `stage` bytes; a0 / a1 are the addresses of its first
    payload byte and one past its last.  The data buffer is 16-byte aligned: the host entry copies the bytes from
    offsets[0] on, a keep_offsets device slice hands over its parent buffer, so byte o sits at o (mod 16)."""
    offs = np.asarray(offsets, np.int64)
    n = len(offs) - 1
    base = 0 if keep_offsets else -int(offs[0])
    i0 = np.arange(0, n, JS_THREADS)
    o0, o1 = offs[i0], offs[np.minimum(i0 + JS_THREADS, n)]
    lo, hi = (o0 + base) & ~15, (o1 + base + 15) & ~15
    return (stage > 0) & (o1 > o0) & (hi - lo <= stage)


def staging_mix(rb, off, keep_offsets):
    col = rb.column(0)
    if off is not None:
        col = col.slice(off, len(col) - off)
    offs = np.frombuffer(col.buffers()[1], np.int32)[col.offset:col.offset + len(col) + 1]
    st = cta_staged(offs, stage_bytes(int(offs[-1]) - int(offs[0]), len(col)), keep_offsets)
    return "staged" if st.all() else "inplace" if not st.any() else "mixed"


# ---- inputs -----------------------------------------------------------------------------------------------------------
STRS = ["", "plain", 'q"uote', "back\\slash", "tab\tnl\nret\r", "é", "漢字", "\U0001F600", "\x00c\x1f", "/",
        "\u007f\u0080߿ࠀ￿\U00010000\U0010FFFF"]


def _f64(i):
    """A double from i: ordinary values, subnormals, huge, -0.0 and integers past 2^53 in turn."""
    k = i % 6
    if k == 0:
        return (i * 0.37) - 1e3
    if k == 1:
        return math.ldexp((i * 2654435761) % 2 ** 52 + 1, -1074)  # subnormal / tiny
    if k == 2:
        return math.ldexp((i * 40503) % 2 ** 53 + 1, 900)
    if k == 3:
        return -0.0
    if k == 4:
        return float(2 ** 53 + 2 * i)
    return 1.0 / (i + 3)


def flat_record(i, extra=None):
    rec = {"id": (i * 7919) - (2 ** 62 if i % 11 == 5 else 0), "f": _f64(i), "s": STRS[i % len(STRS)] + str(i),
           "b": i % 3 == 0, "z": None}
    if extra:
        rec.update(extra)
    return json.dumps(rec, ensure_ascii=i % 2 == 0).encode()


def binary_batch(payloads):
    return pa.record_batch([pa.array(payloads, pa.binary())], names=["__value__"])


def pad_record(i, length):
    """A flat record of exactly `length` bytes (≥ 24)."""
    head = b'{"id":%d,"s":"' % i
    body = length - len(head) - 2
    assert body >= 0, length
    return head + bytes(97 + (i + k) % 26 for k in range(body)) + b'"}'


def window_payloads():
    """30 CTAs of 48-byte payloads, except CTA 5 whose bytes are exactly the staging size and CTA 9 with 16 bytes more:
    every CTA starts 16-byte aligned, so CTA 5 fills the staging buffer to its last byte, CTA 9 is parsed in place, and
    the last CTA's window ends on the column's last byte."""
    n_cta, base = 30, 48
    lens = np.full(n_cta * JS_THREADS, base, np.int64)
    s = stage_bytes(lens.sum(), len(lens))
    for _ in range(10):
        lens[:] = base
        for t, extra in ((5, 0), (9, 16)):
            total = s + extra
            lens[t * JS_THREADS:(t + 1) * JS_THREADS] = total // JS_THREADS
            lens[t * JS_THREADS:t * JS_THREADS + total % JS_THREADS] += 1
        new = stage_bytes(lens.sum(), len(lens))
        if new == s:
            break
        s = new
    assert stage_bytes(lens.sum(), len(lens)) == s and (JS_THREADS * base) % 16 == 0 and s % 16 == 0
    return [pad_record(i, int(n)) for i, n in enumerate(lens)], s


def avg_payloads(target_total, n):
    lens = np.full(n, target_total // n, np.int64)
    lens[:target_total - int(lens.sum())] += 1
    return [pad_record(i, int(x)) for i, x in enumerate(lens)]


def field_records(k, n=300):
    """k fields of every scalar type; later records list their keys rotated, so the key lookup wraps around."""
    out = []
    for i in range(n):
        items = []
        for j in range(k):
            name = "f%02d" % j
            v = [i * 31 + j, _f64(i + j), "v%d_%dé" % (i, j), (i + j) % 2 == 0, None][j % 5]
            items.append((name, v))
        if i:
            r = i % k
            items = items[r:] + items[:r]
        out.append(json.dumps(dict(items), ensure_ascii=i % 2 == 1).encode())
    return out


N47, N48, N49 = "n" * 47, "m" * 48, "L" * 48 + "x"
N49U = "é" * 24 + "y"  # 49 bytes of UTF-8


def _esc_all(name):
    """Every character of `name` as \\u escapes (a surrogate pair above the BMP)."""
    return "".join(json.dumps(ch)[1:-1] if ord(ch) > 0xFFFF else "\\u%04x" % ord(ch) for ch in name)


def names_records(wide):
    """Keys that are prefixes of each other, names of 47, 48 and 49 bytes (inline vs pool), keys written with escapes in
    the first record and in later ones, duplicate keys and unknown keys that extend known ones."""
    first = b'{"a": 1, "ab": "x", "abc": 2.5, "abcd": true, "%s": 1, "%s": 2, "%s": 3, "%s": "u", "\\u0061b\\u00e9": 5, "\\ud83d\\ude00": 6' % (
        N47.encode(), N48.encode(), N49.encode(), N49U.encode())
    if wide:
        first += b"".join(b', "w%02d": %d' % (j, j) for j in range(12))
    out = [first + b"}"]
    for i in range(1, 400):
        k = i % 6
        if k == 0:
            p = b'{"abcd": false, "abc": %d.5, "ab": "y%d", "a": %d}' % (i, i, i)  # reversed
        elif k == 1:
            p = b'{"a": %d, "a": %d, "abcde": 1, "ab ": 2, "%s": %d, "%s": %d}' % (i, i + 1, N48.encode() + b"z", i, N49.encode(), i)
        elif k == 2:
            p = b'{"%s": %d, "%s": "%s", "\\u0061\\u0062": "e%d", "\\ud83d\\ude00": %d, "ab\\u00e9": %d}' % (
                _esc_all(N49).encode(), i, _esc_all(N49U).encode(), _esc_all("é%d" % i).encode(), i, i, i)
        elif k == 3:
            p = ('{"\U0001F600": %d, "abé": %d, "%s": %d, "%s": %d}' % (i, i, N47, i, N47[:-1], i)).encode()
        elif k == 4:
            p = b'{"ab": null, "ab": "last%d", "abc": 1e%d, "zz": {"a": [1, "\\u00e9"]}}' % (i, i % 300)
        else:
            p = b'{}'
        if wide and i % 2:
            p = p[:-1] + (b", " if p != b"{}" else b"") + b", ".join(b'"w%02d": %d' % (j, i * j) for j in range(11, -1, -1)) + b"}"
        out.append(p)
    return out


ESC_VALUES = [b'\\"', b"\\\\", b"\\/", b"\\b", b"\\f", b"\\n", b"\\r", b"\\t", b"\\u0000", b"\\u007f", b"\\u007F", b"\\u0080",
              b"\\u07ff", b"\\u07FF", b"\\u0800", b"\\uffff", b"\\uFFFF", b"\\ud800\\udc00", b"\\uD800\\uDC00", b"\\udbff\\udfff",
              b"\\uDBFF\\uDFFF", b"\\uDbFf\\uDfFf", b"\\ud83d\\ude00", b"\\u00e9t\\u00E9"]
RAW_VALUES = ["\u007f", "\u0080", "߿", "ࠀ", "�", "￿", "\U00010000", "\U0010FFFF", "aé漢\U0001F600z"]


def string_payloads():
    out = [b'{"s": "", "t": "x", "i": 0, "f": 0.5}'] * 2  # the slice from payload 1 infers the same schema
    for i in range(2, 600):
        e = ESC_VALUES[i % len(ESC_VALUES)]
        r = RAW_VALUES[i % len(RAW_VALUES)].encode()
        s = [e, r, b"", e * 3 + r, r + e + b"tail", b"x" * (i % 40) + e][i % 6]
        # quoted numbers, some written with escapes: decoded first, then parsed
        q = [b"%d" % i, b"1\\u0032", b"\\u002d7", b"\\u0031e\\u0032", b"+\\u0035", b"\\u0039" * 18][i % 6]
        qf = [b"0.25", b"\\u0031.\\u0035", b"-\\u0030.0", b"1e-\\u0033\\u0030\\u0038", b"2.5e\\u002b3", b"\\u0030." + b"\\u0031" * 30][i % 6]
        out.append(b'{"s": "%s", "t": "%s", "i": "%s", "f": "%s"}' % (s, r, q, qf))
    return out


def long_string_payloads(mixed):
    big = ("é" * 100 + "A\\n" * 50).encode()
    if mixed:
        p = [flat_record(i) for i in range(4000)]
        p[1500] = b'{"id": 1, "s": "%s"}' % (big * 250)  # 70 KB
        return p
    return [b'{"id": %d, "s": "%s"}' % (i, big * (240 + i)) for i in range(8)] + [flat_record(i) for i in range(300)]


def list_payloads():
    first = b'{"li": [1, 2], "lf": [1.5, 2], "lb": [true], "ls": ["a", "\\u00e9\\n"], "ln": [], "lnn": [null], "id": 0}'
    out = [first]
    for i in range(1, 700):
        k = i % 5
        if k == 0:
            p = b'{"li": [], "lf": [], "lb": [], "ls": [], "ln": [], "lnn": [], "id": %d}' % i
        elif k == 1:
            p = b'{"li": [null, %d, "3"], "lf": [null, %d.25, "1e\\u0033"], "lb": [null, false], "ls": [null, "", "\\ud83d\\ude00", "t\\"%d"], "ln": [null], "lnn": [null, null], "id": %d}' % (i, i, i, i)
        elif k == 2:
            p = b'{"li": null, "lf": null, "lb": null, "ls": null, "ln": null, "lnn": null, "id": %d}' % i
        elif k == 3:
            p = b'{"id": %d}' % i
        else:
            p = ('{"ls": ["%s", "é\U0001F600"], "li": [%d], "lf": [%r], "id": %d}' % ("x" * (i % 50), -i, _f64(i), i)).encode()
        out.append(p)
    return out


def struct_payloads():
    first = b'{"st": {"a": 1, "s": "x", "f": 0.5, "b": true}, "id": 0}'
    out = [first]
    for i in range(1, 700):
        k = i % 6
        if k == 0:
            p = b'{"st": null, "id": %d}' % i
        elif k == 1:
            p = b'{"id": %d}' % i
        elif k == 2:
            p = b'{"st": {}, "id": %d}' % i
        elif k == 3:
            p = b'{"st": {"s": "\\ud83d\\ude00\\t%d", "\\u0061": %d, "zz": [1, {"q": "\\u00e9"}]}, "id": %d}' % (i, i, i)
        elif k == 4:
            p = b'{"st": {"b": false, "f": "2.\\u0035", "a": "7", "s": "%s", "s": "last"}, "id": %d}' % ("é".encode() * (i % 9), i)
        else:
            p = ('{"st": {"a": %d, "s": "%s", "f": %r, "b": true}, "id": %d}' % (i, "y" * (i % 70), _f64(i), i)).encode()
        out.append(p)
    return out


# malformed strings (the text between and including the quotes): bugs 1-4 and 6 of the decoder's history
BAD_STRINGS = {
    "high_then_bmp": b'"\\ud800\\u0041"',
    "lone_low": b'"\\udc00"',
    "high_then_bad_hex": b'"\\ud800\\uzzzz"',
    "lone_high_end": b'"ab\\ud800"',
    "bad_hex": b'"\\u12G4"',
    "short_u": b'"\\u12"',
    "bad_escape": b'"\\x41"',
    "raw_ff": b'"\xff"',
    "overlong": b'"\xc0\xaf"',
    "raw_surrogate": b'"\xed\xa0\x80"',
    "truncated_seq": b'"\xe2\x82"',
    "control": b'"a\x01b"',
}
CONTEXTS = {  # where the malformed string stands in a record
    "value": lambda i, b: b'{"id": %d, "s": %s, "l": ["a"], "st": {"k": "v"}}' % (i, b),
    "key": lambda i, b: b'{"id": %d, %s: 1, "s": "x"}' % (i, b),
    "unknown": lambda i, b: b'{"id": %d, "s": "x", "zz": %s}' % (i, b),
    "skipped_nested": lambda i, b: b'{"id": %d, "zz": {"q": [1, %s]}, "s": "x"}' % (i, b),
    "list": lambda i, b: b'{"id": %d, "l": ["a", %s]}' % (i, b),
    "struct": lambda i, b: b'{"id": %d, "st": {"k": %s}}' % (i, b),
    "struct_key": lambda i, b: b'{"id": %d, "st": {%s: "v"}}' % (i, b),
}
ERR_N = 300
ERR_AT = {"first": 0, "middle": ERR_N // 2, "last": ERR_N - 1}


def error_payloads(bad, ctx, where):
    good = [b'{"id": %d, "s": "ok\\u00e9", "l": ["a", "b"], "st": {"k": "v"}}' % i for i in range(ERR_N)]
    at = ERR_AT[where]
    good[at] = CONTEXTS[ctx](at, BAD_STRINGS[bad])
    return good


# ---- cases ------------------------------------------------------------------------------------------------------------
BIG = (1 << 20) + 3


def _payload_fn(name):
    kind, *rest = name.split(":")
    if kind == "flat":
        return lambda: [flat_record(i) for i in range(int(rest[0]))]
    if kind == "nullblank":
        def f():
            p = [flat_record(i) for i in range(1000)]
            for i in (0, 127, 128, 255, 256, 511, 999):
                p[i] = None
            for i in (126, 129, 640):
                p[i] = b""
            for i in (383, 384):
                p[i] = b" \n\t "
            return p
        return f
    if kind == "multi":
        return lambda: [b"\n".join(flat_record(i * 3 + k) for k in range(i % 3 + 1)) + (b" " if i % 2 else b"") for i in range(777)]
    if kind == "longrun":
        return lambda: [flat_record(i, {"pad": "x" * 1900} if 10 * 128 <= i < 12 * 128 else None) for i in range(4096)]
    if kind == "window":
        return lambda: window_payloads()[0]
    if kind == "avg":
        return lambda: avg_payloads(256 * 1024 + int(rest[0]), 1024)
    if kind == "fields":
        return lambda: field_records(int(rest[0]))
    if kind == "names":
        return lambda: names_records(rest[0] == "wide")
    if kind == "strings":
        return string_payloads
    if kind == "longstr":
        return lambda: long_string_payloads(rest[0] == "mixed")
    if kind == "lists":
        return list_payloads
    if kind == "structs":
        return struct_payloads
    if kind == "err":
        return lambda: error_payloads(*rest)
    raise ValueError(name)


def _case(cases, name, *, single=True, mix=None, slices=(), nested=False, expect="ok", err_where=None, qnum=0):
    """qnum: launches of json_quoted_numbers_kernel, one per Int64 / Float64 column of a pass that met a quoted number
    written with escapes."""
    cases.append(dict(id=f"c{len(cases)}", name=name, single=single, mix=mix, slices=list(slices), nested=nested,
                      expect=expect, err_where=err_where, qnum=qnum))


def all_cases():
    cases = []
    for n in (1, 127, 128, 129, (1 << 17) - 1, (1 << 17) + 1, BIG):
        _case(cases, f"flat:{n}", mix="staged", slices=(3,) if n in (129, (1 << 17) + 1) else ())
    _case(cases, "nullblank", single=False, mix="staged", slices=(1, 7))
    _case(cases, "multi", single=False, mix="staged", slices=(5,))
    _case(cases, "longrun", mix="mixed", slices=(3,))
    _case(cases, "window", mix="mixed")
    _case(cases, "avg:-100", mix="staged")  # averages 255.9 bytes
    _case(cases, "avg:100", mix="inplace")  # 256.1 bytes: no staging
    for k in (1, 16, 17, 63, 64):  # wide records average more than 256 bytes
        _case(cases, f"fields:{k}", mix="staged" if k == 1 else "inplace")
    _case(cases, "fields:65", expect="Unsupported")
    _case(cases, "names:narrow", mix="staged")
    _case(cases, "names:wide", mix="staged")
    _case(cases, "strings", mix="staged", slices=(1,), qnum=2)
    _case(cases, "longstr:inplace", mix="inplace")
    _case(cases, "longstr:mixed", mix="mixed")
    _case(cases, "lists", nested=True, mix="staged")
    _case(cases, "structs", nested=True, mix="staged", qnum=2)
    for bad in BAD_STRINGS:
        for ctx in CONTEXTS:
            for where in ERR_AT:
                _case(cases, f"err:{bad}:{ctx}:{where}", expect="Process", err_where=where)
    return cases


# ---- child: runs the library -----------------------------------------------------------------------------------------
def _child(spec_path):
    import ctypes as C

    from arkflow_b200 import _lib as L
    from arkflow_b200.arrow_ffi import DeviceBatch
    from arkflow_b200.processor import ArkError, JsonToArrowProcessor, MessageBatch, _check

    spec = json.load(open(spec_path))
    d = os.path.dirname(spec_path)
    lib = L.lib()
    _check(lib.ark_b200_init(0))
    lib.ark_kernel_timing_enable(1)
    report = {}
    for c in spec["cases"]:
        with pa.ipc.open_file(os.path.join(spec["inputs"], c["file"])) as r:
            rb = r.get_batch(0)
        for run in c["runs"]:
            x = rb if run["off"] is None else rb.slice(run["off"], rb.num_rows - run["off"])
            lib.ark_kernel_timing_reset()
            res = {}
            try:
                p = JsonToArrowProcessor({})
                if run["device"]:
                    out = p.process_device(DeviceBatch.from_arrow(x, keep_offsets=run["off"] is not None))
                    out = out.to_arrow()
                else:
                    out = p.process(MessageBatch.new_arrow(x)).batches[0].record_batch
                with pa.ipc.new_file(os.path.join(d, run["id"] + ".arrow"), out.schema) as w:
                    w.write_batch(out)
            except ArkError as e:
                res["error"], res["message"] = e.kind, e.message
            counts = {}
            for name in KERNELS:
                ms, n = C.c_double(), C.c_int64()
                lib.ark_kernel_timing_get(name.encode(), C.byref(ms), C.byref(n))
                counts[name] = n.value
            res["counts"] = counts
            report[run["id"]] = res
    json.dump(report, open(os.path.join(d, "report.json"), "w"))
    print("CHILD_OK")


def _run_child(tmp, inputs_dir, cases, env):
    spec = os.path.join(tmp, "spec.json")
    json.dump({"cases": cases, "inputs": inputs_dir}, open(spec, "w"))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), spec], capture_output=True, text=True, timeout=1200,
                       env=dict(os.environ, **env))
    assert r.returncode == 0 and "CHILD_OK" in r.stdout, r.stdout[-2000:] + r.stderr[-3000:]
    return json.load(open(os.path.join(tmp, "report.json")))


# ---- parent: inputs, the oracle and the comparison --------------------------------------------------------------------
_INPUTS, _ORACLE = {}, {}


def _input(name):
    if name not in _INPUTS:
        _INPUTS[name] = binary_batch(_payload_fn(name)())
    return _INPUTS[name]


def _sliced(name, off):
    rb = _input(name)
    return rb if off is None else rb.slice(off, rb.num_rows - off)


def _oracle(name, off):
    """The oracle's batch, or the OracleError kind."""
    import oracle.json_oracle as jo
    from oracle.sql_oracle import OracleError

    k = (name, off)
    if k not in _ORACLE:
        old, jo.NESTED = jo.NESTED, True
        try:
            _ORACLE[k] = jo.json_to_arrow(_sliced(name, off))
        except OracleError as e:
            _ORACLE[k] = e.kind
        finally:
            jo.NESTED = old
    return _ORACLE[k]


def _runs(c):
    """(device, offset) of each run of case c: host and device on the whole batch, then each slice both ways (the device
    slice keeps its offsets: data pointer not 16-byte aligned, offsets[0] != 0, validity starting inside a byte).  Nested
    outputs are read back through the host entry only (the Python DeviceBatch mirror holds flat columns)."""
    runs = [(False, None)] + ([] if c["nested"] else [(True, None)])
    for off in c["slices"]:
        runs += [(False, off), (True, off)]
    return runs


def _expand(cases):
    for c in cases:
        c["file"] = c["name"].replace(":", "_") + ".arrow"
        c["runs"] = [dict(id=f"{c['id']}_{k}", device=dev, off=off) for k, (dev, off) in enumerate(_runs(c))]
    return cases


@pytest.fixture(scope="module")
def inputs_dir(tmp_path_factory):
    return str(tmp_path_factory.mktemp("json_inputs"))


def _write_inputs(inputs_dir, cases):
    for c in cases:
        path = os.path.join(inputs_dir, c["file"])
        if not os.path.exists(path):
            rb = _input(c["name"])
            with pa.ipc.new_file(path, rb.schema) as w:
                w.write_batch(rb)


def _f64_bits(a):
    bits = np.frombuffer(a.buffers()[1], np.uint64)[a.offset:a.offset + len(a)] if len(a) else np.zeros(0, np.uint64)
    return a.is_valid().to_numpy(zero_copy_only=False), bits


def same_array(g, w, what):
    assert g.type == w.type and len(g) == len(w), (what, g.type, w.type, len(g), len(w))
    if pa.types.is_floating(w.type):
        gv, gb = _f64_bits(g)
        wv, wb = _f64_bits(w)
        assert np.array_equal(gv, wv), (what, "validity")
        bad = np.flatnonzero(wv & (gb != wb))
        assert len(bad) == 0, (what, len(bad), [(int(i), hex(gb[i]), hex(wb[i])) for i in bad[:5]])
    elif pa.types.is_struct(w.type):
        assert g.is_valid().equals(w.is_valid()), (what, "struct validity")
        for k in range(w.type.num_fields):
            wc = w.field(k)
            # the oracle's builder leaves defaults under a NULL struct row; the decoder's children are NULL there
            wc = pc.if_else(w.is_valid(), wc, pa.nulls(len(w), wc.type))
            same_array(g.field(k), wc, what + (w.type.field(k).name,))
    elif pa.types.is_list(w.type):
        assert g.is_valid().equals(w.is_valid()), (what, "list validity")
        assert pc.list_value_length(g).fill_null(0).equals(pc.list_value_length(w).fill_null(0)), (what, "list lengths")
        same_array(g.flatten(), w.flatten(), what + ("item",))
    else:
        assert g.equals(w), (what, _first_diff(g, w))


def _first_diff(g, w):
    for i in range(min(len(g), len(w))):
        if g[i] != w[i]:
            return i, g[i], w[i]
    return None


def compare(got, want, what):
    try:
        got.validate(full=True)
    except pa.ArrowInvalid as e:
        raise AssertionError((what, "invalid result", str(e))) from None
    assert got.schema.names == want.schema.names, (what, got.schema, want.schema)
    assert [f.type for f in got.schema] == [f.type for f in want.schema], (what, got.schema, want.schema)
    assert got.num_rows == want.num_rows, (what, got.num_rows, want.num_rows)
    for name, g, w in zip(want.schema.names, got.columns, want.columns):
        same_array(g, w, (what, name))
    if any(pa.types.is_struct(t) or pa.types.is_list(t) for t in want.schema.types):
        assert got.to_pylist() == want.to_pylist(), what


def _utf8_arrays(a):
    """Utf8 arrays of `a` (nested children included) that the decoder fills with json_strings_kernel: non-empty ones."""
    t = a.type
    if pa.types.is_string(t):
        return int(len(a) > 0)
    if pa.types.is_list(t):
        return _utf8_arrays(a.flatten()) if len(a) else 0
    if pa.types.is_struct(t):
        return sum(_utf8_arrays(a.field(k)) for k in range(t.num_fields)) if len(a) else 0
    return 0


def expected_counts(env, c, want):
    """Launches of the route: the optimistic pass (1) falls back to count + parse when a payload is NULL, blank or holds
    several records; ARK_JSON_TWO_PASS goes there directly.  Each Struct column adds its span pass.  Quoted numbers
    written with escapes are parsed by json_quoted_numbers_kernel after the pass that met them."""
    two_pass = "ARK_JSON_TWO_PASS" in env
    if want.num_columns == 0:
        return dict.fromkeys(KERNELS, 0)
    rows = want.num_rows
    structs = sum(1 for t in want.schema.types if pa.types.is_struct(t) and t.num_fields and rows)
    lists = [a for a in want.columns if pa.types.is_list(a.type)]
    parse = (1 if two_pass or c["single"] else 2) + structs
    return {"json_parse_kernel": parse, "json_count_kernel": int(two_pass or not c["single"]),
            "json_strings_kernel": sum(_utf8_arrays(a) for a in want.columns),
            "json_list_count_kernel": sum(1 for a in lists if rows), "json_list_fill_kernel": sum(1 for a in lists if len(a.flatten())),
            "json_quoted_numbers_kernel": c["qnum"]}


def _check_run(path, tmp, c, run, res):
    env = PATHS[path]
    what = (path, c["name"], "device" if run["device"] else "host", run["off"])
    counts = res["counts"]
    want = _oracle(c["name"], run["off"]) if c["expect"] != "Unsupported" else "Unsupported"
    if c["expect"] != "ok":
        assert want == c["expect"], (what, "oracle", want)
        assert res.get("error") == c["expect"], (what, res)
        assert counts["json_strings_kernel"] == 0, (what, counts)
        if c["err_where"] == "first":  # schema inference rejects the first record: nothing launches
            assert counts["json_parse_kernel"] == 0 and counts["json_count_kernel"] == 0, (what, counts)
        elif c["err_where"]:  # the count pass validates every string of every record and reports it
            assert counts["json_count_kernel"] == 1, (what, counts)
            assert counts["json_parse_kernel"] == (0 if "ARK_JSON_TWO_PASS" in env else 1), (what, counts)
        return
    assert "error" not in res, (what, res)
    assert not isinstance(want, str), (what, "oracle", want)
    with pa.ipc.open_file(os.path.join(str(tmp), run["id"] + ".arrow")) as r:
        got = r.get_batch(0) if r.num_record_batches else r.schema.empty_table().to_batches()[0]
    compare(got, want, what)
    assert counts == expected_counts(env, c, want), (what, counts, expected_counts(env, c, want))
    if c["mix"] and run["off"] is None:  # the staged / in-place mix the case claims, for its whole batch
        mix = "inplace" if "ARK_JSON_NO_STAGE" in env else staging_mix(_input(c["name"]), None, False)
        assert mix == ("inplace" if "ARK_JSON_NO_STAGE" in env else c["mix"]), (what, mix)


def _check_path(path, tmp, inputs_dir, cases):
    _expand(cases)
    _write_inputs(inputs_dir, cases)
    report = _run_child(str(tmp), inputs_dir, cases, PATHS[path])
    for c in cases:
        for run in c["runs"]:
            _check_run(path, tmp, c, run, report[run["id"]])


# ---- CPU: the oracle's string policy and the cases' staging mix ----------------------------------------------------------
@pytest.mark.parametrize("payload", [b'{"s": "\\ud800"}', b'{"s": "\\udc00"}', b'{"s": "\\ud800\\u0041"}', b'{"\\udfff": 1}',
                                     b'{"a": 1, "zz": "\\ud83d"}', b'{"a": 1, "zz": {"q": ["\\udc00"]}}', b'{"a": ["\\ud800x"]}',
                                     b'{"a": {"\\ud800": 1}}'])
def test_oracle_rejects_unpaired_surrogates(payload):
    import oracle.json_oracle as jo
    from oracle.sql_oracle import OracleError

    for nested in (False, True):
        old, jo.NESTED = jo.NESTED, nested
        try:
            with pytest.raises(OracleError) as e:
                jo.json_to_arrow(binary_batch([b'{"a": 1}', payload]))
            assert e.value.kind == "Process"
            with pytest.raises(OracleError) as e:
                jo.json_to_arrow(binary_batch([payload]))
            assert e.value.kind == "Process"
        finally:
            jo.NESTED = old


def test_oracle_keeps_paired_surrogates_and_decodes_quoted_numbers():
    import oracle.json_oracle as jo

    rb = jo.json_to_arrow(binary_batch([b'{"\\ud83d\\ude00": "\\uD83D\\uDE00x", "i": 1}', b'{"i": "1\\u0032"}']))
    assert rb.schema.names == ["\U0001F600", "i"]
    assert rb.column(0).to_pylist() == ["\U0001F600x", None] and rb.column(1).to_pylist() == [1, 12]


def test_cases_have_the_staging_mix_they_claim():
    """The staging model, applied to every case that claims a mix: the whole batch on the host entry and device."""
    for c in all_cases():
        if c["mix"]:
            rb = _input(c["name"])
            for keep in (False, True):
                assert staging_mix(rb, None, keep) == c["mix"], (c["name"], keep)
    payloads, s = window_payloads()
    offs = np.concatenate([[0], np.cumsum([len(p) for p in payloads])])
    st = cta_staged(offs, s, False)
    assert st[5] and not st[9] and st.sum() == len(st) - 1
    assert offs[6 * JS_THREADS] - offs[5 * JS_THREADS] == s and offs[-1] % 16 == 0


# ---- GPU ----------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("path", list(PATHS))
def test_decoder_matches_oracle(gpu, tmp_path, inputs_dir, path):
    _check_path(path, tmp_path, inputs_dir, all_cases())


def _csv_read_all(path):
    from arkflow_b200.input import FileInput
    from arkflow_b200.processor import ArkError

    inp = FileInput({"input_type": {"type": "csv", "path": path}, "batch_size": 1000})
    inp.connect()
    got = []
    while True:
        try:
            got.append(inp.read()[0].record_batch)
        except ArkError as e:
            if e.kind == "EOF":
                return pa.Table.from_batches(got)
            raise


@pytest.mark.gpu
def test_csv_rejects_invalid_utf8(gpu, tmp_path):
    """A Utf8 field or header name that is not UTF-8 is a Process error naming the line, as pyarrow.csv rejects such a
    field of a string column (left to itself pyarrow infers Binary, a type arrow-csv's inference never yields); valid
    multi-byte text round-trips.  arrow-csv reads the header as UTF-8 strings, so a header that is not fails too."""
    import pyarrow.csv as pacsv

    from arkflow_b200.processor import ArkError

    as_strings = pacsv.ConvertOptions(column_types={"s": pa.string(), "t": pa.string()})
    rows = [b"%d,name\xc3\xa9%d,\xf0\x9f\x98\x80" % (i, i) for i in range(2500)]
    ok = str(tmp_path / "ok.csv")
    open(ok, "wb").write(b"id,s,t\n" + b"\n".join(rows) + b"\n")
    got = _csv_read_all(ok)
    want = pacsv.read_csv(ok, convert_options=as_strings)
    assert got.column("s").to_pylist() == want.column("s").to_pylist() and got.column("t").to_pylist() == want.column("t").to_pylist()
    for at in (0, 1250, 2499):
        for bad in (b"\xff", b"\xc0\xaf", b"\xed\xa0\x80", b"ab\xe2\x82"):
            r = list(rows)
            r[at] = b"%d,%s,x" % (at, bad)
            p = str(tmp_path / "bad.csv")
            open(p, "wb").write(b"id,s,t\n" + b"\n".join(r) + b"\n")
            with pytest.raises(pa.ArrowInvalid):
                pacsv.read_csv(p, convert_options=as_strings)
            with pytest.raises(ArkError) as e:
                _csv_read_all(p)
            assert e.value.kind == "Process" and "line %d" % (at + 2) in e.value.message, (at, bad, e.value.message)
    p = str(tmp_path / "badhead.csv")
    open(p, "wb").write(b"id,s\xff,t\n" + b"\n".join(rows) + b"\n")
    with pytest.raises(ArkError) as e:
        _csv_read_all(p)
    assert e.value.kind == "Process"


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    _child(sys.argv[1])
