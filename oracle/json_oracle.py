"""CPU oracle for `json_to_arrow` — TEST INFRASTRUCTURE (see oracle/__init__.py).

Restates JsonToArrowProcessor::process (crates/arkflow-plugin/src/processor/json.rs:48-61) and
component::json::try_to_arrow (crates/arkflow-plugin/src/component/json.rs:22-58) on top of the
published behaviour of arrow-json 55.2.0 (third-party; pinned in Cargo.lock, not vendored):
  * to_binary(value_field) keeps the non-null payloads (core/lib.rs:355-371), joined with a newline;
  * infer_json_schema(.., Some(1)): types from the FIRST record only, first-seen field order, every
    field nullable; integer fitting i64 -> Int64, other numbers -> Float64, bool -> Boolean,
    string -> Utf8, null -> Null (array/object -> List/Struct: outside this library's subset);
  * decoding is non-strict: unknown keys ignored, missing keys -> NULL;
  * numeric columns accept JSON numbers and quoted numbers; Int64 parses as integer, else as f64 and
    truncates (error when out of range); Utf8 accepts only strings, Boolean only true/false;
  * every top-level value must be an object.
PARITY STATUS: unpinned by the reference beyond row counts / is_err (json.rs:170-266); the type
inference table is from the arrow-json documentation.
"""
from __future__ import annotations

import json
import re
from typing import Optional

import pyarrow as pa

from .sql_oracle import OracleError

# Nested values (List / Struct columns).  The library does not decode them yet (DESIGN.md §10 item 0), so the default
# mirrors it and reports Unsupported; NESTED = True is the restatement of arrow-json's behaviour the next round's
# kernels will be checked against (tests/test_oracle_golden.py pins it to processor/json.rs:170-207).
NESTED = False

_NUM_RE = re.compile(rb"^[+-]?(\d+)(\.\d+)?([eE][+-]?\d+)?$|^[+-]?\.\d+([eE][+-]?\d+)?$")
_INT_RE = re.compile(rb"^[+-]?\d+$")


class _Num:
    __slots__ = ("text",)

    def __init__(self, text: str):
        self.text = text


def _bad_constant(s):
    raise ValueError("invalid JSON constant " + s)


def _decoder():
    return json.JSONDecoder(parse_int=_Num, parse_float=_Num, parse_constant=_bad_constant,
                            object_pairs_hook=lambda pairs: ("obj", pairs))


def _iter_values(data: str):
    dec = _decoder()
    pos, n = 0, len(data)
    while True:
        while pos < n and data[pos] in " \t\r\n":
            pos += 1
        if pos >= n:
            return
        v, pos = dec.raw_decode(data, pos)
        yield v


def _infer_type(v) -> pa.DataType:
    if v is None:
        return pa.null()
    if isinstance(v, bool):
        return pa.bool_()
    if isinstance(v, _Num):
        if _INT_RE.match(v.text.encode()) and -(2 ** 63) <= int(v.text) <= 2 ** 63 - 1:
            return pa.int64()
        return pa.float64()
    if isinstance(v, str):
        return pa.utf8()
    if NESTED and isinstance(v, list):
        # arrow-json infer_json_schema: the element type is the coercion of the elements' types
        # (Int64 + Float64 → Float64, anything + Null → that thing, an empty array → List<Null>)
        t = pa.null()
        for x in v:
            xt = _infer_type(x)
            if t == pa.null():
                t = xt
            elif xt == pa.null() or xt == t:
                pass
            elif {t, xt} == {pa.int64(), pa.float64()}:
                t = pa.float64()
            else:
                raise OracleError("Unsupported", "JSON array of mixed types")
        return pa.list_(pa.field("item", t, True))
    if NESTED and isinstance(v, tuple) and v[0] == "obj":
        fields, seen = [], set()
        for k, x in v[1]:
            if k not in seen:
                seen.add(k)
                fields.append(pa.field(k, _infer_type(x), True))
        return pa.struct(fields)
    raise OracleError("Unsupported", "nested JSON value (List/Struct column)")


def _to_i64(text: bytes) -> int:
    if _INT_RE.match(text):
        v = int(text)
        if -(2 ** 63) <= v <= 2 ** 63 - 1:
            return v
    if not _NUM_RE.match(text):
        raise OracleError("Process", "Arrow JSON Reader Error: Json error: failed to parse number")
    f = float(text)
    if not (-9223372036854777856.0 < f < 9223372036854775808.0):
        raise OracleError("Process", "Arrow JSON Reader Error: Json error: failed to parse number")
    return int(f)


def _to_f64(text: bytes) -> float:
    if not _NUM_RE.match(text):
        raise OracleError("Process", "Arrow JSON Reader Error: Json error: failed to parse number")
    return float(text)


def _check_no_surrogates(v):
    stack = [v]
    while stack:
        x = stack.pop()
        if isinstance(x, str):
            try:
                x.encode("utf-8")
            except UnicodeEncodeError:
                raise OracleError("Process", "Arrow JSON Reader Error: Json error: invalid string: unpaired surrogate escape")
        elif isinstance(x, list):
            stack.extend(x)
        elif isinstance(x, tuple) and x[0] == "obj":
            for k, e in x[1]:
                stack.append(k)
                stack.append(e)


def json_to_arrow(rb: pa.RecordBatch, value_field: str = "__value__", fields_to_include: Optional[set] = None) -> pa.RecordBatch:
    if value_field not in rb.schema.names:
        raise OracleError("Process", "not found column")
    col = rb.column(value_field)
    if col.type != pa.binary():
        raise OracleError("Process", "not support data type")
    payloads = [v.as_py() for v in col if v.is_valid]
    try:
        data = b"\n".join(payloads).decode("utf-8")
    except UnicodeDecodeError:
        raise OracleError("Process", "Schema inference error: Json error: invalid UTF-8")
    try:
        values = list(_iter_values(data))
    except (ValueError, json.JSONDecodeError) as e:
        raise OracleError("Process", f"Arrow JSON Reader Error: Json error: {e}")
    # Python's json decodes a lone or mispaired surrogate escape ("\ud800", "\udc00", "\ud800A") to a surrogate
    # code point, which no UTF-8 string can hold; an arrow-rs StringArray is always valid UTF-8, so such a string is
    # a Process error wherever it stands: a key, a value, an unknown field or inside a nested value.
    for v in values:
        _check_no_surrogates(v)
    if not values:
        return pa.RecordBatch.from_arrays([], schema=pa.schema([]))
    first = values[0]
    if not (isinstance(first, tuple) and first[0] == "obj"):
        raise OracleError("Process", "Schema inference error: Json error: Expected JSON record to be an object")
    fields, seen = [], set()
    for k, v in first[1]:
        if k in seen:
            continue
        seen.add(k)
        if fields_to_include is not None and k not in fields_to_include:
            continue
        fields.append((k, _infer_type(v)))
    def convert(x, t):
        if x is None:
            return None
        if t == pa.int64() or t == pa.float64():
            if isinstance(x, _Num):
                text = x.text.encode()
            elif isinstance(x, str):
                text = x.encode()
            else:
                raise OracleError("Process", "Arrow JSON Reader Error: Json error: expected a number")
            return _to_i64(text) if t == pa.int64() else _to_f64(text)
        if t == pa.bool_():
            if not isinstance(x, bool):
                raise OracleError("Process", "Arrow JSON Reader Error: Json error: expected a boolean")
            return x
        if t == pa.utf8():
            if not isinstance(x, str):
                raise OracleError("Process", "Arrow JSON Reader Error: Json error: expected a string")
            return x
        if pa.types.is_list(t):
            if not isinstance(x, list):
                raise OracleError("Process", "Arrow JSON Reader Error: Json error: expected an array")
            return [convert(e, t.value_type) for e in x]
        if pa.types.is_struct(t):
            if not (isinstance(x, tuple) and x[0] == "obj"):
                raise OracleError("Process", "Arrow JSON Reader Error: Json error: expected an object")
            rec = {}
            for k, e in x[1]:
                rec[k] = e
            return {f.name: convert(rec.get(f.name), f.type) for f in t}
        raise OracleError("Process", "Arrow JSON Reader Error: Json error: expected null")

    cols = {k: [] for k, _ in fields}
    for v in values:
        if not (isinstance(v, tuple) and v[0] == "obj"):
            raise OracleError("Process", "Arrow JSON Reader Error: Json error: expected { got a non-object value")
        rec = {}
        for k, x in v[1]:
            rec[k] = x  # duplicate keys: the last one wins
        for k, t in fields:
            x = rec.get(k)
            if x is None:
                cols[k].append(None)
            elif pa.types.is_list(t) or pa.types.is_struct(t):
                cols[k].append(convert(x, t))
            elif t == pa.int64() or t == pa.float64():
                if isinstance(x, _Num):
                    text = x.text.encode()
                elif isinstance(x, str):
                    text = x.encode()
                else:
                    raise OracleError("Process", "Arrow JSON Reader Error: Json error: expected a number")
                cols[k].append(_to_i64(text) if t == pa.int64() else _to_f64(text))
            elif t == pa.bool_():
                if not isinstance(x, bool):
                    raise OracleError("Process", "Arrow JSON Reader Error: Json error: expected a boolean")
                cols[k].append(x)
            elif t == pa.utf8():
                if not isinstance(x, str):
                    raise OracleError("Process", "Arrow JSON Reader Error: Json error: expected a string")
                cols[k].append(x)
            else:  # Null column: only nulls
                raise OracleError("Process", "Arrow JSON Reader Error: Json error: expected null")
    arrays = [pa.array(cols[k], type=t) for k, t in fields]
    return pa.RecordBatch.from_arrays(arrays, schema=pa.schema([pa.field(k, t, True) for k, t in fields]))


# ------------------------------------------------------------------------------------------------
# arrow_to_json  (crates/arkflow-plugin/src/processor/json.rs:78-113 + core/lib.rs:280-302)
# ------------------------------------------------------------------------------------------------
def _lexical_f64(x: float) -> str:
    """lexical-core's default float text (arrow-json 55.2 writes finite f64 through lexical_core::write):
    shortest round-trip digits (= Python repr digits); positional with at least ".0" while the
    scientific exponent is in [-5, 9], d.ddde±x otherwise."""
    import math

    if math.isnan(x) or math.isinf(x):
        return "null"
    if x == 0:
        return "-0.0" if math.copysign(1.0, x) < 0 else "0.0"
    r = repr(abs(x))
    mant, _, ex = r.partition("e")
    ip, _, fp = mant.partition(".")
    digits = (ip + fp).lstrip("0")
    e10 = (int(ex) if ex else 0) - len(fp)
    stripped = digits.rstrip("0")
    e10 += len(digits) - len(stripped)
    ds = stripped
    sci = e10 + len(ds) - 1
    if -5 <= sci <= 9:
        if e10 >= 0:
            s = ds + "0" * e10 + ".0"
        elif -e10 < len(ds):
            s = ds[: len(ds) + e10] + "." + ds[len(ds) + e10:]
        else:
            s = "0." + "0" * (-e10 - len(ds)) + ds
    else:
        s = ds[0] + "." + (ds[1:] if len(ds) > 1 else "0") + "e" + str(sci)
    return ("-" if x < 0 else "") + s


def arrow_to_json_lines(rb: pa.RecordBatch, fields_to_include: Optional[set] = None) -> list[bytes]:
    """LineDelimitedWriter with default options: schema order, NULL fields omitted, no whitespace."""
    names = [n for n in rb.schema.names if fields_to_include is None or n in fields_to_include]
    cols = [(n, rb.column(rb.schema.names.index(n))) for n in names]
    lines = []
    for i in range(rb.num_rows):
        parts = []
        for n, c in cols:
            v = c[i]
            if not v.is_valid or c.type == pa.null():
                continue
            key = json.dumps(n, ensure_ascii=False)
            if c.type == pa.int64():
                val = str(v.as_py())
            elif c.type == pa.float64():
                val = _lexical_f64(v.as_py())
            elif c.type == pa.bool_():
                val = "true" if v.as_py() else "false"
            elif c.type == pa.utf8():
                val = json.dumps(v.as_py(), ensure_ascii=False)
            elif c.type == pa.binary():
                val = '"' + v.as_py().hex() + '"'
            else:
                raise OracleError("Unsupported", f"arrow_to_json of {c.type}")
            parts.append(f"{key}:{val}")
        lines.append(("{" + ",".join(parts) + "}").encode("utf-8"))
    return lines


def arrow_to_json(rb: pa.RecordBatch, fields_to_include: Optional[set] = None) -> pa.RecordBatch:
    """ArrowToJsonProcessor::process: the original columns + a non-null Binary `__value__` column."""
    lines = arrow_to_json_lines(rb, fields_to_include)
    if len(lines) != rb.num_rows:
        raise OracleError("Process", "Creating an Arrow record batch failed")
    fields = list(rb.schema) + [pa.field("__value__", pa.binary(), nullable=False)]
    return pa.RecordBatch.from_arrays(list(rb.columns) + [pa.array(lines, pa.binary())], schema=pa.schema(fields))
