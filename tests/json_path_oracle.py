"""CPU oracle for the JSON path functions of the `sql` processor — TEST INFRASTRUCTURE, not product code.

Restates datafusion-functions-json 0.47 over jiter 0.9 (third-party, registered by the reference's sql.rs:18-24; not
vendored, so what follows is its published behaviour, not a run of it):
    * jiter_json_find: from the document's first value, a string path element selects the FIRST key of an object that
      equals it once escapes are decoded; an integer selects an array element.  A key applied to an array, an index
      applied to an object, a missing key or an index past the end finds nothing.
    * The walk is lazy: it parses exactly what it passes over and the value it lands on.  Bytes after that are never
      read, so trailing garbage after a found value does not matter; anything malformed before it gives NULL.
    * json_get_int: an integer that fits i64; json_get_float: any number (an integer converted exactly, so "-0" is +0.0);
      json_get_bool: true / false; json_get_str: a string, unescaped; json_as_text: a string unescaped, NULL for null,
      the raw source text otherwise; json_get_json: the raw source text of any value; json_length: elements of an array
      or keys of an object; json_contains: whether the path resolves (jiter only peeks at the value found).
Python's json module is used only to convert number text.

Unverified assumptions (no crate source or binary is available to check them):
    * A bare Binary first argument: the crate's coercion of it is not known, so it is Unsupported here.
    * json_contains on a NULL document: the crate maps every row through jiter_json_find(None, ..).is_some(), which is
      false, not NULL; followed here.
    * The reference docs write array access as '1' (json_get_str('["apple", ...]', '1') = banana).  In the crate a string
      path element is an object key, so '1' on an array finds nothing.  The docs and the crate contradict each other;
      this oracle follows the crate: only an integer literal indexes an array.
    * Numbers: 1e400 (out of range) gives NULL (jiter's NumberOutOfRange); "-0" is the integer 0 (json_get_float +0.0,
      json_get_int 0) while "-0.0" is the float -0.0; integers beyond i64 convert to the nearest double.
    * Trailing garbage after a found value is ignored (the lazy walk), and "12x" yields the number 12.
    * Nesting deeper than 256 containers is malformed; strings the walk passes over must have well-formed escapes.
    * json_length is UInt64 in the crate; it is Int64 here (the column type the plan reads).
"""
from __future__ import annotations

import json
import re
from typing import Optional

import pyarrow as pa

import oracle.sql_oracle as S
from oracle.sql_oracle import E, OracleError

JSON_FUNCS = {"json_get_str": "Utf8", "json_get_int": "Int64", "json_get_float": "Float64", "json_get_bool": "Boolean",
              "json_get_json": "Utf8", "json_as_text": "Utf8", "json_contains": "Boolean", "json_length": "Int64"}
MAX_PATH = 8
MAX_DEPTH = 256
_PA = {"Utf8": pa.string(), "Int64": pa.int64(), "Float64": pa.float64(), "Boolean": pa.bool_()}
_NUM_RE = re.compile(rb"-?(?:0|[1-9][0-9]*)(?:\.[0-9]+)?(?:[eE][+-]?[0-9]+)?")
_ESC = {ord('"'): '"', ord("\\"): "\\", ord("/"): "/", ord("b"): "\b", ord("f"): "\f", ord("n"): "\n", ord("r"): "\r",
        ord("t"): "\t"}


class _Bad(Exception):
    """The document is malformed where the walk reads it."""


def _ws(b: bytes, i: int) -> int:
    while i < len(b) and b[i] in b" \t\n\r":
        i += 1
    return i


def _at(b: bytes, i: int) -> int:
    if i >= len(b):
        raise _Bad()
    return b[i]


def _hex4(b: bytes, i: int) -> int:
    h = b[i:i + 4]
    if len(h) < 4 or not all(c in b"0123456789abcdefABCDEF" for c in h):
        raise _Bad()
    return int(h, 16)


def _string(b: bytes, i: int) -> tuple[int, str]:
    """b[i] is the opening quote → (position after the closing quote, decoded text)."""
    i += 1
    out = []
    while True:
        c = _at(b, i)
        if c == 0x22:
            return i + 1, "".join(out)
        if c < 0x20:
            raise _Bad()
        if c != 0x5C:
            j = i
            while j < len(b) and b[j] not in (0x22, 0x5C) and b[j] >= 0x20:
                j += 1
            out.append(b[i:j].decode("utf-8"))
            i = j
            continue
        e = _at(b, i + 1)
        if e in _ESC:
            out.append(_ESC[e])
            i += 2
            continue
        if e != ord("u"):
            raise _Bad()
        cp = _hex4(b, i + 2)
        i += 6
        if 0xDC00 <= cp <= 0xDFFF:
            raise _Bad()
        if 0xD800 <= cp <= 0xDBFF:
            if b[i:i + 2] != b"\\u":
                raise _Bad()
            lo = _hex4(b, i + 2)
            if not 0xDC00 <= lo <= 0xDFFF:
                raise _Bad()
            cp = 0x10000 + ((cp - 0xD800) << 10) + (lo - 0xDC00)
            i += 6
        out.append(chr(cp))


def _number(b: bytes, i: int) -> tuple[int, bytes]:
    m = _NUM_RE.match(b, i)
    if not m:
        raise _Bad()
    end = m.end()
    if end < len(b) and 0x30 <= b[end] <= 0x39:  # a leading zero followed by a digit
        raise _Bad()
    return end, m.group(0)


def _skip(b: bytes, i: int, depth: int = 0) -> tuple[int, int]:
    """A whole value from b[i] (no leading whitespace) → (its end, its element count when it is a container)."""
    c = _at(b, i)
    if c in (0x7B, 0x5B):
        if depth >= MAX_DEPTH:
            raise _Bad()
        close = 0x7D if c == 0x7B else 0x5D
        i = _ws(b, i + 1)
        if _at(b, i) == close:
            return i + 1, 0
        n = 0
        while True:
            if c == 0x7B:
                if _at(b, i) != 0x22:
                    raise _Bad()
                i, _ = _string(b, i)
                i = _ws(b, i)
                if _at(b, i) != 0x3A:
                    raise _Bad()
                i = _ws(b, i + 1)
            i, _ = _skip(b, i, depth + 1)
            n += 1
            i = _ws(b, i)
            d = _at(b, i)
            if d == close:
                return i + 1, n
            if d != 0x2C:
                raise _Bad()
            i = _ws(b, i + 1)
            if c == 0x5B and _at(b, i) == 0x5D:
                raise _Bad()  # trailing comma
    if c == 0x22:
        return _string(b, i)[0], 0
    for lit in (b"true", b"false", b"null"):
        if c == lit[0]:
            if b[i:i + len(lit)] != lit:
                raise _Bad()
            return i + len(lit), 0
    return _number(b, i)[0], 0


def _find(b: bytes, path: list) -> Optional[int]:
    """jiter_json_find: the position of the value the path leads to, None when it leads nowhere."""
    i = _ws(b, 0)
    _at(b, i)
    for el in path:
        c = b[i]
        if isinstance(el, str) and c == 0x7B:
            i = _ws(b, i + 1)
            if _at(b, i) == 0x7D:
                return None
            while True:
                if _at(b, i) != 0x22:
                    raise _Bad()
                i, key = _string(b, i)
                i = _ws(b, i)
                if _at(b, i) != 0x3A:
                    raise _Bad()
                i = _ws(b, i + 1)
                _at(b, i)
                if key == el:
                    break
                i, _ = _skip(b, i, 1)
                i = _ws(b, i)
                d = _at(b, i)
                if d == 0x7D:
                    return None
                if d != 0x2C:
                    raise _Bad()
                i = _ws(b, i + 1)
        elif isinstance(el, int) and not isinstance(el, bool) and c == 0x5B:
            i = _ws(b, i + 1)
            if _at(b, i) == 0x5D:
                return None
            for _ in range(el):
                i, _ = _skip(b, i, 1)
                i = _ws(b, i)
                d = _at(b, i)
                if d == 0x5D:
                    return None
                if d != 0x2C:
                    raise _Bad()
                i = _ws(b, i + 1)
                if _at(b, i) == 0x5D:
                    raise _Bad()  # trailing comma
        else:
            return None
    return i


def json_call(fn: str, doc: Optional[str], path: list):
    """One row of one json_* call.  None is SQL NULL."""
    if doc is None:
        return False if fn == "json_contains" else None
    b = doc.encode("utf-8")
    try:
        i = _find(b, path)
        if fn == "json_contains":
            return i is not None
        if i is None:
            return None
        c = b[i]
        if fn == "json_get_str" or (fn == "json_as_text" and c == 0x22):
            return _string(b, i)[1] if c == 0x22 else None
        if fn == "json_get_bool":
            for lit, v in ((b"true", True), (b"false", False)):
                if b[i:i + len(lit)] == lit:
                    return v
            return None
        if fn in ("json_get_int", "json_get_float"):
            if c in b'"{[tfn':
                return None
            _, text = _number(b, i)
            v = json.loads(text)
            if fn == "json_get_int":
                return v if isinstance(v, int) and -2**63 <= v < 2**63 else None
            v = float(v)
            return None if v in (float("inf"), float("-inf")) else v
        end, n = _skip(b, i, 0)
        if fn == "json_length":
            return n if c in b"{[" else None
        if fn == "json_as_text" and c == ord("n"):
            return None
        return b[i:end].decode("utf-8")
    except _Bad:
        return False if fn == "json_contains" else None


# ------------------------------------------------------------------------------------------------
# binding: the json_* calls of a query → hidden columns, then the sql oracle
# ------------------------------------------------------------------------------------------------
def _unsupported(msg: str):
    raise OracleError("Unsupported", "SQL outside the GPU subset: " + msg)


def _bind_call(e: E, ctx_types: dict) -> tuple[str, bool, list]:
    """→ (document column, read through CAST(Binary AS STRING), path)."""
    what = e.name + "()"
    if e.star or not e.args:
        _unsupported(what + " without a JSON document argument")
    if len(e.args) > 1 + MAX_PATH:
        _unsupported(f"{what} with more than {MAX_PATH} path elements")
    doc = e.args[0]
    col = doc if doc.kind == "col" else doc.args[0] if doc.kind == "cast" and doc.to == "Utf8" and doc.args[0].kind == "col" else None
    t = ctx_types.get(col.name) if col is not None else None
    if col is not None and t is None:
        raise OracleError("Process", f"Execution query error: Schema error: No field named {col.name}.")
    if not (t == "Utf8" or (t == "Binary" and col is not doc)):
        _unsupported(what + ": the JSON document must be a Utf8 column or CAST(<Binary column> AS STRING)")
    path = []
    for a in e.args[1:]:
        if a.kind == "lit" and a.vtype == "Utf8":
            path.append(a.value)
        elif a.kind == "lit" and a.vtype == "Int64" and a.value >= 0:
            path.append(int(a.value))
        else:
            _unsupported(what + ": a path element must be a string or non-negative integer literal")
    return col.name, t == "Binary", path


def _arrow_kind(t: pa.DataType) -> str:
    if pa.types.is_string(t):
        return "Utf8"
    if pa.types.is_binary(t):
        return "Binary"
    return str(t)


def json_column(rb: pa.RecordBatch, fn: str, doc_col: str, path: list, cast: bool = False) -> pa.Array:
    docs = rb.column(rb.schema.get_field_index(doc_col)).to_pylist()
    if cast:
        try:
            docs = [None if d is None else d.decode("utf-8") for d in docs]
        except UnicodeDecodeError:
            raise OracleError("Process", "Collection query results error: Arrow error: Cast error: Cannot cast binary to string: invalid utf-8 sequence")
    return pa.array([json_call(fn, d, path) for d in docs], _PA[JSON_FUNCS[fn]])


def sql_process_json(rb: pa.RecordBatch, query: str, table_name: str = "flow") -> Optional[pa.RecordBatch]:
    """oracle.sql_oracle.sql_process with the json_* calls evaluated first, each distinct call once, as hidden columns."""
    q = S.parse(query)
    vis = q.alias or q.table
    types = {f.name: _arrow_kind(f.type) for f in rb.schema}
    calls: dict[str, tuple] = {}

    def rewrite(e: Optional[E]) -> Optional[E]:
        if e is None:
            return None
        if e.kind == "func" and e.name in JSON_FUNCS and not q.joins:
            doc, cast, path = _bind_call(e, types)
            name = S.display(e, vis)
            if name not in calls:
                calls[name] = (f"__json{len(calls)}", e.name, doc, cast, path)
            return E("col", name=calls[name][0])
        e.args = [rewrite(a) for a in e.args]
        return e

    for it in q.select:
        it.expr = rewrite(it.expr)
    q.where = rewrite(q.where)
    q.group_by = [rewrite(g) for g in q.group_by]
    if not calls or rb.num_rows == 0:
        return S.sql_process(rb, query, table_name)
    cols, names = list(rb.columns), list(rb.schema.names)
    for name, (hidden, fn, doc, cast, path) in calls.items():
        cols.append(json_column(rb, fn, doc, path, cast))
        names.append(hidden)
    wide = pa.record_batch(cols, names=names)
    saved = S.parse
    S.parse = lambda _text: q
    try:
        out = S.sql_process(wide, query, table_name)
    finally:
        S.parse = saved
    if out is None:
        return None
    keep, renamed = [], []
    for k, f in enumerate(out.schema):
        n = f.name
        for name, (hidden, *_rest) in calls.items():
            n = n.replace(f"{vis}.{hidden}", name)
            if n == hidden and f.name == hidden and any(it.expr is not None and it.expr.kind == "col" and it.expr.name == hidden and not it.alias for it in q.select):
                n = name
        if re.fullmatch(r"__json\d+", n):
            continue  # SELECT * never expands the hidden columns
        keep.append(k)
        renamed.append(n)
    return pa.record_batch([out.column(k) for k in keep], names=renamed)
