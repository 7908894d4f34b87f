"""CPU oracle for the CSV scan of the `file` input (csrc/csv.cu) — TEST INFRASTRUCTURE (see oracle/__init__.py).

The reference reads a CSV file with DataFusion's `ctx.read_csv(path, CsvReadOptions::default())`
(crates/arkflow-plugin/src/input/file.rs:229-237), which is arrow-csv 55.2 over csv-core.  This module restates, in
plain Python and without pyarrow.csv, the contract the library documents for that scan:

  * a record is one line; `\\n` and `\\r\\n` both end a line and the last line needs no terminator;
  * an empty line (nothing but `\\r` before its `\\n`) is skipped: it is no record and counts toward no batch, but it
    still counts as a physical line in error messages;
  * `"` opens a quoted field when it is the field's first byte, `""` inside it is one quote; elsewhere `"` is data;
  * an empty field, quoted or not, is NULL for every type;
  * column names come from the first line that is not empty, or are column_1, column_2, … without a header;
  * types come from the first 1000 records: Int64 when every non-empty value is [+-]?digits within i64, Float64 when
    they are decimals or nan / inf / infinity (any case, optional sign), Int64 with Float64 gives Float64, Boolean for
    true / false in any case, Utf8 for anything else or any other mix; a column without a value in the sample is Utf8;
  * Float64 values are correctly rounded (Python's float() is);
  * errors name the FIRST failing line in file order by its 1-based physical line number; within one line a wrong
    number of fields comes first, then a value that does not parse, then invalid UTF-8 in a Utf8 field;
  * more than 32 columns is Unsupported.

Where this contract differs from arrow-csv (csrc/csv.cu's header names the first three):
  * quoted fields may not contain line breaks: a line break always ends the record;
  * dates and timestamps stay Utf8 (arrow-csv infers Date32 / Timestamp);
  * the sample is the first 1000 records as here, but arrow-csv's integer pattern has no leading `+`: `+5` is Utf8
    there and Int64 here;
  * an integer beyond i64 is Float64 here when its column is inferred and a parse error after the sample; arrow-csv
    infers Int64 from the digits and fails on the value;
  * bytes between a closing quote and the next delimiter (`"ab"cd`) are a field-count error here; csv-core appends
    them to the field;
  * a quoted field that never closes ends at the end of its line;
  * invalid UTF-8 in a numeric or Boolean field after the sample is reported as a value that does not parse.
"""
from __future__ import annotations

import re
from typing import Optional

import pyarrow as pa

from .sql_oracle import OracleError

SAMPLE_ROWS = 1000
MAX_COLS = 32

_INT_RE = re.compile(rb"[+-]?[0-9]+\Z")
_DEC_RE = re.compile(rb"[+-]?([0-9]+\.?[0-9]*|\.[0-9]+)([eE][+-]?[0-9]+)?\Z")
_SPECIAL_RE = re.compile(rb"([+-]?)(nan|inf|infinity)\Z", re.I)

_PREFIX = "Read input failed: Arrow error: "


def _err_fields(line):
    return OracleError("Process", _PREFIX + "Csv error: incorrect number of fields for line %d" % line)


def _err_value(line):
    return OracleError("Process", _PREFIX + "Parser error: Error while parsing value of line %d" % line)


def _err_utf8(line):
    return OracleError("Process", _PREFIX + "Csv error: Encountered invalid UTF-8 data for line %d" % line)


def records(data: bytes) -> list[tuple[int, bytes]]:
    """(physical line number, line without its terminator) of every line that is not empty."""
    out = []
    pieces = data.split(b"\n")
    if pieces[-1] == b"":
        pieces.pop()  # the bytes after the last terminator are a line only when there are any
    for k, ln in enumerate(pieces):
        ln = ln.rstrip(b"\r")
        if ln:
            out.append((k + 1, ln))
    return out


def _field(line: bytes, pos: int, delim: int) -> tuple[bytes, int]:
    """The decoded field that starts at `pos` and the position just after it (after a closing quote, if any)."""
    if pos < len(line) and line[pos] == 0x22:
        pos += 1
        start = pos
        while pos < len(line):
            if line[pos] == 0x22:
                if pos + 1 < len(line) and line[pos + 1] == 0x22:
                    pos += 2
                    continue
                break
            pos += 1
        body = line[start:pos].replace(b'""', b'"')
        return body, min(pos + 1, len(line))
    end = line.find(bytes([delim]), pos)
    if end < 0:
        end = len(line)
    return line[pos:end], end


def split_all(line: bytes, delim: int) -> list[bytes]:
    """Every field of a line (the header, and the sample rows during inference).  Splitting stops at a field that is
    not followed by a delimiter."""
    out, pos = [], 0
    while True:
        f, pos = _field(line, pos, delim)
        out.append(f)
        if pos < len(line) and line[pos] == delim:
            pos += 1
            continue
        return out


def split_n(line: bytes, delim: int, n: int) -> Optional[list[bytes]]:
    """Exactly n fields, or None when the line has fewer or more."""
    out, pos = [], 0
    for c in range(n):
        f, pos = _field(line, pos, delim)
        out.append(f)
        if c + 1 == n:
            break
        if pos < len(line) and line[pos] == delim:
            pos += 1
        else:
            return None
    return out if pos == len(line) else None


def _is_i64(v: bytes) -> bool:
    return bool(_INT_RE.match(v)) and -(2 ** 63) <= int(v) <= 2 ** 63 - 1


def _is_f64(v: bytes) -> bool:
    return bool(_SPECIAL_RE.match(v) or _DEC_RE.match(v))


def _is_bool(v: bytes) -> bool:
    return v.lower() in (b"true", b"false")


def _merge(cur: Optional[str], v: bytes) -> Optional[str]:
    if not v:
        return cur
    t = "i64" if _is_i64(v) else "f64" if _is_f64(v) else "bool" if _is_bool(v) else "str"
    if cur is None or cur == t:
        return t
    if {cur, t} == {"i64", "f64"}:
        return "f64"
    return "str"


def _to_f64(v: bytes) -> float:
    m = _SPECIAL_RE.match(v)
    if m:
        if m.group(2).lower() == b"nan":
            return float("nan")
        return float("-inf") if m.group(1) == b"-" else float("inf")
    return float(v.decode("ascii"))  # correctly rounded; the grammar was checked by _DEC_RE


_ARROW = {"i64": pa.int64(), "f64": pa.float64(), "bool": pa.bool_(), "str": pa.utf8()}


def csv_read(data: bytes, has_header: bool = True, delim: bytes = b",", batch_rows: Optional[int] = None) -> list[pa.RecordBatch]:
    """The batches the scan returns, each of `batch_rows` records but the last (one batch without `batch_rows`); no
    batches when the file has no data record.  Raises the error of the first failing line."""
    d = delim[0]
    recs = records(data)
    if not recs:
        return []
    head = split_all(recs[0][1], d)
    if has_header:
        for h in head:
            try:
                h.decode("utf-8")
            except UnicodeDecodeError:
                raise _err_utf8(recs[0][0])
        names = [h.decode("utf-8") for h in head]
        recs = recs[1:]
    else:
        names = ["column_%d" % (i + 1) for i in range(len(head))]
    nc = len(names)
    if nc > MAX_COLS:
        raise OracleError("Unsupported", "csv input: more than 32 columns")
    types: list[Optional[str]] = [None] * nc
    for _, ln in recs[:SAMPLE_ROWS]:
        for c, v in enumerate(split_all(ln, d)[:nc]):
            types[c] = _merge(types[c], v)
    types = [t or "str" for t in types]
    schema = pa.schema([pa.field(n, _ARROW[t], True) for n, t in zip(names, types)])

    cols: list[list] = [[] for _ in range(nc)]
    for line_no, ln in recs:
        fields = split_n(ln, d, nc)
        if fields is None:
            raise _err_fields(line_no)
        row, bad_utf8 = [], False
        for t, v in zip(types, fields):
            if not v:
                row.append(None)
            elif t == "i64":
                if not _is_i64(v):
                    raise _err_value(line_no)
                row.append(int(v))
            elif t == "f64":
                if not _is_f64(v):
                    raise _err_value(line_no)
                row.append(_to_f64(v))
            elif t == "bool":
                if not _is_bool(v):
                    raise _err_value(line_no)
                row.append(v.lower() == b"true")
            else:
                try:
                    row.append(v.decode("utf-8"))
                except UnicodeDecodeError:
                    bad_utf8 = True  # reported only when no value of the line fails to parse
                    row.append(None)
        if bad_utf8:
            raise _err_utf8(line_no)
        for c, x in enumerate(row):
            cols[c].append(x)
    n = len(recs)
    step = batch_rows or max(n, 1)
    out = []
    for r0 in range(0, n, step):
        arrays = [pa.array(cols[c][r0:r0 + step], type=schema.field(c).type) for c in range(nc)]
        out.append(pa.RecordBatch.from_arrays(arrays, schema=schema))
    return out
