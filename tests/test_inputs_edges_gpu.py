"""The `generate` and `file` inputs (csrc/inputs.cu) at their edges, against plain references.

CSV scans are compared with oracle/csv_oracle.py (itself checked on the CPU by tests/test_csv_oracle_cpu.py), NDJSON
scans with oracle/json_oracle.py or with values derived from the record index, `generate` with `payload * n`.  Every
file is written from a seed or an index into tmp_path.  Every result is compared as whole arrays: schema names, types
and nullability, Array.equals per column, Float64 by bit pattern with the NULL slots masked, validate(full=True) on every
batch, through both read() and read_device().to_arrow().  Errors are compared by kind and by the full message, line
number included.  Where a case claims a route, the launch counts of the kernels (ark_kernel_timing_get) assert it.
"""
import ctypes as C
import json
import random

import numpy as np
import pyarrow as pa
import pytest

import number_corpus as NC
from arkflow_b200.input import FileInput, GenerateInput
from arkflow_b200.processor import ArkError
from oracle.csv_oracle import csv_read
from oracle.json_oracle import json_to_arrow
from oracle.sql_oracle import OracleError, sql_process

pytestmark = pytest.mark.gpu

PFX = "Read input failed: Arrow error: "
CHUNK = 8 << 20  # file_connect uploads the file in pinned chunks of this size, two in flight


@pytest.fixture(scope="module", autouse=True)
def timing(gpu):
    gpu.ark_kernel_timing_enable(1)
    yield gpu
    gpu.ark_kernel_timing_enable(0)


def launches(lib, name):
    ms, n = C.c_double(), C.c_int64()
    lib.ark_kernel_timing_get(name.encode(), C.byref(ms), C.byref(n))
    return n.value


def scan(path, kind, device=False, **cfg):
    """(batches, error): every batch up to EOF (error None) or up to the first other error."""
    it = {"type": kind, "path": str(path)}
    if "has_header" in cfg:
        it["has_header"] = cfg.pop("has_header")
    out = []
    try:
        inp = FileInput(dict(cfg, input_type=it))
        inp.connect()
        while True:
            out.append(inp.read_device().to_arrow() if device else inp.read()[0].record_batch)
    except ArkError as e:
        return out, (None if e.kind == "EOF" else e)


def same_batch(got, want, what=""):
    got.validate(full=True)
    assert got.schema.names == want.schema.names, what
    assert [str(t) for t in got.schema.types] == [str(t) for t in want.schema.types], what
    assert [f.nullable for f in got.schema] == [f.nullable for f in want.schema], what
    assert got.num_rows == want.num_rows, what
    for i, (g, w) in enumerate(zip(got.columns, want.columns)):
        assert g.null_count == w.null_count, (what, i)
        if pa.types.is_floating(w.type):
            assert g.is_valid().equals(w.is_valid()), (what, i)
            gb, wb = (x.fill_null(0.0).to_numpy(zero_copy_only=False).view(np.uint64) for x in (g, w))
            assert np.array_equal(gb, wb), (what, i, np.flatnonzero(gb != wb)[:5])
        else:
            assert g.equals(w), (what, i)


def same_batches(got, want, what=""):
    assert [b.num_rows for b in got] == [b.num_rows for b in want], what
    for k, (g, w) in enumerate(zip(got, want)):
        same_batch(g, w, (what, "batch", k))


def check_csv(tmp_path, data, batch_size=None, has_header=True, name="t.csv"):
    """Scans `data` both ways and compares with the oracle: the batches, or the error (kind and whole message).
    Returns what the oracle said."""
    p = tmp_path / name
    p.write_bytes(data)
    try:
        want = csv_read(data, has_header=has_header, batch_rows=batch_size)
    except OracleError as e:
        want = e
    cfg = {} if batch_size is None else {"batch_size": batch_size}
    if not has_header:
        cfg["has_header"] = False
    for device in (False, True):
        got, err = scan(p, "csv", device, **cfg)
        if isinstance(want, OracleError):
            assert err is not None, ("no error", want.message)
            assert (err.kind, err.message) == (want.kind, want.message)
        else:
            assert err is None, err.message
            same_batches(got, want, "device" if device else "host")
    return want


def expect_error(tmp_path, data, message, kind="Process", **kw):
    want = check_csv(tmp_path, data, **kw)
    assert isinstance(want, OracleError) and (want.kind, want.message) == (kind, message if kind != "Process" else PFX + message)


# ---- a CSV table that holds every kind of field -------------------------------------------------------------------------
_FLOATS = None


def float_strings():
    global _FLOATS
    if _FLOATS is None:
        c = NC.corpus(seed=7, per_class=40)
        _FLOATS = [s for k in sorted(c) for s in c[k]]
    return _FLOATS


STRS = ["plain", '"quoted, comma"', '"say ""hi"""', '"""lead"', '"trail"""', '""""""', '""""', "é漢\U0001F600", '"é,""漢"""', 'in"side',
        "x" * 15, "y" * 16, "z" * 17, "a", " ", '"' + "w" * 16 + '"']


def rich_rows(n, null_rows=()):
    """n records of id Int64, f Float64, b Boolean, s Utf8, q Int64 (quoted), e (always empty → Utf8, all NULL)."""
    fl = float_strings()
    rows = []
    for i in range(n):
        f = "" if i in null_rows or i % 13 == 5 else fl[(i * 31) % len(fl)]
        b = ["true", "FALSE", "TrUe", "fAlSe", '"true"', ""][i % 6]
        s = "" if i in null_rows else STRS[i % len(STRS)]
        q = '""' if i % 9 == 4 else '"%d"' % (i * 7919 - 40000)
        rows.append("%d,%s,%s,%s,%s," % (i - 5, f, b, s, q))
    return rows


def csv_bytes(rows, header="id,f,b,s,q,e", eol="\n", last_eol=True):
    lines = ([header] if header is not None else []) + rows
    return (eol.join(lines) + (eol if last_eol else "")).encode()


# ---- line index and upload ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def big_files(tmp_path_factory):
    """Two files of a little over 20 MiB: three upload chunks, the last one partial.  Every row is fixed-width with an odd
    width, so rows straddle both chunk boundaries, and distinct: its values follow from its index."""
    d = tmp_path_factory.mktemp("big")
    n = (20 << 20) // 29 + 5000
    idx = np.arange(n, dtype=np.int64)
    v = (idx * 2654435761) % 10 ** 9
    csv = b"id,v,s\n" + b"".join(b"%08d,%09d,rr%07x\n" % (i, x, i) for i, x in zip(idx.tolist(), v.tolist()))
    nj = b"".join(b'{"id":%8d,"v":%9d, "s":"rr%07x"}\n' % (i, x, i) for i, x in zip(idx.tolist(), v.tolist()))
    assert len(csv) > 2 * CHUNK + (1 << 20) and len(nj) > 2 * CHUNK + (1 << 20)
    assert (len(csv) - 7) % 29 == 0 and len(nj) % 47 == 0 and CHUNK % 29 and CHUNK % 47 and len(csv) % CHUNK and len(nj) % CHUNK
    (d / "big.csv").write_bytes(csv)
    (d / "big.json").write_bytes(nj)
    want = pa.record_batch({"id": pa.array(idx), "v": pa.array(v), "s": pa.array(["rr%07x" % i for i in range(n)])})
    return d, want


@pytest.mark.parametrize("kind,fname,cfg", [("csv", "big.csv", {}), ("csv", "big.csv", {"batch_size": 250_000}),
                                            ("json", "big.json", {"batch_size": 300_001})])
def test_a_file_of_three_upload_chunks_arrives_byte_for_byte(big_files, kind, fname, cfg):
    d, want = big_files
    got, err = scan(d / fname, kind, device="batch_size" in cfg, **cfg)
    assert err is None
    step = cfg.get("batch_size", want.num_rows)
    same_batches(got, [want.slice(o, step) for o in range(0, want.num_rows, step)])


@pytest.mark.parametrize("kind", ["csv", "json"])
@pytest.mark.parametrize("data", [b"", b"\n", b"\r\n", b"\n\n\r\n\n", b"\r"], ids=["0 bytes", "LF", "CRLF", "blank lines", "CR"])
def test_a_file_without_records_is_eof_on_the_first_read(timing, tmp_path, kind, data):
    p = tmp_path / "empty"
    p.write_bytes(data)
    timing.ark_kernel_timing_reset()
    for device in (False, True):
        assert scan(p, kind, device) == ([], None)
    assert launches(timing, "csv_parse_kernel") == 0 and launches(timing, "json_parse_kernel") == 0


@pytest.mark.parametrize("data", [b"x", b"a,b", b"a,b\n", b"\n\na,b\r\n\n"], ids=["1 byte", "header", "header LF", "header among blanks"])
def test_a_csv_file_with_a_header_only_is_eof_on_the_first_read(timing, tmp_path, data):
    timing.ark_kernel_timing_reset()
    assert check_csv(tmp_path, data) == []
    assert launches(timing, "csv_parse_kernel") == 0
    one = check_csv(tmp_path, data, has_header=False)  # the same bytes are one record without a header
    assert len(one) == 1 and one[0].num_rows == 1


@pytest.mark.parametrize("eol,last", [("\n", True), ("\n", False), ("\r\n", True), ("\r\n", False)])
def test_csv_line_endings(tmp_path, eol, last):
    rows = rich_rows(300, null_rows=(0, 7, 8, 299))
    want = check_csv(tmp_path, csv_bytes(rows, eol=eol, last_eol=last))
    same_batches(want, csv_read(csv_bytes(rows)))
    if eol == "\r\n":  # mixed: every third line ends in LF alone
        mixed = "".join(r + ("\n" if i % 3 == 0 else "\r\n") for i, r in enumerate(["id,f,b,s,q,e"] + rows)).encode()
        same_batches(check_csv(tmp_path, mixed), want)


def with_blanks(rows, eol="\n"):
    """Blank lines before the header, after it, in the middle alone and in runs, and at the end."""
    out = ["", "", rows[0], ""]
    for i, r in enumerate(rows[1:]):
        out.append(r)
        if i % 5 == 2:
            out.append("")
        if i % 11 == 3:
            out += ["", "\r", ""]
    return (eol.join(out + ["", "", ""]) + eol).encode()


@pytest.mark.parametrize("eol", ["\n", "\r\n"])
@pytest.mark.parametrize("batch_size", [None, 7])
def test_csv_blank_lines_are_no_records(tmp_path, eol, batch_size):
    rows = rich_rows(100)
    want = check_csv(tmp_path, with_blanks(["id,f,b,s,q,e"] + rows, eol), batch_size=batch_size)
    same_batches(want, csv_read(csv_bytes(rows), batch_rows=batch_size))  # the oracle: the same table as without them
    for tail in (b"\n\n", b"\r\n\r\n"):  # a file that ends in an empty line
        assert check_csv(tmp_path, b"a,b\n1,2\n3,4" + tail)[0].num_rows == 2


N_SPLIT = 300


@pytest.mark.parametrize("batch_size", [1, 2, N_SPLIT - 1, N_SPLIT, N_SPLIT + 1, 127, 128, 129])
def test_csv_batches_hold_batch_size_records_and_concatenate_to_the_whole(timing, tmp_path, batch_size):
    """Blank lines do not count toward a batch: every batch but the last has exactly batch_size records."""
    rows = rich_rows(N_SPLIT, null_rows=(0, 7, 8, N_SPLIT - 1))
    data = with_blanks(["id,f,b,s,q,e"] + rows)
    timing.ark_kernel_timing_reset()
    want = check_csv(tmp_path, data, batch_size=batch_size)
    n_batches = -(-N_SPLIT // batch_size)
    assert [b.num_rows for b in want] == [batch_size] * (N_SPLIT // batch_size) + ([N_SPLIT % batch_size] if N_SPLIT % batch_size else [])
    assert pa.Table.from_batches(want).combine_chunks().to_batches()[0].equals(csv_read(data)[0])
    # the route: one parse per batch and scan, one string kernel per Utf8 column (s and e) of each batch
    assert launches(timing, "csv_parse_kernel") == 2 * n_batches
    assert launches(timing, "csv_strings_kernel") == 2 * 2 * n_batches


# ---- CSV records --------------------------------------------------------------------------------------------------------
def test_csv_numbers_at_their_limits(tmp_path):
    ints = ["-9223372036854775808", "9223372036854775807", "-0", "+0", "0007", "-000", "+9223372036854775807", '"12"', ""]
    specials = [s + w for w in ("nan", "NaN", "NAN", "inf", "Inf", "INF", "infinity", "Infinity", "INFINITY", "iNfInItY") for s in ("", "+", "-")]
    fl = NC.HARD + float_strings() + specials + ["-0.0", "1.", ".5", "-.5e1", "1E5", "00.10", '"2.5"', "5", "+7", ""]
    bools = ["true", "false", "TRUE", "FALSE", "True", "tRuE", "fALSe", '"false"', ""]
    n = len(fl)
    rows = ["%s,%s,%s" % (ints[i % len(ints)], fl[i], bools[i % len(bools)]) for i in range(n)]
    want = check_csv(tmp_path, csv_bytes(rows, header="i,f,b"))
    assert [str(t) for t in want[0].schema.types] == ["int64", "double", "bool"]
    assert want[0].column("i").to_pylist()[:4] == [-2 ** 63, 2 ** 63 - 1, 0, 0]
    # one past each end of i64: Float64 inside the sample, an error after it
    assert str(check_csv(tmp_path, b"i\n1\n9223372036854775808\n")[0].schema.types[0]) == "double"
    body = "\n".join(["i"] + ["%d" % k for k in range(1000)])
    for past in ("9223372036854775808", "-9223372036854775809", "99999999999999999999999"):
        expect_error(tmp_path, (body + "\n" + past + "\n").encode(), "Parser error: Error while parsing value of line 1002")
    assert check_csv(tmp_path, (body + "\n9223372036854775807\n-9223372036854775808\n").encode())[0].num_rows == 1002


def test_csv_quoting(tmp_path):
    recs = ['"first",mid,last', 'first,mid,"last"', '"a,b","c,,d",","', '"""x","x""","""""', '"""""","""","a""""b"', '"","",""',
            '"12","true","1.5"', 'é"漢,"é,漢","""é"""', '"\U0001F600","é""",","', ' , ,"  "', 'un"quoted"x,q""q,"', 'x,y,"open,z']
    for w in (0, 1, 15, 16, 17, 70_000):
        recs += ["%s,%d,x" % ("s" * w, w), '"%s",%d,"y"' % ('q""' * (w // 3) + "q" * (w % 3), w)]
    want = check_csv(tmp_path, csv_bytes(recs, header="a,b,c"))[0]
    assert want.column("a").to_pylist()[:6] == ["first", "first", "a,b", '"x', '""', None]
    assert want.column("c").to_pylist()[10:12] == [None, "open,z"] and want.column("b")[10].as_py() == 'q""q'
    alone = check_csv(tmp_path, b'a\n"only"\n""\n""""\n"x,y"\nplain\n')[0]  # one column: a quoted field alone on its line
    assert alone.column(0).to_pylist() == ["only", None, '"', "x,y", "plain"]
    typed = check_csv(tmp_path, b'i,f,b\n"1","2.5","TRUE"\n"-7","1e3","false"\n"","",""\n')[0]
    assert typed.to_pydict() == {"i": [1, -7, None], "f": [2.5, 1000.0, None], "b": [True, False, None]}


def test_csv_nulls(timing, tmp_path):
    # rows 4-7 are one batch in which every column, whatever its type, is all NULL
    rows = ["1,1.5,true,x", "2,2.5,false,y", "3,nan,TRUE,z", "4,4,true,w"] + [",,,"] * 4 + ["9,9.5,false,v"]
    want = check_csv(tmp_path, csv_bytes(rows, header="i,f,b,s"), batch_size=4)
    assert [str(t) for t in want[0].schema.types] == ["int64", "double", "bool", "string"]
    assert [c.null_count for c in want[1].columns] == [4, 4, 4, 4] and [c.null_count for c in want[0].columns] == [0, 0, 0, 0]
    p = tmp_path / "nonull.csv"
    p.write_bytes(csv_bytes(["%d,%d.5,true,s%d" % (i, i, i) for i in range(77)], header="i,f,b,s"))
    for device in (False, True):  # no NULL anywhere: no validity buffer at all
        (b,), err = scan(p, "csv", device)
        assert err is None and all(c.null_count == 0 and c.buffers()[0] is None for c in b.columns)
    for k in (0, 7, 8, 76):
        rows = ["%s,%s,%s,%s" % (("", "", "", "") if i == k else (i, "%d.5" % i, "true", "s%d" % i)) for i in range(77)]
        assert check_csv(tmp_path, csv_bytes(rows, header="i,f,b,s"))[0].column("s").is_null().to_pylist().index(True) == k


def test_csv_inference_sample_is_the_first_1000_records(tmp_path):
    base = ["%d,,%d,%d" % (i, i, i) for i in range(1000)]
    head = "a,late,mix,c"
    late = check_csv(tmp_path, csv_bytes(base + ["5,filled,1,2"], header=head))[0]  # 1001 records
    assert str(late.schema.types[1]) == "string" and late.column("late").to_pylist() == [None] * 1000 + ["filled"]
    inside = base[:999] + ["5,,2.5,true"]  # exactly 1000 records: the last one still decides
    t = check_csv(tmp_path, csv_bytes(inside, header=head))[0]
    assert [str(x) for x in t.schema.types] == ["int64", "string", "double", "string"] and t.num_rows == 1000
    expect_error(tmp_path, csv_bytes(base + ["5,,2.5,1"], header=head), "Parser error: Error while parsing value of line 1002")
    # blank lines are not records: they do not use up the sample, and the message counts them
    expect_error(tmp_path, with_blanks([head] + base + ["5,,2.5,1"]), "Parser error: Error while parsing value of line %d" %
                 (with_blanks([head] + base + ["5,,2.5,1"]).split(b"\n").index(b"5,,2.5,1") + 1))
    # without a header the sample is records 1-1000 as well
    expect_error(tmp_path, csv_bytes(base + ["5,,2.5,1"], header=None), "Parser error: Error while parsing value of line 1001", has_header=False)
    t = check_csv(tmp_path, csv_bytes(base[:999] + ["5,,2.5,1"], header=None), has_header=False)[0]
    assert t.schema.names == ["column_1", "column_2", "column_3", "column_4"] and str(t.schema.types[2]) == "double"


def test_csv_width_and_header_names(tmp_path):
    one = check_csv(tmp_path, b"only\n1\n\n2\n\n")[0]
    assert one.to_pydict() == {"only": [1, 2]}
    kinds = ["%d", "%d.25", "true", "s%d"]
    rows = [",".join(kinds[c % 4].replace("%d", str(i * 32 + c)) for c in range(32)) for i in range(50)]
    wide = check_csv(tmp_path, csv_bytes(rows, header=",".join("c%d" % c for c in range(32))))[0]
    assert wide.num_columns == 32
    rows33 = [r + ",x" for r in rows]
    expect_error(tmp_path, csv_bytes(rows33, header=",".join("c%d" % c for c in range(33))), "csv input: more than 32 columns", kind="Unsupported")
    dup = check_csv(tmp_path, 'x,,x,"é,"\n1,2,3,4\n'.encode())[0]
    assert dup.schema.names == ["x", "", "x", "é,"]
    nh = check_csv(tmp_path, csv_bytes(rich_rows(40), header=None), has_header=False)[0]
    assert nh.schema.names == ["column_%d" % i for i in range(1, 7)] and nh.num_rows == 40


def good(n, k0=0):
    return [b"%d,%d.5,true,s%d" % (i, i, i) for i in range(k0, k0 + n)]


def lines(*parts):
    return b"i,f,b,s\n" + b"".join(x + b"\n" for p in parts for x in p)


@pytest.mark.parametrize("bad,message", [
    (b"5,1.5,true", "Csv error: incorrect number of fields for line 1202"),
    (b"5", "Csv error: incorrect number of fields for line 1202"),
    (b"5,1.5,true,s,extra", "Csv error: incorrect number of fields for line 1202"),
    (b"5,1.5,true,s,", "Csv error: incorrect number of fields for line 1202"),
    (b'5,1.5,true,"s"x', "Csv error: incorrect number of fields for line 1202"),
    (b"5.0,1.5,true,s", "Parser error: Error while parsing value of line 1202"),
    (b"5,1.5.1,true,s", "Parser error: Error while parsing value of line 1202"),
    (b"5,1.5,yes,s", "Parser error: Error while parsing value of line 1202"),
    (b"5,1.5,true,\xe9", "Csv error: Encountered invalid UTF-8 data for line 1202"),
    (b"5,1.5,true,\"a\xed\xa0\x80\"", "Csv error: Encountered invalid UTF-8 data for line 1202"),
    (b"\xff,1.5,true,s", "Parser error: Error while parsing value of line 1202"),
    # several faults in one line: the field count first, then a bad value, then invalid UTF-8
    (b"x,1.5,true,\xff,extra", "Csv error: incorrect number of fields for line 1202"),
    (b"5,1.5,maybe,\xff", "Parser error: Error while parsing value of line 1202"),
])
def test_csv_errors_carry_the_message_and_the_physical_line(timing, tmp_path, bad, message):
    timing.ark_kernel_timing_reset()
    expect_error(tmp_path, lines(good(1200), [bad], good(300, 1200)), message)
    assert launches(timing, "csv_strings_kernel") == 0  # the failing batch (the file's only one) copies no string


def test_csv_invalid_utf8_in_the_header_and_in_the_sample(tmp_path):
    expect_error(tmp_path, b"\n\na,\xffb\n1,2\n", "Csv error: Encountered invalid UTF-8 data for line 3")
    expect_error(tmp_path, b"a,b\n1,x\n2,\xc3\x28\n", "Csv error: Encountered invalid UTF-8 data for line 3")
    expect_error(tmp_path, b"a,b\n1,x\n\xff,y\n", "Csv error: Encountered invalid UTF-8 data for line 3")  # a is Utf8 by inference


@pytest.mark.parametrize("first,second,message", [
    (b"5,1.5,true,\xff", b"5,1.5,true", "Csv error: Encountered invalid UTF-8 data for line 1502"),
    (b"5,1.5,true", b"5,1.5,true,\xff", "Csv error: incorrect number of fields for line 1502"),
    (b"z,1.5,true,s", b"5,1.5,true,s,s", "Parser error: Error while parsing value of line 1502"),
    (b"5,1.5,true,s,s", b"z,1.5,true,s", "Csv error: incorrect number of fields for line 1502"),
])
def test_csv_two_bad_lines_in_one_batch_name_the_first(tmp_path, first, second, message):
    expect_error(tmp_path, lines(good(1500), [first], good(4000, 1500), [second], good(500, 5500)), message)


def test_csv_a_bad_line_in_the_second_batch_comes_after_a_good_first_batch(tmp_path):
    data = lines(good(1500), [b""], good(700, 1500), [b"5,1.5"], good(300, 2200))
    p = tmp_path / "second.csv"
    p.write_bytes(data)
    assert isinstance(check_csv(tmp_path, data, batch_size=1500), OracleError)
    for device in (False, True):
        got, err = scan(p, "csv", device, batch_size=1500)
        same_batches(got, csv_read(lines(good(1500))))
        assert (err.kind, err.message) == ("Process", PFX + "Csv error: incorrect number of fields for line 2203")


@pytest.mark.parametrize("query,grouped", [
    ("SELECT s, id, f FROM flow WHERE id >= 100 AND f < 1500.5", False),
    ("SELECT s, COUNT(*), SUM(id), MIN(f) FROM flow GROUP BY s", True),
])
def test_csv_scan_with_a_query(tmp_path, query, grouped):
    rows = ["%d,%d.25,%s,%s,%d," % (i - 5, i, ["true", "FALSE", ""][i % 3], STRS[i % len(STRS)], i * 7919 - 40000) for i in range(2000)]
    data = with_blanks(["id,f,b,s,q,e"] + rows)
    p = tmp_path / "q.csv"
    p.write_bytes(data)
    want = sql_process(csv_read(data)[0], query)
    (got,), err = scan(p, "csv", query={"query": query})
    assert err is None
    got.validate(full=True)
    if grouped:
        key = lambda b: sorted(zip(*[c.to_pylist() for c in b.columns]), key=repr)
        assert got.schema.names == want.schema.names and key(got) == key(want)
    else:
        assert got.equals(want)


# ---- NDJSON through the file input --------------------------------------------------------------------------------------
def nd_records(n):
    return [json.dumps({"id": i * 7919 - 4000, "f": i / 8.0, "s": STRS[i % len(STRS)] + str(i), "b": i % 3 == 0},
                       ensure_ascii=i % 2 == 0).encode() for i in range(n)]


def nd_oracle(payloads, batch_size=None):
    whole = json_to_arrow(pa.record_batch({"__value__": pa.array(payloads, pa.binary())}))
    step = batch_size or whole.num_rows
    return [whole.slice(o, step) for o in range(0, whole.num_rows, step)]


@pytest.mark.parametrize("eol", ["\n", "\r\n"])
@pytest.mark.parametrize("batch_size", [None, 1, 2, N_SPLIT - 1, N_SPLIT, N_SPLIT + 1, 127, 128, 129])
def test_ndjson_lines_blank_lines_and_batches(tmp_path, eol, batch_size):
    """Empty lines are no records for NDJSON either: every batch but the last has batch_size records."""
    recs = nd_records(N_SPLIT)
    p = tmp_path / "t.json"
    data = with_blanks([r.decode() for r in recs], eol)
    p.write_bytes(data.rstrip(b"\r\n") if batch_size in (None, 2) else data)  # the last record without a terminator, too
    cfg = {} if batch_size is None else {"batch_size": batch_size}
    for device in (False, True):
        got, err = scan(p, "json", device, **cfg)
        assert err is None
        same_batches(got, nd_oracle(recs, batch_size), (eol, batch_size, device))


def test_ndjson_lines_of_spaces_are_dropped_by_the_decoder(timing, tmp_path):
    """A line of spaces is a line (it takes a slot of its batch window) that holds no record.  A window of nothing but
    such lines yields no batch: the scan moves on to the next window."""
    recs = nd_records(10)
    body = [b"  ", recs[0], b" \t ", recs[1]] + [b"   "] * 4 + recs[2:]
    p = tmp_path / "spaces.json"
    p.write_bytes(b"\n".join(body) + b"\n")
    timing.ark_kernel_timing_reset()
    got, err = scan(p, "json", batch_size=4)
    assert err is None
    assert [b.num_rows for b in got] == [2, 4, 4]  # windows: 2 records + 2 space lines, 4 space lines (no batch), 4, 4
    same_batches([pa.Table.from_batches(got).combine_chunks().to_batches()[0]], nd_oracle(recs))
    assert launches(timing, "rebase_offsets_kernel") == 4  # four windows were decoded for three batches


def test_ndjson_schema_is_merged_over_the_first_1000_records(tmp_path):
    """DataFusion infers an NDJSON file's schema once, over its first schema_infer_max_records = 1000 records
    (NdJsonReadOptions::default(), file.rs:219-226), and arrow-json's decoder, which is not strict, ignores a key the
    schema lacks: a field first seen at record 1000 is a column, one first seen at record 1001 is dropped."""
    def write(name, n_before):
        rows = [b'{"a": %d}' % i for i in range(n_before)] + [b'{"a": 0.5, "b": "new"}'] + [b'{"a": %d, "b": "x"}' % i for i in range(5)]
        p = tmp_path / name
        p.write_bytes(b"\n\n" + b"\n\n".join(rows) + b"\n")  # empty lines do not use up the sample
        return p
    n = 999
    want_in = pa.record_batch({"a": pa.array([float(i) for i in range(n)] + [0.5] + [float(i) for i in range(5)]),
                               "b": pa.array([None] * n + ["new"] + ["x"] * 5, pa.utf8())})
    for device in (False, True):
        (got,), err = scan(write("in.json", n), "json", device)
        assert err is None
        same_batch(got, want_in)
    n = 1000  # record 1001 brings `b` and a fractional `a`: the schema is fixed as {a: Int64}
    (got,), err = scan(write("out.json", n), "json")
    assert err is None and got.schema.names == ["a"] and str(got.schema.types[0]) == "int64"
    assert got.column("a").to_pylist() == list(range(n)) + [0] + list(range(5))


# ---- generate -----------------------------------------------------------------------------------------------------------
def payload_of(length, seed=1):
    """ASCII for short payloads; longer ones mix in multi-byte UTF-8, cut so that the text has exactly `length` bytes."""
    rng = random.Random(seed * 1000003 + length)
    out, size = [], 0
    while size < length:
        ch = rng.choice("abcxyz0189 {}:,é漢\U0001F600")
        if size + len(ch.encode()) > length:
            ch = "p"
        out.append(ch)
        size += len(ch.encode())
    assert len("".join(out).encode()) == length
    return "".join(out)


def check_generate(ctx, batch_size, lib):
    raw = ctx.encode()
    lib.ark_kernel_timing_reset()
    inp = GenerateInput({"context": ctx, "interval": "1ns", "batch_size": batch_size})
    want_off = np.arange(batch_size + 1, dtype=np.int64) * len(raw)
    for k, device in enumerate((False, True, False)):  # the replicated column is built once and shared by every read
        b = inp.read_device().to_arrow() if device else inp.read()[0].record_batch
        b.validate(full=True)
        assert b.schema.names == ["__value__"] and b.schema.types == [pa.binary()] and not b.schema.field(0).nullable
        col = b.column(0)
        assert len(col) == batch_size and col.null_count == 0
        off = np.frombuffer(col.buffers()[1], np.int32)[col.offset:col.offset + batch_size + 1]
        assert np.array_equal(off - off[0], want_off)
        data = bytes(col.buffers()[2] or b"")[int(off[0]):int(off[-1])]
        assert data == raw * batch_size, (len(raw), batch_size, k)
    assert launches(lib, "replicate_kernel") == 1


@pytest.mark.parametrize("length", [0, 1, 2, 15, 16, 17, 31, 33, 63, 255, 4096, 49_152, 49_153, 200_000])
def test_generate_replicates_a_context_of_any_length(timing, length):
    """16 bytes per thread: lengths around the vector width, a last partial group, and contexts beyond 48 KiB."""
    ctx = payload_of(length)
    for batch_size in ((0, 1, 2, 15, 16, 17, 1000) if length <= 4096 else (1, 3, 17)):
        check_generate(ctx, batch_size, timing)


@pytest.mark.parametrize("count,batch_size,reads", [(0, 1, 0), (0, 4, 0), (3, 4, 0), (4, 4, 1), (8, 4, 2), (10, 4, 2), (5, 1, 5)])
def test_generate_count_and_batch_size(gpu, count, batch_size, reads):
    """generate.rs:71-80: EOF once `count` messages were produced, or when the next batch would exceed it."""
    inp = GenerateInput({"context": "é{}", "interval": "1ns", "count": count, "batch_size": batch_size})
    for _ in range(reads):
        assert inp.read()[0].record_batch.column(0).to_pylist() == ["é{}".encode()] * batch_size
    for _ in range(2):
        with pytest.raises(ArkError) as e:
            inp.read()
        assert e.value.kind == "EOF"


def test_generate_refuses_a_batch_beyond_a_binary_array_before_it_allocates(timing):
    timing.ark_kernel_timing_reset()
    inp = GenerateInput({"context": "x" * 1000, "interval": "1ns", "batch_size": 2_147_484})  # 2 147 484 000 bytes > 2^31 - 1
    for read in (inp.read, inp.read_device):
        with pytest.raises(ArkError) as e:
            read()
        assert e.value.kind == "Process" and e.value.message == "generate: batch_size x context exceeds a Binary array's 2 GiB"
    assert launches(timing, "replicate_kernel") == 0
    ok = GenerateInput({"context": "x" * 1000, "interval": "1ns", "batch_size": 2_147})
    assert ok.read()[0].record_batch.column(0)[2_146].as_py() == b"x" * 1000
