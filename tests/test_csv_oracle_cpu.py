"""oracle/csv_oracle.py checked on the CPU before any kernel is compared with it: against Arrow C++'s CSV reader over
a seeded corpus kept to the ground where the two readers agree (no dates, no leading `+`, no NA spellings, no line
breaks inside quotes), and against hand-written tables for every rule of the contract in the oracle's docstring."""
import io
import random
import struct

import pyarrow as pa
import pyarrow.csv as pacsv
import pytest

from oracle.csv_oracle import csv_read, records, split_all, split_n
from oracle.sql_oracle import OracleError
from number_corpus import HARD

PFX = "Read input failed: Arrow error: "


def one(data, **kw):
    bs = csv_read(data, **kw)
    assert len(bs) == 1
    return bs[0]


def bits(arr):
    return [None if x is None else struct.unpack("<Q", struct.pack("<d", x))[0] for x in arr.to_pylist()]


def corpus_file(seed, n, eol):
    rng = random.Random(seed)
    words = ["plain", "with space", "é漢", "semi;colon", "x"]
    lines = ["id,i,f,b,s,q"]
    for k in range(n):
        i = "" if rng.random() < 0.1 else str(rng.randrange(-2 ** 63, 2 ** 63) if k % 7 == 0 else rng.randrange(-99, 99))
        f = "" if rng.random() < 0.1 else rng.choice([repr(rng.uniform(-1e6, 1e6)), "%de%d" % (rng.randrange(1, 10 ** 17), rng.randrange(-330, 300)),
                                                     str(rng.randrange(-5, 5)), rng.choice(HARD)])
        b = rng.choice(["true", "FALSE", "True", "false", ""])
        s = rng.choice(words) + str(k) if rng.random() < 0.9 else ""
        q = rng.choice(['"a,b%d"' % k, '"say ""hi"""', '""""', '"%d"' % k, '""', "bare%d" % k])
        lines.append(",".join([str(k), i, f, b, s, q]))
        if k % 37 == 5:
            lines.append("")  # both readers skip empty lines
    return (eol.join(lines) + (eol if seed % 2 else "")).encode()


@pytest.mark.parametrize("seed,n,eol", [(1, 50, "\n"), (2, 1500, "\n"), (3, 1500, "\r\n"), (4, 999, "\n")])
def test_oracle_agrees_with_arrow_cpp_where_the_readers_agree(seed, n, eol):
    data = corpus_file(seed, n, eol)
    want = pacsv.read_csv(io.BytesIO(data), convert_options=pacsv.ConvertOptions(
        null_values=[""], strings_can_be_null=True, quoted_strings_can_be_null=True)).combine_chunks()
    got = one(data)
    assert got.num_rows == n and got.schema.names == want.schema.names
    assert [str(t) for t in got.schema.types] == [str(t) for t in want.schema.types] == ["int64", "int64", "double", "bool", "string", "string"]
    for name in want.schema.names:
        g, w = got.column(name), want.column(name).combine_chunks()
        if name == "f":
            assert bits(g) == bits(w)
        else:
            assert g.equals(w), name


def test_lines_terminators_and_empty_lines():
    assert records(b"") == [] and records(b"\n") == [] and records(b"\r\n\n\r\r\n") == []
    assert records(b"a\nb") == [(1, b"a"), (2, b"b")] and records(b"a\nb\n") == [(1, b"a"), (2, b"b")]
    assert records(b"\n\na\r\n\r\n\nb\r\n\n") == [(3, b"a"), (6, b"b")]
    assert records(b" \n") == [(1, b" ")]  # a line of spaces is a record
    for data in (b"", b"\n", b"\n\r\n\n", b"a,b", b"a,b\n", b"a,b\n\n\n"):
        assert csv_read(data) == []
    want = one(b"a,b\n1,x\n2,y\n").to_pydict()
    assert want == {"a": [1, 2], "b": ["x", "y"]}
    for data in (b"a,b\n1,x\n2,y", b"a,b\r\n1,x\r\n2,y\r\n", b"a,b\r\n1,x\n2,y\r\n", b"\n\na,b\n\n1,x\n\r\n\n2,y\n\n"):
        assert one(data).to_pydict() == want


def test_quoting():
    assert split_all(b'"a,b",c,"d"', 44) == [b"a,b", b"c", b"d"]
    assert split_all(b'"""x","x""","""""",""""', 44) == [b'"x', b'x"', b'""', b'"']
    assert split_all(b'a"b,""', 44) == [b'a"b', b""]  # a quote inside an unquoted field is data
    assert split_all(b'"open,x', 44) == [b"open,x"]   # a quoted field that never closes ends with its line
    assert split_n(b'"ab"cd,e', 44, 2) is None and split_n(b'e,"ab"cd', 44, 2) is None
    assert split_n(b"1,2,", 44, 2) is None and split_n(b"1,2,", 44, 3) == [b"1", b"2", b""]
    b = one('n,s,t\n"1","é,""漢""","true"\n"","",""\n'.encode())
    assert [str(t) for t in b.schema.types] == ["int64", "string", "bool"]
    assert b.to_pydict() == {"n": [1, None], "s": ['é,"漢"', None], "t": [True, None]}


def test_types_and_inference():
    b = one(b"i,f,m,b,s,c,e,p\n"
            b"-9223372036854775808,1.5,1,true,x,1,,+5\n"
            b"9223372036854775807,nan,2.5,FALSE,2,true,,-0\n"
            b"007,-Infinity,,TrUe,,,,0\n")
    assert [str(t) for t in b.schema.types] == ["int64", "double", "double", "bool", "string", "string", "string", "int64"]
    assert b.column("i").to_pylist() == [-2 ** 63, 2 ** 63 - 1, 7] and b.column("p").to_pylist() == [5, 0, 0]
    assert bits(b.column("f")) == [0x3FF8000000000000, 0x7FF8000000000000, 0xFFF0000000000000]
    assert b.column("m").to_pylist() == [1.0, 2.5, None] and b.column("b").to_pylist() == [True, False, True]
    assert b.column("c").to_pylist() == ["1", "true", None] and b.column("e").null_count == 3
    # one past i64 inside the sample makes the column Float64; a date stays Utf8
    b = one(b"a,d\n9223372036854775808,2024-01-02\n1,2024-01-03\n")
    assert [str(t) for t in b.schema.types] == ["double", "string"] and b.column("a").to_pylist() == [9223372036854775808.0, 1.0]
    for sp in ("nan", "NaN", "+NAN", "-nan", "inf", "+Inf", "-INF", "infinity", "-InFiNiTy", "+INFINITY"):
        x = one(("f\n%s\n" % sp).encode()).column(0)
        assert str(x.type) == "double"
        want = 0x7FF8000000000000 if "nan" in sp.lower() else (0xFFF0000000000000 if sp[0] == "-" else 0x7FF0000000000000)
        assert bits(x) == [want], sp
    assert bits(one(("f\n" + "\n".join(HARD) + "\n").encode()).column(0)) == [struct.unpack("<Q", struct.pack("<d", float(h)))[0] for h in HARD]


def test_the_sample_is_the_first_1000_records():
    rows = ["a,b"] + ["%d," % i for i in range(1000)]
    b = one(("\n".join(rows + ["7,late"]) + "\n").encode())  # b: no evidence in the sample → Utf8, filled after it
    assert [str(t) for t in b.schema.types] == ["int64", "string"] and b.column("b").to_pylist() == [None] * 1000 + ["late"]
    b = one(("\n".join(rows[:1000] + ["2.5,"]) + "\n").encode())  # record 1000 is still in the sample
    assert str(b.schema.types[0]) == "double" and b.num_rows == 1000
    with pytest.raises(OracleError) as e:  # record 1001 is not; blank lines do not count toward the sample
        csv_read(("\n\n" + "\n".join(rows + ["2.5,"]) + "\n").encode())
    assert e.value.kind == "Process" and e.value.message == PFX + "Parser error: Error while parsing value of line 1004"
    with pytest.raises(OracleError) as e:
        csv_read(("\n".join(rows[1:] + ["2.5,"]) + "\n").encode(), has_header=False)
    assert e.value.message == PFX + "Parser error: Error while parsing value of line 1001"


def test_header_names_width_and_batches():
    b = one(b"x,,x\n1,2,3\n")
    assert b.schema.names == ["x", "", "x"] and [c.to_pylist() for c in b.columns] == [[1], [2], [3]]
    b = one(b"1,a\n2,b\n", has_header=False)
    assert b.schema.names == ["column_1", "column_2"] and b.to_pydict() == {"column_1": [1, 2], "column_2": ["a", "b"]}
    assert all(f.nullable for f in b.schema)
    assert one((",".join("c%d" % i for i in range(32)) + "\n" + ",".join(["1"] * 32) + "\n").encode()).num_columns == 32
    with pytest.raises(OracleError) as e:
        csv_read((",".join("c%d" % i for i in range(33)) + "\n").encode())
    assert e.value.kind == "Unsupported"
    data = b"a\n" + b"".join(b"%d\n\n" % i for i in range(10))
    bs = csv_read(data, batch_rows=4)
    assert [x.num_rows for x in bs] == [4, 4, 2] and pa.Table.from_batches(bs).column(0).to_pylist() == list(range(10))
    assert one(b"a;b\n1;x,y\n", delim=b";").to_pydict() == {"a": [1], "b": ["x,y"]}


@pytest.mark.parametrize("data,msg", [
    (b"a,b\n1,2\n3\n", "Csv error: incorrect number of fields for line 3"),
    (b"a,b\n1,2\n\n\n3,4,5\n", "Csv error: incorrect number of fields for line 5"),
    (b"a,b\n1,2,\n", "Csv error: incorrect number of fields for line 2"),
    (b"\n\xff,b\n1,2\n", "Csv error: Encountered invalid UTF-8 data for line 2"),
    (b"a,b\n1,x\n2,\xc3\n", "Csv error: Encountered invalid UTF-8 data for line 3"),
    (b"a,b\n1,x\n" * 1 + b"1,x\n" * 1000 + b"\xff,x\n", "Parser error: Error while parsing value of line 1003"),
    # one line, several faults: the field count first, then a bad value, then invalid UTF-8
    (b"a,b\n" + b"1,x\n" * 1000 + b"z,\xff,3\n", "Csv error: incorrect number of fields for line 1002"),
    (b"a,b\n" + b"x,1\n" * 1000 + b"\xff,z\n", "Parser error: Error while parsing value of line 1002"),
    # two bad lines: the first in file order is named
    (b"a,b\n" + b"1,x\n" * 1000 + b"1,\xff\n" + b"1,x\n" * 50 + b"z,x\n", "Csv error: Encountered invalid UTF-8 data for line 1002"),
    (b"a,b\n" + b"1,x\n" * 1000 + b"z,x\n" + b"1,x\n" * 50 + b"1\n", "Parser error: Error while parsing value of line 1002"),
])
def test_errors_name_the_first_failing_physical_line(data, msg):
    with pytest.raises(OracleError) as e:
        csv_read(data)
    assert e.value.kind == "Process" and e.value.message == PFX + msg
