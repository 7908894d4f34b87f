"""The Boolean and validity bitmaps of every producer that packs one from a byte per row, and the null count it exports
with them (csrc/bitmap.cu).

Each producer runs at row counts that cover the byte tail and the 2048-row block edge of pack_bits_kernel.  Its device
result is read as the library exported it, without going through pyarrow: the raw null_count, whether buffers[0] is
present, and the bytes of the validity and Boolean bitmaps.  The policy each producer keeps:
  * exact: the file inputs (CSV, NDJSON, Avro) and the decoders (json_to_arrow, protobuf_to_arrow) export the exact
    null count, and a validity bitmap only when it is > 0;
  * unknown: query outputs (SQL projection, join gathers, GROUP BY keys and aggregates) export null_count -1 with a
    bitmap whenever the output has rows and can hold NULLs (a nullable input or an outer-join miss), else 0 and none.
Validity bitmaps must equal the expected validity bit for bit, zero padding in the last byte included; Boolean value
bits must equal the expected values in every non-NULL row and be zero past the last row.
"""
import json
from collections import namedtuple

import numpy as np
import pyarrow as pa
import pytest

from arkflow_b200 import arrow_ffi as F
from arkflow_b200.arrow_ffi import DeviceBatch
from arkflow_b200.input import FileInput
from arkflow_b200.processor import ArkError, JsonToArrowProcessor, ProtobufToArrowProcessor, SqlProcessor
from oracle import protobuf_oracle as O
from oracle.avro_oracle import block_bytes, header, record_schema

pytestmark = pytest.mark.gpu

NS = [0, 1, 7, 8, 9, 2047, 2048, 2049, 1_000_003]

Raw = namedtuple("Raw", "name length offset null_count validity values children")


def _dev_bytes(ptr, nbytes):
    import torch

    if nbytes == 0:
        return b""
    return torch.as_tensor(F._CudaPtr(ptr, nbytes, "|u1", 1, None), device="cuda").cpu().numpy().tobytes()


def _raw(a, s):
    n, nb = a.length, (a.length + 7) // 8
    kids = [_raw(a.children[i].contents, s.children[i].contents) for i in range(a.n_children)]
    return Raw(s.name.decode(), n, a.offset, a.null_count,
               _dev_bytes(a.buffers[0], nb) if a.n_buffers > 0 and a.buffers[0] else None,
               _dev_bytes(a.buffers[1], nb) if s.format == b"b" else None,
               {k.name: k for k in kids})


def columns(db):
    """name → Raw of every top-level column of a device result (nothing when the call produced no batch)."""
    if db is None:
        return {}
    a, s = db._owner.dev.array, db._owner.sch
    return {c.name: c for c in (_raw(a.children[i].contents, s.children[i].contents) for i in range(a.n_children))}


def check(col, valid, values=None, exact=True, bitmap=False, what=""):
    """`valid` / `values`: the expected validity and Boolean values (numpy bool) in the column's row order.  exact: the
    exported null_count is the number of NULLs and a bitmap is present only when there are any.  Otherwise (unknown)
    the bitmap is present with null_count -1 when `bitmap` and the column has rows, and absent with 0 when not."""
    n = len(valid)
    nulls = int(n - valid.sum())
    assert (col.length, col.offset) == (n, 0), what
    if exact:
        has = nulls > 0
        assert col.null_count == nulls, (what, col.null_count, nulls)
    else:
        has = bitmap and n > 0
        assert col.null_count == (-1 if has else 0), (what, col.null_count)
    assert (col.validity is not None) == has, what
    if has:
        assert col.validity == np.packbits(valid, bitorder="little").tobytes(), what
    else:
        assert nulls == 0, what
    if values is not None:
        assert len(col.values) == (n + 7) // 8, what
        bits = np.unpackbits(np.frombuffer(col.values, np.uint8), bitorder="little").astype(bool)
        assert np.array_equal(bits[:n] & valid, values & valid), (what, np.flatnonzero((bits[:n] ^ values) & valid)[:5])
        assert not bits[n:].any(), what


def read_file(path, kind):
    """Every batch of a `file` input, left in HBM."""
    inp = FileInput({"input_type": {"type": kind, "path": str(path)}})
    inp.connect()
    out = []
    try:
        while True:
            out.append(inp.read_device())
    except ArkError as e:
        assert e.kind == "EOF", e.message
    return out


def one_batch(batches, n):
    """The single batch a file of n ≤ 4 Mi records is read as (none when n == 0)."""
    assert len(batches) == (1 if n else 0)
    return columns(batches[0]) if batches else None


def binary(payloads):
    return pa.record_batch([pa.array(payloads, pa.binary())], names=["__value__"])


def table(n):
    """i Int64; b Boolean; x Int64 with a NULL in row 0 and every 4th row after it, so every non-empty batch has NULLs."""
    i = np.arange(n, dtype=np.int64)
    x = pa.array(i * 7 - 20, mask=(i % 4 == 0))
    return pa.record_batch({"i": pa.array(i), "b": pa.array(i % 3 == 0), "x": x}), i


# ---- producers -------------------------------------------------------------------------------------------------------
def csv_input(n, tmp_path):
    i = np.arange(n)
    b_valid, b_val, x_valid = i % 5 != 1, i % 3 == 0, i % 4 != 1
    lines = ["%d,%s,%s" % (k, ("true" if b_val[k] else "false") if b_valid[k] else "", k * 3 if x_valid[k] else "")
             for k in range(n)]
    p = tmp_path / "t.csv"
    p.write_text("i,b,x\n" + "".join(s + "\n" for s in lines))
    cols = one_batch(read_file(p, "csv"), n)
    if cols is None:
        return
    check(cols["i"], np.ones(n, bool), what="i")
    check(cols["b"], b_valid, b_val, what="b")
    check(cols["x"], x_valid, what="x")


def ndjson_input(n, tmp_path):
    i = np.arange(n)
    b_valid, b_val, x_valid = i % 5 != 1, i % 3 == 0, i % 4 != 1
    p = tmp_path / "t.json"
    p.write_text("".join(json.dumps({"b": bool(b_val[k]) if b_valid[k] else None, "x": int(k) if x_valid[k] else None}) + "\n"
                         for k in range(n)))
    cols = one_batch(read_file(p, "json"), n)
    if cols is None:
        return
    check(cols["b"], b_valid, b_val, what="b")
    check(cols["x"], x_valid, what="x")


def json_to_arrow(n, tmp_path):
    """A Bool scalar, a nullable Int64 scalar, a List<Int64> and a Struct {a: Int64}; row 0 holds every field, so the
    schema taken from it has every type."""
    i = np.arange(n)
    b_valid, b_val, x_valid, l_valid, s_valid = i % 5 != 1, i % 3 == 0, i % 4 != 1, i % 6 != 2, i % 7 != 3
    recs = [json.dumps({"b": bool(b_val[k]) if b_valid[k] else None, "x": int(k) if x_valid[k] else None,
                        "l": list(range(k, k + k % 3 + 1)) if l_valid[k] else None,
                        "s": {"a": int(k)} if s_valid[k] else None}).encode() for k in range(n)]
    out = JsonToArrowProcessor({}).process_device(DeviceBatch.from_arrow(binary(recs)))
    cols = columns(out)
    if n == 0:
        assert cols == {}
        return
    check(cols["b"], b_valid, b_val, what="b")
    check(cols["x"], x_valid, what="x")
    check(cols["l"], l_valid, what="l")
    check(cols["l"].children["item"], np.ones(int(((i % 3 + 1) * l_valid).sum()), bool), what="l.item")
    check(cols["s"], s_valid, what="s")
    check(cols["s"].children["a"], s_valid, what="s.a")


def avro_input(n, tmp_path):
    """A boolean and a ["null", "boolean"] field."""
    i = np.arange(n)
    b_val, nb_valid, nb_val = i % 3 == 0, i % 5 != 1, i % 2 == 0
    recs = [bytes([int(b_val[k])]) + (bytes([2, int(nb_val[k])]) if nb_valid[k] else b"\x00") for k in range(n)]
    data = header(record_schema([("b", "boolean"), ("nb", ["null", "boolean"])]))
    if n:
        data += block_bytes(n, b"".join(recs))
    p = tmp_path / "t.avro"
    p.write_bytes(data)
    cols = one_batch(read_file(p, "avro"), n)
    if cols is None:
        return
    check(cols["b"], np.ones(n, bool), b_val, what="b")
    check(cols["nb"], nb_valid, nb_val, what="nb")


def protobuf_to_arrow(n, tmp_path):
    """A proto3 bool field (never NULL: an absent field is false)."""
    d = tmp_path / "pb"
    d.mkdir()
    (d / "m.proto").write_text(O.proto_text("t", "M", [O.PbField("b", 1, "bool")]))
    val = np.arange(n) % 3 == 0
    out = ProtobufToArrowProcessor({"proto_inputs": [str(d)], "message_type": "t.M"}).process_device(
        DeviceBatch.from_arrow(binary([b"\x08\x01" if v else b"" for v in val])))
    cols = columns(out)
    if n == 0 and not cols:
        return
    check(cols["b"], np.ones(n, bool), val, what="b")


def sql_projection(n, tmp_path):
    """A Boolean column, a nullable column and a computed Boolean through the filter kernel (every row passes)."""
    rb, i = table(n)
    out = SqlProcessor({"query": "SELECT b, x, x > 5 AS c FROM flow WHERE i >= 0"}).process_device(DeviceBatch.from_arrow(rb))
    cols = columns(out)
    if n == 0:
        assert cols == {}
        return
    x_valid = i % 4 != 0
    check(cols["b"], np.ones(n, bool), i % 3 == 0, exact=False, bitmap=False, what="b")
    check(cols["x"], x_valid, exact=False, bitmap=True, what="x")
    check(cols["c"], x_valid, i * 7 - 20 > 5, exact=False, bitmap=True, what="c")


def group_by(n, tmp_path):
    """A Boolean key; a nullable Int64 key g (n groups: NULL in row 0 only) with SUM(x), NULL for the groups whose x is
    NULL."""
    rb, i = table(n)
    rb = pa.record_batch({"b": rb.column("b"), "g": pa.array(i, mask=(i == 0)), "x": rb.column("x")})
    dev = SqlProcessor({"query": "SELECT b, COUNT(*) AS c FROM flow GROUP BY b"}).process_device(DeviceBatch.from_arrow(rb))
    cols = columns(dev)
    if n == 0:
        assert cols == {}
        return
    got = dev.to_arrow()
    keys = np.array(got.column("b").to_pylist(), bool)
    want = {True: int((i % 3 == 0).sum()), False: int((i % 3 != 0).sum())}
    assert dict(zip(keys.tolist(), got.column("c").to_pylist())) == {k: v for k, v in want.items() if v}
    check(cols["b"], np.ones(len(keys), bool), keys, exact=False, bitmap=False, what="b key")

    dev = SqlProcessor({"query": "SELECT g, SUM(x) AS s FROM flow GROUP BY g"}).process_device(DeviceBatch.from_arrow(rb))
    cols, got = columns(dev), dev.to_arrow()
    g = got.column("g").to_pylist()
    assert sorted(g, key=lambda v: -1 if v is None else v) == [None] + list(range(1, n))
    g_valid = np.array([v is not None for v in g])
    row = np.array([0 if v is None else v for v in g])  # the group's only row
    check(cols["g"], g_valid, exact=False, bitmap=True, what="g key")
    check(cols["s"], row % 4 != 0, exact=False, bitmap=True, what="SUM(x)")


def join(n, tmp_path):
    """a JOIN c and a LEFT JOIN c on k, gathering a's Boolean b and nullable x and c's Boolean cb and Int64 cy.  For the
    inner join c holds every key; for the outer one every third key of a finds no row in c."""
    a, i = table(n)
    a = pa.record_batch({"id": a.column("i"), "k": a.column("i"), "b": a.column("b"), "x": a.column("x")})
    for jt, keep in (("", np.ones(n, bool)), ("LEFT ", i % 3 != 2)):
        k = i[keep]
        c = pa.record_batch({"k": pa.array(k), "cb": pa.array(k % 2 == 0), "cy": pa.array(k * 5)})
        q = f"SELECT a.id, a.b, a.x, c.cb, c.cy FROM a {jt}JOIN c ON a.k = c.k"
        dev = SqlProcessor({"query": q}).process_tables_device({"a": DeviceBatch.from_arrow(a), "c": DeviceBatch.from_arrow(c)})
        cols = columns(dev)
        if n == 0:
            assert all(col.length == 0 for col in cols.values())
            continue
        ids = np.array(dev.to_arrow().column("id").to_pylist(), np.int64)
        assert np.array_equal(np.sort(ids), i)
        miss = bool(jt)  # an outer join's other side gets a bitmap whether or not a row finds no match
        check(cols["b"], np.ones(n, bool), ids % 3 == 0, exact=False, bitmap=False, what=(jt, "b"))
        check(cols["x"], ids % 4 != 0, exact=False, bitmap=True, what=(jt, "x"))
        check(cols["cb"], keep[ids], ids % 2 == 0, exact=False, bitmap=miss, what=(jt, "cb"))
        check(cols["cy"], keep[ids], exact=False, bitmap=miss, what=(jt, "cy"))


PRODUCERS = {f.__name__: f for f in (csv_input, ndjson_input, json_to_arrow, avro_input, protobuf_to_arrow, sql_projection,
                                     group_by, join)}


@pytest.mark.parametrize("n", NS)
@pytest.mark.parametrize("producer", list(PRODUCERS))
def test_bitmaps_and_null_counts(gpu, tmp_path, producer, n):
    PRODUCERS[producer](n, tmp_path)
