"""oracle/buffer_oracle.py's concat_batches (arrow-rs concat_batches with a chosen batch's schema) on the CPU: equal to
pyarrow's own concatenation for same-schema members, and the first-schema, type and nullability rules."""
import numpy as np
import pyarrow as pa
import pytest

from oracle.buffer_oracle import batch_processor, concat_batches, memory_drain, sliding_windows, window_drain
from oracle.sql_oracle import OracleError


def members(seed, sizes):
    rng = np.random.default_rng(seed)
    out = []
    for n in sizes:
        mask = rng.random(n) < 0.3
        out.append(pa.record_batch({
            "i": pa.array(rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64), mask=mask),
            "f": pa.array(rng.random(n).astype(np.float32)),
            "u": pa.array(rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32), mask=~mask),
            "b": pa.array([bool(x) for x in rng.integers(0, 2, n)], pa.bool_()),
            "s": pa.array(["é" * int(k) for k in rng.integers(0, 5, n)], pa.utf8()),
            "n": pa.nulls(n),
        }))
    return out


@pytest.mark.parametrize("sizes", [[1], [0], [3, 0, 9], [7, 8, 9, 17, 1, 2]])
def test_same_schema_equals_concat_tables(sizes):
    bs = members(len(sizes), sizes)
    got = concat_batches(bs[0].schema, bs)
    want = pa.concat_tables([pa.Table.from_batches([b]) for b in bs]).combine_chunks()
    got.validate(full=True)
    assert got.schema == want.schema and got.num_rows == sum(sizes)
    assert pa.Table.from_batches([got]).equals(want)


def test_schema_batch_gives_names_and_nullability():
    a = pa.record_batch([pa.array([1, 2], pa.int64())], schema=pa.schema([pa.field("x", pa.int64(), nullable=False)]))
    b = pa.record_batch([pa.array([3, None], pa.int64())], schema=pa.schema([pa.field("y", pa.int64())]))
    got = concat_batches(b.schema, [a, b])  # positional: a's "x" lands under b's "y"
    assert got.schema.names == ["y"] and got.schema.field(0).nullable and got.column(0).to_pylist() == [1, 2, 3, None]
    with pytest.raises(OracleError) as e:
        concat_batches(a.schema, [a, b])
    assert e.value.kind == "Process"
    assert e.value.message == ("Merge batches failed: Invalid argument error: Column 'x' is declared as non-nullable but "
                               "contains null values")
    # a non-nullable field may take members without NULLs, validity buffer or not
    c = pa.record_batch([pa.array([None, 5], pa.int64()).slice(1)], schema=pa.schema([pa.field("z", pa.int64())]))
    assert c.column(0).buffers()[0] is not None
    assert concat_batches(a.schema, [a, c]).column(0).to_pylist() == [1, 2, 5]


def test_types_must_match_by_position():
    a = pa.record_batch({"x": pa.array([1], pa.int64())})
    for other in (pa.record_batch({"x": pa.array([1], pa.int32())}), pa.record_batch({"x": pa.array(["1"])})):
        with pytest.raises(OracleError) as e:
            concat_batches(a.schema, [a, other])
        assert e.value.kind == "Process" and e.value.message.startswith("Merge batches failed: ")


def test_empty_inputs_and_null_fields():
    s = pa.schema([pa.field("a", pa.int32(), nullable=False), pa.field("n", pa.null())])
    e = concat_batches(s, [])
    assert e.schema == s and e.num_rows == 0
    rb = pa.record_batch([pa.array([1, 2], pa.int32()), pa.nulls(2)], schema=s)
    got = concat_batches(s, [rb, rb.slice(1)])
    assert got.num_rows == 3 and got.column(1).null_count == 3 and got.schema == s
    assert concat_batches(pa.schema([]), [pa.record_batch([pa.nulls(3)], names=["q"])]).num_rows == 3


def test_drains_pick_the_call_sites_schema_batch():
    def one(name, v, nullable=True):
        return pa.record_batch([pa.array([v], pa.int64())], schema=pa.schema([pa.field(name, pa.int64(), nullable=nullable)]))

    old, mid, new = one("old", 1), one("mid", 2), one("new", 3)
    assert memory_drain([old, mid, new]).schema.names == ["old"]
    assert window_drain([("p", old), ("q", mid), ("p", new)]).schema.names == ["new"]  # input p's newest batch
    assert window_drain([("p", old), ("q", mid), ("p", new)]).column(0).to_pylist() == [3, 1, 2]
    assert [b.schema.names for b in sliding_windows([old, mid, new], 2, 1)] == [["old"], ["mid"]]
    assert [b.schema.names for b in batch_processor([old, mid, new, old], 2)] == [["old"], ["new"]]
    with pytest.raises(OracleError):
        memory_drain([one("x", 1, nullable=False), pa.record_batch({"y": pa.array([None], pa.int64())})])
