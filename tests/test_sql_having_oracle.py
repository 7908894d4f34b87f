"""tests/having_oracle.py on the CPU: against pyarrow's Acero where the semantics coincide, against hand-written tables
for alias dereferencing, all-NULL groups and global aggregates, and for every planning error.  Also: the new query
forms construct a `sql` processor without a GPU (the query is parsed there; it is bound on the first batch)."""
import math

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

from arkflow_b200.processor import SqlProcessor
from having_oracle import PLAN, sql_process_having
from oracle.sql_oracle import OracleError


def table(n=3000, seed=3, n_keys=29):
    rng = np.random.default_rng(seed)
    k = rng.integers(0, n_keys, n)
    v = rng.integers(-1000, 1000, n)
    return pa.record_batch({
        "sensor": pa.array([None if x == 4 else f"s{x}" for x in k], pa.utf8()),
        "value": pa.array(v, pa.int64(), mask=rng.random(n) < 0.05),
        "f": pa.array(v.astype(np.float64) * 0.37, pa.float64()),
    })


def by_key(rb, key):
    return {r[key]: r for r in rb.to_pylist()}


def acero(rb, having):
    """GROUP BY sensor with sum / count / count(value) / min / max / avg in Acero, then HAVING as a pc filter."""
    g = pa.Table.from_batches([rb]).group_by("sensor").aggregate(
        [("value", "sum"), ([], "count_all"), ("value", "count"), ("value", "min"), ("value", "max"), ("f", "mean")])
    return g.filter(having(g))


@pytest.mark.parametrize("having,acero_having", [
    ("count(*) > 100", lambda g: pc.greater(g["count_all"], 100)),
    ("sum(value) > 0 AND count(value) < 104", lambda g: pc.and_kleene(pc.greater(g["value_sum"], 0), pc.less(g["value_count"], 104))),
    ("min(value) > -999 OR max(value) < 998", lambda g: pc.or_kleene(pc.greater(g["value_min"], -999), pc.less(g["value_max"], 998))),
    ("sensor IS NULL OR sensor > 's2'", lambda g: pc.or_kleene(pc.is_null(g["sensor"]), pc.greater(g["sensor"], "s2"))),
])
def test_against_acero(having, acero_having):
    rb = table()
    q = ("SELECT sensor, sum(value), count(*), count(value), min(value), max(value), avg(f), max(value) - min(value) AS spread "
         f"FROM flow GROUP BY sensor HAVING {having}")
    got = sql_process_having(rb, q)
    want = acero(rb, acero_having)
    assert 0 < got.num_rows < 30
    g, w = by_key(got, "sensor"), {r["sensor"]: r for r in want.to_pylist()}
    assert g.keys() == w.keys()
    for k, r in g.items():
        a = w[k]
        assert (r["sum(flow.value)"], r["count(*)"], r["count(flow.value)"], r["min(flow.value)"], r["max(flow.value)"]) == \
               (a["value_sum"], a["count_all"], a["value_count"], a["value_min"], a["value_max"])
        assert r["spread"] == a["value_max"] - a["value_min"]
        n = a["count_all"]
        assert math.isclose(r["avg(flow.f)"], a["f_mean"], rel_tol=0, abs_tol=2 * n * 2 ** -53 * 370 * n)


def test_schema_names_and_nullability():
    got = sql_process_having(table(), "SELECT sensor, count(*) AS c, sum(value) / count(*), count(*) > 5 AS hot, avg(value) * 2, "
                                      "CAST(count(*) AS STRING) FROM flow GROUP BY sensor HAVING c > 0")
    assert [(f.name, str(f.type), f.nullable) for f in got.schema] == [
        ("sensor", "string", True), ("c", "int64", False), ("sum(flow.value) / count(*)", "int64", True),
        ("hot", "bool", False), ("avg(flow.value) * Int64(2)", "double", True), ("count(*)", "string", False)]


def test_alias_dereferencing():
    rb = pa.record_batch({"sensor": ["a", "a", "b", "c", "c", "c"], "value": [1, 2, 3, 4, 5, 6]})
    got = sql_process_having(rb, "SELECT sensor, count(*) AS value FROM flow GROUP BY sensor HAVING value >= 2")
    assert sorted(got.to_pylist(), key=str) == [{"sensor": "a", "value": 2}, {"sensor": "c", "value": 3}]
    got = sql_process_having(rb, "SELECT sensor, max(value) - min(value) AS spread FROM flow GROUP BY sensor HAVING spread > 1")
    assert got.to_pylist() == [{"sensor": "c", "spread": 2}]


def test_all_null_groups():
    rb = pa.record_batch({"sensor": ["a", "a", "b", None], "value": pa.array([None, None, 1, None], pa.int64())})
    got = sql_process_having(rb, "SELECT sensor, sum(value) FROM flow GROUP BY sensor HAVING sum(value) IS NULL")
    assert sorted(got.to_pylist(), key=lambda r: str(r["sensor"])) == [{"sensor": None, "sum(flow.value)": None},
                                                                      {"sensor": "a", "sum(flow.value)": None}]
    got = sql_process_having(rb, "SELECT sensor FROM flow GROUP BY sensor HAVING sum(value) > 0 OR NOT (max(value) < 5)")
    assert got.to_pylist() == [{"sensor": "b"}]  # NULL drops the group


def test_global_aggregates():
    rb = pa.record_batch({"value": pa.array([1, 2, 3], pa.int64())})
    assert sql_process_having(rb, "SELECT count(*), sum(value) FROM flow HAVING sum(value) = 6").num_rows == 1
    assert sql_process_having(rb, "SELECT count(*), sum(value) FROM flow HAVING sum(value) = 7").num_rows == 0
    empty = "SELECT count(*), sum(value) FROM flow WHERE value > 9"  # the aggregate over no row: one group
    assert sql_process_having(rb, empty + " HAVING count(*) = 0").to_pylist() == [{"count(*)": 0, "sum(flow.value)": None}]
    assert sql_process_having(rb, empty + " HAVING sum(value) IS NOT NULL").num_rows == 0
    assert sql_process_having(rb.slice(0, 0), "SELECT count(*) FROM flow HAVING count(*) = 0") is None  # ProcessResult::None


def test_limit():
    rb = table()
    full = sql_process_having(rb, "SELECT sensor, count(*) FROM flow GROUP BY sensor HAVING count(*) > 100")
    for n in (0, 3, 1000):
        got = sql_process_having(rb, f"SELECT sensor, count(*) FROM flow GROUP BY sensor HAVING count(*) > 100 LIMIT {n}")
        assert got.schema == full.schema and got.num_rows == min(n, full.num_rows)


@pytest.mark.parametrize("query,message", [
    ("SELECT value FROM flow HAVING value > 1",
     "HAVING clause references: flow.value > Int64(1) must appear in the GROUP BY clause or be used in an aggregate function"),
    ("SELECT sensor, value + 1 FROM flow GROUP BY sensor",
     'Column in SELECT must be in GROUP BY or an aggregate function: While expanding wildcard, column "value" must appear in the '
     "GROUP BY clause or must be part of an aggregate function"),
    ("SELECT sensor FROM flow GROUP BY sensor HAVING value > 1",
     'Column in HAVING must be in GROUP BY or an aggregate function: While expanding wildcard, column "value" must appear in the '
     "GROUP BY clause or must be part of an aggregate function"),
    ("SELECT sum(count(*)) + 1 FROM flow", "nested aggregates are not allowed"),
    ("SELECT sensor FROM flow GROUP BY sensor HAVING max(sum(value)) > 1", "nested aggregates are not allowed"),
])
def test_planning_errors(query, message):
    with pytest.raises(OracleError) as e:
        sql_process_having(table(), query)
    assert e.value.kind == "Process" and e.value.message == PLAN + message


@pytest.mark.parametrize("q", [
    "SELECT sensor, max(value) - min(value) AS spread FROM flow GROUP BY sensor HAVING count(*) > 100",
    "SELECT sensor, count(*) AS c FROM flow GROUP BY sensor HAVING c > 5 LIMIT 10",
    "SELECT count(*) FROM flow HAVING count(*) > 0",
    "SELECT sensor, count(*) FROM flow GROUP BY sensor LIMIT 0",
    "SELECT concat(sensor, ':', count(*)), count(*) > 5 AS hot FROM flow GROUP BY sensor",
])
def test_new_forms_construct_without_a_gpu(lib, q):
    SqlProcessor({"query": q})


def test_having_on_a_join_is_unsupported():
    with pytest.raises(OracleError) as e:
        sql_process_having(table(), "SELECT * FROM a JOIN b ON a.k = b.k HAVING count(*) > 1")
    assert e.value.kind == "Unsupported"
