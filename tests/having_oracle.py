"""HAVING, expressions over aggregates and LIMIT in aggregate queries, restated over oracle/sql_oracle.py.

DataFusion 47 plans these queries as Aggregate → Filter → Projection → Limit.  This oracle does the same:
- the aggregate is a *frame*: every GROUP BY key, then every distinct aggregate call of SELECT and HAVING, computed by
  `sql_process` itself (keys from each group's first row, aggregates as the oracle computes them everywhere else);
- HAVING and the SELECT items are rewritten so that each key and each aggregate call reads a frame column, and are
  evaluated over the frame by the oracle's own expression evaluator, as a WHERE and a projection: a group whose HAVING
  is NULL is dropped (Kleene logic), arithmetic, coercions, errors and nullability are those of a projection;
- LIMIT n keeps n groups of the result after HAVING.
json_* calls are evaluated first by tests/json_path_oracle.py's helpers, as the library does.

Assumptions, none pinned by the reference's tests:
- SELECT aliases are dereferenced in HAVING (datafusion-sql's `resolve_aliases_to_exprs`): an unqualified column named
  as a SELECT alias stands for that item's expression, also where an input column has the same name.
- Without ORDER BY, which n groups LIMIT returns is unspecified.  This oracle returns the first n of its own group
  order, so a LIMIT result is to be compared as n distinct groups, each equal to the unlimited result's row for its key.
- The planning errors are ARK_ERR_PROCESS with these texts after "Execution query error: Error during planning: ":
  `HAVING clause references: <expr> must appear in the GROUP BY clause or be used in an aggregate function` (HAVING in
  a query with neither GROUP BY nor an aggregate; <expr> as DataFusion displays it), `Column in SELECT|HAVING must be in
  GROUP BY or an aggregate function: While expanding wildcard, column "<name>" must appear in the GROUP BY clause or must
  be part of an aggregate function`, and `nested aggregates are not allowed`.
"""
from __future__ import annotations

import copy
from typing import Optional

import numpy as np
import pyarrow as pa

import json_path_oracle as J
import oracle.sql_oracle as S
from oracle.sql_oracle import E, OracleError, Query, SelectItem

PLAN = "Execution query error: Error during planning: "


def parse(query: str) -> tuple[Query, Optional[E]]:
    """sql_oracle's parse with the HAVING clause taken out of the token stream: (query, having)."""
    if len(S._tokenize(query)) == 1:
        return S.parse(query), None  # the parser's own error
    ps = S._Parser(query)
    having = None
    for i, t in enumerate(ps.t):
        if t.kind == "id" and t.text.upper() == "HAVING":
            ps.p = i + 1
            having = ps.expr()
            ps.t = ps.t[:i] + ps.t[ps.p:]
            ps.p = 0
            break
    return ps.parse(), having


def _plain(e: E) -> bool:
    """The aggregate SELECT items sql_process evaluates itself: keys, aggregates, CAST(<aggregate> AS STRING), literals."""
    if e.kind == "cast" and e.to == "Utf8" and e.args[0].kind == "func" and e.args[0].name in S._AGG:
        return True
    return (e.kind == "func" and e.name in S._AGG) or e.kind in ("col", "lit")


def _with_query(rb: pa.RecordBatch, q: Query, table_name: str) -> Optional[pa.RecordBatch]:
    saved = S.parse
    S.parse = lambda _text: q
    try:
        return S.sql_process(rb, "<frame>", table_name)
    finally:
        S.parse = saved


def sql_process_having(rb: pa.RecordBatch, query: str, table_name: str = "flow") -> Optional[pa.RecordBatch]:
    """The sql processor's result for any query of the subset; None ⇔ ProcessResult::None (an empty batch)."""
    q, having = parse(query)
    has_agg = bool(q.group_by) or any(not it.star and S._has_agg(it.expr) for it in q.select) or S._has_agg(having)
    if having is None and (not has_agg or (q.limit < 0 and all(it.star or _plain(it.expr) for it in q.select))):
        return J.sql_process_json(rb, query, table_name)
    if q.joins:
        raise OracleError("Unsupported", "HAVING on a join query" if having is not None else "LIMIT on a join query")
    if rb.num_rows == 0:
        return None
    if q.table != table_name:
        raise OracleError("Process", f"Execution query error: Error during planning: table '{q.table}' not found")
    vis = q.alias or q.table
    if S._has_agg(q.where):
        raise OracleError("Process", PLAN + "Aggregate functions are not allowed in the WHERE clause")
    if having is not None and not has_agg:
        raise OracleError("Process", PLAN + f"HAVING clause references: {S.display(having, vis)} must appear in the GROUP BY "
                                            "clause or be used in an aggregate function")

    # json_* calls → hidden input columns (json_path_oracle.sql_process_json)
    types = {f.name: J._arrow_kind(f.type) for f in rb.schema}
    calls: dict[str, tuple] = {}

    def json_rw(e: Optional[E]) -> Optional[E]:
        if e is None:
            return None
        if e.kind == "func" and e.name in J.JSON_FUNCS:
            doc, cast, path = J._bind_call(e, types)
            name = S.display(e, vis)
            if name not in calls:
                calls[name] = (f"__json{len(calls)}", e.name, doc, cast, path)
            return E("col", name=calls[name][0])
        e.args = [json_rw(a) for a in e.args]
        return e

    for it in q.select:
        it.expr = json_rw(it.expr)
    q.where = json_rw(q.where)
    q.group_by = [json_rw(g) for g in q.group_by]
    having = json_rw(having)
    wide = rb
    if calls:
        cols, names = list(rb.columns), list(rb.schema.names)
        for hidden, fn, doc, cast, path in calls.values():
            cols.append(J.json_column(rb, fn, doc, path, cast))
            names.append(hidden)
        wide = pa.record_batch(cols, names=names)
    ctx_in = S._Ctx(vis, wide)

    # the frame: keys, then every distinct aggregate call
    for it in q.select:
        if it.star:
            raise OracleError("Process", "Execution query error: Error during planning: SELECT * with GROUP BY")
    key_disp = [S.display(g, vis) for g in q.group_by]
    frame_items = [SelectItem(g, alias=f"__k{i}") for i, g in enumerate(q.group_by)]
    aggs: dict[str, str] = {}

    def rw(e: E, clause: str, aliases: bool) -> E:
        if e.kind == "func" and e.name in S._AGG:
            if any(S._has_agg(a) for a in e.args):
                raise OracleError("Process", PLAN + "nested aggregates are not allowed")
            d = S.display(e, vis)
            if d not in aggs:
                aggs[d] = f"__a{len(aggs)}"
                frame_items.append(SelectItem(e, alias=aggs[d]))
            return E("col", name=aggs[d])
        if e.kind == "col":
            if aliases and not e.qual:
                for it in q.select:
                    if it.alias and it.alias == e.name:
                        return rw(copy.deepcopy(it.expr), clause, False)
            d = S.display(e, vis)
            if d in key_disp:
                return E("col", name=f"__k{key_disp.index(d)}")
            ctx_in.resolve(e)
            raise OracleError("Process", PLAN + f"Column in {clause} must be in GROUP BY or an aggregate function: While expanding "
                                                f"wildcard, column \"{e.name}\" must appear in the GROUP BY clause or must be part of "
                                                "an aggregate function")
        e = copy.copy(e)
        e.args = [rw(a, clause, aliases) for a in e.args]
        return e

    items = [(it, rw(it.expr, "SELECT", False)) for it in q.select]
    having_rw = rw(having, "HAVING", True) if having is not None else None
    frame = _with_query(wide, Query(frame_items, q.table, q.alias, [], q.where, q.group_by, -1), table_name)

    # the stage: HAVING as a WHERE, the items as a projection, then LIMIT
    ctx = S._Ctx(vis, frame)
    sel = None
    if having_rw is not None:
        t = ctx.type_of(having_rw)
        if t not in ("Boolean", "Null"):
            raise OracleError("Process", PLAN + "Cannot create filter with non-boolean predicate")
        m = ctx.eval(having_rw)
        sel = np.nonzero(m.values.astype(bool) & m.valid)[0]
    cols, fields = [], []
    for it, e in items:
        v = ctx.eval(e, sel)
        if v.dtype == "Null":
            raise OracleError("Unsupported", "NULL-typed projection")
        name = it.alias or (it.expr.name if it.expr.kind == "col" else S.display(it.expr, vis))
        for call, (hidden, *_rest) in calls.items():
            name = call if name == hidden else name.replace(f"{vis}.{hidden}", call)
        arr = S._vec_to_arrow(v)
        cols.append(arr)
        fields.append(pa.field(name, arr.type, ctx.nullable_of(e)))
    out = pa.RecordBatch.from_arrays(cols, schema=pa.schema(fields))
    return out.slice(0, q.limit) if q.limit >= 0 else out
