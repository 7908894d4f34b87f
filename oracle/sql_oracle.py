"""CPU oracle for the `sql` processor — TEST INFRASTRUCTURE, not product code.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this package.  The product path (arkflow_b200/) never does.

What it restates
    SqlProcessor::process / execute_query     crates/arkflow-plugin/src/processor/sql.rs:108-149, 209-220
    execute_query_with_statement              crates/arkflow-plugin/src/processor/sql.rs:188-204
and, because the arithmetic behind those 250 lines lives in third-party crates that are NOT under
the reference's tree (datafusion 47.0.0, arrow 55.2.0, sqlparser 0.55.0 — pinned in Cargo.lock, not
vendored; no Rust toolchain in this image), the published semantics of those crates for the SQL
subset the BASELINE configs exercise:
    * identifiers are lower-cased unless quoted; result columns are named as DataFusion's
      schema_name() does (value, sum(flow.value), count(*), flow.value + Int64(1), alias);
    * Int64 + - * wrap; Int64 / and % by zero raise; Int64 ∘ Float64 coerces to Float64;
    * Float64 comparisons follow IEEE-754 totalOrder (arrow-ord: NaN > +inf, -0.0 < +0.0, = is bitwise);
    * AND / OR are Kleene; WHERE keeps rows whose predicate is TRUE (NULL drops the row);
    * SUM(Int64) → Int64 wrapping, SUM(Float64) → Float64, COUNT → Int64 non-null,
      AVG → Float64 = f64 sum / count, MIN/MAX keep the type; aggregates skip NULLs; a NULL group
      key forms its own group;
    * inner equi-join: NULL keys never match; `SELECT *` = left columns then right columns;
    * empty input batch → ProcessResult::None (sql.rs:211-213); an all-filtered batch → 0-row batch.
GROUP BY / JOIN output order is unspecified in DataFusion: compare as multisets.

PARITY STATUS: "parity unpinned" for SUM/AVG values, GROUP BY contents and join contents — the
reference's own tests pin only shapes, COUNT(*) = 5 (core/lib.rs:1857) and one filter cardinality
(core/lib.rs:2183-2196); those pins are checked in tests/test_oracle_golden.py.  The mechanics
(filter/take/hash) run on pyarrow 24 / numpy; every rule where Arrow C++ differs from arrow-rs
(float totalOrder, naming, empty-result shapes) is encoded explicitly below.
"""
from __future__ import annotations

import math
import re
from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc


class OracleError(Exception):
    """kind mirrors arkflow_core::Error variants: 'Process' | 'Config' | 'Unsupported'."""

    def __init__(self, kind: str, message: str):
        super().__init__(message)
        self.kind, self.message = kind, message


# ------------------------------------------------------------------------------------------------
# tokenizer / parser (independent restatement of the same SQL subset the library accepts)
# ------------------------------------------------------------------------------------------------
_TOKEN_RE = re.compile(
    r"""\s*(?:
        (?P<num>(?:\d+\.\d*|\.\d+|\d+)(?:[eE][+-]?\d+)?) |
        (?P<id>[A-Za-z_][A-Za-z_0-9]*) |
        "(?P<qid>(?:[^"]|"")*)" |
        '(?P<str>(?:[^']|'')*)' |
        (?P<op><=|>=|<>|!=|==|[-+*/%=<>(),.;])
    )""",
    re.X,
)

_RESERVED = {"SELECT", "FROM", "WHERE", "GROUP", "BY", "HAVING", "ORDER", "LIMIT", "JOIN", "INNER", "LEFT", "RIGHT",
             "FULL", "CROSS", "ON", "USING", "AND", "OR", "NOT", "AS", "IS", "NULL", "UNION", "CASE", "DISTINCT",
             "TRUE", "FALSE", "BETWEEN", "IN", "LIKE", "OFFSET"}


@dataclass
class Tok:
    kind: str  # num | id | qid | str | op | end
    text: str


def _tokenize(sql: str) -> list[Tok]:
    out, pos = [], 0
    sql = sql.rstrip()
    while pos < len(sql):
        m = _TOKEN_RE.match(sql, pos)
        if not m or m.end() == pos:
            raise OracleError("Process", f"SQL query error: unexpected character at {pos}")
        pos = m.end()
        for k in ("num", "id", "qid", "str", "op"):
            if m.group(k) is not None:
                t = m.group(k)
                if k == "qid":
                    t = t.replace('""', '"')
                if k == "str":
                    t = t.replace("''", "'")
                if k == "op" and t == "<>":
                    t = "!="
                if k == "op" and t == "==":
                    t = "="
                out.append(Tok(k, t))
                break
    out.append(Tok("end", ""))
    return out


@dataclass
class E:
    kind: str  # col | lit | bin | un | func | cast | isnull
    name: str = ""
    qual: str = ""
    value: object = None
    vtype: str = ""  # Int64 | Float64 | Utf8 | Boolean | Null
    op: str = ""
    args: list = field(default_factory=list)
    star: bool = False
    negated: bool = False
    to: str = ""


@dataclass
class SelectItem:
    expr: Optional[E]
    alias: str = ""
    star: bool = False
    star_qual: str = ""


@dataclass
class Query:
    select: list
    table: str
    alias: str
    joins: list  # [(table, alias, on_expr)]
    where: Optional[E]
    group_by: list
    limit: int = -1


class _Parser:
    def __init__(self, sql):
        self.t = _tokenize(sql)
        self.p = 0

    def cur(self):
        return self.t[self.p]

    def kw(self, w):
        c = self.cur()
        return c.kind == "id" and c.text.upper() == w

    def accept_kw(self, w):
        if self.kw(w):
            self.p += 1
            return True
        return False

    def accept_op(self, o):
        c = self.cur()
        if c.kind == "op" and c.text == o:
            self.p += 1
            return True
        return False

    def err(self, what):
        raise OracleError("Process", f"SQL query error: Expected {what}, found: {self.cur().text or 'EOF'}")

    def ident(self, what="identifier"):
        c = self.cur()
        if c.kind == "qid":
            self.p += 1
            return c.text
        if c.kind == "id" and c.text.upper() not in _RESERVED:
            self.p += 1
            return c.text.lower()
        self.err(what)

    def parse(self) -> Query:
        if self.cur().kind == "id" and self.cur().text.upper() in ("INSERT", "UPDATE", "DELETE", "CREATE", "DROP", "ALTER", "SET"):
            raise OracleError("Process", "SQL query error: DDL/DML/statements are not allowed")
        if not self.accept_kw("SELECT"):
            self.err("SELECT")
        if self.kw("DISTINCT"):
            raise OracleError("Unsupported", "SELECT DISTINCT")
        sel = [self.select_item()]
        while self.accept_op(","):
            sel.append(self.select_item())
        if not self.accept_kw("FROM"):
            self.err("FROM")
        table, alias = self.table_ref()
        joins = []
        while True:
            jtype = "inner"
            if not self.accept_kw("INNER"):
                for w in ("LEFT", "RIGHT"):  # LEFT [OUTER] JOIN / RIGHT [OUTER] JOIN
                    if self.accept_kw(w):
                        jtype = w.lower()
                        self.accept_kw("OUTER")
            for w in ("FULL", "CROSS"):
                if self.kw(w):
                    raise OracleError("Unsupported", w + " JOIN")
            if self.accept_kw("JOIN"):
                jt, ja = self.table_ref()
                if not self.accept_kw("ON"):
                    self.err("ON")
                joins.append((jt, ja, self.expr(), jtype))
            elif jtype != "inner":
                self.err("JOIN")
            else:
                break
        where = self.expr() if self.accept_kw("WHERE") else None
        group_by = []
        if self.accept_kw("GROUP"):
            if not self.accept_kw("BY"):
                self.err("BY")
            group_by.append(self.expr())
            while self.accept_op(","):
                group_by.append(self.expr())
        if self.kw("HAVING"):
            raise OracleError("Unsupported", "HAVING")
        order_by = []
        if self.accept_kw("ORDER"):
            if not self.accept_kw("BY"):
                self.err("BY")
            while True:
                order_by.append(self.expr())
                if not self.accept_kw("ASC"):
                    self.accept_kw("DESC")
                if self.accept_kw("NULLS") and not (self.accept_kw("FIRST") or self.accept_kw("LAST")):
                    self.err("FIRST or LAST")
                if not self.accept_op(","):
                    break
        for w in ("UNION", "OFFSET"):
            if self.kw(w):
                raise OracleError("Unsupported", w)
        limit = -1
        if self.accept_kw("LIMIT"):
            if self.cur().kind != "num":
                self.err("a number")
            limit = int(self.cur().text)
            self.p += 1
        while self.accept_op(";"):
            pass
        if self.cur().kind != "end":
            self.err("end of statement")
        if order_by and (group_by or not any((not it.star) and _has_agg(it.expr) for it in sel)):
            # ORDER BY survives only where it cannot change the result: an aggregate query without GROUP BY has one row
            raise OracleError("Unsupported", "ORDER BY")
        return Query(sel, table, alias, joins, where, group_by, limit)

    def table_ref(self):
        name = self.ident("table name")
        while self.accept_op("."):
            name = self.ident("table name")
        alias = ""
        if self.accept_kw("AS"):
            alias = self.ident("alias")
        elif self.cur().kind == "qid" or (self.cur().kind == "id" and self.cur().text.upper() not in _RESERVED):
            alias = self.ident("alias")
        return name, alias

    def select_item(self):
        if self.accept_op("*"):
            return SelectItem(None, star=True)
        c = self.cur()
        if c.kind in ("id", "qid") and self.t[self.p + 1].text == "." and self.t[self.p + 2].text == "*":
            q = c.text if c.kind == "qid" else c.text.lower()
            self.p += 3
            return SelectItem(None, star=True, star_qual=q)
        e = self.expr()
        alias = ""
        if self.accept_kw("AS"):
            alias = self.ident("alias")
        elif self.cur().kind == "qid" or (self.cur().kind == "id" and self.cur().text.upper() not in _RESERVED):
            alias = self.ident("alias")
        return SelectItem(e, alias)

    def expr(self):
        return self.or_()

    def or_(self):
        l = self.and_()
        while self.accept_kw("OR"):
            l = E("bin", op="OR", args=[l, self.and_()])
        return l

    def and_(self):
        l = self.not_()
        while self.accept_kw("AND"):
            l = E("bin", op="AND", args=[l, self.not_()])
        return l

    def not_(self):
        if self.accept_kw("NOT"):
            return E("un", op="NOT", args=[self.not_()])
        return self.cmp()

    def cmp(self):
        l = self.add()
        while True:
            c = self.cur()
            if c.kind == "op" and c.text in ("=", "!=", "<", "<=", ">", ">="):
                self.p += 1
                l = E("bin", op=c.text, args=[l, self.add()])
            elif self.kw("IS"):
                self.p += 1
                neg = self.accept_kw("NOT")
                if not self.accept_kw("NULL"):
                    raise OracleError("Unsupported", "IS TRUE/FALSE")
                l = E("isnull", args=[l], negated=neg)
            elif self.kw("BETWEEN") or self.kw("IN") or self.kw("LIKE"):
                raise OracleError("Unsupported", self.cur().text.upper())
            else:
                return l

    def add(self):
        l = self.mul()
        while self.cur().kind == "op" and self.cur().text in "+-" and self.cur().text:
            op = self.cur().text
            self.p += 1
            l = E("bin", op=op, args=[l, self.mul()])
        return l

    def mul(self):
        l = self.unary()
        while self.cur().kind == "op" and self.cur().text in ("*", "/", "%"):
            op = self.cur().text
            self.p += 1
            l = E("bin", op=op, args=[l, self.unary()])
        return l

    def unary(self):
        if self.accept_op("-"):
            inner = self.unary()
            if inner.kind == "lit" and inner.vtype == "Int64":
                v = -inner.value
                if v < -(2 ** 63):
                    v += 2 ** 64
                inner.value = v
                return inner
            if inner.kind == "lit" and inner.vtype == "Float64":
                inner.value = -inner.value
                return inner
            return E("un", op="NEG", args=[inner])
        if self.accept_op("+"):
            return self.unary()
        return self.primary()

    def type_name(self):
        c = self.cur()
        if c.kind != "id":
            self.err("a data type")
        self.p += 1
        u = c.text.upper()
        if u == "DOUBLE":
            self.accept_kw("PRECISION")
            return "Float64"
        if u in ("FLOAT8",):
            return "Float64"
        if u in ("BIGINT", "INT8"):
            return "Int64"
        if u in ("BOOLEAN", "BOOL"):
            return "Boolean"
        if u in ("STRING", "TEXT", "VARCHAR", "CHAR"):
            return "Utf8"
        if u in ("BYTEA", "BINARY", "VARBINARY"):
            return "Binary"
        raise OracleError("Unsupported", "CAST to " + u)

    def primary(self):
        c = self.cur()
        if self.accept_op("("):
            e = self.expr()
            if not self.accept_op(")"):
                self.err(")")
            return e
        if c.kind == "num":
            self.p += 1
            if re.search(r"[.eE]", c.text) or int(c.text) > 2 ** 63 - 1:
                return E("lit", value=float(c.text), vtype="Float64")
            return E("lit", value=int(c.text), vtype="Int64")
        if c.kind == "str":
            self.p += 1
            return E("lit", value=c.text, vtype="Utf8")
        if c.kind == "id":
            u = c.text.upper()
            if u == "NULL":
                self.p += 1
                return E("lit", value=None, vtype="Null")
            if u in ("TRUE", "FALSE"):
                self.p += 1
                return E("lit", value=(u == "TRUE"), vtype="Boolean")
            if u == "CASE":
                raise OracleError("Unsupported", "CASE")
            if u == "CAST":
                self.p += 1
                if not self.accept_op("("):
                    self.err("(")
                inner = self.expr()
                if not self.accept_kw("AS"):
                    self.err("AS")
                to = self.type_name()
                if not self.accept_op(")"):
                    self.err(")")
                return E("cast", args=[inner], to=to)
            if self.t[self.p + 1].kind == "op" and self.t[self.p + 1].text == "(" and u not in _RESERVED:
                self.p += 2
                f = E("func", name=c.text.lower())
                if self.kw("DISTINCT"):
                    raise OracleError("Unsupported", "aggregate DISTINCT")
                if self.accept_op("*"):
                    f.star = True
                elif not (self.cur().kind == "op" and self.cur().text == ")"):
                    f.args.append(self.expr())
                    while self.accept_op(","):
                        f.args.append(self.expr())
                if not self.accept_op(")"):
                    self.err(")")
                return f
        if c.kind in ("id", "qid"):
            name = self.ident("expression")
            e = E("col", name=name)
            if self.cur().kind == "op" and self.cur().text == "." and self.t[self.p + 1].kind in ("id", "qid"):
                self.p += 1
                e.qual, e.name = name, self.ident("column")
            return e
        self.err("an expression")


def parse_expr(text: str) -> E:
    """SessionContext::parse_sql_expr: one scalar expression and nothing after it (expr/mod.rs:111)."""
    ps = _Parser(text)
    if len(ps.t) == 1:
        raise OracleError("Process", "SQL query error: Expected an expression, found: EOF")
    e = ps.expr()
    if ps.p != len(ps.t) - 1:
        ps.err("end of expression")
    return e


def parse(sql: str) -> Query:
    toks = _tokenize(sql)
    if len(toks) == 1:
        raise OracleError("Process", "SQL query error: Expected a statement, found: EOF")
    return _Parser(sql).parse()


# ------------------------------------------------------------------------------------------------
# naming (DataFusion schema_name)
# ------------------------------------------------------------------------------------------------
def _fmt_f64(v: float) -> str:
    if math.isnan(v):
        return "NaN"
    if math.isinf(v):
        return "inf" if v > 0 else "-inf"
    if v == math.floor(v) and abs(v) < 1e15:
        return "%d" % int(v)
    return repr(v)


def display(e: E, table: str) -> str:
    if e.kind == "col":
        return f"{e.qual or table}.{e.name}"
    if e.kind == "lit":
        if e.vtype == "Null":
            return "NULL"
        if e.vtype == "Int64":
            return f"Int64({e.value})"
        if e.vtype == "Float64":
            return f"Float64({_fmt_f64(e.value)})"
        if e.vtype == "Boolean":
            return f"Boolean({'true' if e.value else 'false'})"
        return f'Utf8("{e.value}")'
    if e.kind == "bin":
        return f"{display(e.args[0], table)} {e.op} {display(e.args[1], table)}"
    if e.kind == "un":
        return ("NOT " + display(e.args[0], table)) if e.op == "NOT" else f"(- {display(e.args[0], table)})"
    if e.kind == "cast":
        return display(e.args[0], table)
    if e.kind == "isnull":
        return display(e.args[0], table) + (" IS NOT NULL" if e.negated else " IS NULL")
    if e.kind == "func":
        nm = "avg" if e.name == "mean" else e.name
        inner = "*" if e.star else ",".join(display(a, table) for a in e.args)
        return f"{nm}({inner})"
    raise AssertionError(e.kind)


# ------------------------------------------------------------------------------------------------
# vectorised evaluation: a value is (dtype, numpy values, numpy valid mask)
# ------------------------------------------------------------------------------------------------
@dataclass
class Vec:
    dtype: str  # Int64 | Float64 | Boolean | Utf8 | Binary | Null
    values: object  # np.ndarray (int64/float64/bool) or pa.Array for strings
    valid: np.ndarray


_PA2D = {pa.int64(): "Int64", pa.float64(): "Float64", pa.bool_(): "Boolean", pa.utf8(): "Utf8", pa.binary(): "Binary",
         pa.null(): "Null"}
_D2PA = {v: k for k, v in _PA2D.items()}


def _col_vec(arr: pa.Array) -> Vec:
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks()
    d = _PA2D.get(arr.type)
    if d is None:
        raise OracleError("Unsupported", f"column type {arr.type}")
    n = len(arr)
    valid = np.ones(n, dtype=bool) if arr.null_count == 0 else np.asarray(arr.is_valid())
    if d in ("Int64", "Float64"):
        vals = np.asarray(arr.fill_null(0)).astype(np.int64 if d == "Int64" else np.float64, copy=False)
    elif d == "Boolean":
        vals = np.asarray(arr.fill_null(False)).astype(bool)
    elif d == "Null":
        vals = np.zeros(n, dtype=np.int64)
        valid = np.zeros(n, dtype=bool)
    else:
        vals = arr
    return Vec(d, vals, valid)


def total_order_key(x: np.ndarray) -> np.ndarray:
    """IEEE-754 totalOrder as a monotone int64 key (f64::total_cmp)."""
    b = np.ascontiguousarray(x, dtype=np.float64).view(np.int64)
    return b ^ ((b >> 63).view(np.uint64) >> np.uint64(1)).view(np.int64)


def _cmp(op, a, b):
    return {"=": a == b, "!=": a != b, "<": a < b, "<=": a <= b, ">": a > b, ">=": a >= b}[op]


class _Ctx:
    def __init__(self, table: str, rb: pa.RecordBatch):
        self.table, self.rb, self.n = table, rb, rb.num_rows

    def resolve(self, e: E) -> int:
        if e.qual and e.qual != self.table:
            raise OracleError("Process", f"Execution query error: Schema error: No field named {e.qual}.{e.name}.")
        names = self.rb.schema.names
        if e.name not in names:
            raise OracleError("Process", f"Execution query error: Schema error: No field named {e.name}.")
        return names.index(e.name)

    def type_of(self, e: E) -> str:
        if e.kind == "col":
            t = _PA2D.get(self.rb.schema.field(self.resolve(e)).type)
            if t is None:
                raise OracleError("Unsupported", "column type")
            return t
        if e.kind == "lit":
            return e.vtype
        if e.kind == "bin":
            l, r = self.type_of(e.args[0]), self.type_of(e.args[1])
            num = ("Int64", "Float64", "Null")
            if e.op in ("AND", "OR"):
                if l not in ("Boolean", "Null") or r not in ("Boolean", "Null"):
                    raise OracleError("Process", "Execution query error: Error during planning: boolean op on non-boolean")
                return "Boolean"
            if e.op in ("=", "!=", "<", "<=", ">", ">="):
                ok = (l in num and r in num) or (l in ("Utf8", "Binary") and r in ("Utf8", "Binary")) or (l == r == "Boolean")
                if not ok:
                    if {l, r} & {"Utf8", "Binary"} and {l, r} & {"Int64", "Float64"}:
                        raise OracleError("Unsupported", "string/number comparison")
                    raise OracleError("Process", "Execution query error: Error during planning: cannot compare")
                return "Boolean"
            if l not in num or r not in num:
                raise OracleError("Process", "Execution query error: Error during planning: Cannot coerce arithmetic expression")
            return "Float64" if "Float64" in (l, r) else "Int64"
        if e.kind == "un":
            t = self.type_of(e.args[0])
            if e.op == "NOT":
                if t not in ("Boolean", "Null"):
                    raise OracleError("Process", "Execution query error: Error during planning: NOT on non-boolean")
                return "Boolean"
            if t not in ("Int64", "Float64"):
                raise OracleError("Process", "Execution query error: Error during planning: negation of non-numeric")
            return t
        if e.kind == "cast":
            return e.to
        if e.kind == "isnull":
            self.type_of(e.args[0])
            return "Boolean"
        if e.kind == "func":
            if e.name == "concat" and e.args:
                for a in e.args:  # the library's subset: Utf8 columns and string / NULL literals
                    if a.kind == "col":
                        if self.type_of(a) not in ("Utf8", "Int64", "Boolean"):
                            raise OracleError("Unsupported", f"concat() over a {self.type_of(a)} argument")
                    elif not (a.kind == "lit" and a.vtype in ("Utf8", "Null")):
                        raise OracleError("Unsupported", "concat() over a computed argument")
                return "Utf8"
            raise OracleError("Unsupported", f"scalar function {e.name}()")
        raise AssertionError

    def nullable_of(self, e: E) -> bool:
        if e.kind == "func" and e.name == "concat":
            return True  # ScalarUDFImpl::is_nullable default; the values themselves are never NULL
        if e.kind == "col":
            return self.rb.schema.field(self.resolve(e)).nullable
        if e.kind == "lit":
            return e.vtype == "Null"
        if e.kind == "isnull":
            return False
        return any(self.nullable_of(a) for a in e.args)

    def eval(self, e: E, sel: Optional[np.ndarray] = None) -> Vec:
        """Evaluate on the rows `sel` (index array) or on all rows."""
        n = self.n if sel is None else len(sel)
        if e.kind == "col":
            arr = self.rb.column(self.resolve(e))
            if sel is not None:
                arr = arr.take(pa.array(sel, type=pa.int64()))
            return _col_vec(arr)
        if e.kind == "lit":
            if e.vtype == "Null":
                return Vec("Null", np.zeros(n, dtype=np.int64), np.zeros(n, dtype=bool))
            if e.vtype == "Int64":
                return Vec("Int64", np.full(n, e.value, dtype=np.int64), np.ones(n, dtype=bool))
            if e.vtype == "Float64":
                return Vec("Float64", np.full(n, e.value, dtype=np.float64), np.ones(n, dtype=bool))
            if e.vtype == "Boolean":
                return Vec("Boolean", np.full(n, e.value, dtype=bool), np.ones(n, dtype=bool))
            return Vec("Utf8", pa.array([e.value] * n, type=pa.utf8()), np.ones(n, dtype=bool))
        if e.kind == "bin":
            self.type_of(e)
            a, b = self.eval(e.args[0], sel), self.eval(e.args[1], sel)
            if e.op in ("AND", "OR"):
                at, bt = a.values.astype(bool) & a.valid, b.values.astype(bool) & b.valid
                af, bf = (~a.values.astype(bool)) & a.valid, (~b.values.astype(bool)) & b.valid
                if e.op == "AND":
                    res_false = af | bf
                    res_true = at & bt
                else:
                    res_true = at | bt
                    res_false = af & bf
                return Vec("Boolean", res_true, res_true | res_false)
            valid = a.valid & b.valid
            if e.op in ("=", "!=", "<", "<=", ">", ">="):
                if a.dtype in ("Utf8", "Binary"):
                    la = a.values.cast(pa.binary()).to_pylist()
                    lb = b.values.cast(pa.binary()).to_pylist()
                    res = np.array([(_cmp(e.op, x, y) if (x is not None and y is not None) else False) for x, y in zip(la, lb)],
                                   dtype=bool).reshape(n)
                    return Vec("Boolean", res, valid)
                if a.dtype == "Boolean" and b.dtype == "Boolean":
                    return Vec("Boolean", _cmp(e.op, a.values.astype(np.int8), b.values.astype(np.int8)), valid)
                if "Float64" in (a.dtype, b.dtype):
                    ka = total_order_key(a.values.astype(np.float64))
                    kb = total_order_key(b.values.astype(np.float64))
                    return Vec("Boolean", _cmp(e.op, ka, kb), valid)
                return Vec("Boolean", _cmp(e.op, a.values, b.values), valid)
            # arithmetic
            if "Float64" in (a.dtype, b.dtype):
                x, y = a.values.astype(np.float64), b.values.astype(np.float64)
                with np.errstate(all="ignore"):
                    if e.op == "+":
                        r = x + y
                    elif e.op == "-":
                        r = x - y
                    elif e.op == "*":
                        r = x * y
                    elif e.op == "/":
                        r = x / y
                    else:
                        r = np.fmod(x, y)
                return Vec("Float64", r, valid)
            x, y = a.values.astype(np.int64), b.values.astype(np.int64)
            with np.errstate(all="ignore"):
                if e.op == "+":
                    r = x + y
                elif e.op == "-":
                    r = x - y
                elif e.op == "*":
                    r = x * y
                else:
                    if np.any((y == 0) & valid):
                        raise OracleError("Process", "Collection query results error: Arrow error: Divide by zero error")
                    # arrow-arith div_checked / mod_checked: i64::MIN / -1 and i64::MIN % -1 both overflow (checked_div / checked_rem → None)
                    if np.any((x == np.iinfo(np.int64).min) & (y == -1) & valid):
                        raise OracleError("Process", "Collection query results error: Arrow error: Arithmetic overflow: Overflow happened on: "
                                                     f"-9223372036854775808 {e.op} -1")
                    ys = np.where(y == 0, 1, y)
                    q = np.abs(x.astype(object)) // np.abs(ys.astype(object))  # truncating division, exact
                    q = np.where((x < 0) != (ys < 0), -q, q)
                    if e.op == "/":
                        r = np.array([int(v) for v in q], dtype=object)
                    else:
                        r = x.astype(object) - q * ys.astype(object)
                    r = np.array([((int(v) + 2 ** 63) % 2 ** 64) - 2 ** 63 for v in r], dtype=np.int64).reshape(n)
            return Vec("Int64", r, valid)
        if e.kind == "un":
            a = self.eval(e.args[0], sel)
            self.type_of(e)
            if e.op == "NOT":
                return Vec("Boolean", ~a.values.astype(bool), a.valid)
            if a.dtype == "Float64":
                return Vec("Float64", -a.values, a.valid)
            with np.errstate(all="ignore"):
                return Vec("Int64", (0 - a.values.astype(np.int64)), a.valid)
        if e.kind == "cast":
            a = self.eval(e.args[0], sel)
            return _cast(a, e.to)
        if e.kind == "isnull":
            a = self.eval(e.args[0], sel)
            r = a.valid if e.negated else ~a.valid
            return Vec("Boolean", r.copy(), np.ones(n, dtype=bool))
        if e.kind == "func":
            self.type_of(e)
            # datafusion-functions ConcatFunc: NULL arguments count as empty strings, the result is never NULL
            import pyarrow.compute as pc

            parts = []
            for a in e.args:
                v = self.eval(a, sel)
                if v.dtype in ("Int64", "Boolean"):
                    v = _cast(v, "Utf8")  # concat() coerces its arguments to strings
                if v.dtype == "Null":
                    parts.append(pa.array([""] * n, type=pa.utf8()))
                else:
                    arr = v.values if isinstance(v.values, (pa.Array, pa.ChunkedArray)) else pa.array(v.values)
                    parts.append(pc.if_else(pa.array(v.valid), arr, pa.scalar("", pa.utf8())))
            out = pc.binary_join_element_wise(*parts, pa.scalar("", pa.utf8())) if n else pa.array([], type=pa.utf8())
            return Vec("Utf8", out, np.ones(n, dtype=bool))
        raise AssertionError


def _cast(a: Vec, to: str) -> Vec:
    if a.dtype == to or a.dtype == "Null":
        return Vec(to if a.dtype == "Null" else a.dtype, a.values, a.valid) if a.dtype != "Null" else a
    if a.dtype == "Int64" and to == "Float64":
        return Vec("Float64", a.values.astype(np.float64), a.valid)
    if a.dtype == "Float64" and to == "Int64":
        x = a.values
        bad = a.valid & ~((x > -9223372036854777856.0) & (x < 9223372036854775808.0))
        if np.any(bad):
            raise OracleError("Process", "Collection query results error: Arrow error: Cast error")
        with np.errstate(all="ignore"):
            return Vec("Int64", np.trunc(np.where(a.valid, x, 0.0)).astype(np.int64), a.valid)
    if a.dtype == "Boolean" and to == "Int64":
        return Vec("Int64", a.values.astype(np.int64), a.valid)
    if a.dtype == "Boolean" and to == "Float64":
        return Vec("Float64", a.values.astype(np.float64), a.valid)
    if a.dtype == "Int64" and to == "Boolean":
        return Vec("Boolean", a.values != 0, a.valid)
    if a.dtype == "Float64" and to == "Boolean":
        return Vec("Boolean", a.values != 0.0, a.valid)
    if a.dtype == "Binary" and to == "Utf8":
        for v in a.values.to_pylist():
            if v is not None:
                try:
                    v.decode("utf-8")
                except UnicodeDecodeError:
                    raise OracleError("Process", "Collection query results error: Arrow error: Invalid UTF-8")
        return Vec("Utf8", a.values.cast(pa.utf8()), a.valid)
    if a.dtype == "Utf8" and to == "Binary":
        return Vec("Binary", a.values.cast(pa.binary()), a.valid)
    if a.dtype == "Int64" and to == "Utf8":  # arrow-cast: lexical decimal text
        return Vec("Utf8", pa.array([str(int(v)) if ok else None for v, ok in zip(a.values.tolist(), a.valid.tolist())], pa.utf8()), a.valid)
    if a.dtype == "Boolean" and to == "Utf8":  # arrow-cast: "true" / "false"
        return Vec("Utf8", pa.array([("true" if v else "false") if ok else None for v, ok in zip(a.values.tolist(), a.valid.tolist())], pa.utf8()), a.valid)
    raise OracleError("Unsupported", f"CAST {a.dtype} → {to}")


def _vec_to_arrow(v: Vec) -> pa.Array:
    mask = ~v.valid if not v.valid.all() else None
    if v.dtype in ("Utf8", "Binary"):
        arr = v.values
        if mask is not None:
            arr = pc.if_else(pa.array(v.valid), arr, pa.nulls(len(arr), arr.type))
        return arr
    if v.dtype == "Null":
        return pa.nulls(len(v.valid))
    return pa.array(v.values, type=_D2PA[v.dtype], mask=mask)


_AGG = {"sum", "count", "avg", "mean", "min", "max"}


def _has_agg(e: Optional[E]) -> bool:
    if e is None:
        return False
    if e.kind == "func" and e.name in _AGG:
        return True
    return any(_has_agg(a) for a in e.args)


def _empty_schema_batch() -> pa.RecordBatch:
    return pa.RecordBatch.from_arrays([], schema=pa.schema([]))


def sum_exact(xs: list[float]) -> float:
    """The IEEE-754 sum of `xs` without intermediate rounding, total over non-finite inputs: NaN when a NaN or both
    infinities occur, ±inf when infinities of one sign occur, else the correctly rounded exact sum — ±inf when that
    leaves the double range.  (Any summation order yields the same NaN / ±inf in the non-finite cases.)"""
    if any(math.isnan(x) for x in xs):
        return math.nan
    pinf, ninf = math.inf in xs, -math.inf in xs
    if pinf or ninf:
        return math.nan if pinf and ninf else (math.inf if pinf else -math.inf)
    try:
        return math.fsum(xs)
    except OverflowError:  # fsum gives up once a partial sum leaves the double range: sum exactly, round once
        from fractions import Fraction

        s = sum(Fraction(x) for x in xs)
        try:
            return float(s)  # int / int true division: correctly rounded
        except OverflowError:
            return math.inf if s > 0 else -math.inf


def group_sum_exact(values: np.ndarray, codes: np.ndarray, k: int) -> list[float]:
    """Correctly-rounded per-group Float64 sums (sum_exact) — the reference point of the tolerance."""
    order = np.argsort(codes, kind="stable")
    sv, sc = values[order], codes[order]
    bounds = np.searchsorted(sc, np.arange(k + 1))
    return [sum_exact(sv[bounds[i]:bounds[i + 1]].tolist()) for i in range(k)]


def sql_process(rb: pa.RecordBatch, query: str, table_name: str = "flow") -> Optional[pa.RecordBatch]:
    """SqlProcessor::process (sql.rs:209-220).  None ⇔ ProcessResult::None."""
    q = parse(query)  # construction-time parse (sql.rs:91-98)
    if rb.num_rows == 0:
        return None
    if q.joins:
        raise OracleError("Unsupported", "JOIN in a single-table processor call")
    if q.table != table_name:
        raise OracleError("Process", f"Execution query error: Error during planning: table '{q.table}' not found")
    vis = q.alias or q.table
    ctx = _Ctx(vis, rb)
    has_agg = bool(q.group_by) or any((not it.star) and _has_agg(it.expr) for it in q.select)
    if _has_agg(q.where):
        raise OracleError("Process", "Execution query error: Error during planning: Aggregate functions are not allowed in the WHERE clause")

    sel = None
    if q.where is not None:
        t = ctx.type_of(q.where)
        if t not in ("Boolean", "Null"):
            raise OracleError("Process", "Execution query error: Error during planning: Cannot create filter with non-boolean predicate")
        m = ctx.eval(q.where)
        sel = np.nonzero(m.values.astype(bool) & m.valid)[0]

    if not has_agg:
        cols, fields = [], []
        for it in q.select:
            if it.star:
                if it.star_qual and it.star_qual != vis:
                    raise OracleError("Process", "Execution query error: Error during planning: Invalid qualifier " + it.star_qual)
                for i, f in enumerate(rb.schema):
                    if f.type not in _PA2D:
                        raise OracleError("Unsupported", f"column type {f.type}")
                    arr = rb.column(i)
                    cols.append(arr if sel is None else arr.take(pa.array(sel, type=pa.int64())))
                    fields.append(pa.field(f.name, f.type, f.nullable))
            else:
                v = ctx.eval(it.expr, sel)
                if v.dtype == "Null":
                    raise OracleError("Unsupported", "NULL-typed projection")
                name = it.alias or (it.expr.name if it.expr.kind == "col" else display(it.expr, vis))
                arr = _vec_to_arrow(v)
                cols.append(arr)
                fields.append(pa.field(name, arr.type, ctx.nullable_of(it.expr)))
        out = pa.RecordBatch.from_arrays(cols, schema=pa.schema(fields))
        if q.limit >= 0:
            out = out.slice(0, q.limit)
        return out

    # ---- aggregate ----
    if q.limit >= 0:
        raise OracleError("Unsupported", "LIMIT on aggregate")
    n_sel = rb.num_rows if sel is None else len(sel)
    key_disp, key_arrays = [], []
    for g in q.group_by:
        if g.kind != "col":
            raise OracleError("Unsupported", "GROUP BY expression")
        arr = rb.column(ctx.resolve(g))
        if arr.type not in (pa.int64(), pa.utf8(), pa.binary(), pa.bool_()):
            raise OracleError("Unsupported", f"GROUP BY key type {arr.type}")
        key_arrays.append(arr if sel is None else arr.take(pa.array(sel, type=pa.int64())))
        key_disp.append(display(g, vis))
    if len(key_arrays) > 2:
        raise OracleError("Unsupported", "more than two GROUP BY keys")
    # group codes: dictionary-encode each key (NULL = its own group), combine
    if key_arrays:
        codes = np.zeros(n_sel, dtype=np.int64)
        for arr in key_arrays:
            d = arr.dictionary_encode(null_encoding="encode")
            idx = np.asarray(d.indices).astype(np.int64)
            codes = codes * max(len(d.dictionary), 1) + idx
        uniq, first, inv = np.unique(codes, return_index=True, return_inverse=True)
        k = len(uniq)
        inv = inv.reshape(-1)
    else:
        k, inv, first = 1, np.zeros(n_sel, dtype=np.int64), np.zeros(1, dtype=np.int64)
        if n_sel == 0:
            first = np.zeros(0, dtype=np.int64)
    if key_arrays and n_sel == 0:
        k = 0

    cols, fields = [], []
    for it in q.select:
        if it.star:
            raise OracleError("Process", "Execution query error: Error during planning: SELECT * with GROUP BY")
        e = it.expr
        cast_str = e.kind == "cast" and e.to == "Utf8" and e.args[0].kind == "func" and e.args[0].name in _AGG
        if cast_str:
            e = e.args[0]

        def _finish():
            if cast_str:  # CAST(<Int64 aggregate> AS STRING): arrow-cast's decimal text, NULL stays NULL
                if cols[-1].type != pa.int64():
                    raise OracleError("Unsupported", f"CAST({cols[-1].type} aggregate AS STRING)")
                import pyarrow.compute as pc

                cols[-1] = pc.cast(cols[-1], pa.utf8())
                fields[-1] = pa.field(fields[-1].name, pa.utf8(), fields[-1].nullable)

        if e.kind == "func" and e.name in _AGG:
            fn = "avg" if e.name == "mean" else e.name
            name = it.alias or display(E("func", name=fn, args=e.args, star=e.star), vis)
            count_star = fn == "count" and (e.star or (len(e.args) == 1 and e.args[0].kind == "lit" and e.args[0].vtype != "Null"))
            if count_star:
                cnt = np.bincount(inv, minlength=k).astype(np.int64)
                cols.append(pa.array(cnt, type=pa.int64()))
                fields.append(pa.field(name, pa.int64(), False))
                _finish()
                continue
            if len(e.args) != 1 or e.star:
                raise OracleError("Process", f"Execution query error: Error during planning: {fn} expects one argument")
            if _has_agg(e.args[0]):
                raise OracleError("Process", "Execution query error: Error during planning: nested aggregate")
            v = ctx.eval(e.args[0], sel)
            if fn == "count":
                cnt = np.bincount(inv[v.valid], minlength=k).astype(np.int64)
                cols.append(pa.array(cnt, type=pa.int64()))
                fields.append(pa.field(name, pa.int64(), False))
                _finish()
                continue
            if v.dtype not in ("Int64", "Float64"):
                if fn in ("min", "max"):
                    raise OracleError("Unsupported", f"{fn} over {v.dtype}")
                raise OracleError("Process", f"Execution query error: Error during planning: {fn} does not support {v.dtype}")
            gi, gv = inv[v.valid], v.values[v.valid]
            cnt = np.bincount(gi, minlength=k).astype(np.int64)
            some = cnt > 0
            if fn == "sum":
                if v.dtype == "Int64":
                    acc = np.zeros(k, dtype=np.int64)
                    with np.errstate(all="ignore"):
                        np.add.at(acc, gi, gv)
                    cols.append(pa.array(acc, type=pa.int64(), mask=~some))
                    fields.append(pa.field(name, pa.int64(), True))
                else:
                    acc = np.array(group_sum_exact(gv, gi, k), dtype=np.float64).reshape(k)
                    cols.append(pa.array(acc, type=pa.float64(), mask=~some))
                    fields.append(pa.field(name, pa.float64(), True))
            elif fn == "avg":
                acc = np.array(group_sum_exact(gv.astype(np.float64), gi, k), dtype=np.float64).reshape(k)
                with np.errstate(all="ignore"):
                    avg = acc / np.where(some, cnt, 1).astype(np.float64)
                cols.append(pa.array(avg, type=pa.float64(), mask=~some))
                fields.append(pa.field(name, pa.float64(), True))
            else:
                if v.dtype == "Float64":
                    keys = total_order_key(gv)
                    init = np.iinfo(np.int64).max if fn == "min" else np.iinfo(np.int64).min
                    acc = np.full(k, init, dtype=np.int64)
                    (np.minimum if fn == "min" else np.maximum).at(acc, gi, keys)
                    back = acc ^ ((acc >> 63).view(np.uint64) >> np.uint64(1)).view(np.int64)
                    cols.append(pa.array(back.view(np.float64), type=pa.float64(), mask=~some))
                    fields.append(pa.field(name, pa.float64(), True))
                else:
                    init = np.iinfo(np.int64).max if fn == "min" else np.iinfo(np.int64).min
                    acc = np.full(k, init, dtype=np.int64)
                    (np.minimum if fn == "min" else np.maximum).at(acc, gi, gv)
                    cols.append(pa.array(acc, type=pa.int64(), mask=~some))
                    fields.append(pa.field(name, pa.int64(), True))
        elif e.kind == "col":
            d = display(e, vis)
            if d not in key_disp:
                ctx.resolve(e)
                raise OracleError("Process", "Execution query error: Error during planning: Column in SELECT must be in GROUP BY or an aggregate function")
            karr = key_arrays[key_disp.index(d)]
            cols.append(karr.take(pa.array(first[:k], type=pa.int64())))
            fields.append(pa.field(it.alias or e.name, karr.type, rb.schema.field(ctx.resolve(e)).nullable))
        elif e.kind == "lit":
            if e.vtype == "Null":
                raise OracleError("Unsupported", "NULL literal in aggregate SELECT")
            t = _D2PA[e.vtype]
            cols.append(pa.array([e.value] * k, type=t))
            fields.append(pa.field(it.alias or display(e, vis), t, False))
        else:
            raise OracleError("Unsupported", "expression in aggregate SELECT list")
        _finish()
    return pa.RecordBatch.from_arrays(cols, schema=pa.schema(fields))


def sql_join(tables: dict[str, pa.RecordBatch], query: str) -> pa.RecordBatch:
    """JoinOperation's `ctx.sql(query).collect()` (buffer/join.rs:111-131) for one equi-join: inner, or LEFT / RIGHT
    [OUTER] as in the shipped temporary_list example (examples/redis_temporary_example.yaml:29): rows of the preserved
    side without a match appear once with NULLs for the other side's columns, whose fields become nullable (DataFusion
    HashJoinExec / build_join_schema).  PARITY unpinned: the reference holds no join assertion."""
    q = parse(query)
    if not q.joins:
        if q.table not in tables:
            raise OracleError("Process", f"Execution query error: Error during planning: table '{q.table}' not found")
        r = sql_process(tables[q.table], query, q.table)
        return r if r is not None else _empty_schema_batch()
    if len(q.joins) != 1 or q.where is not None or q.group_by or q.limit >= 0:
        raise OracleError("Unsupported", "join shape")
    jt, ja, on, jtype = q.joins[0]
    for t in (q.table, jt):
        if t not in tables:
            raise OracleError("Process", f"Execution query error: Error during planning: table '{t}' not found")
    L, R = tables[q.table], tables[jt]
    lvis, rvis = q.alias or q.table, ja or jt

    def side(c: E):
        if c.qual == lvis:
            return 0, c.name
        if c.qual == rvis:
            return 1, c.name
        if c.qual:
            raise OracleError("Process", f"Execution query error: Schema error: No field named {c.qual}.{c.name}.")
        inl, inr = c.name in L.schema.names, c.name in R.schema.names
        if inl and inr:
            raise OracleError("Process", "Execution query error: Schema error: Ambiguous reference")
        if inl:
            return 0, c.name
        if inr:
            return 1, c.name
        raise OracleError("Process", f"Execution query error: Schema error: No field named {c.name}.")

    if not (on.kind == "bin" and on.op == "=" and on.args[0].kind == "col" and on.args[1].kind == "col"):
        raise OracleError("Unsupported", "join condition")
    (s0, n0), (s1, n1) = side(on.args[0]), side(on.args[1])
    if s0 == s1:
        raise OracleError("Unsupported", "join condition on one table")
    lk, rk = (n0, n1) if s0 == 0 else (n1, n0)
    lkeys, rkeys = L.column(lk).to_pylist(), R.column(rk).to_pylist()
    build: dict = {}
    for j, kv in enumerate(rkeys):
        if kv is not None:
            build.setdefault(kv, []).append(j)
    li, ri = [], []
    matched_r = set()
    for i, kv in enumerate(lkeys):
        hits = build.get(kv, ()) if kv is not None else ()
        for j in hits:
            li.append(i)
            ri.append(j)
            matched_r.add(j)
        if not hits and jtype == "left":
            li.append(i)
            ri.append(None)
    if jtype == "right":
        for j in range(len(rkeys)):
            if j not in matched_r:
                li.append(None)
                ri.append(j)
    li, ri = pa.array(li, type=pa.int64()), pa.array(ri, type=pa.int64())
    cols, fields = [], []
    null_side = {"left": 1, "right": 0}.get(jtype)  # the side whose columns turn NULL for unmatched rows

    def add_all(s):
        T, idx = (L, li) if s == 0 else (R, ri)
        for i, f in enumerate(T.schema):
            cols.append(T.column(i).take(idx))
            fields.append(pa.field(f.name, f.type, f.nullable or s == null_side))

    for it in q.select:
        if it.star:
            if not it.star_qual:
                add_all(0)
                add_all(1)
            elif it.star_qual == lvis:
                add_all(0)
            elif it.star_qual == rvis:
                add_all(1)
            else:
                raise OracleError("Process", "Execution query error: Error during planning: Invalid qualifier")
        elif it.expr.kind == "col":
            s, nm = side(it.expr)
            T, idx = (L, li) if s == 0 else (R, ri)
            f = T.schema.field(nm)
            cols.append(T.column(nm).take(idx))
            fields.append(pa.field(it.alias or nm, f.type, f.nullable or s == null_side))
        else:
            raise OracleError("Unsupported", "computed join projection")
    return pa.RecordBatch.from_arrays(cols, schema=pa.schema(fields))


# ------------------------------------------------------------------------------------------------
# expr::evaluate_expr  (crates/arkflow-plugin/src/expr/mod.rs:92-122)
# ------------------------------------------------------------------------------------------------
def _references_column(e: E) -> bool:
    return e.kind == "col" or any(_references_column(a) for a in e.args)


def evaluate_expr(text: str, rb: pa.RecordBatch) -> tuple[bool, pa.Array]:
    """→ (is_scalar, values).  ColumnarValue::Scalar when the expression references no column (a literal
    evaluates to a scalar, and datum::apply keeps scalar ∘ scalar a scalar), else an array of rb.num_rows.
    PARITY: pinned by expr/mod.rs:133-212 — `0.9` → Scalar Float64(0.9); concat(name, ' is here') → the three
    joined strings; `invalid sql` and `1 + name` → errors."""
    e = parse_expr(text)
    if _has_agg(e):
        raise OracleError("Process", "Error during planning: aggregate functions are not valid in a scalar expression")
    scalar = not _references_column(e)
    base = pa.RecordBatch.from_arrays([pa.array([0], pa.int64())], names=["\x01dummy"]) if scalar else rb
    ctx = _Ctx("flow", base)
    ctx.type_of(e)
    v = ctx.eval(e)
    if v.dtype == "Null":
        raise OracleError("Unsupported", "NULL-typed projection")
    return scalar, _vec_to_arrow(v)
