"""The JSON path functions without a GPU: the oracle (tests/json_path_oracle.py) against hand-written values for every
rule it restates, the reference docs' examples where they agree with the crate, and the forms the library refuses at
bind time (Unsupported, raised before any device work), display names, and expression evaluation, which does not bind
the calls.  Join queries import their tables before binding, so their check is in test_json_functions_gpu.py.
"""
import math

import pyarrow as pa
import pytest

from arkflow_b200.processor import ArkError, MessageBatch, SqlProcessor
from json_path_oracle import json_call, sql_process_json

J = json_call


@pytest.mark.parametrize("fn,doc,path,want", [
    # every value kind through every function
    ("json_get_str", '{"a":"x"}', ["a"], "x"),
    ("json_get_str", '{"a":1}', ["a"], None),
    ("json_get_int", '{"a":1}', ["a"], 1),
    ("json_get_int", '{"a":1.0}', ["a"], None),
    ("json_get_int", '{"a":1e2}', ["a"], None),
    ("json_get_int", '{"a":"1"}', ["a"], None),
    ("json_get_float", '{"a":1}', ["a"], 1.0),
    ("json_get_float", '{"a":-2.5e-3}', ["a"], -0.0025),
    ("json_get_float", '{"a":true}', ["a"], None),
    ("json_get_bool", '{"a":true}', ["a"], True),
    ("json_get_bool", '{"a":false}', ["a"], False),
    ("json_get_bool", '{"a":0}', ["a"], None),
    ("json_get_json", '{"a": {"b" : [1, 2]} }', ["a"], '{"b" : [1, 2]}'),
    ("json_get_json", '{"a":"x\\n"}', ["a"], '"x\\n"'),
    ("json_get_json", '{"a":null}', ["a"], "null"),
    ("json_as_text", '{"a":"x\\n"}', ["a"], "x\n"),
    ("json_as_text", '{"a":-1.50}', ["a"], "-1.50"),
    ("json_as_text", '{"a":true}', ["a"], "true"),
    ("json_as_text", '{"a":[1, {"b":2}]}', ["a"], '[1, {"b":2}]'),
    ("json_as_text", '{"a":null}', ["a"], None),
    ("json_length", '{"a":[1,[2,3],{}]}', ["a"], 3),
    ("json_length", '{"a":{"x":1,"y":2}}', ["a"], 2),
    ("json_length", '{"a":[]}', ["a"], 0),
    ("json_length", '{"a":"abc"}', ["a"], None),
    ("json_length", '[1,2', [], None),
    ("json_contains", '{"a":null}', ["a"], True),
    ("json_contains", '{"a":1}', ["b"], False),
    ("json_contains", None, ["a"], False),
    ("json_get_int", None, ["a"], None),
    # paths: keys, indices, mismatched containers, empty path
    ("json_get_int", '[10,20,30]', [2], 30),
    ("json_get_int", '[10,20,30]', [3], None),
    ("json_get_int", '[10,20,30]', ["1"], None),
    ("json_get_int", '{"1":5}', [1], None),
    ("json_get_int", '7', [], 7),
    ("json_get_str", '{"a":[{"b":"deep"}]}', ["a", 0, "b"], "deep"),
    ("json_get_int", '{"a":{"b":{"c":{"d":{"e":{"f":{"g":{"h":8}}}}}}}}', list("abcdefgh"), 8),
    ("json_length", '{"a":{"b":{"c":{"d":{"e":{"f":{"g":{"h":[1,2]}}}}}}}}', list("abcdefgh"), 2),
    # duplicate keys: the first wins, even when the path fails inside it
    ("json_get_int", '{"a":1,"a":2}', ["a"], 1),
    ("json_get_int", '{"a":{"x":1},"a":{"b":2}}', ["a", "b"], None),
    # escaped keys and values, surrogate pairs
    ("json_get_int", '{"k\\u0065y":1}', ["key"], 1),
    ("json_get_int", '{"\\"q\\"":3}', ['"q"'], 3),
    ("json_get_str", '{"a":"\\ud83d\\ude00 \\u00e9\\t"}', ["a"], "\U0001F600 é\t"),
    ("json_get_str", '{"a":"\\ud83d"}', ["a"], None),
    ("json_get_str", '{"a":"\\q"}', ["a"], None),
    ("json_get_str", '{"é":"ü"}', ["é"], "ü"),
    # whitespace everywhere; brackets and quotes inside strings
    ("json_get_int", ' \t\n{ "s" : "]}\\"[{" , "a" :\r\n 4 } ', ["a"], 4),
    ("json_get_int", '{"s":["}", {"t":"]"}], "a":5}', ["a"], 5),
    # malformed and truncated documents; the lazy walk ignores what lies after a found value
    ("json_get_int", '{"a":1', ["a"], 1),
    ("json_get_int", '{"a":1}garbage', ["a"], 1),
    ("json_get_int", '{"a":12x}', ["a"], 12),
    ("json_get_int", '{"b":[1,}, "a":1}', ["a"], None),
    ("json_get_int", '{"b":01, "a":1}', ["a"], None),
    ("json_get_int", '{"a":', ["a"], None),
    ("json_get_int", '', [], None),
    ("json_get_int", '{"a" 1}', ["a"], None),
    ("json_get_json", '{"a":[1,2}', ["a"], None),
    ("json_contains", '{"a":[1,2', ["a"], True),
    ("json_contains", '[1,]', [1], False),
    ("json_contains", '{"b":tru,"a":1}', ["a"], False),
    ("json_get_bool", '{"a":tru}', ["a"], None),
    ("json_get_str", '{"a":"x', ["a"], None),
    ("json_get_str", '{"a":"x\ny"}', ["a"], None),
    # integer limits and float conversions
    ("json_get_int", '9223372036854775807', [], 2**63 - 1),
    ("json_get_int", '-9223372036854775808', [], -2**63),
    ("json_get_int", '9223372036854775808', [], None),
    ("json_get_int", '-9223372036854775809', [], None),
    ("json_get_int", '-0', [], 0),
    ("json_get_float", '9223372036854775808', [], 9223372036854775808.0),
    ("json_get_float", '1e400', [], None),
    ("json_get_float", '4.9406564584124654e-324', [], 5e-324),
    ("json_get_float", '0.1', [], 0.1),
])
def test_oracle_rules(fn, doc, path, want):
    got = J(fn, doc, path)
    assert got == want and type(got) is type(want), (fn, doc, path, got, want)


def test_oracle_signed_zero():
    assert math.copysign(1.0, J("json_get_float", "-0", [])) == 1.0  # the integer 0
    assert math.copysign(1.0, J("json_get_float", "-0.0", [])) == -1.0


def test_oracle_nesting_limit():
    assert J("json_length", "[" * 256 + "]" * 256, []) == 1
    assert J("json_length", "[" * 257 + "]" * 257, []) is None


def test_reference_doc_examples_that_agree():
    # docs/docs/sql/7-scalar_functions.md, "JSON Functions"
    assert J("json_contains", '{"a": {"b": 1}}', ["a"]) is True
    assert J("json_contains", '{"user": {"name": "John", "age": 30}}', ["user"]) is True
    assert J("json_get_str", '{"user": {"name": "John"}}', ["user", "name"]) == "John"
    assert J("json_get_int", '{"user": {"id": 12345, "age": 30}}', ["user", "id"]) == 12345
    # the docs write indices as '1'; the crate reads a string as a key (an unverified contradiction, see the oracle)
    assert J("json_get_str", '["apple", "banana", "orange"]', [1]) == "banana"
    assert J("json_get_str", '["apple", "banana", "orange"]', ["1"]) is None


def test_oracle_query_names_and_groups():
    rb = pa.record_batch({"doc": pa.array(['{"s":"a","v":1}', '{"s":"b","v":2.5}', '{"s":"a","v":3}', None])})
    out = sql_process_json(rb, "SELECT json_get_str(doc,'s'), count(*), sum(json_get_float(doc,'v')) FROM flow "
                               "GROUP BY json_get_str(doc,'s')")
    assert out.schema.names == ['json_get_str(flow.doc,Utf8("s"))', "count(*)", 'sum(json_get_float(flow.doc,Utf8("v")))']
    assert sorted(zip(*[c.to_pylist() for c in out.columns]), key=str) == sorted([("a", 2, 4.0), ("b", 1, 2.5), (None, 1, None)], key=str)
    out = sql_process_json(rb, "SELECT json_get_int(doc,'v') + 1, json_get_int(doc, 'x', 0) AS x FROM flow")
    assert out.schema.names == ['json_get_int(flow.doc,Utf8("v")) + Int64(1)', "x"]


def _bind_error(query, rb=None):
    rb = rb if rb is not None else pa.record_batch({"doc": pa.array(['{"a":1}']), "b": pa.array([b"{}"]), "n": pa.array([1])})
    with pytest.raises(ArkError) as e:
        SqlProcessor({"query": query}).process(MessageBatch.new_arrow(rb))
    return e.value


@pytest.mark.parametrize("query,needle", [
    ("SELECT json_get_int(b, 'a') FROM flow", "json_get_int(): the JSON document"),
    ("SELECT json_get_str('{\"a\":1}', 'a') FROM flow", "json_get_str(): the JSON document"),
    ("SELECT json_get_str(concat(doc, 'x'), 'a') FROM flow", "json_get_str(): the JSON document"),
    ("SELECT json_get_int(CAST(n AS STRING), 'a') FROM flow", "json_get_int(): the JSON document"),
    ("SELECT json_length(json_get_json(doc, 'a')) FROM flow", "json_length(): the JSON document"),
    ("SELECT json_get_int(doc, -1) FROM flow", "path element"),
    ("SELECT json_get_int(doc, n) FROM flow", "path element"),
    ("SELECT json_get_int(doc, 'a' || 'b') FROM flow", None),
    ("SELECT json_get_int(doc, 1.5) FROM flow", "path element"),
    ("SELECT json_get_int(doc, true) FROM flow", "path element"),
    ("SELECT json_get_int(doc, NULL) FROM flow", "path element"),
    ("SELECT json_get_int(doc, 'a','b','c','d','e','f','g','h','i') FROM flow", "more than 8 path elements"),
    ("SELECT json_get_int() FROM flow", "without a JSON document"),
    ("SELECT json_get(doc, 'a') FROM flow", "scalar function json_get()"),
])
def test_unsupported_forms(lib, query, needle):
    e = _bind_error(query)
    assert e.kind in ("Unsupported", "Process"), e.message
    if needle is not None:
        assert e.kind == "Unsupported" and needle in e.message, e.message


def test_unknown_document_column_is_a_planning_error(lib):
    e = _bind_error("SELECT json_get_int(nope, 'a') FROM flow")
    assert e.kind == "Process" and "No field named nope" in e.message


def test_group_by_float_key_stays_unsupported(lib):
    e = _bind_error("SELECT json_get_float(doc, 'a'), count(*) FROM flow GROUP BY json_get_float(doc, 'a')")
    assert e.kind == "Unsupported" and "GROUP BY key of type Float64" in e.message


def test_expression_evaluation_does_not_bind_json_calls(lib):
    from arkflow_b200.expr import evaluate_expr

    rb = pa.record_batch({"doc": pa.array(['{"a":1}'])})
    with pytest.raises(ArkError) as e:
        evaluate_expr("json_get_int(doc, 'a')", rb)
    assert e.value.kind == "Unsupported" and "scalar function json_get_int()" in e.value.message
