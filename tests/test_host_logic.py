"""Host-side mirror of the reference interface: Schema, PartitionSpec, PartitionCursor, local
dataframes, function wrapper.  Cases follow the reference's own unit tests
(tests/fugue/collections/test_partition.py, tests/fugue/dataframe/*)."""
import json
from collections import OrderedDict

import pandas as pd
import pyarrow as pa
import pytest
from pytest import raises

from fugue_b200.dataframe import ArrayDataFrame, ArrowDataFrame, PandasDataFrame, df_eq
from fugue_b200.partition import KEYWORD_ROWCOUNT, PartitionCursor, PartitionSpec, parse_presort_exp
from fugue_b200.schema import Schema, SchemaError


def test_schema_expressions():
    s = Schema("a:int,b:str,c:double,d:long,e:bool,f:datetime")
    assert s.names == list("abcdef")
    assert s.types[0] == pa.int32() and s.types[3] == pa.int64() and s.types[2] == pa.float64()
    assert str(s) == "a:int,b:str,c:double,d:long,e:bool,f:datetime"
    assert s == "a:int,b:str,c:double,d:long,e:bool,f:datetime"
    assert Schema(s.pa_schema) == s
    assert "a" in s and "z" not in s and ["a", "b"] in s and "a:int" in s and "a:long" not in s
    assert s.extract(["c", "a"]) == "c:double,a:int"
    assert s.exclude(["a", "b"]) == "c:double,d:long,e:bool,f:datetime"
    assert (Schema("a:int") + "b:str") == "a:int,b:str"
    assert s.index_of_key("c") == 2
    with raises(SchemaError):
        Schema("a:int,a:str")
    with raises(SchemaError):
        Schema("a")
    with raises(KeyError):
        s.index_of_key("x")


def test_schema_transform():
    s = Schema("a:int,b:str")
    assert s.transform("*") == s
    assert s.transform("*,c:double") == "a:int,b:str,c:double"
    assert s.transform("*-a") == "b:str"
    assert s.transform("*~x") == s
    assert s.transform("x:long") == "x:long"
    assert s.transform("*", "c:long") == "a:int,b:str,c:long"
    assert s.union("c:int") == "a:int,b:str,c:int"
    assert s.intersect(["b", "z"]) == "b:str"
    assert s.rename({"a": "x"}) == "x:int,b:str"


def test_parse_presort_exp():
    assert parse_presort_exp(None) == OrderedDict()
    assert parse_presort_exp("c") == OrderedDict([("c", True)])
    assert parse_presort_exp("         c") == OrderedDict([("c", True)])
    assert parse_presort_exp("c           desc") == OrderedDict([("c", False)])
    assert parse_presort_exp("b desc, c asc") == OrderedDict([("b", False), ("c", True)])
    assert parse_presort_exp("DESC DESC, ASC ASC") == OrderedDict([("DESC", False), ("ASC", True)])
    assert parse_presort_exp([("b", False), ("c", True)]) == OrderedDict([("b", False), ("c", True)])
    assert parse_presort_exp("`` desc, `a b` asc, ````, `中国`") == OrderedDict(
        [("", False), ("a b", True), ("`", True), ("中国", True)])
    for bad in ["b dsc, c asc", "c true", "c true, c true", "a b dsc, c asc"]:
        with raises(SyntaxError):
            parse_presort_exp(bad)
    with raises(SyntaxError):
        parse_presort_exp([("b", "desc"), ("c", "asc")])


def test_partition_spec():
    p = PartitionSpec()
    assert p.partition_by == [] and p.num_partitions == "0" and p.algo == "default" and p.empty
    assert PartitionSpec(None).empty and PartitionSpec(PartitionSpec(None)).empty
    p = PartitionSpec(json.dumps(dict(partition_by=["a", "b", "c"], num_partitions=1)))
    assert p.partition_by == ["a", "b", "c"] and p.num_partitions == "1" and not p.empty
    p = PartitionSpec(dict(by=["a", "b", "c"], presort="d asc,e desc"))
    assert dict(d=True, e=False) == dict(p.presort) and p.num_partitions == "0"
    p = PartitionSpec(by=["a ", "b", "c"], num=5, presort="d,`e ` desc", algo="EvEN")
    assert p.partition_by == ["a ", "b", "c"] and p.num_partitions == "5"
    assert dict(p.presort) == {"d": True, "e ": False} and p.algo == "even"
    p = PartitionSpec(partition_by=["a", "b", "c"], presort="d,e desc", algo="EvEN",
                      num_partitions="ROWCOUNT*3", row_limit=4, size_limit="5k")
    p2 = PartitionSpec(p)
    assert p2.jsondict == p.jsondict and p2.presort_expr == "d ASC,e DESC"
    assert p.get_num_partitions(**{KEYWORD_ROWCOUNT: lambda: 7}) == 21
    assert PartitionSpec("per_row") == PartitionSpec(num="ROWCOUNT", algo="even")
    assert PartitionSpec(by="abc") == PartitionSpec(by=["abc"]) == PartitionSpec("abc")
    assert PartitionSpec(["abc", "def"]) == PartitionSpec(by=["abc", "def"]) == PartitionSpec(("abc", "def"))
    assert PartitionSpec(4) == PartitionSpec(num=4)
    raises(SyntaxError, lambda: PartitionSpec(partition_by=["a", "b", "c"], presort="a asc,e desc"))
    raises(SyntaxError, lambda: PartitionSpec(partition_by=["a", "b", "b"]))
    raises(SyntaxError, lambda: PartitionSpec(partition_by=123))
    raises(TypeError, lambda: PartitionSpec(1.1))
    raises(SyntaxError, lambda: PartitionSpec(presort="a xsc,e desc"))
    raises(SyntaxError, lambda: PartitionSpec(presort="a asc,a desc"))
    raises(SyntaxError, lambda: PartitionSpec(presort=[("a", "asc"), "b"]))
    p = PartitionSpec(dict(partition_by=["a"], presort="d asc,e desc"))
    sch = Schema("a:int,b:int,d:int,e:int")
    assert dict(p.get_sorts(sch)) == dict(a=True, d=True, e=False)
    assert dict(p.get_sorts(sch, with_partition_keys=False)) == dict(d=True, e=False)
    assert PartitionSpec(dict(partition_by=["e", "a"])).get_key_schema(sch) == "e:int,a:int"
    a = PartitionSpec(by=["a", "b"])
    b = PartitionSpec(a, by=["a"], num=2)
    assert a.partition_by == ["a", "b"] and b.partition_by == ["a"] and b.num_partitions == "2"
    with raises(KeyError):
        p.get_sorts(Schema("x:int"))


def test_partition_spec_determinism():
    """The id properties tests/fugue/collections/test_partition.py:242-253 asserts (there through
    triad's ``to_uuid``, which calls ``__uuid__``)."""
    uid = lambda spec: spec.__uuid__()  # noqa: E731
    assert uid(PartitionSpec(num=0)) == uid(PartitionSpec())
    assert uid(PartitionSpec(by=["a"], num=2)) == uid(PartitionSpec(num="2", by=["a"]))
    assert uid(PartitionSpec(by=["a", "b"])) != uid(PartitionSpec(by=["b", "a"]))
    assert uid(PartitionSpec(by=["a"], presort="b")) != uid(PartitionSpec(by=["a"], presort="b desc"))
    assert uid(PartitionSpec(by=["a"], algo="hash")) != uid(PartitionSpec(by=["a"], algo="even"))
    assert uid(PartitionSpec(PartitionSpec(by=["a"], num=3))) == uid(PartitionSpec(by=["a"], num=3))


def test_presort_forms_and_spec_equality():
    """Presort given as text, pairs, bare names or a mix; quoted names; specs compare by meaning
    (tests/fugue/collections/test_partition.py:20-56, 170-212)."""
    od = OrderedDict
    assert parse_presort_exp("DESC DESC, ASC ASC") == od([("DESC", False), ("ASC", True)])
    assert parse_presort_exp("`` desc, `a b` asc, ````, `中国`") == od([("", False), ("a b", True), ("`", True),
                                                                      ("中国", True)])
    assert parse_presort_exp([("", False), ("a b", True), "中国"]) == od([("", False), ("a b", True), ("中国", True)])
    same = [PartitionSpec(by=["a"], presort=p) for p in
            ("b DESC, c", [("b", False), ("c", True)], [("b", False), "c"], od([("b", False), ("c", True)]))]
    assert all(x.presort == same[0].presort and x == same[0] for x in same)
    other = PartitionSpec(by=["a"], presort="c,b DESC")
    assert other.presort != same[0].presort and other != same[0]
    assert PartitionSpec(other, presort=same[0].presort) == same[0]          # override while copying
    assert len(PartitionSpec(other, presort=[]).presort) == 0
    assert PartitionSpec(by=["a"], presort=["b", "c"]) == dict(presort="b asc, c", by=["a"])
    assert PartitionSpec(num=10, by=["a"], presort=["b", "c"]) != PartitionSpec(num=10, by=["a"], presort=["c", "b"])
    for bad in ("a b asc,a desc", [("a",), ("b")], ["a", ["b", True]]):
        with raises(SyntaxError):
            PartitionSpec(presort=bad)


def test_num_partitions_expressions():
    """tests/fugue/collections/test_partition.py:228-241."""
    by = dict(partition_by=["b", "a"])
    assert PartitionSpec(by).get_num_partitions() == 0
    assert PartitionSpec(dict(by, num=123)).get_num_partitions() == 123
    p = PartitionSpec(dict(by, num="(x + Y) * 2"))
    assert p.get_num_partitions(x=lambda: 1, Y=lambda: 2) == 6
    with raises(Exception):
        p.get_num_partitions(x=lambda: 1)
    p = PartitionSpec(dict(by, num="min(ROWCOUNT,CONCURRENCY)"))
    assert p.get_num_partitions(**{KEYWORD_ROWCOUNT: lambda: 100, "CONCURRENCY": lambda: 90}) == 90
    with raises(Exception):
        PartitionSpec(num="__import__('os').getpid()").get_num_partitions()   # no builtins in the expression


def test_partition_cursor():
    # tests/fugue/collections/test_partition.py (test_partition_cursor)
    p = PartitionSpec(dict(partition_by=["b", "a"]))
    s = Schema("a:int,b:int,c:int,d:int")
    c = p.get_cursor(s, 2)
    pt = c.row_schema.extract(p.partition_by)
    assert pt == "b:int,a:int" and c.key_schema == "b:int,a:int"
    c.set([1, 2, 2, 2], 5, 6)
    assert [2, 1] == c.key_value_array
    assert dict(a=1, b=2) == c.key_value_dict
    assert 2 == c["c"] and [1, 2, 2, 2] == c.row
    assert 5 == c.partition_no and 2 == c.physical_partition_no and 6 == c.slice_no
    c.set(lambda: [3, 4, 5, 6], 7, 0)  # lazily evaluated first row
    assert c.key_value_array == [4, 3] and c.partition_no == 7


def test_local_dataframes():
    df = ArrayDataFrame([[1, 2.0], [None, 3.5]], "a:long,b:double")
    assert df.is_local and df.is_bounded and df.count() == 2 and not df.empty
    assert df.as_array() == [[1, 2.0], [None, 3.5]]
    assert df.peek_array() == [1, 2.0] and df.peek_dict() == dict(a=1, b=2.0)
    assert df[["b"]].schema == "b:double"
    assert df.rename({"a": "x"}).schema == "x:long,b:double"
    assert df.as_arrow().schema == df.schema.pa_schema
    p = PandasDataFrame(pd.DataFrame({"a": [1, 2], "b": ["x", None]}), "a:int,b:str")
    assert p.as_array() == [[1, "x"], [2, None]]
    assert ArrowDataFrame(None, "a:int").empty
    assert df_eq(df, [[None, 3.5], [1, 2.0]], "a:long,b:double", throw=True)
    assert not df_eq(df, [[None, 3.5], [1, 2.1]], "a:long,b:double")
    assert not df_eq(df, [[None, 3.5], [1, 2.0]], "a:long,c:double")
    assert df_eq(df, [[None, 3.5], [1, 2.0 + 1e-10]], "a:long,b:double", throw=True)


def test_join_schemas():
    """Key schema / output schema rule of every join type (fugue/dataframe/utils.py:152-226; cases of
    tests/fugue/dataframe/test_utils.py:55-88)."""
    from fugue_b200.join import get_join_schemas

    a, b, c = (ArrayDataFrame([], s) for s in ("a:int,b:int", "c:int", "d:str,a:int"))
    assert get_join_schemas(a, b, how="cross", on=[]) == ("", "a:int,b:int,c:int")
    for how, on in (("inner", ["a"]), ("inner", []), ("Left_Outer", None)):          # keys given or inferred
        assert get_join_schemas(a, c, how=how, on=on) == ("a:int", "a:int,b:int,d:str")
    for how in ("SEMI", "LEFT_Semi", "Anti", "left_Anti"):                             # left columns only
        assert get_join_schemas(c, a, how=how, on=["a"]) == ("a:int", "d:str,a:int")
    wide1, wide2 = ArrayDataFrame([], "a:int,b:int,c:int"), ArrayDataFrame([], "c:int,b:int,x:int")
    assert get_join_schemas(wide1, wide2, how="inner", on=["c", "b"]) == ("b:int,c:int", "a:int,b:int,c:int,x:int")
    for exc, l, r, how, on in [
        (Exception, a, b, None, []), (ValueError, a, b, "x", []), (ValueError, a, c, "outer", ["a"]),
        (SchemaError, a, b, "CROSS", ["a"]), (SchemaError, a, c, "CROSS", ["a"]), (SchemaError, a, c, "CROSS", []),
        (SchemaError, a, b, "inner", ["a"]), (SchemaError, wide1, wide2, "inner", ["a"]),
        (SchemaError, wide1, wide2, "inner", ["c"]), (SchemaError, wide1, wide2, "full_outer", ["b"]),  # b, c common
    ]:
        with raises(exc):
            get_join_schemas(l, r, how=how, on=on)
