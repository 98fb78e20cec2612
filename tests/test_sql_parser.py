"""The SELECT parser of B200SQLEngine (host logic): SQL text -> column expressions (fugue_b200.column)."""
import pytest
from pytest import raises

from fugue_b200.sql import StructuredRawSQL, _parse_select


def parse(items, rest):
    return _parse_select(items, rest, f"SELECT {items} FROM {rest}")


def test_group_by_having_order_limit():
    st = parse("key, SUM(v0) AS s, COUNT(*) AS c", "t GROUP BY key HAVING SUM(v0) >= 7 OR key = 1 ORDER BY s DESC, key LIMIT 3")
    assert [str(c) for c in st.columns] == ["key", "SUM(v0) AS s", "COUNT(*) AS c"]
    assert st.table == "t" and [str(g) for g in st.group_by] == ["key"]
    assert str(st.having) == "|(>=(SUM(v0),7),==(key,1))"
    assert st.order_by == [("s", False), ("key", True)] and st.limit == 3 and not st.distinct


def test_expressions_and_aliases():
    st = parse("DISTINCT a.key k, (v0 + 1.5e2) * -2 AS w, CAST(v1 AS long) AS q, COALESCE(x, 0) c, 'it''s' AS s, "
               "`odd name`, COUNT(*), MAX(v0), COUNT(DISTINCT key) AS d",
               "`my table` AS a WHERE NOT (key > 3 AND v0 IS NOT NULL) OR key IN (1,2) OR v1 NOT BETWEEN 0 AND 1")
    assert st.distinct and st.table == "my table"
    assert [str(c) for c in st.columns] == [
        "key AS k", "*(+(v0,150.0),-2) AS w", "CAST(v1 AS long) AS q", "COALESCE(x,0) AS c", "'it\\'s' AS s",
        "odd name", "COUNT(*) AS count", "MAX(v0) AS v0", "COUNT(DISTINCT key) AS d"]
    assert str(st.where) == "|(|(~(&(>(key,3),NOT_NULL(v0))),|(==(key,1),==(key,2))),~(&(>=(v1,0),<=(v1,1))))"


def test_precedence():
    st = parse("a + b * c - d / 2 AS x, -a * 2 AS y, NOT a = 1 AND b <> 2 OR c AS z, a - -1 AS w", "t")
    assert [str(c) for c in st.columns] == [
        "-(+(a,*(b,c)),/(d,2)) AS x", "*(-(a),2) AS y", "|(&(~(==(a,1)),!=(b,2)),c) AS z", "-(a,-1) AS w"]


def test_rejections():
    with raises(NotImplementedError):
        parse("key", "(SELECT * FROM t)")
    with raises(NotImplementedError):
        parse("key", "t UNION SELECT key FROM u")
    with raises(NotImplementedError):
        parse("key", "t LIMIT x")
    with raises(ValueError):
        parse("key", "t WHERE SUM(v) > 1")
    with raises(NotImplementedError):
        parse("key ; DROP", "t")


def test_structured_raw_sql_pieces():
    """tests/fugue/collections/test_sql.py:34-88 (without the sqlglot transpile cases)."""
    from fugue_b200.sql import TempTableName

    def marked(sql):
        return "".join(t if not ref else "!" + t + "!" for ref, t in StructuredRawSQL.from_expr(sql)._statements)

    t1, t2 = TempTableName(), TempTableName()
    assert t1.key != t2.key and str(t1) == f"<tmpdf:{t1.key}>"
    assert marked("") == "" and marked(f"{t1}") == f"!{t1.key}!" and marked(f" {t1} ") == f" !{t1.key}! "
    assert marked(f"SELECT {t1}.* FROM {t1} NATURAL JOIN {t2} WHERE {t2}.x<1") == \
        f"SELECT !{t1.key}!.* FROM !{t1.key}! NATURAL JOIN !{t2.key}! WHERE !{t2.key}!.x<1"
    assert StructuredRawSQL.from_expr("SELECT * FROM abc", dialect="y").dialect == "y"
    with raises(SyntaxError):
        StructuredRawSQL.from_expr("SELECT * FROM <tmpdf:abc")

    pieces = [(False, "SELECT * FROM"), (True, "tb1"), (False, "NATURAL JOIN"), (True, "tb2")]
    q = StructuredRawSQL(pieces, dialect="x")
    assert q.dialect == "x" and q.construct() == "SELECT * FROM tb1 NATURAL JOIN tb2"
    assert q.construct({"tb1": "tt"}) == "SELECT * FROM tt NATURAL JOIN tb2"       # unknown names stay
    assert q.construct(lambda n: n + "_", dialect="x") == "SELECT * FROM tb1_ NATURAL JOIN tb2_"
    with raises(NotImplementedError):
        q.construct(dialect="y")                                                    # would need sqlglot
    assert StructuredRawSQL(pieces).construct(dialect="y") == q.construct()         # no source dialect: as is

    uid = lambda *a, **k: StructuredRawSQL(*a, **k).__uuid__()  # noqa: E731
    same = [(False, "SELECT * FROM"), (True, "tb1")]
    assert uid(same) == uid(list(same)) and uid(same) != uid(same, dialect="x")
    assert uid(same) != uid([(False, "SELECT * from"), (True, "tb1")])


class _FakeDF:
    """Stands in for an engine dataframe: records what the SQL engine asks of it."""

    def __init__(self, names):
        from fugue_b200.schema import Schema

        self.schema = Schema(",".join(f"{n}:long" for n in names))
        self.columns = list(names)
        self.picked = None

    def __getitem__(self, cols):
        out = _FakeDF(cols)
        out.picked = list(cols)
        return out


class _FakeEngine:
    is_distributed = False

    def __init__(self):
        self.calls = []

    def to_df(self, df):
        return df

    def select(self, df, cols, where=None, having=None):
        self.calls.append((cols, where, having))
        return _FakeDF([c.output_name for c in cols.all_cols])


def test_sql_engine_hands_select_the_right_trees():
    from fugue_b200.sql import B200SQLEngine

    eng = _FakeEngine()
    sql = B200SQLEngine(eng)
    t = _FakeDF(["key", "v0", "v1"])
    out = sql.select({"t": t}, "SELECT key, SUM(v0 * 2) AS s FROM t WHERE v1 > 0 GROUP BY key HAVING COUNT(*) > 5")
    cols, where, having = eng.calls[-1]
    assert [str(c) for c in cols.all_cols] == ["key", "SUM(*(v0,2)) AS s"] and not cols.is_distinct
    assert str(where) == ">(v1,0)" and str(having) == ">(COUNT(*),5)"
    assert out.columns == ["key", "s"]
    # a GROUP BY key that is not selected rides along as a hidden column and is dropped afterwards
    out = sql.select({"t": t}, "SELECT MAX(v0) AS m FROM t GROUP BY key, v1 + 1")
    cols, _, _ = eng.calls[-1]
    assert [str(c) for c in cols.all_cols] == ["MAX(v0) AS m", "key AS __fb_g0", "+(v1,1) AS __fb_g1"]
    assert out.picked == ["m"]
    # select-list keys must all be in GROUP BY; GROUP BY needs an aggregate
    with raises(ValueError):
        sql.select({"t": t}, "SELECT key, v1, SUM(v0) AS s FROM t GROUP BY key")
    with raises(NotImplementedError):
        sql.select({"t": t}, "SELECT key FROM t GROUP BY key")
    with raises(KeyError):
        sql.select({"t": t}, "SELECT key FROM nope")
    out = sql.select({"t": t}, "SELECT DISTINCT key k, v0 FROM t")
    assert eng.calls[-1][0].is_distinct and out.columns == ["k", "v0"]


class _JoinRecorder:
    """Records the join the SQL engine asks for: (method, left, right, keyword arguments)."""
    is_distinct = False

    def __init__(self):
        self.calls = []

    def to_df(self, df):
        return df

    def __getattr__(self, name):
        if name not in ("join", "range_join", "asof_join"):
            raise AttributeError(name)

        def method(df1, df2, **kw):
            self.calls.append((name, df1, df2, kw))
            return df1

        return method


_TA, _TB = _FakeDF(["k", "j", "v"]), _FakeDF(["k", "j", "w"])


def _join_call(rest, tables=None):
    from fugue_b200.sql import B200SQLEngine

    eng = _JoinRecorder()
    B200SQLEngine(eng).select(tables or {"a": _TA, "b": _TB}, "SELECT * FROM " + rest)
    (call,) = eng.calls
    return call


@pytest.mark.parametrize("rest,how,on", [
    ("a JOIN b ON a.k = b.k", "inner", ["k"]),
    ("a INNER JOIN b USING (k)", "inner", ["k"]),
    ("a inner join b using (k, j)", "inner", ["k", "j"]),
    ("a LEFT JOIN b ON a.k = b.k", "left_outer", ["k"]),
    ("a LEFT OUTER JOIN b ON b.k = a.k", "left_outer", ["k"]),
    ("a RIGHT JOIN b ON a.k = b.k", "right_outer", ["k"]),
    ("a RIGHT OUTER JOIN b ON a.k = b.k", "right_outer", ["k"]),
    ("a FULL JOIN b ON a.k = b.k", "full_outer", ["k"]),
    ("a FULL OUTER JOIN b ON a.k = b.k AND a.j = b.j", "full_outer", ["k", "j"]),
    ("a SEMI JOIN b ON a.k = b.k", "semi", ["k"]),
    ("a LEFT SEMI JOIN b ON a.k = b.k", "semi", ["k"]),
    ("a ANTI JOIN b USING (k)", "anti", ["k"]),
    ("a LEFT ANTI JOIN b ON a.k = b.k", "anti", ["k"]),
    ("a CROSS JOIN b", "cross", None),
    ("a AS x JOIN b AS y ON x.k = y.k", "inner", ["k"]),
    ("a x LEFT JOIN b y ON (y.k = x.k) AND (x.j = y.j)", "left_outer", ["k", "j"]),
    ("a x left\n  outer join b ON (x.k = b.k AND a.j = b.j)", "left_outer", ["k", "j"]),
    ("`a` JOIN `b` ON `a`.`k` = `b`.`k`", "inner", ["k"]),
    ("a JOIN b ON k = k", "inner", ["k"]),
    # the join texts that used to run another join
    ("a LEFT JOIN b ON a.k = b.k AND a.k = b.k", "left_outer", ["k"]),     # ran with on=['k', 'k']
    ("a LEFT JOIN b ON a.k = b.k AND b.k = a.k", "left_outer", ["k"]),
    ("a NATURAL JOIN b", "inner", None),                                     # NATURAL was read as a's alias
    ("a NATURAL LEFT JOIN b", "left_outer", None),
    ("a x NATURAL FULL OUTER JOIN b", "full_outer", None),
    # raw_sql's dataframes have generated names (_0, _1) the text cannot spell: any qualifier may stand for them
    ("_0 JOIN _1 ON orders.k = prices.k", "inner", ["k"]),
    ("_0 o LEFT JOIN _1 ON o.k = p.k", "left_outer", ["k"]),
])
def test_join_spellings(rest, how, on):
    tables = {"_0": _TA, "_1": _TB} if rest.startswith("_0") else None
    name, d1, d2, kw = _join_call(rest, tables)
    assert name == "join" and d1 is _TA and d2 is _TB and kw == dict(how=how, on=on)


@pytest.mark.parametrize("rest", [
    "a OUTER JOIN b USING (k)",             # ran an inner join: OUTER was read as a's alias
    "a CROSS JOIN b ON a.k = b.k",          # ran the cross product and dropped the ON
    "a CROSS JOIN b USING (k)",
    "a JOIN b ON a.k = a.k",                # ran an inner join on k: both operands name a
    "a x JOIN b y ON y.k = y.k",
    "a JOIN b ON z.k = q.k",                # ran an inner join on k: neither qualifier names a table
    "a x JOIN b y ON a.k = q.k",
    "a JOIN b",                             # ran a natural join; SQLite runs a cross join
    "a LEFT JOIN b",
    "a NATURAL JOIN b USING (k)",
    "a NATURAL JOIN b ON a.k = b.k",
    "a NATURAL CROSS JOIN b",
    "a JOIN b ON a.k = b.j",
    "a JOIN b ON a.k = b.k OR a.j = b.j",
    "a JOIN b ON a.k < b.k",
    "a x y JOIN b ON a.k = b.k",
])
def test_join_texts_that_must_not_run(rest):
    from fugue_b200.sql import B200SQLEngine

    eng = _JoinRecorder()
    with raises(NotImplementedError):
        B200SQLEngine(eng).select({"a": _TA, "b": _TB}, "SELECT * FROM " + rest)
    assert eng.calls == []
