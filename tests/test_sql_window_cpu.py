"""Explicit window nodes (``over(partition_by=.., order_by=..)``) and the SQL ``OVER`` / ``QUALIFY`` grammar on CPU:
the nodes the parser builds, SQL's default frame, every rejection (before any device work), the fingerprints that
keep explicit and bare nodes apart, the GROUP BY plan of a window over aggregates, and print -> parse as a fixed
point."""
import datetime
import random

import pytest

from fugue_b200.colmap import ColumnMap
from fugue_b200.column import (Kind, SelectColumns, all_cols, col, functions as f, has_bare_window, is_explicit,
                               lit, to_sql)
from fugue_b200.sql import _parse_select


def _item(text: str):
    st = _parse_select(text, "FROM t", "SELECT " + text + " FROM t")
    assert len(st.columns) == 1
    return st.columns[0]


def _same(a, b) -> bool:
    return a.fingerprint() == b.fingerprint()


@pytest.mark.parametrize("text,node", [
    ("SUM(v) OVER (PARTITION BY k) AS s", f.sum(col("v")).over(partition_by=["k"]).alias("s")),
    ("SUM(v) OVER () AS s", f.sum(col("v")).over(partition_by=[]).alias("s")),
    ("COUNT(*) OVER (PARTITION BY k, j) AS c", f.count(all_cols()).over(partition_by=["k", "j"]).alias("c")),
    ("AVG(v) OVER (PARTITION BY k ORDER BY t ROWS BETWEEN 6 PRECEDING AND CURRENT ROW) AS m",
     f.avg(col("v")).over(rows=(-6, 0), partition_by=["k"], order_by=["t"]).alias("m")),
    ("MIN(v) OVER (ORDER BY t DESC ROWS BETWEEN 2 FOLLOWING AND UNBOUNDED FOLLOWING) AS m",
     f.min(col("v")).over(rows=(2, None), partition_by=[], order_by=[("t", False)]).alias("m")),
    ("MAX(v) OVER (ORDER BY t ROWS 3 PRECEDING) AS m",
     f.max(col("v")).over(rows=(-3, 0), order_by=["t"]).alias("m")),
    ("SUM(v) OVER (ORDER BY t ROWS UNBOUNDED PRECEDING) AS m",
     f.sum(col("v")).over(running=True, order_by=["t"]).alias("m")),
    ("SUM(v) OVER (PARTITION BY k ORDER BY t RANGE BETWEEN 5 PRECEDING AND 2 FOLLOWING) AS r",
     f.sum(col("v")).over(range=(-5, 2), partition_by=["k"], order_by=["t"]).alias("r")),
    ("SUM(v) OVER (ORDER BY d RANGE BETWEEN INTERVAL '7' DAY PRECEDING AND CURRENT ROW) AS r",
     f.sum(col("v")).over(range=(-datetime.timedelta(days=7), 0), order_by=["d"]).alias("r")),
    ("SUM(v) OVER (ORDER BY d RANGE INTERVAL '0 12:00:00' DAY TO SECOND PRECEDING) AS r",
     f.sum(col("v")).over(range=(-datetime.timedelta(hours=12), 0), order_by=["d"]).alias("r")),
    ("ROW_NUMBER() OVER (PARTITION BY k ORDER BY ts DESC NULLS LAST) AS rn",
     f.row_number().over(partition_by=["k"], order_by=[("ts", False)]).alias("rn")),
    ("RANK() OVER (ORDER BY t) AS r", f.rank().over(order_by=["t"]).alias("r")),
    ("DENSE_RANK() OVER (PARTITION BY k ORDER BY t ASC) AS r",
     f.dense_rank().over(partition_by=["k"], order_by=["t"]).alias("r")),
    ("LAG(v) OVER (PARTITION BY k ORDER BY t) AS l", f.lag(col("v")).over(partition_by=["k"], order_by=["t"]).alias("l")),
    ("LEAD(v, 2, -1) OVER (ORDER BY t) AS l", f.lead(col("v"), 2, -1).over(order_by=["t"]).alias("l")),
    ("PERCENTILE_DISC(0.25) WITHIN GROUP (ORDER BY v) OVER (PARTITION BY k) AS p",
     f.percentile_disc(col("v"), 0.25).over(partition_by=["k"]).alias("p")),
    ("SUM(v) OVER (PARTITION BY k % 4 ORDER BY t + 1 DESC, j) AS s",
     f.sum(col("v")).over(range=(None, 0), partition_by=[col("k") % 4], order_by=[(col("t") + 1, False), "j"]).alias("s")),
])
def test_every_over_form_gives_its_node(text, node):
    got = _item(text)
    assert is_explicit(got) and not has_bare_window(got)
    assert _same(got, node), (to_sql(got), to_sql(node))


def test_default_frame_is_sql_s():
    # with ORDER BY: RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW, which includes the current row's peers
    assert _item("SUM(v) OVER (PARTITION BY k ORDER BY t) AS s").kwargs["range"] == (None, 0)
    # without ORDER BY: the whole partition
    assert _item("SUM(v) OVER (PARTITION BY k) AS s").kwargs["running"] is False
    assert _item("SUM(v) OVER (ORDER BY t ROWS BETWEEN UNBOUNDED PRECEDING AND UNBOUNDED FOLLOWING) AS s"
                 ).kwargs["running"] is False
    # the builders keep their own default (the whole partition) for explicit nodes too
    assert f.sum(col("v")).over(order_by=["t"]).kwargs["running"] is False
    # the variance family has no RANGE frame, so its SQL default is refused, with the running form suggested
    with pytest.raises(NotImplementedError, match="ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW"):
        _item("STDDEV(v) OVER (PARTITION BY k ORDER BY t) AS s")
    assert _item("STDDEV(v) OVER (PARTITION BY k ORDER BY t ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW) AS s"
                 ).kwargs["running"] is True
    assert _item("STDDEV(v) OVER (PARTITION BY k) AS s").kwargs["running"] is False


@pytest.mark.parametrize("text,exc", [
    ("SUM(v) OVER (ORDER BY t GROUPS BETWEEN 1 PRECEDING AND CURRENT ROW) AS s", NotImplementedError),
    ("SUM(v) OVER (ORDER BY t ROWS 1 PRECEDING EXCLUDE CURRENT ROW) AS s", NotImplementedError),
    ("SUM(v) OVER w AS s", NotImplementedError),
    ("SUM(v) OVER (ORDER BY t NULLS FIRST) AS s", NotImplementedError),
    ("SUM(v) OVER (ORDER BY t DESC NULLS FIRST) AS s", NotImplementedError),
    ("ROW_NUMBER() AS rn", NotImplementedError),
    ("RANK() AS r", NotImplementedError),
    ("DENSE_RANK() AS r", NotImplementedError),
    ("LAG(v) AS l", NotImplementedError),
    ("LEAD(v, 1) AS l", NotImplementedError),
    ("SUM(ROW_NUMBER() OVER (ORDER BY t)) OVER () AS s", ValueError),
    ("SUM(ROW_NUMBER() OVER (ORDER BY t)) AS s", ValueError),
    ("SUM(v) OVER (PARTITION BY ROW_NUMBER() OVER (ORDER BY t)) AS s", ValueError),
    ("SUM(v) OVER (ORDER BY RANK() OVER (ORDER BY t)) AS s", ValueError),
    ("ROW_NUMBER() OVER (ORDER BY t ROWS 1 PRECEDING) AS s", ValueError),
    ("PERCENTILE_CONT(0.5) WITHIN GROUP (ORDER BY v) OVER (ORDER BY t) AS p", ValueError),
    ("SUM(v) OVER (ORDER BY t, j RANGE BETWEEN 1 PRECEDING AND CURRENT ROW) AS s", ValueError),
    ("LAG(v, j) OVER (ORDER BY t) AS l", ValueError),
    ("SUM(v) OVER (ORDER BY t ROWS BETWEEN UNBOUNDED FOLLOWING AND CURRENT ROW) AS s", ValueError),
])
def test_rejections_of_the_select_list(text, exc):
    with pytest.raises(exc):
        _item(text)


@pytest.mark.parametrize("rest", [
    "FROM t WHERE ROW_NUMBER() OVER (ORDER BY t) > 1",
    "FROM t GROUP BY RANK() OVER (ORDER BY t)",
    "FROM t GROUP BY k HAVING SUM(SUM(v)) OVER () > 1",
])
def test_windows_outside_the_select_list_and_qualify(rest):
    with pytest.raises(ValueError):
        _parse_select("k, SUM(v) AS s", rest, "SELECT k, SUM(v) AS s " + rest)


def test_named_windows_are_refused():
    with pytest.raises(NotImplementedError):
        _parse_select("k", "FROM t WINDOW w AS (ORDER BY t)", "SELECT k FROM t WINDOW w AS (ORDER BY t)")


def test_qualify_sits_between_having_and_order_by():
    st = _parse_select("k, v, ROW_NUMBER() OVER (PARTITION BY k ORDER BY t DESC) AS rn",
                       "FROM t WHERE v > 0 QUALIFY rn = 1 ORDER BY k LIMIT 5", "")
    assert st.qualify is not None and st.qualify.kind == Kind.BINARY and st.order_by == [("k", True)]
    assert st.limit == 5 and st.where is not None
    st = _parse_select("k, SUM(v) AS s", "FROM t GROUP BY k HAVING SUM(v) > 0 "
                       "QUALIFY RANK() OVER (ORDER BY SUM(v) DESC) <= 3", "")
    assert st.having is not None and is_explicit(st.qualify.args[0])


def test_builder_rules_for_explicit_nodes():
    with pytest.raises(ValueError):  # a spec, or nothing: over() alone still is no ROW_NUMBER form
        f.row_number().over()
    assert is_explicit(f.row_number().over(partition_by=[]))
    with pytest.raises(ValueError):
        f.lag(col("v")).over(rows=(-1, 0), order_by=["t"])
    with pytest.raises(ValueError):
        f.median(col("v")).over(order_by=["t"])
    with pytest.raises(ValueError):
        f.median(col("v")).over(running=True, partition_by=["k"])
    with pytest.raises(NotImplementedError):  # the variance family keeps its frame rule
        f.var_samp(col("v")).over(range=(None, 0), order_by=["t"])
    with pytest.raises(NotImplementedError):
        f.corr(col("x"), col("y")).over(rows=(-1, 1), order_by=["t"])
    with pytest.raises(ValueError):
        f.sum(col("v")).over(partition_by="k")  # a list, not a name
    with pytest.raises(ValueError):
        f.sum(col("v")).over(order_by=[("t", "desc")])
    with pytest.raises(ValueError):
        f.sum(col("v")).over(partition_by=[all_cols()])
    with pytest.raises(ValueError):
        f.sum(col("v")).over(partition_by=[f.row_number().over(order_by=["t"])])
    with pytest.raises(ValueError):  # a bare window never reads an aggregation; an explicit one may
        f.sum(f.sum(col("v"))).over()
    assert is_explicit(f.sum(f.sum(col("v"))).over(partition_by=[]))


def test_column_map_rejects_explicit_nodes_and_select_rejects_bare_ones():
    with pytest.raises(ValueError):
        ColumnMap("k", f.sum(col("v")).over(partition_by=["k"]).alias("s"))
    with pytest.raises(ValueError):
        ColumnMap("k", (col("v") / f.sum(col("v")).over(partition_by=[])).alias("share"))
    ColumnMap("k", f.sum(col("v")).over().alias("s"))  # a bare node: the PartitionSpec's partition
    assert has_bare_window(col("v") - f.lag(col("v")))
    assert not has_bare_window(col("v") - f.lag(col("v")).over(order_by=["t"]))


def test_fingerprints_separate_explicit_and_bare_nodes():
    bare = f.sum(col("v")).over()
    assert not _same(bare, f.sum(col("v")).over(partition_by=[]))
    assert not _same(f.sum(col("v")).over(partition_by=["k"]), f.sum(col("v")).over(partition_by=["j"]))
    assert not _same(f.sum(col("v")).over(order_by=["t"]), f.sum(col("v")).over(order_by=[("t", False)]))
    assert _same(f.sum(col("v")).over(partition_by=[]), f.sum(col("v")).over(order_by=[]))  # both OVER ()
    assert _same(f.sum(col("v")).over(partition_by=["k"]), f.sum(col("v")).over(partition_by=[col("k").alias("x")]))
    assert _same(f.rank().over(order_by=["t"]), f.rank().over(order_by=[("t", True)]))
    from fugue_b200.colmap import _collect_windows

    out = {}
    _collect_windows((f.sum(col("v")).over(partition_by=["k"]) + f.sum(col("v")).over(partition_by=["k"]).alias("y")
                      + f.sum(col("v")).over()).alias("z"), out)
    assert len(out) == 2  # equal explicit nodes once, never merged with the bare one
    # bare nodes print as they always did
    assert str(f.sum(col("v")).over(running=True)) == "SUM(v) OVER (ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW)"
    assert str(f.sum(col("v")).over(rows=(-6, 0), partition_by=["k"], order_by=[("t", False)])) == \
        "SUM(v) OVER (PARTITION BY k ORDER BY t DESC ROWS BETWEEN 6 PRECEDING AND CURRENT ROW)"


def test_group_by_windows_are_aggregating_and_never_group_keys():
    """The two-stage plan: a window that reads aggregates makes the SELECT aggregating, it is not a group key,
    and its aggregates (arguments, PARTITION BY, ORDER BY) are found as outputs of the group-by stage and
    rewritten to read them."""
    from fugue_b200.expr import find_aggs, rewrite

    rank = f.rank().over(order_by=[(f.sum(col("v")), False)]).alias("r")
    share = (f.sum(col("v")) / f.sum(f.sum(col("v"))).over(partition_by=[col("g")])).alias("share")
    sel = SelectColumns(col("k"), col("g"), rank, share)
    assert sel.has_agg and [to_sql(k) for k in sel.group_keys] == ["k", "g"]
    found = []
    for c in sel.all_cols:
        find_aggs(c, found)
    assert len({a.fingerprint() for a in found}) == 1 and to_sql(found[0]) == "SUM(v)"
    hidden = {found[0].fingerprint(): col("__fb_a0")}
    out = [rewrite(c, lambda e: hidden.get(e.alias("").cast(None).fingerprint())) for c in (rank, share)]
    assert to_sql(out[0]) == "RANK() OVER (ORDER BY __fb_a0 DESC) AS r"
    assert to_sql(out[1]) == "__fb_a0/SUM(__fb_a0) OVER (PARTITION BY g) AS share"
    # a window over the groups without an aggregation is not a key either
    sel = SelectColumns(col("k"), f.sum(col("v")).alias("s"), f.row_number().over(order_by=["k"]).alias("rn"))
    assert [to_sql(k) for k in sel.group_keys] == ["k"]


def _random_tree(rng: random.Random):
    def scalar(depth: int):
        r = rng.random()
        if depth > 1 or r < 0.5:
            return col(rng.choice(["a", "b", "k", "t"]))
        if r < 0.7:
            return scalar(depth + 1) + rng.randint(1, 9)
        if r < 0.85:
            return scalar(depth + 1) * scalar(depth + 1)
        return f.coalesce(scalar(depth + 1), rng.randint(0, 3))

    pb = [scalar(1) for _ in range(rng.randint(0, 2))]
    ob = [(scalar(1), rng.random() < 0.5) for _ in range(rng.randint(0, 2))]
    head = rng.choice(["SUM", "COUNT", "AVG", "MIN", "MAX", "ROW_NUMBER", "RANK", "DENSE_RANK", "LAG", "LEAD",
                       "PERCENTILE_CONT", "STDDEV"])
    if head in ("ROW_NUMBER", "RANK", "DENSE_RANK"):
        w = getattr(f, head.lower())().over(partition_by=pb, order_by=ob)
    elif head in ("LAG", "LEAD"):
        w = getattr(f, head.lower())(scalar(1), rng.randint(0, 3), rng.choice([None, 0, 7])).over(
            partition_by=pb, order_by=ob)
    elif head == "PERCENTILE_CONT":
        w = f.percentile_cont(scalar(1), rng.choice([0, 0.25, 0.5, 1])).over(partition_by=pb)
    else:
        frames = [{}, {"running": True}] if head == "STDDEV" else \
            [{}, {"running": True}, {"rows": (-rng.randint(0, 9), rng.randint(0, 9))}, {"rows": (None, 2)},
             {"rows": (-1, None)}] + ([{"range": (None, 0)}, {"range": (-rng.randint(1, 9), 0)},
                                        {"range": (0, None)}] if len(ob) == 1 else [])
        arg = all_cols() if head == "COUNT" and rng.random() < 0.3 else scalar(1)
        w = getattr(f, head.lower())(arg).over(partition_by=pb, order_by=ob, **rng.choice(frames))
    r = rng.random()
    e = w if r < 0.5 else (col("a") - w if r < 0.75 else w * lit(2))
    return e.alias("x")


def test_print_then_parse_is_a_fixed_point_on_random_trees():
    rng = random.Random(7)
    for _ in range(400):
        e = _random_tree(rng)
        text = to_sql(e)
        back = _item(text)
        assert to_sql(back) == text
        assert _same(back, e), text


def test_raw_sql_takes_explicit_expressions_as_pieces_and_refuses_bare_ones():
    from fugue_b200 import api as fa
    from fugue_b200.execution_engine import B200ExecutionEngine

    seen = []

    class _SQL:
        @staticmethod
        def select(dfs, statement):
            seen.append(statement.construct())
            raise RuntimeError("stop")

    E = type("E", (B200ExecutionEngine,), {"sql_engine": property(lambda self: _SQL())})
    e2 = E.__new__(E)
    e2.to_df = lambda df, schema=None: df  # type: ignore
    with pytest.raises(RuntimeError):
        fa.raw_sql("SELECT k,", f.sum(col("v")).over(partition_by=["k"]).alias("s"), "FROM t", engine=e2)
    assert seen == ["SELECT k, SUM(v) OVER (PARTITION BY k) AS s FROM t"]
    with pytest.raises(NotImplementedError):
        fa.raw_sql("SELECT k,", f.sum(col("v")).over().alias("s"), "FROM t", engine=e2)


def test_engines_refuse_before_touching_the_device():
    from fugue_b200.dist import DistributedB200Engine
    from fugue_b200.execution_engine import B200ExecutionEngine

    rn = f.row_number().over(partition_by=["k"], order_by=["t"])
    eng = B200ExecutionEngine.__new__(B200ExecutionEngine)
    eng.to_df = lambda df, schema=None: (_ for _ in ()).throw(AssertionError("must reject first"))  # type: ignore
    with pytest.raises(ValueError):  # a window in WHERE / HAVING
        eng.select(None, SelectColumns(col("k")), where=rn > 1)
    with pytest.raises(ValueError):
        eng.select(None, SelectColumns(col("k"), f.sum(col("v")).alias("s")), having=rn > 1)
    with pytest.raises(NotImplementedError):  # a bare node in select / assign / filter
        eng.select(None, SelectColumns(col("k"), f.row_number().alias("rn")))
    dist = DistributedB200Engine.__new__(DistributedB200Engine)
    dist._world = 2
    dist.to_df = eng.to_df  # type: ignore
    assert dist.get_current_parallelism() == 2
    for call in (lambda: dist.select(None, SelectColumns(col("k"), rn.alias("rn"))),
                 lambda: dist.assign(None, [rn.alias("rn")]),
                 lambda: dist.filter(None, rn == 1)):
        with pytest.raises(NotImplementedError, match="multi-GPU"):
            call()
