"""Value frames of window nodes (``over(range=(start, end))``, fugue_b200/column.py): builders, every malformed
frame, SQL text and fingerprints, and that the existing ROWS / running / whole-partition nodes keep theirs."""
import datetime

import pytest

from fugue_b200.column import all_cols, col, functions as f, to_sql

TD = datetime.timedelta


def test_builders_store_the_frame():
    for a in [f.sum(col("v")), f.count(col("v")), f.count(all_cols()), f.avg(col("v")), f.min(col("v")),
              f.max(col("v")), f.first(col("v")), f.last(col("v"))]:
        for rng in [(-7, 0), (-0.5, 0.5), (TD(days=-7), 0), (None, 0), (0, 0), (0, None), (1, 3), (None, -2)]:
            e = a.over(range=rng)
            assert e.kwargs == {"range": rng}
            assert e.func == a.func


@pytest.mark.parametrize("bad", [(1,), (1, 2, 3), [-1, 0], "(-1, 0)", -1, None.__class__])
def test_not_a_pair(bad):
    with pytest.raises(ValueError):
        f.sum(col("v")).over(range=bad)


@pytest.mark.parametrize("bad", [(True, 0), (0, False), (float("nan"), 0), (0, float("inf")), (-float("inf"), 0),
                                 ("1", 2), (1, 2j), (0, datetime.date(2020, 1, 1))])
def test_bad_bounds(bad):
    with pytest.raises(ValueError):
        f.sum(col("v")).over(range=bad)


def test_start_after_end_and_combinations():
    for bad in [(1, 0), (0.5, 0.25), (TD(days=1), TD(hours=1)), (TD(seconds=1), 0), (0, TD(microseconds=-1))]:
        with pytest.raises(ValueError):
            f.sum(col("v")).over(range=bad)
    with pytest.raises(ValueError):
        f.sum(col("v")).over(range=(TD(days=-1), 3))  # a timedelta and a non-zero number
    with pytest.raises(ValueError):
        f.sum(col("v")).over(running=True, range=(-1, 0))
    with pytest.raises(ValueError):
        f.sum(col("v")).over(rows=(-1, 0), range=(-1, 0))
    with pytest.raises(ValueError):
        f.sum(col("v")).over(running=True, range=(None, None))
    with pytest.raises(ValueError):
        f.count_distinct(col("v")).over(range=(-1, 0))
    f.sum(col("v")).over(range=(-2**63, 2**63 - 1))
    f.sum(col("v")).over(range=(-1e300, 1e300))
    f.sum(col("v")).over(range=(TD(days=-3), TD(days=3)))


def test_whole_partition_collapses_and_nothing_else_does():
    a = f.sum(col("v")).alias("s")
    assert a.over(range=(None, None)).fingerprint() == a.over().fingerprint()
    assert str(a.over(range=(None, None))) == str(a.over())
    assert a.over(range=(None, 0)).fingerprint() != a.over(running=True).fingerprint()
    assert a.over(range=(None, 0)).fingerprint() != a.over(rows=(None, 0)).fingerprint()
    assert a.over(range=(0, None)).fingerprint() != a.over(rows=(0, None)).fingerprint()
    assert a.over(range=(-1, 0)).fingerprint() != a.over(rows=(-1, 0)).fingerprint()
    assert a.over(range=(-1, 0)).fingerprint() == a.over(range=(-1, 0)).fingerprint()
    assert a.over(range=(-1, 0)).fingerprint() != a.over(range=(-1.0, 0)).fingerprint()  # the offset's type is kept
    # a zero bound of any type is CURRENT ROW, stored as the int 0
    assert a.over(range=(-0.0, TD(0))).kwargs == {"range": (0, 0)}
    assert a.over(range=(-0.0, TD(0))).fingerprint() == a.over(range=(0, 0)).fingerprint()


def test_text():
    assert str(f.avg(col("v")).over(range=(-7, 0))) == "AVG(v) OVER (RANGE BETWEEN 7 PRECEDING AND CURRENT ROW)"
    assert str(f.sum(col("v")).over(range=(None, 0))) == \
        "SUM(v) OVER (RANGE BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW)"
    assert str(f.sum(col("v")).over(range=(0, 0))) == "SUM(v) OVER (RANGE BETWEEN CURRENT ROW AND CURRENT ROW)"
    assert str(f.max(col("v")).over(range=(-0.5, 0.5))) == \
        "MAX(v) OVER (RANGE BETWEEN 0.5 PRECEDING AND 0.5 FOLLOWING)"
    assert str(f.count(all_cols()).over(range=(1, None))) == \
        "COUNT(*) OVER (RANGE BETWEEN 1 FOLLOWING AND UNBOUNDED FOLLOWING)"
    assert str(f.avg(col("v")).over(range=(TD(days=-7), 0)).alias("a7")) == \
        "AVG(v) OVER (RANGE BETWEEN INTERVAL '7' DAY PRECEDING AND CURRENT ROW) AS a7"
    assert str(f.sum(col("v")).over(range=(TD(hours=-36), TD(seconds=30, microseconds=5)))) == \
        "SUM(v) OVER (RANGE BETWEEN INTERVAL '1 12:00:00' DAY TO SECOND PRECEDING AND " \
        "INTERVAL '0 00:00:30.000005' DAY TO SECOND FOLLOWING)"
    assert to_sql((col("v") - f.avg(col("v")).over(range=(-6, 0))).alias("d")) == \
        "v-AVG(v) OVER (RANGE BETWEEN 6 PRECEDING AND CURRENT ROW) AS d"


def test_types_and_aliases_follow_the_rows_form():
    import pyarrow as pa

    from fugue_b200.schema import Schema

    sch = Schema("i:int,x:double,s:str")
    for e in [f.sum(col("i")), f.sum(col("x")), f.avg(col("i")), f.count(col("s")), f.min(col("i")),
              f.max(col("x")), f.first(col("s")), f.last(col("i"))]:
        w = e.over(range=(-3, 1))
        assert w.infer_type(sch) == e.over(rows=(-3, 1)).infer_type(sch)
        assert w.infer_alias().output_name == e.over(rows=(-3, 1)).infer_alias().output_name
    assert f.sum(col("i")).over(range=(-1, 1)).infer_type(sch) == pa.int64()


def test_rows_and_running_nodes_are_unchanged():
    # the text and fingerprints pinned before range frames existed
    assert str(f.sum(col("v")).over(rows=(-6, 0))) == "SUM(v) OVER (ROWS BETWEEN 6 PRECEDING AND CURRENT ROW)"
    assert str(f.sum(col("v")).over(running=True)) == \
        "SUM(v) OVER (ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW)"
    assert str(f.sum(col("v")).over()) == "SUM(v) OVER ()"
    assert f.sum(col("v")).over(rows=(-6, 0)).kwargs == {"rows": (-6, 0)}
    assert f.sum(col("v")).over(running=True).kwargs == {"running": True}
    assert f.sum(col("v")).over().kwargs == {"running": False}
    assert f.sum(col("v")).over(rows=(None, 0)).fingerprint() == f.sum(col("v")).over(running=True).fingerprint()
    assert f.sum(col("v")).over(rows=(-6, 0)).fingerprint() == "26ecb00582f0ba337f2423c9579e5a9d2d95e6db"
    assert f.sum(col("v")).over(running=True).fingerprint() == "1fb58254ddb00110983f365071ff43628bf615b7"
    assert f.sum(col("v")).over().fingerprint() == "426352a42c68da5af89ad5b3210ffc8339ac98af"
    m = f.avg(col("x")).over(rows=(-2, 3)).alias("m")
    assert str(m) == "AVG(x) OVER (ROWS BETWEEN 2 PRECEDING AND 3 FOLLOWING) AS m"
    assert m.fingerprint() == "99cbed2c310685798bd43acc7de5b9af35f24d5a"
