"""Moving frames of window nodes (``over(rows=(start, end))``, fugue_b200/column.py) and their place in the
ColumnMap plan on CPU: builders, validation, normalisation to the running / whole-partition nodes, SQL text,
types, that a frame map is never fused, and that select / filter / assign / raw_sql still reject them."""
import os
import re

import pyarrow as pa
import pytest
import torch

from fugue_b200 import kernels as K
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import Kind, SelectColumns, all_cols, col, functions as f, has_window, is_agg, to_sql
from fugue_b200.schema import Schema
from fugue_b200.table import B200Table

AGGS = [f.sum(col("v")), f.count(col("v")), f.count(all_cols()), f.avg(col("v")), f.min(col("v")), f.max(col("v")),
        f.first(col("v")), f.last(col("v"))]


def test_every_window_aggregate_takes_a_frame():
    for a in AGGS:
        for rows in [(-6, 0), (-2, 2), (0, None), (1, 5), (None, -1), (-3, -1), (5, 7), (0, 0)]:
            e = a.over(rows=rows)
            assert e.kind == Kind.WINDOW and has_window(e) and not is_agg(e)
            assert e.kwargs == {"rows": rows} and e.head == a.head and e.args == a.args


def test_frame_validation():
    for bad in [(1,), (1, 2, 3), [-1, 0], "(-1, 0)", -1, (None,)]:
        with pytest.raises(ValueError):
            f.sum(col("v")).over(rows=bad)
    for bad in [(True, 0), (0, False), (-1.0, 0), (0, "1"), (None, 2.5)]:
        with pytest.raises(ValueError):
            f.sum(col("v")).over(rows=bad)
    with pytest.raises(ValueError):
        f.sum(col("v")).over(rows=(1, 0))
    with pytest.raises(ValueError):
        f.sum(col("v")).over(running=True, rows=(-1, 0))
    with pytest.raises(ValueError):
        f.sum(col("v")).over(running=True, rows=(None, 0))
    with pytest.raises(ValueError):  # rankings and LAG / LEAD take no frame
        f.row_number().over(rows=(-1, 0))
    with pytest.raises(ValueError):
        f.lag(col("v")).over(rows=(-1, 0))
    with pytest.raises(ValueError):
        f.count_distinct(col("v")).over(rows=(-1, 0))
    # empty frames are legal
    f.sum(col("v")).over(rows=(None, -1))
    f.sum(col("v")).over(rows=(5, 7))
    f.sum(col("v")).over(rows=(-2**63 + 1, 2**63 - 1))


def test_equal_frames_make_equal_nodes():
    for a in AGGS:
        run, whole = a.over(running=True), a.over()
        r2, w2 = a.over(rows=(None, 0)), a.over(rows=(None, None))
        assert r2.kwargs == run.kwargs == {"running": True} and w2.kwargs == whole.kwargs == {"running": False}
        assert r2.fingerprint() == run.fingerprint() and w2.fingerprint() == whole.fingerprint()
        assert str(r2) == str(run) and str(w2) == str(whole)
    assert f.sum(col("v")).over(rows=(-1, 0)).fingerprint() == f.sum(col("v")).over(rows=(-1, 0)).fingerprint()
    assert f.sum(col("v")).over(rows=(-1, 0)).fingerprint() != f.sum(col("v")).over(rows=(-2, 0)).fingerprint()
    assert f.sum(col("v")).over(rows=(0, None)).fingerprint() != f.sum(col("v")).over().fingerprint()


def test_text_forms():
    assert str(f.sum(col("v")).over(rows=(-6, 0))) == "SUM(v) OVER (ROWS BETWEEN 6 PRECEDING AND CURRENT ROW)"
    assert str(f.avg(col("v")).over(rows=(-2, 2))) == "AVG(v) OVER (ROWS BETWEEN 2 PRECEDING AND 2 FOLLOWING)"
    assert str(f.max(col("v")).over(rows=(0, None))) == \
        "MAX(v) OVER (ROWS BETWEEN CURRENT ROW AND UNBOUNDED FOLLOWING)"
    assert str(f.count(all_cols()).over(rows=(1, 5))) == "COUNT(*) OVER (ROWS BETWEEN 1 FOLLOWING AND 5 FOLLOWING)"
    assert str(f.min(col("v")).over(rows=(None, -1)).alias("m")) == \
        "MIN(v) OVER (ROWS BETWEEN UNBOUNDED PRECEDING AND 1 PRECEDING) AS m"
    assert to_sql((col("v") - f.avg(col("v")).over(rows=(-6, 0))).alias("d")) == \
        "v-AVG(v) OVER (ROWS BETWEEN 6 PRECEDING AND CURRENT ROW) AS d"
    assert to_sql(f.last(col("my v")).over(rows=(-3, -1)).cast(int)) == \
        "CAST(LAST(`my v`) OVER (ROWS BETWEEN 3 PRECEDING AND 1 PRECEDING) AS long)"


def test_alias_and_type_inference_ignore_the_frame():
    sch = Schema("k:long,i:int,v:double,s:str,d:date")
    for e in [f.sum(col("i")), f.sum(col("v")), f.avg(col("i")), f.count(col("s")), f.count(all_cols()),
              f.min(col("i")), f.max(col("v")), f.first(col("s")), f.last(col("d"))]:
        for rows in [(-6, 0), (1, 3), (None, -1), (0, None)]:
            w = e.over(rows=rows)
            assert w.infer_type(sch) == e.over().infer_type(sch)
            assert w.infer_alias().output_name == e.over().infer_alias().output_name
    assert f.sum(col("i")).over(rows=(-1, 1)).infer_type(sch) == pa.int64()
    assert f.min(col("i")).over(rows=(-1, 1)).infer_type(sch) == pa.int32()


def test_frame_maps_are_never_fused():
    t = B200Table(Schema("k:long,x:double"), [torch.arange(16, dtype=torch.int64), torch.arange(16, dtype=torch.float64)])
    for w in [f.sum(col("x")).over(rows=(-2, 0)).alias("m"), (col("x") - f.avg(col("x")).over(rows=(-6, 0))).alias("d"),
              f.count(all_cols()).over(rows=(1, 5)).alias("c")]:
        cm = ColumnMap("k", "x", w)
        assert cm.has_window and cm.fusion_units(t) is None


def test_select_filter_assign_raw_sql_reject_frame_nodes():
    from fugue_b200 import api as fa
    from fugue_b200.execution_engine import B200ExecutionEngine

    eng = B200ExecutionEngine.__new__(B200ExecutionEngine)  # no device needed to reject the input
    eng.to_df = lambda df, schema=None: (_ for _ in ()).throw(AssertionError("must reject first"))  # type: ignore
    w = f.sum(col("x")).over(rows=(-2, 0))
    with pytest.raises(NotImplementedError):
        eng.select(None, SelectColumns(col("k"), w.alias("m")))
    with pytest.raises(NotImplementedError):
        eng.select(None, SelectColumns(col("k")), where=w > 1)
    with pytest.raises(NotImplementedError):
        eng.filter(None, w > 1)
    with pytest.raises(NotImplementedError):
        eng.assign(None, [w.alias("m")])
    with pytest.raises(NotImplementedError):
        fa.raw_sql("SELECT * FROM", w, engine=eng)


def test_tile_width_constant_mirrors_the_header():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "include", "fugue_b200.h")) as fh:
        h = fh.read()
    assert int(re.search(r"#define FB_FRAME_TILE_MAX_WIDTH (\d+)", h).group(1)) == K.FRAME_TILE_MAX_WIDTH
    assert int(re.search(r"#define FB_FRAME_UNBOUNDED_START (\d+)", h).group(1)) == K.FRAME_UNBOUNDED_START
    assert int(re.search(r"#define FB_FRAME_UNBOUNDED_END (\d+)", h).group(1)) == K.FRAME_UNBOUNDED_END
