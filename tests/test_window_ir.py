"""Window nodes of the column IR (``Kind.WINDOW``, fugue_b200/column.py) and their place in the ColumnMap plan
(fugue_b200/colmap.py) on CPU: builders, errors, ``is_agg``, printing, types, and that a map with a window
function is never fused into the scatter kernel while row-wise maps plan as before."""
import numpy as np
import pyarrow as pa
import pytest
import torch

from fugue_b200.colmap import ColumnMap
from fugue_b200.column import (Kind, SelectColumns, all_cols, col, functions as f, has_window, is_agg, lit,
                               to_sql)
from fugue_b200.schema import Schema
from fugue_b200.table import B200Table


def test_kind_value_is_appended():
    assert [int(k) for k in Kind] == list(range(8)) and Kind.WINDOW == 7 and Kind.AGG == 6


def test_builders_make_window_nodes():
    for e in [f.sum(col("v")).over(), f.count(col("v")).over(running=True), f.count(all_cols()).over(),
              f.avg(col("v")).over(), f.min(col("v")).over(), f.max(col("v")).over(running=True),
              f.first(col("v")).over(), f.last(col("v")).over(running=True), f.row_number(), f.rank(),
              f.dense_rank(), f.lag(col("v")), f.lead(col("v"), 2, 0)]:
        assert e.kind == Kind.WINDOW and has_window(e) and not is_agg(e)
    assert f.sum(col("v")).over().kwargs == {"running": False}
    assert f.lag(col("v")).kwargs == {"n": 1, "default": None}
    assert f.lead("v", n=0, default="x").kwargs == {"n": 0, "default": "x"}


def test_over_needs_a_plain_aggregation():
    for bad in [col("v"), col("v") + 1, lit(1), f.coalesce(col("v"), 0), f.row_number()]:
        with pytest.raises(ValueError):
            bad.over()
    with pytest.raises(ValueError):
        f.count_distinct(col("v")).over()
    with pytest.raises(ValueError):
        f.sum(f.max(col("v"))).over()
    with pytest.raises(ValueError):
        f.first(all_cols()).over()
    with pytest.raises(ValueError):
        f.sum(col("v")).over(running=1)


def test_lag_lead_arguments_are_checked():
    for n in [-1, 1.0, True, "1"]:
        with pytest.raises(ValueError):
            f.lag(col("v"), n)
    with pytest.raises(ValueError):
        f.lead(col("v"), 1, [1])
    with pytest.raises(ValueError):
        f.lag(all_cols())
    with pytest.raises(ValueError):
        f.lag(f.sum(col("v")))


def test_is_agg_does_not_look_inside_a_window():
    share = col("v") / f.sum(col("v")).over()
    assert not is_agg(share) and has_window(share)
    assert is_agg(f.sum(col("v"))) and not has_window(f.sum(col("v")))
    assert is_agg(f.sum(col("v")) + f.row_number())
    with pytest.raises(ValueError):
        ColumnMap(f.sum(col("x")))
    ColumnMap("k", share.alias("share"))  # a window map is a map


def test_text_forms():
    assert str(f.sum(col("v")).over()) == "SUM(v) OVER ()"
    assert str(f.sum(col("v")).over(running=True).alias("r")) == \
        "SUM(v) OVER (ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW) AS r"
    assert str(f.count(all_cols()).over()) == "COUNT(*) OVER ()"
    assert str(f.row_number().alias("rn")) == "ROW_NUMBER() OVER () AS rn"
    assert str(f.lag(col("v"), 2, 0.5)) == "LAG(v,2,0.5) OVER ()"
    assert str(f.lead(col("s"), 1, "x")) == "LEAD(s,1,'x') OVER ()"
    assert to_sql((col("v") / f.sum(col("v")).over()).alias("share")) == "v/SUM(v) OVER () AS share"
    assert to_sql(f.last(col("my v")).over(running=True)) == \
        "LAST(`my v`) OVER (ROWS BETWEEN UNBOUNDED PRECEDING AND CURRENT ROW)"
    assert to_sql(f.lag(col("v")).cast(int)) == "CAST(LAG(v,1,NULL) OVER () AS long)"
    assert f.lag(col("v")).fingerprint() != f.lead(col("v")).fingerprint()
    assert f.sum(col("v")).over().fingerprint() != f.sum(col("v")).over(running=True).fingerprint()


def test_alias_and_type_inference():
    sch = Schema("k:long,i:int,v:double,s:str,d:date")
    assert f.sum(col("v")).over().infer_alias().output_name == "v"
    assert f.lag(col("s")).infer_alias().output_name == "s"
    assert f.row_number().infer_alias().output_name == ""
    assert f.count(all_cols()).over().infer_alias().output_name == ""
    types = {"SUM(i)": (f.sum(col("i")).over(), pa.int64()), "SUM(v)": (f.sum(col("v")).over(), pa.float64()),
             "AVG": (f.avg(col("i")).over(), pa.float64()), "COUNT": (f.count(col("s")).over(), pa.int64()),
             "MIN": (f.min(col("i")).over(running=True), pa.int32()), "LAST": (f.last(col("d")).over(), pa.date32()),
             "LAG": (f.lag(col("s")), pa.string()), "RN": (f.row_number(), pa.int64()),
             "RANK": (f.rank(), pa.int64()), "DR": (f.dense_rank(), pa.int64())}
    for name, (e, tp) in types.items():
        assert e.infer_type(sch) == tp, name
    with pytest.raises(ValueError):  # a ranking needs an alias
        SelectColumns(col("k"), f.row_number()).assert_all_with_names()


def _table() -> B200Table:
    n = 16
    cols = [torch.arange(n, dtype=torch.int64), torch.arange(n, dtype=torch.float64)]
    return B200Table(Schema("k:long,x:double"), cols)


def test_window_maps_are_never_fused_and_row_wise_maps_plan_as_before():
    t = _table()
    assert ColumnMap("k", "x").fusion_units(t) is not None
    assert ColumnMap("k", (col("x") * 2 + 1).alias("w")).fusion_units(t) is not None
    for w in [f.row_number().alias("rn"), f.sum(col("x")).over(running=True).alias("r"),
              (col("x") - f.lag(col("x"))).alias("dx"), f.lag(col("x"), 0).alias("same")]:
        cm = ColumnMap("k", "x", w)
        assert cm.has_window and cm.fusion_units(t) is None
    assert not ColumnMap("k", "x").has_window


def test_window_argument_may_not_hold_a_window():
    from fugue_b200.colmap import _collect_windows
    from fugue_b200.column import ColumnExpr

    with pytest.raises(ValueError):  # the builders refuse it ...
        f.sum(f.row_number()).over()
    with pytest.raises(NotImplementedError):  # ... and so does the evaluator for a hand-made tree
        _collect_windows(ColumnExpr(Kind.WINDOW, "SUM", [f.row_number()], {"running": False}), {})
    out = {}
    _collect_windows((f.sum(col("x")).over() + f.sum(col("x")).over().alias("y") * f.row_number()).alias("z"), out)
    assert len(out) == 2  # equal nodes (alias aside) are computed once


def test_select_filter_raw_sql_reject_window_nodes():
    """``fa.select / assign / filter / raw_sql`` check before touching the device."""
    from fugue_b200 import api as fa
    from fugue_b200.execution_engine import B200ExecutionEngine

    eng = B200ExecutionEngine.__new__(B200ExecutionEngine)  # no device needed to reject the input
    eng.to_df = lambda df, schema=None: (_ for _ in ()).throw(AssertionError("must reject first"))  # type: ignore
    with pytest.raises(NotImplementedError):
        eng.select(None, SelectColumns(col("k"), f.row_number().alias("rn")))
    with pytest.raises(NotImplementedError):
        eng.select(None, SelectColumns(col("k")), where=f.row_number() > 1)
    with pytest.raises(NotImplementedError):
        eng.filter(None, f.lag(col("x")) > 1)
    with pytest.raises(NotImplementedError):
        eng.assign(None, [f.row_number().alias("rn")])
    with pytest.raises(NotImplementedError):
        fa.raw_sql("SELECT * FROM", f.row_number(), engine=eng)
