"""Explicit window nodes (``over(partition_by=.., order_by=..)``, SQL's ``OVER (PARTITION BY .. ORDER BY ..)``) restated
in plain Python and numpy for the tests (DESIGN §7p).  Test infrastructure only: nothing here touches the device.

:func:`select` takes an Arrow table and output ``ColumnExpr`` trees, as the SQL parser or the builders give them, and
returns python values per output in input row order.  Every distinct explicit window node is evaluated on its own:
its PARTITION BY / ORDER BY expressions and its arguments become temporary columns (:func:`column`), then the bare node
(spec removed) goes to the map references with keys = the partition columns and presort = the order pairs:
``_range_oracle.window_map``, which serves RANGE nodes itself and hands ROWS nodes to ``_frame_oracle`` and the rest
to ``oracle.window``.  So the semantics are theirs (§7d): NaN is NULL, -0.0 equals 0.0, NULLs last in every
direction, ties in input order.  Two rules of the engine are applied around them:

* dates, timestamps and booleans reach the references as their integer storage (partition and order keys too, except
  the one order key of a RANGE frame with an offset), and MIN / MAX / FIRST / LAST / LAG / LEAD come back as the type;
  a uint64 argument of SUM / AVG / MIN / MAX is its int64 bit pattern (§7e's limit);
* the expressions around the windows (arithmetic on a window result, QUALIFY) go through ``oracle.expressions``.
"""
import datetime
from collections import OrderedDict
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import pyarrow as pa

import _range_oracle as RO
from fugue_b200.column import ColumnExpr, Kind, col
from oracle import expressions as ox
from oracle import scalar as osc
from oracle import string_build as osb
from oracle import window as W

_TEMPORAL_STORAGE = (pa.types.is_date32, pa.types.is_date64, pa.types.is_timestamp)


def _storage(a: pa.Array) -> pa.Array:
    if pa.types.is_date32(a.type):
        return a.view(pa.int32())
    if pa.types.is_date64(a.type) or pa.types.is_timestamp(a.type):
        return a.view(pa.int64())
    return a


def column(e: ColumnExpr, table: pa.Table) -> pa.Array:
    """A row-wise expression of the forms the tests put in PARTITION BY / ORDER BY and window arguments, one Python
    value at a time: a column, ``CAST(float AS BIGINT)`` (truncation; a NaN or infinite value has no defined result),
    ``UPPER``, integer ``+ - * %`` (int64, wrapping; ``%`` truncated), a date or timestamp plus or minus a whole
    number of its units, and a literal.  Anything else goes to ``oracle.expressions`` on a pandas frame of the table."""
    n = table.num_rows
    if e.kind == Kind.NAMED and e.as_type is None:
        return table.column(e.name).combine_chunks()
    if e.kind == Kind.NAMED and e.as_type == pa.int64():
        a = table.column(e.name).combine_chunks()
        out = []
        for x in a.to_pylist():
            if isinstance(x, float) and not np.isfinite(x):
                raise ValueError(f"CAST({x} AS BIGINT) has no defined result")
            out.append(None if x is None else int(x))
        return pa.array(out, type=pa.int64())
    if e.kind == Kind.CALL and e.func == "UPPER" and e.as_type is None:
        return pa.array([osb.upper(x) for x in column(e.args[0], table).to_pylist()], type=pa.string())
    if e.kind == Kind.BINARY and e.op in ("+", "-", "*", "%") and e.as_type is None:
        left = column(e.left, table)
        if e.right.kind == Kind.LITERAL and not isinstance(e.right.value, (int, float)):  # a date + an interval
            tp = left.type
            assert any(f(tp) for f in _TEMPORAL_STORAGE) and e.op in ("+", "-"), str(e)
            unit = "D" if pa.types.is_date32(tp) else ("ms" if pa.types.is_date64(tp) else tp.unit)
            per, mul = W._PER_UNIT_US[unit]
            us = e.right.value // datetime.timedelta(microseconds=1)
            assert (us * mul) % per == 0
            step = (us * mul // per) * (1 if e.op == "+" else -1)
            vals = [None if x is None else x + step for x in _storage(left).to_pylist()]
            return pa.array(vals, type=_storage(left).type).view(tp)
        right = column(e.right, table)
        assert pa.types.is_integer(left.type) and pa.types.is_integer(right.type), str(e)
        out = []
        for a, b in zip(left.to_pylist(), right.to_pylist()):
            if a is None or b is None:
                out.append(None)
            elif e.op == "%":
                out.append(osc.mod(a, b, False))
            else:
                out.append(osc.wrap(a + b if e.op == "+" else a - b if e.op == "-" else a * b))
        return pa.array(out, type=pa.int64())
    if e.kind == Kind.LITERAL:
        return pa.array([e.value] * n, type=pa.scalar(e.value).type)
    return pa.array(ox.evaluate(e, W._pandas(table)), from_pandas=True)


def _window(node: ColumnExpr, table: pa.Table) -> pa.Array:
    """One explicit window node (no alias, no cast) over ``table``, in input row order."""
    cols: Dict[str, pa.Array] = {}

    def temp(x: ColumnExpr, stem: str) -> str:
        nm = f"{stem}{len(cols)}"
        cols[nm] = column(x, table)
        return nm

    keys = [temp(x, "__p") for x in node.kwargs["partition_by"]]
    presort: "OrderedDict[str, bool]" = OrderedDict()
    for x, asc in node.kwargs["order_by"]:
        presort.setdefault(temp(x, "__o"), asc)
    offset = "range" in node.kwargs and any(b is not None and b != 0 for b in node.kwargs["range"])
    for nm in keys + ([] if offset else list(presort)):  # integer storage sorts and groups as the value
        cols[nm] = _storage(cols[nm])
    fn = node.func
    kw = {k: v for k, v in node.kwargs.items() if k not in ("partition_by", "order_by")}
    args, back = [], None
    for a in node.args:
        if a.kind == Kind.WILDCARD:
            args.append(a)
            continue
        nm = temp(a, "__a")
        tp = cols[nm].type
        typed = fn in ("MIN", "MAX", "FIRST", "LAST", "LAG", "LEAD")
        if any(f(tp) for f in _TEMPORAL_STORAGE) or tp == pa.bool_():
            cols[nm] = cols[nm].cast(pa.int8()) if tp == pa.bool_() else _storage(cols[nm])
            back = tp if typed else None
        elif tp in (pa.float16(), pa.float32()) and fn in ("MIN", "MAX"):
            # totalOrder on the stored bits (numpy's float conversions may quiet a signalling NaN): an integer key
            ib = pa.int16() if tp == pa.float16() else pa.int32()
            b = np.asarray(cols[nm].view(ib).fill_null(0).to_numpy(zero_copy_only=False)).astype(np.int64)
            key = np.where(b >= 0, b, b ^ ((1 << (ib.bit_width - 1)) - 1))
            cols[nm], back = pa.array(key, type=pa.int64(), mask=~np.asarray(cols[nm].is_valid())), ("key", tp, ib)
        elif tp == pa.uint64() and fn in ("SUM", "AVG", "MIN", "MAX"):
            cols[nm], back = cols[nm].view(pa.int64()), (tp if typed else None)
        if back is not None and fn in ("LAG", "LEAD") and kw["default"] is not None:
            d = W.offset_default(kw["default"], tp)
            kw["default"] = (d.cast(pa.int8()) if tp == pa.bool_() else _storage(d))[0].as_py()
        args.append(col(nm))
    bare = ColumnExpr(Kind.WINDOW, node.head, args, kw).alias("__w")
    sub = pa.table(cols) if cols else pa.table({"__n": pa.nulls(table.num_rows, pa.int8())})
    out = pa.array(RO.window_map(sub, keys, presort, [bare])["__w"], type=_result_type(fn, args, sub))
    if isinstance(back, tuple):  # a totalOrder key back to the float's bits
        _, tp, ib = back
        k = np.asarray(out.fill_null(0).to_numpy(zero_copy_only=False))
        bits = np.where(k >= 0, k, k ^ ((1 << (ib.bit_width - 1)) - 1)).astype(ib.to_pandas_dtype())
        out = pa.array(bits, type=ib, mask=~np.asarray(out.is_valid())).view(tp)
    elif back is not None:
        out = out.cast(back) if back == pa.bool_() else out.view(back)
    return out


def _result_type(fn: str, args: List[ColumnExpr], sub: pa.Table) -> Optional[pa.DataType]:
    if fn in ("ROW_NUMBER", "RANK", "DENSE_RANK", "COUNT"):
        return pa.int64()
    if fn == "AVG":
        return pa.float64()
    tp = sub.column(args[0].name).type
    if fn == "SUM":
        return pa.float64() if pa.types.is_floating(tp) else pa.int64()
    return tp


def _replace(e: Any, table: pa.Table, temps: Dict[str, pa.Array]) -> Any:
    if not isinstance(e, ColumnExpr):
        return e
    if e.kind == Kind.WINDOW:
        bare = e.alias("").cast(None)
        uid = "__w" + bare.fingerprint()[:12]
        if uid not in temps:
            temps[uid] = _window(bare, table)
        rep = col(uid)
        if e.as_type is not None:
            rep = rep.cast(e.as_type)
        return rep.alias(e.as_name) if e.as_name else rep
    if e.has_args:
        return ColumnExpr(e.kind, e.head, [_replace(a, table, temps) for a in e.args],
                          {k: _replace(v, table, temps) for k, v in e.kwargs.items()}, e.is_distinct, e.as_name,
                          e.as_type)
    return e


def select(table: pa.Table, columns: Sequence[ColumnExpr], qualify: Optional[ColumnExpr] = None
           ) -> Tuple[Dict[str, list], List[int]]:
    """(output name -> python values, the input rows kept): ``SELECT columns FROM table QUALIFY qualify``, rows in
    input order; dates and timestamps as their integer storage (``storage_list``).  Window results read directly are
    returned as the window gives them; any other expression goes through ``oracle.expressions``."""
    temps: Dict[str, pa.Array] = {}
    exprs = [_replace(c.infer_alias(), table, temps) for c in columns]
    q = None if qualify is None else _replace(qualify, table, temps)
    full = table
    for k, a in temps.items():
        full = full.append_column(k, a)
    keep = list(range(table.num_rows))
    if q is not None:
        pdf = W._pandas(full.select(_names(q)))
        keep = np.flatnonzero(ox._predicate(q, pdf)).tolist()
    out: Dict[str, list] = {}
    for e in exprs:
        if e.kind == Kind.NAMED and e.as_type is None:
            vals = storage_list(full.column(e.name))
        else:
            s = ox.evaluate(e.alias(""), W._pandas(full.select(_names(e))))
            vals = [None if x is None or x is np.nan or (x is not None and str(x) == "<NA>") else x
                    for x in (s.tolist() if hasattr(s, "tolist") else [s] * table.num_rows)]
        out[e.output_name] = [vals[i] for i in keep]
    return out, keep


def storage_list(a: Any) -> list:
    """Python values of an Arrow column; dates and timestamps as their integer storage (days or the type's unit since
    the epoch), which holds every value, also those outside Python's ``datetime``."""
    a = a.combine_chunks() if isinstance(a, pa.ChunkedArray) else a
    return (_storage(a) if any(f(a.type) for f in _TEMPORAL_STORAGE) else a).to_pylist()


def _names(e: ColumnExpr) -> List[str]:
    found: List[str] = []

    def walk(x: Any) -> None:
        if isinstance(x, ColumnExpr):
            if x.kind == Kind.NAMED:
                found.append(x.name)
            if x.has_args:
                for a in list(x.args) + list(x.kwargs.values()):
                    walk(a)

    walk(e)
    return list(dict.fromkeys(found))
