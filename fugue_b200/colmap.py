"""``ColumnMap``: a per-row map of ``fa.transform`` written as column expressions (K4).

The reference applies the map function to every partition after grouping
(``PandasMapEngine.map_dataframe``, fugue/execution/native_execution_engine.py:156-164).  A map that is
a list of column expressions needs no second pass on the GPU: the B200 map engine evaluates affine
expressions (``x * a + y * b + c`` over at most two columns of one class) inside the scatter kernel
of the hash partition, between the gather from the staged tile and the store
(``fb_partition_apply_map``).  Everything else is still evaluated on the device, by the expression
evaluator (K8) over the partitioned table - calling the object does exactly that.

Window functions (K9) make the map depend on the partitioning: ``f.sum(col("v")).over(running=True)``,
``f.row_number()``, ``f.lag(col("v"))`` ... are evaluated over the logical partitions of the table
(``table.logical_offsets``, rows in presort order; a table without them is one partition), with SQL
window semantics.  The map engine sorts by (keys, presort) first for such a map.

    fa.transform(df, ColumnMap("key", "v", f.sum(col("v")).over(running=True).alias("run"),
                               (col("v") / f.sum(col("v")).over()).alias("share")),
                 schema="key:long,v:double,run:double,share:double", partition=PartitionSpec(by="key", presort="t"))

    fa.transform(df, ColumnMap("key", "v0", (col("v0") * 2 + col("v1")).alias("w")),
                 schema="key:long,v0:double,w:double", partition=PartitionSpec(by="key", algo="hash", num=256))
"""
import datetime
import math
import struct
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import pyarrow as pa
import torch

from . import aggregates as A
from . import kernels as K
from .aggregates import bivariate_of
from .column import (AGGREGATES, DISTRIBUTIONS, EWM_HEADS, PERCENTILES, VALUE_HEADS, ColumnExpr, Kind, SelectColumns,
                     bivariate_xy, col as _col, ewm_alpha, has_window, has_explicit_window, is_agg, is_explicit,
                     result_type)
from .table import B200Table, _storage_dtype, narrow, widen


def _f64_bits(v: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", float(v)))[0]


class ColumnMap:
    def __init__(self, *columns: Any):
        assert len(columns) > 0, "ColumnMap needs at least one output column"
        self.columns: List[ColumnExpr] = [_col(c) for c in columns]
        for c in self.columns:
            if is_agg(c):
                raise ValueError(f"{c} is an aggregation: a map is row-wise")
            if has_explicit_window(c):
                raise ValueError(f"{c}: a ColumnMap's windows run over the PartitionSpec's partitions and presort; "
                                 "drop partition_by / order_by, or use the node in select / assign / filter")
        self.has_window = any(has_window(c) for c in self.columns)

    def select(self, t: B200Table) -> SelectColumns:
        return SelectColumns(*self.columns).replace_wildcard(t.schema).assert_all_with_names()

    def __call__(self, t: B200Table) -> B200Table:
        """Unfused evaluation on the device (one pass of the expression evaluator over ``t``)."""
        from . import expr as X

        cols = self.select(t).all_cols
        src = _with_windows(t, cols) if self.has_window else t
        if src is not t:
            cols = [X.rewrite(c, src.window_column) for c in cols]
        out = X.project(src, cols)
        keep = t.partition_keys is not None and all(k in out.schema for k in t.partition_keys)
        return B200Table(out.schema, out.columns, out.valid, out.dictionaries, t.offsets if keep else None,
                         t.partition_keys if keep else None)

    # ---- fusion plan -----------------------------------------------------------------------------
    def fusion_units(self, t: B200Table) -> Optional[List[Tuple[Any, Any, int, int, int, int, pa.DataType]]]:
        """One ``(x, y, mode, a, b, c, type)`` per output column if EVERY column can be produced by the
        scatter kernel's epilogue (plain 8-byte NULL-free columns and affine expressions of them), else None.
        A map with window functions depends on the logical partitions: never fused."""
        if self.has_window:
            return None
        units = []
        for e in self.select(t).all_cols:
            u = _unit_of(e, t)
            if u is None:
                return None
            units.append(u)
        return units


def _plain_column(e: ColumnExpr, t: B200Table) -> Optional[int]:
    if e.kind != Kind.NAMED or e.as_type is not None or e.name not in t.schema:
        return None
    i = t.schema.index_of_key(e.name)
    if t.columns[i].element_size() != 8 or t.valid[i] is not None or e.name in t.dictionaries:
        return None
    if t.columns[i].data_ptr() % 16 != 0:
        return None
    return i


def _term(e: ColumnExpr, t: B200Table) -> Optional[Tuple[Any, int]]:
    """``col`` | ``-col`` | ``col * lit`` | ``lit * col`` -> (coefficient, column index)."""
    if e.as_type is not None:
        return None
    if e.kind == Kind.NAMED:
        i = _plain_column(e, t)
        return None if i is None else (1, i)
    if e.kind == Kind.UNARY and e.op == "-":
        i = _plain_column(e.arg, t)
        return None if i is None else (-1, i)
    if e.kind == Kind.BINARY and e.op == "*":
        for c, l in ((e.left, e.right), (e.right, e.left)):
            if l.kind == Kind.LITERAL and l.as_type is None and type(l.value) in (int, float):
                i = _plain_column(c, t)
                if i is not None:
                    return (l.value, i)
    return None


def _unit_of(e: ColumnExpr, t: B200Table) -> Optional[Tuple[Any, Any, int, int, int, int, pa.DataType]]:
    i = _plain_column(e, t)
    if i is not None:
        return (t.columns[i], None, K.MAP_COPY, 0, 0, 0, t.schema.types[i])
    if e.as_type is not None:
        return None
    # peel: ((term [+-] term) [+-] lit) in exactly this association, so that the rounding order of the
    # fused form (a*x + b*y) + c is the evaluator's
    const: Any = None
    body = e
    if e.kind == Kind.BINARY and e.op in ("+", "-") and e.right.kind == Kind.LITERAL and e.right.as_type is None \
            and type(e.right.value) in (int, float) and e.left.as_type is None:
        const = e.right.value if e.op == "+" else -e.right.value
        body = e.left
    terms = []
    first = _term(body, t)
    if first is not None:
        terms = [first]
    elif body.kind == Kind.BINARY and body.op in ("+", "-") and body.as_type is None:
        a, b = _term(body.left, t), _term(body.right, t)
        if a is None or b is None:
            return None
        terms = [a, (b[0] if body.op == "+" else -b[0], b[1])]
    else:
        return None
    if const is None and len(terms) == 1 and terms[0][0] == 1:
        return None  # plain column with an alias only: handled as copy by the caller's NAMED case
    cols = [t.columns[i] for _, i in terms]
    tps = [t.schema.types[i] for _, i in terms]
    if all(tp == pa.float64() for tp in tps):
        coef = [_f64_bits(c) for c, _ in terms] + [0]
        cbits = _f64_bits(-0.0 if const is None else const)  # x + (-0.0) == x for every x, signed zeros included
        return (cols[0], cols[1] if len(cols) > 1 else None, K.MAP_AFFINE_F64, coef[0], coef[1], cbits, pa.float64())
    if all(tp == pa.int64() for tp in tps) and all(type(c) is int for c, _ in terms) and type(const or 0) is int:
        coef = [c & ((1 << 64) - 1) for c, _ in terms] + [0]
        return (cols[0], cols[1] if len(cols) > 1 else None, K.MAP_AFFINE_I64, coef[0], coef[1],
                (const or 0) & ((1 << 64) - 1), pa.int64())
    return None


# ---- window functions (K9) ---------------------------------------------------------------------------
class _WindowTable(B200Table):
    """The map's input plus one temporary column per distinct window node; ``window_column`` is the
    ``expr.rewrite`` mapper that makes a tree read those columns."""

    def window_column(self, node: ColumnExpr) -> Optional[ColumnExpr]:
        if node.kind != Kind.WINDOW:
            return None
        return _col(self.window_names[node.alias("").cast(None).fingerprint()])


def _collect_windows(e: Any, out: Dict[str, ColumnExpr]) -> None:
    if not isinstance(e, ColumnExpr):
        return
    if e.kind == Kind.WINDOW:
        for a in e.args:
            if has_window(a):
                raise NotImplementedError(f"window function inside the argument of {e}")
        bare = e.alias("").cast(None)
        out.setdefault(bare.fingerprint(), bare)
        return
    for a in list(e.args) + list(e.kwargs.values()):
        _collect_windows(a, out)


def _with_windows(t: B200Table, cols: List[ColumnExpr]) -> B200Table:
    """Evaluate every window node of ``cols`` over the logical partitions of ``t``: arguments pre-projected
    by the evaluator (K8), running / partition aggregates and ranks by the segmented scan (K9), moving
    frames (``rows``) by the frame kernel, value frames (``range``) by the bounds kernel (or the peer groups)
    and the block tree, all with the same finishers, FIRST / LAST / partition values / LAG / LEAD by row
    gathers, percentiles by the quantile kernel (K10), one call per argument column with all its q values,
    FIRST_VALUE / LAST_VALUE / NTH_VALUE by one ``fb_window_value`` call per frame, NTILE / PERCENT_RANK / CUME_DIST by
    one ``fb_window_distribution`` call over the peer heads."""
    from . import expr as X
    from . import sort as S
    from .schema import Schema

    nodes: Dict[str, ColumnExpr] = {}
    for c in cols:
        _collect_windows(c, nodes)
    n, dev = t.num_rows, t.device
    # ---- arguments: plain columns as they are, anything else through one evaluator pass
    pre = [_col(nm) for nm in t.schema.names]
    arg_name: Dict[str, str] = {}
    for bare in nodes.values():
        for a in bare.args:
            if a.kind == Kind.WILDCARD:
                continue
            uid = a.fingerprint()
            if uid in arg_name:
                continue
            if a.kind == Kind.NAMED and a.as_type is None:
                if a.name not in t.schema:
                    raise KeyError(f"column {a.name} is not in {t.schema}")
                arg_name[uid] = a.name
            else:
                arg_name[uid] = f"__fb_wa{len(arg_name)}"
                pre.append(a.alias(arg_name[uid]))
    base = X.project(t, pre) if len(pre) > len(t.schema) else t
    # ---- segments: the logical partitions, one segment when the table has none
    off = t.logical_offsets
    if off is None:
        off = torch.tensor([0, n], dtype=torch.int64, device=dev)
    lengths = off[1:] - off[:-1]
    rows = torch.arange(n, dtype=torch.int64, device=dev)
    bounds: Dict[str, torch.Tensor] = {}

    def seg_first() -> torch.Tensor:  # first row of every row's partition
        if "first" not in bounds:
            bounds["first"] = torch.repeat_interleave(off[:-1], lengths, output_size=n)
        return bounds["first"]

    def seg_last() -> torch.Tensor:  # last row of every row's partition
        if "last" not in bounds:
            bounds["last"] = torch.repeat_interleave(off[1:] - 1, lengths, output_size=n)
        return bounds["last"]

    def peer_heads() -> torch.Tensor:  # first row of every group of rows equal on all presort columns
        heads = S.group_starts(t, list(getattr(t, "logical_order", None) or []))
        heads[off[:-1][lengths > 0]] = True
        return heads

    # ---- scans: collected first, all run in one call per frame (None: the running scan)
    scans: Dict[Any, List[Any]] = {}
    quantiles: Dict[str, List[Tuple[float, int]]] = {}  # argument column -> its (q, CONT | DISC) pairs
    moments: Dict[str, int] = {}  # argument column of a variance -> its column of the moments scan
    shapes: Dict[str, int] = {}  # argument column of a skewness or kurtosis -> its column of the shape-moments scan
    comoments: Dict[Tuple[str, str], int] = {}  # (x, y) argument columns of a pair -> its pair of the co-moments scan
    ewms: Dict[Tuple[Any, ...], int] = {}  # (argument column, _ewm_decay) -> its column of the ewm scan
    ewm_spread: set = set()  # the ewm scan columns an EWM_VAR or EWM_STD reads
    pair_sums: Dict[Tuple[str, str], Tuple[Any, Any]] = {}  # (x, y) -> the running SUM scans of x and y over the pair
    finish: List[Any] = []     # per node: (fingerprint, fn(scan results) -> (column, validity, type, dictionary))
    values: Dict[Any, List[Any]] = {}  # frame -> (values, validity, nth) of its FIRST / LAST / NTH_VALUE nodes
    dist: Dict[str, Any] = {"PERCENT_RANK": False, "CUME_DIST": False, "NTILE": []}  # this spec's distribution heads

    def scan(op: int, v: Any, m: Any, frame: Any = None) -> Tuple[Any, int]:
        cols_ = scans.setdefault(frame, [])
        cols_.append((op, v, m))
        return frame, len(cols_) - 1

    for uid, bare in nodes.items():
        fn = bare.func
        if fn in ("LAG", "LEAD"):
            finish.append((uid, _offset_value(base, bare, arg_name, rows, seg_first, seg_last)))
            continue
        if fn in PERCENTILES:
            name = arg_name[bare.arg.fingerprint()]
            qs = quantiles.setdefault(name, [])
            qs.append((bare.kwargs["q"], K.QUANTILE_CONT if fn == "PERCENTILE_CONT" else K.QUANTILE_DISC))
            finish.append((uid, _percentile_value(base, name, len(qs) - 1, fn == "PERCENTILE_CONT", lengths, n)))
            continue
        if fn == "ROW_NUMBER":
            finish.append((uid, lambda r, rows=rows: (rows - seg_first() + 1, None, pa.int64(), None)))
            continue
        if fn in ("RANK", "DENSE_RANK"):
            heads = peer_heads()
            if fn == "RANK":
                i = scan(K.AGG_MAX_I64, torch.where(heads, rows - seg_first() + 1, torch.zeros_like(rows)), None)
            else:
                i = scan(K.AGG_SUM_I64, heads.to(torch.int64), None)
            finish.append((uid, lambda r, i=i: (r[i][0], None, pa.int64(), None)))
            continue
        if fn in DISTRIBUTIONS:  # one fb_window_distribution call for all of them
            if fn == "NTILE":
                dist["NTILE"].append(bare.kwargs["n"])
                key: Any = ("NTILE", len(dist["NTILE"]) - 1)
            else:
                dist[fn] = True
                key = (fn,)
            finish.append((uid, lambda r, key=key: (r[("dist",) + key], None, result_type_of(key[0]), None)))
            continue
        if fn in VALUE_HEADS:  # one fb_window_value call per frame for all of them
            kw = bare.kwargs
            if "range" in kw:
                vframe: Any = ("range",) + _range_offsets(t, kw["range"])
            else:
                vframe = ("rows",) + (kw["rows"] if "rows" in kw else ((None, 0) if kw.get("running") else (None, None)))
            name = arg_name[bare.arg.fingerprint()]
            ci = base.schema.index_of_key(name)
            nth = kw["n"] if fn == "NTH_VALUE" else (1 if fn == "FIRST_VALUE" else K.VALUE_LAST)
            vcols = values.setdefault(vframe, [])
            vcols.append((base.columns[ci], base.valid[ci], nth))
            finish.append((uid, lambda r, j=(vframe, len(vcols) - 1), tp=base.schema.types[ci],
                           d=base.dictionaries.get(name): (*r[("value",) + j], tp, d)))
            continue
        if fn in EWM_HEADS:  # the ewm scan: one column per argument and decay, shared by its heads
            name = arg_name[bare.arg.fingerprint()]
            A.check_argument(fn, name, base.schema.types[base.schema.index_of_key(name)], name in base.dictionaries)
            j = ewms.setdefault((name,) + _ewm_decay(t, bare), len(ewms))
            if fn != "EWM_MEAN":  # a variance reads W, W2 and C as well; a mean alone writes only count and mean
                ewm_spread.add(j)
            finish.append((uid, lambda r, j=j, fn=fn, kw=bare.kwargs: (
                *A.ewm_of(fn, *r[("ewm", j)], kw.get("bias", False), kw["min_periods"]), pa.float64(), None)))
            continue
        frame = bare.kwargs.get("rows")  # ROWS BETWEEN frame[0] AND frame[1]: the moving-frame kernel
        if "range" in bare.kwargs:  # RANGE BETWEEN: ("range", key class or None, start, end), the block tree
            frame = ("range",) + _range_offsets(t, bare.kwargs["range"])
        whole = None if frame is not None or bare.kwargs["running"] else seg_last

        def at_end(x: torch.Tensor, whole: Any = whole) -> torch.Tensor:  # partition value: the scan at its last row
            return x if whole is None else x[whole()]

        family = AGGREGATES[fn].family
        if family == "bivariate":  # the co-moments scan, one pair per (x, y) shared by its functions; no frames
            xy = tuple(arg_name[a.fingerprint()] for a in bivariate_xy(bare))
            for nm in xy:
                A.check_argument(fn, nm, base.schema.types[base.schema.index_of_key(nm)], nm in base.dictionaries)
            if xy not in comoments:
                comoments[xy] = len(comoments)
                # the means follow AVG, as on the hash route: each side's float64 SUM over the pair rows, over their
                # count (the scan's running means stay finite where that sum overflows)
                vx, vy = (base.valid[base.schema.index_of_key(nm)] for nm in xy)
                p = vx if vy is None else (vy if vx is None else (vx & vy).contiguous())
                pair_sums[xy] = tuple(scan(K.AGG_SUM_F64, A.f64_values(base, nm), p) for nm in xy)

            def pair(r: Any, j: int = comoments[xy], sums: Any = pair_sums[xy], e: Any = at_end, fn: str = fn) -> Any:
                m, _, _, sxx, syy, sxy = (e(x) for x in r[("comoments", j)])
                mx, my = (e(r[s][0]) / m.to(torch.float64) for s in sums)
                return (*bivariate_of(fn, m, mx, my, sxx, syy, sxy), result_type(fn, None), None)

            finish.append((uid, pair))
            continue
        if fn == "COUNT" or bare.arg.kind == Kind.WILDCARD:  # COUNT(x), COUNT(*)
            m = None if bare.arg.kind == Kind.WILDCARD else base.valid[base.schema.index_of_key(
                arg_name[bare.arg.fingerprint()])]
            i = scan(K.AGG_COUNT, None, m, frame)
            finish.append((uid, lambda r, i=i, e=at_end: (*A.finish_basic("COUNT", None, e(r[i][1]), None), None)))
            continue
        name = arg_name[bare.arg.fingerprint()]
        ci = base.schema.index_of_key(name)
        c, m, tp, d = base.columns[ci], base.valid[ci], base.schema.types[ci], base.dictionaries.get(name)
        A.check_argument(fn, name, tp, d is not None)
        if family == "pick":
            # first / last valid row so far: MIN / MAX of the row number over the valid rows, then a gather
            i = scan(*A.reduce_input(fn, rows, pa.int64()), m, frame)

            def pick(r: Any, i: Any = i, e: Any = at_end, c: Any = c, m: Any = m, tp: Any = tp, d: Any = d) -> Any:
                idx = torch.where(e(r[i][1]) > 0, e(r[i][0]), torch.full_like(rows, -1))
                (g,), (gv,) = K.gather_rows([c], [m], idx.contiguous(), want_valid=True)
                return g, gv, tp, d

            finish.append((uid, pick))
            continue
        if d is not None:  # MIN / MAX of the ranks, mapped back to codes
            rank, rm = S.string_ranks(base, name)
            i = scan(*A.reduce_input(fn, rank, pa.int64()), rm, frame)
            finish.append((uid, lambda r, i=i, e=at_end, d=d, tp=tp: A.finish_string(e(r[i][0]), e(r[i][1]), d, tp)))
            continue
        if family == "variance":  # the moments scan; frames are rejected by over()
            j = moments.setdefault(name, len(moments))
            finish.append((uid, lambda r, j=j, e=at_end, fn=fn: (
                *A.variance_of(fn, e(r[("moments", j)][1]), e(r[("moments", j)][0])), pa.float64(), None)))
            continue
        if family == "shape":  # the shape-moments scan; frames are rejected by over()
            j = shapes.setdefault(name, len(shapes))
            finish.append((uid, lambda r, j=j, e=at_end, fn=fn: (
                *A.shape_of(fn, *(e(x) for x in r[("shape", j)])), pa.float64(), None)))
            continue
        i = scan(*A.reduce_input(fn, c, tp), m, frame)
        finish.append((uid, lambda r, i=i, e=at_end, fn=fn, tp=tp: (
            *A.finish_basic(fn, e(r[i][0]), e(r[i][1]), tp), None)))

    def range_bounds(cls: Optional[int], start: Any, end: Any) -> Tuple[torch.Tensor, torch.Tensor]:
        """First and last row of every row's RANGE frame."""
        if cls is not None:  # an offset: a search over the one presort key
            name = t.logical_order[0]
            i = t.schema.index_of_key(name)
            tp = t.schema.types[i]
            key = widen(t.columns[i], tp).contiguous()
            kv = S.float_key_valid(key, t.valid[i]) if cls == K.RANGE_KEY_F64 else t.valid[i]
            asc = (getattr(t, "logical_ascending", None) or [True])[0]
            return K.window_range_bounds(off.contiguous(), key, kv, cls, asc, start, end)
        # CURRENT ROW / UNBOUNDED only: the current row's peer group, or the partition's end
        heads = peer_heads()
        peer_first = torch.cummax(torch.where(heads, rows, torch.zeros_like(rows)), 0).values
        ends = torch.ones_like(heads)
        ends[:-1] = heads[1:]  # the next row starts a peer group (or a partition)
        peer_last = torch.flip(torch.cummin(torch.flip(torch.where(ends, rows, torch.full_like(rows, n)), [0]), 0)
                               .values, [0])
        return (seg_first() if start is None else peer_first), (seg_last() if end is None else peer_last)

    results: Dict[Tuple[Any, int], Any] = {}
    for frame, spec in scans.items():
        if frame is None:
            res = K.segmented_scan(off.contiguous(), n, spec)
        elif frame[0] == "range":
            lo, hi = range_bounds(*frame[1:])
            res = K.window_bounded(lo.contiguous(), hi.contiguous(), spec)
        else:
            res = K.window_frame(off.contiguous(), n, frame[0], frame[1], spec)
        results.update(((frame, j), r) for j, r in enumerate(res))
    for vframe, vcols in values.items():
        how = ("bounds",) + tuple(b.contiguous() for b in range_bounds(*vframe[1:])) if vframe[0] == "range" else vframe
        results.update((("value", vframe, j), r) for j, r in enumerate(K.window_value(off.contiguous(), n, how, vcols)))
    if dist["PERCENT_RANK"] or dist["CUME_DIST"] or dist["NTILE"]:
        pr, cd, nts = K.window_distribution(off.contiguous(), peer_heads().contiguous(), dist["PERCENT_RANK"],
                                            dist["CUME_DIST"], dist["NTILE"])
        results.update({("dist", "PERCENT_RANK"): pr, ("dist", "CUME_DIST"): cd})
        results.update((("dist", "NTILE", j), x) for j, x in enumerate(nts))
    for name, qs in quantiles.items():
        results[("quantile", name)] = K.segmented_quantile(off.contiguous(), *quantile_input(base, name), qs)

    def f64_valid(name: str) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
        return A.f64_values(base, name), base.valid[base.schema.index_of_key(name)]

    if moments:
        mcols = [f64_valid(name) for name in moments]
        results.update((("moments", j), r) for j, r in enumerate(K.segmented_moments(off.contiguous(), n, mcols)))
    if shapes:
        scols = [f64_valid(name) for name in shapes]
        results.update((("shape", j), r) for j, r in enumerate(K.segmented_shape_moments(off.contiguous(), n, scols)))
    if comoments:
        pairs = [f64_valid(x) + f64_valid(y) for x, y in comoments]
        results.update((("comoments", j), r) for j, r in enumerate(K.segmented_comoments(off.contiguous(), n, pairs)))
    if ewms:
        ecols = [f64_valid(name) + (alpha, adjust, pos, _ewm_times(t) if pos == K.EWM_TIMES else None, scale,
                                    j in ewm_spread) for (name, alpha, adjust, pos, scale), j in ewms.items()]
        results.update((("ewm", j), r) for j, r in enumerate(K.segmented_ewm(off.contiguous(), n, ecols)))
    names, types, columns, valid = list(base.schema.names), list(base.schema.types), list(base.columns), list(base.valid)
    dicts = dict(base.dictionaries)
    window_names: Dict[str, str] = {}
    for uid, fn in finish:
        c, v, tp, d = fn(results)
        nm = f"__fb_w{len(window_names)}"
        window_names[uid] = nm
        names.append(nm)
        types.append(tp)
        columns.append(narrow(c, tp))
        valid.append(v)
        if d is not None:
            dicts[nm] = d
    out = _WindowTable(Schema([pa.field(a, b) for a, b in zip(names, types)]), columns, valid, dicts)
    out.window_names = window_names
    return out


def result_type_of(fn: str) -> pa.DataType:
    """The result type of a distribution head: NTILE is int64, PERCENT_RANK and CUME_DIST float64."""
    return pa.int64() if fn == "NTILE" else pa.float64()


def evaluate_windows(t: B200Table, exprs: List[ColumnExpr]) -> _WindowTable:
    """Evaluate every explicit window node (``over(partition_by=.., order_by=..)``) of ``exprs`` over ``t``: ``t``
    plus one column per distinct node, rows in ``t``'s order; ``window_column`` rewrites a tree to read them.

    Window arguments and PARTITION BY / ORDER BY expressions are pre-projected in one evaluator pass (K8).  The
    nodes are grouped by spec; for each spec the rows are sorted (stable radix sort: partition expressions
    ascending, then the order expressions in their directions, NULLs last; input order breaks ties), only the
    columns its windows read are gathered, ``_with_windows`` runs over the partitions, and the spec's outputs go back
    to input row order in one launch (``_to_input_order``).  ``OVER ()`` needs no sort."""
    from collections import OrderedDict

    from . import expr as X
    from . import sort as S
    from .schema import Schema

    nodes: Dict[str, ColumnExpr] = {}
    for e in exprs:
        _collect_windows(e, nodes)
    pre = [_col(nm) for nm in t.schema.names]
    temps: Dict[str, str] = {}

    def temp(e: ColumnExpr) -> str:
        if e.kind == Kind.NAMED and e.as_type is None:
            if e.name not in t.schema:
                raise KeyError(f"column {e.name} is not in {t.schema}")
            return e.name
        uid = e.fingerprint()
        if uid not in temps:
            temps[uid] = f"__fb_ws{len(temps)}"
            pre.append(e.alias(temps[uid]))
        return temps[uid]

    specs: Dict[Any, List[Tuple[str, ColumnExpr]]] = {}  # (partition columns, order pairs) -> (uid, map node)
    for uid, node in nodes.items():
        if not is_explicit(node):
            raise NotImplementedError(f"{node}: a window function needs PARTITION BY / ORDER BY; use "
                                      "over(partition_by=.., order_by=..) or a ColumnMap of fa.transform")
        pb = tuple(temp(x) for x in node.kwargs["partition_by"])
        ob = tuple((temp(x), asc) for x, asc in node.kwargs["order_by"])
        args = [a if a.kind == Kind.WILDCARD else _col(temp(a)) for a in node.args]
        kw = {k: v for k, v in node.kwargs.items() if k not in ("partition_by", "order_by")}
        specs.setdefault((pb, ob), []).append((uid, ColumnExpr(Kind.WINDOW, node.head, args, kw)))
    base = X.project(t, pre) if len(pre) > len(t.schema) else t
    for members in specs.values():  # a LAG / LEAD default the argument's type cannot hold fails before the sorts
        for _, m in members:
            if m.func in ("LAG", "LEAD") and m.kwargs["default"] is not None:
                offset_default(m.kwargs["default"], base.schema.types[base.schema.index_of_key(m.arg.name)], m)
    n, dev = t.num_rows, t.device
    names, types = list(t.schema.names), list(t.schema.types)
    columns, valid, dicts = list(t.columns), list(t.valid), dict(t.dictionaries)
    window_names: Dict[str, str] = {}
    for (pb, ob), members in specs.items():
        read = list(dict.fromkeys(list(pb) + [c for c, _ in ob] +
                                  [a.name for _, m in members for a in m.args if a.kind == Kind.NAMED]))
        sub = base.select(read or base.schema.names[:1])  # a table of no columns has no rows
        sub = B200Table(sub.schema, sub.columns, sub.valid, sub.dictionaries)
        idx = None
        if (pb or ob) and n > 1:
            order: "OrderedDict[str, bool]" = OrderedDict((c, True) for c in pb)
            for c, asc in ob:
                order.setdefault(c, asc)
            idx = S.argsort_rows(sub, order, "last")
            sub = S.take_rows(sub, idx)
        sub.logical_offsets = S.logical_offsets(sub, list(pb)) if pb and n > 0 else \
            torch.tensor([0, n], dtype=torch.int64, device=dev)
        sub.logical_order = [c for c, _ in ob]
        sub.logical_ascending = [asc for _, asc in ob]
        w = _with_windows(sub, [m for _, m in members])
        at = [w.schema.index_of_key(w.window_names[m.fingerprint()]) for _, m in members]
        outs, outv = [w.columns[i] for i in at], [w.valid[i] for i in at]
        if idx is not None:
            outs, outv = _to_input_order(outs, outv, idx)
        for (uid, _), i, c, v in zip(members, at, outs, outv):
            nm = f"__fb_w{len(window_names)}"
            window_names[uid] = nm
            names.append(nm)
            types.append(w.schema.types[i])
            columns.append(c)
            valid.append(v)
            if w.schema.names[i] in w.dictionaries:
                dicts[nm] = w.dictionaries[w.schema.names[i]]
    out = _WindowTable(Schema([pa.field(a, b) for a, b in zip(names, types)]), columns, valid, dicts)
    out.window_names = window_names
    return out


def _to_input_order(cols: List[torch.Tensor], valid: List[Optional[torch.Tensor]], idx: torch.Tensor) -> Any:
    """Columns in sorted order (row i is input row ``idx[i]``) back in input order.  One column: one ``fb_scatter_rows``
    launch; more: the inverse permutation and one ``fb_gather_rows`` launch, whose coalesced stores win once several
    columns are moved (100 M rows on an H100 at 700 W: 7.9 ms against 11.7 ms for one float64 column, 23.6 ms against
    19.8 ms for three; DESIGN §7p, §10)."""
    if len(cols) == 1:
        return K.scatter_rows(cols, valid, idx)
    inv = torch.empty_like(idx)
    inv[idx] = torch.arange(int(idx.shape[0]), dtype=torch.int64, device=idx.device)
    return K.gather_rows(cols, valid, inv, want_valid=False)


def quantile_input(t: B200Table, name: str) -> Tuple[torch.Tensor, Optional[torch.Tensor], int]:
    """Column ``name`` as the 8-byte values, validity and value class of the quantile kernel: floats as
    float64, unsigned integers as uint64, strings as their dictionary rank, everything else as int64."""
    from . import sort as S

    i = t.schema.index_of_key(name)
    c, m, tp = t.columns[i], t.valid[i], t.schema.types[i]
    if name in t.dictionaries:
        return S._unsigned_order_key(t, name, True), m, K.RANGE_KEY_U64
    if pa.types.is_floating(tp):
        return widen(c, tp).contiguous(), m, K.RANGE_KEY_F64
    return widen(c, tp).contiguous(), m, K.RANGE_KEY_U64 if pa.types.is_unsigned_integer(tp) else K.RANGE_KEY_I64


def _percentile_value(base: B200Table, name: str, j: int, cont: bool, lengths: torch.Tensor, n: int) -> Any:
    """The finisher of a percentile node: its per-partition result repeated over the partition's rows; a
    DISC result is the picked row's own value (any type), gathered."""
    i = base.schema.index_of_key(name)
    c, m, tp = base.columns[i], base.valid[i], base.schema.types[i]
    if cont and (name in base.dictionaries or not (pa.types.is_integer(tp) or pa.types.is_floating(tp))):
        raise NotImplementedError(f"PERCENTILE_CONT needs an integer or float column; {name} is {tp}")

    def run(r: Any) -> Any:
        count, outs = r[("quantile", name)]
        has = torch.repeat_interleave(count > 0, lengths, output_size=n)
        res = torch.repeat_interleave(outs[j], lengths, output_size=n)
        if cont:
            return res.contiguous(), has.to(torch.uint8), pa.float64(), None
        (g,), (gv,) = K.gather_rows([c], [m], res.contiguous(), want_valid=True)
        return g, gv, tp, base.dictionaries.get(name)

    return run


def _ewm_decay(t: B200Table, node: ColumnExpr) -> Tuple[float, bool, int, float]:
    """(alpha, adjust, positions, 1 / halflife) of an EWM node for ``K.segmented_ewm``: pandas' alpha, and for a time
    decay the halflife as a number (whole or not) of units of the single ascending order column of ``t``."""
    kw = node.kwargs
    if not kw["times"]:
        return ewm_alpha(kw), kw["adjust"], K.EWM_OBSERVATIONS if kw["ignore_na"] else K.EWM_ROWS, 1.0
    name = _ewm_time_column(t, node)
    tp = t.schema[name].type
    h = kw["halflife"]
    if pa.types.is_integer(tp):
        if isinstance(h, datetime.timedelta):
            raise ValueError(f"{node}: a timedelta halflife needs a temporal order column; {name} is {tp}")
        units = float(h)
    else:
        if not isinstance(h, datetime.timedelta):
            raise ValueError(f"{node}: the temporal order column {name} ({tp}) needs a timedelta halflife, got {h!r}")
        # any number of units, whole or not: only the scale 1 / halflife reaches the device
        unit = "D" if pa.types.is_date32(tp) else ("ms" if pa.types.is_date64(tp) else tp.unit)
        us = h // datetime.timedelta(microseconds=1)
        units = us * 1000.0 if unit == "ns" else us / (86_400_000_000 if unit == "D" else _TIME_UNIT_US[unit])
    return ewm_alpha(kw), kw["adjust"], K.EWM_TIMES, 1.0 / units


def _ewm_time_column(t: B200Table, node: Any = None) -> str:
    """The order column of a time decay: the single ascending presort (or ORDER BY) column of ``t``, an integer, date,
    timestamp or duration column."""
    order = list(getattr(t, "logical_order", None) or [])
    if len(order) != 1:
        raise ValueError(f"{node}: time decay needs exactly one presort / ORDER BY column, got {order}")
    if not (getattr(t, "logical_ascending", None) or [True])[0]:
        raise ValueError(f"{node}: time decay needs ascending times; {order[0]} is sorted descending")
    tp = t.schema[order[0]].type
    if order[0] in t.dictionaries or not (pa.types.is_integer(tp) or pa.types.is_date(tp) or
                                          pa.types.is_timestamp(tp) or pa.types.is_duration(tp)):
        raise ValueError(f"{node}: time decay needs an integer or temporal order column; {order[0]} is {tp}")
    return order[0]


def _ewm_times(t: B200Table) -> torch.Tensor:
    """The time-decay order column of ``t`` as contiguous int64; ValueError for a NULL time."""
    i = t.schema.index_of_key(_ewm_time_column(t))
    if t.valid[i] is not None and not bool(t.valid[i].all()):
        raise ValueError(f"time decay needs non-NULL times; {t.schema.names[i]} holds a NULL")
    return widen(t.columns[i], t.schema.types[i]).contiguous()


_TIME_UNIT_US = {"s": 1_000_000, "ms": 1_000, "us": 1}  # microseconds per unit ("ns": 1 / 1000)


def _range_offsets(t: B200Table, frame: Tuple[Any, Any]) -> Tuple[Optional[int], Any, Any]:
    """A ``range=(start, end)`` frame against the presort of ``t``: ``(key class, start, end)`` with the
    offsets in the presort column's storage units (int) or as floats, or ``(None, start, end)`` when every
    bound is CURRENT ROW (0) or UNBOUNDED (None), which needs no offset arithmetic and works with any presort.
    Raises ValueError for a frame the presort cannot serve."""
    if all(b is None or b == 0 for b in frame):
        return (None,) + tuple(frame)
    order = list(getattr(t, "logical_order", None) or [])
    if len(order) != 1:
        raise ValueError(f"a RANGE frame with an offset needs exactly one presort column, got {order}: {frame}")
    name = order[0]
    tp = t.schema[name].type
    temporal = pa.types.is_date(tp) or pa.types.is_timestamp(tp) or pa.types.is_duration(tp) or \
        pa.types.is_time64(tp)
    if name in t.dictionaries or not (pa.types.is_integer(tp) or pa.types.is_floating(tp) or temporal):
        raise ValueError(f"a RANGE frame with an offset needs a numeric or temporal presort column; {name} is {tp}")
    if pa.types.is_floating(tp):
        cls = K.RANGE_KEY_F64
    else:
        cls = K.RANGE_KEY_U64 if pa.types.is_unsigned_integer(tp) else K.RANGE_KEY_I64
    unit = "D" if pa.types.is_date32(tp) else ("ms" if pa.types.is_date64(tp) else getattr(tp, "unit", None))

    def offset(b: Any) -> Any:
        if b is None:
            return None
        if isinstance(b, datetime.timedelta):
            if not temporal:
                raise ValueError(f"a timedelta RANGE offset needs a temporal presort column; {name} is {tp}")
            us = b // datetime.timedelta(microseconds=1)
            if unit == "ns":
                return us * 1000
            per = 86_400_000_000 if unit == "D" else _TIME_UNIT_US[unit]
            if us % per:
                raise ValueError(f"RANGE offset {b} is not a whole number of {unit} units of {name} ({tp})")
            return us // per
        if cls == K.RANGE_KEY_F64:
            try:
                return float(b)
            except OverflowError as e:
                raise ValueError(f"RANGE offset {b} does not fit a float64 key ({name} is {tp})") from e
        if isinstance(b, float):
            raise ValueError(f"a float RANGE offset {b} on the {tp} presort column {name}: give an int")
        return b

    start, end = offset(frame[0]), offset(frame[1])
    for b in (start, end):
        if b is not None and cls != K.RANGE_KEY_F64 and not -(1 << 63) <= b < (1 << 63):
            raise ValueError(f"RANGE offset {b} on {name} ({tp}) is outside the int64 range")
    return cls, start, end


_INT_RANGE = {8: (-(1 << 7), 1 << 7), 16: (-(1 << 15), 1 << 15), 32: (-(1 << 31), 1 << 31), 64: (-(1 << 63), 1 << 63)}


def offset_default(default: Any, tp: pa.DataType, what: Any) -> Optional[int]:
    """The storage of LAG / LEAD's ``default`` in a column of type ``tp``, as the unsigned integer of the storage's
    bits (None for a string column, whose dictionary code is found when the gather runs).  The default is converted
    as a literal in a CAST to ``tp`` would be: float16 / float32 round to nearest, once, from the float64 value (a
    NaN keeps its sign and the top bits of its payload, as ``table.narrow``), integers take the type's range (uint64
    all of ``[0, 2^64)``), bool takes True / False, a date or timestamp column takes DATE / TIMESTAMP literals in its
    own units (a naive timestamp is UTC, an aware one is converted to UTC), a duration column a timedelta.  A default
    the type cannot hold raises ValueError: a non-integer number for an integer column, an integer out of range (of
    float64 too, for a float column), a number for a temporal column, a temporal literal that is not a whole number of
    the column's units, a string for a column that is not a string, anything but a string for one that is."""
    from .expr import _in_unit, time_unit

    def bad(why: str) -> ValueError:
        return ValueError(f"{what}: the default {default!r} {why} ({tp})")

    if pa.types.is_string(tp) or pa.types.is_large_string(tp):
        if not isinstance(default, str):
            raise bad("is not a string, the column is")
        return None
    width = _storage_dtype(tp).itemsize * 8
    if isinstance(default, str):
        raise bad("is a string, the column is not")
    if pa.types.is_boolean(tp):
        if not isinstance(default, bool):
            raise bad("is not a boolean")
        return int(default)
    if isinstance(default, bool):
        raise bad("is a boolean, the column is not")
    if pa.types.is_floating(tp):
        if not isinstance(default, (int, float)):
            raise bad("is not a number")
        try:
            x = float(default)
        except OverflowError as e:
            raise bad("is out of the float64 range") from e
        if tp == pa.float16() and not math.isnan(x):
            # numpy's float64 -> half rounds once; torch's CPU conversion rounds twice, through float32
            with np.errstate(over="ignore"):
                return int(np.array([x], np.float64).astype(np.float16).view(np.uint16)[0])
        v = torch.tensor([x], dtype=torch.float64)
        return int(narrow(v, tp).view(_BITS[width])[0]) & ((1 << width) - 1)
    unit = time_unit(tp)
    if unit is not None:
        kind, code = unit
        if not isinstance(default, (datetime.date, datetime.timedelta)) or \
                (kind == "span") != isinstance(default, datetime.timedelta):
            raise bad("is not a " + ("timedelta" if kind == "span" else "DATE or TIMESTAMP literal"))
        if isinstance(default, datetime.datetime) and default.tzinfo is not None:
            default = default.astimezone(datetime.timezone.utc).replace(tzinfo=None)
        v, exact = _in_unit(default, code)
        if not exact:
            raise bad("is not a whole number of the column's units")
        lo, hi = _INT_RANGE[width]
    elif pa.types.is_integer(tp):
        if isinstance(default, float):
            if not default.is_integer():
                raise bad("is not an integer")
            default = int(default)
        if not isinstance(default, int):
            raise bad("is not an integer")
        v = default
        lo, hi = (0, 1 << tp.bit_width) if pa.types.is_unsigned_integer(tp) else _INT_RANGE[tp.bit_width]
    else:
        raise bad("has no conversion to the column's type")
    if not lo <= v < hi:
        raise bad("is out of the column's range")
    return v & ((1 << width) - 1)


_BITS = {8: torch.uint8, 16: torch.int16, 32: torch.int32, 64: torch.int64}


def _offset_value(base: B200Table, bare: ColumnExpr, arg_name: Dict[str, str], rows: torch.Tensor,
                  seg_first: Any, seg_last: Any) -> Any:
    """LAG / LEAD: a gather of the row ``n`` before / after, NULL (then ``default``) across a partition bound.
    The default is converted to the argument's type here, when the plan is built (``offset_default``); ``n`` is
    clamped to the row count, so that ``rows + n`` cannot wrap: every ``n`` at or past a partition's length gives
    the default on all its rows."""
    name = arg_name[bare.arg.fingerprint()]
    ci = base.schema.index_of_key(name)
    c, m, tp = base.columns[ci], base.valid[ci], base.schema.types[ci]
    k, default = min(bare.kwargs["n"], int(rows.shape[0])), bare.kwargs["default"]
    d = base.dictionaries.get(name)
    bits = None if default is None else offset_default(default, tp, bare)

    def run(_: Any) -> Any:
        if bare.func == "LAG":
            src = rows - k
            ok = src >= seg_first()
        else:
            src = rows + k
            ok = src <= seg_last()
        idx = torch.where(ok, src, torch.full_like(src, -1)).contiguous()
        (g,), (gv,) = K.gather_rows([c], [m], idx, want_valid=True)
        dd = d
        if default is not None:
            if dd is not None:
                hit = dd.index(default).as_py() if len(dd) > 0 else -1
                if hit is None or hit < 0:
                    hit = len(dd)
                    dd = pa.concat_arrays([dd, pa.array([default], type=dd.type)])
                fill = torch.full_like(g, hit)
            else:
                gb = g.view(_BITS[g.element_size() * 8])
                signed = bits - (1 << (8 * g.element_size())) if gb.dtype != torch.uint8 and \
                    bits >= (1 << (8 * g.element_size() - 1)) else bits
                fill = torch.full_like(gb, signed).view(g.dtype)
            g = torch.where(ok, g, fill).contiguous()
            gv = torch.where(ok, gv, torch.ones_like(gv)).contiguous()
        return g, gv, tp, dd

    return run
