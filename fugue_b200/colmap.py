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
import struct
from typing import Any, Dict, List, Optional, Tuple

import pyarrow as pa
import torch

from . import kernels as K
from .column import ColumnExpr, Kind, SelectColumns, col as _col, has_window, is_agg
from .table import B200Table


def _f64_bits(v: float) -> int:
    return struct.unpack("<Q", struct.pack("<d", float(v)))[0]


class ColumnMap:
    def __init__(self, *columns: Any):
        assert len(columns) > 0, "ColumnMap needs at least one output column"
        self.columns: List[ColumnExpr] = [_col(c) for c in columns]
        for c in self.columns:
            if is_agg(c):
                raise ValueError(f"{c} is an aggregation: a map is row-wise")
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
    by the evaluator (K8), running / partition aggregates and ranks by the segmented scan (K9), FIRST /
    LAST / partition values / LAG / LEAD by row gathers."""
    from . import expr as X
    from . import sort as S
    from .schema import Schema
    from .table import _storage_dtype

    nodes: Dict[str, ColumnExpr] = {}
    for c in cols:
        _collect_windows(c, nodes)
    n, dev = t.num_rows, t.device
    # ---- arguments: plain columns as they are, anything else through one evaluator pass
    pre = [_col(nm) for nm in t.schema.names]
    arg_name: Dict[str, str] = {}
    for bare in nodes.values():
        if not bare.args or bare.arg.kind == Kind.WILDCARD:
            continue
        a = bare.arg
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

    # ---- scans: collected first, all run in one call
    scans: List[Any] = []
    finish: List[Any] = []     # per node: (fingerprint, fn(scan results) -> (column, validity, type, dictionary))

    def scan(op: int, v: Any, m: Any) -> int:
        scans.append((op, v, m))
        return len(scans) - 1

    for uid, bare in nodes.items():
        fn = bare.func
        if fn in ("LAG", "LEAD"):
            finish.append((uid, _offset_value(base, bare, arg_name, rows, seg_first, seg_last)))
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
        running = bare.kwargs["running"]
        whole = None if running else seg_last

        def at_end(x: torch.Tensor, whole: Any = whole) -> torch.Tensor:  # partition value: the scan at its last row
            return x if whole is None else x[whole()]

        if bare.arg.kind == Kind.WILDCARD:  # COUNT(*)
            i = scan(K.AGG_COUNT, None, None)
            finish.append((uid, lambda r, i=i, e=at_end: (e(r[i][1]), None, pa.int64(), None)))
            continue
        name = arg_name[bare.arg.fingerprint()]
        ci = base.schema.index_of_key(name)
        c, m, tp = base.columns[ci], base.valid[ci], base.schema.types[ci]
        if fn == "COUNT":
            i = scan(K.AGG_COUNT, None, m)
            finish.append((uid, lambda r, i=i, e=at_end: (e(r[i][1]), None, pa.int64(), None)))
            continue
        if fn in ("FIRST", "LAST"):
            # first / last valid row so far: MIN / MAX of the row number over the valid rows, then a gather
            i = scan(K.AGG_MIN_I64 if fn == "FIRST" else K.AGG_MAX_I64, rows, m)

            def pick(r: Any, i: int = i, e: Any = at_end, c: Any = c, m: Any = m, tp: Any = tp, name: str = name) -> Any:
                idx = torch.where(e(r[i][1]) > 0, e(r[i][0]), torch.full_like(rows, -1))
                (g,), (gv,) = K.gather_rows([c], [m], idx.contiguous(), want_valid=True)
                return g, gv, tp, base.dictionaries.get(name)

            finish.append((uid, pick))
            continue
        if name in base.dictionaries:
            raise NotImplementedError(f"{fn} on a string column: {bare}")
        is_f = pa.types.is_floating(tp)
        if fn in ("SUM", "AVG"):
            f64 = fn == "AVG" or is_f
            v8 = c.to(torch.float64 if f64 else torch.int64).contiguous()
            i = scan(K.AGG_SUM_F64 if f64 else K.AGG_SUM_I64, v8, m)
            out_tp = pa.float64() if f64 else pa.int64()

            def total(r: Any, i: int = i, e: Any = at_end, avg: bool = fn == "AVG", out_tp: Any = out_tp) -> Any:
                v, cnt = e(r[i][0]), e(r[i][1])
                if avg:
                    v = v / cnt.to(torch.float64)
                return v.contiguous(), (cnt > 0).to(torch.uint8), out_tp, None

            finish.append((uid, total))
            continue
        if fn in ("MIN", "MAX"):
            v8 = c if c.element_size() == 8 else c.to(torch.float64 if is_f else torch.int64).contiguous()
            op = {("MIN", True): K.AGG_MIN_F64, ("MAX", True): K.AGG_MAX_F64,
                  ("MIN", False): K.AGG_MIN_I64, ("MAX", False): K.AGG_MAX_I64}[(fn, is_f)]
            i = scan(op, v8, m)

            def extreme(r: Any, i: int = i, e: Any = at_end, tp: Any = tp, dt: Any = c.dtype) -> Any:
                v, cnt = e(r[i][0]), e(r[i][1])
                return v.to(dt).contiguous(), (cnt > 0).to(torch.uint8), tp, None

            finish.append((uid, extreme))
            continue
        raise NotImplementedError(f"window function {fn}")  # pragma: no cover - builders admit no other
    results = K.segmented_scan(off.contiguous(), n, scans) if scans else []
    names, types, columns, valid = list(base.schema.names), list(base.schema.types), list(base.columns), list(base.valid)
    dicts = dict(base.dictionaries)
    window_names: Dict[str, str] = {}
    for uid, fn in finish:
        c, v, tp, d = fn(results)
        nm = f"__fb_w{len(window_names)}"
        window_names[uid] = nm
        names.append(nm)
        types.append(tp)
        columns.append(c if c.dtype == _storage_dtype(tp) else c.to(_storage_dtype(tp)))
        valid.append(v)
        if d is not None:
            dicts[nm] = d
    out = _WindowTable(Schema([pa.field(a, b) for a, b in zip(names, types)]), columns, valid, dicts)
    out.window_names = window_names
    return out


def _offset_value(base: B200Table, bare: ColumnExpr, arg_name: Dict[str, str], rows: torch.Tensor,
                  seg_first: Any, seg_last: Any) -> Any:
    """LAG / LEAD: a gather of the row ``n`` before / after, NULL (then ``default``) across a partition bound."""
    name = arg_name[bare.arg.fingerprint()]
    ci = base.schema.index_of_key(name)
    c, m, tp = base.columns[ci], base.valid[ci], base.schema.types[ci]
    k, default = bare.kwargs["n"], bare.kwargs["default"]

    def run(_: Any) -> Any:
        if bare.func == "LAG":
            src = rows - k
            ok = src >= seg_first()
        else:
            src = rows + k
            ok = src <= seg_last()
        idx = torch.where(ok, src, torch.full_like(src, -1)).contiguous()
        (g,), (gv,) = K.gather_rows([c], [m], idx, want_valid=True)
        d = base.dictionaries.get(name)
        if default is not None:
            if d is not None:
                if not isinstance(default, str):
                    raise NotImplementedError(f"non-string default of {bare} on a string column")
                hit = d.index(default).as_py() if len(d) > 0 else -1
                if hit is None or hit < 0:
                    hit = len(d)
                    d = pa.concat_arrays([d, pa.array([default], type=d.type)])
                fill = torch.full_like(g, hit)
            elif isinstance(default, str):
                raise NotImplementedError(f"string default of {bare} on a {tp} column")
            else:
                fill = torch.full((), default, dtype=torch.float64 if isinstance(default, float) else torch.int64,
                                  device=g.device).to(g.dtype).expand_as(g)
            g = torch.where(ok, g, fill).contiguous()
            gv = torch.where(ok, gv, torch.ones_like(gv)).contiguous()
        return g, gv, tp, d

    return run
