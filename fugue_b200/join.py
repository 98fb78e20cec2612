"""Device join driver for ``B200ExecutionEngine.join`` (kernels: csrc/fb_join.cu).

Reference semantics:
  * schema rule ``get_join_schemas``   fugue/dataframe/utils.py:152-226
  * join types / NULL keys             fugue/execution/native_execution_engine.py:230-241,
                                       fugue_test/execution_suite.py:366-543
"""
import datetime
from collections import OrderedDict
from typing import Any, List, Optional, Tuple

import pyarrow as pa
import pyarrow.compute as pc
import torch

from . import kernels as K
from .dataframe import B200DataFrame
from .schema import Schema, SchemaError
from .sort import _unsigned_order_key, argsort_rows, float_key, float_key_valid, group_starts, take_rows
from .table import B200Table, widen

_JOIN_TYPES = ["semi", "left_semi", "anti", "left_anti", "inner", "left_outer", "right_outer",
               "full_outer", "cross"]


def get_join_schemas(df1: Any, df2: Any, how: str, on: Optional[List[str]]) -> Tuple[Schema, Schema]:
    """(key schema, output schema) - fugue/dataframe/utils.py:152-226."""
    assert how is not None, "how can't be None"
    how = how.lower()
    if how not in _JOIN_TYPES:
        if how == "outer":
            raise ValueError("'how' must use left_outer, right_outer, full_outer for outer joins")
        raise ValueError(f"{how} is not a valid join type")
    on = list(on) if on is not None else []
    if len(on) != len(set(on)):
        raise AssertionError(f"{on} has duplication")
    if how != "cross" and len(on) == 0:
        other = set(df2.columns)
        on = [c for c in df1.columns if c in other]
        if len(on) == 0:
            raise SchemaError(f"no common columns between {df1.columns} and {df2.columns}")
    schema2 = df2.schema
    if how in ["semi", "left_semi", "anti", "left_anti"]:
        schema2 = schema2.extract(on)
    if not (on in df1.schema and on in schema2):
        raise SchemaError(f"{on} is not the intersection of {df1.schema} & {df2.schema}")
    for k in on:
        if df1.schema[k].type != schema2[k].type:
            raise SchemaError(f"join key {k} has different types: {df1.schema[k].type} vs {schema2[k].type}")
    cm = df1.schema.intersect(on)
    if how == "cross":
        cs = df1.schema.intersect(schema2.names)
        if len(cs) > 0:
            raise SchemaError(f"invalid cross join, two dataframes have common columns {cs}")
    elif len(on) == 0:
        raise SchemaError("join on columns must be specified")
    else:  # the output holds one column of each name: a common column must be a key
        cs = [c for c in df1.schema.names if c in schema2.names and c not in on]
        if len(cs) > 0:
            raise SchemaError(f"{cs} are in both dataframes but not join keys {on}")
    return cm, df1.schema.union(schema2)


def _key64(t1: B200Table, t2: B200Table, keys: List[str]):
    """One 8-byte surrogate key per row on both sides + validity (NULL in any key -> never matches).
    A NaN in a float key counts as NULL: it never matches, on either key path, as in the reference, where
    pandas holds NULL as NaN.  exact == False means the surrogate is a hash and matches must be verified."""
    def cols_of(t: B200Table, remap=None):
        out, val = [], None
        for k in keys:
            i = t.schema.index_of_key(k)
            c, tp = t.columns[i], t.schema.types[i]
            if pa.types.is_floating(tp):  # bits with -0.0 read as 0.0; a NaN clears the row's validity
                c, not_nan = float_key(c, tp, None)
                if not_nan is not None:
                    val = not_nan if val is None else val & not_nan
            if remap is not None and k in remap:
                m = remap[k]
                c = m[c.long().clamp(min=0)]
                bad = (c < 0).to(torch.uint8) ^ 1
                val = bad if val is None else val & bad
            out.append(c.contiguous())
            if t.valid[i] is not None:
                val = t.valid[i] if val is None else val & t.valid[i]
        return out, val

    # string keys: translate the right side's dictionary codes into the left side's code space
    remap = {}
    for k in keys:
        if k in t1.dictionaries or k in t2.dictionaries:
            d1, d2 = t1.dictionaries[k], t2.dictionaries[k]
            pos = pc.index_in(d2, value_set=d1).fill_null(-1)
            remap[k] = torch.from_numpy(pos.to_numpy(zero_copy_only=False).astype("int32")).to(t2.device)
    c1, v1 = cols_of(t1)
    c2, v2 = cols_of(t2, remap)
    if len(keys) == 1 and c1[0].element_size() == 8:
        return c1[0].view(torch.int64), v1, c2[0].view(torch.int64), v2, True
    if len(keys) == 1:
        return c1[0].to(torch.int64), v1, c2[0].to(torch.int64), v2, True
    return K.row_hash64(c1), v1, K.row_hash64(c2), v2, False


def _verify(t1: B200Table, t2: B200Table, keys: List[str], li: torch.Tensor, ri: torch.Tensor):
    """Drop hash-collision candidates of a multi-column key (both indices >= 0)."""
    ok = torch.ones(li.shape[0], dtype=torch.bool, device=li.device)
    for k in keys:
        a = t1.column(k)[li]
        b = t2.column(k)[ri]
        if k in t1.dictionaries:  # compare decoded codes through the left dictionary
            d1, d2 = t1.dictionaries[k], t2.dictionaries[k]
            pos = pc.index_in(d2, value_set=d1).fill_null(-1)
            m = torch.from_numpy(pos.to_numpy(zero_copy_only=False).astype("int32")).to(li.device)
            b = m[b.long()]
        tp = t1.schema[k].type
        if pa.types.is_floating(tp):  # compare values: -0.0 == 0.0, also for float16 (stored as int16)
            a, b = widen(a, tp), widen(b, tp)
        ok &= a == b
    return ok


RADIX_JOIN_MIN_ROWS = 2_000_000
RADIX_JOIN_PARTITIONS = 256


def _radix_partition(t: B200Table, key64: torch.Tensor, kvalid: Optional[torch.Tensor], num: int):
    """Hash-partition the surrogate key together with every column (and mask) of the table, so
    that build, probe and the output gathers all walk the data partition by partition
    (radix join: the hash table and the gathered rows stay L2-resident)."""
    cols: List[torch.Tensor] = [key64]
    index = {}
    for i, c in enumerate(t.columns):
        index[("c", i)] = len(cols)
        cols.append(c)
    for i, v in enumerate(t.valid):
        if v is not None:
            index[("v", i)] = len(cols)
            cols.append(v)
    if kvalid is not None:
        index["kv"] = len(cols)
        cols.append(kvalid)
    out, part_offsets = K.partition_columns(cols, [0], num, [kvalid])
    pt = B200Table(t.schema, [out[index[("c", i)]] for i in range(len(t.columns))],
                   [out[index[("v", i)]] if ("v", i) in index else None for i in range(len(t.columns))],
                   t.dictionaries)
    return pt, out[0], (out[index["kv"]] if kvalid is not None else None), part_offsets


def device_join(engine: Any, df1: B200DataFrame, df2: B200DataFrame, how: str,
                on: Optional[List[str]]) -> B200DataFrame:
    key_schema, out_schema = get_join_schemas(df1, df2, how, on)
    how = how.lower()
    keys = key_schema.names
    t1, t2 = df1.native, df2.native
    dev = t1.device
    n1, n2 = t1.num_rows, t2.num_rows
    if how == "cross":
        total = n1 * n2
        o = torch.arange(total, dtype=torch.int64, device=dev)
        li, ri = (o // max(n2, 1)), (o % max(n2, 1))
        return _assemble(t1, t2, keys, out_schema, li, ri, how)
    k1, v1, k2, v2, exact = _key64(t1, t2, keys)
    if getattr(t1, "global_num_partitions", None) or getattr(t2, "global_num_partitions", None):
        k1, k2 = K.scramble64(k1), K.scramble64(k2)  # shuffled input: see kernels.scramble64
    parts = 0
    po1 = po2 = None
    if min(n1, n2) >= RADIX_JOIN_MIN_ROWS:
        parts = RADIX_JOIN_PARTITIONS
        t1, k1, v1, po1 = _radix_partition(t1, k1, v1, parts)
        t2, k2, v2, po2 = _radix_partition(t2, k2, v2, parts)
    if how in ("semi", "left_semi", "anti", "left_anti"):
        if exact:
            counts = K.JoinTable(k2, v2, parts, po2).probe_counts(k1, v1, outer=False)
            hit = counts > 0
        else:
            li, ri = K.JoinTable(k2, v2, parts, po2).probe(k1, v1, outer=False)
            ok = _verify(t1, t2, keys, li, ri)
            hit = torch.zeros(n1, dtype=torch.bool, device=dev)
            hit[li[ok]] = True
        keep = hit if how in ("semi", "left_semi") else ~hit
        li = K.compact_indices((keep).contiguous())
        cols, valid = K.gather_rows(t1.columns, t1.valid, li, want_valid=False)
        return B200DataFrame(B200Table(out_schema, cols, valid, t1.dictionaries))
    if exact and how in ("inner", "left_outer") and n2 < (1 << 31) \
            and len(t1.columns) + sum(v is not None for v in t1.valid) <= K.JOIN2_MAX_COLS \
            and len(t2.columns) <= K.JOIN2_MAX_COLS:
        return _fused_join(t1, t2, keys, out_schema, k1, v1, k2, v2, parts, po2, how == "left_outer", po1)
    if how == "right_outer":
        # probe with the right side so that every right row appears
        tab = K.JoinTable(k1, v1, parts, po1)
        ri, li = tab.probe(k2, v2, outer=True)
        if not exact:
            li, ri = _drop_collisions(t1, t2, keys, li, ri, outer_side="right")
        return _assemble(t1, t2, keys, out_schema, li, ri, how)
    tab = K.JoinTable(k2, v2, parts, po2)
    li, ri = tab.probe(k1, v1, outer=how in ("left_outer", "full_outer"))
    if not exact:
        li, ri = _drop_collisions(t1, t2, keys, li, ri, outer_side="left" if how != "inner" else None)
    if how == "full_outer":
        matched = tab.matched_mask(ri) if exact else _matched_mask(n2, ri)
        extra = K.compact_indices((matched == 0).contiguous())
        li = torch.cat([li, torch.full_like(extra, -1)])
        ri = torch.cat([ri, extra])
    return _assemble(t1, t2, keys, out_schema, li, ri, how)


def _fused_join(t1: B200Table, t2: B200Table, keys: List[str], out_schema: Schema, k1: torch.Tensor,
                v1: Optional[torch.Tensor], k2: torch.Tensor, v2: Optional[torch.Tensor], parts: int,
                po2: Optional[torch.Tensor], outer: bool, po1: Optional[torch.Tensor] = None) -> B200DataFrame:
    """Inner / left outer join on one 8-byte key through the fused kernels (K.join_fused): the probe
    side's columns (and validity masks, as 1-byte columns) are copied, the build side's non-key columns
    are gathered - straight into the output table."""
    left: List[torch.Tensor] = list(t1.columns)
    lmask_at = {}
    for i, v in enumerate(t1.valid):
        if v is not None:
            lmask_at[i] = len(left)
            left.append(v)
    names2 = [n for n in t2.schema.names if n not in keys]
    idx2 = [t2.schema.index_of_key(n) for n in names2]
    louts, routs, rvout, _ = K.join_fused(k1.contiguous(), v1, k2.contiguous(), v2, left,
                                          [t2.columns[i] for i in idx2], [t2.valid[i] for i in idx2], outer, parts, po2, po1)
    ncol1 = len(t1.columns)
    lvalid = [louts[lmask_at[i]] if i in lmask_at else None for i in range(ncol1)]
    dicts = dict(t1.dictionaries)
    dicts.update({n: t2.dictionaries[n] for n in names2 if n in t2.dictionaries})
    return B200DataFrame(B200Table(out_schema, louts[:ncol1] + routs, lvalid + rvout, dicts))


def _matched_mask(n: int, ri: torch.Tensor) -> torch.Tensor:
    m = torch.zeros(n, dtype=torch.uint8, device=ri.device)
    m[ri[ri >= 0]] = 1
    return m


def _drop_collisions(t1, t2, keys, li, ri, outer_side):
    both = (li >= 0) & (ri >= 0)
    ok = torch.ones_like(both)
    if bool(both.any()):
        ok[both] = _verify(t1, t2, keys, li[both], ri[both])
    if outer_side is None:
        return li[ok], ri[ok]
    # a false candidate of an outer join degrades to "unmatched" unless the row has a true match
    probe = li if outer_side == "left" else ri
    n = (t1 if outer_side == "left" else t2).num_rows
    has = torch.zeros(n, dtype=torch.bool, device=li.device)
    has[probe[ok & both]] = True
    keep = ok.clone()
    bad = ~ok
    first_bad = torch.zeros_like(bad)
    if bool(bad.any()):
        # keep one NULL-extended row for probe rows that lost all their candidates
        idx = K.compact_indices((bad).contiguous())
        rows = probe[idx]
        lost = ~has[rows]
        uniq, inv = torch.unique(rows[lost], return_inverse=True)
        firsts = torch.full((uniq.numel(),), li.numel(), dtype=torch.int64, device=li.device)
        firsts.scatter_reduce_(0, inv, idx[lost], reduce="amin")
        first_bad[firsts] = True
    keep |= first_bad
    li, ri = li.clone(), ri.clone()
    if outer_side == "left":
        ri[first_bad] = -1
    else:
        li[first_bad] = -1
    return li[keep], ri[keep]


ASOF_JOIN_TYPES = ["inner", "left_outer"]
ASOF_DIRECTIONS = {"backward": K.ASOF_BACKWARD, "forward": K.ASOF_FORWARD, "nearest": K.ASOF_NEAREST}


def get_asof_schemas(df1: Any, df2: Any, on: Optional[List[str]], asof: str) -> Tuple[List[str], Schema]:
    """(equality keys, output schema) of an as-of join.  ``on=None`` takes every common column but ``asof``; an
    empty list is one group.  The output is ``df1.schema`` followed by df2's columns other than the keys and
    ``asof``; any other common column raises SchemaError, as ``get_join_schemas`` does."""
    if not isinstance(asof, str):
        raise ValueError(f"asof must be one column name, got {asof!r}")
    if on is None:
        other = set(df2.columns)
        on = [c for c in df1.columns if c in other and c != asof]
    on = list(on)
    if len(on) != len(set(on)):
        raise AssertionError(f"{on} has duplication")
    if asof in on:
        raise ValueError(f"the as-of column {asof} is also an equality key {on}")
    for k in on + [asof]:
        if k not in df1.schema or k not in df2.schema:
            raise SchemaError(f"{k} is not in both {df1.schema} and {df2.schema}")
        if df1.schema[k].type != df2.schema[k].type:
            raise SchemaError(f"join key {k} has different types: {df1.schema[k].type} vs {df2.schema[k].type}")
    names2 = [n for n in df2.schema.names if n not in on and n != asof]
    common = [n for n in names2 if n in df1.schema]
    if common:
        raise SchemaError(f"{common} are common columns of {df1.schema} and {df2.schema} but not join keys")
    return on, Schema(df1.schema, df2.schema.extract(names2))


def asof_key_class(name: str, tp: pa.DataType, is_string: bool, what: str = "an as-of column") -> int:
    """The ``RANGE_KEY_*`` class of an as-of column: the key types RANGE frames take; anything else is a ValueError."""
    temporal = pa.types.is_date(tp) or pa.types.is_timestamp(tp) or pa.types.is_duration(tp) or \
        pa.types.is_time64(tp)
    if is_string or not (pa.types.is_integer(tp) or pa.types.is_floating(tp) or temporal):
        raise ValueError(f"{what} must be numeric or temporal; {name} is {tp}")
    if pa.types.is_floating(tp):
        return K.RANGE_KEY_F64
    return K.RANGE_KEY_U64 if pa.types.is_unsigned_integer(tp) else K.RANGE_KEY_I64


def asof_tolerance(name: str, tp: pa.DataType, tolerance: Any) -> Any:
    """``tolerance`` in the as-of column's units, by the rules of a RANGE frame's offset (``colmap._range_offsets``):
    an int in storage units, a float for float columns, a timedelta as a whole number of the column's units.
    None stays None; a negative tolerance is a ValueError."""
    from types import SimpleNamespace

    from .colmap import _range_offsets
    from .column import _range_frame

    if tolerance is None:
        return None
    tol = _range_frame((tolerance, tolerance))[0]
    if tol == 0:
        return 0.0 if pa.types.is_floating(tp) else 0
    if (tol.total_seconds() if isinstance(tol, datetime.timedelta) else tol) < 0:
        raise ValueError(f"tolerance must be >= 0, got {tolerance!r}")
    presort = SimpleNamespace(logical_order=[name], schema=Schema([pa.field(name, tp)]), dictionaries={})
    return _range_offsets(presort, (tol, tol))[1]  # type: ignore[arg-type]


def device_asof_join(df1: B200DataFrame, df2: B200DataFrame, on: Optional[List[str]], asof: str, how: str = "inner",
                     direction: str = "backward", allow_exact_matches: bool = True,
                     tolerance: Any = None) -> B200DataFrame:
    """As-of join (``pandas.merge_asof`` semantics, DESIGN §7q): every left row, in input order, with the right
    row of equal key whose ``asof`` value is the latest at or before its own (``backward``), the earliest at or
    after (``forward``) or the closer of those two (``nearest``, ties to the backward one)."""
    how = how.lower() if isinstance(how, str) else how
    if how not in ASOF_JOIN_TYPES:
        raise ValueError(f"an as-of join is {' or '.join(ASOF_JOIN_TYPES)}, got {how!r}")
    if direction not in ASOF_DIRECTIONS:
        raise ValueError(f"direction must be one of {list(ASOF_DIRECTIONS)}, got {direction!r}")
    if not isinstance(allow_exact_matches, bool):
        raise ValueError(f"allow_exact_matches must be a bool, got {allow_exact_matches!r}")
    keys, out_schema = get_asof_schemas(df1, df2, on, asof)
    t1, t2 = df1.native, df2.native
    tp = t1.schema[asof].type
    cls = asof_key_class(asof, tp, asof in t1.dictionaries or asof in t2.dictionaries)
    tol = asof_tolerance(asof, tp, tolerance)
    return _asof_assemble(t1, t2, keys, out_schema, asof_rows(t1, t2, keys, asof, cls, direction,
                                                                allow_exact_matches, tol), how)


def _asof_value(t: B200Table, name: str, cls: int) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """Order codes of an as-of column and its validity (a float NaN is NULL)."""
    i = t.schema.index_of_key(name)
    v = t.valid[i]
    if cls == K.RANGE_KEY_F64:
        v = float_key_valid(widen(t.columns[i], t.schema.types[i]), v)
    return _unsigned_order_key(t, name, True), v


def sorted_runs(t1: B200Table, t2: B200Table, keys: List[str], by: str,
                values: List[Tuple[torch.Tensor, Optional[torch.Tensor]]], keep: Optional[torch.Tensor] = None
                ) -> Optional[Tuple[torch.Tensor, List[torch.Tensor], torch.Tensor, torch.Tensor]]:
    """Steps 1 and 2 of the as-of and range joins (DESIGN §7q, §7r).  ``values`` are (order codes, validity) of
    df2's value columns, ``by`` first.  1: the right rows that can match - a valid key, every value valid, and
    ``keep`` (uint8, None: all) - sorted by (keys..., by) with the stable ``argsort_rows``.  2: the runs of equal
    keys, and every left row's run through a ``JoinTable`` over the run heads.  Returns None when no right row is
    kept, else (the kept right rows in sorted order, each value's codes in that order, per left row its run or -1,
    the runs' int64 offsets)."""
    dev = t1.device
    n1, n2 = t1.num_rows, t2.num_rows
    # 1. right side: drop the rows that can never match, sort the rest by (keys..., by), stable
    if keys:
        k1, v1, k2, v2, exact = _key64(t1, t2, keys)
        keep = v2 if keep is None else (keep if v2 is None else v2 & keep)
    for _, av2 in values:
        keep = av2 if keep is None else (keep if av2 is None else keep & av2)
    kept = torch.arange(n2, dtype=torch.int64, device=dev) if keep is None else K.compact_indices(keep.contiguous())
    sub = take_rows(B200Table(t2.schema.extract(keys + [by]), [t2.column(k) for k in keys + [by]],
                              [t2.valid[t2.schema.index_of_key(k)] for k in keys + [by]],
                              {k: t2.dictionaries[k] for k in keys if k in t2.dictionaries}), kept)
    if kept.shape[0] == 0:
        return None
    perm = argsort_rows(sub, OrderedDict([(k, True) for k in keys] + [(by, True)]))
    rows = kept[perm].contiguous()
    codes = [c[rows].contiguous() for c, _ in values]
    # 2. runs of equal keys, and every left row's run
    if keys:
        heads = K.compact_indices(group_starts(take_rows(sub, perm), keys).contiguous())
        head_rows = rows[heads]
        tab = K.JoinTable(k2[head_rows].contiguous(), None)
        if exact:  # one surrogate per key value: the first match is the run
            run = torch.empty(n1, dtype=torch.int64, device=dev)
            tab.probe_counts(k1.contiguous(), v1, outer=False, first=run)
        else:  # hashed surrogates: a candidate run counts only if its head has the row's key values
            li, ri = tab.probe(k1.contiguous(), v1, outer=False)
            ok = _verify(t1, t2, keys, li, head_rows[ri])
            run = torch.full((n1,), -1, dtype=torch.int64, device=dev)
            run[li[ok]] = ri[ok]
        run_offsets = torch.cat([heads, torch.tensor([rows.shape[0]], dtype=torch.int64, device=dev)])
    else:  # one group
        run = torch.zeros(n1, dtype=torch.int64, device=dev)
        run_offsets = torch.tensor([0, rows.shape[0]], dtype=torch.int64, device=dev)
    return rows, codes, run, run_offsets.contiguous()


def asof_rows(t1: B200Table, t2: B200Table, keys: List[str], asof: str, cls: int, direction: str,
              allow_exact_matches: bool, tolerance: Any) -> torch.Tensor:
    """Per left row, the right row it matches, -1 for none (int64)."""
    dev = t1.device
    n1 = t1.num_rows
    if n1 == 0:
        return torch.empty(0, dtype=torch.int64, device=dev)
    runs = sorted_runs(t1, t2, keys, asof, [_asof_value(t2, asof, cls)])
    if runs is None:
        return torch.full((n1,), -1, dtype=torch.int64, device=dev)
    rows, (codes,), run, run_offsets = runs
    # 3. the search
    c1, av1 = _asof_value(t1, asof, cls)
    return K.asof_search(run, run_offsets, c1, av1, codes, rows, cls, ASOF_DIRECTIONS[direction],
                         allow_exact_matches, tolerance)


def _asof_assemble(t1: B200Table, t2: B200Table, keys: List[str], out_schema: Schema, match: torch.Tensor,
                   how: str) -> B200DataFrame:
    """df1's rows (all, or the matched ones for ``inner``) with df2's output columns gathered from their match."""
    names2 = out_schema.names[len(t1.columns):]
    idx2 = [t2.schema.index_of_key(n) for n in names2]
    lcols, lvalid = list(t1.columns), list(t1.valid)
    if how == "inner":
        li = K.compact_indices((match >= 0).contiguous())
        lcols, lvalid = K.gather_rows(lcols, lvalid, li, want_valid=False)
        match = match[li].contiguous()
    rcols, rvalid = K.gather_rows([t2.columns[i] for i in idx2], [t2.valid[i] for i in idx2], match,
                                  want_valid=how == "left_outer")
    dicts = dict(t1.dictionaries)
    dicts.update({n: t2.dictionaries[n] for n in names2 if n in t2.dictionaries})
    return B200DataFrame(B200Table(out_schema, lcols + rcols, lvalid + rvalid, dicts))


def _assemble(t1: B200Table, t2: B200Table, keys: List[str], out_schema: Schema, li: torch.Tensor,
              ri: torch.Tensor, how: str) -> B200DataFrame:
    """Gather the output columns: df1's columns, then df2's non-key columns; key columns of
    NULL-extended left rows (right/full outer) come from the right side."""
    l_null = how in ("right_outer", "full_outer")
    r_null = how in ("left_outer", "full_outer")
    lcols, lvalid = K.gather_rows(t1.columns, t1.valid, li, want_valid=l_null)
    names2 = [n for n in t2.schema.names if n not in keys]
    idx2 = [t2.schema.index_of_key(n) for n in names2]
    rcols, rvalid = K.gather_rows([t2.columns[i] for i in idx2], [t2.valid[i] for i in idx2], ri,
                                  want_valid=r_null)
    dicts = dict(t1.dictionaries)
    dicts.update({n: t2.dictionaries[n] for n in names2 if n in t2.dictionaries})
    if l_null and len(keys) > 0:
        kidx2 = [t2.schema.index_of_key(k) for k in keys]
        kc, kv = K.gather_rows([t2.columns[i] for i in kidx2], [t2.valid[i] for i in kidx2], ri, want_valid=True)
        from_right = li < 0
        for k, c2, v2 in zip(keys, kc, kv):
            i1 = t1.schema.index_of_key(k)
            if k in t1.dictionaries:  # translate right codes into the left dictionary, extending it
                d1, d2 = t1.dictionaries[k], t2.dictionaries[k]
                merged = pa.concat_arrays([d1, d2.filter(pc.invert(pc.is_in(d2, value_set=d1)))])
                pos = pc.index_in(d2, value_set=merged)
                m = torch.from_numpy(pos.to_numpy(zero_copy_only=False).astype("int32")).to(li.device)
                c2 = m[c2.long().clamp(min=0)]
                dicts[k] = merged
            lcols[i1] = torch.where(from_right, c2.to(lcols[i1].dtype), lcols[i1])
            lvalid[i1] = torch.where(from_right, v2, lvalid[i1])
    return B200DataFrame(B200Table(out_schema, lcols + rcols, lvalid + rvalid, dicts))


RANGE_JOIN_TYPES = ["inner", "left_outer"]
RANGE_CLOSED = {"both": K.RANGE_CLOSED_LEFT | K.RANGE_CLOSED_RIGHT, "left": K.RANGE_CLOSED_LEFT,
                "right": K.RANGE_CLOSED_RIGHT, "neither": 0}
_SIGN64 = -(1 << 63)


def get_range_schemas(df1: Any, df2: Any, on: Optional[List[str]], at: str, start: str,
                      end: str) -> Tuple[List[str], Schema]:
    """(equality keys, output schema) of a range join.  ``on=None`` takes every common column but ``at``; an empty
    list is one group.  ``at`` is a column of df1, ``start`` and ``end`` (possibly one column) of df2, all of one
    type.  The output is ``df1.schema`` followed by df2's columns other than the keys (``start`` and ``end``
    included); any other common column raises SchemaError, as ``get_asof_schemas`` does."""
    for arg, name in (("at", at), ("start", start), ("end", end)):
        if not isinstance(name, str):
            raise ValueError(f"{arg} must be one column name, got {name!r}")
    if on is None:
        other = set(df2.columns)
        on = [c for c in df1.columns if c in other and c != at]
    on = list(on)
    if len(on) != len(set(on)):
        raise AssertionError(f"{on} has duplication")
    for name in (at, start, end):
        if name in on:
            raise ValueError(f"the range column {name} is also an equality key {on}")
    for k in on:
        if k not in df1.schema or k not in df2.schema:
            raise SchemaError(f"{k} is not in both {df1.schema} and {df2.schema}")
        if df1.schema[k].type != df2.schema[k].type:
            raise SchemaError(f"join key {k} has different types: {df1.schema[k].type} vs {df2.schema[k].type}")
    if at not in df1.schema:
        raise SchemaError(f"{at} is not in {df1.schema}")
    for name in (start, end):
        if name not in df2.schema:
            raise SchemaError(f"{name} is not in {df2.schema}")
        if df2.schema[name].type != df1.schema[at].type:
            raise SchemaError(f"range columns have different types: {at} is {df1.schema[at].type}, {name} is "
                              f"{df2.schema[name].type}")
    names2 = [n for n in df2.schema.names if n not in on]
    common = [n for n in names2 if n in df1.schema]
    if common:
        raise SchemaError(f"{common} are common columns of {df1.schema} and {df2.schema} but not join keys")
    return on, Schema(df1.schema, df2.schema.extract(names2))


def device_range_join(df1: B200DataFrame, df2: B200DataFrame, on: Optional[List[str]], at: str, start: str,
                      end: str, how: str = "inner", closed: str = "both") -> B200DataFrame:
    """Range join (DESIGN §7r): every left row, in input order, with every right row of equal key whose interval
    [start, end] (sides open or closed by ``closed``: both, left, right, neither) holds its ``at`` value, in
    ascending (start, right input order)."""
    how = how.lower() if isinstance(how, str) else how
    if how not in RANGE_JOIN_TYPES:
        raise ValueError(f"a range join is {' or '.join(RANGE_JOIN_TYPES)}, got {how!r}")
    if not isinstance(closed, str) or closed not in RANGE_CLOSED:
        raise ValueError(f"closed must be one of {list(RANGE_CLOSED)}, got {closed!r}")
    keys, out_schema = get_range_schemas(df1, df2, on, at, start, end)
    t1, t2 = df1.native, df2.native
    is_string = at in t1.dictionaries or start in t2.dictionaries or end in t2.dictionaries
    cls = asof_key_class(at, t1.schema[at].type, is_string, "a range column")
    li, ri = range_pairs(t1, t2, keys, at, start, end, cls, RANGE_CLOSED[closed], how == "left_outer")
    return _assemble(t1, t2, keys, out_schema, li, ri, how)


def range_pairs(t1: B200Table, t2: B200Table, keys: List[str], at: str, start: str, end: str, cls: int, closed: int,
                outer: bool) -> Tuple[torch.Tensor, torch.Tensor]:
    """The (left row, right row) pairs of a range join in output order; right row -1 for an unmatched left row of
    an outer join."""
    dev = t1.device
    n1 = t1.num_rows
    if n1 == 0:
        return torch.empty(0, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.int64, device=dev)
    # 1-2. the intervals that can match (valid bounds, start <= end) sorted by (keys..., start), and the runs
    s2 = _asof_value(t2, start, cls)
    e2 = s2 if end == start else _asof_value(t2, end, cls)
    ordered = ((s2[0] ^ _SIGN64) <= (e2[0] ^ _SIGN64)).to(torch.uint8)
    runs = sorted_runs(t1, t2, keys, start, [s2, e2], ordered)
    if runs is None:
        if outer:
            return torch.arange(n1, dtype=torch.int64, device=dev), torch.full((n1,), -1, dtype=torch.int64, device=dev)
        return torch.empty(0, dtype=torch.int64, device=dev), torch.empty(0, dtype=torch.int64, device=dev)
    rows, (starts, ends), run, run_offsets = runs
    # 3. the MAX tree over the end codes, sign-flipped so that the signed MAX orders them
    ends = (ends ^ _SIGN64).contiguous()
    tree = K.window_tree(K.AGG_MAX_I64, ends)
    # 4-6. count, offsets, emit
    c1, av1 = _asof_value(t1, at, cls)
    counts = K.range_join_count(run, run_offsets, c1, av1, starts, ends, tree, closed, outer)
    offsets, total = K.exclusive_scan(counts)
    return K.range_join_emit(run, run_offsets, c1, av1, starts, ends, tree, rows, closed, outer, counts, offsets,
                             total)

