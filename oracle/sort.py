"""Oracle: exact CPU reference for the device sort, the logical partitions and ``take`` (numpy only).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Every column becomes a pair per row: a NULL flag and the dense rank of the value among the column's valid values
(``np.unique(..., return_inverse=True)``).  Ranks are exact for every storage type:

* integers on their int64 / uint64 values (no detour through float64, so exact near 2^63 and for uint64 >= 2^63);
* floats with -0.0 read as 0.0, and NaN of either sign (any payload) read as NULL (DESIGN §7d);
* strings as Python ``str``, i.e. in code-point order (the order of their UTF-8 bytes);
* bool, date and timestamp on their integer storage.

``argsort`` is ``np.lexsort`` over the (flag, rank) pairs, the least significant column first and the row number
last of all, so it is a stable row permutation.  DESC negates the rank; ``na_position`` places the flag.
``group_heads`` and ``take`` use the same pairs: NULL == NULL, a NaN is NULL, -0.0 == 0.0.  ``take`` is
``native_execution_engine.py:350-384``: a stable sort, then the first ``n`` rows of every ``groupby(dropna=False)``
group, in sorted order.
"""
from collections import OrderedDict
from typing import List, Sequence, Tuple

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc


def _array(table: pa.Table, name: str) -> pa.Array:
    a = table.column(name).combine_chunks()
    if pa.types.is_dictionary(a.type):
        a = a.cast(a.type.value_type)
    return a


def null_and_rank(table: pa.Table, name: str) -> Tuple[np.ndarray, np.ndarray]:
    """(bool NULL flag, int64 dense rank among the valid values; 0 under NULL) of one column."""
    a = _array(table, name)
    n, tp = len(a), a.type
    null = np.zeros(n, dtype=bool) if a.null_count == 0 else \
        ~np.asarray(pc.is_valid(a).to_numpy(zero_copy_only=False), dtype=bool)
    if pa.types.is_string(tp) or pa.types.is_large_string(tp):
        vals = np.array(["" if x is None else x for x in a.to_pylist()], dtype=object)
    elif pa.types.is_floating(tp):
        vals = np.asarray(a.cast(pa.float64()).fill_null(0.0).to_numpy(zero_copy_only=False), dtype=np.float64)
        null = null | np.isnan(vals)
        vals = np.where(vals == 0, 0.0, vals)  # -0.0 -> 0.0
    elif pa.types.is_boolean(tp):
        vals = np.asarray(a.fill_null(False).to_numpy(zero_copy_only=False), dtype=np.int64)
    elif pa.types.is_unsigned_integer(tp):
        vals = np.asarray(a.fill_null(0).to_numpy(zero_copy_only=False)).astype(np.uint64)
    elif pa.types.is_integer(tp):
        vals = np.asarray(a.fill_null(0).to_numpy(zero_copy_only=False)).astype(np.int64)
    elif pa.types.is_temporal(tp):  # date / timestamp / duration: their integer storage
        store = pa.int32() if tp.bit_width == 32 else pa.int64()
        vals = np.asarray(a.view(store).fill_null(0).to_numpy(zero_copy_only=False)).astype(np.int64)
    else:
        raise NotImplementedError(f"oracle sort of {tp}")
    rank = np.zeros(n, dtype=np.int64)
    ok = ~null
    if ok.any():
        _, inv = np.unique(vals[ok], return_inverse=True)
        rank[ok] = inv.reshape(-1)
    return null, rank


def argsort(table: pa.Table, sorts: "OrderedDict[str, bool]", na_position: str = "last") -> np.ndarray:
    """Stable row permutation that sorts ``table`` by ``sorts`` (name -> ascending)."""
    if na_position not in ("first", "last"):
        raise ValueError(na_position)
    n = table.num_rows
    keys: List[np.ndarray] = [np.arange(n, dtype=np.int64)]  # least significant: the row number (stability)
    for name, asc in reversed(list(sorts.items())):
        null, rank = null_and_rank(table, name)
        keys.append(rank if asc else -rank)
        keys.append(~null if na_position == "first" else null)
    return np.lexsort(keys).astype(np.int64) if n else np.zeros(0, dtype=np.int64)


def group_heads(table: pa.Table, keys: Sequence[str]) -> np.ndarray:
    """For a table in which equal key tuples are adjacent: True at the first row of every group."""
    n = table.num_rows
    head = np.zeros(n, dtype=bool)
    if n == 0:
        return head
    head[0] = True
    for name in keys:
        null, rank = null_and_rank(table, name)
        head[1:] |= (null[1:] != null[:-1]) | (~null[1:] & (rank[1:] != rank[:-1]))
    return head


def logical_offsets(table: pa.Table, keys: Sequence[str]) -> np.ndarray:
    """int64 offsets (groups + 1) of the groups of a key-sorted table."""
    return np.concatenate([np.flatnonzero(group_heads(table, keys)), [table.num_rows]]).astype(np.int64)


def group_ids(table: pa.Table, keys: Sequence[str]) -> np.ndarray:
    """Dense group number per row (groups numbered in ascending key order, NULLs last)."""
    n = table.num_rows
    order = argsort(table, OrderedDict((k, True) for k in keys))
    gid = np.empty(n, dtype=np.int64)
    gid[order] = np.cumsum(group_heads(table.take(pa.array(order)), keys)) - 1
    return gid


def take(table: pa.Table, n: int, sorts: "OrderedDict[str, bool]", na_position: str,
         partition_by: Sequence[str]) -> pa.Table:
    """First ``n`` rows after a stable sort by ``sorts``, per group of ``partition_by`` when given."""
    order = argsort(table, sorts, na_position)
    if len(partition_by) == 0:
        return table.take(pa.array(order[:max(n, 0)], type=pa.int64()))
    g = group_ids(table, partition_by)[order]
    by_group = np.argsort(g, kind="stable")  # rows of a group together, still in sorted order
    gs = g[by_group]
    first = np.concatenate([[True], gs[1:] != gs[:-1]]) if len(gs) else np.zeros(0, dtype=bool)
    starts = np.flatnonzero(first)
    within = np.arange(len(gs)) - np.repeat(starts, np.diff(np.concatenate([starts, [len(gs)]])))
    keep = np.zeros(len(order), dtype=bool)
    keep[by_group] = within < n
    return table.take(pa.array(order[keep], type=pa.int64()))
