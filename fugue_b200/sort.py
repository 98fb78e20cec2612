"""Device sort (LSD radix passes of the partition kernels), logical partitions, ``take``.

Reference semantics:
  * presort inside a partition   fugue/execution/native_execution_engine.py:107-115, 157-160
                                 (``pdf.sort_values(presort_keys, ascending=...)``)
  * ``take``                     fugue/execution/native_execution_engine.py:350-384
                                 (sort with ``na_position`` then ``head(n)`` per group; NULL keys form
                                 a group: ``groupby(dropna=False)``)
  * logical partitions           one per distinct key tuple, NULLs grouped (SURVEY.md 3.2)

A column becomes an order-preserving UNSIGNED 64-bit key (sign bit flipped for signed ints, the
usual total-order transform for floats - with NaN as NULL and -0.0 as 0.0, see ``float_key_bits`` -,
dictionary rank for strings, complement for DESC); (key,
row index) pairs are sorted with one stable 8-bit radix pass (``fb_radix_pass``) per varying byte, the
least significant sort column first; NULLS FIRST/LAST is one more pass on the validity flag.  The
payload is gathered once at the end (``fb_gather_rows``).  Key preparation uses torch integer ops on
the device; the passes and the gather are the library's kernels.
"""
from collections import OrderedDict
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import torch

from . import _lib
from . import kernels as K
from .table import B200Table, widen

_SIGN = -(1 << 63)


# Float sort and grouping keys (DESIGN §7d): a NaN of either sign is NULL, and -0.0 equals 0.0.  Only the
# order and the grouping follow this rule; the rows keep their own bits.
def float_key_bits(c: torch.Tensor) -> torch.Tensor:
    """Bit pattern (int64 for float64, int32 for float32) of a float key column, -0.0 read as 0.0."""
    z = torch.where(c == 0, torch.zeros_like(c), c)
    return z.view(torch.int64 if c.dtype == torch.float64 else torch.int32)


def float_key_valid(c: torch.Tensor, v: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """Validity (uint8) of a float key column with NaN rows cleared; None when every row is valid."""
    ok = c == c
    if v is not None:
        return v & ok.to(torch.uint8)
    return None if bool(ok.all()) else ok.to(torch.uint8)


def float_key(c: torch.Tensor, tp: pa.DataType,
              v: Optional[torch.Tensor]) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """(bits, validity) of a stored float key column of arrow type ``tp`` under §7d.  float16 (stored as int16) is
    widened to float64 first, exactly, so its bits are int64; float32 / float64 keep their width."""
    w = widen(c, tp) if tp == pa.float16() else c
    return float_key_bits(w), float_key_valid(w, v)


def dictionary_order(d: pa.Array) -> np.ndarray:
    """The entries of a string dictionary in code-point (UTF-8 byte) order, as their codes; NULL entries last.
    The position of an entry's code here is its rank."""
    return pc.sort_indices(d).to_numpy()


def _unsigned_order_key(t: B200Table, name: str, ascending: bool) -> torch.Tensor:
    """int64 tensor whose bit pattern, read as unsigned, orders like the column."""
    i = t.schema.index_of_key(name)
    c, tp = t.columns[i], t.schema.types[i]
    if name in t.dictionaries:  # strings: rank of every dictionary entry in sorted order
        d = t.dictionaries[name]
        order = dictionary_order(d)
        rank = np.empty(len(d), dtype=np.int64)
        rank[order] = np.arange(len(d), dtype=np.int64)
        r = torch.from_numpy(rank).to(c.device)
        key = r[c.long().clamp(min=0)] if len(d) > 0 else torch.zeros_like(c, dtype=torch.int64)
    elif pa.types.is_floating(tp):
        b = float_key_bits(widen(c, tp))
        key = b ^ ((b >> 63) | _SIGN)  # negative: flip all bits; non-negative: flip the sign bit
    elif tp in (pa.uint8(), pa.bool_()):
        key = c.to(torch.int64)
    elif tp == pa.uint16():
        key = c.to(torch.int64) & 0xFFFF
    elif tp == pa.uint32():
        key = c.to(torch.int64) & 0xFFFFFFFF
    elif tp == pa.uint64():
        key = c  # the int64 bit view already is the unsigned value
    else:  # signed integers, dates, timestamps
        key = c.to(torch.int64) ^ _SIGN
    if not ascending:
        key = ~key
    return key.contiguous()


def string_ranks(t: B200Table, name: str) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """A string column as the rank of every row's dictionary entry (int64, see ``dictionary_order``) and its
    validity: a NULL row or a row whose entry is NULL is not valid (None: every row is valid).  MIN / MAX of
    the ranks are MIN / MAX of the strings in code-point order; ``codes_of_ranks`` maps them back."""
    i = t.schema.index_of_key(name)
    rank, v = _unsigned_order_key(t, name, True), t.valid[i]
    d = t.dictionaries[name]
    if d.null_count > 0:
        ok = torch.from_numpy(d.is_valid().to_numpy(zero_copy_only=False).astype(np.uint8)).to(rank.device)
        c = t.columns[i].long()
        if v is not None:
            c = torch.where(v.bool(), c, torch.zeros_like(c))  # a NULL row's stored code means nothing
        hit = ok[c]
        v = hit if v is None else v & hit
    return rank, v


def codes_of_ranks(d: pa.Array, ranks: torch.Tensor) -> torch.Tensor:
    """The int32 codes of dictionary ``d`` whose ranks are ``ranks`` (the inverse of ``string_ranks``)."""
    if len(d) == 0:
        return torch.zeros(ranks.shape, dtype=torch.int32, device=ranks.device)
    order = torch.from_numpy(dictionary_order(d).astype(np.int32)).to(ranks.device)
    return order[ranks.clamp(0, len(d) - 1)].contiguous()


def _radix_sort_pairs(key: torch.Tensor, idx: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """Stable sort of (key, idx) pairs by the unsigned value of key; only varying bytes get a pass."""
    lib = _lib.load()
    dev = key.device
    n = int(key.shape[0])
    if n <= 1:
        return key, idx
    lo, hi = int(key.min().item()), int(key.max().item())
    diff = (lo ^ hi) & 0xFFFFFFFFFFFFFFFF
    # signed min/max are not the unsigned extremes when signs differ: then every byte may vary
    if (lo < 0) != (hi < 0):
        diff = 0xFFFFFFFFFFFFFFFF
    nbytes = (diff.bit_length() + 7) // 8
    scratch = torch.empty(K.partition_scratch_bytes(dev, n, 256) + 256, dtype=torch.uint8, device=dev)
    offsets = torch.empty(257, dtype=torch.int64, device=dev)
    k2, i2 = torch.empty_like(key), torch.empty_like(idx)
    widths = _lib.i32_array([8, 8])
    for b in range(nbytes):
        _lib.check(lib.fb_radix_pass(dev.index, K._stream_ptr(dev), n, key.data_ptr(), 8 * b, 2,
                                     _lib.ptr_array([key.data_ptr(), idx.data_ptr()]), widths,
                                     _lib.ptr_array([k2.data_ptr(), i2.data_ptr()]), scratch.data_ptr(),
                                     scratch.numel(), offsets.data_ptr()))
        key, k2 = k2, key
        idx, i2 = i2, idx
    return key, idx


def argsort_rows(t: B200Table, sorts: "OrderedDict[str, bool]", na_position: str = "last") -> torch.Tensor:
    """Row permutation that sorts the table by ``sorts`` (name -> ascending), stable."""
    if na_position not in ("first", "last"):
        raise ValueError(f"invalid na_position {na_position}")
    dev = t.device
    n = t.num_rows
    idx = torch.arange(n, dtype=torch.int64, device=dev)
    for name, asc in reversed(list(sorts.items())):
        key = _unsigned_order_key(t, name, asc)
        i = t.schema.index_of_key(name)
        v = t.valid[i]
        if pa.types.is_floating(t.schema.types[i]):
            v = float_key_valid(widen(t.columns[i], t.schema.types[i]), v)
        if v is not None:
            # the value stored under a NULL is undefined (Arrow / parquet leave garbage there): give all
            # NULL rows one constant key, so that they keep the order set by the less significant columns
            key = torch.where(v.bool(), key, torch.zeros_like(key))
        _, idx = _radix_sort_pairs(key[idx].contiguous(), idx)
        if v is not None:
            flag = v.to(torch.int64) if na_position == "first" else (1 - v.to(torch.int64))
            _, idx = _radix_sort_pairs(flag[idx].contiguous(), idx)
    return idx


def take_rows(t: B200Table, idx: torch.Tensor) -> B200Table:
    cols, valid = K.gather_rows(t.columns, t.valid, idx.contiguous(), want_valid=False)
    return B200Table(t.schema, cols, valid, t.dictionaries)


def sort_table(t: B200Table, sorts: "OrderedDict[str, bool]", na_position: str = "last") -> B200Table:
    if len(sorts) == 0 or t.num_rows <= 1:
        return t
    return take_rows(t, argsort_rows(t, sorts, na_position))


def group_starts(t: B200Table, keys: List[str]) -> torch.Tensor:
    """For a table in which equal key tuples are adjacent: bool mask, True at the first row of
    every logical partition (NULL == NULL for grouping; float keys: NaN is NULL and -0.0 equals 0.0)."""
    n = t.num_rows
    first = torch.zeros(n, dtype=torch.bool, device=t.device)
    if n == 0:
        return first
    first[0] = True
    for k in keys:
        i = t.schema.index_of_key(k)
        c, v = t.columns[i], t.valid[i]
        if pa.types.is_floating(t.schema.types[i]):
            c, v = float_key(c, t.schema.types[i], v)
        if v is None:
            diff = c[1:] != c[:-1]
        else:
            diff = (v[1:] != v[:-1]) | ((v[1:] != 0) & (c[1:] != c[:-1]))
        first[1:] |= diff
    return first


def logical_offsets(t: B200Table, keys: List[str]) -> torch.Tensor:
    """int64 offsets (length groups + 1) of the logical partitions of a key-sorted table."""
    starts = K.compact_indices((group_starts(t, keys)).contiguous())
    end = torch.tensor([t.num_rows], dtype=torch.int64, device=t.device)
    return torch.cat([starts, end])


def take(t: B200Table, n: int, sorts: "OrderedDict[str, bool]", na_position: str,
         partition_by: List[str]) -> B200Table:
    """First ``n`` rows (per logical partition when ``partition_by`` is given) after sorting."""
    if not isinstance(n, int) or isinstance(n, bool):
        raise ValueError("n needs to be an integer")
    if len(partition_by) == 0:
        s = sort_table(t, sorts, na_position)
        return s.slice(0, min(n, s.num_rows))
    full: "OrderedDict[str, bool]" = OrderedDict((k, True) for k in partition_by)
    for k, v in sorts.items():
        if k not in full:
            full[k] = v
    # group columns first (any consistent order groups equal keys; NULL keys last), presort inside
    idx = argsort_rows(t, OrderedDict((k, v) for k, v in full.items()), na_position)
    if any(k in sorts for k in partition_by):  # a partition key re-listed in presort keeps its own direction
        full2 = OrderedDict((k, sorts.get(k, True)) for k in partition_by)
        for k, v in sorts.items():
            if k not in full2:
                full2[k] = v
        idx = argsort_rows(t, full2, na_position)
    s = take_rows(t, idx)
    first = group_starts(s, partition_by)
    pos = torch.arange(s.num_rows, dtype=torch.int64, device=s.device)
    start_of = torch.cummax(torch.where(first, pos, torch.zeros_like(pos)), 0).values
    keep = K.compact_indices(((pos - start_of) < n).contiguous())
    return take_rows(s, keep)
