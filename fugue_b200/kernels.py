"""Thin tensor-level wrappers over the C ABI.

torch is used here only as the owner of device memory and streams; every
operation is a call into ``libfugue_b200.so``.
"""
import ctypes as C
import struct
from typing import Any, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib

MAX_PARTITIONS = 1024
MAX_KEYS = 8


def _stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _check_cols(cols: Sequence[torch.Tensor]) -> Tuple[torch.device, int]:
    assert len(cols) > 0, "no columns"
    dev = cols[0].device
    n = cols[0].shape[0]
    for c in cols:
        if not c.is_cuda:
            raise _lib.FugueB200KernelError("fugue_b200 kernels need CUDA tensors (no CPU path)")
        if c.device != dev or c.dim() != 1 or c.shape[0] != n or not c.is_contiguous():
            raise ValueError("columns must be 1-d contiguous tensors of equal length on one device")
        if c.element_size() not in (1, 2, 4, 8):
            raise ValueError(f"unsupported column width {c.element_size()}")
    return dev, n


def _valid_ptrs(valid: Optional[Sequence[Optional[torch.Tensor]]], nkeys: int):
    if valid is None or all(v is None for v in valid):
        return None
    assert len(valid) == nkeys
    for v in valid:
        if v is not None:
            assert v.dtype == torch.uint8 and v.is_contiguous() and v.is_cuda
    return _lib.ptr_array([0 if v is None else v.data_ptr() for v in valid])


def partition_ids(keys: Sequence[torch.Tensor], num: int,
                  valid: Optional[Sequence[Optional[torch.Tensor]]] = None) -> torch.Tensor:
    """K1: ``hash_pandas_object(df[keys], index=False) % num`` per row (int32 tensor)."""
    lib = _lib.load()
    dev, n = _check_cols(keys)
    out = torch.empty(n, dtype=torch.int32, device=dev)
    vp = _valid_ptrs(valid, len(keys))
    _lib.check(lib.fb_partition_ids(
        dev.index, _stream_ptr(dev), n, len(keys),
        _lib.ptr_array([k.data_ptr() for k in keys]),
        _lib.i32_array([k.element_size() for k in keys]),
        vp, num, out.data_ptr()))
    return out


def partition_scratch_bytes(device: torch.device, nrows: int, num: int) -> int:
    return int(_lib.load().fb_partition_scratch_bytes(device.index, nrows, num))


class PartitionPlan:
    """Result of pass 1 (histogram + scan): partition offsets and the chunk bases
    needed by pass 2.  Holds references to the key columns it was built from."""

    def __init__(self, keys, valid, num, scratch, offsets):
        self.keys = list(keys)
        self.valid = None if valid is None else list(valid)
        self.num = num
        self.scratch = scratch
        self.offsets = offsets  # int64 [num + 1] on device
        self.nrows = self.keys[0].shape[0]


def partition_plan(keys: Sequence[torch.Tensor], num: int,
                   valid: Optional[Sequence[Optional[torch.Tensor]]] = None,
                   scratch: Optional[torch.Tensor] = None,
                   offsets: Optional[torch.Tensor] = None) -> PartitionPlan:
    lib = _lib.load()
    dev, n = _check_cols(keys)
    need = partition_scratch_bytes(dev, n, num)
    if scratch is None or scratch.numel() < need:
        scratch = torch.empty(max(need, 256), dtype=torch.uint8, device=dev)
    if offsets is None:
        offsets = torch.empty(num + 1, dtype=torch.int64, device=dev)
    vp = _valid_ptrs(valid, len(keys))
    _lib.check(lib.fb_partition_plan(
        dev.index, _stream_ptr(dev), n, len(keys),
        _lib.ptr_array([k.data_ptr() for k in keys]),
        _lib.i32_array([k.element_size() for k in keys]),
        vp, num, scratch.data_ptr(), scratch.numel(), offsets.data_ptr()))
    return PartitionPlan(keys, valid, num, scratch, offsets)


def partition_apply(plan: PartitionPlan, cols: Sequence[torch.Tensor],
                    out: Optional[Sequence[torch.Tensor]] = None, sm_reserve: int = 0, cols_per_launch: int = 0
                    ) -> List[torch.Tensor]:
    """Pass 2 for ``cols``; ``sm_reserve`` SMs stay free for kernels that co-run (multi-GPU exchange);
    ``cols_per_launch`` is a tuning argument of the fast kernel: 8-byte columns per group, all groups in one
    launch (0 = default, 2)."""
    lib = _lib.load()
    dev, n = _check_cols(list(cols) + plan.keys)
    if out is None:
        out = [torch.empty_like(c) for c in cols]
    else:
        _check_cols(list(out) + plan.keys)
    vp = _valid_ptrs(plan.valid, len(plan.keys))
    _lib.check(lib.fb_partition_apply_ex(
        dev.index, _stream_ptr(dev), n, len(plan.keys),
        _lib.ptr_array([k.data_ptr() for k in plan.keys]),
        _lib.i32_array([k.element_size() for k in plan.keys]),
        vp, plan.num, plan.scratch.data_ptr(), plan.scratch.numel(), plan.offsets.data_ptr(),
        len(cols), _lib.ptr_array([c.data_ptr() for c in cols]),
        _lib.i32_array([c.element_size() for c in cols]),
        _lib.ptr_array([o.data_ptr() for o in out]), int(sm_reserve), int(cols_per_launch)))
    return list(out)


MAP_COPY, MAP_AFFINE_F64, MAP_AFFINE_I64 = 0, 1, 2


def partition_apply_map(plan: PartitionPlan, units: Sequence[Tuple[torch.Tensor, Optional[torch.Tensor], int, int, int, int]],
                        out: Optional[Sequence[torch.Tensor]] = None, sm_reserve: int = 0) -> List[torch.Tensor]:
    """K4: pass 2 with a fused map epilogue.  ``units`` = one ``(x, y or None, mode, a, b, c)`` per output
    column (8-byte columns; a / b / c are 64-bit patterns): ``MAP_COPY`` x, ``MAP_AFFINE_F64``
    (a*x + b*y) + c in float64, ``MAP_AFFINE_I64`` a*x + b*y + c in wrapping int64."""
    lib = _lib.load()
    xs = [u[0] for u in units]
    dev, n = _check_cols(xs + [u[1] for u in units if u[1] is not None] + plan.keys)
    assert all(c.element_size() == 8 for c in xs) and plan.num <= 256
    if out is None:
        out = [torch.empty_like(x) for x in xs]
    maps = (_lib.MapUnit * len(units))()
    for i, (x, y, mode, a, b, c) in enumerate(units):
        maps[i].src2 = 0 if y is None else y.data_ptr()
        maps[i].mode = mode
        maps[i].a, maps[i].b, maps[i].c = a & ((1 << 64) - 1), b & ((1 << 64) - 1), c & ((1 << 64) - 1)
    tail = torch.empty(int(lib.fb_partition_map_tail_bytes(len(units))), dtype=torch.uint8, device=dev)
    vp = _valid_ptrs(plan.valid, len(plan.keys))
    _lib.check(lib.fb_partition_apply_map(
        dev.index, _stream_ptr(dev), n, len(plan.keys),
        _lib.ptr_array([k.data_ptr() for k in plan.keys]),
        _lib.i32_array([k.element_size() for k in plan.keys]),
        vp, plan.num, plan.scratch.data_ptr(), plan.scratch.numel(), plan.offsets.data_ptr(),
        len(units), _lib.ptr_array([x.data_ptr() for x in xs]), _lib.ptr_array([o.data_ptr() for o in out]),
        maps, tail.data_ptr(), int(sm_reserve)))
    tail.record_stream(torch.cuda.current_stream(dev))
    return list(out)


def partition_columns(cols: Sequence[torch.Tensor], key_idx: Sequence[int], num: int,
                      key_valid: Optional[Sequence[Optional[torch.Tensor]]] = None,
                      out: Optional[Sequence[torch.Tensor]] = None,
                      scratch: Optional[torch.Tensor] = None,
                      offsets: Optional[torch.Tensor] = None
                      ) -> Tuple[List[torch.Tensor], torch.Tensor]:
    """K1+K2+K3 through ``fb_partition_cols``: stable hash partition of ``cols``."""
    lib = _lib.load()
    dev, n = _check_cols(cols)
    need = partition_scratch_bytes(dev, n, num)
    if scratch is None or scratch.numel() < need:
        scratch = torch.empty(max(need, 256), dtype=torch.uint8, device=dev)
    if offsets is None:
        offsets = torch.empty(num + 1, dtype=torch.int64, device=dev)
    if out is None:
        out = [torch.empty_like(c) for c in cols]
    vp = _valid_ptrs(key_valid, len(key_idx))
    _lib.check(lib.fb_partition_cols(
        dev.index, _stream_ptr(dev), n, len(cols),
        _lib.ptr_array([c.data_ptr() for c in cols]),
        _lib.i32_array([c.element_size() for c in cols]),
        _lib.i32_array(list(key_idx)), len(key_idx), vp, num,
        _lib.ptr_array([o.data_ptr() for o in out]), offsets.data_ptr(),
        scratch.data_ptr(), scratch.numel()))
    return list(out), offsets


def bits_to_bytes(bits: torch.Tensor, bit_offset: int, nrows: int) -> torch.Tensor:
    lib = _lib.load()
    out = torch.empty(nrows, dtype=torch.uint8, device=bits.device)
    _lib.check(lib.fb_bits_to_bytes(bits.device.index, _stream_ptr(bits.device), bits.data_ptr(),
                                    bit_offset, nrows, out.data_ptr()))
    return out


def bytes_to_bits(mask: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    lib = _lib.load()
    n = mask.shape[0]
    out = torch.empty((n + 7) // 8, dtype=torch.uint8, device=mask.device)
    nulls = torch.zeros(1, dtype=torch.int64, device=mask.device)
    _lib.check(lib.fb_bytes_to_bits(mask.device.index, _stream_ptr(mask.device), mask.data_ptr(), n,
                                    out.data_ptr(), nulls.data_ptr()))
    return out, nulls


def copy_segments(src_cols: Sequence[torch.Tensor], dst_cols: Sequence[torch.Tensor],
                  src_off: torch.Tensor, dst_off: torch.Tensor, seg_len: torch.Tensor,
                  max_len: Optional[int] = None, src_table: Optional[torch.Tensor] = None,
                  src_ptrs: Optional[Sequence[int]] = None) -> None:
    """For every column: dst[dst_off[s]:+len[s]] = table[src_table[s]][src_off[s]:+len[s]].
    ``src_ptrs`` (ntables x ncols raw device pointers, [table][col]) replaces ``src_cols`` when the
    sources are peer-GPU buffers mapped through symmetric memory."""
    lib = _lib.load()
    dev = dst_cols[0].device
    nseg = int(seg_len.shape[0])
    ncols = len(dst_cols)
    if nseg == 0 or ncols == 0:
        return
    ptrs = list(src_ptrs) if src_ptrs is not None else [c.data_ptr() for c in src_cols]
    ptr_src = torch.tensor(ptrs, dtype=torch.int64, device=dev)
    ptr_dst = torch.tensor([c.data_ptr() for c in dst_cols], dtype=torch.int64, device=dev)
    widths = torch.tensor([c.element_size() for c in dst_cols], dtype=torch.int32, device=dev)
    for t in (src_off, dst_off, seg_len):
        assert t.dtype == torch.int64 and t.is_cuda and t.is_contiguous()
    if max_len is None:
        max_len = int(seg_len.max().item())
    _lib.check(lib.fb_copy_segments(dev.index, _stream_ptr(dev), ncols, ptr_src.data_ptr(),
                                    ptr_dst.data_ptr(), widths.data_ptr(), nseg,
                                    0 if src_table is None else src_table.data_ptr(), src_off.data_ptr(),
                                    dst_off.data_ptr(), seg_len.data_ptr(), int(max_len)))


def copy_runs_dma(device: torch.device, src_ptrs: Any, dst_ptrs: Any, nbytes: Any) -> None:
    """``nruns`` device-to-device copies on the copy engines (numpy uint64 arrays of raw pointers /
    byte counts); sources may be peer buffers mapped through symmetric memory."""
    import numpy as np

    lib = _lib.load()
    src = np.ascontiguousarray(src_ptrs, dtype=np.uint64)
    dst = np.ascontiguousarray(dst_ptrs, dtype=np.uint64)
    nb = np.ascontiguousarray(nbytes, dtype=np.uint64)
    assert src.shape == dst.shape == nb.shape and src.ndim == 1
    if src.size == 0:
        return
    _lib.check(lib.fb_copy_runs_dma(device.index, _stream_ptr(device), int(src.size), src.ctypes.data,
                                    dst.ctypes.data, nb.ctypes.data))


def copy_runs_dma_streams(device: torch.device, src_ptrs: Any, dst_ptrs: Any, nbytes: Any, streams: Any,
                          prefer_overlap: bool = True) -> None:
    """:func:`copy_runs_dma` with one CUDA stream per run (raw ``cudaStream_t`` values): the whole
    exchange of a column group is enqueued by ONE call."""
    import numpy as np

    lib = _lib.load()
    src = np.ascontiguousarray(src_ptrs, dtype=np.uint64)
    dst = np.ascontiguousarray(dst_ptrs, dtype=np.uint64)
    nb = np.ascontiguousarray(nbytes, dtype=np.uint64)
    st = np.ascontiguousarray(streams, dtype=np.uint64)
    assert src.shape == dst.shape == nb.shape == st.shape and src.ndim == 1
    if src.size == 0:
        return
    _lib.check(lib.fb_copy_runs_dma_streams(device.index, int(src.size), src.ctypes.data, dst.ctypes.data,
                                            nb.ctypes.data, st.ctypes.data, 1 if prefer_overlap else 0))


def pull_runs_tma(device: torch.device, src_ptrs: Any, dst_ptrs: Any, nbytes: Any, max_ctas: int = 16) -> None:
    """The same runs as :func:`copy_runs_dma`, moved by the persistent TMA pull kernel on ``max_ctas`` SMs."""
    import numpy as np

    lib = _lib.load()
    src = np.ascontiguousarray(src_ptrs, dtype=np.uint64)
    dst = np.ascontiguousarray(dst_ptrs, dtype=np.uint64)
    nb = np.ascontiguousarray(nbytes, dtype=np.uint64)
    assert src.shape == dst.shape == nb.shape and src.ndim == 1
    if src.size == 0:
        return
    _lib.check(lib.fb_pull_runs_tma(device.index, _stream_ptr(device), int(src.size), src.ctypes.data,
                                    dst.ctypes.data, nb.ctypes.data, int(max_ctas)))


# A table that went through the multi-GPU shuffle holds, on every rank, only keys whose partitioner hash % N
# falls into the rank's range.  Local radix partitions of the same keys by the same hash would then fill only
# a fraction of their partitions (and overflow the hash-table regions sized for an even spread).  Local
# operators therefore hash a bijective re-coding of such keys: k * odd constant (mod 2^64) - equal keys stay
# equal, the partition ids become independent of the shuffle's.
_SCRAMBLE = 0x9E3779B97F4A7C15 - (1 << 64)
_UNSCRAMBLE = pow(0x9E3779B97F4A7C15, -1, 1 << 64) - (1 << 64)


def scramble64(k: torch.Tensor) -> torch.Tensor:
    return k * _SCRAMBLE


def unscramble64(k: torch.Tensor) -> torch.Tensor:
    return k * _UNSCRAMBLE


AGG_SUM_F64, AGG_SUM_I64, AGG_COUNT, AGG_MIN_I64, AGG_MAX_I64, AGG_MIN_F64, AGG_MAX_F64 = range(7)
# group-by only: deviations from the group mean (sum of d and of d * d, d = x - SUM / COUNT); each needs an
# AGG_SUM_F64 of the same f64 column and validity and an AGG_COUNT of the same validity in the same call
AGG_DEV_F64, AGG_DEV2_F64 = 7, 8
# group-by only: cross deviations of a pair (sum of dx * dy over the rows where the pair validity is set).  An
# AGG_CODEV_F64 names x and the pair validity; the AGG_DEV_F64 right after it names y with the same validity, and
# the call needs AGG_SUM_F64 of x and of y and an AGG_COUNT, all of that same validity tensor
AGG_CODEV_F64 = 9
# group-by only: sums of d^3 and d^4, tied like AGG_DEV2_F64 to the AGG_SUM_F64 and AGG_COUNT of their column
AGG_DEV3_F64, AGG_DEV4_F64 = 10, 11
MAX_AGGS = 16


GROUPBY_PARTITION_MIN_ROWS = 4_000_000   # below this the table fits in L2 anyway
GROUPBY_PARTITIONS = 256
# initialise + aggregate the table in L2-sized batches of regions (fb_groupby_u64 d_part_offsets): off, because
# the group-by's atomics are bound by the L2 atomic rate, not by DRAM, so batching did not pay
GROUPBY_BATCHED = False


def groupby_u64(keys: torch.Tensor, key_valid: Optional[torch.Tensor],
                vals: Sequence[Optional[torch.Tensor]], val_valid: Sequence[Optional[torch.Tensor]],
                ops: Sequence[int], capacity: Optional[int] = None, max_capacity: Optional[int] = None,
                partition: Optional[bool] = None
                ) -> Tuple[torch.Tensor, Optional[torch.Tensor], List[torch.Tensor], int]:
    """K6: hash group-by of an 8-byte key column with up to ``MAX_AGGS`` (16) aggregates.
    Returns (group keys, key validity or None, aggregate columns as int64 bit patterns, ngroups)."""
    lib = _lib.load()
    dev, n = _check_cols([keys])
    assert keys.element_size() == 8 and len(vals) == len(ops) == len(val_valid) <= MAX_AGGS
    for v in vals:
        assert v is None or (v.element_size() == 8 and v.is_cuda and v.is_contiguous() and v.shape[0] == n)
    naggs = len(ops)
    num_parts = 0
    part_offsets = None
    if partition is None:
        partition = n >= GROUPBY_PARTITION_MIN_ROWS
    if partition and n > 0:
        # radix-partition (key, values, masks) on the key first: rows of one partition are then
        # contiguous and the aggregation sweeps the hash table region by region (L2-resident)
        uniq: List[torch.Tensor] = [keys]
        for t in list(vals) + [key_valid] + list(val_valid):
            if t is not None and all(t.data_ptr() != u.data_ptr() for u in uniq):
                uniq.append(t)
        pout, part_offsets = partition_columns(uniq, [0], GROUPBY_PARTITIONS, [key_valid])
        remap = {u.data_ptr(): o for u, o in zip(uniq, pout)}
        keys = remap[keys.data_ptr()]
        key_valid = None if key_valid is None else remap[key_valid.data_ptr()]
        vals = [None if v is None else remap[v.data_ptr()] for v in vals]
        val_valid = [None if v is None else remap[v.data_ptr()] for v in val_valid]
        num_parts = GROUPBY_PARTITIONS
    if n == 0:  # nothing to aggregate: no groups
        e = torch.empty(0, dtype=torch.int64, device=dev)
        return (e, None if key_valid is None else torch.empty(0, dtype=torch.uint8, device=dev),
                [e.clone() for _ in range(naggs)], 0)
    hard_max = 1 << max(1, (2 * max(n, 1) - 1).bit_length())   # >= 2n: every row may be its own group
    if max_capacity is not None:
        hard_max = min(hard_max, max_capacity)
    if capacity is None:
        capacity = min(hard_max, 1 << 25)
        if part_offsets is not None and n >= (1 << 22):
            # size the table from the data: count the distinct keys of ONE hash partition exactly (1/256 of
            # the rows, a few hundred kilobytes) and scale up.  A table of the right size halves the init and
            # extract passes and keeps a region L2-resident; an under-estimate only costs the retry below.
            po = part_offsets[:2].tolist()
            if po[1] - po[0] >= 1024:
                _, _, _, d0 = groupby_u64(keys[po[0]:po[1]], None if key_valid is None else key_valid[po[0]:po[1]],
                                          [], [], [], partition=False)
                est = int(d0 * num_parts * 1.6) + 1024   # load factor <= ~0.62
                capacity = max(1 << 16, min(hard_max, 1 << (est - 1).bit_length()))
    capacity = max(2, 1 << (int(capacity) - 1).bit_length())
    status = torch.zeros(4, dtype=torch.int64, device=dev)
    vp = _lib.ptr_array([0 if v is None else v.data_ptr() for v in vals])
    vv = _lib.ptr_array([0 if v is None else v.data_ptr() for v in val_valid])
    opa = _lib.i32_array(list(ops))
    while True:
        nbytes = int(lib.fb_groupby_table_bytes(capacity, naggs))
        table = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        parts = num_parts if capacity >= 2 * max(num_parts, 1) else 0
        _lib.check(lib.fb_groupby_u64(dev.index, _stream_ptr(dev), n, keys.data_ptr(),
                                      0 if key_valid is None else key_valid.data_ptr(), naggs, vp, vv, opa,
                                      capacity, parts, table.data_ptr(), status.data_ptr(),
                                      part_offsets.data_ptr() if (part_offsets is not None and GROUPBY_BATCHED)
                                      else 0))
        # extract right away and read overflow flag + group count with ONE host sync (an overflowing attempt
        # wastes its extract; that is the rare path)
        bound = min(n, capacity) + 2  # upper bound on the number of groups
        out_keys = torch.empty(bound, dtype=torch.int64, device=dev)
        out_valid = torch.empty(bound, dtype=torch.uint8, device=dev) if key_valid is not None else None
        out_aggs = [torch.empty(bound, dtype=torch.int64, device=dev) for _ in range(naggs)]
        d_ptrs = torch.tensor([a.data_ptr() for a in out_aggs] or [0], dtype=torch.int64, device=dev)
        _lib.check(lib.fb_groupby_extract(dev.index, _stream_ptr(dev), capacity, naggs, opa, table.data_ptr(),
                                          out_keys.data_ptr(), 0 if out_valid is None else out_valid.data_ptr(),
                                          d_ptrs.data_ptr(), status.data_ptr()))
        overflow, ngroups = (int(x) for x in status[:2].tolist())
        if overflow == 0:
            break
        del table, out_keys, out_valid, out_aggs
        if parts > 0:
            # Region mode gives every hash partition capacity / num_parts slots.  Keys concentrated in a few
            # partitions (say, the input is one partition of an earlier 256-way hash partition) overflow their
            # region however large the table grows.  Retry at this capacity with ONE region over the whole
            # table and keep it (the rows may stay partitioned: the whole-table kernel does not care).
            num_parts = 0
            continue
        if capacity >= hard_max:
            raise _lib.FugueB200KernelError("group-by hash table overflow at the maximum capacity")
        capacity *= 4
    return (out_keys[:ngroups], None if out_valid is None else out_valid[:ngroups],
            [a[:ngroups] for a in out_aggs], ngroups)


SCAN_MAX_COLS = 8


def _segments(offsets: torch.Tensor) -> Tuple[torch.device, int]:
    assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous()
    return offsets.device, int(offsets.shape[0]) - 1


def _check_rows(t: Optional[torch.Tensor], dev: torch.device, nrows: int, dtype: Optional[torch.dtype] = None) -> None:
    """``t`` is None or a contiguous column of ``nrows`` values on ``dev``: of ``dtype``, or of any 8-byte type."""
    if t is not None:
        assert (t.element_size() == 8 if dtype is None else t.dtype == dtype)
        assert t.device == dev and t.is_contiguous() and t.shape[0] == nrows


def _ptrs(ts: Sequence[Optional[torch.Tensor]]) -> Any:
    return _lib.ptr_array([0 if t is None else t.data_ptr() for t in ts])


def _batched(items: Sequence[Any], dev: torch.device, outputs: Any, scratch_bytes: Any, launch: Any) -> List[Any]:
    """Runs ``items`` ``SCAN_MAX_COLS`` at a time: per batch, ``outputs(*item)`` allocates each item's output tensors,
    ``scratch_bytes(n)`` sizes the scratch of n items, and ``launch(batch, outs, scratch)`` calls the kernel with
    ``outs[k]``, the pointer array of every item's k-th output.  Returns the outputs per item."""
    res: List[Any] = []
    for b in range(0, len(items), SCAN_MAX_COLS):
        batch = items[b:b + SCAN_MAX_COLS]
        outs = [outputs(*it) for it in batch]
        nb = int(scratch_bytes(len(batch)))
        scratch = torch.empty(max(nb, 8), dtype=torch.uint8, device=dev)
        _lib.check(launch(batch, [_ptrs(o) for o in zip(*outs)], scratch))
        res.extend(outs)
    return res


def _op_batched(columns: Sequence[Tuple[int, Optional[torch.Tensor], Optional[torch.Tensor]]], nrows: int,
                dev: torch.device, scratch_bytes: Any, launch: Any) -> List[Tuple[Optional[torch.Tensor], torch.Tensor]]:
    """:func:`_batched` over ``(op, values or None, validity or None)`` columns with ``(values, count)`` outputs:
    ``launch(n, ops, vals, valid, out_vals, out_count, scratch, scratch_bytes)``."""

    def outputs(op: int, v: Optional[torch.Tensor], m: Optional[torch.Tensor]) -> Tuple[Optional[torch.Tensor], torch.Tensor]:
        assert (v is None) == (op == AGG_COUNT)
        _check_rows(v, dev, nrows)
        _check_rows(m, dev, nrows, torch.uint8)
        return None if v is None else torch.empty_like(v), torch.empty(nrows, dtype=torch.int64, device=dev)

    return _batched(columns, dev, outputs, scratch_bytes, lambda batch, outs, scratch: launch(
        len(batch), _lib.i32_array([op for op, _, _ in batch]), _ptrs([v for _, v, _ in batch]),
        _ptrs([m for _, _, m in batch]), *outs, scratch.data_ptr(), scratch.numel()))


def _stat_outputs(dev: torch.device, nrows: int, nf64: int) -> Tuple[torch.Tensor, ...]:
    return (torch.empty(nrows, dtype=torch.int64, device=dev),) + tuple(
        torch.empty(nrows, dtype=torch.float64, device=dev) for _ in range(nf64))


def _value_batched(columns: Sequence[Tuple[torch.Tensor, Optional[torch.Tensor]]], nrows: int, dev: torch.device,
                   nf64: int, scratch_bytes: Any, launch: Any) -> List[Tuple[torch.Tensor, ...]]:
    """:func:`_batched` over ``(float64 values, validity or None)`` columns with a count and ``nf64`` float64 outputs:
    ``launch(n, vals, valid, out_count, *outs, scratch, scratch_bytes)``."""

    def outputs(v: torch.Tensor, m: Optional[torch.Tensor]) -> Tuple[torch.Tensor, ...]:
        _check_rows(v, dev, nrows, torch.float64)
        _check_rows(m, dev, nrows, torch.uint8)
        return _stat_outputs(dev, nrows, nf64)

    return _batched(columns, dev, outputs, scratch_bytes, lambda batch, outs, scratch: launch(
        len(batch), _ptrs([v for v, _ in batch]), _ptrs([m for _, m in batch]), *outs, scratch.data_ptr(),
        scratch.numel()))


def segmented_scan(offsets: torch.Tensor, nrows: int,
                   columns: Sequence[Tuple[int, Optional[torch.Tensor], Optional[torch.Tensor]]]
                   ) -> List[Tuple[Optional[torch.Tensor], torch.Tensor]]:
    """K9: inclusive scan restarting at every segment ``[offsets[s], offsets[s + 1])``.  ``columns`` = one
    ``(op, values or None, validity or None)`` per scan (``AGG_*`` ops; 8-byte values, none for
    ``AGG_COUNT``).  Returns per scan ``(running op over the valid rows or None for COUNT, running count of
    the valid rows)``; up to ``SCAN_MAX_COLS`` scans share one launch sequence."""
    lib = _lib.load()
    dev, nseg = _segments(offsets)
    return _op_batched(columns, nrows, dev, lambda n: lib.fb_segmented_scan_scratch_bytes(nrows, n),
                       lambda *args: lib.fb_segmented_scan(dev.index, _stream_ptr(dev), nrows, nseg,
                                                           offsets.data_ptr(), *args))


def segmented_moments(offsets: torch.Tensor, nrows: int,
                      columns: Sequence[Tuple[torch.Tensor, Optional[torch.Tensor]]]
                      ) -> List[Tuple[torch.Tensor, torch.Tensor]]:
    """K9: running moments restarting at every segment ``[offsets[s], offsets[s + 1])``.  ``columns`` = one
    ``(float64 values, validity or None)`` per column.  Returns per column ``(running count of the valid rows
    (int64), running M2 = sum of (x - mean)^2 over them (float64, 0 where the count is 0))``; up to
    ``SCAN_MAX_COLS`` columns share one launch sequence."""
    lib = _lib.load()
    dev, nseg = _segments(offsets)
    return _value_batched(columns, nrows, dev, 1, lambda n: lib.fb_segmented_moments_scratch_bytes(nrows, n),
                          lambda *args: lib.fb_segmented_moments(dev.index, _stream_ptr(dev), nrows, nseg,
                                                                 offsets.data_ptr(), *args))


def segmented_shape_moments(offsets: torch.Tensor, nrows: int,
                            columns: Sequence[Tuple[torch.Tensor, Optional[torch.Tensor]]]
                            ) -> List[Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]]:
    """K9: running shape moments restarting at every segment ``[offsets[s], offsets[s + 1])``.  ``columns`` = one
    ``(float64 values, validity or None)`` per column.  Returns per column ``(running count of the valid rows (int64),
    M2, M3, M4)``, Mk = sum of (x - mean)^k over them (float64, 0 where the count is 0); up to ``SCAN_MAX_COLS``
    columns share one launch sequence."""
    lib = _lib.load()
    dev, nseg = _segments(offsets)
    return _value_batched(columns, nrows, dev, 3, lambda n: lib.fb_segmented_shape_moments_scratch_bytes(nrows, n),
                          lambda *args: lib.fb_segmented_shape_moments(dev.index, _stream_ptr(dev), nrows, nseg,
                                                                       offsets.data_ptr(), *args))


def segmented_comoments(offsets: torch.Tensor, nrows: int,
                        pairs: Sequence[Tuple[torch.Tensor, Optional[torch.Tensor], torch.Tensor, Optional[torch.Tensor]]]
                        ) -> List[Tuple[torch.Tensor, ...]]:
    """K9: running co-moments restarting at every segment ``[offsets[s], offsets[s + 1])``.  ``pairs`` = one
    ``(float64 x, validity of x or None, float64 y, validity of y or None)`` per pair; the kernel takes the rows
    where both are valid.  Returns per pair ``(count (int64), mean x, mean y, Sxx, Syy, Sxy)`` of those rows up to
    each row (float64, 0 where the count is 0); up to ``SCAN_MAX_COLS`` pairs share one launch sequence."""
    lib = _lib.load()
    dev, nseg = _segments(offsets)

    def outputs(x: torch.Tensor, mx: Optional[torch.Tensor], y: torch.Tensor,
                my: Optional[torch.Tensor]) -> Tuple[torch.Tensor, ...]:
        for v in (x, y):
            _check_rows(v, dev, nrows, torch.float64)
        for m in (mx, my):
            _check_rows(m, dev, nrows, torch.uint8)
        return _stat_outputs(dev, nrows, 5)

    return _batched(pairs, dev, outputs, lambda n: lib.fb_segmented_comoments_scratch_bytes(nrows, n),
                    lambda batch, outs, scratch: lib.fb_segmented_comoments(
                        dev.index, _stream_ptr(dev), nrows, nseg, offsets.data_ptr(), len(batch),
                        *[_ptrs([p[i] for p in batch]) for i in range(4)], *outs, scratch.data_ptr(),
                        scratch.numel()))


EWM_ROWS = 0           # FB_EWM_*: the positions of fb_segmented_ewm: row index (pandas' ignore_na=False),
EWM_OBSERVATIONS = 1   # observation ordinal (ignore_na=True),
EWM_TIMES = 2          # an int64 times column, decaying by 0.5^(dt * scale)


def segmented_ewm(offsets: torch.Tensor, nrows: int,
                  columns: Sequence[Tuple[torch.Tensor, Optional[torch.Tensor], float, bool, int,
                                          Optional[torch.Tensor], float, bool]]) -> List[Tuple[Any, ...]]:
    """K9: running exponentially weighted moments restarting at every segment ``[offsets[s], offsets[s + 1])``.
    ``columns`` = one ``(float64 values, validity or None, alpha, adjust, positions, int64 times or None, scale,
    spread)`` per column, ``positions`` one of ``EWM_*`` (``times`` and ``scale`` = 1 / halflife only for
    ``EWM_TIMES``).  An observation is a valid, non-NaN value.  Returns per column ``(count of observations (int64),
    weighted mean, W, W2, C)`` up to each row (float64, 0 where the count is 0), with W / W2 the sums of the weights
    and of their squares and C the weighted sum of squared deviations from the mean, each weight a share of the total
    without ``adjust`` (``fb_segmented_ewm``); W, W2 and C are None unless ``spread``, and then not written.  Up to
    ``SCAN_MAX_COLS`` columns share one launch sequence."""
    lib = _lib.load()
    dev, nseg = _segments(offsets)

    def outputs(v: torch.Tensor, m: Optional[torch.Tensor], alpha: float, adjust: bool, pos: int,
                times: Optional[torch.Tensor], scale: float, spread: bool) -> Tuple[Any, ...]:
        _check_rows(v, dev, nrows, torch.float64)
        _check_rows(m, dev, nrows, torch.uint8)
        assert (times is not None) == (pos == EWM_TIMES)
        _check_rows(times, dev, nrows, torch.int64)
        return _stat_outputs(dev, nrows, 4 if spread else 1) + (() if spread else (None, None, None))

    return _batched(columns, dev, outputs, lambda n: lib.fb_segmented_ewm_scratch_bytes(nrows, n),
                    lambda batch, outs, scratch: lib.fb_segmented_ewm(
                        dev.index, _stream_ptr(dev), nrows, nseg, offsets.data_ptr(), len(batch),
                        _ptrs([c[0] for c in batch]), _ptrs([c[1] for c in batch]),
                        _lib.f64_array([c[2] for c in batch]), _lib.i32_array([c[3] for c in batch]),
                        _lib.i32_array([c[4] for c in batch]), _ptrs([c[5] for c in batch]),
                        _lib.f64_array([c[6] for c in batch]), *outs, scratch.data_ptr(), scratch.numel()))


FRAME_TILE_MAX_WIDTH = 1024   # FB_FRAME_TILE_MAX_WIDTH: widest frame of the one-pass kernel
FRAME_UNBOUNDED_START = 1
FRAME_UNBOUNDED_END = 2


def window_frame(offsets: torch.Tensor, nrows: int, start: Optional[int], end: Optional[int],
                 columns: Sequence[Tuple[int, Optional[torch.Tensor], Optional[torch.Tensor]]]
                 ) -> List[Tuple[Optional[torch.Tensor], torch.Tensor]]:
    """K9: ``ROWS BETWEEN start AND end`` over every segment ``[offsets[s], offsets[s + 1])``: per row, the
    op over the valid rows of ``[max(first, i + start), min(last, i + end)]`` (``None``: unbounded) and
    their count, 0 where the count is 0.  ``columns`` and the result are shaped as in
    :func:`segmented_scan`; up to ``SCAN_MAX_COLS`` columns share one launch sequence."""
    lib = _lib.load()
    dev, nseg = _segments(offsets)
    # a bound past every segment is unbounded: exact, as no segment is longer than the table
    if start is not None and start <= -nrows:
        start = None
    if end is not None and end >= nrows:
        end = None
    flags = (FRAME_UNBOUNDED_START if start is None else 0) | (FRAME_UNBOUNDED_END if end is None else 0)
    s, e = (0 if start is None else start), (0 if end is None else end)
    return _op_batched(columns, nrows, dev, lambda n: lib.fb_window_frame_scratch_bytes(nrows, n, s, e, flags),
                       lambda *args: lib.fb_window_frame(dev.index, _stream_ptr(dev), nrows, nseg, offsets.data_ptr(),
                                                         s, e, flags, *args))


RANGE_KEY_I64 = 0   # FB_RANGE_KEY_*: how fb_window_range_bounds reads the 8-byte presort key
RANGE_KEY_U64 = 1
RANGE_KEY_F64 = 2


def window_range_bounds(offsets: torch.Tensor, keys: torch.Tensor, valid: Optional[torch.Tensor], key_class: int,
                        ascending: bool, start: Optional[Any], end: Optional[Any]) -> Tuple[torch.Tensor, torch.Tensor]:
    """K9: ``RANGE BETWEEN start AND end`` over every segment ``[offsets[s], offsets[s + 1])``, each sorted by
    one key (``keys``: 8-byte values of ``key_class``; ``valid``: uint8 validity with a float key's NaN rows
    cleared, NULLs last).  Offsets are ints (``RANGE_KEY_I64`` / ``_U64``, within int64) or floats
    (``RANGE_KEY_F64``), ``None`` unbounded.  Returns per row the first and last row of its frame (int64;
    last < first: empty)."""
    lib = _lib.load()
    assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous()
    dev = offsets.device
    nseg = int(offsets.shape[0]) - 1
    n = int(keys.shape[0])
    assert keys.element_size() == 8 and keys.device == dev and keys.is_contiguous()
    if valid is not None:
        assert valid.dtype == torch.uint8 and valid.device == dev and valid.is_contiguous() and valid.shape[0] == n

    def bits(b: Any) -> int:
        if b is None:
            return 0
        if key_class == RANGE_KEY_F64:
            return struct.unpack("<Q", struct.pack("<d", float(b)))[0]
        assert -(1 << 63) <= b < (1 << 63), f"offset {b} outside int64"
        return int(b) & ((1 << 64) - 1)

    flags = (FRAME_UNBOUNDED_START if start is None else 0) | (FRAME_UNBOUNDED_END if end is None else 0)
    lo = torch.empty(n, dtype=torch.int64, device=dev)
    hi = torch.empty(n, dtype=torch.int64, device=dev)
    nb = int(lib.fb_window_range_bounds_scratch_bytes(nseg))
    scratch = torch.empty(max(nb, 8), dtype=torch.uint8, device=dev)
    _lib.check(lib.fb_window_range_bounds(
        dev.index, _stream_ptr(dev), n, nseg, offsets.data_ptr(), keys.data_ptr(),
        0 if valid is None else valid.data_ptr(), key_class, 0 if ascending else 1, bits(start), bits(end), flags,
        lo.data_ptr(), hi.data_ptr(), scratch.data_ptr(), scratch.numel()))
    return lo, hi


def window_bounded(lo: torch.Tensor, hi: torch.Tensor,
                   columns: Sequence[Tuple[int, Optional[torch.Tensor], Optional[torch.Tensor]]]
                   ) -> List[Tuple[Optional[torch.Tensor], torch.Tensor]]:
    """K9: per row i, the op over the valid rows of ``[lo[i], hi[i]]`` (clamped to the table; hi < lo: empty)
    and their count, 0 where the count is 0.  ``columns`` and the result are shaped as in
    :func:`segmented_scan`; up to ``SCAN_MAX_COLS`` columns share one tree build and query."""
    lib = _lib.load()
    dev = lo.device
    nrows = int(lo.shape[0])
    for b_ in (lo, hi):
        assert b_.dtype == torch.int64 and b_.is_cuda and b_.is_contiguous() and b_.shape[0] == nrows
    return _op_batched(columns, nrows, dev, lambda n: lib.fb_window_bounded_scratch_bytes(nrows, n),
                       lambda *args: lib.fb_window_bounded(dev.index, _stream_ptr(dev), nrows, lo.data_ptr(),
                                                           hi.data_ptr(), *args))


VALUE_LAST = 0   # FB_VALUE_LAST: the frame's last row


def _i64_array(vals: Sequence[int]) -> Any:
    arr = (C.c_int64 * max(len(vals), 1))()
    for i, v in enumerate(vals):
        arr[i] = int(v)
    return arr


def window_value(offsets: Optional[torch.Tensor], nrows: int, frame: Any,
                 columns: Sequence[Tuple[torch.Tensor, Optional[torch.Tensor], int]]
                 ) -> List[Tuple[torch.Tensor, torch.Tensor]]:
    """K9: FIRST_VALUE / LAST_VALUE / NTH_VALUE (``fb_window_value``).  ``frame`` is ``("rows", start, end)`` over the
    segments ``offsets`` (``None``: unbounded; as :func:`window_frame`) or ``("bounds", lo, hi)``, every row's first
    and last frame row (int64, as :func:`window_range_bounds` returns them).  ``columns`` = one ``(values of any width,
    validity or None, nth)`` per column: nth >= 1 picks the frame's nth row, ``VALUE_LAST`` its last.  Returns per
    column (value, uint8 validity): NULL for an empty frame, a pick past its end or a NULL at the picked row.  Up to
    ``SCAN_MAX_COLS`` columns share one launch."""
    lib = _lib.load()
    dev = columns[0][0].device
    lo = hi = None
    start = end = flags = 0
    nseg = 0
    if frame[0] == "rows":
        _, s, e = frame
        dev, nseg = _segments(offsets)
        if s is not None and s <= -nrows:
            s = None
        if e is not None and e >= nrows:
            e = None
        flags = (FRAME_UNBOUNDED_START if s is None else 0) | (FRAME_UNBOUNDED_END if e is None else 0)
        start, end = (0 if s is None else s), (0 if e is None else e)
    else:
        _, lo, hi = frame
        for b_ in (lo, hi):
            assert b_.dtype == torch.int64 and b_.device == dev and b_.is_contiguous() and b_.shape[0] == nrows
    res: List[Tuple[torch.Tensor, torch.Tensor]] = []
    for b in range(0, len(columns), SCAN_MAX_COLS):
        batch = columns[b:b + SCAN_MAX_COLS]
        for v, m, nth in batch:
            assert v.device == dev and v.is_contiguous() and v.dim() == 1 and v.shape[0] == nrows
            assert v.element_size() in (1, 2, 4, 8)
            assert nth == VALUE_LAST or nth >= 1
            _check_rows(m, dev, nrows, torch.uint8)
        outs = [(torch.empty_like(v), torch.empty(nrows, dtype=torch.uint8, device=dev)) for v, _, _ in batch]
        _lib.check(lib.fb_window_value(
            dev.index, _stream_ptr(dev), nrows, nseg, 0 if offsets is None else offsets.data_ptr(), start, end, flags,
            0 if lo is None else lo.data_ptr(), 0 if hi is None else hi.data_ptr(), len(batch),
            _i64_array([min(nth, nrows + 1) for _, _, nth in batch]),
            _lib.i32_array([v.element_size() for v, _, _ in batch]), _ptrs([v for v, _, _ in batch]),
            _ptrs([m for _, m, _ in batch]), _ptrs([o for o, _ in outs]), _ptrs([ov for _, ov in outs])))
        res.extend(outs)
    return res


def window_distribution(offsets: torch.Tensor, heads: torch.Tensor, percent_rank: bool, cume_dist: bool,
                        ntiles: Sequence[int]) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor], List[torch.Tensor]]:
    """K9: PERCENT_RANK, CUME_DIST and NTILE(n) of every row over the segments ``offsets`` (``fb_window_distribution``);
    ``heads`` (bool or uint8, one per row) marks the first row of every peer group.  Returns (float64 PERCENT_RANK or
    None, float64 CUME_DIST or None, one int64 column per n of ``ntiles``); ``SCAN_MAX_COLS`` NTILEs a launch."""
    lib = _lib.load()
    dev, nseg = _segments(offsets)
    nrows = int(heads.shape[0])
    heads = heads.view(torch.uint8) if heads.dtype == torch.bool else heads
    _check_rows(heads, dev, nrows, torch.uint8)
    pr = torch.empty(nrows, dtype=torch.float64, device=dev) if percent_rank else None
    cd = torch.empty(nrows, dtype=torch.float64, device=dev) if cume_dist else None
    nts = [torch.empty(nrows, dtype=torch.int64, device=dev) for _ in ntiles]
    nb = int(lib.fb_window_distribution_scratch_bytes(nrows))
    scratch = torch.empty(max(nb, 8), dtype=torch.uint8, device=dev)
    for b in range(0, max(len(ntiles), 1), SCAN_MAX_COLS):
        ns, outs = ntiles[b:b + SCAN_MAX_COLS], nts[b:b + SCAN_MAX_COLS]
        assert all(n >= 1 for n in ns)
        first = b == 0
        _lib.check(lib.fb_window_distribution(
            dev.index, _stream_ptr(dev), nrows, nseg, offsets.data_ptr(), heads.data_ptr(),
            0 if pr is None or not first else pr.data_ptr(), 0 if cd is None or not first else cd.data_ptr(),
            len(ns), _i64_array([min(n, 1 << 62) for n in ns]), _ptrs(outs), scratch.data_ptr(), scratch.numel()))
    return pr, cd, nts


QUANTILE_TILE_ROWS = 2048   # FB_QUANTILE_TILE_ROWS: longest segment of the one-pass shared-memory path
QUANTILE_MAX_Q = 16
QUANTILE_CONT = 0
QUANTILE_DISC = 1


def segmented_quantile(offsets: torch.Tensor, values: torch.Tensor, valid: Optional[torch.Tensor], value_class: int,
                       quantiles: Sequence[Tuple[float, int]]) -> Tuple[torch.Tensor, List[torch.Tensor]]:
    """K10: exact quantiles of every segment ``[offsets[s], offsets[s + 1])`` of one column (``values``: 8-byte
    values of ``value_class``, a ``RANGE_KEY_*``; ``valid``: uint8 validity or None; f64 NaN is NULL too).
    ``quantiles`` = ``(q, QUANTILE_CONT | QUANTILE_DISC)`` pairs; up to ``QUANTILE_MAX_Q`` share one call.
    Returns (per segment the non-NULL count m, per pair a result per segment: f64 for CONT, 0 where m = 0;
    for DISC the int64 row of the picked value, -1 where m = 0)."""
    lib = _lib.load()
    assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous()
    dev = offsets.device
    nseg = int(offsets.shape[0]) - 1
    n = int(values.shape[0])
    assert values.element_size() == 8 and values.device == dev and values.is_contiguous()
    if valid is not None:
        assert valid.dtype == torch.uint8 and valid.device == dev and valid.is_contiguous() and valid.shape[0] == n
    count = torch.empty(nseg, dtype=torch.int64, device=dev)
    outs = [torch.empty(nseg, dtype=torch.float64 if kind == QUANTILE_CONT else torch.int64, device=dev)
            for _, kind in quantiles]
    if nseg == 0 or not quantiles:
        return count, outs
    lengths = offsets[1:] - offsets[:-1]
    long_rows = int(torch.where(lengths > QUANTILE_TILE_ROWS, lengths, 0).sum()) if n > QUANTILE_TILE_ROWS else 0
    nb = int(lib.fb_quantile_scratch_bytes(dev.index, n, long_rows))
    scratch = torch.empty(max(nb, 8), dtype=torch.uint8, device=dev)
    for b in range(0, len(quantiles), QUANTILE_MAX_Q):
        batch = quantiles[b:b + QUANTILE_MAX_Q]
        qs = (C.c_double * len(batch))(*[float(q) for q, _ in batch])
        _lib.check(lib.fb_segmented_quantile(
            dev.index, _stream_ptr(dev), n, nseg, offsets.data_ptr(), values.data_ptr(),
            0 if valid is None else valid.data_ptr(), value_class, len(batch), qs,
            _lib.i32_array([kind for _, kind in batch]), count.data_ptr(),
            _lib.ptr_array([o.data_ptr() for o in outs[b:b + QUANTILE_MAX_Q]]), scratch.data_ptr(), scratch.numel()))
    return count, outs


def exclusive_scan(counts: torch.Tensor) -> Tuple[torch.Tensor, int]:
    """Exclusive prefix sum of an int64 device vector (own kernels); returns (offsets, total)."""
    lib = _lib.load()
    dev = counts.device
    n = int(counts.shape[0])
    out = torch.empty(n, dtype=torch.int64, device=dev)
    total = torch.zeros(1, dtype=torch.int64, device=dev)
    nb = int(lib.fb_exclusive_scan_scratch_bytes(n))
    scratch = torch.empty(max(nb, 8), dtype=torch.uint8, device=dev)
    _lib.check(lib.fb_exclusive_scan_i64(dev.index, _stream_ptr(dev), n, counts.data_ptr(), out.data_ptr(),
                                         total.data_ptr(), scratch.data_ptr(), scratch.numel()))
    return out, int(total.item())


class JoinTable:
    """Hash multimap of the build side of a join (K7)."""

    def __init__(self, keys: torch.Tensor, valid: Optional[torch.Tensor], num_parts: int = 0,
                 part_offsets: Optional[torch.Tensor] = None):
        """num_parts > 1: ``keys`` (and later the probe keys) were hash-partitioned into that many
        partitions with ``partition_columns``; the table is then used region by region
        (``part_offsets``: the partition offsets of ``keys``, lets the build work in L2-sized batches)."""
        lib = _lib.load()
        dev, n = _check_cols([keys])
        assert keys.element_size() == 8
        self.nbuild = n
        self.capacity = max(2, 1 << (2 * max(n, 1)).bit_length())  # load factor <= 0.5
        if num_parts > 1:
            self.capacity = max(self.capacity, 4 * num_parts)
        self.num_parts = num_parts if num_parts > 1 else 0
        self.table = torch.empty(int(lib.fb_join_table_bytes(self.capacity)), dtype=torch.uint8, device=dev)
        self.status = torch.zeros(4, dtype=torch.int64, device=dev)

        def build() -> None:
            _lib.check(lib.fb_join_build_u64(dev.index, _stream_ptr(dev), n, keys.data_ptr(),
                                             0 if valid is None else valid.data_ptr(), self.capacity,
                                             self.num_parts, self.table.data_ptr(), self.status.data_ptr(),
                                             0 if (part_offsets is None or self.num_parts == 0)
                                             else part_offsets.data_ptr()))

        build()
        # Region mode gives every partition capacity / num_parts slots: a skewed build side (hot key,
        # low cardinality) can overflow its region, and the kernel then reports status[0] = 1 instead
        # of inserting.  Fall back to ONE region over the whole table (load factor <= 0.5: cannot
        # overflow; the inputs may stay partitioned, the probes just use the same single region).
        if self.num_parts > 0 and int(self.status[0].item()) != 0:
            self.num_parts = 0
            self.status.zero_()
            build()
            if int(self.status[0].item()) != 0:  # pragma: no cover - load factor 0.5 always has room
                raise _lib.FugueB200KernelError("join hash table overflow")
        self.device = dev

    def probe_counts(self, keys: torch.Tensor, valid: Optional[torch.Tensor], outer: bool,
                     first: Optional[torch.Tensor] = None) -> torch.Tensor:
        lib = _lib.load()
        n = int(keys.shape[0])
        counts = torch.empty(n, dtype=torch.int64, device=self.device)
        _lib.check(lib.fb_join_probe_count_u64(self.device.index, _stream_ptr(self.device), n, keys.data_ptr(),
                                               0 if valid is None else valid.data_ptr(), self.capacity,
                                               self.num_parts, self.table.data_ptr(), 1 if outer else 0,
                                               counts.data_ptr(), 0 if first is None else first.data_ptr()))
        return counts

    def probe(self, keys: torch.Tensor, valid: Optional[torch.Tensor], outer: bool
              ) -> Tuple[torch.Tensor, torch.Tensor]:
        """(probe_row, build_row) pairs of all matches, probe-row major; build_row == -1 marks the
        NULL-extended row of an outer join."""
        lib = _lib.load()
        n = int(keys.shape[0])
        first = torch.empty(n, dtype=torch.int64, device=self.device)
        counts = self.probe_counts(keys, valid, outer, first)
        offsets, total = exclusive_scan(counts)
        pi = torch.empty(total, dtype=torch.int64, device=self.device)
        bi = torch.empty(total, dtype=torch.int64, device=self.device)
        _lib.check(lib.fb_join_probe_write_u64(self.device.index, _stream_ptr(self.device), n, keys.data_ptr(),
                                               0 if valid is None else valid.data_ptr(), self.capacity,
                                               self.num_parts, self.table.data_ptr(), 1 if outer else 0,
                                               offsets.data_ptr(), pi.data_ptr(), bi.data_ptr(),
                                               counts.data_ptr(), first.data_ptr()))
        return pi, bi

    def matched_mask(self, build_idx: torch.Tensor) -> torch.Tensor:
        lib = _lib.load()
        m = torch.zeros(self.nbuild, dtype=torch.uint8, device=self.device)
        _lib.check(lib.fb_join_mark_matched(self.device.index, _stream_ptr(self.device), build_idx.data_ptr(),
                                            int(build_idx.shape[0]), m.data_ptr()))
        return m


JOIN2_MAX_COLS = 48


def join_fused(probe_keys: torch.Tensor, probe_valid: Optional[torch.Tensor], build_keys: torch.Tensor,
               build_valid: Optional[torch.Tensor], left_cols: Sequence[torch.Tensor],
               right_cols: Sequence[torch.Tensor], right_valid: Sequence[Optional[torch.Tensor]], outer: bool,
               num_parts: int = 0, build_part_offsets: Optional[torch.Tensor] = None,
               probe_part_offsets: Optional[torch.Tensor] = None
               ) -> Tuple[List[torch.Tensor], List[torch.Tensor], List[Optional[torch.Tensor]], int]:
    """K7 fast path (inner / left outer on one 8-byte key): build a 4-byte-slot table over ``build_keys``,
    probe it once (match count + first match per probe row, output size), then write the OUTPUT columns
    directly: ``left_cols`` copied from the probe rows, ``right_cols`` gathered from the matched build rows
    (with ``outer``: NULL-extended, a validity mask per right column).  Returns
    (left outputs, right outputs, right validity or None each, number of output rows)."""
    lib = _lib.load()
    dev, nb = _check_cols([build_keys])
    _, npr = _check_cols([probe_keys])
    assert build_keys.element_size() == 8 and probe_keys.element_size() == 8
    assert len(left_cols) <= JOIN2_MAX_COLS and len(right_cols) <= JOIN2_MAX_COLS and nb < (1 << 32) - 1
    capacity = max(4, 1 << (2 * max(nb, 1)).bit_length())  # load factor <= 0.5
    parts = num_parts if (num_parts > 1 and capacity >= 4 * num_parts) else 0
    table = torch.empty(int(lib.fb_join2_table_bytes(capacity)), dtype=torch.uint8, device=dev)
    status = torch.zeros(4, dtype=torch.int64, device=dev)

    def build() -> None:
        _lib.check(lib.fb_join2_build(dev.index, _stream_ptr(dev), nb, build_keys.data_ptr(),
                                      0 if build_valid is None else build_valid.data_ptr(), capacity, parts,
                                      table.data_ptr(), status.data_ptr(),
                                      0 if (build_part_offsets is None or parts == 0) else build_part_offsets.data_ptr()))

    cnt = torch.empty(npr, dtype=torch.int32, device=dev)
    first = torch.empty(npr, dtype=torch.int32, device=dev)
    tile_base = torch.empty(int(lib.fb_join2_tiles_bytes(npr)) // 8, dtype=torch.int64, device=dev)
    total = torch.zeros(1, dtype=torch.int64, device=dev)

    def probe() -> None:
        _lib.check(lib.fb_join2_probe(dev.index, _stream_ptr(dev), npr, probe_keys.data_ptr(),
                                      0 if probe_valid is None else probe_valid.data_ptr(), build_keys.data_ptr(),
                                      capacity, parts, table.data_ptr(), 1 if outer else 0, cnt.data_ptr(),
                                      first.data_ptr(), tile_base.data_ptr(), total.data_ptr(), status.data_ptr()))

    if parts > 0 and build_part_offsets is not None and probe_part_offsets is not None:
        # both sides hash-partitioned: build and probe region batch by region batch (L2-resident)
        _lib.check(lib.fb_join2_build_probe(
            dev.index, _stream_ptr(dev), nb, build_keys.data_ptr(), 0 if build_valid is None else build_valid.data_ptr(),
            build_part_offsets.data_ptr(), npr, probe_keys.data_ptr(),
            0 if probe_valid is None else probe_valid.data_ptr(), probe_part_offsets.data_ptr(), capacity, parts,
            table.data_ptr(), 1 if outer else 0, cnt.data_ptr(), first.data_ptr(), tile_base.data_ptr(),
            total.data_ptr(), status.data_ptr()))
    else:
        build()
        probe()
    # ONE host read per join: the output size (needed to allocate) together with the overflow flag of the
    # build.  A skewed build side can overflow its region (capacity / num_parts slots): redo with one region.
    both = torch.cat([status[:1], total]).tolist()
    if parts > 0 and both[0] != 0:
        parts = 0
        build()
        probe()
        both = torch.cat([status[:1], total]).tolist()
        if both[0] != 0:  # pragma: no cover - load factor 0.5 always has room
            raise _lib.FugueB200KernelError("join hash table overflow")
    nout = int(both[1])
    louts = [torch.empty(nout, dtype=c.dtype, device=dev) for c in left_cols]
    routs = [torch.empty(nout, dtype=c.dtype, device=dev) for c in right_cols]
    rvout = [torch.empty(nout, dtype=torch.uint8, device=dev) if (outer or v is not None) else None
             for v in right_valid]
    if nout > 0:
        _lib.check(lib.fb_join2_emit(
            dev.index, _stream_ptr(dev), npr, probe_keys.data_ptr(), build_keys.data_ptr(), capacity, parts,
            table.data_ptr(), cnt.data_ptr(), first.data_ptr(), tile_base.data_ptr(),
            len(left_cols), _lib.ptr_array([c.data_ptr() for c in left_cols]),
            _lib.ptr_array([c.data_ptr() for c in louts]), _lib.i32_array([c.element_size() for c in left_cols]),
            len(right_cols), _lib.ptr_array([c.data_ptr() for c in right_cols]),
            _lib.ptr_array([c.data_ptr() for c in routs]), _lib.i32_array([c.element_size() for c in right_cols]),
            _lib.ptr_array([0 if v is None else v.data_ptr() for v in right_valid]),
            _lib.ptr_array([0 if v is None else v.data_ptr() for v in rvout])))
    return louts, routs, rvout, nout


def gather_rows(cols: Sequence[torch.Tensor], valid: Sequence[Optional[torch.Tensor]], idx: torch.Tensor,
                want_valid: bool) -> Tuple[List[torch.Tensor], List[Optional[torch.Tensor]]]:
    """out[c][o] = cols[c][idx[o]]; idx < 0 gives NULL (needs want_valid)."""
    lib = _lib.load()
    if len(cols) == 0:
        return [], []
    dev = idx.device
    n = int(idx.shape[0])
    outs = [torch.empty(n, dtype=c.dtype, device=dev) for c in cols]
    need_v = [want_valid or v is not None for v in valid]
    outv = [torch.empty(n, dtype=torch.uint8, device=dev) if nv else None for nv in need_v]
    sp = torch.tensor([c.data_ptr() for c in cols], dtype=torch.int64, device=dev)
    dp = torch.tensor([c.data_ptr() for c in outs], dtype=torch.int64, device=dev)
    w = torch.tensor([c.element_size() for c in cols], dtype=torch.int32, device=dev)
    sv = torch.tensor([0 if v is None else v.data_ptr() for v in valid], dtype=torch.int64, device=dev)
    dv = torch.tensor([0 if v is None else v.data_ptr() for v in outv], dtype=torch.int64, device=dev)
    _lib.check(lib.fb_gather_rows(dev.index, _stream_ptr(dev), len(cols), sp.data_ptr(), dp.data_ptr(),
                                  w.data_ptr(), sv.data_ptr(), dv.data_ptr(), idx.data_ptr(), n))
    return outs, outv


def scatter_rows(cols: Sequence[torch.Tensor], valid: Sequence[Optional[torch.Tensor]], idx: torch.Tensor
                 ) -> Tuple[List[torch.Tensor], List[Optional[torch.Tensor]]]:
    """out[c][idx[i]] = cols[c][i], validity likewise (None stays None): the inverse of ``gather_rows`` for a
    permutation ``idx`` (``fb_scatter_rows``; only argsort results may be passed), all columns in one launch."""
    lib = _lib.load()
    if len(cols) == 0:
        return [], []
    dev = idx.device
    n = int(idx.shape[0])
    assert all(int(c.shape[0]) == n for c in cols), "scatter_rows: every column needs one row per index"
    outs = [torch.empty(n, dtype=c.dtype, device=dev) for c in cols]
    outv = [None if v is None else torch.empty(n, dtype=torch.uint8, device=dev) for v in valid]
    sp = torch.tensor([c.data_ptr() for c in cols], dtype=torch.int64, device=dev)
    dp = torch.tensor([c.data_ptr() for c in outs], dtype=torch.int64, device=dev)
    w = torch.tensor([c.element_size() for c in cols], dtype=torch.int32, device=dev)
    sv = torch.tensor([0 if v is None else v.data_ptr() for v in valid], dtype=torch.int64, device=dev)
    dv = torch.tensor([0 if v is None else v.data_ptr() for v in outv], dtype=torch.int64, device=dev)
    _lib.check(lib.fb_scatter_rows(dev.index, _stream_ptr(dev), len(cols), sp.data_ptr(), dp.data_ptr(),
                                   w.data_ptr(), sv.data_ptr(), dv.data_ptr(), idx.contiguous().data_ptr(), n))
    return outs, outv


ASOF_BACKWARD, ASOF_FORWARD, ASOF_NEAREST = 0, 1, 2   # FB_ASOF_*


def asof_search(run: torch.Tensor, run_offsets: torch.Tensor, left_codes: torch.Tensor,
                left_valid: Optional[torch.Tensor], right_codes: torch.Tensor, right_rows: torch.Tensor, key_class: int,
                direction: int, allow_exact_matches: bool, tolerance: Optional[Any]) -> torch.Tensor:
    """``fb_asof_search``: per left row i, the right row it matches in its run ``run[i]`` (-1: none) of the sorted
    right side, or -1.  ``right_codes`` (order codes, ascending within each run ``[run_offsets[r],
    run_offsets[r + 1])``: only argsort results may be passed) and ``right_rows`` (the sort permutation) are in sorted
    order; ``left_codes`` / ``left_valid`` in left order.  ``tolerance``: None, an int >= 0 for the integer classes,
    a float for ``RANGE_KEY_F64``."""
    lib = _lib.load()
    dev = run.device
    n = int(run.shape[0])
    for t in (run, run_offsets, right_rows):
        assert t.dtype == torch.int64 and t.is_cuda and t.is_contiguous()
    for t in (left_codes, right_codes):
        assert t.element_size() == 8 and t.device == dev and t.is_contiguous()
    assert left_codes.shape[0] == n and right_codes.shape[0] == right_rows.shape[0]
    if left_valid is not None:
        assert left_valid.dtype == torch.uint8 and left_valid.device == dev and left_valid.is_contiguous()
    if tolerance is None:
        tol = 0
    elif key_class == RANGE_KEY_F64:
        tol = struct.unpack("<Q", struct.pack("<d", float(tolerance)))[0]
    else:
        assert 0 <= tolerance < (1 << 63), f"tolerance {tolerance} outside [0, 2^63)"
        tol = int(tolerance)
    out = torch.empty(n, dtype=torch.int64, device=dev)
    _lib.check(lib.fb_asof_search(dev.index, _stream_ptr(dev), n, run.data_ptr(), run_offsets.data_ptr(),
                                  left_codes.data_ptr(), 0 if left_valid is None else left_valid.data_ptr(),
                                  right_codes.data_ptr(), right_rows.data_ptr(), key_class, direction,
                                  1 if allow_exact_matches else 0, 0 if tolerance is None else 1, tol,
                                  out.data_ptr()))
    return out


RANGE_CLOSED_LEFT, RANGE_CLOSED_RIGHT = 1, 2   # FB_RANGE_CLOSED_*


def window_tree(op: int, values: torch.Tensor) -> torch.Tensor:
    """``fb_window_tree``: the levels >= 1 of the aligned block tree of ``op`` (an ``AGG_*`` op) over one column of
    8-byte values without NULLs, as the uint8 scratch that holds them (layout: include/fugue_b200.h)."""
    lib = _lib.load()
    dev, n = _check_cols([values])
    assert values.element_size() == 8
    nb = int(lib.fb_window_bounded_scratch_bytes(n, 1))
    tree = torch.empty(max(nb, 8), dtype=torch.uint8, device=dev)
    _lib.check(lib.fb_window_tree(dev.index, _stream_ptr(dev), n, 1, _lib.i32_array([op]),
                                  _ptrs([values]), _ptrs([None]), tree.data_ptr(), tree.numel()))
    return tree


def _range_join_args(run: torch.Tensor, run_offsets: torch.Tensor, left_codes: torch.Tensor,
                     left_valid: Optional[torch.Tensor], start_codes: torch.Tensor, end_keys: torch.Tensor,
                     tree: torch.Tensor) -> List[Any]:
    dev = run.device
    for t in (run, run_offsets, end_keys):
        assert t.dtype == torch.int64 and t.is_cuda and t.is_contiguous()
    for t in (left_codes, start_codes):
        assert t.element_size() == 8 and t.device == dev and t.is_contiguous()
    assert left_codes.shape[0] == run.shape[0] and start_codes.shape[0] == end_keys.shape[0]
    if left_valid is not None:
        assert left_valid.dtype == torch.uint8 and left_valid.device == dev and left_valid.is_contiguous()
    assert tree.dtype == torch.uint8 and tree.device == dev
    return [dev.index, _stream_ptr(dev), int(run.shape[0]), run.data_ptr(), run_offsets.data_ptr(),
            left_codes.data_ptr(), 0 if left_valid is None else left_valid.data_ptr(), int(start_codes.shape[0]),
            start_codes.data_ptr(), end_keys.data_ptr(), tree.data_ptr(), tree.numel()]


def range_join_count(run: torch.Tensor, run_offsets: torch.Tensor, left_codes: torch.Tensor,
                     left_valid: Optional[torch.Tensor], start_codes: torch.Tensor, end_keys: torch.Tensor,
                     tree: torch.Tensor, closed: int, outer: bool) -> torch.Tensor:
    """``fb_range_join_count``: per left row the number of intervals of its run ``run[i]`` (-1: none) that hold its
    value (1 for none when ``outer``).  In sorted right order: ``start_codes`` (order codes, ascending within each
    run: only argsort results may be passed), ``end_keys`` (end codes ^ 2^63 as int64) and ``tree``
    (``window_tree(AGG_MAX_I64, end_keys)``); ``closed`` is ``RANGE_CLOSED_*`` flags."""
    lib = _lib.load()
    args = _range_join_args(run, run_offsets, left_codes, left_valid, start_codes, end_keys, tree)
    counts = torch.empty(int(run.shape[0]), dtype=torch.int64, device=run.device)
    _lib.check(lib.fb_range_join_count(*args, closed, 1 if outer else 0, counts.data_ptr()))
    return counts


def range_join_emit(run: torch.Tensor, run_offsets: torch.Tensor, left_codes: torch.Tensor,
                    left_valid: Optional[torch.Tensor], start_codes: torch.Tensor, end_keys: torch.Tensor,
                    tree: torch.Tensor, right_rows: torch.Tensor, closed: int, outer: bool, counts: torch.Tensor,
                    offsets: torch.Tensor, total: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """``fb_range_join_emit``: the ``total`` (left row, right row) pairs counted by :func:`range_join_count`, each
    left row's at ``offsets[i]`` (its exclusive scan) in ascending (start, right row) order; ``right_rows`` maps
    sorted positions to right rows, and -1 stands for the unmatched row of an outer join."""
    lib = _lib.load()
    args = _range_join_args(run, run_offsets, left_codes, left_valid, start_codes, end_keys, tree)
    for t in (right_rows, counts, offsets):
        assert t.dtype == torch.int64 and t.device == run.device and t.is_contiguous()
    assert right_rows.shape[0] == start_codes.shape[0] and counts.shape[0] == offsets.shape[0] == run.shape[0]
    li = torch.empty(total, dtype=torch.int64, device=run.device)
    ri = torch.empty(total, dtype=torch.int64, device=run.device)
    if total == 0:
        return li, ri
    _lib.check(lib.fb_range_join_emit(*args, right_rows.data_ptr(), closed, 1 if outer else 0, counts.data_ptr(),
                                      offsets.data_ptr(), li.data_ptr(), ri.data_ptr()))
    return li, ri


def row_hash64(keys: Sequence[torch.Tensor], valid: Optional[Sequence[Optional[torch.Tensor]]] = None
               ) -> torch.Tensor:
    """64-bit hash of each row's key tuple (same function as the partitioner, before ``% num``)."""
    lib = _lib.load()
    dev, n = _check_cols(keys)
    out = torch.empty(n, dtype=torch.int64, device=dev)
    vp = _valid_ptrs(valid, len(keys))
    _lib.check(lib.fb_row_hash64(dev.index, _stream_ptr(dev), n, len(keys),
                                 _lib.ptr_array([k.data_ptr() for k in keys]),
                                 _lib.i32_array([k.element_size() for k in keys]), vp, out.data_ptr()))
    return out


def compact_indices(mask: torch.Tensor) -> torch.Tensor:
    """Row numbers (int64, increasing) where ``mask`` (bool / uint8 device vector) is set."""
    lib = _lib.load()
    if mask.dtype == torch.bool:
        mask = mask.view(torch.uint8)
    assert mask.dtype == torch.uint8 and mask.is_cuda and mask.is_contiguous()
    dev = mask.device
    n = int(mask.shape[0])
    out = torch.empty(n, dtype=torch.int64, device=dev)
    cnt = torch.zeros(1, dtype=torch.int64, device=dev)
    nb = int(lib.fb_compact_scratch_bytes(n))
    scratch = torch.empty(max(nb, 8), dtype=torch.uint8, device=dev)
    _lib.check(lib.fb_compact_indices(dev.index, _stream_ptr(dev), mask.data_ptr(), n, out.data_ptr(),
                                      cnt.data_ptr(), scratch.data_ptr(), scratch.numel()))
    return out[:int(cnt.item())]


# ---- K8: column-expression evaluator -----------------------------------------------------------
EXPR_MAX_COLS, EXPR_MAX_OUTS, EXPR_MAX_INS, EXPR_NREGS = 16, 16, 96, 4
T_I8, T_I16, T_I32, T_I64, T_U8, T_F32, T_F64, T_U16, T_U32, T_F16 = range(10)
XK_NONE, XK_REG, XK_COL, XK_IMM, XK_NULL = range(5)
XF_B_I2F = 1
XF_COND_SHIFT = 8  # X_SEL: the condition's temporary is flags >> 8
(X_MOV, X_ST, X_OUT, X_I2F, X_F2I, X_NEG_I, X_NEG_F, X_NOT, X_IS_NULL, X_NOT_NULL, X_TOBOOL_I, X_TOBOOL_F,
 X_ADD_I, X_SUB_I, X_RSUB_I, X_MUL_I, X_ADD_F, X_SUB_F, X_RSUB_F, X_MUL_F, X_DIV_F, X_RDIV_F,
 X_LT_I, X_LE_I, X_GT_I, X_GE_I, X_EQ_I, X_NE_I, X_LT_F, X_LE_F, X_GT_F, X_GE_F, X_EQ_F, X_NE_F,
 X_AND, X_OR, X_COALESCE, X_RCOALESCE, X_LOOKUP,
 X_SEL, X_MOD_I, X_RMOD_I, X_MOD_F, X_RMOD_F, X_ABS_I, X_ABS_F, X_FLOOR_F, X_CEIL_F, X_ROUND_F, X_ROUND_I,
 X_SQRT, X_EXP, X_LN, X_LOG10, X_POW, X_RPOW, X_GREATEST_I, X_LEAST_I, X_GREATEST_F, X_LEAST_F,
 X_MULSAT_I, X_FLOORDIV_I, X_TS_PART, X_TS_TRUNC, X_TS_INDEX, X_TS_ADDMON) = range(66)
XF_UNIT_SHIFT = 8  # X_TS_ADDMON: the unit is flags >> 8; X_TS_PART / TRUNC / INDEX: imm = field or part | unit << 8
TU_DAY, TU_S, TU_MS, TU_US, TU_NS = range(5)  # enum fb_time_unit: what one count of a temporal value is
TIME_FIELDS = ("year", "month", "day", "hour", "minute", "second", "quarter", "dow", "isodow", "doy", "week",
               "isoyear")  # enum fb_time_field, in order
TIME_PARTS = ("year", "quarter", "month", "week", "day", "hour", "minute", "second")  # enum fb_time_part, in order

# storage dtype of each K8 type: uint16 / uint32 / float16 live in the signed tensors of their width
EXPR_STORAGE = {T_I8: torch.int8, T_I16: torch.int16, T_I32: torch.int32, T_I64: torch.int64, T_U8: torch.uint8,
                T_F32: torch.float32, T_F64: torch.float64, T_U16: torch.int16, T_U32: torch.int32,
                T_F16: torch.int16}
_EXPR_TYPE_OF_DTYPE = {torch.int8: T_I8, torch.int16: T_I16, torch.int32: T_I32, torch.int64: T_I64,
                       torch.uint8: T_U8, torch.bool: T_U8, torch.float32: T_F32, torch.float64: T_F64}


def expr_type_of(dtype: torch.dtype) -> int:
    """The K8 type that reads a tensor of ``dtype`` as a signed integer or a float of its width."""
    return _EXPR_TYPE_OF_DTYPE[dtype]


def eval_expr(nrows: int, device: torch.device, cols: Sequence[torch.Tensor],
              valid: Sequence[Optional[torch.Tensor]], program: Sequence[Tuple[int, int, int, int, int]],
              out_dtypes: Sequence[torch.dtype], want_valid: Sequence[bool],
              col_types: Optional[Sequence[int]] = None, out_types: Optional[Sequence[int]] = None
              ) -> Tuple[List[torch.Tensor], List[Optional[torch.Tensor]]]:
    """Run one accumulator-machine ``program`` (tuples ``(op, operand_kind, b, flags, imm_bits)``, see
    include/fugue_b200.h K8) over all rows; ``X_OUT b`` writes output ``b``.  Returns the output
    columns (``out_dtypes``) and (where asked for) their validity byte masks.
    ``col_types`` / ``out_types`` are the K8 types (``T_*``) of the columns and outputs: the storage
    dtype alone does not say whether 16 bits hold an int16, a uint16 or a float16.  Left out, every
    tensor is read and written as the signed integer or float of its dtype (``expr_type_of``)."""
    lib = _lib.load()
    col_types = [expr_type_of(c.dtype) for c in cols] if col_types is None else list(col_types)
    out_types = [expr_type_of(dt) for dt in out_dtypes] if out_types is None else list(out_types)
    assert len(col_types) == len(cols) and len(out_types) == len(out_dtypes)
    for dt, tp in zip(out_dtypes, out_types):
        assert dt.itemsize == EXPR_STORAGE[tp].itemsize, f"{dt} output can't hold K8 type {tp}"
    outs = [torch.empty(nrows, dtype=dt, device=device) for dt in out_dtypes]
    outv = [torch.empty(nrows, dtype=torch.uint8, device=device) if w else None for w in want_valid]
    if nrows == 0:
        return outs, outv
    prog = (_lib.ExprIns * len(program))()
    for i, (op, kind, b, flags, imm) in enumerate(program):
        prog[i].op, prog[i].kind, prog[i].b, prog[i].flags = op, kind, b, flags
        imm &= (1 << 64) - 1
        prog[i].imm = imm - (1 << 64) if imm >= (1 << 63) else imm
    tables = {b for op, kind, b, _, _ in program if op == X_LOOKUP}  # per-entry tables: any length
    for j, (c, tp) in enumerate(zip(cols, col_types)):
        assert c.is_cuda and c.is_contiguous() and (j in tables or c.shape[0] == nrows)
        assert c.element_size() == EXPR_STORAGE[tp].itemsize, f"{c.dtype} column can't hold K8 type {tp}"
    _lib.check(lib.fb_eval_expr(
        device.index, _stream_ptr(device), nrows, len(cols), _lib.ptr_array([c.data_ptr() for c in cols]),
        _lib.i32_array(col_types),
        _lib.ptr_array([0 if v is None else v.data_ptr() for v in valid]), len(program), prog, len(outs),
        _lib.i32_array(out_types),
        _lib.ptr_array([o.data_ptr() for o in outs]),
        _lib.ptr_array([0 if v is None else v.data_ptr() for v in outv])))
    return outs, outv


# ---- K11: string functions over a dictionary's entries ------------------------------------------
LIKE_MAX_TOKENS, LIKE_ONE, LIKE_ANY = 1024, 256, 257


def string_length(offsets: torch.Tensor, data: torch.Tensor, valid: Optional[torch.Tensor]) -> torch.Tensor:
    """Code points of every entry of a device dictionary (int64 ``offsets`` of n + 1 entries, uint8 UTF-8
    ``data``, uint8 ``valid`` or None); 0 for a NULL entry."""
    lib = _lib.load()
    dev = offsets.device
    n = int(offsets.shape[0]) - 1
    out = torch.empty(n, dtype=torch.int64, device=dev)
    _lib.check(lib.fb_string_length(dev.index, _stream_ptr(dev), n, offsets.data_ptr(), data.data_ptr(),
                                    0 if valid is None else valid.data_ptr(), out.data_ptr()))
    return out


def string_like(offsets: torch.Tensor, data: torch.Tensor, valid: Optional[torch.Tensor],
                tokens: Sequence[int]) -> Tuple[torch.Tensor, torch.Tensor]:
    """(match, validity) of every entry, uint8 each: the entries against a pattern compiled to ``tokens``
    (literal bytes, ``LIKE_ONE`` for ``_``, ``LIKE_ANY`` for ``%``)."""
    lib = _lib.load()
    dev = offsets.device
    n = int(offsets.shape[0]) - 1
    out = torch.empty(n, dtype=torch.uint8, device=dev)
    out_valid = torch.empty(n, dtype=torch.uint8, device=dev)
    toks = (C.c_int16 * max(len(tokens), 1))(*tokens)
    _lib.check(lib.fb_string_like(dev.index, _stream_ptr(dev), n, offsets.data_ptr(), data.data_ptr(),
                                  0 if valid is None else valid.data_ptr(), len(tokens), toks, out.data_ptr(),
                                  out_valid.data_ptr()))
    return out, out_valid


# ---- K12: string-building functions over a dictionary's entries ---------------------------------
STR_MAX_LITERAL, STR_MAX_TOKENS, STR_SELF = 256, 1024, 256
(STR_COPY, STR_UPPER, STR_LOWER, STR_SUBSTR, STR_LTRIM, STR_RTRIM, STR_TRIM, STR_REPLACE, STR_FORMAT) = range(9)


def string_transform(op: int, offsets: torch.Tensor, data: torch.Tensor, valid: Optional[torch.Tensor],
                     src: Optional[torch.Tensor] = None, start: int = 0, length: Optional[int] = None,
                     lits: Sequence[bytes] = (), tokens: Sequence[int] = (), null_is_empty: bool = False,
                     out_offsets: Optional[torch.Tensor] = None, out_data: Optional[torch.Tensor] = None
                     ) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """One ``fb_string_transform`` call over the entries of a device dictionary (int64 ``offsets``, uint8
    ``data`` and ``valid``), or over the entries ``src`` (int64) when given.  Without ``out_data`` it is the
    measure call and returns (byte length int64, validity uint8) per output; with ``out_offsets`` /
    ``out_data`` it fills the bytes and returns (None, None).  ``lits``: up to two literal arguments."""
    lib = _lib.load()
    dev = offsets.device
    n = int(src.shape[0]) if src is not None else int(offsets.shape[0]) - 1
    lit0, lit1 = (list(lits) + [b"", b""])[:2]
    toks = (C.c_int16 * max(len(tokens), 1))(*tokens)
    out_len = out_valid = None
    if out_data is None:
        out_len = torch.empty(n, dtype=torch.int64, device=dev)
        out_valid = torch.empty(n, dtype=torch.uint8, device=dev)
    _lib.check(lib.fb_string_transform(
        dev.index, _stream_ptr(dev), op, n, offsets.data_ptr(), data.data_ptr(),
        0 if valid is None else valid.data_ptr(), 0 if src is None else src.data_ptr(), start,
        0 if length is None else length, int(length is not None), len(lit0), lit0, len(lit1), lit1, len(tokens),
        toks, int(null_is_empty), 0 if out_len is None else out_len.data_ptr(),
        0 if out_valid is None else out_valid.data_ptr(), 0 if out_offsets is None else out_offsets.data_ptr(),
        0 if out_data is None else out_data.data_ptr()))
    return out_len, out_valid


def string_hash(offsets: torch.Tensor, data: torch.Tensor, valid: Optional[torch.Tensor], bits: int = 64
                ) -> torch.Tensor:
    """A 64-bit hash of every entry's bytes (its low ``bits`` kept), as int64; 0 for a NULL entry."""
    lib = _lib.load()
    dev = offsets.device
    n = int(offsets.shape[0]) - 1
    out = torch.empty(n, dtype=torch.int64, device=dev)
    _lib.check(lib.fb_string_hash(dev.index, _stream_ptr(dev), n, offsets.data_ptr(), data.data_ptr(),
                                  0 if valid is None else valid.data_ptr(), bits, out.data_ptr()))
    return out


def string_first_equal(offsets: torch.Tensor, data: torch.Tensor, valid: Optional[torch.Tensor],
                       sorted_hash: torch.Tensor, sorted_idx: torch.Tensor) -> torch.Tensor:
    """Per entry: the smallest entry id with equal bytes (int64), from the stably sorted (hash, entry) pairs."""
    lib = _lib.load()
    dev = offsets.device
    n = int(offsets.shape[0]) - 1
    out = torch.empty(n, dtype=torch.int64, device=dev)
    _lib.check(lib.fb_string_first_equal(dev.index, _stream_ptr(dev), n, offsets.data_ptr(), data.data_ptr(),
                                         0 if valid is None else valid.data_ptr(), sorted_hash.data_ptr(),
                                         sorted_idx.data_ptr(), out.data_ptr()))
    return out


# ---- K15: regular expressions over a dictionary's entries ---------------------------------------
def _program_on(prog: Any, dev: torch.device) -> torch.Tensor:
    return torch.frombuffer(bytearray(bytes(prog)), dtype=torch.uint8).to(dev)


def regex_match(offsets: torch.Tensor, data: torch.Tensor, valid: Optional[torch.Tensor], prog: Any
                ) -> Tuple[torch.Tensor, torch.Tensor]:
    """(match, validity) of every entry, uint8 each, for a ``regex.match_program``."""
    lib = _lib.load()
    dev = offsets.device
    n = int(offsets.shape[0]) - 1
    out = torch.empty(n, dtype=torch.uint8, device=dev)
    out_valid = torch.empty(n, dtype=torch.uint8, device=dev)
    dprog = _program_on(prog, dev)
    _lib.check(lib.fb_regex_match(dev.index, _stream_ptr(dev), n, offsets.data_ptr(), data.data_ptr(),
                                  0 if valid is None else valid.data_ptr(), C.addressof(prog), dprog.data_ptr(),
                                  out.data_ptr(), out_valid.data_ptr()))
    return out, out_valid


def regex_transform(offsets: torch.Tensor, data: torch.Tensor, valid: Optional[torch.Tensor], prog: Any,
                    out_offsets: Optional[torch.Tensor] = None, out_data: Optional[torch.Tensor] = None
                    ) -> Tuple[Optional[torch.Tensor], Optional[torch.Tensor]]:
    """One ``fb_regex_transform`` call (``regex.extract_program`` / ``replace_program``) with the measure / write
    contract of ``string_transform``."""
    lib = _lib.load()
    dev = offsets.device
    n = int(offsets.shape[0]) - 1
    out_len = out_valid = None
    if out_data is None:
        out_len = torch.empty(n, dtype=torch.int64, device=dev)
        out_valid = torch.empty(n, dtype=torch.uint8, device=dev)
    dprog = _program_on(prog, dev)
    _lib.check(lib.fb_regex_transform(
        dev.index, _stream_ptr(dev), n, offsets.data_ptr(), data.data_ptr(), 0 if valid is None else valid.data_ptr(),
        C.addressof(prog), dprog.data_ptr(), 0 if out_len is None else out_len.data_ptr(),
        0 if out_valid is None else out_valid.data_ptr(), 0 if out_offsets is None else out_offsets.data_ptr(),
        0 if out_data is None else out_data.data_ptr()))
    return out_len, out_valid


def regex_host(offsets: np.ndarray, data: np.ndarray, valid: Optional[np.ndarray], prog: Any
               ) -> Tuple[np.ndarray, np.ndarray, Optional[np.ndarray]]:
    """Either regex call on the CPU over host arrays (int64 ``offsets``, uint8 ``data`` / ``valid``), by the same
    per-entry code as the kernels: (0 / 1 match or byte length per entry (int64), validity, result offsets and
    bytes as one (offsets, data) pair, None for a match program)."""
    lib = _lib.load()
    n = int(offsets.shape[0]) - 1
    data = data if data.size else np.zeros(1, dtype=np.uint8)
    out = np.zeros(max(n, 1), dtype=np.int64)
    out_valid = np.zeros(max(n, 1), dtype=np.uint8)
    vp = 0 if valid is None else valid.ctypes.data
    _lib.check(lib.fb_debug_regex_host(n, offsets.ctypes.data, data.ctypes.data, vp, C.addressof(prog),
                                       out.ctypes.data, out_valid.ctypes.data, 0, 0))
    if prog.op == 0:
        return out[:n], out_valid[:n], None
    offs = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(out[:n], out=offs[1:])
    buf = np.zeros(max(int(offs[-1]), 1), dtype=np.uint8)
    _lib.check(lib.fb_debug_regex_host(n, offsets.ctypes.data, data.ctypes.data, vp, C.addressof(prog),
                                       0, 0, offs.ctypes.data, buf.ctypes.data))
    return out[:n], out_valid[:n], (offs, buf)


# ---- K13: string casts over a dictionary's entries ----------------------------------------------
(PARSE_I8, PARSE_I16, PARSE_I32, PARSE_I64, PARSE_U8, PARSE_U16, PARSE_U32, PARSE_U64, PARSE_F32, PARSE_F64,
 PARSE_BOOL, PARSE_DATE32, PARSE_DATE64) = range(13)
PARSE_TS, PARSE_TS_ZONED = 16, 8  # PARSE_TS + TU_S .. TU_NS (+ PARSE_TS_ZONED)
PARSE_OK, PARSE_NULL, PARSE_INVALID, PARSE_UNDECIDED = range(4)


def string_parse(offsets: torch.Tensor, data: torch.Tensor, valid: Optional[torch.Tensor], target: int
                 ) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, Optional[int]]:
    """Every entry of a device dictionary parsed to ``target`` (a ``PARSE_*`` code): (value int64, validity uint8,
    status uint8 per entry, the smallest entry whose status is ``PARSE_INVALID`` / ``PARSE_UNDECIDED`` or None).
    The last one is the only value read back to the host."""
    lib = _lib.load()
    dev = offsets.device
    n = int(offsets.shape[0]) - 1
    out = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    out_valid = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
    status = torch.empty(max(n, 1), dtype=torch.uint8, device=dev)
    first_bad = torch.empty(1, dtype=torch.int64, device=dev)
    _lib.check(lib.fb_string_parse(dev.index, _stream_ptr(dev), n, offsets.data_ptr(), data.data_ptr(),
                                   0 if valid is None else valid.data_ptr(), target, out.data_ptr(),
                                   out_valid.data_ptr(), status.data_ptr(), first_bad.data_ptr()))
    bad = int(first_bad.item())  # UINT64_MAX reads as -1
    return out[:n], out_valid[:n], status[:n], (None if bad < 0 else bad)


def string_parse_host(offsets: np.ndarray, data: np.ndarray, valid: Optional[np.ndarray], target: int
                      ) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """``string_parse`` on the CPU over host arrays (int64 ``offsets``, uint8 ``data`` / ``valid``), by the same
    parse routines: (value int64, validity uint8, status uint8)."""
    lib = _lib.load()
    n = int(offsets.shape[0]) - 1
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    data = np.ascontiguousarray(data, dtype=np.uint8) if len(data) else np.zeros(1, dtype=np.uint8)
    out = np.empty(max(n, 1), dtype=np.int64)
    out_valid = np.empty(max(n, 1), dtype=np.uint8)
    status = np.empty(max(n, 1), dtype=np.uint8)
    if valid is not None:
        valid = np.ascontiguousarray(valid, dtype=np.uint8)
    _lib.check(lib.fb_debug_string_parse_host(n, offsets.ctypes.data, data.ctypes.data,
                                              0 if valid is None else valid.ctypes.data, target, out.ctypes.data,
                                              out_valid.ctypes.data, status.ctypes.data))
    return out[:n], out_valid[:n], status[:n]


# ---- K14: casts to string, one text per value ----------------------------------------------------
FMT_I64, FMT_U64, FMT_BOOL, FMT_F64, FMT_DATE32, FMT_DATE64 = range(6)
FMT_TS, FMT_TS_FRAC = 8, 16  # FMT_TS + TU_S .. TU_NS (+ FMT_TS_FRAC: the unit's fraction digits on every value)


def value_format(values: torch.Tensor, valid: Optional[torch.Tensor], kind: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """The text of every value (one 8-byte word each: an int64 / uint64 / float64 bit pattern / date or timestamp
    count, ``kind`` a ``FMT_*`` code) on the device: (offsets int64, n + 1 entries; UTF-8 bytes uint8, at least one
    byte).  A value whose ``valid`` byte is 0 gets no bytes."""
    from .strings import _scan

    lib = _lib.load()
    dev = values.device
    n = int(values.shape[0])
    values = values.contiguous()
    vp = 0 if valid is None else valid.contiguous().data_ptr()
    lengths = torch.empty(n, dtype=torch.int64, device=dev)
    _lib.check(lib.fb_value_format(dev.index, _stream_ptr(dev), n, values.data_ptr(), vp, kind, lengths.data_ptr(),
                                   0, 0))
    offsets, total = _scan(lengths)
    data = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
    _lib.check(lib.fb_value_format(dev.index, _stream_ptr(dev), n, values.data_ptr(), vp, kind, 0,
                                   offsets.data_ptr(), data.data_ptr()))
    return offsets, data


def value_format_host(values: np.ndarray, valid: Optional[np.ndarray], kind: int) -> Tuple[np.ndarray, np.ndarray]:
    """``value_format`` on the CPU over host arrays (8-byte ``values``, uint8 ``valid``), by the same format
    routines: (offsets int64, UTF-8 bytes uint8)."""
    lib = _lib.load()
    n = int(values.shape[0])
    values = np.ascontiguousarray(values).view(np.uint64)
    if valid is not None:
        valid = np.ascontiguousarray(valid, dtype=np.uint8)
    vp = 0 if valid is None else valid.ctypes.data
    lengths = np.zeros(max(n, 1), dtype=np.int64)
    _lib.check(lib.fb_debug_value_format_host(n, values.ctypes.data, vp, kind, lengths.ctypes.data, 0, 0))
    offsets = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lengths[:n], out=offsets[1:])
    data = np.zeros(max(int(offsets[-1]), 1), dtype=np.uint8)
    _lib.check(lib.fb_debug_value_format_host(n, values.ctypes.data, vp, kind, 0, offsets.ctypes.data,
                                              data.ctypes.data))
    return offsets, data
