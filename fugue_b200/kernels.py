"""Thin tensor-level wrappers over the C ABI.

torch is used here only as the owner of device memory and streams; every
operation is a call into ``libfugue_b200.so``.
"""
from typing import Any, List, Optional, Sequence, Tuple

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


def segmented_scan(offsets: torch.Tensor, nrows: int,
                   columns: Sequence[Tuple[int, Optional[torch.Tensor], Optional[torch.Tensor]]]
                   ) -> List[Tuple[Optional[torch.Tensor], torch.Tensor]]:
    """K9: inclusive scan restarting at every segment ``[offsets[s], offsets[s + 1])``.  ``columns`` = one
    ``(op, values or None, validity or None)`` per scan (``AGG_*`` ops; 8-byte values, none for
    ``AGG_COUNT``).  Returns per scan ``(running op over the valid rows or None for COUNT, running count of
    the valid rows)``; up to ``SCAN_MAX_COLS`` scans share one launch sequence."""
    lib = _lib.load()
    assert offsets.dtype == torch.int64 and offsets.is_cuda and offsets.is_contiguous()
    dev = offsets.device
    nseg = int(offsets.shape[0]) - 1
    res: List[Tuple[Optional[torch.Tensor], torch.Tensor]] = []
    for b in range(0, len(columns), SCAN_MAX_COLS):
        batch = columns[b:b + SCAN_MAX_COLS]
        outs, cnts = [], []
        for op, v, m in batch:
            assert (v is None) == (op == AGG_COUNT)
            if v is not None:
                assert v.element_size() == 8 and v.device == dev and v.is_contiguous() and v.shape[0] == nrows
            if m is not None:
                assert m.dtype == torch.uint8 and m.device == dev and m.is_contiguous() and m.shape[0] == nrows
            outs.append(None if v is None else torch.empty_like(v))
            cnts.append(torch.empty(nrows, dtype=torch.int64, device=dev))
        nb = int(lib.fb_segmented_scan_scratch_bytes(nrows, len(batch)))
        scratch = torch.empty(max(nb, 8), dtype=torch.uint8, device=dev)
        _lib.check(lib.fb_segmented_scan(
            dev.index, _stream_ptr(dev), nrows, nseg, offsets.data_ptr(), len(batch),
            _lib.i32_array([op for op, _, _ in batch]),
            _lib.ptr_array([0 if v is None else v.data_ptr() for _, v, _ in batch]),
            _lib.ptr_array([0 if m is None else m.data_ptr() for _, _, m in batch]),
            _lib.ptr_array([0 if o is None else o.data_ptr() for o in outs]),
            _lib.ptr_array([c.data_ptr() for c in cnts]), scratch.data_ptr(), scratch.numel()))
        res.extend(zip(outs, cnts))
    return res


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
T_I8, T_I16, T_I32, T_I64, T_U8, T_F32, T_F64 = range(7)
XK_NONE, XK_REG, XK_COL, XK_IMM, XK_NULL = range(5)
XF_B_I2F = 1
(X_MOV, X_ST, X_OUT, X_I2F, X_F2I, X_NEG_I, X_NEG_F, X_NOT, X_IS_NULL, X_NOT_NULL, X_TOBOOL_I, X_TOBOOL_F,
 X_ADD_I, X_SUB_I, X_RSUB_I, X_MUL_I, X_ADD_F, X_SUB_F, X_RSUB_F, X_MUL_F, X_DIV_F, X_RDIV_F,
 X_LT_I, X_LE_I, X_GT_I, X_GE_I, X_EQ_I, X_NE_I, X_LT_F, X_LE_F, X_GT_F, X_GE_F, X_EQ_F, X_NE_F,
 X_AND, X_OR, X_COALESCE, X_RCOALESCE) = range(38)

_EXPR_TYPE_OF_DTYPE = {torch.int8: T_I8, torch.int16: T_I16, torch.int32: T_I32, torch.int64: T_I64,
                       torch.uint8: T_U8, torch.bool: T_U8, torch.float32: T_F32, torch.float64: T_F64}


def expr_type_of(dtype: torch.dtype) -> int:
    return _EXPR_TYPE_OF_DTYPE[dtype]


def eval_expr(nrows: int, device: torch.device, cols: Sequence[torch.Tensor],
              valid: Sequence[Optional[torch.Tensor]], program: Sequence[Tuple[int, int, int, int, int]],
              out_dtypes: Sequence[torch.dtype], want_valid: Sequence[bool]
              ) -> Tuple[List[torch.Tensor], List[Optional[torch.Tensor]]]:
    """Run one accumulator-machine ``program`` (tuples ``(op, operand_kind, b, flags, imm_bits)``, see
    include/fugue_b200.h K8) over all rows; ``X_OUT b`` writes output ``b``.  Returns the output
    columns and (where asked for) their validity byte masks."""
    lib = _lib.load()
    outs = [torch.empty(nrows, dtype=dt, device=device) for dt in out_dtypes]
    outv = [torch.empty(nrows, dtype=torch.uint8, device=device) if w else None for w in want_valid]
    if nrows == 0:
        return outs, outv
    prog = (_lib.ExprIns * len(program))()
    for i, (op, kind, b, flags, imm) in enumerate(program):
        prog[i].op, prog[i].kind, prog[i].b, prog[i].flags = op, kind, b, flags
        imm &= (1 << 64) - 1
        prog[i].imm = imm - (1 << 64) if imm >= (1 << 63) else imm
    for c in cols:
        assert c.is_cuda and c.is_contiguous() and c.shape[0] == nrows
    _lib.check(lib.fb_eval_expr(
        device.index, _stream_ptr(device), nrows, len(cols), _lib.ptr_array([c.data_ptr() for c in cols]),
        _lib.i32_array([expr_type_of(c.dtype) for c in cols]),
        _lib.ptr_array([0 if v is None else v.data_ptr() for v in valid]), len(program), prog, len(outs),
        _lib.i32_array([expr_type_of(dt) for dt in out_dtypes]),
        _lib.ptr_array([o.data_ptr() for o in outs]),
        _lib.ptr_array([0 if v is None else v.data_ptr() for v in outv])))
    return outs, outv
