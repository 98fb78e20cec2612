"""Pipelined host -> device -> host ``transform`` for host-resident inputs.

``fa.transform(host_table, fn_typed_on_B200Table, partition=hash spec, as_local=True)`` moves every
byte over PCIe twice; done step by step (to_df, map_dataframe, as_local) that costs
H2D + compute + D2H.  Here the three phases overlap column by column on three CUDA streams:

    copy-in stream : key column(s) first, then the other columns, one H2D per column chunk
    compute stream : pass 1 (histogram/scan) as soon as the keys are on the device, then one
                     ``fb_partition_apply`` per column as soon as that column has arrived
    copy-out stream: D2H of an output column as soon as its scatter has finished

The map function is called once on the partitioned device table right after the work is
enqueued (CUDA stream order makes whatever it launches run after the scatters); result columns
that are passed through untouched start their D2H early, computed columns wait for the function.
PCIe is full duplex, so the wall time approaches max(H2D, D2H) instead of their sum.

Semantics are those of ``B200MapEngine.map_dataframe`` with ``map_func_format_hint == "b200"``
(fugue/execution/execution_engine.py:283-315); only fixed-width, NULL-free columns take this
path, everything else uses the plain engine path.
"""
from typing import Any, List, Optional

import numpy as np
import pyarrow as pa
import torch

from . import kernels as K
from . import sort as S
from .dataframe import ArrowDataFrame, B200DataFrame, DataFrame
from .partition import PartitionSpec
from .schema import Schema
from .table import B200Table, _from_readonly, _np_storage, _storage_dtype


def _eligible(table: pa.Table, schema: Schema, spec: PartitionSpec) -> bool:
    if len(spec.partition_by) == 0 or spec.algo in ("coarse", "even", "rand") or len(spec.presort) > 0:
        return False  # even / rand number the distinct keys first (device sorts): not a one-pass hash partition
    if table.num_rows == 0:
        return False
    for name, tp in zip(schema.names, schema.types):
        if pa.types.is_string(tp) or pa.types.is_large_string(tp) or pa.types.is_boolean(tp):
            return False
        try:
            _storage_dtype(tp)
        except NotImplementedError:
            return False
        col = table.column(name)
        if col.null_count > 0 or col.type != tp:
            return False
    return True


def streaming_transform(engine: Any, local_df: DataFrame, runner: Any, out_schema: Schema,
                        spec: PartitionSpec) -> Optional[DataFrame]:
    """Returns the local result, or None when the input does not qualify for the pipelined path."""
    table = local_df.as_arrow()
    schema = local_df.schema
    if not _eligible(table, schema, spec):
        return None
    dev = engine.device
    n = table.num_rows
    keys = list(spec.partition_by)
    for k in keys:
        if k not in schema:
            raise KeyError(f"{k} not in {schema}")
    num = engine._num_partitions(spec, n)
    if num > K.MAX_PARTITIONS:
        return None
    order = keys + [c for c in schema.names if c not in keys]
    s_cmp = torch.cuda.current_stream(dev)
    s_in, s_out = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
    dcols = {c: torch.empty(n, dtype=_storage_dtype(schema[c].type), device=dev) for c in schema.names}
    outs = {c: torch.empty_like(dcols[c]) for c in schema.names}
    ev_in = {}
    s_in.wait_stream(s_cmp)  # allocations above are ordered before the copies
    with torch.cuda.stream(s_in):
        for c in order:
            pos = 0
            st = _np_storage(schema[c].type)
            for arr in table.column(c).chunks:
                m = len(arr)
                if m == 0:
                    continue
                host = np.frombuffer(arr.buffers()[1], dtype=st, count=m + arr.offset)[arr.offset:]
                dcols[c][pos:pos + m].copy_(_from_readonly(host), non_blocking=True)
                pos += m
            ev = torch.cuda.Event()
            ev.record(s_in)
            ev_in[c] = ev
    for k in keys:
        s_cmp.wait_event(ev_in[k])
    # pass 1 hashes float keys as the logical hash partition of map_dataframe does (DESIGN §7d): -0.0 read as 0.0,
    # NaN as NULL, float16 widened to float64; pass 2 moves the original columns
    kcols, kvalid = [dcols[k] for k in keys], [None] * len(keys)
    for i, k in enumerate(keys):
        if pa.types.is_floating(schema[k].type):
            kcols[i], kvalid[i] = S.float_key(dcols[k], schema[k].type, None)
    scratch = engine._pool.scratch(dev, K.partition_scratch_bytes(dev, n, num))
    plan = K.partition_plan(kcols, num, kvalid, scratch=scratch)
    ev_out = {}
    for c in order:
        s_cmp.wait_event(ev_in[c])
        K.partition_apply(plan, [dcols[c]], [outs[c]])
        ev = torch.cuda.Event()
        ev.record(s_cmp)
        ev_out[c] = ev
    part = B200Table(schema, [outs[c] for c in schema.names], offsets=plan.offsets, partition_keys=keys)
    cursor = spec.get_cursor(schema, 0)
    pdf = B200DataFrame(part)
    cursor.set(lambda: pdf.peek_array(), 0, 0)
    res = engine.to_df(runner(cursor, pdf))
    if res.schema != out_schema:
        raise AssertionError(f"map output {res.schema} mismatches given {out_schema}")
    rt: B200Table = res.native
    plain = all(not (pa.types.is_boolean(tp) or pa.types.is_string(tp) or pa.types.is_large_string(tp))
                and col.element_size() * 8 == tp.bit_width
                for tp, col in zip(out_schema.types, rt.columns))
    if any(v is not None for v in rt.valid) or len(rt.dictionaries) > 0 or not plain:
        return res.as_local()  # rare shapes (NULLs, strings, bool = one byte per row on the device): plain D2H
    ev_f = torch.cuda.Event()
    ev_f.record(s_cmp)
    passthrough = {(t.data_ptr(), t.numel()): c for c, t in outs.items()}
    hosts: List[torch.Tensor] = []
    with torch.cuda.stream(s_out):
        for col in rt.columns:
            src = passthrough.get((col.data_ptr(), col.numel()))
            # a pass-through column starts its D2H as soon as its scatter is done; tables are immutable
            # values (fugue/dataframe/dataframe.py:291-295): a map function must not write into its input
            s_out.wait_event(ev_out[src] if src is not None else ev_f)
            h = torch.empty(col.shape, dtype=col.dtype, pin_memory=True)
            h.copy_(col, non_blocking=True)
            hosts.append(h)
        done = torch.cuda.Event()
        done.record(s_out)
    done.synchronize()
    s_cmp.wait_stream(s_out)
    nout = rt.num_rows
    arrays = [pa.Array.from_buffers(tp, nout, [None, pa.py_buffer(h.numpy())])
              for h, tp in zip(hosts, out_schema.types)]
    return ArrowDataFrame(pa.Table.from_arrays(arrays, schema=out_schema.pa_schema))
