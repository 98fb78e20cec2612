"""``B200Table``: an Arrow-layout columnar table resident in GPU HBM.

One contiguous device buffer per column (Arrow primitive layout, fixed width
1/2/4/8 bytes) plus an optional byte-per-row validity mask.  Strings are
dictionary-encoded on ingest (int32 codes on the device, dictionary on the host);
bools are widened to one byte.  torch tensors are used purely as owners of
device memory.

This is the data type that crosses the engine boundary in place of the pandas
frame of the reference's ``PandasDataFrame`` (fugue/dataframe/pandas_dataframe.py:38)
/ the ``pa.Table`` of ``ArrowDataFrame`` (fugue/dataframe/arrow_dataframe.py:45).
"""
from typing import Any, Dict, List, Optional, Sequence

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import torch

from . import kernels as K
from .schema import Schema

_TORCH_OF_WIDTH = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def _storage_dtype(tp: pa.DataType) -> torch.dtype:
    if pa.types.is_boolean(tp) or tp == pa.uint8():
        return torch.uint8
    if tp == pa.int8():
        return torch.int8
    if tp in (pa.int16(), pa.uint16(), pa.float16()):
        return torch.int16
    if tp in (pa.int32(), pa.uint32(), pa.date32()) or pa.types.is_string(tp) or pa.types.is_large_string(tp):
        return torch.int32
    if tp == pa.float32():
        return torch.float32
    if tp == pa.float64():
        return torch.float64
    if tp in (pa.int64(), pa.uint64()) or pa.types.is_timestamp(tp) or pa.types.is_date64(tp) \
            or pa.types.is_duration(tp) or pa.types.is_time64(tp):
        return torch.int64
    raise NotImplementedError(f"B200Table can't hold arrow type {tp} on the device")


_EXPR_TYPE_OF_STORAGE = {torch.uint8: K.T_U8, torch.int8: K.T_I8, torch.int16: K.T_I16, torch.int32: K.T_I32,
                         torch.int64: K.T_I64, torch.float32: K.T_F32, torch.float64: K.T_F64}


def expr_type(tp: pa.DataType) -> int:
    """The K8 column type (``kernels.T_*``) that reads a column of arrow type ``tp`` by its value."""
    special = {pa.uint16(): K.T_U16, pa.uint32(): K.T_U32, pa.float16(): K.T_F16}
    return special.get(tp, _EXPR_TYPE_OF_STORAGE[_storage_dtype(tp)])


# (mantissa bits, exponent mask) of float16 and float32: where a NaN's sign and payload sit
_NAN_LAYOUT = {torch.float16: (10, 0x7C00), torch.float32: (23, 0x7F800000)}


def _nan_bits_to_f64(x: torch.Tensor, raw: torch.Tensor, small: torch.dtype) -> torch.Tensor:
    """``x`` (float64 from the device conversion of ``raw``, the float16 / float32 bits as int64) with every NaN
    replaced by the float64 NaN of the same sign and payload: the device conversion makes them all one NaN."""
    mbits, emask = _NAN_LAYOUT[small]
    width = 16 if small == torch.float16 else 32
    raw = raw & ((1 << width) - 1)
    nan = ((raw & emask) == emask) & ((raw & ((1 << mbits) - 1)) != 0)
    bits = (0x7FF << 52) | ((raw & ((1 << mbits) - 1)) << (52 - mbits))
    bits = torch.where((raw >> (width - 1)) == 1, bits + (-(1 << 63)), bits)  # the sign bit
    return torch.where(nan, bits, x.view(torch.int64)).view(torch.float64)


def _nan_bits_from_f64(v: torch.Tensor, small: torch.dtype) -> torch.Tensor:
    """``v`` (float64) converted to ``small`` with every NaN keeping its sign and the top bits of its payload (a
    payload that loses all its bits keeps the lowest one, so that it stays a NaN), as the storage integers."""
    mbits, emask = _NAN_LAYOUT[small]
    width = 16 if small == torch.float16 else 32
    store = torch.int16 if small == torch.float16 else torch.int32
    b = v.view(torch.int64)
    mant = (b >> (52 - mbits)) & ((1 << mbits) - 1)
    bits = (((b >> 63) & 1) << (width - 1)) | emask | torch.where(mant == 0, torch.ones_like(mant), mant)
    bits = torch.where(bits >= (1 << (width - 1)), bits - (1 << width), bits)  # as the signed storage integer
    return torch.where(torch.isnan(v), bits.to(store), v.to(small).view(store))


def widen(c: torch.Tensor, tp: pa.DataType) -> torch.Tensor:
    """A stored column as its canonical 64-bit value: float64 for float types, int64 for the rest.
    uint16 / uint32 zero-extend, float16 is decoded from its int16 storage (exactly, a NaN's sign and payload
    too); uint64 values >= 2**63 stay int64 bit patterns.  Returns ``c`` itself when it already is that."""
    if tp == pa.float16():
        return _nan_bits_to_f64(c.view(torch.float16).to(torch.float64), c.to(torch.int64), torch.float16)
    if tp == pa.float32():
        return _nan_bits_to_f64(c.to(torch.float64), c.view(torch.int32).to(torch.int64), torch.float32)
    if pa.types.is_floating(tp):
        return c.to(torch.float64)
    if tp == pa.uint16():
        return c.to(torch.int64) & 0xFFFF
    if tp == pa.uint32():
        return c.to(torch.int64) & 0xFFFFFFFF
    return c.to(torch.int64)


def narrow(v: torch.Tensor, tp: pa.DataType) -> torch.Tensor:
    """The inverse of ``widen`` for a value the type can hold: the storage of arrow type ``tp``."""
    sd = _storage_dtype(tp)
    if v.dtype == sd:
        return v
    if tp == pa.float16():
        return _nan_bits_from_f64(v.to(torch.float64), torch.float16)
    if tp == pa.float32():
        return _nan_bits_from_f64(v.to(torch.float64), torch.float32).view(torch.float32)
    return v.to(sd)


def _np_storage(tp: pa.DataType) -> np.dtype:
    return {torch.uint8: np.dtype("u1"), torch.int8: np.dtype("i1"), torch.int16: np.dtype("i2"),
            torch.int32: np.dtype("i4"), torch.int64: np.dtype("i8"), torch.float32: np.dtype("f4"),
            torch.float64: np.dtype("f8")}[_storage_dtype(tp)]


class B200Table:
    def __init__(self, schema: Schema, columns: Sequence[torch.Tensor],
                 valid: Optional[Sequence[Optional[torch.Tensor]]] = None,
                 dictionaries: Optional[Dict[str, pa.Array]] = None,
                 offsets: Optional[torch.Tensor] = None,
                 partition_keys: Optional[List[str]] = None):
        self.schema = schema if isinstance(schema, Schema) else Schema(schema)
        self.columns: List[torch.Tensor] = list(columns)
        assert len(self.columns) == len(self.schema), "column count != schema"
        self.valid: List[Optional[torch.Tensor]] = list(valid) if valid is not None else [None] * len(self.columns)
        self.dictionaries: Dict[str, pa.Array] = dict(dictionaries or {})
        # physical partitioning metadata (set by the engine after a hash partition)
        self.offsets = offsets                # int64 [num + 1] on the device
        self.partition_keys = partition_keys  # key column names the offsets refer to
        self.logical_offsets: Optional[torch.Tensor] = None  # set after a device presort: one segment
        #                                                      per distinct key tuple (logical partition)
        self.logical_order: Optional[List[str]] = None  # presort columns the rows of a logical partition are
        #                                                 sorted by (peers of RANK / DENSE_RANK are equal on all)
        self.logical_ascending: Optional[List[bool]] = None  # their directions (NULLs last either way)
        # multi-GPU shuffle result (fugue_b200/dist.py): int64 [world, nown + 1] on the HOST; owned
        # partition j is the concatenation over source ranks s of rows
        # [segment_offsets[s, j], segment_offsets[s, j + 1]) - see compacted()
        self.segment_offsets: Optional[torch.Tensor] = None
        n = self.columns[0].shape[0] if self.columns else 0
        for c in self.columns:
            assert c.dim() == 1 and c.shape[0] == n and c.is_contiguous()
        self._nrows = n

    # ---- basic properties ---------------------------------------------------------------
    @property
    def num_rows(self) -> int:
        return self._nrows

    def __len__(self) -> int:
        return self._nrows

    @property
    def column_names(self) -> List[str]:
        return self.schema.names

    @property
    def device(self) -> torch.device:
        return self.columns[0].device if self.columns else torch.device("cuda", torch.cuda.current_device())

    @property
    def num_partitions(self) -> int:
        if self.offsets is None and self.segment_offsets is not None:
            return int(self.segment_offsets.shape[1]) - 1
        return 1 if self.offsets is None else int(self.offsets.shape[0]) - 1

    def compacted(self) -> "B200Table":
        """A multi-GPU shuffle leaves every owned partition as one segment per source rank
        (``segment_offsets``).  This returns the table with every partition contiguous (``offsets``),
        rows inside a partition in (source rank, source row) order: one local segment copy."""
        if self.segment_offsets is None or self.offsets is not None:
            return self
        from .dist import compact_plan

        src, dst, ln, off = compact_plan(self.segment_offsets)
        dev = self.device
        cols = list(self.columns) + [v for v in self.valid if v is not None]
        outs = [torch.empty_like(c) for c in cols]
        if self._nrows > 0:
            K.copy_segments(cols, outs, src.to(dev), dst.to(dev), ln.to(dev), max_len=int(ln.max()))
        ncol = len(self.columns)
        it = iter(outs[ncol:])
        valid = [None if v is None else next(it) for v in self.valid]
        res = B200Table(self.schema, outs[:ncol], valid, self.dictionaries, off.to(dev), self.partition_keys)
        for a in ("global_partition_range", "global_num_partitions"):
            if hasattr(self, a):
                setattr(res, a, getattr(self, a))
        return res

    def nbytes(self) -> int:
        return sum(c.numel() * c.element_size() for c in self.columns)

    def column(self, name: str) -> torch.Tensor:
        return self.columns[self.schema.index_of_key(name)]

    def typed_column(self, name: str) -> torch.Tensor:
        """Column viewed with the natural torch dtype of its arrow type (float64 as float64...)."""
        return self.column(name)

    def select(self, names: Sequence[str]) -> "B200Table":
        idx = [self.schema.index_of_key(n) for n in names]
        keep = self.partition_keys is not None and all(k in names for k in self.partition_keys)
        return B200Table(self.schema.extract(list(names)), [self.columns[i] for i in idx],
                         [self.valid[i] for i in idx],
                         {k: v for k, v in self.dictionaries.items() if k in names},
                         self.offsets if keep else None, self.partition_keys if keep else None)

    def rename(self, columns: Dict[str, str]) -> "B200Table":
        sch = self.schema.rename(columns)
        return B200Table(sch, self.columns, self.valid,
                         {columns.get(k, k): v for k, v in self.dictionaries.items()}, self.offsets,
                         None if self.partition_keys is None else [columns.get(k, k) for k in self.partition_keys])

    def slice(self, start: int, stop: int) -> "B200Table":
        return B200Table(self.schema, [c[start:stop] for c in self.columns],
                         [None if v is None else v[start:stop] for v in self.valid], self.dictionaries)

    def with_columns(self, schema: Schema, columns: Sequence[torch.Tensor],
                     valid: Optional[Sequence[Optional[torch.Tensor]]] = None) -> "B200Table":
        return B200Table(schema, columns, valid, self.dictionaries, self.offsets, self.partition_keys)

    # ---- host <-> device ---------------------------------------------------------------
    @staticmethod
    def from_arrow(table: pa.Table, device: Optional[torch.device] = None,
                   schema: Optional[Schema] = None) -> "B200Table":
        if not torch.cuda.is_available():
            from ._lib import FugueB200KernelError
            raise FugueB200KernelError("B200Table needs a CUDA device (no CPU fallback)")
        device = device or torch.device("cuda", torch.cuda.current_device())
        sch = schema or Schema(table.schema)
        cols: List[torch.Tensor] = []
        valids: List[Optional[torch.Tensor]] = []
        dicts: Dict[str, pa.Array] = {}
        for name, tp in zip(sch.names, sch.types):
            col = table.column(name)
            chunks = list(col.chunks) if isinstance(col, pa.ChunkedArray) else [col]
            is_str = pa.types.is_string(tp) or pa.types.is_large_string(tp)
            if is_str or len(chunks) == 0:
                # dictionary encoding needs one dictionary: combine on the host (ingest, not hot path)
                arr = col.combine_chunks() if isinstance(col, pa.ChunkedArray) and len(chunks) > 0 \
                    else (chunks[0] if chunks else pa.array([], type=tp))
                if isinstance(arr, pa.ChunkedArray):
                    arr = pa.array([], type=tp)
                chunks = [arr]
            prepared = []
            for arr in chunks:  # no host-side concatenation: every chunk is copied to its slice
                if arr.type != tp and not pa.types.is_dictionary(arr.type):
                    arr = arr.cast(tp)
                if is_str:
                    enc = arr if pa.types.is_dictionary(arr.type) else arr.dictionary_encode()
                    dicts[name] = enc.dictionary
                    arr = enc.indices.cast(pa.int32())
                elif pa.types.is_boolean(tp):
                    arr = pc.cast(arr, pa.uint8())
                prepared.append(arr)
            n = sum(len(a) for a in prepared)
            st = _np_storage(tp)
            dcol = torch.empty(n, dtype=_storage_dtype(tp), device=device)
            has_nulls = any(a.null_count > 0 for a in prepared)
            dvalid = torch.ones(n, dtype=torch.uint8, device=device) if has_nulls else None
            pos = 0
            for arr in prepared:
                m = len(arr)
                if m == 0:
                    continue
                bufs = arr.buffers()
                host = np.frombuffer(bufs[1], dtype=st, count=m + arr.offset)[arr.offset:]
                dcol[pos:pos + m].copy_(_from_readonly(host), non_blocking=True)
                if arr.null_count > 0 and bufs[0] is not None:
                    bits = np.frombuffer(bufs[0], dtype=np.uint8)
                    dbits = _from_readonly(bits).to(device, non_blocking=True)
                    dvalid[pos:pos + m].copy_(K.bits_to_bytes(dbits, arr.offset, m))
                pos += m
            cols.append(dcol)
            valids.append(dvalid)
        return B200Table(sch, cols, valids, dicts)

    def to_arrow(self) -> pa.Table:
        arrays = []
        n = self._nrows
        for (name, tp), col, v in zip(zip(self.schema.names, self.schema.types), self.columns, self.valid):
            host = torch.empty(col.shape, dtype=col.dtype, pin_memory=True)
            host.copy_(col, non_blocking=True)
            vbuf = None
            nulls = 0
            if v is not None:
                bits, nn = K.bytes_to_bits(v)
                hb = torch.empty(bits.shape, dtype=torch.uint8, pin_memory=True)
                hb.copy_(bits, non_blocking=True)
                torch.cuda.current_stream(col.device).synchronize()
                nulls = int(nn.item())
                vbuf = pa.py_buffer(hb.numpy())
            else:
                torch.cuda.current_stream(col.device).synchronize()
            data = pa.py_buffer(host.numpy())
            if pa.types.is_string(tp) or pa.types.is_large_string(tp):
                idx = pa.Array.from_buffers(pa.int32(), n, [vbuf, data], null_count=nulls)
                arr = pa.DictionaryArray.from_arrays(idx, self.dictionaries[name]).cast(tp)
            elif pa.types.is_boolean(tp):
                arr = pa.Array.from_buffers(pa.uint8(), n, [vbuf, data], null_count=nulls).cast(pa.bool_())
            else:
                arr = pa.Array.from_buffers(tp, n, [vbuf, data], null_count=nulls)
            arrays.append(arr)
        return pa.Table.from_arrays(arrays, schema=self.schema.pa_schema)

    def to_pandas(self):
        return self.to_arrow().to_pandas()

    def __repr__(self) -> str:
        return f"B200Table({self.schema}, rows={self._nrows}, partitions={self.num_partitions})"


def _from_readonly(a: np.ndarray) -> torch.Tensor:
    """torch tensor over a read-only numpy view (Arrow buffers are immutable; we only read)."""
    import warnings

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        return torch.from_numpy(a)
