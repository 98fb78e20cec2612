"""``B200ExecutionEngine`` / ``B200MapEngine``: the drop-in boundary of the hot path.

Mirrors the reference ABCs (names, argument meaning, error behaviour):
  * ``MapEngine.map_dataframe``      fugue/execution/execution_engine.py:283-315
      native implementation          fugue/execution/native_execution_engine.py:81-169
  * ``ExecutionEngine``              fugue/execution/execution_engine.py:338-1241
      to_df :93-114, repartition :488-502, persist :513-537, broadcast :504-511,
      join :539-561, aggregate :889-939, convert_yield_dataframe :941-960
The arithmetic runs in ``libfugue_b200.so`` through ``fugue_b200.kernels``; there is
no CPU implementation of the partition/join/aggregate steps in this package.
"""
import logging
from typing import Any, Callable, Dict, List, Optional

import pandas as pd
import pyarrow as pa
import torch

from . import kernels as K
from .dataframe import (ArrowDataFrame, B200DataFrame, DataFrame, LocalDataFrame, PandasDataFrame,
                        as_fugue_df)
from .lifecycle import FUGUE_GLOBAL_CONF, EngineLifecycle
from .partition import KEYWORD_PARALLELISM, KEYWORD_ROWCOUNT, PartitionCursor, PartitionSpec
from .schema import Schema
from .table import B200Table

FUGUE_B200_CONF_DEVICE = "fugue.b200.device"
FUGUE_B200_CONF_DEFAULT_PARTITIONS = "fugue.b200.default.partitions"
FUGUE_B200_DEFAULT_PARTITIONS = 256


def assert_or_throw(cond: bool, exc: Any) -> None:
    if not cond:
        e = exc() if callable(exc) and not isinstance(exc, type) else exc
        if isinstance(e, str):
            raise AssertionError(e)
        raise e


class _ScratchPool:
    """Reusable scratch / offsets buffers so no device allocation happens in steady state."""

    def __init__(self) -> None:
        self._scratch: Dict[Any, torch.Tensor] = {}

    def scratch(self, device: torch.device, nbytes: int) -> torch.Tensor:
        cur = self._scratch.get(device)
        if cur is None or cur.numel() < nbytes:
            cur = torch.empty(max(nbytes, 1 << 20), dtype=torch.uint8, device=device)
            self._scratch[device] = cur
        return cur


class B200MapEngine:
    """fugue/execution/execution_engine.py:277-335 (MapEngine facet)."""

    def __init__(self, execution_engine: "B200ExecutionEngine"):
        assert_or_throw(isinstance(execution_engine, B200ExecutionEngine),
                        lambda: TypeError(f"{self} expects a B200ExecutionEngine"))
        self._execution_engine = execution_engine

    @property
    def execution_engine(self) -> "B200ExecutionEngine":
        return self._execution_engine

    @property
    def execution_engine_constraint(self):
        return B200ExecutionEngine

    @property
    def is_distributed(self) -> bool:
        return self._execution_engine.is_distributed

    @property
    def log(self) -> logging.Logger:
        return self._execution_engine.log

    @property
    def conf(self) -> Dict[str, Any]:
        return self._execution_engine.conf

    def to_df(self, df: Any, schema: Any = None) -> DataFrame:
        return self._execution_engine.to_df(df, schema)

    def map_dataframe(
        self,
        df: DataFrame,
        map_func: Callable[[PartitionCursor, LocalDataFrame], LocalDataFrame],
        output_schema: Any,
        partition_spec: PartitionSpec,
        on_init: Optional[Callable[[int, DataFrame], Any]] = None,
        map_func_format_hint: Optional[str] = None,
    ) -> DataFrame:
        engine = self._execution_engine
        output_schema = Schema(output_schema)
        is_coarse = partition_spec.algo == "coarse"
        presort = partition_spec.get_sorts(df.schema, with_partition_keys=is_coarse)
        cursor = partition_spec.get_cursor(df.schema, 0)
        edf = engine.to_df(df)
        if on_init is not None:
            on_init(0, edf)
        keyed = len(partition_spec.partition_by) > 0 and not is_coarse
        cmap = getattr(map_func, "column_map", None)
        windowed = map_func_format_hint == "b200" and cmap is not None and cmap.has_window
        if windowed:
            # window functions (K9) need every logical partition contiguous and in presort order on one device
            assert_or_throw(not is_coarse, NotImplementedError(
                "window functions over algo='coarse' partitions: a coarse partition is not a logical partition"))
            assert_or_throw(keyed or partition_spec.num_partitions == "0", NotImplementedError(
                "window functions without partition keys but with num: the partitions of a key-less split are "
                "not logical partitions; give keys, or no num for one partition over the whole table"))
            assert_or_throw(not self.is_distributed, NotImplementedError(
                "window functions on the multi-GPU engine: the presort is local to each rank before the shuffle, "
                "so rows of one key from different ranks would not be merged in presort order"))
        if map_func_format_hint == "b200" and (len(presort) > 0 or windowed):
            # device presort: sort by (partition keys, presort) first; the stable hash partition below
            # keeps that order inside every physical partition, so logical partitions (distinct key
            # tuples) come out contiguous and presorted; their boundaries go to table.logical_offsets
            from collections import OrderedDict

            from . import sort as S

            order = OrderedDict((k, True) for k in (partition_spec.partition_by if keyed else []))
            for k, v in presort.items():
                order[k] = v
            edf = B200DataFrame(S.sort_table(edf.native, order))
        if keyed and cmap is not None and map_func_format_hint == "b200" and len(presort) == 0 and not windowed:
            fused = engine._repartition_fused_map(edf, partition_spec, cmap, output_schema)  # K4
            if fused is not None:
                return fused
        if keyed:
            edf = engine.repartition(edf, partition_spec)  # K1+K2+K3 on the device
        if map_func_format_hint == "b200":
            # device-vectorised map: the function is typed on B200Table and is called once per
            # device table, the physical partitions delimited by table.offsets (after a multi-GPU
            # shuffle: by table.segment_offsets, one segment per source rank and partition)
            if (len(presort) > 0 or windowed) and keyed:
                from . import sort as S

                if edf.native.segment_offsets is not None:
                    edf = B200DataFrame(edf.native.compacted())
                edf.native.logical_offsets = S.logical_offsets(edf.native, partition_spec.partition_by)
            if windowed:
                t = edf.native
                t = B200Table(t.schema, t.columns, t.valid, t.dictionaries, t.offsets, t.partition_keys)
                t.logical_offsets = edf.native.logical_offsets if keyed else \
                    torch.tensor([0, t.num_rows], dtype=torch.int64, device=t.device)
                t.logical_order = list(presort.keys())
                edf = B200DataFrame(t)
            cursor.set(lambda: edf.peek_array(), 0, 0)
            out = map_func(cursor, edf)
            res = engine.to_df(out)
            assert_or_throw(res.schema == output_schema,
                            lambda: f"map output {res.schema} mismatches given {output_schema}")
            return res
        return self._map_on_host(edf, map_func, output_schema, partition_spec, cursor, presort, keyed)

    # Python callbacks typed on pandas/arrow/lists run per logical partition on the host, exactly
    # as native_execution_engine.py:104-169 does; the device did the physical partitioning.
    def _map_on_host(self, edf: B200DataFrame, map_func: Any, output_schema: Schema,
                     spec: PartitionSpec, cursor: PartitionCursor, presort: Any, keyed: bool) -> DataFrame:
        engine = self._execution_engine
        presort_keys = list(presort.keys())
        presort_asc = list(presort.values())
        if keyed and edf.native.segment_offsets is not None:
            edf = B200DataFrame(edf.native.compacted())  # multi-GPU shuffle result: make partitions contiguous
        pdf = edf.as_pandas()
        outs: List[pd.DataFrame] = []

        def run(sub: pd.DataFrame, partition_no: int) -> None:
            if presort_keys:
                sub = sub.sort_values(presort_keys, ascending=presort_asc)
            sub = sub.reset_index(drop=True)
            input_df = PandasDataFrame(sub, edf.schema)
            cursor.set(lambda: input_df.peek_array(), partition_no, 0)
            out = map_func(cursor, input_df)
            outs.append(as_fugue_df(out).as_pandas())

        if not keyed:
            if len(spec.partition_by) == 0 and spec.num_partitions != "0":
                import numpy as np

                n = spec.get_num_partitions(**{KEYWORD_ROWCOUNT: lambda: len(pdf),
                                               KEYWORD_PARALLELISM: lambda: 1})
                if presort_keys:
                    pdf = pdf.sort_values(presort_keys, ascending=presort_asc).reset_index(drop=True)
                    presort_keys = []
                for p, sub in enumerate(np.array_split(pdf, n)):
                    if len(sub) > 0:
                        run(sub, p)
            else:
                run(pdf, 0)
        elif len(pdf) > 0:
            offsets = edf.native.offsets.cpu().tolist()
            no = 0
            for p in range(len(offsets) - 1):
                if offsets[p + 1] == offsets[p]:
                    continue
                part = pdf.iloc[offsets[p]:offsets[p + 1]]
                for _, sub in part.groupby(spec.partition_by, dropna=False, sort=True):
                    no += 1
                    run(sub, no)
        if not outs:
            return engine.to_df(ArrowDataFrame(None, output_schema))
        res = pd.concat(outs, ignore_index=True)
        return engine.to_df(PandasDataFrame(res, output_schema))


def decompose_aggs(agg_cols: List[Any]) -> Any:
    """Two-level form of plain aggregations: ``partial`` (computed per sub-group), ``final`` (computed
    over the partials) and ``post`` = [(name, sum column, count column)] for AVG = SUM / COUNT.
    Used for the multi-GPU group-by (partials per rank) and for COUNT(DISTINCT x) (partials per
    distinct (keys, x))."""
    from .column import Kind, agg as _agg, col

    partial: List[Any] = []
    final: List[Any] = []
    post: List[Any] = []
    for i, a in enumerate(agg_cols):
        assert_or_throw(a.kind == Kind.AGG and a.output_name != "",
                        lambda: ValueError(f"{a} must be a named aggregation"))
        tmp = f"__p{i}"
        if a.func in ("SUM", "MIN", "MAX"):
            partial.append(_agg(a.func, a.arg, tmp))
            final.append(_agg(a.func, col(tmp), a.output_name))
        elif a.func == "COUNT":
            partial.append(_agg("COUNT", a.arg, tmp))
            final.append(_agg("SUM", col(tmp), a.output_name))
        elif a.func == "AVG":
            partial.append(_agg("SUM", a.arg, tmp + "s"))
            partial.append(_agg("COUNT", a.arg, tmp + "c"))
            final.append(_agg("SUM", col(tmp + "s"), tmp + "s"))
            final.append(_agg("SUM", col(tmp + "c"), tmp + "c"))
            post.append((a.output_name, tmp + "s", tmp + "c"))
        else:
            raise NotImplementedError(f"{a.func} has no partial / final decomposition")
    return partial, final, post


def finish_avgs(res: "B200DataFrame", post: List[Any], want: List[str]) -> "B200DataFrame":
    """Replace the (sum, count) column pairs of ``decompose_aggs`` by their quotient."""
    if not post:
        return res
    t: B200Table = res.native
    fields, cols, valid = [], [], []
    drop = {x for p_ in post for x in p_[1:]}
    avg_at = {p_[1]: p_ for p_ in post}
    for name, tp, c, v in zip(t.schema.names, t.schema.types, t.columns, t.valid):
        if name in avg_at:
            out, sname, cname = avg_at[name]
            sc, cc = t.column(sname), t.column(cname)
            fields.append(pa.field(out, pa.float64()))
            cols.append((sc.to(torch.float64) / cc.to(torch.float64)).contiguous())
            valid.append((cc > 0).to(torch.uint8))
        elif name not in drop:
            fields.append(pa.field(name, tp))
            cols.append(c)
            valid.append(v)
    res = B200DataFrame(B200Table(Schema(fields), cols, valid, t.dictionaries))
    return res[want] if res.columns != want else res


class B200ExecutionEngine(EngineLifecycle):
    """The engine object ``fa.engine_context`` / ``fa.transform(engine=...)`` see.  Context / global / stop
    protocol: ``EngineLifecycle`` (fugue_b200/lifecycle.py)."""

    def __init__(self, conf: Any = None, **kwargs: Any):
        self._conf: Dict[str, Any] = {**FUGUE_GLOBAL_CONF, **dict(conf or {})}  # execution_engine.py:351-354
        self._conf.update(kwargs)
        self._log = logging.getLogger("fugue_b200")
        if not torch.cuda.is_available():
            from ._lib import FugueB200KernelError

            raise FugueB200KernelError(
                "B200ExecutionEngine needs a CUDA device: this engine has no CPU fallback")
        from . import _lib

        _lib.load()  # fail loudly here if the CUDA library is missing
        self._device = torch.device("cuda", int(self._conf.get(FUGUE_B200_CONF_DEVICE,
                                                               torch.cuda.current_device())))
        self._map_engine = B200MapEngine(self)
        self._pool = _ScratchPool()

    def __repr__(self) -> str:
        return f"B200ExecutionEngine({self._device})"

    # ---- facets / properties ----------------------------------------------------------
    @property
    def conf(self) -> Dict[str, Any]:
        return self._conf

    @property
    def log(self) -> logging.Logger:
        return self._log

    @property
    def device(self) -> torch.device:
        return self._device

    @property
    def is_distributed(self) -> bool:
        return False

    @property
    def map_engine(self) -> B200MapEngine:
        return self._map_engine

    def create_default_map_engine(self) -> B200MapEngine:
        return B200MapEngine(self)

    @property
    def sql_engine(self) -> Any:
        if getattr(self, "_sql_engine", None) is None:
            self._sql_engine = self.create_default_sql_engine()
        return self._sql_engine

    def create_default_sql_engine(self) -> Any:
        from .sql import B200SQLEngine

        return B200SQLEngine(self)

    def get_current_parallelism(self) -> int:
        return 1

    def stop_engine(self) -> None:
        """Called once, when the engine leaves its last context (or by ``stop()``): drops the cached scratch
        buffers.  The engine object stays usable; scratch is re-allocated on demand."""
        self._pool = _ScratchPool()

    # ---- ingest -----------------------------------------------------------------------
    def to_df(self, df: Any, schema: Any = None) -> B200DataFrame:
        """Any dataframe-like -> engine dataframe; returns the input itself if it already is one
        (execution_engine.py:107-112)."""
        if isinstance(df, B200DataFrame):
            assert_or_throw(schema is None or Schema(schema) == df.schema,
                            lambda: ValueError(f"schema {schema} doesn't match {df.schema}"))
            return df
        if isinstance(df, B200Table):
            return B200DataFrame(df, schema)
        if isinstance(df, DataFrame):
            res = B200DataFrame(B200Table.from_arrow(df.as_arrow(), self._device,
                                                     Schema(schema) if schema is not None else df.schema))
            if df.has_metadata:
                res.reset_metadata(df.metadata)
            return res
        local = as_fugue_df(df, schema)
        return B200DataFrame(B200Table.from_arrow(local.as_arrow(), self._device, local.schema))

    def persist(self, df: Any, lazy: bool = False, **kwargs: Any) -> B200DataFrame:
        return self.to_df(df)  # already materialised in HBM

    def broadcast(self, df: Any) -> B200DataFrame:
        return self.to_df(df)

    def convert_yield_dataframe(self, df: DataFrame, as_local: bool) -> DataFrame:
        return df.as_local() if as_local else df

    # ---- repartition (K1+K2+K3) ---------------------------------------------------------
    def _num_partitions(self, spec: PartitionSpec, nrows: int) -> int:
        n = spec.get_num_partitions(**{KEYWORD_ROWCOUNT: lambda: nrows,
                                       KEYWORD_PARALLELISM: lambda: self.get_current_parallelism()})
        if n <= 0:
            n = int(self._conf.get(FUGUE_B200_CONF_DEFAULT_PARTITIONS, FUGUE_B200_DEFAULT_PARTITIONS))
        return n

    def repartition(self, df: Any, partition_spec: PartitionSpec) -> B200DataFrame:
        """Physical repartition.  With keys every algo co-locates equal keys by hashing them
        (``hash_pandas_object(df[keys]) % num``, fugue_dask/_utils.py:146-169); without keys the
        single-device table already is one physical partition."""
        edf = self.to_df(df)
        keys = partition_spec.partition_by
        t: B200Table = edf.native
        for k in keys:
            assert_or_throw(k in t.schema, lambda: KeyError(f"{k} not in {t.schema}"))
        if partition_spec.algo in ("even", "rand"):
            return self._repartition_even_rand(edf, partition_spec)
        if len(keys) == 0:
            return edf
        num = self._num_partitions(partition_spec, t.num_rows)
        if t.offsets is not None and t.partition_keys == keys and t.num_partitions == num:
            return edf  # already partitioned this way
        if num > K.MAX_PARTITIONS:
            return self._repartition_wide(edf, keys, num)
        kidx = [t.schema.index_of_key(k) for k in keys]
        kvalid = [t.valid[i] for i in kidx]
        # validity masks travel as extra 1-byte columns
        cols = list(t.columns)
        vpos: Dict[int, int] = {}
        for i, v in enumerate(t.valid):
            if v is not None:
                vpos[i] = len(cols)
                cols.append(v)
        scratch = self._pool.scratch(t.device, K.partition_scratch_bytes(t.device, t.num_rows, num))
        out, offsets = K.partition_columns(cols, kidx, num, kvalid, scratch=scratch)
        ncol = len(t.columns)
        valid = [out[vpos[i]] if i in vpos else None for i in range(ncol)]
        res = B200Table(t.schema, out[:ncol], valid, t.dictionaries, offsets, list(keys))
        rdf = B200DataFrame(res)
        if edf.has_metadata:
            rdf.reset_metadata(edf.metadata)
        return rdf

    def _repartition_fused_map(self, edf: B200DataFrame, spec: PartitionSpec, cmap: Any,
                               output_schema: Schema) -> Optional[B200DataFrame]:
        """Hash partition + per-row map in ONE pass over the table (K4): pass 1 as usual, pass 2 with the
        map evaluated in the scatter kernel's epilogue (``fb_partition_apply_map``).  Returns None when
        the map (or the table) does not qualify - the caller then partitions and evaluates the map with
        the expression evaluator, still on the device."""
        t: B200Table = edf.native
        keys = list(spec.partition_by)
        if self.is_distributed or spec.algo in ("even", "rand") or t.num_rows == 0:
            return None
        for k in keys:
            if k not in t.schema:
                return None
        num = self._num_partitions(spec, t.num_rows)
        if num > 256 or (t.offsets is not None and t.partition_keys == keys and t.num_partitions == num):
            return None
        units = cmap.fusion_units(t)
        if units is None:
            return None
        names = [c.output_name for c in cmap.select(t).all_cols]
        got = Schema([pa.field(n, u[6]) for n, u in zip(names, units)])
        assert_or_throw(got == output_schema, lambda: f"map output {got} mismatches given {output_schema}")
        kidx = [t.schema.index_of_key(k) for k in keys]
        scratch = self._pool.scratch(t.device, K.partition_scratch_bytes(t.device, t.num_rows, num))
        plan = K.partition_plan([t.columns[i] for i in kidx], num, [t.valid[i] for i in kidx], scratch=scratch)
        outs = K.partition_apply_map(plan, [u[:6] for u in units])
        outs = [o.view(torch.float64) if u[6] == pa.float64() else
                (o.view(torch.int64) if o.dtype != torch.int64 and u[2] != K.MAP_COPY else o)
                for o, u in zip(outs, units)]
        plain = {n: u for n, u in zip(names, units) if u[2] == K.MAP_COPY}
        keep = all(k in plain and plain[k][0].data_ptr() == t.column(k).data_ptr() for k in keys)
        res = B200Table(output_schema, outs, None, {}, plan.offsets if keep else None, keys if keep else None)
        return B200DataFrame(res)

    def _repartition_wide(self, edf: B200DataFrame, keys: List[str], num: int) -> B200DataFrame:
        """More physical partitions than one radix pass separates (``num=65536``, ``PartitionSpec("per_row")``
        = ROWCOUNT partitions, fugue/collections/partition.py:95,115,186-207): the partition id
        ``hash % num`` of every row (K1) is sorted with stable byte-wise radix passes - the same
        partition kernels in digit mode, one pass per varying byte of the id - carrying the row number,
        and the table is gathered once.  Stable like the single-pass path, so the result is the same
        partition-contiguous table the oracle produces; ``offsets`` has ``num + 1`` entries."""
        from . import sort as S

        t: B200Table = edf.native
        dev, n = t.device, t.num_rows
        assert_or_throw(num < (1 << 32), NotImplementedError(f"num_partitions={num} >= 2^32"))
        kidx = [t.schema.index_of_key(k) for k in keys]
        if n == 0:
            res = B200Table(t.schema, t.columns, t.valid, t.dictionaries,
                            torch.zeros(num + 1, dtype=torch.int64, device=dev), list(keys))
            return B200DataFrame(res)
        pid = K.partition_ids([t.columns[i] for i in kidx], num, [t.valid[i] for i in kidx]).to(torch.int64)
        spid, idx = S._radix_sort_pairs(pid.contiguous(), torch.arange(n, dtype=torch.int64, device=dev))
        moved = S.take_rows(t, idx)
        offsets = torch.searchsorted(spid.contiguous(), torch.arange(num + 1, dtype=torch.int64, device=dev))
        res = B200Table(t.schema, moved.columns, moved.valid, t.dictionaries, offsets, list(keys))
        rdf = B200DataFrame(res)
        if edf.has_metadata:
            rdf.reset_metadata(edf.metadata)
        return rdf

    def _repartition_even_rand(self, edf: B200DataFrame, spec: PartitionSpec) -> B200DataFrame:
        """``algo="even"`` / ``"rand"`` with the meaning the distributed backends give them
        (fugue_dask/_utils.py:62-121): without keys the rows are cut into ``num`` equal contiguous
        ranges (rand: after a random permutation); with keys the distinct key tuples are numbered (in
        key order; rand: in random order) and spread evenly over ``num`` partitions, ``num <= 0``
        meaning one partition per group.  Built from the device sort (radix passes) and gathers."""
        from collections import OrderedDict

        from . import sort as S

        t: B200Table = edf.native
        keys = list(spec.partition_by)
        n, dev = t.num_rows, t.device
        rand = spec.algo == "rand"
        num = spec.get_num_partitions(**{KEYWORD_ROWCOUNT: lambda: n,
                                         KEYWORD_PARALLELISM: lambda: self.get_current_parallelism()})
        gen = torch.Generator(device=dev).manual_seed(int(self._conf.get("fugue.b200.rand.seed", 0)))

        def even_offsets(total: int, parts: int) -> torch.Tensor:
            return (torch.arange(parts + 1, dtype=torch.int64, device=dev) * total) // max(parts, 1)

        if len(keys) == 0:
            if num <= 1 or n == 0:
                return edf if not rand or n == 0 else B200DataFrame(
                    S.take_rows(t, torch.randperm(n, device=dev, generator=gen)))
            src = S.take_rows(t, torch.randperm(n, device=dev, generator=gen)) if rand else t
            res = B200Table(src.schema, src.columns, src.valid, src.dictionaries, even_offsets(n, num), [])
        else:
            if n == 0:
                return edf
            st = S.sort_table(t, OrderedDict((k, True) for k in keys), "first")
            gid = torch.cumsum(S.group_starts(st, keys).to(torch.int64), 0) - 1   # dense group number per row
            ngroups = int(gid[-1].item()) + 1
            if num <= 0:
                num = ngroups
            if rand:
                gid = torch.randperm(ngroups, device=dev, generator=gen)[gid]
            pid = (gid * num) // ngroups
            if rand:  # groups are no longer in partition order: one stable radix pass per varying byte
                spid, idx = S._radix_sort_pairs(pid.contiguous(), torch.arange(n, dtype=torch.int64, device=dev))
                st, pid = S.take_rows(st, idx), spid
            offsets = torch.searchsorted(pid.contiguous(), torch.arange(num + 1, dtype=torch.int64, device=dev))
            res = B200Table(st.schema, st.columns, st.valid, st.dictionaries, offsets, keys)
        rdf = B200DataFrame(res)
        if edf.has_metadata:
            rdf.reset_metadata(edf.metadata)
        return rdf

    # ---- aggregate (K6) -----------------------------------------------------------------
    def aggregate(self, df: Any, partition_spec: Optional[PartitionSpec], agg_cols: List[Any]) -> B200DataFrame:
        """``ExecutionEngine.aggregate`` (execution_engine.py:889-939): ``partition_spec.partition_by``
        are the GROUP BY keys, ``agg_cols`` named aggregation expressions.  Plain ``FUNC(column)``
        aggregations go straight to the sm_90a hash group-by kernel; anything richer
        (``(max(b) * 2).cast("int32")``, aggregations of expressions) goes through :meth:`select`,
        which evaluates the inner / outer expressions with the device evaluator around that kernel."""
        from .column import SelectColumns, col, is_agg

        assert_or_throw(len(agg_cols) > 0, ValueError("agg_cols can't be empty"))
        for a in agg_cols:
            assert_or_throw(is_agg(a), lambda: ValueError(f"{a} is not an aggregation"))
        agg_cols = [a.infer_alias() for a in agg_cols]
        for a in agg_cols:
            assert_or_throw(a.output_name != "", lambda: ValueError(f"{a} must have an alias"))
        if self._plain_aggs(agg_cols):
            return self._aggregate_named(df, partition_spec, agg_cols)
        keys = [] if partition_spec is None else list(partition_spec.partition_by)
        return self.select(df, SelectColumns(*[col(k) for k in keys], *agg_cols))

    @staticmethod
    def _plain_aggs(agg_cols: List[Any]) -> bool:
        """``SUM/COUNT/MIN/MAX/AVG`` of a named column (or ``*``) without casts: what the group-by
        kernel takes directly (and what the distributed engine decomposes into partial / final)."""
        from .column import ColumnExpr, Kind

        return all(isinstance(a, ColumnExpr) and a.kind == Kind.AGG and a.as_type is None and not a.is_distinct
                   and a.func in ("SUM", "COUNT", "MIN", "MAX", "AVG", "FIRST", "LAST")
                   and a.arg.kind in (Kind.NAMED, Kind.WILDCARD) and a.arg.as_type is None
                   and not (a.func in ("FIRST", "LAST") and a.arg.kind == Kind.WILDCARD)
                   for a in agg_cols)

    def _aggregate_named(self, df: Any, partition_spec: Optional[PartitionSpec],
                         agg_cols: List[Any]) -> B200DataFrame:
        """GROUP BY on named key columns with ``SUM/COUNT/MIN/MAX/AVG`` of named columns."""
        import pyarrow as pa

        edf = self.to_df(df)
        t: B200Table = edf.native
        keys = [] if partition_spec is None else list(partition_spec.partition_by)
        n = t.num_rows
        dev = t.device
        # ---- the 8-byte group key
        multi = len(keys) > 1
        kidx = [t.schema.index_of_key(k) for k in keys]

        def key_bits64(c: torch.Tensor) -> torch.Tensor:
            if c.dtype == torch.float64:
                return torch.where(c == 0, torch.zeros_like(c), c).view(torch.int64)  # -0.0 groups with 0.0
            if c.dtype == torch.float32:
                return torch.where(c == 0, torch.zeros_like(c), c).view(torch.int32).to(torch.int64)
            return c if c.dtype == torch.int64 else c.to(torch.int64)

        if len(keys) == 1:
            ki = kidx[0]
            kcol, kvalid, ktype = t.columns[ki], t.valid[ki], t.schema.types[ki]
            key64 = key_bits64(kcol)
        elif multi:
            # several key columns: group on the 64-bit hash of the key tuple (same hash as the
            # partitioner) and carry MIN/MAX of every key column as hidden aggregates: a group whose
            # MIN != MAX (or that mixes NULL and non-NULL) is a hash collision -> error instead of a
            # silently merged group.  The key values of the output are the MINs.
            kb = [key_bits64(t.columns[i]).contiguous() for i in kidx]
            key64 = K.row_hash64(kb, [t.valid[i] for i in kidx])
            kvalid, ktype = None, None
        else:
            key64, kvalid, ktype = torch.zeros(n, dtype=torch.int64, device=dev), None, None
        # ---- aggregates
        vals: List[Any] = []
        vvalid: List[Any] = []
        ops: List[int] = []
        plan: List[Any] = []  # (name, kind, slots..., out_type)

        def add(v: Any, m: Any, op: int) -> int:
            vals.append(v)
            vvalid.append(m)
            ops.append(op)
            return len(ops) - 1

        key_slots: List[Any] = []
        if multi:
            for i, kbits in zip(kidx, kb):
                m = t.valid[i]
                key_slots.append((add(kbits, m, K.AGG_MIN_I64), add(kbits, m, K.AGG_MAX_I64),
                                  add(None, m, K.AGG_COUNT) if m is not None else None))
            rows_slot = add(None, None, K.AGG_COUNT)
        rowno: Any = None
        for a in agg_cols:
            fn, arg = a.func, a.arg.name
            if fn == "COUNT":
                if arg == "*":
                    plan.append((a.output_name, "plain", add(None, None, K.AGG_COUNT), pa.int64(), None))
                else:
                    ci = t.schema.index_of_key(arg)
                    plan.append((a.output_name, "plain", add(None, t.valid[ci], K.AGG_COUNT), pa.int64(), None))
                continue
            ci = t.schema.index_of_key(arg)
            c, m, tp = t.columns[ci], t.valid[ci], t.schema.types[ci]
            if fn in ("FIRST", "LAST"):
                # first / last non-NULL value in input row order: MIN / MAX of the row number over the
                # rows where the value is not NULL, then one gather (works for every column type)
                if rowno is None:
                    rowno = torch.arange(n, dtype=torch.int64, device=dev)
                cnt = add(None, m, K.AGG_COUNT)
                plan.append((a.output_name, "pick", add(rowno, m, K.AGG_MIN_I64 if fn == "FIRST" else K.AGG_MAX_I64),
                             tp, (cnt, ci)))
                continue
            assert_or_throw(arg not in t.dictionaries, NotImplementedError(f"{fn} on a string column"))
            is_f = pa.types.is_floating(tp)
            c8 = c if c.element_size() == 8 else c.to(torch.float64 if is_f else torch.int64)
            # non-null count -> result validity.  A global aggregate (no keys) always carries it: over an
            # empty input (or an empty shard of a multi-GPU aggregate) SUM / MIN / MAX are NULL, not 0
            nn = add(None, m, K.AGG_COUNT) if (m is not None or len(keys) == 0) else None
            if fn == "SUM":
                plan.append((a.output_name, "plain", add(c8, m, K.AGG_SUM_F64 if is_f else K.AGG_SUM_I64),
                             pa.float64() if is_f else pa.int64(), nn))
            elif fn in ("MIN", "MAX"):
                op = {("MIN", True): K.AGG_MIN_F64, ("MAX", True): K.AGG_MAX_F64,
                      ("MIN", False): K.AGG_MIN_I64, ("MAX", False): K.AGG_MAX_I64}[(fn, is_f)]
                plan.append((a.output_name, "plain", add(c8, m, op), tp, nn))
            elif fn == "AVG":
                cf = c8 if is_f else c8.to(torch.float64)
                cnt = nn if nn is not None else add(None, None, K.AGG_COUNT)
                plan.append((a.output_name, "avg", add(cf, m, K.AGG_SUM_F64), pa.float64(), cnt))
            else:
                raise NotImplementedError(f"aggregation {fn}")
        assert_or_throw(len(ops) <= K.MAX_AGGS, NotImplementedError(
            f"{len(ops)} accumulators needed, one kernel call handles {K.MAX_AGGS}"))
        shuffled = getattr(t, "global_num_partitions", None) is not None and len(keys) > 0
        if shuffled:  # see kernels.scramble64: local partitions must not reuse the shuffle's hash
            key64 = K.scramble64(key64)
        gkeys, gvalid, gaggs, ng = K.groupby_u64(key64, kvalid, vals, vvalid, ops)
        if shuffled:
            gkeys = K.unscramble64(gkeys)
        if len(keys) == 0 and ng == 0:  # SQL: a global aggregate of an empty table is one row
            gaggs = [torch.zeros(1, dtype=torch.int64, device=dev) for _ in ops]
            ng = 1
        # ---- assemble the output table
        fields, cols, valids = [], [], []
        if multi:
            from .table import _storage_dtype

            bad = torch.zeros((), dtype=torch.bool, device=dev)
            for k, i, (smin, smax, scnt) in zip(keys, kidx, key_slots):
                bad |= (gaggs[smin] != gaggs[smax]).any() if scnt is None else \
                    (((gaggs[scnt] > 0) & (gaggs[smin] != gaggs[smax])) |
                     ((gaggs[scnt] > 0) & (gaggs[scnt] != gaggs[rows_slot]))).any()
                kc = t.columns[i]
                raw = gaggs[smin]
                if kc.dtype == torch.float64:
                    out_k = raw.view(torch.float64)
                elif kc.dtype == torch.float32:
                    out_k = raw.to(torch.int32).view(torch.float32)
                else:
                    out_k = raw if kc.dtype == torch.int64 else raw.to(kc.dtype)
                fields.append(pa.field(k, t.schema.types[i]))
                cols.append(out_k.contiguous())
                valids.append(None if scnt is None else (gaggs[scnt] > 0).to(torch.uint8))
            assert_or_throw(not bool(bad), RuntimeError(
                "64-bit hash collision between two distinct key tuples in a multi-column GROUP BY"))
        if len(keys) == 1:
            kc = t.columns[ki]
            if kc.dtype == torch.float64:
                out_k = gkeys.view(torch.float64)
            elif kc.dtype == torch.float32:
                out_k = gkeys.to(torch.int32).view(torch.float32)
            else:
                out_k = gkeys if kc.dtype == torch.int64 else gkeys.to(kc.dtype)
            fields.append(pa.field(keys[0], ktype))
            cols.append(out_k.contiguous())
            valids.append(gvalid)
        dicts = {k: t.dictionaries[k] for k in keys if k in t.dictionaries}
        for name, kind, slot, tp, nn in plan:
            raw = gaggs[slot]
            if kind == "pick":
                cnt, ci = nn
                has = gaggs[cnt] > 0
                idx = torch.where(has, raw, torch.zeros_like(raw))
                fields.append(pa.field(name, tp))
                cols.append(t.columns[ci][idx].contiguous() if n > 0 else t.columns[ci][:0])
                valids.append(has.to(torch.uint8))
                if t.schema.names[ci] in t.dictionaries:
                    dicts[name] = t.dictionaries[t.schema.names[ci]]
                continue
            v = None if nn is None else (gaggs[nn] > 0).to(torch.uint8)
            if kind == "avg":
                cnt = gaggs[nn].to(torch.float64)
                col = raw.view(torch.float64) / cnt
                v = (gaggs[nn] > 0).to(torch.uint8)
            elif pa.types.is_floating(tp):
                col = raw.view(torch.float64)
                if tp == pa.float32():
                    col = col.to(torch.float32)
            else:
                from .table import _storage_dtype

                sd = _storage_dtype(tp)
                col = raw if sd == torch.int64 else raw.to(sd)
            fields.append(pa.field(name, tp))
            cols.append(col.contiguous())
            valids.append(v)
        return B200DataFrame(B200Table(Schema(fields), cols, valids, dicts))

    # ---- select / filter / assign (K8) ---------------------------------------------------
    def select(self, df: Any, cols: Any, where: Any = None, having: Any = None) -> B200DataFrame:
        """``ExecutionEngine.select`` (execution_engine.py:736-806): ``SELECT cols FROM df [WHERE ...]
        [GROUP BY inferred keys] [HAVING ...]``.  Row-wise expressions run in the device evaluator
        (one pass per SELECT list), aggregations in the hash group-by kernel; nothing goes through
        SQL text.  Pins: fugue_test/execution_suite.py:98-155."""
        from . import expr as X
        from . import relational as R
        from .column import ColumnExpr, Kind, SelectColumns, agg as _agg, col, has_window, is_agg

        for e in list(cols.all_cols) + [where, having]:
            assert_or_throw(not has_window(e), lambda: NotImplementedError(
                f"{e}: a window function needs PARTITION BY / ORDER BY; use it in a ColumnMap of fa.transform"))
        edf = self.to_df(df)
        t: B200Table = edf.native
        sel: SelectColumns = cols.replace_wildcard(t.schema).assert_all_with_names()
        if where is not None:
            assert_or_throw(not is_agg(where), lambda: ValueError(f"{where} has aggregation functions"))
            t = X.filter_table(t, where)
        if not sel.has_agg:
            assert_or_throw(having is None, ValueError("HAVING needs an aggregation"))
            res = B200DataFrame(X.project(t, sel.all_cols))
            return R.distinct(self, res) if sel.is_distinct else res
        # ---- aggregation: pre-project (group keys, aggregation arguments) -> group-by -> post-project
        pre: List[Any] = []        # expressions of the temporary table
        pre_names: Dict[str, str] = {}
        key_names: List[str] = []

        def temp(e: Any, prefix: str) -> str:
            """Name of the temporary column holding ``e`` (plain columns keep their name)."""
            if e.kind == Kind.NAMED and e.as_type is None:
                if e.name not in pre_names:
                    pre_names[e.name] = e.name
                    pre.append(col(e.name))
                return e.name
            uid = e.fingerprint()
            if uid not in pre_names:
                pre_names[uid] = f"__fb_{prefix}{len(pre_names)}"
                pre.append(e.alias(pre_names[uid]))
            return pre_names[uid]

        key_of: Dict[str, str] = {}  # uuid of a group-key expression -> its column in the group table
        for k in sel.group_keys:
            nm = temp(k, "k")
            key_of[k.fingerprint()] = nm
            if nm not in key_names:
                key_names.append(nm)
        aggs: List[ColumnExpr] = []
        for c in sel.all_cols:
            X.find_aggs(c, aggs)
        if having is not None:
            X.find_aggs(having, aggs)
        agg_col: Dict[str, str] = {}  # uuid of FUNC(arg) -> its column in the group table
        named_aggs: List[ColumnExpr] = []
        distinct_on: Any = None       # ([temporary columns of the DISTINCT argument], is wildcard)
        distinct_outs: List[str] = []
        for a in aggs:
            bare = a.alias("").cast(None)
            uid = bare.fingerprint()
            if uid in agg_col:
                continue
            assert_or_throw(a.func in ("SUM", "COUNT", "MIN", "MAX", "AVG", "FIRST", "LAST"),
                            NotImplementedError(f"aggregation {a.func}"))
            assert_or_throw(not is_agg(a.arg), ValueError(f"nested aggregation {a}"))
            out = f"__fb_a{len(agg_col)}"
            agg_col[uid] = out
            if a.is_distinct:
                # COUNT(DISTINCT x): group by (keys, x) first, then count the sub-groups per key
                assert_or_throw(a.func == "COUNT", NotImplementedError(f"DISTINCT aggregation {a}"))
                dn = [temp(col(n), "d") for n in t.schema.names] if a.arg.kind == Kind.WILDCARD \
                    else [temp(a.arg, "d")]
                assert_or_throw(distinct_on is None or distinct_on[0] == dn, NotImplementedError(
                    "COUNT(DISTINCT ...) of different arguments in one SELECT"))
                distinct_on = (dn, a.arg.kind == Kind.WILDCARD)
                distinct_outs.append(out)
                continue
            if a.arg.kind == Kind.WILDCARD:
                named_aggs.append(_agg(a.func, col("*"), out))
            elif a.arg.kind == Kind.LITERAL:
                nm = temp(a.arg.alias("").cast(a.arg.as_type), "l")
                named_aggs.append(_agg(a.func, col(nm), out))
            else:
                named_aggs.append(_agg(a.func, col(temp(a.arg, "v")), out))
        if len(pre) == 0:  # e.g. SELECT COUNT(*) FROM t
            tmp = t
        else:
            tmp = X.project(t, pre)
        # (self.aggregate, not the local kernel wrapper: the distributed engine shuffles partials here)
        if distinct_on is None:
            g = self.aggregate(B200DataFrame(tmp), PartitionSpec(by=key_names) if key_names else None,
                               named_aggs).native
        else:
            dn, wildcard = distinct_on
            partial, final, post = decompose_aggs(named_aggs)
            lvl1 = key_names + [d for d in dn if d not in key_names]
            g1 = self.aggregate(B200DataFrame(tmp), PartitionSpec(by=lvl1),
                                partial if partial else [_agg("COUNT", col("*"), "__fb_n")])
            final = final + [_agg("COUNT", col("*") if wildcard else col(dn[0]), o) for o in distinct_outs]
            g2 = self.aggregate(g1, PartitionSpec(by=key_names) if key_names else None, final)
            g = finish_avgs(g2, post, key_names + [a.output_name for a in named_aggs] + distinct_outs).native

        def to_group_table(e: Any) -> Any:
            def mapper(node: Any) -> Any:
                if node.kind == Kind.AGG:
                    return col(agg_col[node.alias("").cast(None).fingerprint()])
                if node.kind == Kind.LITERAL:
                    return None
                uid = node.alias("").cast(None).fingerprint()
                if uid in key_of:
                    return col(key_of[uid])
                return None
            return X.rewrite(e, mapper)

        if having is not None:
            g = X.filter_table(g, to_group_table(having.alias("")))
        outs = [to_group_table(c).alias(c.output_name) for c in sel.all_cols]
        res = B200DataFrame(X.project(g, outs))
        # MIN/MAX/plain keys keep the input type when the expression says so (correct_select_schema)
        fix = {}
        for c in sel.all_cols:
            tp = c.infer_type(edf.schema)
            if tp is not None and tp != res.schema[c.output_name].type:
                fix[c.output_name] = tp
        if fix:
            res = B200DataFrame(X.project(res.native, [col(n).cast(fix[n]) if n in fix else col(n)
                                                       for n in res.schema.names]))
        return R.distinct(self, res) if sel.is_distinct else res

    def filter(self, df: Any, condition: Any) -> B200DataFrame:
        """``ExecutionEngine.filter`` (execution_engine.py:808-834): rows where ``condition`` is TRUE
        (predicate evaluated on the device, stream compaction + gather).  Pins: execution_suite.py:85-95."""
        from . import expr as X
        from .column import has_window, is_agg

        assert_or_throw(not is_agg(condition), lambda: ValueError(f"{condition} has aggregation functions"))
        assert_or_throw(not has_window(condition), lambda: NotImplementedError(
            f"{condition}: a window function needs PARTITION BY / ORDER BY; use it in a ColumnMap of fa.transform"))
        edf = self.to_df(df)
        res = B200DataFrame(X.filter_table(edf.native, condition))
        if edf.has_metadata:
            res.reset_metadata(edf.metadata)
        return res

    def assign(self, df: Any, columns: List[Any]) -> B200DataFrame:
        """``ExecutionEngine.assign`` (execution_engine.py:836-887): replace / append columns.
        Pins: execution_suite.py:157-174."""
        from .column import SelectColumns, col, has_window

        SelectColumns(*columns).assert_no_wildcard().assert_all_with_names().assert_no_agg()
        for c in columns:
            assert_or_throw(not has_window(c), lambda: NotImplementedError(
                f"{c}: a window function needs PARTITION BY / ORDER BY; use it in a ColumnMap of fa.transform"))
        edf = self.to_df(df)
        pos = {n: i for i, n in enumerate(edf.schema.names)}
        cols: List[Any] = [col(n) for n in pos]
        for c in columns:
            c = c.infer_alias()
            if c.output_name in pos:
                cols[pos[c.output_name]] = c
            else:
                cols.append(c)
        return self.select(edf, SelectColumns(*cols))

    # ---- join (K7) ----------------------------------------------------------------------
    def join(self, df1: Any, df2: Any, how: str, on: Optional[List[str]] = None) -> B200DataFrame:
        """``ExecutionEngine.join`` (execution_engine.py:539-561; native :230-241): equi-join on the
        common columns, NULL keys never match, output schema ``df1.schema`` U (``df2.schema`` - keys)."""
        from .join import device_join

        return device_join(self, self.to_df(df1), self.to_df(df2), how, on)

    # ---- set operations, NULL handling, sampling, IO (fugue_b200/relational.py) -----------
    def union(self, df1: Any, df2: Any, distinct: bool = True) -> B200DataFrame:
        from . import relational as R

        return R.union(self, self.to_df(df1), self.to_df(df2), distinct)

    def subtract(self, df1: Any, df2: Any, distinct: bool = True) -> B200DataFrame:
        from . import relational as R

        return R.subtract(self, self.to_df(df1), self.to_df(df2), distinct)

    def intersect(self, df1: Any, df2: Any, distinct: bool = True) -> B200DataFrame:
        from . import relational as R

        return R.intersect(self, self.to_df(df1), self.to_df(df2), distinct)

    def distinct(self, df: Any) -> B200DataFrame:
        from . import relational as R

        return R.distinct(self, self.to_df(df))

    def dropna(self, df: Any, how: str = "any", thresh: Optional[int] = None,
               subset: Optional[List[str]] = None) -> B200DataFrame:
        from . import relational as R

        return R.dropna(self.to_df(df), how, thresh, subset)

    def fillna(self, df: Any, value: Any, subset: Optional[List[str]] = None) -> B200DataFrame:
        from . import relational as R

        return R.fillna(self.to_df(df), value, subset)

    def sample(self, df: Any, n: Optional[int] = None, frac: Optional[float] = None, replace: bool = False,
               seed: Optional[int] = None) -> B200DataFrame:
        from . import relational as R

        return R.sample(self.to_df(df), n, frac, replace, seed)

    def load_df(self, path: Any, format_hint: Any = None, columns: Any = None, **kwargs: Any) -> B200DataFrame:
        from . import relational as R

        return R.load_df(self, path, format_hint, columns, **kwargs)

    def save_df(self, df: Any, path: str, format_hint: Any = None, mode: str = "overwrite",
                partition_spec: Optional[PartitionSpec] = None, force_single: bool = False, **kwargs: Any) -> None:
        from . import relational as R

        R.save_df(self, df, path, format_hint, mode, **kwargs)

    def take(self, df: Any, n: int, presort: Any, na_position: str = "last",
             partition_spec: Optional[PartitionSpec] = None) -> B200DataFrame:
        """``ExecutionEngine.take`` (execution_engine.py:708-734; native :350-384) on the device."""
        from . import sort as S
        from .partition import parse_presort_exp

        partition_spec = partition_spec or PartitionSpec()
        assert_or_throw(isinstance(n, int) and not isinstance(n, bool), ValueError("n needs to be an integer"))
        sorts = parse_presort_exp(presort) if presort else None
        if not sorts:
            sorts = partition_spec.presort
        edf = self.to_df(df)
        for k in list(sorts.keys()) + list(partition_spec.partition_by):
            assert_or_throw(k in edf.schema, lambda: KeyError(f"{k} not in {edf.schema}"))
        return B200DataFrame(S.take(edf.native, n, sorts, na_position, list(partition_spec.partition_by)))
