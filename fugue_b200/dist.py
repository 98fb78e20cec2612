"""Multi-GPU hash repartition: one process per GPU, rows range-sharded (SURVEY.md 8e).

    pass 1 on the local shard (rank records + per-partition counts)        libfugue_b200.so
 -> counts to every rank through a symmetric-memory control buffer          (no NCCL, no SM-filling kernel)
 -> pass 2 (scatter) column group by column group into this rank's slice of a symmetric ARENA
 -> while group k+1 scatters, the COPY ENGINES pull group k over NVLink / NVSwitch: physical
    partition p is owned by rank p*world//num, so the partitions one rank owns are contiguous in
    every source's partitioned table and the exchange is ONE run per (source rank, column)
 -> the result keeps the received runs in (source rank, partition) order: an owned partition is a
    list of `world` segments (``B200Table.segment_offsets``), rows inside it ordered by (source
    rank, source row) = the stable partition of the concatenated table.  ``B200Table.compacted()``
    makes every partition contiguous with one local segment copy when a consumer needs that.

The reference has no shuffle of its own (Dask: set_index + repartition(divisions),
fugue_dask/_utils.py:124-130, 166-169; Spark: df.repartition, fugue_spark/_utils/partition.py:23);
the contract honoured is SURVEY.md 3.3: equal keys land in the same physical partition.

The planning functions work on CPU tensors with any torch.distributed backend, so the
world-size-2 ``gloo`` tests (tests/test_dist_cpu.py) cover this logic without a GPU.
"""
import os
from typing import Any, Dict, List, Optional, Sequence, Tuple

# The exchange runs ~10 streams at once (scatter, control, one copy-engine stream per peer).  With the
# default of 8 hardware work queues streams alias each other's queue and pick up false dependencies
# (measured: the barrier kernel and the copies waited for scatter kernels of OTHER streams).  Must be
# set before the CUDA context exists; harmless if the application already set it.
os.environ.setdefault("CUDA_DEVICE_MAX_CONNECTIONS", "32")

import numpy as np  # noqa: E402
import pyarrow as pa  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from .column import Kind
from .dataframe import B200DataFrame
from .execution_engine import B200ExecutionEngine, assert_or_throw
from .partition import PartitionSpec
from .table import B200Table


def owner_range(num: int, world: int, rank: int) -> Tuple[int, int]:
    """Physical partitions [lo, hi) owned by ``rank`` (balanced contiguous ranges)."""
    return rank * num // world, (rank + 1) * num // world


class ExchangePlan:
    """Everything derived from the count matrix ``counts[src][p]``."""

    def __init__(self, counts: torch.Tensor, rank: int):
        world, num = counts.shape
        self.world, self.num, self.rank = world, num, rank
        self.counts = counts
        lo, hi = owner_range(num, world, rank)
        self.lo, self.hi = lo, hi
        bounds = [owner_range(num, world, r) for r in range(world)]
        # rows this rank sends to every destination / receives from every source
        self.send_rows = [int(counts[rank, a:b].sum()) for a, b in bounds]
        self.recv_rows = [int(counts[s, lo:hi].sum()) for s in range(world)]
        self.total_recv = sum(self.recv_rows)
        # received layout: [src 0: partitions lo..hi) | src 1: ... ]; wanted: partition-major
        mine = counts[:, lo:hi]                                   # [world, nown]
        recv_base = torch.zeros(world, dtype=torch.int64)
        recv_base[1:] = torch.cumsum(torch.tensor(self.recv_rows[:-1], dtype=torch.int64), 0)
        within = torch.cumsum(mine, 1) - mine                     # offset of p inside src's run
        src_off = recv_base[:, None] + within                     # [world, nown]
        flat_pm = mine.t().contiguous().reshape(-1)               # partition-major lengths
        dst_off = torch.cumsum(flat_pm, 0) - flat_pm
        self.seg_src_off = src_off.t().contiguous().reshape(-1)   # partition-major order
        # pull exchange: the same runs addressed inside every SOURCE rank's partitioned table
        src_part_off = torch.cumsum(counts, 1) - counts            # [world, num] offset of p in src table
        self.pull_src_off = src_part_off[:, lo:hi].t().contiguous().reshape(-1)
        self.pull_src_rank = torch.arange(world, dtype=torch.int32).repeat(hi - lo)
        self.rows_per_rank = counts.sum(1)                        # local row count of every rank
        self.max_seg = int(flat_pm.max()) if flat_pm.numel() > 0 else 0
        self.seg_dst_off = dst_off
        self.seg_len = flat_pm
        part_counts = mine.sum(0)
        self.out_offsets = torch.zeros(hi - lo + 1, dtype=torch.int64)
        self.out_offsets[1:] = torch.cumsum(part_counts, 0)
        # one-run-per-source exchange: source s's rows for this rank are the contiguous range
        # [pull_start[s], pull_start[s] + recv_rows[s]) of its partitioned table and land at
        # recv_base[s]; the received (source, partition) runs are delimited by segment_offsets
        self.recv_base = recv_base
        self.pull_start = src_part_off[:, lo]                      # [world]
        seg = torch.zeros(world, hi - lo + 1, dtype=torch.int64)
        seg[:, 1:] = torch.cumsum(mine, 1)
        self.segment_offsets = seg + recv_base[:, None]            # [world, nown + 1]


def gather_counts(local_counts: torch.Tensor, group: Any = None) -> torch.Tensor:
    """all-gather of the per-partition row counts -> CPU int64 matrix [world, num]."""
    world = dist.get_world_size(group)
    out = torch.empty(world * local_counts.numel(), dtype=torch.int64, device=local_counts.device)
    dist.all_gather_into_tensor(out, local_counts.contiguous(), group=group)
    return out.view(world, -1).cpu()


def exchange_column(col: torch.Tensor, plan: ExchangePlan, group: Any = None) -> torch.Tensor:
    out = torch.empty(plan.total_recv, dtype=col.dtype, device=col.device)
    dist.all_to_all_single(out, col, output_split_sizes=plan.recv_rows, input_split_sizes=plan.send_rows,
                           group=group)
    return out


def rearrange_cpu(recv: Sequence[torch.Tensor], plan: ExchangePlan) -> List[torch.Tensor]:
    """CPU restatement of fb_copy_segments, used by the gloo tests only."""
    outs = [torch.empty_like(c) for c in recv]
    for s, d, n in zip(plan.seg_src_off.tolist(), plan.seg_dst_off.tolist(), plan.seg_len.tolist()):
        for c, o in zip(recv, outs):
            o[d:d + n] = c[s:s + n]
    return outs


def compact_plan(segment_offsets: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]:
    """(source, partition) runs -> partition-contiguous order.  Returns (src_off, dst_off, len) of
    the runs in (partition, source) order and the offsets[nown + 1] of the compacted table."""
    lens = segment_offsets[:, 1:] - segment_offsets[:, :-1]        # [world, nown]
    flat = lens.t().contiguous().reshape(-1)
    dst = torch.cumsum(flat, 0) - flat
    src = segment_offsets[:, :-1].t().contiguous().reshape(-1)
    off = torch.zeros(lens.shape[1] + 1, dtype=torch.int64)
    off[1:] = torch.cumsum(lens.sum(0), 0)
    return src, dst, flat, off


FUGUE_B200_CONF_DIST_GROUP_COLS = "fugue.b200.dist.group_cols"    # payload columns per scatter/exchange group
FUGUE_B200_CONF_DIST_EXCHANGE = "fugue.b200.dist.exchange"        # "dma" (copy engines) | "tma" | "kernel" (SM pulls)
FUGUE_B200_CONF_DIST_DMA_PIECES = "fugue.b200.dist.dma_pieces"    # copy-engine streams per peer
FUGUE_B200_CONF_DIST_SM_RESERVE = "fugue.b200.dist.sm_reserve"    # SMs the persistent scatter leaves free
_BARRIER_TIMEOUT_MS = 120_000   # a rank that died must not hang the others' GPUs forever
_CTL_SLOTS = 1024                                                 # counts per rank and parity (K.MAX_PARTITIONS)


class DistributedB200Engine(B200ExecutionEngine):
    """``B200ExecutionEngine`` whose ``repartition`` shuffles across the GPUs of the process group."""

    def __init__(self, conf: Any = None, group: Any = None, **kwargs: Any):
        super().__init__(conf, **kwargs)
        assert_or_throw(dist.is_initialized(), RuntimeError(
            "DistributedB200Engine needs an initialised torch.distributed process group"))
        self._group = group
        self._world = dist.get_world_size(group)
        self._rank = dist.get_rank(group)
        self._arena: Optional[torch.Tensor] = None
        self._ctl: Optional[torch.Tensor] = None
        self._step = 0
        self._trace: Optional[List[Any]] = None
        # at 2 GPUs scatter and exchange take about as long and groups of 2 interleave them best; from 4 GPUs
        # on the exchange dominates and the copy engines lose more to a running scatter than an earlier start
        # wins, so groups of 4.  These sizes were chosen on another GPU generation and are not measured on H100.
        gc = self._conf.get(FUGUE_B200_CONF_DIST_GROUP_COLS, "2" if self._world == 2 else "4")
        self._group_cols = [max(1, int(x)) for x in str(gc).split(",")]  # columns per group; last repeats
        self._exchange = str(self._conf.get(FUGUE_B200_CONF_DIST_EXCHANGE, "dma"))
        assert_or_throw(self._exchange in ("dma", "kernel", "tma"), ValueError(f"unknown exchange {self._exchange}"))
        # copy-engine streams per peer (pieces every run is cut into): 8 GPUs: 1, 4: 2, 2: 4
        self._dma_pieces = max(1, min(8, int(self._conf.get(FUGUE_B200_CONF_DIST_DMA_PIECES,
                                                            max(1, min(4, 6 // max(1, self._world - 1)))))))
        self._dma_overlap_flag = bool(int(self._conf.get("fugue.b200.dist.dma_overlap_flag", 1)))
        self._sm_reserve = int(self._conf.get(FUGUE_B200_CONF_DIST_SM_RESERVE,
                                              1 if self._exchange == "dma" else 16))

    @property
    def is_distributed(self) -> bool:
        return True

    def get_current_parallelism(self) -> int:
        return self._world

    # ---- symmetric memory: the arena (this rank's partitioned columns, readable by every peer over
    #      NVLink) and a small control buffer for the per-partition counts
    def _ensure_arena(self, nbytes: int) -> None:
        """Collective: all ranks call this with the same ``nbytes`` (derived from the gathered counts)."""
        import torch.distributed._symmetric_memory as symm_mem

        if self._arena is not None and self._arena.numel() >= nbytes:
            return
        cap = ((int(nbytes * 1.25) + (1 << 21) - 1) >> 21) << 21
        self._arena = None  # release the old mapping first
        self._arena = symm_mem.empty(cap, dtype=torch.uint8, device=self._device)
        self._arena_hdl = symm_mem.rendezvous(self._arena, group=self._group or dist.group.WORLD)

    def _ensure_ctl(self) -> None:
        import torch.distributed._symmetric_memory as symm_mem

        if self._ctl is not None:
            return
        dev = self._device
        self._ctl = symm_mem.empty(2 * _CTL_SLOTS, dtype=torch.int64, device=dev)
        self._ctl_hdl = symm_mem.rendezvous(self._ctl, group=self._group or dist.group.WORLD)
        self._ctl_peers = [[self._ctl_hdl.get_buffer(s, (_CTL_SLOTS,), torch.int64, par * _CTL_SLOTS)
                            for s in range(self._world)] for par in range(2)]
        self._counts_dev = torch.empty(self._world, _CTL_SLOTS, dtype=torch.int64, device=dev)
        self._counts_host = torch.empty(self._world, _CTL_SLOTS, dtype=torch.int64, pin_memory=True)
        self._s_ctl = torch.cuda.Stream(dev, priority=-1)  # barrier kernels must not queue behind the scatter
        self._s_dma = [torch.cuda.Stream(dev) for _ in range(1 + (self._world - 1) * 8)]
        self._s_alloc = torch.cuda.Stream(dev)  # allocation-only stream (see _shuffle_table)

    def _post_counts(self, local_counts: torch.Tensor) -> torch.cuda.Event:
        """Stream-ordered all-gather of ``local_counts`` (int64[num], device) over symmetric memory:
        own slot <- counts; barrier; read every peer's slot; copy the matrix to pinned host memory.
        Returns the event after which ``self._counts_host[:, :num]`` is valid.  Two slots used
        alternately: a rank rewrites a slot only after passing the NEXT call's barrier, which every
        peer reaches after its reads of this call."""
        self._ensure_ctl()
        num = int(local_counts.shape[0])
        par = self._step & 1
        self._ctl[par * _CTL_SLOTS:par * _CTL_SLOTS + num].copy_(local_counts)
        self._ctl_hdl.barrier(channel=0, timeout_ms=_BARRIER_TIMEOUT_MS)
        for s in range(self._world):
            self._counts_dev[s, :num].copy_(self._ctl_peers[par][s][:num])
        self._counts_host.copy_(self._counts_dev, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(self._device))
        return ev

    def _mark(self, label: str, stream: Any = None) -> None:
        """Timeline probe (tools/dist_probe.py --trace): a timed event on ``stream`` when tracing is on."""
        if self._trace is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(stream if stream is not None else torch.cuda.current_stream(self._device))
            self._trace.append((label, ev))

    @staticmethod
    def _col_offsets(nrows: int, widths: List[int]) -> List[int]:
        off, out = 0, []
        for w in widths:
            out.append(off)
            off += (nrows * w + 255) & ~255
        out.append(off)
        return out

    def repartition(self, df: Any, partition_spec: PartitionSpec) -> B200DataFrame:
        """Shuffle (module docstring): pass 1 -> counts over symmetric memory -> per column group:
        scatter into the arena, then - overlapping the next group's scatter - one copy-engine pull per
        (source rank, column) over NVLink.  The only host wait is for the count matrix (16 KB), and it
        happens while the first scatter is already running."""
        from . import kernels as K

        keys = partition_spec.partition_by
        edf = self.to_df(df)
        if len(keys) == 0 or self._world == 1:
            return super().repartition(edf, partition_spec)
        t: B200Table = edf.native
        for k in keys:
            assert_or_throw(k in t.schema, lambda: KeyError(f"{k} not in {t.schema}"))
        num = self._num_partitions(partition_spec, t.num_rows)
        assert_or_throw(num <= min(K.MAX_PARTITIONS, _CTL_SLOTS), NotImplementedError(
            f"num_partitions={num}: the multi-GPU exchange handles up to {K.MAX_PARTITIONS} partitions"))
        assert_or_throw(num >= self._world, ValueError(
            f"num_partitions={num} must be >= the number of GPUs ({self._world})"))
        if (t.segment_offsets is not None and t.partition_keys == list(keys)
                and getattr(t, "global_num_partitions", None) == num):
            return edf  # already shuffled this way
        t = self._globalize_dictionaries(t)  # string columns: one code space on all ranks
        res, _ = self._shuffle_table(t, list(keys), num)
        rdf = B200DataFrame(res)
        if edf.has_metadata:
            rdf.reset_metadata(edf.metadata)
        return rdf

    def _shuffle_table(self, t: B200Table, keys: List[str], num: int,
                       col_events: Optional[List[Optional[torch.cuda.Event]]] = None
                       ) -> Tuple[B200Table, List[List[torch.cuda.Event]]]:
        """The exchange itself.  ``col_events[i]`` (optional): event after which column i of ``t`` is on
        the device (host -> device copies still in flight: the pipelined host-to-host transform); pass 1
        waits for the key columns, the scatter of a group for its columns.  Returns the shuffled table and,
        per output column, the events after which that column is complete (its group's pulls), so that a
        device -> host copy of an early column can overlap the exchange of the later ones."""
        from . import kernels as K

        dev = t.device
        world, rank = self._world, self._rank
        kidx = [t.schema.index_of_key(k) for k in keys]
        kvalid = [t.valid[i] for i in kidx]
        cols = list(t.columns)
        vpos: Dict[int, int] = {}
        for i, v in enumerate(t.valid):
            if v is not None:
                vpos[i] = len(cols)
                cols.append(v)
        widths = [c.element_size() for c in cols]
        s_main = torch.cuda.current_stream(dev)
        if col_events is not None:
            col_events = list(col_events) + [None] * (len(cols) - len(col_events))
            for i in kidx:
                if col_events[i] is not None:
                    s_main.wait_event(col_events[i])
        # ---- pass 1 on the local shard; counts to everybody (stream-ordered, host reads them later)
        scratch = self._pool.scratch(dev, K.partition_scratch_bytes(dev, t.num_rows, num))
        self._mark("start")
        plan_local = K.partition_plan([t.columns[i] for i in kidx], num, kvalid, scratch=scratch)
        self._mark("pass1")
        ev_counts = self._post_counts(plan_local.offsets[1:] - plan_local.offsets[:-1])
        self._mark("counts")
        self._step += 1
        # 8-byte columns first (fast kernel), cut into groups (the first group small: the exchange can
        # start as soon as it is scattered); narrow columns (validity masks ...) last
        order = sorted(range(len(cols)), key=lambda i: (widths[i] != 8, i))
        groups: List[List[int]] = []
        a0, gi0 = 0, 0
        while a0 < len(order):
            per = self._group_cols[min(gi0, len(self._group_cols) - 1)]
            groups.append(order[a0:a0 + per])
            a0 += per
            gi0 += 1
        my_off = self._col_offsets(t.num_rows, widths)
        s_ctl = self._s_ctl

        def scatter_all() -> List[torch.cuda.Event]:
            parts = [self._arena[my_off[i]:my_off[i] + t.num_rows * w].view(c.dtype)
                     for i, (c, w) in enumerate(zip(cols, widths))]
            evs = []
            for idx in groups:
                if col_events is not None:
                    for i in idx:
                        if col_events[i] is not None:
                            s_main.wait_event(col_events[i])
                K.partition_apply(plan_local, [cols[i] for i in idx], [parts[i] for i in idx],
                                  sm_reserve=self._sm_reserve)
                ev = torch.cuda.Event()
                ev.record(s_main)
                evs.append(ev)
                self._mark(f"scatter{len(evs) - 1}")
            return evs

        def barriers(ev_sc: Optional[List[torch.cuda.Event]]) -> List[torch.cuda.Event]:
            """Per group, on the control stream: after this rank's scatter of the group, a barrier over
            all ranks ("group k sits in every arena"); the returned events release the pulls."""
            evs = []
            with torch.cuda.stream(s_ctl):
                for gi in range(len(groups)):
                    if ev_sc is not None:
                        s_ctl.wait_event(ev_sc[gi])
                    self._arena_hdl.barrier(channel=1, timeout_ms=_BARRIER_TIMEOUT_MS)
                    ev = torch.cuda.Event()
                    ev.record(s_ctl)
                    evs.append(ev)
                    self._mark(f"barrier{gi}")
            return evs

        # Everything that does not need the counts is enqueued BEFORE the host waits for them: the
        # scatters (if the local shard fits the arena; peers' reads of the previous call are over: every
        # call ends with a barrier) and the per-group barriers.  Ranks must agree on the number of
        # barriers: they are issued whenever an arena exists (a collective property), scattered or not.
        ev_sc: Optional[List[torch.cuda.Event]] = None
        ev_b: Optional[List[torch.cuda.Event]] = None
        if self._arena is not None:
            if self._arena.numel() >= my_off[-1]:
                ev_sc = scatter_all()
            ev_b = barriers(ev_sc)
        ev_counts.synchronize()
        # ---- host plan from the count matrix (numpy, a few microseconds)
        c = self._counts_host.numpy()[:, :num]
        lo, hi = owner_range(num, world, rank)
        mine = c[:, lo:hi]
        rows = c.sum(1)
        recv_rows = mine.sum(1)
        recv_base = np.cumsum(recv_rows) - recv_rows
        pull_start = c[:, :lo].sum(1)
        total_recv = int(recv_rows.sum())
        seg = np.zeros((world, hi - lo + 1), dtype=np.int64)
        np.cumsum(mine, axis=1, out=seg[:, 1:])
        seg += recv_base[:, None]
        need = max(self._col_offsets(int(r), widths)[-1] for r in rows)
        if self._arena is None or self._arena.numel() < need:
            # first call / growth: every rank takes this branch (same matrix, same capacity everywhere)
            torch.cuda.synchronize(dev)
            self._ensure_arena(need)
            ev_sc = scatter_all()
            ev_b = barriers(ev_sc)
        base = [int(x) for x in self._arena_hdl.buffer_ptrs]
        peer_off = [self._col_offsets(int(rows[s]), widths) for s in range(world)]
        # The receive buffers come from the pool of a stream that never runs work: a block in that pool
        # is idle on the device (the allocator returns it only after the events of every stream recorded
        # below have passed), so the pulls may write it at once.  Allocated on the main stream they would
        # have to wait for an event BEHIND the scatters enqueued above - the exchange of group 0 would
        # start when the last scatter is over.
        with torch.cuda.stream(self._s_alloc):
            outs = [torch.empty(total_recv, dtype=cc.dtype, device=dev) for cc in cols]
        optr = [o.data_ptr() for o in outs]
        pieces = self._dma_pieces
        streams = self._s_dma[:1 + (world - 1) * pieces]
        sptr = [st.cuda_stream for st in streams]
        col_done: List[List[torch.cuda.Event]] = [[] for _ in cols]
        for gi, idx in enumerate(groups):
            if self._exchange == "dma":
                # own rows: local copy on stream 0 as soon as this rank's scatter of the group is done;
                # peers: stream j pulls from rank + j (every rank starts on a different source)
                streams[0].wait_event(ev_sc[gi])
                for st in streams[1:]:
                    st.wait_event(ev_b[gi])
                src, dst, nb, stq = [], [], [], []
                for j in range(world):
                    sr = (rank + j) % world
                    if recv_rows[sr] == 0:
                        continue
                    for i in idx:
                        a_src = base[sr] + peer_off[sr][i] + int(pull_start[sr]) * widths[i]
                        a_dst = optr[i] + int(recv_base[sr]) * widths[i]
                        total = int(recv_rows[sr]) * widths[i]
                        if j == 0 or pieces == 1:
                            src.append(a_src), dst.append(a_dst), nb.append(total), stq.append(sptr[j])
                            continue
                        # one copy engine does not saturate the link from one peer: with few peers every run is cut
                        # into `pieces` parts on different streams so that several engines share it
                        step = ((total + pieces - 1) // pieces + 255) & ~255
                        for q in range(pieces):
                            o = q * step
                            if o >= total:
                                break
                            src.append(a_src + o), dst.append(a_dst + o), nb.append(min(step, total - o))
                            stq.append(sptr[1 + (j - 1) * pieces + q])
                if self._trace is not None:
                    self._mark(f"dmaB{gi}.s1", streams[1])
                K.copy_runs_dma_streams(dev, src, dst, nb, stq, self._dma_overlap_flag)
                if self._trace is not None:
                    self._mark(f"dma{gi}.s1", streams[1])
                evs = []
                for st in streams:
                    ev = torch.cuda.Event()
                    ev.record(st)
                    evs.append(ev)
                for i in idx:
                    col_done[i] = evs
                continue
            with torch.cuda.stream(s_ctl):
                s_ctl.wait_event(ev_b[gi])
                if self._exchange == "tma":
                    # persistent TMA pull kernel on the SMs the scatter leaves free; peers first (rotated,
                    # so that not every rank starts on the same source), own rows last
                    order_s = [(rank + j) % world for j in range(1, world)] + [rank]
                    rs = [(base[sr] + peer_off[sr][i] + int(pull_start[sr]) * widths[i],
                           optr[i] + int(recv_base[sr]) * widths[i], int(recv_rows[sr]) * widths[i])
                          for i in idx for sr in order_s if recv_rows[sr] > 0]
                    for a in range(0, len(rs), 64):
                        K.pull_runs_tma(dev, [r[0] for r in rs[a:a + 64]], [r[1] for r in rs[a:a + 64]],
                                        [r[2] for r in rs[a:a + 64]], max(1, self._sm_reserve))
                else:  # "kernel": fb_copy_segments with peer pointers (16-byte loads over NVLink)
                    src_ptrs = [base[sr] + peer_off[sr][i] for sr in range(world) for i in idx]
                    K.copy_segments(None, [outs[i] for i in idx], torch.from_numpy(pull_start).to(dev),
                                    torch.from_numpy(recv_base).to(dev), torch.from_numpy(recv_rows).to(dev),
                                    max_len=int(recv_rows.max()),
                                    src_table=torch.arange(world, dtype=torch.int32, device=dev), src_ptrs=src_ptrs)
                ev = torch.cuda.Event()
                ev.record(s_ctl)
                for i in idx:
                    col_done[i] = [ev]
        if self._trace is not None:
            for j, st in enumerate(streams):
                self._mark(f"dma_done.s{j}", st)
        for st in streams:
            s_ctl.wait_stream(st)
        with torch.cuda.stream(s_ctl):
            # nobody overwrites an arena that is still being read
            self._arena_hdl.barrier(channel=1, timeout_ms=_BARRIER_TIMEOUT_MS)
        s_main.wait_stream(s_ctl)
        self._mark("end")
        for o in outs:
            o.record_stream(s_main)
            for st in streams:
                o.record_stream(st)
            o.record_stream(s_ctl)
        ncol = len(t.columns)
        valid = [outs[vpos[i]] if i in vpos else None for i in range(ncol)]
        res = B200Table(t.schema, outs[:ncol], valid, t.dictionaries, None, list(keys))
        res.segment_offsets = torch.from_numpy(seg)          # [world, nown + 1] (host)
        res.global_partition_range = (lo, hi)               # which physical partitions this GPU owns
        res.global_num_partitions = num
        return res, col_done

    # ---- host table in, host table out: H2D / shuffle / D2H overlapped column by column -----------
    def streaming_transform(self, local_df: Any, runner: Any, out_schema: Any, spec: PartitionSpec) -> Any:
        """``fa.transform(host_table, device_function, hash spec, as_local=True)`` across GPUs with the three
        stages overlapped (the single-GPU counterpart is fugue_b200/streaming.py): every column is copied
        to the device on its own, scattered and exchanged as soon as it has arrived (one column per
        group), and copied back to pinned host memory as soon as its pulls are done - PCIe runs full
        duplex while the GPUs shuffle.  Returns None when the input does not qualify (NULLs, strings,
        presort ...): the caller then takes the step-by-step path."""
        import numpy as np  # noqa: F811
        import pyarrow as pa

        from .dataframe import ArrowDataFrame
        from .streaming import _eligible
        from .table import _from_readonly, _np_storage, _storage_dtype

        table = local_df.as_arrow()
        schema = local_df.schema
        keys = list(spec.partition_by)
        if not _eligible(table, schema, spec) or any(k not in schema for k in keys) or spec.algo in ("even", "rand"):
            return None
        n = table.num_rows
        num = self._num_partitions(spec, n)
        if num > 1024 or num < self._world:
            return None
        dev = self._device
        s_cmp = torch.cuda.current_stream(dev)
        if getattr(self, "_s_h2d", None) is None:
            self._s_h2d, self._s_d2h = torch.cuda.Stream(dev), torch.cuda.Stream(dev)
        s_in, s_out = self._s_h2d, self._s_d2h
        names = schema.names
        order = keys + [c for c in names if c not in keys]
        dcols = {c: torch.empty(n, dtype=_storage_dtype(schema[c].type), device=dev) for c in names}
        ev_in: Dict[str, torch.cuda.Event] = {}
        s_in.wait_stream(s_cmp)
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
        t = B200Table(schema, [dcols[c] for c in names])
        saved = self._group_cols
        self._group_cols = [1]  # ship every column as soon as it is there
        try:
            shuffled, col_done = self._shuffle_table(t, keys, num, [ev_in[c] for c in names])
        finally:
            self._group_cols = saved
        cursor = spec.get_cursor(schema, 0)
        pdf = B200DataFrame(shuffled)
        cursor.set(lambda: pdf.peek_array(), 0, 0)
        res = self.to_df(runner(cursor, pdf))
        if res.schema != out_schema:
            raise AssertionError(f"map output {res.schema} mismatches given {out_schema}")
        rt: B200Table = res.native
        plain = all(not (pa.types.is_boolean(tp) or pa.types.is_string(tp) or pa.types.is_large_string(tp))
                    and col.element_size() * 8 == tp.bit_width for tp, col in zip(out_schema.types, rt.columns))
        if any(v is not None for v in rt.valid) or len(rt.dictionaries) > 0 or not plain:
            return res.as_local()
        ev_f = torch.cuda.Event()
        ev_f.record(s_cmp)
        passthrough = {(c.data_ptr(), c.numel()): i for i, c in enumerate(shuffled.columns)}
        hosts: List[torch.Tensor] = []
        with torch.cuda.stream(s_out):
            for col in rt.columns:
                src = passthrough.get((col.data_ptr(), col.numel()))
                if src is not None and col_done[src]:
                    for ev in col_done[src]:   # this column's pulls are done; later columns still travel
                        s_out.wait_event(ev)
                else:
                    s_out.wait_event(ev_f)
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

    def _globalize_dictionaries(self, t: B200Table) -> B200Table:
        return self._globalize_tables([t])[0]

    def _globalize_tables(self, tables: List[B200Table]) -> List[B200Table]:
        """String columns are dictionary encoded per rank and per table; before rows travel (and
        before codes are hashed as partition keys) every rank re-codes them against ONE union
        dictionary per column name - over all ranks and over all the given tables, so that the two
        sides of a join hash equal strings to equal codes: the dictionaries are gathered on the
        host (small), the union is taken in first-appearance order (identical everywhere), and the
        codes are remapped on the device."""
        names = sorted({k for t in tables for k in t.dictionaries})
        if len(names) == 0:
            return tables
        import pyarrow as pa
        import pyarrow.compute as pc

        local = {k: [x for t in tables if k in t.dictionaries for x in t.dictionaries[k].to_pylist()]
                 for k in names}
        gathered: List[Any] = [None] * self._world
        dist.all_gather_object(gathered, local, group=self._group)
        unions = {k: pc.unique(pa.array([x for g in gathered for x in g.get(k, [])], type=pa.string()))
                  for k in names}
        out = []
        for t in tables:
            cols = list(t.columns)
            dicts: Dict[str, Any] = {}
            for k in t.dictionaries:
                pos = pc.index_in(t.dictionaries[k], value_set=unions[k]).to_numpy(zero_copy_only=False).astype("int32")
                i = t.schema.index_of_key(k)
                if len(pos) > 0:
                    m = torch.from_numpy(pos).to(t.device)
                    cols[i] = m[cols[i].long().clamp_(min=0)].contiguous()
                dicts[k] = unions[k]
            nt = B200Table(t.schema, cols, t.valid, dicts, t.offsets, t.partition_keys)
            nt.segment_offsets = t.segment_offsets
            for a in ("global_partition_range", "global_num_partitions"):
                if hasattr(t, a):
                    setattr(nt, a, getattr(t, a))
            out.append(nt)
        return out

    # ---- distributed relational operators (BASELINE configs 4 and 5) -------------------------
    def _shuffle_partitions(self) -> int:
        from .execution_engine import FUGUE_B200_CONF_DEFAULT_PARTITIONS, FUGUE_B200_DEFAULT_PARTITIONS

        n = int(self._conf.get(FUGUE_B200_CONF_DEFAULT_PARTITIONS, FUGUE_B200_DEFAULT_PARTITIONS))
        return max(n, self._world)

    def aggregate(self, df: Any, partition_spec: Optional[PartitionSpec], agg_cols: List[Any]) -> B200DataFrame:
        """GROUP BY across GPUs: local partial aggregation (K6) -> shuffle of the partials by key
        (pull exchange) -> final aggregation of the partials.  Every group ends up on exactly one
        rank; the result stays sharded.  SUM/COUNT/MIN/MAX decompose directly, AVG as SUM + COUNT."""

        keys = [] if partition_spec is None else list(partition_spec.partition_by)
        if self._world > 1:
            # MIN / MAX of a string column or expression compare dictionary ranks, and every rank has its own
            # dictionary
            t = self.to_df(df).native

            def is_str(a: Any) -> bool:
                if a.kind == Kind.NAMED and a.name in t.dictionaries:
                    return True
                tp = a.infer_type(t.schema)
                return tp is not None and (pa.types.is_string(tp) or pa.types.is_large_string(tp))

            assert_or_throw(not any(a.func in ("MIN", "MAX") and is_str(a.arg) for a in agg_cols if a.kind == Kind.AGG),
                            lambda: NotImplementedError("MIN / MAX of a string column or expression across GPUs: "
                                                        "string dictionaries are per rank"))
        if self._world == 1 or not self._plain_aggs(agg_cols):
            # aggregations of expressions / expressions of aggregations: the base class evaluates the
            # row-wise parts locally and comes back here with plain FUNC(column) aggregations
            return super().aggregate(df, partition_spec, agg_cols)
        from .execution_engine import decompose_aggs, finish_avgs

        partial, final, post = decompose_aggs(agg_cols)
        local = super().aggregate(df, partition_spec, partial)
        if len(keys) == 0:
            # global aggregate: every rank reduces its partial row; gather the W partial rows everywhere
            shuffled = self._allgather_rows(local)
        else:
            shuffled = self.repartition(local, PartitionSpec(by=keys, num=self._shuffle_partitions()))
        res = super().aggregate(shuffled, partition_spec, final)
        return finish_avgs(res, post, keys + [a.output_name for a in agg_cols])

    def _allgather_rows(self, df: B200DataFrame) -> B200DataFrame:
        t: B200Table = df.native
        cols, valid = [], []
        for c, v in zip(t.columns, t.valid):
            out = torch.empty(c.shape[0] * self._world, dtype=c.dtype, device=c.device)
            dist.all_gather_into_tensor(out, c.contiguous(), group=self._group)
            cols.append(out)
            if v is None:
                v = torch.ones(c.shape[0], dtype=torch.uint8, device=c.device)
            vo = torch.empty(c.shape[0] * self._world, dtype=torch.uint8, device=c.device)
            dist.all_gather_into_tensor(vo, v.contiguous(), group=self._group)
            valid.append(vo)
        return B200DataFrame(B200Table(t.schema, cols, valid, t.dictionaries))

    def join(self, df1: Any, df2: Any, how: str, on: Optional[List[str]] = None) -> B200DataFrame:
        """Equi-join across GPUs: co-partition both sides on the join keys with the same hash and the
        same partition -> rank ownership (two pull exchanges), then join locally (K7).  Rows with equal
        keys of both tables are on the same rank; NULL keys are co-located too (they never match, but
        outer joins must still emit them exactly once).  Cross joins are not distributed."""
        from .join import get_join_schemas

        if self._world == 1:
            return super().join(df1, df2, how, on)
        e1, e2 = self.to_df(df1), self.to_df(df2)
        key_schema, _ = get_join_schemas(e1, e2, how, on)
        assert_or_throw(how.lower() != "cross", NotImplementedError("distributed cross join"))
        spec = PartitionSpec(by=key_schema.names, num=self._shuffle_partitions())
        # one code space for string columns of BOTH sides before their codes are hashed
        g1, g2 = self._globalize_tables([e1.native, e2.native])
        return super().join(self.repartition(B200DataFrame(g1), spec), self.repartition(B200DataFrame(g2), spec),
                            how, on)
