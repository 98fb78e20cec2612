"""Every path of the K7 hash join against the exact CPU reference (oracle/join.py).

``kernels.JoinTable`` (16-byte multimap: right / full outer, semi, anti, multi-column keys) and ``kernels.join_fused``
(4-byte slots, output columns written by the kernel: inner / left outer on one 8-byte key) each run one of these:

==================== ================================================================================
``table16``            ``JoinTable(k, v)``: one table
``table16-region``     ``JoinTable(k, v, 256)``: one table region per hash partition
``table16-batched``    ``JoinTable(k, v, 256, offsets)``: regions cleared and built in L2-sized batches
``table16-fallback``   a region overflowed; the table was rebuilt as one region
``fused``              ``join_fused`` without partitions
``fused-region``       ``join_fused(..., build_part_offsets=po)``: region mode, build in batches
``fused-build-probe``  both offsets: build and probe batch by batch, probe of batch b next to build of b + 1
``fused-fallback``     a region overflowed; whole-table build and probe
==================== ================================================================================

A spy on the C entry points (tests/_join_spy.py) asserts the path of every result.  Pairs are compared exactly:
``JoinTable.probe`` must return the reference's (probe row, build row) pairs, probe rows not decreasing along the
output and the build rows of one probe row as a set; ``join_fused`` carries a row-id column on each side, and every
other column must equal the row it came from.  Engine-level tests compare whole output rows of ``engine.join``
with ``oracle.join.join_rows`` as multisets.
"""
import functools
from typing import List, Optional

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

import fugue_b200.join as J  # noqa: E402
from fugue_b200 import api as fa  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200.column import SelectColumns, col  # noqa: E402
from fugue_b200.dataframe import B200DataFrame  # noqa: E402
from fugue_b200.table import B200Table  # noqa: E402
from oracle import join as oj  # noqa: E402

from _join_spy import Launches  # noqa: E402

DEV = "cuda:0"
NPARTS = J.RADIX_JOIN_PARTITIONS
INT64_MIN, INT64_MAX = -(2**63), 2**63 - 1
ODD = np.int64(0x9E3779B97F4A7C15 - (1 << 64))


@pytest.fixture
def launches(monkeypatch):
    return Launches(monkeypatch)


def _dev(a: Optional[np.ndarray]):
    return None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def _np(t) -> np.ndarray:
    return t.cpu().numpy()


def _pids(keys: np.ndarray) -> np.ndarray:
    return _np(K.partition_ids([_dev(keys)], NPARTS)) if len(keys) else np.zeros(0, np.int32)


# ---- data -----------------------------------------------------------------------------------------------
DISTS = ["distinct", "unique-build", "three", "special", "null-build", "null-probe", "nulls-both"]
SHAPES = [(0, 700), (700, 0), (1, 700), (700, 1), (31, 40), (33, 20), (4095, 3000), (4096, 4096), (4097, 5000),
          (100_003, 60_000)]


def _keys(dist: str, rng: np.random.Generator, npr: int, nb: int):
    """(probe keys, probe validity, build keys, build validity); duplicates per key stay small, so the output
    stays within a few times the probe side."""
    pv = bv = None
    if dist in ("distinct", "null-build", "null-probe"):
        ids = rng.permutation(npr + nb).astype(np.int64) * ODD
        pk, bk = ids[:npr].copy(), ids[npr // 2: npr // 2 + nb].copy()
        if dist == "null-build":
            bv = np.zeros(nb, np.uint8)
        elif dist == "null-probe":
            pv = np.zeros(npr, np.uint8)
    elif dist == "unique-build":
        bk = rng.permutation(nb).astype(np.int64) * 7 - 3 if nb else np.zeros(0, np.int64)
        pk = rng.choice(bk, npr) if nb else np.zeros(npr, np.int64)
        pk[rng.random(npr) < 0.2] = -(10**12)            # absent key
    elif dist == "three":
        three = np.array([5, -7, 1 << 40], dtype=np.int64)
        nb = min(nb, 15)                                 # up to five copies of each key
        pk, bk = rng.choice(three, npr), rng.choice(three, nb)
    elif dist == "special":
        spec = np.array([0, -1, INT64_MIN, INT64_MAX], dtype=np.int64)
        bk = rng.permutation(max(nb, 1)).astype(np.int64)[:nb] * ODD
        bk[: min(nb, 12)] = np.tile(spec, 3)[: min(nb, 12)]   # each special up to three times
        pk = np.where(rng.random(npr) < 0.5, rng.choice(spec, npr), rng.choice(bk, npr) if nb else 3)
        pv = (rng.random(npr) > 0.3).astype(np.uint8)
        bv = (rng.random(nb) > 0.3).astype(np.uint8)
    elif dist == "nulls-both":
        pk = rng.integers(0, max(npr, 2) // 2, npr).astype(np.int64) * ODD
        bk = rng.permutation(nb).astype(np.int64) * ODD
        pv = (rng.random(npr) > 0.3).astype(np.uint8)
        bv = (rng.random(nb) > 0.3).astype(np.uint8)
    else:
        raise ValueError(dist)
    return pk.astype(np.int64), pv, bk.astype(np.int64), bv


def _payload(rng: np.random.Generator, n: int, side: str):
    """A row-id column and one column of every width (floats as random bit patterns, NaN payloads included),
    with a validity mask on some."""
    rid = np.arange(n, dtype=np.int64) + (0 if side == "l" else 10**12)
    cols = [rid, rng.integers(0, 256, n).astype(np.uint8), rng.integers(-2**15, 2**15, n).astype(np.int16),
            rng.integers(-2**31, 2**31, n).astype(np.int32).view(np.float32),
            rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64).view(np.float64)]
    masks = [None, (rng.random(n) > 0.2).astype(np.uint8), None, (rng.random(n) > 0.5).astype(np.uint8),
             (rng.random(n) > 0.1).astype(np.uint8)]
    return cols, masks


@functools.lru_cache(maxsize=None)
def dataset(npr: int, nb: int, dist: str, partitioned: bool):
    rng = np.random.default_rng([npr, nb, DISTS.index(dist)])
    pk, pv, bk, bv = _keys(dist, rng, npr, nb)
    lcols, lmasks = _payload(rng, len(pk), "l")
    rcols, rmasks = _payload(rng, len(bk), "r")
    ppo = bpo = None
    if partitioned:   # rows in hash-partition order, as ``partition_columns`` leaves them
        def part(k, v, cols, masks):
            pid = _pids(k)
            perm = np.argsort(pid, kind="stable")
            off = np.concatenate([[0], np.cumsum(np.bincount(pid, minlength=NPARTS))]).astype(np.int64)
            return k[perm], None if v is None else v[perm], _permute(cols, perm), _permute(masks, perm), off
        pk, pv, lcols, lmasks, ppo = part(pk, pv, lcols, lmasks)
        bk, bv, rcols, rmasks, bpo = part(bk, bv, rcols, rmasks)
    return pk, pv, bk, bv, lcols, lmasks, rcols, rmasks, ppo, bpo


def _permute(cols: List[Optional[np.ndarray]], perm: np.ndarray) -> List[Optional[np.ndarray]]:
    """Rows reordered by ``perm``; a row-id column (the first of ``_payload``'s) keeps numbering positions."""
    out = [None if c is None else c[perm] for c in cols]
    if cols[0] is not None:
        out[0] = cols[0]
    return out


def _max_region_load(bk: np.ndarray, bv: Optional[np.ndarray]) -> int:
    k = bk if bv is None else bk[bv.astype(bool)]
    return int(np.bincount(_pids(k), minlength=NPARTS).max()) if len(k) else 0


# ---- checks ---------------------------------------------------------------------------------------------
def assert_pairs(li: np.ndarray, ri: np.ndarray, exp_p: np.ndarray, exp_b: np.ndarray) -> None:
    """Same pairs as the reference; probe rows in output order never decrease (probe-row-major)."""
    assert len(li) == len(exp_p), (len(li), len(exp_p))
    assert np.all(np.diff(li) >= 0), "output is not probe-row major"
    order = np.lexsort((ri, li))
    assert np.array_equal(li[order], exp_p)
    bad = np.flatnonzero(ri[order] != exp_b)
    assert bad.size == 0, (bad[:5], li[order][bad[:5]], ri[order][bad[:5]], exp_b[bad[:5]])


def check_table16(pk, pv, bk, bv, num_parts=0, po=None, outer_modes=(False, True)):
    tab = K.JoinTable(_dev(bk), _dev(bv), num_parts, _dev(po))
    for outer in outer_modes:
        li, ri = tab.probe(_dev(pk), _dev(pv), outer)
        exp_p, exp_b = oj.join_pairs(pk, pv, bk, bv, outer)
        assert_pairs(_np(li), _np(ri), exp_p, exp_b)
        assert np.array_equal(_np(tab.probe_counts(_dev(pk), _dev(pv), outer)), oj.probe_counts(pk, pv, bk, bv, outer))
        if not outer:
            assert np.array_equal(_np(tab.matched_mask(ri)), oj.matched_build_rows(pk, pv, bk, bv))
    torch.cuda.synchronize()


def _bits(a: np.ndarray) -> np.ndarray:
    return a.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def _valid_at(mask: Optional[np.ndarray], rows: np.ndarray):
    """mask[rows] where rows >= 0 (1 without a mask); rows < 0 give 0."""
    if mask is None:
        return (rows >= 0).astype(np.uint8)
    return np.where(rows >= 0, mask[np.maximum(rows, 0)] if len(mask) else 0, 0)


def check_fused(pk, pv, bk, bv, lcols, lmasks, rcols, rmasks, outer_modes=(False, True), **kw):
    # the engine's layout: left columns, then the left validity masks as 1-byte columns
    left = list(lcols) + [m for m in lmasks if m is not None]
    for outer in outer_modes:
        louts, routs, rvout, nout = K.join_fused(_dev(pk), _dev(pv), _dev(bk), _dev(bv), [_dev(c) for c in left],
                                                 [_dev(c) for c in rcols], [_dev(m) for m in rmasks], outer,
                                                 **{k: (_dev(v) if k.endswith("offsets") else v) for k, v in kw.items()})
        louts, routs = [_np(c) for c in louts], [_np(c) for c in routs]
        rvout = [None if v is None else _np(v) for v in rvout]
        exp_p, exp_b = oj.join_pairs(pk, pv, bk, bv, outer)
        assert nout == len(exp_p) == len(louts[0])
        li = louts[0]
        has = np.ones(nout, bool) if rvout[0] is None else rvout[0].astype(bool)
        ri = np.where(has, routs[0] - 10**12, -1)
        assert_pairs(li, ri, exp_p, exp_b)
        for src, out in zip(left, louts):
            assert np.array_equal(_bits(out), _bits(src[li]))
        for src, m, out, vo in zip(rcols, rmasks, routs, rvout):
            assert np.array_equal(_bits(out[has]), _bits(src[ri[has]]))
            if vo is None:
                assert not outer and m is None
                continue
            assert np.array_equal(vo, np.where(has, _valid_at(m, ri), 0))              # NULL-extended rows: validity 0 in every right column
    torch.cuda.synchronize()


# ---- every path, every key distribution, every size ----------------------------------------------------
PATHS = ["table16", "table16-region", "table16-batched", "fused", "fused-region", "fused-build-probe"]


def _run_path(path: str, npr: int, nb: int, dist: str, launches) -> str:
    partitioned = path in ("table16-batched", "fused-region", "fused-build-probe")
    pk, pv, bk, bv, lcols, lmasks, rcols, rmasks, ppo, bpo = dataset(npr, nb, dist, partitioned)
    launches.clear()
    if path.startswith("table16"):
        check_table16(pk, pv, bk, bv, 0 if path == "table16" else NPARTS, bpo)
        family = "table16"
    else:
        kw = {} if path == "fused" else dict(num_parts=NPARTS, build_part_offsets=bpo)
        if path == "fused-build-probe":
            kw["probe_part_offsets"] = ppo
        check_fused(pk, pv, bk, bv, lcols, lmasks, rcols, rmasks, **kw)
        family = "fused"
    got = launches.path(family)
    want = path
    first = [c for c in launches.calls if c.name in ("fb_join_build_u64", "fb_join2_build", "fb_join2_build_probe")][0]
    if path not in ("table16", "fused"):
        if first.parts == 0:   # join_fused uses regions only when every region has at least 4 slots
            assert family == "fused" and first.capacity < 4 * NPARTS, first
            want = "fused"
        elif _max_region_load(bk, bv) > first.capacity // first.parts and not (first.name == "fb_join2_build_probe"
                                                                             and npr == 0):
            want = f"{family}-fallback"
    assert got == want, (got, want, launches.calls)
    if partitioned and got == path:
        assert launches.batches(family) == 1     # these sizes fit one batch; the 4.2 M tests run several
    return got


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{a}x{b}" for a, b in SHAPES])
@pytest.mark.parametrize("path", PATHS)
def test_path_matches_oracle(path, shape, launches):
    seen = {dist: _run_path(path, shape[0], shape[1], dist, launches) for dist in DISTS}
    if shape == (100_003, 60_000):   # with room in every region the requested path holds
        assert seen["distinct"] == seen["unique-build"] == seen["nulls-both"] == path, seen


# ---- duplicates across output windows of pass B ---------------------------------------------------------
@functools.lru_cache(maxsize=None)
def hot_dataset():
    """One build key with 9 000 copies (> 2 windows of 4 096 output slots) among 1.1 M unique keys, all probe
    keys in the hot key's hash partition.  Probe rows 16..23 (owned by one thread of tile 0), 4095 / 4096 (the
    tile edge) and 9000..9003 hold the hot key; row 19 is a NULL in between; the others match once or never."""
    rng = np.random.default_rng(77)
    cand = np.arange(1, 1_200_001, dtype=np.int64) * 1_000_003
    pid = _pids(cand)
    hot = cand[0]
    same = cand[1:][pid[1:] == pid[0]]
    others = cand[1:][pid[1:] != pid[0]]
    bk = np.concatenate([np.full(9000, hot), same[: len(same) // 2], others[:1_100_000 - len(same)]])
    bk = bk[rng.permutation(len(bk))]
    npr = 12_000
    pk = rng.choice(same, npr)                                     # half of them have no build row
    hot_rows = np.array(list(range(16, 24)) + [4095, 4096, 9000, 9001, 9002, 9003])
    pk[hot_rows] = hot
    pv = np.ones(npr, np.uint8)
    pv[19] = 0
    lcols, lmasks = _payload(rng, npr, "l")
    rcols, rmasks = _payload(rng, len(bk), "r")
    return pk, pv, bk, lcols, lmasks, rcols, rmasks, int(pid[0])


@pytest.mark.parametrize("path", ["fused", "table16", "fused-build-probe"])
def test_duplicates_across_output_windows(path, launches):
    pk, pv, bk, lcols, lmasks, rcols, rmasks, hot_part = hot_dataset()
    exp_p, _ = oj.join_pairs(pk, pv, bk, None, False)
    assert np.bincount(exp_p, minlength=len(pk))[[16, 20, 4095, 4096]].tolist() == [9000] * 4
    assert np.bincount(exp_p, minlength=len(pk))[19] == 0
    launches.clear()
    if path == "table16":
        check_table16(pk, pv, bk, None)
    elif path == "fused":
        check_fused(pk, pv, bk, None, lcols, lmasks, rcols, rmasks)
    else:
        pid = _pids(bk)
        perm = np.argsort(pid, kind="stable")
        bpo = np.concatenate([[0], np.cumsum(np.bincount(pid, minlength=NPARTS))]).astype(np.int64)
        ppo = np.zeros(NPARTS + 1, np.int64)
        ppo[hot_part + 1:] = len(pk)                                # every probe row is in the hot partition
        check_fused(pk, pv, bk[perm], None, lcols, lmasks, _permute(rcols, perm), _permute(rmasks, perm), num_parts=NPARTS,
                    build_part_offsets=bpo, probe_part_offsets=ppo)
        assert launches.batches() == 1
    assert launches.path() == path, launches.calls


# ---- 4.2 M rows: several batches, duplicate build keys in the first or the last batch only ---------------
N_BIG = 4_200_000


def _batch_partitions(budget: int, slot: int, nrows: int):
    cap = 1 << (2 * nrows).bit_length()
    per = budget // (cap // NPARTS * slot)
    return [(p, min(p + per, NPARTS)) for p in range(0, NPARTS, per)]


@functools.lru_cache(maxsize=None)
def big_dataset(dup_batch: str):
    """4.2 M unique build keys, then 20 k rows of the partitions of one batch of the build-probe path copy the key
    of the row before them in the same partition; 4.2 M probe rows, 10 % absent keys, 5 % NULL."""
    rng = np.random.default_rng(42 if dup_batch == "first" else 43)
    bk = rng.permutation(N_BIG).astype(np.int64) * ODD
    pid = _pids(bk)
    batches = _batch_partitions(24 << 20, 4, N_BIG)
    assert len(batches) == 3
    p0, p1 = batches[0] if dup_batch == "first" else batches[-1]
    rows = np.flatnonzero((pid >= p0) & (pid < p1))
    rows = rows[np.argsort(pid[rows], kind="stable")]
    q = np.flatnonzero(pid[rows[1:]] == pid[rows[:-1]])[::40][:20_000] + 1
    bk[rows[q]] = bk[rows[q - 1]]
    dup = np.unique(bk, return_counts=True)[1] > 1
    assert dup.sum() > 10_000
    pk = rng.choice(bk, N_BIG)
    pk[rng.random(N_BIG) < 0.1] = 12345                             # (almost surely) absent
    pv = (rng.random(N_BIG) > 0.05).astype(np.uint8)
    ppid, bpid = _pids(pk), pid
    pperm, bperm = np.argsort(ppid, kind="stable"), np.argsort(bpid, kind="stable")
    ppo = np.concatenate([[0], np.cumsum(np.bincount(ppid, minlength=NPARTS))]).astype(np.int64)
    bpo = np.concatenate([[0], np.cumsum(np.bincount(bpid, minlength=NPARTS))]).astype(np.int64)
    pk, pv, bk = pk[pperm], pv[pperm], bk[bperm]
    # duplicates only in the chosen batch
    dup_keys = np.unique(bk)[np.unique(bk, return_counts=True)[1] > 1]
    dpid = _pids(dup_keys)
    assert dpid.min() >= p0 and dpid.max() < p1
    lcols = [np.arange(N_BIG, dtype=np.int64), rng.integers(0, 256, N_BIG).astype(np.uint8)]
    rcols = [np.arange(N_BIG, dtype=np.int64) + 10**12, rng.integers(-2**31, 2**31, N_BIG).astype(np.int32)]
    rmasks = [None, (rng.random(N_BIG) > 0.2).astype(np.uint8)]
    return pk, pv, bk, ppo, bpo, lcols, rcols, rmasks


@pytest.mark.parametrize("dup_batch", ["last", "first"])
def test_duplicates_in_one_batch_only(dup_batch, launches):
    pk, pv, bk, ppo, bpo, lcols, rcols, rmasks = big_dataset(dup_batch)
    launches.clear()
    check_fused(pk, pv, bk, None, lcols, [None, None], rcols, rmasks, outer_modes=(False,), num_parts=NPARTS,
                build_part_offsets=bpo, probe_part_offsets=ppo)
    assert (launches.path(), launches.batches()) == ("fused-build-probe", 3), launches.calls
    if dup_batch == "last":
        launches.clear()
        check_fused(pk, pv, bk, None, lcols, [None, None], rcols, rmasks, outer_modes=(True,), num_parts=NPARTS,
                    build_part_offsets=bpo)
        assert (launches.path(), launches.batches()) == ("fused-region", 2), launches.calls
    else:
        launches.clear()
        check_table16(pk, pv, bk, None, NPARTS, bpo, outer_modes=(False,))
        assert (launches.path(), launches.batches()) == ("table16-batched", 4), launches.calls


def test_build_probe_batch_counts_follow_the_budget(launches):
    """1 batch up to 2 M build rows, 2 at 2.2 M, 3 at 4.2 M (24 MiB of 4-byte slots per batch)."""
    rng = np.random.default_rng(3)
    for nb, want in ((2_000_000, 1), (2_200_000, 2)):
        bk = rng.permutation(nb).astype(np.int64) * ODD
        pk = bk[rng.integers(0, nb, 5000)]
        pid, ppid = _pids(bk), _pids(pk)
        bperm, pperm = np.argsort(pid, kind="stable"), np.argsort(ppid, kind="stable")
        bpo = np.concatenate([[0], np.cumsum(np.bincount(pid, minlength=NPARTS))]).astype(np.int64)
        ppo = np.concatenate([[0], np.cumsum(np.bincount(ppid, minlength=NPARTS))]).astype(np.int64)
        launches.clear()
        check_fused(pk[pperm], None, bk[bperm], None, [np.arange(5000, dtype=np.int64)], [None],
                    [np.arange(nb, dtype=np.int64) + 10**12], [None], outer_modes=(False,), num_parts=NPARTS,
                    build_part_offsets=bpo, probe_part_offsets=ppo)
        assert (launches.path(), launches.batches()) == ("fused-build-probe", want)
    assert len(_batch_partitions(24 << 20, 4, N_BIG)) == 3


# ---- scan, compaction, gather ---------------------------------------------------------------------------
SCAN_SIZES = [0, 1, 4095, 4096, 4097, 512 * 4096 + 1]


@pytest.mark.parametrize("n", SCAN_SIZES)
def test_exclusive_scan(n):
    rng = np.random.default_rng(n)
    c = rng.integers(0, 1 << 20, n).astype(np.int64)
    c[rng.random(n) < 0.3] = 0
    out, total = K.exclusive_scan(_dev(c))
    assert np.array_equal(_np(out), np.cumsum(c) - c) and total == int(c.sum())


@pytest.mark.parametrize("n", SCAN_SIZES)
def test_compact_indices(n):
    rng = np.random.default_rng(n + 1)
    for p in (0.0, 0.3, 1.0):
        m = (rng.random(n) < p).astype(np.uint8) * rng.integers(1, 256, n).astype(np.uint8)
        assert np.array_equal(_np(K.compact_indices(_dev(m))), np.flatnonzero(m))
        assert np.array_equal(_np(K.compact_indices(_dev(m.astype(bool)))), np.flatnonzero(m))


@pytest.mark.parametrize("n", [1, 4097, 100_003])
def test_gather_rows_every_width(n):
    rng = np.random.default_rng(n + 2)
    src_n = 5000
    cols, masks = _payload(rng, src_n, "r")
    idx = rng.integers(-1, src_n, n).astype(np.int64)
    idx[: min(n, 3)] = -1
    for want_valid in (False, True):
        use = idx if want_valid else np.abs(idx)
        outs, outv = K.gather_rows([_dev(c) for c in cols], [_dev(m) for m in masks], _dev(use), want_valid)
        has = use >= 0
        for c, m, o, v in zip(cols, masks, outs, outv):
            o = _np(o)
            assert np.array_equal(_bits(o[has]), _bits(c[use[has]])) and not _bits(o[~has]).any()
            if v is None:
                assert m is None and not want_valid
                continue
            assert np.array_equal(_np(v), np.where(has, _valid_at(m, use), 0))


# ---- engine level ---------------------------------------------------------------------------------------
HOWS = ["inner", "left_outer", "right_outer", "full_outer", "semi", "anti"]
KEY_KINDS = ["int8", "int16", "int32", "int64", "bool", "float32", "float64", "string", "date", "timestamp", "two"]


def _key_array(kind: str, rng: np.random.Generator, n: int, side: str) -> pa.Array:
    null = rng.random(n) < (0.97 if kind == "bool" else 0.1)
    if kind == "int8":
        return pa.array(rng.integers(-128, 128, n).astype(np.int8), mask=null)
    if kind in ("int16", "int32"):
        pool = rng.integers(-30_000, 30_000, 600)
        return pa.array(rng.choice(pool, n).astype(kind), mask=null)
    if kind == "int64":
        pool = np.concatenate([[0, -1, INT64_MIN, INT64_MAX, INT64_MAX - 1], rng.integers(INT64_MIN, INT64_MAX, 595)])
        return pa.array(rng.choice(pool, n), mask=null)
    if kind == "bool":
        return pa.array(rng.random(n) < 0.5, mask=null)
    if kind in ("float32", "float64"):
        pool = np.concatenate([[0.0, -0.0, np.inf, -np.inf, 5e-324 if kind == "float64" else 1e-45, -3.5],
                               np.round(rng.standard_normal(594), 2)]).astype(kind)
        return pa.array(rng.choice(pool, n), mask=null)
    if kind == "string":   # the right side holds strings the left does not, first seen in another order
        pool = [f"s{i}" for i in (range(0, 300) if side == "l" else range(500, 150, -1))]
        return pa.array(rng.choice(np.array(pool), n).tolist(), mask=null)
    if kind == "date":
        return pa.array(rng.integers(-2000, 2000, n).astype(np.int32), mask=null).cast(pa.date32())
    if kind == "timestamp":
        pool = rng.integers(-(10**15), 10**15, 600)
        return pa.array(rng.choice(pool, n), mask=null).cast(pa.timestamp("us"))
    raise ValueError(kind)


def _engine_tables(kind: str, seed: int, n1: int = 1500, n2: int = 1200):
    rng = np.random.default_rng([seed, KEY_KINDS.index(kind)])
    lk: dict = {}
    rk: dict = {}
    if kind == "two":   # multi-column key: 64-bit hash surrogate + verification
        for d, n, side in ((lk, n1, "l"), (rk, n2, "r")):
            f = np.array([0.0, -0.0, 1.5, -2.0, np.inf])[rng.integers(0, 5, n)]
            d["kf"] = pa.array(f, mask=rng.random(n) < 0.05)
            d["ks"] = _key_array("string", rng, n, side)
            d["ks"] = pa.array([None if v is None else v[:2] for v in d["ks"].to_pylist()])   # ~40 values
    else:
        lk["k"], rk["k"] = _key_array(kind, rng, n1, "l"), _key_array(kind, rng, n2, "r")
    left = pa.table({**lk, "lrow": pa.array(np.arange(n1)), "lv": pa.array(rng.standard_normal(n1), mask=rng.random(n1) < 0.1)})
    right = pa.table({"rs": pa.array(rng.choice(np.array(["x", "yy", "zzz"]), n2).tolist(), mask=rng.random(n2) < 0.1),
                      **rk, "rrow": pa.array(np.arange(n2)), "r8": pa.array(rng.integers(-128, 128, n2).astype(np.int8),
                                                                             mask=rng.random(n2) < 0.2)})
    return left, right, list(lk)


def _edf(tbl: pa.Table, shuffled: bool = False) -> B200DataFrame:
    t = B200Table.from_arrow(tbl)
    if shuffled:
        t.global_num_partitions = 8   # as the multi-GPU shuffle leaves it: keys are re-coded by scramble64
    return B200DataFrame(t)


def _check_engine_join(e, left: pa.Table, right: pa.Table, how: str, on: List[str], shuffled: bool = False,
                       ldf: Optional[B200DataFrame] = None, rdf: Optional[B200DataFrame] = None):
    """engine.join of ``left`` and ``right`` (or of ``ldf`` / ``rdf``, which hold the same rows) against the
    reference: output schema and rows."""
    got = e.join(_edf(left, shuffled) if ldf is None else ldf, _edf(right, shuffled) if rdf is None else rdf, how,
                 on).native.to_arrow()
    names = oj.output_names(left, right, how, on)
    schema = {**{f.name: f.type for f in right.schema}, **{f.name: f.type for f in left.schema}}
    assert [(f.name, f.type) for f in got.schema] == [(n, schema[n]) for n in names], got.schema
    exp = oj.join_rows(left, right, how, on)
    res = oj.rows_of(got)
    assert res == exp, (how, sum(res.values()), sum(exp.values()), list((res - exp).items())[:3],
                        list((exp - res).items())[:3])


@pytest.fixture(scope="module")
def e():
    return fa.make_execution_engine("b200")


@pytest.mark.parametrize("radix", [False, True], ids=["default", "radix1000"])
@pytest.mark.parametrize("kind", KEY_KINDS)
def test_engine_join_types_and_key_types(e, kind, radix, monkeypatch, launches):
    if radix:
        monkeypatch.setattr(J, "RADIX_JOIN_MIN_ROWS", 1000)
    left, right, on = _engine_tables(kind, 1)
    for how in HOWS:
        launches.clear()
        _check_engine_join(e, left, right, how, on)
        first = [c for c in launches.calls if c.name in ("fb_join_build_u64", "fb_join2_build", "fb_join2_build_probe")][0]
        assert first.parts == (NPARTS if radix else 0), launches.calls
        fused = how in ("inner", "left_outer") and on != ["kf", "ks"]
        assert (first.name != "fb_join_build_u64") == fused, launches.calls


@pytest.mark.parametrize("radix", [False, True], ids=["default", "radix1000"])
def test_engine_shuffled_input(e, radix, monkeypatch, launches):
    """Inputs of a multi-GPU shuffle (``global_num_partitions`` set): the join hashes ``scramble64`` of the keys."""
    if radix:
        monkeypatch.setattr(J, "RADIX_JOIN_MIN_ROWS", 1000)
    for kind in ("int64", "two"):
        left, right, on = _engine_tables(kind, 2)
        for how in HOWS:
            _check_engine_join(e, left, right, how, on, shuffled=True)


def test_engine_cross_join(e):
    left, right, _ = _engine_tables("int32", 3, 40, 30)
    _check_engine_join(e, left.drop(["k"]), right.drop(["k"]), "cross", [])


def test_engine_forced_hash_collisions(e, monkeypatch):
    """Two-column keys join on a 64-bit hash; with the hash cut to 3 bits almost every candidate is a false one:
    ``_verify`` drops them, ``_drop_collisions`` keeps one NULL-extended row for outer probe rows whose only
    candidates are false, and the full outer join marks matched rows through ``_matched_mask``."""
    real = K.row_hash64
    monkeypatch.setattr(K, "row_hash64", lambda cols, valid=None: real(cols, valid) & 7)
    rng = np.random.default_rng(4)

    def side(n: int, strings: List[str], tag: str) -> pa.Table:
        # 5 x 8 key pairs per side, 5 x 4 of them on both sides: every row has candidates, many only false ones
        f = np.array([0.0, -0.0, 1.5, -2.0, np.inf])[rng.integers(0, 5, n)]
        return pa.table({"kf": pa.array(f, mask=rng.random(n) < 0.05),
                         "ks": pa.array(rng.choice(np.array(strings), n).tolist(), mask=rng.random(n) < 0.05),
                         tag: pa.array(np.arange(n))})

    left, right = side(1000, list("abcdefgh"), "lrow"), side(800, list("lkjihgfe"), "rrow")
    for how in HOWS:
        _check_engine_join(e, left, right, how, ["kf", "ks"])


NAN_BITS = [0x7FF8000000000000, 0xFFF8000000000000 - (1 << 64), 0x7FF8000000000123]


def _nan_tables(rng, n: int):
    f = np.round(rng.standard_normal(n), 1)
    bits = f.view(np.int64)
    sel = rng.random(n) < 0.3
    bits[sel] = np.array(NAN_BITS, np.int64)[rng.integers(0, 3, int(sel.sum()))]
    f32 = f.astype(np.float32)
    f32[sel] = np.float32("nan")
    f32.view(np.int32)[sel & (rng.random(n) < 0.5)] = np.int32(-4194304)   # -NaN
    return pa.table({"k": pa.array(f), "k32": pa.array(f32), "k2": pa.array(rng.integers(0, 2, n)),
                     "v": pa.array(np.arange(n))})


def test_engine_nan_keys_never_match(e):
    """A valid NaN key (quiet, negative, with a payload) matches nothing, on one-column and two-column keys,
    as in the reference, where NaN is NULL."""
    rng = np.random.default_rng(5)
    left = _nan_tables(rng, 400)
    right = _nan_tables(rng, 300).rename_columns(["k", "k32", "k2", "w"])
    for on in (["k"], ["k32"], ["k", "k2"]):
        l_ = left.select(on + ["v"])
        r_ = right.select(on + ["w"])
        for how in HOWS:
            _check_engine_join(e, l_, r_, how, on)
            if how in ("semi", "inner"):
                got = e.join(_edf(l_), _edf(r_), how, on).native.to_arrow()
                assert not any(isinstance(x, float) and x != x for x in got.column(on[0]).to_pylist())


def test_engine_nan_key_from_a_select(e):
    """``0.0 / 0.0`` in a select yields a valid NaN; as a join key it matches nothing."""
    src = pa.table({"a": pa.array([0.0, 1.0, 0.0, 4.0]), "b": pa.array([0.0, 2.0, 0.0, 8.0]), "v": pa.array([1, 2, 3, 4])})
    sdf = e.select(_edf(src), SelectColumns((col("a") / col("b")).alias("k"), col("v")))
    sel = sdf.native.to_arrow()
    ks = sel.column("k").to_pylist()
    assert ks[0] != ks[0] and ks[2] != ks[2] and sel.column("k").null_count == 0
    # the right side holds the very NaN bit pattern the division produced
    right = pa.table({"k": pa.array([ks[0], 0.5, ks[2]]), "w": pa.array([10, 20, 30])})
    sdf2 = e.select(_edf(src), SelectColumns((col("a") / col("b")).alias("k"), col("v").alias("w")))
    for how in HOWS:
        _check_engine_join(e, sel, right, how, ["k"], ldf=sdf)
        _check_engine_join(e, right.rename_columns(["k", "v"]), sel.rename_columns(["k", "w"]), how, ["k"], rdf=sdf2)


def test_engine_join_column_limit(e, launches):
    """The fused kernels take 48 left columns (validity masks included); the 49th sends the join to the
    16-byte table."""
    rng = np.random.default_rng(6)
    n1, n2 = 500, 400
    right = pa.table({"k": pa.array(rng.integers(0, 300, n2)), "r": pa.array(np.arange(n2))})
    base = {"k": pa.array(rng.integers(0, 300, n1), mask=rng.random(n1) < 0.1)}   # key + its mask: 2 columns
    for extra, path in ((46, "fused"), (47, "table16")):
        widths = [np.int8, np.int16, np.int32, np.int64]
        cols = {f"c{i}": pa.array(rng.integers(-100, 100, n1).astype(widths[i % 4])) for i in range(extra)}
        left = pa.table({**base, **cols})
        for how in ("inner", "left_outer"):
            launches.clear()
            _check_engine_join(e, left, right, how, ["k"])
            assert launches.path() == path, launches.calls


# ---- full size, default thresholds ------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def full_size_tables():
    """4.2 M x 4.2 M, unique build side; 10 % of the probe keys have no match and 2 % are NULL.  The left keys
    spread over every region too: right / full outer joins build on them."""
    rng = np.random.default_rng(8)
    n = N_BIG
    rk = rng.permutation(n).astype(np.int64) * 3 + 1
    lk = rk[rng.integers(0, n, n)]
    absent = rng.random(n) < 0.1
    lk[absent] = np.arange(int(absent.sum())) * 3                   # distinct keys no right row holds
    lv = (rng.random(n) > 0.02).astype(np.uint8)
    left = B200Table("key:long,lrow:long", [_dev(lk), torch.arange(n, device=DEV)],
                     [_dev(lv), None])
    right = B200Table("key:long,rrow:long", [_dev(rk), torch.arange(n, device=DEV)])
    return lk, lv, rk, left, right


def test_full_size_inner_join_build_probe(e, launches):
    lk, lv, rk, left, right = full_size_tables()
    res = e.join(B200DataFrame(left), B200DataFrame(right), "inner", ["key"]).native
    assert (launches.path(), launches.batches()) == ("fused-build-probe", 3), launches.calls
    exp_p, exp_b = oj.join_pairs(lk, lv, rk, None, False)
    li, ri = _np(res.column("lrow")), _np(res.column("rrow"))
    order = np.lexsort((ri, li))
    assert np.array_equal(li[order], exp_p) and np.array_equal(ri[order], exp_b)
    assert np.array_equal(_np(res.column("key"))[order], lk[exp_p])


@pytest.mark.parametrize("how", ["right_outer", "full_outer", "semi", "anti"])
def test_full_size_table16_batched(e, how, launches):
    lk, lv, rk, left, right = full_size_tables()
    res = e.join(B200DataFrame(left), B200DataFrame(right), how, ["key"]).native
    assert (launches.path("table16"), launches.batches("table16")) == ("table16-batched", 4), launches.calls
    li = _np(res.column("lrow"))
    if how in ("semi", "anti"):
        hit = oj.probe_counts(lk, lv, rk, None, False) > 0
        assert np.array_equal(np.sort(li), np.flatnonzero(hit if how == "semi" else ~hit))
        return
    lvalid = res.valid[res.schema.index_of_key("lrow")]
    lvalid = np.ones(len(li), bool) if lvalid is None else _np(lvalid).astype(bool)
    li = np.where(lvalid, li, -1)
    ri = _np(res.column("rrow"))
    rvalid = res.valid[res.schema.index_of_key("rrow")]
    ri = np.where(_np(rvalid).astype(bool), ri, -1) if rvalid is not None else ri
    if how == "right_outer":
        exp_r, exp_l = oj.join_pairs(rk, None, lk, lv, True)
    else:
        exp_l, exp_r = oj.join_pairs(lk, lv, rk, None, True)
        extra = np.flatnonzero(oj.matched_build_rows(lk, lv, rk, None) == 0)
        exp_l, exp_r = np.concatenate([exp_l, np.full(len(extra), -1)]), np.concatenate([exp_r, extra])
    order, eo = np.lexsort((li, ri)), np.lexsort((exp_l, exp_r))
    assert np.array_equal(ri[order], exp_r[eo]) and np.array_equal(li[order], exp_l[eo])
    keys = _np(res.column("key"))[order]
    assert np.array_equal(keys, np.where(exp_l[eo] >= 0, lk[np.maximum(exp_l[eo], 0)], rk[np.maximum(exp_r[eo], 0)]))
