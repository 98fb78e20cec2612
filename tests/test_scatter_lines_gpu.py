"""The fast scatter kernel's write combining with 16-row (128-byte, one L2 line) groups, against the oracle.

Every partition keeps its last rows of a tile that do not fill a 16-row group in shared memory and writes them
with the next tile's rows, so only whole aligned groups are stored until the end of a chunk.  The cases here are
the ones a larger group can break: partitions that get 0, 1, 15, 16 or 17 rows in a tile, long runs of tiles in
which a partition gets nothing, partition and chunk starts at every offset mod 16, a partition holding every row,
skewed keys, few and many partitions, row counts around whole tiles, and every column-group shape (2 columns per
group, which use 16-row groups, and 1 column per group, which uses 4-row groups; the fused map; SMs held back).
Every output must be byte-identical to ``oracle/hash_partition.py``.
"""
import numpy as np
import pytest

from oracle import hash_partition as hp

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

TILE = 4096  # rows per tile of the scatter kernel
G = 16       # rows per write-combined group
_pools = {}


def _dev():
    return torch.device("cuda", 0)


def _sm_count() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _to_dev(a: np.ndarray):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _keys_for(pids: np.ndarray, num: int, rng) -> np.ndarray:
    """int64 keys whose partition (oracle hash % num) is pids[i]."""
    if num not in _pools:
        cand = np.arange(0, 200 * num + 20_000, dtype="int64")
        pid = hp.partition_ids([cand], num)
        _pools[num] = [cand[pid == p] for p in range(num)]
    keys = np.empty(len(pids), dtype="int64")
    for p in np.unique(pids):
        at = np.flatnonzero(pids == p)
        keys[at] = rng.choice(_pools[num][p], len(at))
    return keys


def _crafted_pids(ntiles: int, extra: int, num: int, seed: int) -> np.ndarray:
    """Partition ids tile by tile: the first tile gives every partition 0..15 rows (so partition starts fall on
    every offset mod 16); then partition p gets 0, 1, G - 1, G or G + 1 rows in turn, a block of 32 partitions gets
    nothing for 25 tiles out of every 50, and the last partition takes the rest of the tile.  `extra` random rows
    follow the whole tiles."""
    rng = np.random.default_rng(seed)
    special = np.array([0, 1, G - 1, G, G + 1])
    quiet = slice(num // 2, num // 2 + 32)
    out = []
    for t in range(ntiles):
        counts = np.zeros(num, dtype="int64")
        if t == 0:
            counts[:-1] = rng.integers(0, G, num - 1)
        else:
            counts[:-1] = special[(np.arange(num - 1) + t) % len(special)]
            if (t // 25) % 2 == 1:
                counts[quiet] = 0
        counts[-1] = TILE - counts.sum()
        tile = np.repeat(np.arange(num), counts)
        rng.shuffle(tile)
        out.append(tile)
    out.append(rng.integers(0, num, extra))
    return np.concatenate(out).astype("int64")


def _payload(n: int, ncols: int, seed: int):
    rng = np.random.default_rng(seed + 1)
    return [rng.integers(-(2**63), 2**63 - 1, n, dtype="int64", endpoint=True) for _ in range(ncols)]


def _chunk_starts(pids: np.ndarray, num: int, offsets: np.ndarray) -> np.ndarray:
    """Output row where each full chunk's rows of each partition start (the chunk geometry of the kernel)."""
    ntiles = len(pids) // TILE
    per = -(-ntiles // (2 * _sm_count()))
    starts = []
    seen = np.zeros(num, dtype="int64")
    for t0 in range(0, ntiles, per):
        starts.append(offsets[:-1] + seen)
        seen += np.bincount(pids[t0 * TILE:min(t0 + per, ntiles) * TILE], minlength=num)
    return np.concatenate(starts)


def _check(keys, cols, num, sm_reserve=0, cols_per_launch=0):
    from fugue_b200 import kernels as K

    plan = K.partition_plan([_to_dev(keys)], num)
    out = K.partition_apply(plan, [_to_dev(c) for c in cols], sm_reserve=sm_reserve, cols_per_launch=cols_per_launch)
    torch.cuda.synchronize()
    order, offsets = hp.stable_partition(hp.partition_ids([keys], num), num)
    assert np.array_equal(plan.offsets.cpu().numpy(), offsets)
    for i, (c, o) in enumerate(zip(cols, out)):
        assert np.array_equal(o.cpu().numpy().view("u1"), np.ascontiguousarray(c[order]).view("u1")), \
            f"column {i} differs"
    return offsets


@pytest.mark.parametrize("cols_per_launch", [1, 2])
@pytest.mark.parametrize("ntiles,extra", [(300, 0), (300, 1), (61, 4095)])
def test_crafted_tile_counts(ntiles, extra, cols_per_launch):
    num = 256
    pids = _crafted_pids(ntiles, extra, num, seed=ntiles + extra)
    rng = np.random.default_rng(ntiles)
    keys = _keys_for(pids, num, rng)
    assert np.array_equal(hp.partition_ids([keys], num), pids)
    offsets = _check(keys, [keys] + _payload(len(keys), 3, ntiles), num, cols_per_launch=cols_per_launch)
    assert len(np.unique(offsets[:-1] % G)) == G, "partition starts do not cover every offset mod 16"
    assert len(np.unique(_chunk_starts(pids, num, offsets) % G)) == G, "chunk starts do not cover every offset mod 16"


@pytest.mark.parametrize("cols_per_launch", [1, 2])
@pytest.mark.parametrize("ncols", range(1, 9))
def test_column_counts(ncols, cols_per_launch):
    n = 150 * TILE + 17
    pids = _crafted_pids(150, 17, 256, seed=ncols)
    keys = _keys_for(pids, 256, np.random.default_rng(ncols))
    _check(keys, _payload(n, ncols, ncols), 256, cols_per_launch=cols_per_launch)


@pytest.mark.parametrize("num", [1, 2, 3, 255, 256])
@pytest.mark.parametrize("n", [1000, TILE, 64 * TILE, 64 * TILE + 1, 300 * TILE + 1])
def test_row_counts_and_partition_counts(n, num):
    rng = np.random.default_rng(n + num)
    keys = rng.integers(0, 1 << 16, n).astype("int64")
    _check(keys, [keys] + _payload(n, 2, n), num)


@pytest.mark.parametrize("cols_per_launch", [1, 2])
@pytest.mark.parametrize("num", [3, 256])
def test_one_partition_takes_every_row(num, cols_per_launch):
    n = 200 * TILE + 5
    keys = np.full(n, 12345, dtype="int64")
    _check(keys, [keys] + _payload(n, 3, num), num, cols_per_launch=cols_per_launch)


@pytest.mark.parametrize("cols_per_launch", [1, 2])
@pytest.mark.parametrize("num", [2, 255, 256])
def test_zipf_keys(num, cols_per_launch):
    n = 400 * TILE + 3
    rng = np.random.default_rng(num)
    keys = np.minimum(rng.zipf(1.2, n), 1 << 30).astype("int64")
    _check(keys, [keys] + _payload(n, 3, num), num, cols_per_launch=cols_per_launch)


@pytest.mark.parametrize("cols_per_launch", [1, 2])
@pytest.mark.parametrize("reserve", ["32", "fallback"])
def test_sm_reserve(reserve, cols_per_launch):
    ncols = 8
    sm = {"32": 32, "fallback": _sm_count() - ncols // cols_per_launch + 1}[reserve]
    pids = _crafted_pids(300, 9, 256, seed=5)
    keys = _keys_for(pids, 256, np.random.default_rng(5))
    _check(keys, _payload(len(keys), ncols, 5), 256, sm_reserve=sm, cols_per_launch=cols_per_launch)


@pytest.mark.parametrize("reserve", [0, 32])
@pytest.mark.parametrize("extra", [0, 1234])
def test_fused_map(extra, reserve):
    from fugue_b200 import kernels as K

    pids = _crafted_pids(200, extra, 256, seed=extra)
    keys = _keys_for(pids, 256, np.random.default_rng(extra))
    n = len(keys)
    rng = np.random.default_rng(extra + 1)
    f = [rng.standard_normal(n) for _ in range(2)]
    i = [rng.integers(-(2**62), 2**62, n).astype("int64") for _ in range(2)]
    dk, df, di = _to_dev(keys), [_to_dev(x) for x in f], [_to_dev(x) for x in i]
    bits = lambda x: int(np.array([x], dtype="float64").view("i8")[0])  # noqa: E731
    units = [
        (dk, None, K.MAP_COPY, 0, 0, 0),
        (df[0], df[1], K.MAP_AFFINE_F64, bits(2.0), bits(-0.5), bits(1.25)),
        (di[0], di[1], K.MAP_AFFINE_I64, 3, -7, 11),
    ]
    plan = K.partition_plan([dk], 256)
    out = K.partition_apply_map(plan, units, sm_reserve=reserve)
    torch.cuda.synchronize()
    order, _ = hp.stable_partition(pids, 256)
    u = lambda x: x[order].view("u8")  # noqa: E731
    with np.errstate(over="ignore"):
        exp = [keys[order], (2.0 * f[0][order] + -0.5 * f[1][order]) + 1.25,
               (np.uint64(3) * u(i[0]) + np.uint64(2**64 - 7) * u(i[1]) + np.uint64(11)).view("i8")]
    for k, (o, e) in enumerate(zip(out, exp)):
        assert np.array_equal(o.cpu().numpy().view("u1"), np.ascontiguousarray(e).view("u1")), f"unit {k} differs"
