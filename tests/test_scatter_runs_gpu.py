"""The fast scatter kernel places each CTA's chunks as one run, against the oracle.

Every CTA of a column group takes a run of consecutive chunks and keeps its write-combining state (each partition's
output cursor and its pending rows, fewer than one 16-row group) from one chunk into the next: where a partition's
rows of chunk c end in the output, its rows of chunk c + 1 begin, so nothing is flushed between them.  The cases
here put, at the chunk boundaries inside a run, every pending count 0 .. 15 and 0, 1, 15, 16 or 17 rows of a
partition in the chunk's last tile, for runs of 1 chunk up to all of them (SMs held back make the runs longer), at
both write-group sizes (2 and 1 columns per group).  Every output must be byte-identical to
``oracle/hash_partition.py``.
"""
import numpy as np
import pytest

from oracle import hash_partition as hp

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

TILE = 4096
G = 16
SPECIAL = np.array([0, 1, G - 1, G, G + 1])
_pools = {}


def _sm_count() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _to_dev(a: np.ndarray):
    return torch.from_numpy(np.ascontiguousarray(a)).to(torch.device("cuda", 0))


def _keys_for(pids: np.ndarray, num: int, rng) -> np.ndarray:
    if num not in _pools:
        cand = np.arange(0, 200 * num + 20_000, dtype="int64")
        pid = hp.partition_ids([cand], num)
        _pools[num] = [cand[pid == p] for p in range(num)]
    keys = np.empty(len(pids), dtype="int64")
    for p in np.unique(pids):
        at = np.flatnonzero(pids == p)
        keys[at] = rng.choice(_pools[num][p], len(at))
    return keys


def _pids(ntiles: int, extra: int, num: int, seed: int) -> np.ndarray:
    """Tile t gives partition p < num - 1 one of 0, 1, 15, 16, 17 rows and, every third tile, every third partition
    up to 15 more, so that the pending counts drift through every value mod 16; the last partition takes the rest
    of the tile."""
    rng = np.random.default_rng(seed)
    out = []
    for t in range(ntiles):
        counts = SPECIAL[(np.arange(num) * 3 + t) % len(SPECIAL)]
        if t % 3 == 0:
            counts = counts + np.where(np.arange(num) % 3 == 0, rng.integers(0, G, num), 0)
        counts[-1] = 0
        counts[-1] = TILE - counts.sum()
        tile = np.repeat(np.arange(num), counts)
        rng.shuffle(tile)
        out.append(tile)
    out.append(rng.integers(0, num, extra))
    return np.concatenate(out).astype("int64")


def _runs(ntiles: int, ctas_per_group: int):
    """Tile ranges of the full chunks and the chunk runs of the CTAs of one group (the kernel's geometry)."""
    per = -(-ntiles // (2 * _sm_count()))
    nchunks = -(-ntiles // per)
    s = min(ctas_per_group, nchunks)
    return per, nchunks, [(i * nchunks // s, (i + 1) * nchunks // s) for i in range(s)]


def _check(keys, cols, num, sm_reserve, cols_per_launch):
    from fugue_b200 import kernels as K

    plan = K.partition_plan([_to_dev(keys)], num)
    out = K.partition_apply(plan, [_to_dev(c) for c in cols], sm_reserve=sm_reserve, cols_per_launch=cols_per_launch)
    torch.cuda.synchronize()
    order, offsets = hp.stable_partition(hp.partition_ids([keys], num), num)
    assert np.array_equal(plan.offsets.cpu().numpy(), offsets)
    for i, (c, o) in enumerate(zip(cols, out)):
        assert np.array_equal(o.cpu().numpy().view("u1"), np.ascontiguousarray(c[order]).view("u1")), \
            f"column {i} differs"


@pytest.mark.parametrize("cols_per_launch", [1, 2])
@pytest.mark.parametrize("ctas_per_group", ["all", 7, 2, 1])
def test_runs_across_chunk_boundaries(ctas_per_group, cols_per_launch):
    num, ncols, ntiles, extra = 256, 4, 400, 123
    groups = ncols // cols_per_launch
    cpg = _sm_count() // groups if ctas_per_group == "all" else ctas_per_group
    sm_reserve = _sm_count() - cpg * groups
    pids = _pids(ntiles, extra, num, seed=cpg * 10 + cols_per_launch)
    per, nchunks, runs = _runs(ntiles, cpg)
    # the boundaries between two chunks of one run: each partition's pending count there (its output row, mod 16)
    # and its rows in the last tile before it
    inner = [c for c0, c1 in runs for c in range(c0 + 1, c1)]
    assert inner, "no run spans a chunk boundary"
    counts = np.stack([np.bincount(pids[t * TILE:(t + 1) * TILE], minlength=num) for t in range(ntiles)])
    total = np.bincount(pids, minlength=num)
    at = np.cumsum(counts, axis=0) - counts + (np.cumsum(total) - total)
    pending = {int(v) for c in inner for v in at[c * per] % G}
    last_tile = {int(v) for c in inner for v in counts[c * per - 1]}
    assert pending == set(range(G)), f"pending counts at the boundaries: {sorted(pending)}"
    assert set(SPECIAL.tolist()) <= last_tile
    keys = _keys_for(pids, num, np.random.default_rng(cpg))
    payload = np.random.default_rng(cpg + 1).integers(-(2**63), 2**63 - 1, (ncols - 1, len(keys)), dtype="int64",
                                                       endpoint=True)
    _check(keys, [keys, *payload], num, sm_reserve, cols_per_launch)
