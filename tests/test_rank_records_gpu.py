"""Pass 1 of the hash partition (num <= 256) byte for byte: the rank record of every whole 4096-row tile and the
per-chunk prefix, read back from the plan's scratch buffer and compared with a numpy reference.

Scratch layout (``plan_layout`` in ``csrc/fb_partition.cu``): ``uint32 hist[nchunks][num]`` first (after the scan:
the exclusive prefix of every partition over the chunks), then at ``round256(nchunks * num * 4) + 256`` one
12800-byte record per whole tile: ``uint8 id[4096] | uint16 rank[4096] | uint16 count[256]``.  ``rank`` is the
number of earlier rows of the same partition in the tile (stable, row order); ``count`` the rows per partition.
The chunk geometry (``make_geom``) cuts the whole tiles into at most 2 x #SM chunks; a partial tail tile is a chunk
of its own.
"""
import numpy as np
import pytest

from oracle import hash_partition as hp

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

TILE = 4096
REC = 3 * TILE + 512
WARPS_PER_CTA = 16  # tiles of a chunk are dealt to the 16 warps of its CTA


def _dev():
    return torch.device("cuda", 0)


def _sm_count() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _to_dev(a: np.ndarray):
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _geom(n: int):
    """(tiles per chunk, chunks of whole tiles, chunks) as make_geom computes them."""
    ntiles = n // TILE
    max_chunks = 2 * _sm_count()
    per = -(-ntiles // max_chunks) if ntiles > 0 else 1
    nfull = -(-ntiles // per)
    return per, nfull, nfull + (1 if ntiles * TILE < n else 0)


def _expected(pids: np.ndarray, num: int):
    """(records [ntiles, REC] uint8, hist [nchunks, num] uint32) of the partition ids `pids`."""
    n = len(pids)
    per, nfull, nchunks = _geom(n)
    ntiles = n // TILE
    ids = pids[:ntiles * TILE].reshape(ntiles, TILE)
    key = (np.arange(ntiles, dtype="i8")[:, None] * 256 + ids).ravel()
    order = np.argsort(key, kind="stable")
    sk = key[order]
    first = np.r_[0, np.flatnonzero(sk[1:] != sk[:-1]) + 1]
    start = np.repeat(first, np.diff(np.r_[first, len(sk)]))
    rank = np.empty(len(key), dtype="i8")
    rank[order] = np.arange(len(key)) - start
    count = np.bincount(key, minlength=ntiles * 256).reshape(ntiles, 256)
    rec = np.empty((ntiles, REC), dtype="u1")
    rec[:, :TILE] = ids
    rec[:, TILE:3 * TILE] = rank.reshape(ntiles, TILE).astype("<u2").view("u1")
    rec[:, 3 * TILE:] = count.astype("<u2").view("u1")
    chunk_counts = np.zeros((nchunks, num), dtype="i8")
    for c in range(nfull):
        chunk_counts[c] = count[c * per:min((c + 1) * per, ntiles), :num].sum(axis=0)
    if nchunks > nfull:
        chunk_counts[nfull] = np.bincount(pids[ntiles * TILE:], minlength=num)
    hist = (np.cumsum(chunk_counts, axis=0) - chunk_counts).astype("u4")
    return rec, hist


def _read_scratch(scratch, n: int, num: int):
    _, _, nchunks = _geom(n)
    buf = scratch.cpu().numpy()
    hist = buf[:nchunks * num * 4].view("<u4").reshape(nchunks, num)
    at = ((nchunks * num * 4 + 255) // 256) * 256 + 256
    ntiles = n // TILE
    return buf[at:at + ntiles * REC].reshape(ntiles, REC), hist


def _compare(scratch, pids: np.ndarray, num: int):
    got_rec, got_hist = _read_scratch(scratch, len(pids), num)
    exp_rec, exp_hist = _expected(pids, num)
    bad = np.flatnonzero((got_rec != exp_rec).any(axis=1))
    if len(bad) > 0:
        t = bad[0]
        part = "id" if not np.array_equal(got_rec[t, :TILE], exp_rec[t, :TILE]) else (
            "rank" if not np.array_equal(got_rec[t, TILE:3 * TILE], exp_rec[t, TILE:3 * TILE]) else "count")
        pytest.fail(f"rank records of {len(bad)} tiles differ, the first (tile {t}) in {part}")
    assert np.array_equal(got_hist, exp_hist), "per-chunk prefix differs"


def _check_plan(cols, num, valid=None):
    from fugue_b200 import kernels as K

    dvalid = None if valid is None else [None if v is None else _to_dev(v.astype("u1")) for v in valid]
    plan = K.partition_plan([_to_dev(c) for c in cols], num, dvalid)
    torch.cuda.synchronize()
    pids = hp.partition_ids(cols, num, valid)
    _, offsets = hp.stable_partition(pids, num)
    assert np.array_equal(plan.offsets.cpu().numpy(), offsets)
    _compare(plan.scratch, pids, num)


def _sizes():
    """Row counts: 1 tile, k tiles, k tiles + a tail, one tile per chunk (+ tail), a short last chunk, and enough
    tiles per chunk that every warp ranks several tiles with the same counters."""
    sm2 = 2 * _sm_count()
    return {"1tile": TILE, "ktiles": 37 * TILE, "ktiles_tail": 37 * TILE + 123,
            "1perchunk_tail": (sm2 - 1) * TILE + 4095, "short_last_chunk": (2 * sm2 + 5) * TILE,
            "tiles_per_warp": ((WARPS_PER_CTA + 2) * sm2 - 3) * TILE + 77}


@pytest.mark.parametrize("num", [1, 2, 3, 16, 17, 255, 256])
@pytest.mark.parametrize("size", ["1tile", "ktiles_tail", "short_last_chunk"])
def test_int64_key(num, size):
    n = _sizes()[size]
    rng = np.random.default_rng(num * 7 + n)
    _check_plan([rng.integers(-(2**63), 2**63 - 1, n, dtype="int64", endpoint=True)], num)


@pytest.mark.parametrize("size", ["ktiles", "1perchunk_tail", "tiles_per_warp"])
@pytest.mark.parametrize("num", [16, 256])
def test_int64_key_sizes(size, num):
    n = _sizes()[size]
    rng = np.random.default_rng(n + num)
    _check_plan([rng.integers(0, 1 << 40, n, dtype="int64")], num)


@pytest.mark.parametrize("num", [3, 256])
def test_float_key_as_the_engine_passes_it(num):
    import pyarrow as pa

    from fugue_b200 import sort

    n = 29 * TILE + 1000
    rng = np.random.default_rng(5)
    x = rng.standard_normal(n).round(2)
    x[rng.random(n) < 0.05] = np.nan
    x[rng.random(n) < 0.05] = -0.0
    x[rng.random(n) < 0.05] = 0.0
    bits, v = sort.float_key(_to_dev(x), pa.float64(), None)
    bits_np = bits.cpu().numpy()
    valid = None if v is None else [v.cpu().numpy().astype(bool)]
    _check_plan([bits_np], num, valid)


@pytest.mark.parametrize("num", [17, 256])
def test_multi_column_key_with_nulls(num):
    n = 41 * TILE + 2049
    rng = np.random.default_rng(11)
    a = rng.integers(-1000, 1000, n).astype("int32")
    b = rng.integers(0, 50, n).astype("int64")
    va = rng.random(n) > 0.1
    vb = rng.random(n) > 0.3
    _check_plan([a, b], num, [va, vb])


@pytest.mark.parametrize("num", [1, 16, 256])
def test_all_rows_in_one_partition(num):
    n = 300 * TILE + 5
    _check_plan([np.full(n, 123456789, dtype="int64")], num)


@pytest.mark.parametrize("num", [16, 256])
def test_zipf_keys(num):
    n = 333 * TILE + 4001
    rng = np.random.default_rng(3)
    _check_plan([rng.zipf(1.3, n).astype("int64")], num)


@pytest.mark.parametrize("shift,size", [(0, "ktiles_tail"), (8, "ktiles_tail"), (24, "short_last_chunk"),
                                        (56, "ktiles_tail"), (0, "tiles_per_warp"), (56, "tiles_per_warp")])
def test_radix_digit_pass(shift, size):
    from fugue_b200 import _lib
    from fugue_b200 import kernels as K

    n = _sizes()[size]
    rng = np.random.default_rng(shift + n)
    key = rng.integers(-(2**63), 2**63 - 1, n, dtype="int64", endpoint=True)
    if shift == 56:
        key[rng.random(n) < 0.5] = 0x12 << 56  # half the rows in one digit
    idx = np.arange(n, dtype="int64")
    dk, di = _to_dev(key), _to_dev(idx)
    k2, i2 = torch.empty_like(dk), torch.empty_like(di)
    dev = _dev()
    scratch = torch.empty(K.partition_scratch_bytes(dev, n, 256), dtype=torch.uint8, device=dev)
    offsets = torch.empty(257, dtype=torch.int64, device=dev)
    _lib.check(_lib.load().fb_radix_pass(
        dev.index, K._stream_ptr(dev), n, dk.data_ptr(), shift, 2, _lib.ptr_array([dk.data_ptr(), di.data_ptr()]),
        _lib.i32_array([8, 8]), _lib.ptr_array([k2.data_ptr(), i2.data_ptr()]), scratch.data_ptr(), scratch.numel(),
        offsets.data_ptr()))
    torch.cuda.synchronize()
    pids = ((key.view("u8") >> np.uint64(shift)) & np.uint64(255)).astype("i8")
    order, exp_off = hp.stable_partition(pids, 256)
    assert np.array_equal(offsets.cpu().numpy(), exp_off)
    assert np.array_equal(i2.cpu().numpy(), order)
    _compare(scratch, pids, 256)
