"""Pass 2 with column groups side by side in one launch, and pass 1 with staged key loads, against the oracle.

The fast scatter kernel moves the 8-byte columns in groups of ``cols_per_launch`` columns.  All groups run in
one launch (ngroups x S CTAs, one group per CTA) unless fewer SMs than groups are left free by ``sm_reserve``;
then there is one launch per group.  Every output must be byte-identical to ``oracle/hash_partition.py``
whichever way the columns are split, at sizes around the tile (4096 rows) and chunk boundaries.
"""
import numpy as np
import pytest

from oracle import hash_partition as hp

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

SIZES = [4095, 4096, 4097, 100_003, 1 << 20, 3_000_017]
_cache = {}


def _dev():
    return torch.device("cuda", 0)


def _sm_count() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


def _keys(n: int, kind: str, seed: int):
    rng = np.random.default_rng(seed)
    if kind == "one":
        return [rng.integers(0, 1 << 16, n).astype("int64")]
    if kind == "two":
        return [rng.integers(-(2**40), 2**40, n).astype("int64"), rng.integers(0, 50, n).astype("int32")]
    if kind == "zipf":  # one hot key holds a large share of the rows
        return [np.minimum(rng.zipf(1.3, n), 1 << 20).astype("int64")]
    raise ValueError(kind)


def _table(n: int, nfast: int, kind: str = "one", seed: int = 0):
    """Key columns, then nfast 8-byte columns, then one 4-, 2- and 1-byte column (host arrays)."""
    key = (n, nfast, kind, seed)
    if key not in _cache:
        rng = np.random.default_rng(seed + 1)
        keys = _keys(n, kind, seed)
        fast = [rng.integers(-(2**63), 2**63 - 1, n, dtype="int64", endpoint=True) for _ in range(nfast)]
        narrow = [rng.integers(-(2**31), 2**31, n).astype("int32"), rng.integers(0, 1 << 16, n).astype("uint16"),
                  rng.integers(0, 256, n).astype("uint8")]
        _cache.clear()
        _cache[key] = (keys, fast + narrow)
    return _cache[key]


def _to_dev(a: np.ndarray):
    if a.dtype.kind == "u" and a.dtype.itemsize > 1:
        a = a.view(f"i{a.dtype.itemsize}")
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _expected(keys, num):
    pids = hp.partition_ids(keys, num)
    return hp.stable_partition(pids, num)


def _check(keys, cols, num, sm_reserve=0, cols_per_launch=0):
    from fugue_b200 import kernels as K

    dkeys = [_to_dev(k) for k in keys]
    dcols = [_to_dev(c) for c in cols]
    plan = K.partition_plan(dkeys, num)
    out = K.partition_apply(plan, dcols, sm_reserve=sm_reserve, cols_per_launch=cols_per_launch)
    torch.cuda.synchronize()
    order, offsets = _expected(keys, num)
    assert np.array_equal(plan.offsets.cpu().numpy(), offsets)
    for i, (c, o) in enumerate(zip(cols, out)):
        got = o.cpu().numpy().view("u1")
        exp = np.ascontiguousarray(c[order]).view("u1")
        assert np.array_equal(got, exp), f"column {i} (width {c.dtype.itemsize}) differs"


@pytest.mark.parametrize("cols_per_launch", range(1, 9))
@pytest.mark.parametrize("nfast", [1, 3, 5, 8, 10, 17])
def test_group_sizes(nfast, cols_per_launch):
    keys, cols = _table(100_003, nfast)
    _check(keys, cols, 256, cols_per_launch=cols_per_launch)


@pytest.mark.parametrize("cols_per_launch", [1, 2, 3, 4])
@pytest.mark.parametrize("reserve", ["0", "32", "fallback", "all"])
def test_sm_reserve(reserve, cols_per_launch):
    nfast = 8
    ngroups = -(-nfast // cols_per_launch)
    sm = {"0": 0, "32": 32, "fallback": _sm_count() - ngroups + 1, "all": _sm_count() + 5}[reserve]
    keys, cols = _table(1 << 20, nfast)
    _check(keys, cols, 256, sm_reserve=sm, cols_per_launch=cols_per_launch)


@pytest.mark.parametrize("kind", ["one", "two", "zipf"])
@pytest.mark.parametrize("num", [256, 200])
@pytest.mark.parametrize("n", SIZES)
def test_sizes_and_keys(n, num, kind):
    keys, cols = _table(n, 8, kind, seed=n % 97)
    _check(keys, cols, num)
    if n in (4097, 1 << 20):
        _check(keys, cols, num, cols_per_launch=3)


def test_more_groups_than_one_launch_holds():
    # 70 fast columns in groups of 1: more units than one launch takes (64)
    keys, cols = _table(20_000, 70)
    _check(keys, cols, 256, cols_per_launch=1)


@pytest.mark.parametrize("reserve", ["0", "fallback"])
@pytest.mark.parametrize("n", [100_003, (1 << 20) + 5])
def test_apply_map_across_groups(n, reserve):
    """Fused map units (two-operand ones among them) in groups of 2 (2 + 2 + 1 units)."""
    from fugue_b200 import kernels as K

    rng = np.random.default_rng(7)
    key = rng.integers(0, 1 << 16, n).astype("int64")
    f = [rng.standard_normal(n) for _ in range(3)]
    i = [rng.integers(-(2**62), 2**62, n).astype("int64") for _ in range(3)]
    dk = _to_dev(key)
    df = [_to_dev(x) for x in f]
    di = [_to_dev(x) for x in i]
    bits = lambda x: int(np.array([x], dtype="float64").view("i8")[0])  # noqa: E731
    units = [
        (dk, None, K.MAP_COPY, 0, 0, 0),
        (df[0], df[1], K.MAP_AFFINE_F64, bits(2.0), bits(-0.5), bits(1.25)),  # second unit of group 0
        (di[0], di[1], K.MAP_AFFINE_I64, 3, -7, 11),                          # first unit of group 1
        (df[2], None, K.MAP_AFFINE_F64, bits(0.1), 0, bits(-3.0)),
        (di[2], di[0], K.MAP_AFFINE_I64, -1, 5, 0),                           # alone in group 2
    ]
    sm = {"0": 0, "fallback": _sm_count() - 2}[reserve]
    plan = K.partition_plan([dk], 256)
    out = K.partition_apply_map(plan, units, sm_reserve=sm)
    torch.cuda.synchronize()
    order, _ = _expected([key], 256)
    u = lambda x: x[order].view("u8")  # noqa: E731
    with np.errstate(over="ignore"):
        exp = [
            key[order],
            (2.0 * f[0][order] + -0.5 * f[1][order]) + 1.25,
            (np.uint64(3) * u(i[0]) + np.uint64(2**64 - 7) * u(i[1]) + np.uint64(11)).view("i8"),
            0.1 * f[2][order] + -3.0,
            (np.uint64(2**64 - 1) * u(i[2]) + np.uint64(5) * u(i[0])).view("i8"),
        ]
    for k, (o, e) in enumerate(zip(out, exp)):
        assert np.array_equal(o.cpu().numpy().view("u1"), np.ascontiguousarray(e).view("u1")), f"unit {k} differs"


@pytest.mark.parametrize("n", [4097, 100_003, 1 << 20])
def test_radix_pass_digit_ranking(n):
    """Pass 1 ranks tiles by a radix digit of the key (staged key loads): stable LSD sort of (key, row)."""
    from fugue_b200 import sort

    rng = np.random.default_rng(n)
    key = rng.integers(0, 1 << 40, n, dtype="uint64")
    key[::7] = key[3]  # equal keys: stability shows in the row order
    k, idx = sort._radix_sort_pairs(_to_dev(key), torch.arange(n, dtype=torch.int64, device=_dev()))
    order = np.argsort(key, kind="stable")
    assert np.array_equal(idx.cpu().numpy(), order)
    assert np.array_equal(k.cpu().numpy().view("u8"), key[order])
