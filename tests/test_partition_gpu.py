"""Parity of the sm_90a hash-partition kernels (through the C ABI) with the oracle."""
import os

import numpy as np
import pandas as pd
import pytest

from oracle import hash_partition as hp

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
HERE = os.path.dirname(os.path.abspath(__file__))


def _dev():
    return torch.device("cuda", 0)


def _to_dev(a: np.ndarray):
    if a.dtype == bool:
        return torch.from_numpy(a.view("u1").copy()).to(_dev())
    if a.dtype.kind == "u" and a.dtype.itemsize > 1:
        a = a.view(f"i{a.dtype.itemsize}")
    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _bytes(t) -> np.ndarray:
    return t.cpu().numpy().view("u1")


def test_library_loaded_and_device_is_hopper():
    import ctypes as C

    from fugue_b200 import _lib

    lib = _lib.load()
    sm, mem, maj, mnr = C.c_int(), C.c_size_t(), C.c_int(), C.c_int()
    _lib.check(lib.fb_device_info(0, C.byref(sm), C.byref(mem), C.byref(maj), C.byref(mnr)))
    assert (maj.value, mnr.value) == (9, 0) and sm.value >= 100


def test_partition_ids_golden_vectors():
    from fugue_b200 import kernels as K

    gold = np.load(os.path.join(HERE, "golden", "hash_vectors.npz"), allow_pickle=False)
    for i, combo in enumerate(gold["combos"]):
        names = str(combo).split(",")
        keys = [_to_dev(gold[n]) for n in names]
        for num in (1, 2, 3, 107, 256, 1000, 65536, 2**31 - 1):
            got = K.partition_ids(keys, num).cpu().numpy().astype("int64")
            exp = (gold[f"hash_{i}"] % np.uint64(num)).astype("int64")
            assert np.array_equal(got, exp), (combo, num)


def test_partition_ids_reference_known_answer():
    # tests/fugue_dask/test_utils.py:106-108
    from fugue_b200 import kernels as K

    aa = np.array([0, 1, 1, 2, 3, 4], dtype="int64")
    pids = K.partition_ids([_to_dev(aa)], 3).cpu().numpy()
    buckets = sorted(sorted(aa[pids == p].tolist()) for p in np.unique(pids))
    assert buckets == [[0, 2], [1, 1, 3, 4]]
    keys = np.array([0, 1, 2, 3, 4, -5, 2**62, -(2**63)], dtype="int64")
    assert K.partition_ids([_to_dev(keys)], 256).cpu().tolist() == [99, 18, 81, 147, 63, 29, 114, 81]


def test_partition_ids_null_keys():
    from fugue_b200 import kernels as K

    rng = np.random.default_rng(0)
    n = 10000
    a = rng.integers(0, 50, n).astype("int64")
    b = rng.standard_normal(n)
    va = (rng.random(n) > 0.2).astype("uint8")
    got = K.partition_ids([_to_dev(a), _to_dev(b)], 256, [_to_dev(va), None]).cpu().numpy()
    exp = hp.partition_ids([a, b], 256, [va, None])
    assert np.array_equal(got, exp)


def _check_partition(cols, key_idx, num, valid=None):
    from fugue_b200 import kernels as K

    dcols = [_to_dev(c) for c in cols]
    dvalid = None if valid is None else [None if v is None else _to_dev(v) for v in valid]
    out, off = K.partition_columns(dcols, key_idx, num, dvalid)
    torch.cuda.synchronize()
    exp_cols, exp_off = hp.partition_table(list(cols), key_idx, num, None if valid is None else
                                           [valid[key_idx.index(i)] if i in key_idx else None
                                            for i in range(len(cols))])
    assert np.array_equal(off.cpu().numpy(), exp_off)
    for c, (a, b) in enumerate(zip(out, exp_cols)):
        assert np.array_equal(_bytes(a), np.ascontiguousarray(b).view("u1")), f"column {c} differs"


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 4095, 4096, 4097, 100003, 1 << 20, 3_000_017])
@pytest.mark.parametrize("num", [1, 2, 3, 256])
def test_partition_benchmark_schema_sizes(n, num):
    rng = np.random.default_rng(n * 31 + num)
    cols = [rng.integers(0, 1 << 16, n).astype("int64")] + \
           [rng.integers(-(2**62), 2**62, n).astype("int64") for _ in range(3)] + \
           [rng.standard_normal(n) for _ in range(4)]
    _check_partition(cols, [0], num)


@pytest.mark.parametrize("num", [7, 255, 257, 1000, 1024])
def test_partition_other_partition_counts(num):
    rng = np.random.default_rng(num)
    n = 200_001
    cols = [rng.integers(-1000, 1000, n).astype("int64"), rng.standard_normal(n)]
    _check_partition(cols, [0], num)


def test_partition_mixed_widths_multi_key_nulls():
    rng = np.random.default_rng(11)
    n = 150_000
    cols = [rng.integers(0, 300, n).astype("int32"), rng.integers(0, 5, n).astype("int16"),
            rng.standard_normal(n), rng.integers(0, 255, n).astype("uint8"),
            rng.standard_normal(n).astype("float32"), rng.integers(0, 2, n).astype(bool),
            np.arange(n, dtype="int64")]
    v0 = (rng.random(n) > 0.1).astype("uint8")
    _check_partition(cols, [0, 1], 64, [v0, None])
    _check_partition(cols, [2], 33)
    _check_partition(cols, [0, 1, 3, 5], 256)


def test_partition_skew_and_single_key():
    rng = np.random.default_rng(13)
    n = 500_000
    zipf = np.minimum(rng.zipf(1.2, n), 1 << 20).astype("int64")
    _check_partition([zipf, np.arange(n, dtype="int64")], [0], 256)
    same = np.full(n, 42, dtype="int64")
    _check_partition([same, np.arange(n, dtype="int64")], [0], 256)


def test_partition_matches_live_pandas_hash():
    # the reference expression itself (fugue_dask/_utils.py:155-161), evaluated live
    from fugue_b200 import kernels as K

    rng = np.random.default_rng(17)
    n = 300_000
    df = pd.DataFrame({"key": rng.integers(0, 1 << 16, n), "v": rng.standard_normal(n)})
    ref_pid = pd.util.hash_pandas_object(df[["key"]], index=False).mod(256).astype(int).to_numpy()
    out, off = K.partition_columns([_to_dev(df.key.to_numpy()), _to_dev(df.v.to_numpy())], [0], 256)
    off = off.cpu().numpy()
    assert np.array_equal(np.diff(off), np.bincount(ref_pid, minlength=256))
    k2 = out[0].cpu().numpy()
    v2 = out[1].cpu().numpy()
    order = np.argsort(ref_pid, kind="stable")
    assert np.array_equal(k2, df.key.to_numpy()[order]) and np.array_equal(v2, df.v.to_numpy()[order])


def test_plan_then_apply_column_by_column():
    from fugue_b200 import kernels as K

    rng = np.random.default_rng(19)
    n = 123_457
    cols = [rng.integers(0, 999, n).astype("int64"), rng.standard_normal(n), rng.standard_normal(n)]
    d = [_to_dev(c) for c in cols]
    plan = K.partition_plan([d[0]], 256)
    outs = [K.partition_apply(plan, [c])[0] for c in d]
    exp, exp_off = hp.partition_table(cols, [0], 256)
    assert np.array_equal(plan.offsets.cpu().numpy(), exp_off)
    for a, b in zip(outs, exp):
        assert np.array_equal(_bytes(a), b.view("u1"))


def test_full_size_properties_100m_rows():
    """BASELINE config 2 size (100 M rows x 8 cols): size-independent properties."""
    from fugue_b200 import kernels as K

    n, num = 100_000_000, 256
    g = torch.Generator(device=_dev()).manual_seed(0)
    key = torch.randint(0, 1 << 16, (n,), dtype=torch.int64, device=_dev(), generator=g)
    rowid = torch.arange(n, dtype=torch.int64, device=_dev())
    pay = [torch.randint(-(2**62), 2**62, (n,), dtype=torch.int64, device=_dev(), generator=g)
           for _ in range(2)]
    fcols = [torch.randn(n, dtype=torch.float64, device=_dev(), generator=g) for _ in range(4)]
    cols = [key, rowid] + pay + fcols
    out, off = K.partition_columns(cols, [0], num)
    # offsets are a histogram of the partition ids
    pid_in = K.partition_ids([key], num)
    hist = torch.bincount(pid_in.long(), minlength=num)
    assert torch.equal(off[1:] - off[:-1], hist) and int(off[0]) == 0 and int(off[-1]) == n
    # every output row sits in the partition its key hashes to
    pid_out = K.partition_ids([out[0]], num).long()
    seg = torch.repeat_interleave(torch.arange(num, device=_dev()), hist)
    assert torch.equal(pid_out, seg)
    del pid_out, seg, pid_in
    # stable: row ids increase inside each partition; boundaries are the only descents
    rid = out[1]
    desc = (rid[1:] < rid[:-1]).nonzero().flatten() + 1
    bounds = set(off[1:-1].cpu().tolist())
    assert set(desc.cpu().tolist()) <= bounds
    # rows are moved intact: gather the inputs by output row id and compare bit patterns
    for c in range(len(cols)):
        assert torch.equal(cols[c][rid].view(torch.int64), out[c].view(torch.int64)), c
    # permutation: every row id appears exactly once (checksum of checksums)
    assert int(rid.sum()) == n * (n - 1) // 2
    assert int((rid ^ (rid >> 7)).sum()) == int((rowid ^ (rowid >> 7)).sum())


def _misaligned(a: np.ndarray):
    """``a`` on the device at an address that is 8- but not 16-byte aligned (8-byte columns): a column of a
    device table sliced at row 1."""
    t = torch.empty(len(a) + 1, dtype=_to_dev(a[:1]).dtype, device=_dev())
    t[1:].copy_(_to_dev(a))
    assert t[1:].data_ptr() % 16 == 8 or a.dtype.itemsize < 8
    return t[1:]


def _check_scatter_route(route: str) -> None:
    from fugue_b200 import api as fa
    from fugue_b200 import kernels as K
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.partition import PartitionSpec
    from fugue_b200.table import B200Table

    rng = np.random.default_rng(23)
    n = 1_234_567
    key = rng.integers(0, 1 << 16, n).astype("int64")
    c8 = [rng.integers(-(2**62), 2**62, n).astype("int64") for _ in range(4)] + \
         [rng.standard_normal(n) for _ in range(5)]
    if route.startswith("misaligned"):
        # 8-byte columns at an 8-byte boundary take the generic kernel over all chunks (all-8-byte or mixed widths),
        # next to 16-byte-aligned ones on the fast kernel
        num = int(route.split("_")[-1])
        mixed = "mixed" in route
        cols = [key] + c8 + ([rng.integers(-2**31, 2**31, n).astype("int32"), rng.integers(0, 256, n).astype("uint8")]
                             if mixed else [])
        dcols = [_misaligned(c) if i % 2 == 0 or c.dtype.itemsize < 8 else _to_dev(c) for i, c in enumerate(cols)]
        out, off = K.partition_columns(dcols, [0, 3], num)
        exp, exp_off = hp.partition_table(cols, [0, 3], num)
        assert np.array_equal(off.cpu().numpy(), exp_off)
        for c, (a, b) in enumerate(zip(out, exp)):
            assert np.array_equal(_bytes(a), b.view("u1")), f"column {c} differs"
    elif route.startswith("cols_per_launch"):
        per = int(route.split("_")[-1])
        d = [_to_dev(c) for c in [key] + c8]                          # 10 aligned 8-byte columns
        plan = K.partition_plan([d[0]], 256)
        out = K.partition_apply(plan, d, cols_per_launch=per)
        exp, exp_off = hp.partition_table([key] + c8, [0], 256)
        assert np.array_equal(plan.offsets.cpu().numpy(), exp_off)
        for c, (a, b) in enumerate(zip(out, exp)):
            assert np.array_equal(_bytes(a), b.view("u1")), f"column {c} differs"
    else:
        # a device table sliced at row 1 through engine.repartition / fa.transform; the validity mask travels too
        import pyarrow as pa

        v = rng.random(n) < 0.9
        tbl = pa.table({"k": key, "a": c8[0], "x": pa.array(c8[5], mask=~v),
                        "i": rng.integers(0, 9, n).astype("int32")})
        t = B200Table.from_arrow(tbl, _dev()).slice(1, n)
        e = fa.make_execution_engine("b200")
        spec = PartitionSpec(by="k", algo="hash", num=200)
        assert t.columns[0].data_ptr() % 16 == 8 and t.columns[3].data_ptr() % 16 == 4

        def identity(tb: B200Table) -> B200Table:
            return tb

        if route == "repartition_sliced":
            got = e.repartition(B200DataFrame(t), spec).native
        else:
            got = fa.transform(B200DataFrame(t), identity, schema="*", partition=spec, engine=e, as_fugue=True).native
            assert got.offsets is not None
        cols = [c.cpu().numpy() for c in t.columns] + [t.valid[2].cpu().numpy()]
        assert np.array_equal(cols[4], v[1:].astype("uint8"))
        exp, exp_off = hp.partition_table(cols, [0], 200)
        assert np.array_equal(got.offsets.cpu().numpy(), exp_off)
        for c in range(4):
            assert np.array_equal(_bytes(got.columns[c]), exp[c].view("u1")), f"column {c} differs"
        assert np.array_equal(got.valid[2].cpu().numpy(), exp[4])
        assert got.valid[0] is None and got.valid[1] is None and got.valid[3] is None


@pytest.mark.parametrize("route", ["misaligned_all8_256", "misaligned_mixed_256", "misaligned_mixed_200",
                                   "misaligned_all8_1000", "cols_per_launch_1", "cols_per_launch_8",
                                   "repartition_sliced", "transform_sliced"])
def test_scatter_routes_agree(route):
    """Every route of pass 2: the fast kernel on 16-byte-aligned 8-byte columns (num <= 256) in groups of 1 and 8
    columns per launch, and the generic kernel (all-8-byte or mixed widths) on the rest, also over a device table
    sliced at row 1: the same bits as the oracle."""
    _check_scatter_route(route)
