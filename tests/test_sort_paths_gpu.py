"""The device sort (``fugue_b200/sort.py``) against the exact CPU reference ``oracle/sort.py``: the radix passes,
``argsort_rows`` / ``sort_table`` on every storage type, ``group_starts`` / ``logical_offsets``, ``fa.take``, the
logical partitions ``fa.transform`` hands to a function, window maps and ``aggregate`` on float keys.  Row
permutations are compared exactly, with row ids, so stability is checked too.

Float keys follow one rule (DESIGN §7d): a NaN of either sign is NULL, -0.0 equals 0.0."""
from collections import Counter, OrderedDict

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import _lib
from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from fugue_b200 import sort as S
from fugue_b200.column import all_cols, col, functions as f
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.partition import PartitionSpec
from fugue_b200.table import B200Table
from oracle import sort as O
from test_window_gpu import ALL, ALL_SCHEMA, _check, _input

DEV = torch.device("cuda", 0)
I64_MIN, I64_MAX = -(2**63), 2**63 - 1
NEG_NAN = np.array([-0x0007FFFF00000001], dtype=np.int64).view(np.float64)[0]  # sign bit set, with a payload
POS_NAN_PAYLOAD = np.array([0x7FF0000000000001], dtype=np.int64).view(np.float64)[0]
F64 = np.array([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, 5e-324, -5e-324, 2.2250738585072014e-308, np.nan, NEG_NAN,
                POS_NAN_PAYLOAD, 1.5])
F32 = np.array([0, 0x80000000, 0x3F800000, 0xBF800000, 0x7F800000, 0xFF800000, 1, 0x80000001, 0x7FC00000,
                0xFFC00001, 0x7F800001, 0x3FC00000], dtype=np.uint32).view(np.float32)
KEY_F = np.array([0.0, -0.0, np.nan, NEG_NAN, 1.5, -3.0])  # float keys: the classes {0, -0}, {NaN, -NaN, NULL}


@pytest.fixture(scope="module")
def engine():
    return fa.make_execution_engine("b200")


def _dev(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ---- 1. the radix passes -------------------------------------------------------------------------------------
def _radix_keys(pattern: str, n: int, rng) -> np.ndarray:
    m = max(n // 4, 1)  # a pool of a quarter as many values: ties everywhere
    if pattern == "byte0":
        pool = np.int64(0x1234567890ABCD00) | rng.integers(0, 256, m)
    elif pattern == "byte7":  # same sign: lo ^ hi has only its top byte set
        pool = (rng.integers(0, 128, m) << 56) | np.int64(0x0011223344556677)
    elif pattern == "byte7-signs":
        pool = ((rng.integers(0, 256, m).astype(np.uint64) << np.uint64(56)) | np.uint64(0x0011223344556677)
                ).view(np.int64)
    elif pattern == "every":
        pool = rng.integers(I64_MIN, I64_MAX, m, endpoint=True, dtype=np.int64)
    elif pattern == "equal":  # lo == hi: no pass runs
        pool = np.array([-12345], dtype=np.int64)
    elif pattern == "negative":
        pool = rng.integers(I64_MIN, -1, m, endpoint=True, dtype=np.int64)
    elif pattern == "mixed-signs":
        pool = rng.integers(-1000, 1000, m, dtype=np.int64)
    elif pattern == "specials":
        pool = np.array([0, -1, I64_MIN, I64_MAX], dtype=np.int64)
    else:
        raise ValueError(pattern)
    return np.asarray(pool, dtype=np.int64)[rng.integers(0, len(np.atleast_1d(pool)), n)]


@pytest.mark.parametrize("n", [0, 1, 2, 4095, 4096, 4097, 2**20 + 1, 3_000_017])
@pytest.mark.parametrize("pattern", ["byte0", "byte7", "byte7-signs", "every", "equal", "negative", "mixed-signs",
                                     "specials"])
def test_radix_sort_pairs(pattern, n):
    rng = np.random.default_rng(n + len(pattern))
    key = _radix_keys(pattern, n, rng)
    k, idx = S._radix_sort_pairs(_dev(key), torch.arange(n, dtype=torch.int64, device=DEV))
    order = np.argsort(key.view(np.uint64), kind="stable")
    assert np.array_equal(idx.cpu().numpy(), order)
    assert np.array_equal(k.cpu().numpy(), key[order])


# ---- 2. argsort_rows / sort_table on every storage type --------------------------------------------------------
POOLS = {
    "i8": (pa.int8(), np.array([-128, 127, -1, 0, 1, 5], dtype=np.int8)),
    "i16": (pa.int16(), np.array([-32768, 32767, -1, 0, 255, 256], dtype=np.int16)),
    "i32": (pa.int32(), np.array([-(2**31), 2**31 - 1, -1, 0, 65536, 7], dtype=np.int32)),
    "i64": (pa.int64(), np.array([I64_MIN, I64_MAX, -1, 0, 2**40, 1], dtype=np.int64)),
    "u8": (pa.uint8(), np.array([0, 1, 127, 128, 255], dtype=np.uint8)),
    "u16": (pa.uint16(), np.array([0, 1, 2**15 - 1, 2**15, 2**16 - 1], dtype=np.uint16)),
    "u32": (pa.uint32(), np.array([0, 1, 2**31 - 1, 2**31, 2**32 - 1], dtype=np.uint32)),
    "u64": (pa.uint64(), np.array([0, 1, 2**63 - 1, 2**63, 2**64 - 1], dtype=np.uint64)),
    "f32": (pa.float32(), F32),
    "f64": (pa.float64(), F64),
    "b": (pa.bool_(), np.array([False, True])),
    "d": (pa.date32(), np.array([-1000, -1, 0, 1, 19000], dtype=np.int32)),
    "ts": (pa.timestamp("us"), np.array([-(10**15), -1, 0, 1, 10**15], dtype=np.int64)),
    # first value "z": the dictionary's code order (first appearance) is not the sorted order
    "s": (pa.string(), np.array(["z", "", "a", "é", "日本", "Z", "ab", "a "], dtype=object)),
}
TYPES = list(POOLS)


def _column(name: str, n: int, rng, null_rate: float) -> pa.Array:
    tp, pool = POOLS[name]
    vals = pool[rng.integers(0, len(pool), n)]
    vals[0] = pool[0]
    mask = rng.random(n) < null_rate if null_rate > 0 else None
    if name == "s":
        return pa.array(list(vals), mask=mask, type=pa.string())
    if name in ("d", "ts"):
        return pa.array(vals, mask=mask).view(tp)
    return pa.array(vals, mask=mask, type=tp)


def _garbage_under_nulls(n: int, rng) -> pa.Array:
    """A NULL-heavy int64 column whose storage under NULL is not 0: the sort must not read it."""
    data = rng.integers(-5, 5, n, dtype=np.int64)
    null = rng.random(n) < 0.9
    data[null] = rng.integers(I64_MIN, I64_MAX, int(null.sum()), dtype=np.int64)
    bits = np.packbits(~null, bitorder="little")
    return pa.Array.from_buffers(pa.int64(), n, [pa.py_buffer(bits.tobytes()), pa.py_buffer(data.tobytes())],
                                 null_count=int(null.sum()))


def _typed_table(n: int, seed: int) -> pa.Table:
    rng = np.random.default_rng(seed)
    cols = {"rid": pa.array(np.arange(n, dtype=np.int64))}
    for name in TYPES:
        cols[name] = _column(name, n, rng, 0.2)
        cols[name + "_nn"] = _column(name, n, rng, 0.0)  # no validity mask (floats still hold valid NaN)
    cols["garbage"] = _garbage_under_nulls(n, rng)
    cols["s_allnull"] = pa.array([None] * n, type=pa.string())
    cols["s_one"] = pa.array(["x"] * n, mask=rng.random(n) < 0.3, type=pa.string())
    return pa.table(cols)


@pytest.fixture(scope="module")
def typed():
    t = _typed_table(20_011, 1)
    return t, B200Table.from_arrow(t, DEV)


def _argsort_matches(at: pa.Table, bt: B200Table, sorts, na_position) -> None:
    got = S.argsort_rows(bt, sorts, na_position).cpu().numpy()
    exp = O.argsort(at, sorts, na_position)
    assert np.array_equal(got, exp), (dict(sorts), na_position)


@pytest.mark.parametrize("name", TYPES + ["garbage", "s_allnull", "s_one"])
def test_argsort_rows_on_every_type(typed, name):
    at, bt = typed
    for nm in [name] + ([name + "_nn"] if name in POOLS else []):
        for asc in (True, False):
            for na_position in ("first", "last"):
                _argsort_matches(at, bt, OrderedDict([(nm, asc)]), na_position)


@pytest.mark.parametrize("name,passes", [("u8_nn", 1), ("u16_nn", 2), ("u32_nn", 4), ("b_nn", 1), ("s_nn", 1)])
def test_only_the_varying_bytes_get_a_pass(typed, monkeypatch, name, passes):
    """A narrow key spanning its whole range takes one radix pass per byte of its width, ASC and DESC: an unsigned
    value is zero-extended, not sign-extended from its storage type (which would make every byte vary)."""
    at, bt = typed
    lib = _lib.load()
    shifts = []

    def spy(*a, _real=lib.fb_radix_pass):
        shifts.append(int(a[4]))
        return _real(*a)

    monkeypatch.setattr(lib, "fb_radix_pass", spy)
    for asc in (True, False):
        shifts.clear()
        _argsort_matches(at, bt, OrderedDict([(name, asc)]), "last")
        assert shifts == [8 * b for b in range(passes)], (asc, shifts)


@pytest.mark.parametrize("na_position", ["first", "last"])
@pytest.mark.parametrize("sorts", [
    [("s", True), ("f64", False)],
    [("i8", False), ("u64", True), ("f32", True)],
    [("b", True), ("d", False), ("s", False), ("i64", True)],
    [("garbage", True), ("u32", False), ("ts", True)],
    [("f64_nn", False), ("u16", True), ("s_one", False), ("i16", True)],
])
def test_sort_table_by_several_columns(typed, sorts, na_position):
    at, bt = typed
    sorts = OrderedDict(sorts)
    _argsort_matches(at, bt, sorts, na_position)
    got = S.sort_table(bt, sorts, na_position)
    assert np.array_equal(got.column("rid").cpu().numpy(), O.argsort(at, sorts, na_position))
    exp = at.take(pa.array(O.argsort(at, sorts, na_position)))
    for name in sorts:  # the payload moves with its row, bits and validity included
        i = bt.schema.index_of_key(name)
        g_valid = np.ones(bt.num_rows, dtype=bool) if got.valid[i] is None else got.valid[i].cpu().numpy() != 0
        e_valid = np.asarray(exp.column(name).combine_chunks().is_valid().to_numpy(zero_copy_only=False), dtype=bool)
        assert np.array_equal(g_valid, e_valid), name


def test_sort_large_multi_column():
    rng = np.random.default_rng(9)
    n = 2**20 + 1
    t = pa.table({"a": _column("i32", n, rng, 0.1), "f": _column("f64", n, rng, 0.1), "u": _column("u64", n, rng, 0.1)})
    bt = B200Table.from_arrow(t, DEV)
    for sorts, na_position in [(OrderedDict([("a", True), ("f", False), ("u", True)]), "last"),
                               (OrderedDict([("f", True), ("u", False)]), "first")]:
        _argsort_matches(t, bt, sorts, na_position)


# ---- 3. group_starts / logical_offsets ----------------------------------------------------------------------------
@pytest.mark.parametrize("keys", [[t] for t in TYPES] + [["garbage"], ["s_allnull"], ["f64", "f32"], ["f64_nn"],
                                                         ["i8", "s", "f64"], ["u64", "b", "d", "garbage"]])
def test_group_starts_match_the_oracle(typed, keys):
    at, bt = typed
    order = O.argsort(at, OrderedDict((k, True) for k in keys), "last")
    st = at.take(pa.array(order))
    sbt = S.take_rows(bt, _dev(order))  # the gather keeps the storage under NULL as it was
    assert np.array_equal(S.group_starts(sbt, keys).cpu().numpy(), O.group_heads(st, keys)), keys
    assert np.array_equal(S.logical_offsets(sbt, keys).cpu().numpy(), O.logical_offsets(st, keys)), keys


def test_float_key_example():
    t = pa.table({"k": pa.array([0.0, -0.0, 1.0, np.nan, 0.0, NEG_NAN, -1.0, None], type=pa.float64())})
    bt = B200Table.from_arrow(t, DEV)
    idx = S.argsort_rows(bt, OrderedDict(k=True), "last")
    assert idx.cpu().tolist() == [6, 0, 1, 4, 2, 3, 5, 7]
    st = S.take_rows(bt, idx)
    assert S.logical_offsets(st, ["k"]).cpu().tolist() == [0, 1, 4, 5, 8]
    # values are not rewritten: -0.0 and the NaNs keep their own bits (the last row is the NULL)
    bits = np.array([0.0, -0.0, 1.0, np.nan, 0.0, NEG_NAN, -1.0]).view(np.int64)
    assert st.column("k").cpu().numpy().view(np.int64)[:7].tolist() == bits[[6, 0, 1, 4, 2, 3, 5]].tolist()


# ---- 4. fa.take ------------------------------------------------------------------------------------------------------
def _take_table(n: int, seed: int) -> pa.Table:
    rng = np.random.default_rng(seed)
    m = lambda q: rng.random(n) < q  # noqa: E731
    return pa.table({
        "rid": pa.array(np.arange(n, dtype=np.int64)),
        "k": pa.array(rng.integers(0, 6, n), mask=m(0.1)),
        "kf": pa.array(KEY_F[rng.integers(0, len(KEY_F), n)], mask=m(0.1)),
        "s": pa.array(list(np.array(["q", "", "é", "a"], dtype=object)[rng.integers(0, 4, n)]), mask=m(0.1),
                      type=pa.string()),
        "v": pa.array(rng.integers(0, 5, n), mask=m(0.2)),
        "w": pa.array(F64[rng.integers(0, len(F64), n)], mask=m(0.1)),
    })


def _presort_str(sorts: "OrderedDict[str, bool]") -> str:
    return ",".join(f"{k} {'asc' if a else 'desc'}" for k, a in sorts.items())


def _take(engine, t: pa.Table, n: int, sorts, na_position: str, by) -> list:
    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    res = fa.take(df, n, presort=_presort_str(sorts), na_position=na_position,
                  partition=None if not by else dict(by=by), engine=engine, as_fugue=True)
    return res.as_arrow().column("rid").to_pylist()


@pytest.mark.parametrize("n", [0, 1, 3, 10_000])
@pytest.mark.parametrize("na_position", ["first", "last"])
def test_take_without_partition_in_exact_order(engine, n, na_position):
    t = _take_table(5000, 2)
    for sorts in (OrderedDict([("v", False), ("w", True)]), OrderedDict([("s", True), ("kf", False), ("rid", False)])):
        exp = O.take(t, n, sorts, na_position, []).column("rid").to_pylist()
        assert _take(engine, t, n, sorts, na_position, None) == exp, dict(sorts)


@pytest.mark.parametrize("n", [0, 1, 3, 10_000])
@pytest.mark.parametrize("by", [["kf"], ["k"], ["kf", "s"]])
@pytest.mark.parametrize("na_position", ["first", "last"])
def test_take_per_partition_as_multiset(engine, n, by, na_position):
    t = _take_table(5000, 3)
    sorts = OrderedDict([("w", False), ("v", True)])
    exp = O.take(t, n, sorts, na_position, by).column("rid").to_pylist()
    got = _take(engine, t, n, sorts, na_position, by)
    assert len(got) == len(exp) and Counter(got) == Counter(exp)


@pytest.mark.parametrize("na_position", ["first", "last"])
@pytest.mark.parametrize("key", ["k", "kf"])
def test_take_with_a_partition_key_relisted_desc(engine, key, na_position):
    """A partition key that is also the first presort column keeps the presort's direction: the output is in the
    reference's sorted order exactly."""
    t = _take_table(5000, 4)
    sorts = OrderedDict([(key, False), ("v", True), ("w", False)])
    exp = O.take(t, 2, sorts, na_position, [key]).column("rid").to_pylist()
    assert _take(engine, t, 2, sorts, na_position, [key]) == exp


# ---- 5. the logical partitions fa.transform hands to a function ------------------------------------------------------
def _oracle_groups(t: pa.Table, keys, presort) -> set:
    sorts = OrderedDict((k, True) for k in keys)
    sorts.update(presort)
    st = t.take(pa.array(O.argsort(t, sorts, "last")))
    off = O.logical_offsets(st, keys)
    rid = np.asarray(st.column("rid"))
    return {tuple(rid[a:b].tolist()) for a, b in zip(off[:-1], off[1:])}


@pytest.mark.parametrize("algo,num", [("hash", 0), ("hash", 16), ("hash", K.MAX_PARTITIONS + 976), ("even", 4),
                                      ("rand", 3)])
@pytest.mark.parametrize("keys", [["kf"], ["kf", "k"]])
def test_transform_logical_partitions_are_oracle_groups(engine, keys, algo, num):
    t = _take_table(20_000, 5)
    presort = OrderedDict([("w", False), ("v", True)])
    seen = []

    def record(tb: B200Table) -> B200Table:
        seen.append((tb.logical_offsets.cpu().numpy(), tb.column("rid").cpu().numpy()))
        return tb

    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    fa.transform(df, record, schema="*", partition=PartitionSpec(by=keys, presort=_presort_str(presort), algo=algo,
                                                                  num=num), engine=engine, as_fugue=True)
    assert len(seen) == 1
    off, rid = seen[0]
    got = [tuple(rid[a:b].tolist()) for a, b in zip(off[:-1], off[1:])]
    exp = _oracle_groups(t, keys, presort)
    assert len(got) == len(exp)  # one logical partition per oracle group, none split in two
    assert set(got) == exp       # same rows, in the oracle's presort order


def test_transform_host_function_runs_once_per_oracle_group(engine):
    t = _take_table(3000, 6)
    calls = []

    def record(df: pd.DataFrame) -> pd.DataFrame:
        calls.append(frozenset(df["rid"].tolist()))
        return df[["rid"]]

    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    fa.transform(df, record, schema="rid:long", partition=PartitionSpec(by=["kf", "k"], presort="w desc"), engine=engine,
                 as_fugue=True)
    exp = {frozenset(g) for g in _oracle_groups(t, ["kf", "k"], OrderedDict())}
    assert len(calls) == len(exp)
    assert set(calls) == exp


# ---- 6. window maps on float keys and presort columns -----------------------------------------------------------------
def _window_input(n: int, seed: int) -> pa.Table:
    rng = np.random.default_rng(seed)
    t = _input(n, seed)
    kf = pa.array(KEY_F[rng.integers(0, len(KEY_F), n)], mask=rng.random(n) < 0.05)
    q = pa.array(np.array([0.0, -0.0, np.nan, NEG_NAN, 0.5, -0.5, np.inf])[rng.integers(0, 7, n)],
                 mask=rng.random(n) < 0.1)
    t = t.set_column(t.schema.get_field_index("kf"), "kf", kf)
    return t.set_column(t.schema.get_field_index("q"), "q", q)


@pytest.mark.parametrize("keys,presort", [(["kf"], OrderedDict(q=True)), (["kf"], OrderedDict(q=False)),
                                          (["kf", "k2"], OrderedDict([("q", True), ("p", False)])),
                                          (["k"], OrderedDict(q=True))])
def test_window_functions_on_float_keys_and_presort(engine, keys, presort):
    t = _window_input(3000, 7)
    _check(engine, t, keys, presort, ALL, ALL_SCHEMA)


# ---- 7. aggregate / distinct on a float key ---------------------------------------------------------------------------
def _norm(x):
    if x is None or (isinstance(x, float) and np.isnan(x)):
        return None
    return x + 0.0 if isinstance(x, float) else x


def _agg_table(n: int, seed: int) -> pa.Table:
    rng = np.random.default_rng(seed)
    return pa.table({"kf": pa.array(KEY_F[rng.integers(0, len(KEY_F), n)], mask=rng.random(n) < 0.1),
                     "j": pa.array(rng.integers(0, 3, n)),
                     "v": pa.array(rng.integers(-100, 100, n))})


@pytest.mark.parametrize("keys", [["kf"], ["kf", "j"]])
def test_aggregate_float_key_matches_pandas_groupby(engine, keys):
    t = _agg_table(50_000, 8)
    df = B200DataFrame(B200Table.from_arrow(t, DEV))
    res = engine.aggregate(df, PartitionSpec(by=keys), [f.sum(col("v")).alias("s"), f.count(all_cols()).alias("c")])
    got = res.as_arrow().to_pylist()
    pdf = t.to_pandas()
    exp = pdf.groupby(keys, dropna=False).agg(s=("v", "sum"), c=("v", "size")).reset_index()
    assert len(got) == len(exp)
    g = {tuple(_norm(r[k]) for k in keys): (r["s"], r["c"]) for r in got}
    e = {tuple(_norm(x) for x in row[:len(keys)]): (int(row[-2]), int(row[-1]))
         for row in exp.itertuples(index=False, name=None)}
    assert g == e


@pytest.mark.parametrize("cols", [["kf"], ["kf", "j"]])
def test_distinct_float_key_gives_one_row_for_nan_and_null(engine, cols):
    t = _agg_table(20_000, 9).select(cols)
    res = fa.distinct(B200DataFrame(B200Table.from_arrow(t, DEV)), engine=engine, as_fugue=True).as_arrow()
    got = [tuple(_norm(r[c]) for c in cols) for r in res.to_pylist()]
    exp = {tuple(_norm(x) for x in row) for row in zip(*[t.column(c).to_pylist() for c in cols])}
    assert len(got) == len(exp) and set(got) == exp
