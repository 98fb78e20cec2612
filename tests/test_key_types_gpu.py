"""The keyed operations above the sort on every key type, against exact CPU references: ``engine.aggregate``, the set
operations, ``engine.join``, the logical partitions ``fa.transform`` hands to a device function, a window map and a
pandas host function, ``fa.take`` per partition, and the public ``engine.repartition``.

Every type runs alone and as a two-column key with a string and with a float64 column (the 64-bit row hash with the
MIN/MAX collision check of ``aggregate``, or ``join._verify``).  Groups and matches follow DESIGN §7d: a NaN of either
sign is NULL and -0.0 equals 0.0 for float16, float32 and float64 alike; ``oracle/keys.py`` states the canonical key.
Value pools and their edges are in ``_key_types.py``.  Temporal columns reach the references that work on Python
values as their integer storage, since most of the pool's extremes have no ``datetime``."""
from collections import Counter, OrderedDict

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from _key_types import TYPES, key_array
from fugue_b200 import api as fa
from fugue_b200 import join as J
from fugue_b200 import kernels as K
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import all_cols, col, functions as f
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.partition import PartitionSpec
from fugue_b200.table import B200Table
from oracle import hash_partition as hp
from oracle import join as oj
from oracle import sort as O
from oracle import window as W
from oracle.keys import canonical_rows

DEV = torch.device("cuda", 0)
KEY_SETS = [["k"], ["k", "ks"], ["k", "kf"]]
NUMERIC = [t for t in TYPES if t != "string"]  # types whose storage numpy can hash like hash_pandas_object


@pytest.fixture(scope="module")
def engine():
    return fa.make_execution_engine("b200")


def _strings(rng, n: int, pool) -> pa.Array:
    return pa.array(list(np.array(pool, dtype=object)[rng.integers(0, len(pool), n)]), mask=rng.random(n) < 0.1,
                    type=pa.string())


def _table(name: str, n: int, seed: int, host_safe: bool = False) -> pa.Table:
    rng = np.random.default_rng([seed, TYPES.index(name)])
    return pa.table({
        "rid": pa.array(np.arange(n, dtype=np.int64)),
        "k": key_array(name, n, rng, 0.1, host_safe),
        "ks": _strings(rng, n, ["x", "yy", "", "é"]),
        "kf": key_array("float64", n, rng, 0.1),
        "v": pa.array(rng.integers(-1000, 1000, n), mask=rng.random(n) < 0.2),
    })


def _df(t: pa.Table) -> B200DataFrame:
    return B200DataFrame(B200Table.from_arrow(t, DEV))


def _ints(t: pa.Table) -> pa.Table:
    """Temporal columns viewed as their integer storage, for the references that read Python values."""
    cols = []
    for c in t.columns:
        c = c.combine_chunks()
        if pa.types.is_temporal(c.type):
            c = c.view(pa.int32() if c.type.bit_width == 32 else pa.int64())
        cols.append(c)
    return pa.table(cols, names=t.column_names)


def _types_kept(got: pa.Table, t: pa.Table, names) -> None:
    assert [got.schema.field(c).type for c in names] == [t.schema.field(c).type for c in names]


def _groups(t: pa.Table, keys) -> dict:
    """Canonical key tuple -> its rows, in input order."""
    g: dict = {}
    for i, k in enumerate(canonical_rows(t, keys)):
        g.setdefault(k, []).append(i)
    return g


# ---- a. engine.aggregate ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("region", [False, True], ids=["whole", "region"])
@pytest.mark.parametrize("name", TYPES)
def test_aggregate(engine, monkeypatch, name, region):
    if region:  # the hash-partitioned region path of the group-by
        monkeypatch.setattr(K, "GROUPBY_PARTITION_MIN_ROWS", 64)
    t = _table(name, 4000, 1)
    v = t.column("v").to_pylist()
    aggs = [f.count(all_cols()).alias("n"), f.sum(col("v")).alias("s"), f.min(col("v")).alias("lo"),
            f.max(col("v")).alias("hi"), f.first(col("v")).alias("fv")]
    for keys in KEY_SETS:
        got = engine.aggregate(_df(t), PartitionSpec(by=keys), aggs).native.to_arrow()
        _types_kept(got, t, keys)
        exp = {}
        for k, rows in _groups(t, keys).items():
            vs = [v[i] for i in rows if v[i] is not None]
            exp[k] = (len(rows), sum(vs) if vs else None, min(vs, default=None), max(vs, default=None),
                      vs[0] if vs else None)
        gk = canonical_rows(got, keys)
        assert len(gk) == len(set(gk)) == len(exp), (keys, len(gk), len(exp))  # no group split or merged
        res = dict(zip(gk, zip(*[got.column(c).to_pylist() for c in ("n", "s", "lo", "hi", "fv")])))
        assert res == exp, keys


# ---- b. set operations ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("region", [False, True], ids=["whole", "region"])
@pytest.mark.parametrize("name", TYPES)
def test_set_operations(engine, monkeypatch, name, region):
    if region:
        monkeypatch.setattr(K, "GROUPBY_PARTITION_MIN_ROWS", 64)
    t = _table(name, 1600, 2)
    rng = np.random.default_rng([3, TYPES.index(name)])
    a = t.slice(0, 1000)
    # b: the last 400 rows of a, then rows whose strings a never saw, first seen in another order: the two string
    # dictionaries differ and concat_tables has to merge them
    extra = _table(name, 600, 4).set_column(2, "ks", _strings(rng, 600, ["new", "é", "q", "x"]))
    b = pa.concat_tables([t.slice(600, 400), extra]).combine_chunks()
    b_null = b.set_column(2, "ks", pa.array([None] * b.num_rows, type=pa.string()))
    for cols in (["k"], ["k", "ks", "kf"]):
        ra = set(canonical_rows(a, cols))
        for other in (b, b_null):
            rb = set(canonical_rows(other, cols))
            da, db = _df(a.select(cols)), _df(other.select(cols))
            for op, exp in (("distinct", ra), ("union", ra | rb), ("intersect", ra & rb), ("subtract", ra - rb)):
                if op == "distinct":
                    out = fa.distinct(da, engine=engine, as_fugue=True)
                else:
                    out = getattr(fa, op)(da, db, engine=engine, as_fugue=True)
                got_t = out.as_arrow()
                _types_kept(got_t, t, cols)
                got = canonical_rows(got_t, cols)
                assert len(got) == len(set(got)) and set(got) == exp, (op, cols, other is b_null)


# ---- c. engine.join -------------------------------------------------------------------------------------------------
HOWS = ["inner", "left_outer", "right_outer", "full_outer", "semi", "anti"]


def _join_tables(name: str, seed: int, n1: int = 400, n2: int = 300):
    rng = np.random.default_rng([seed, TYPES.index(name)])
    left = pa.table({"k": key_array(name, n1, rng), "ks": _strings(rng, n1, ["x", "yy", "", "é"]),
                     "kf": key_array("float64", n1, rng), "lrow": pa.array(np.arange(n1))})
    right = pa.table({"rs": _strings(rng, n2, ["a", "b"]), "k": key_array(name, n2, rng),
                      "ks": _strings(rng, n2, ["é", "q", "x", ""]), "kf": key_array("float64", n2, rng),
                      "rrow": pa.array(np.arange(n2))})
    return left, right


@pytest.mark.parametrize("radix", [False, True], ids=["default", "radix"])
@pytest.mark.parametrize("name", TYPES)
def test_join(engine, monkeypatch, name, radix):
    if radix:
        monkeypatch.setattr(J, "RADIX_JOIN_MIN_ROWS", 200)
    left, right = _join_tables(name, 5)
    for on in KEY_SETS:
        lt, rt = left.select(on + ["lrow"]), right.select(["rs"] + on + ["rrow"])
        ldf, rdf = _df(lt), _df(rt)
        for how in HOWS:
            got = engine.join(ldf, rdf, how, on).native.to_arrow()
            names = oj.output_names(lt, rt, how, on)
            assert got.column_names == names
            _types_kept(got, lt, on)
            exp = oj.join_rows(_ints(lt), _ints(rt), how, on)
            res = oj.rows_of(_ints(got))
            assert res == exp, (how, on, sum(res.values()), sum(exp.values()), list((res - exp).items())[:3],
                                list((exp - res).items())[:3])


# ---- d. fa.transform: logical partitions of a device function, and a window map --------------------------------------
def _presort_str(sorts) -> str:
    return ",".join(f"{k} {'asc' if a else 'desc'}" for k, a in sorts.items())


PRESORT = OrderedDict([("v", False), ("rid", True)])


def _oracle_groups(t: pa.Table, keys, presort) -> set:
    sorts = OrderedDict((k, True) for k in keys)
    sorts.update(presort)
    st = t.take(pa.array(O.argsort(t, sorts, "last")))
    off = O.logical_offsets(st, keys)
    rid = np.asarray(st.column("rid"))
    return {tuple(rid[a:b].tolist()) for a, b in zip(off[:-1], off[1:])}


@pytest.mark.parametrize("name", TYPES)
def test_transform_logical_partitions(engine, name):
    t = _table(name, 3000, 6)
    df = _df(t)
    for keys in KEY_SETS:
        exp = _oracle_groups(t, keys, PRESORT)
        assert len(exp) == len(set(canonical_rows(t, keys)))  # the sort reference has the canonical classes
        for algo, num in (("hash", 0), ("hash", 16), ("hash", K.MAX_PARTITIONS + 976), ("even", 4)):
            seen = []

            def record(tb: B200Table) -> B200Table:
                seen.append((tb.logical_offsets.cpu().numpy(), tb.column("rid").cpu().numpy()))
                return tb

            fa.transform(df, record, schema="*", partition=PartitionSpec(by=keys, presort=_presort_str(PRESORT),
                                                                          algo=algo, num=num),
                         engine=engine, as_fugue=True)
            assert len(seen) == 1
            off, rid = seen[0]
            got = [tuple(rid[a:b].tolist()) for a, b in zip(off[:-1], off[1:])]
            assert len(got) == len(exp), (keys, algo, num)  # one logical partition per group, none split in two
            assert set(got) == exp, (keys, algo, num)       # same rows, in presort order


WINDOW = [f.row_number().alias("rn"), f.sum(col("v")).over(running=True).alias("rsv"),
          f.count(all_cols()).over().alias("cnt")]


@pytest.mark.parametrize("name", TYPES)
def test_window_map(engine, name):
    t = _table(name, 2000, 7)
    for keys in KEY_SETS:
        res = fa.transform(_df(t), ColumnMap(col("rid"), *WINDOW), schema="rid:long,rn:long,rsv:long,cnt:long",
                           partition=PartitionSpec(by=keys, presort=_presort_str(PRESORT)), engine=engine,
                           as_fugue=True).as_arrow()
        assert res.num_rows == t.num_rows
        order = np.argsort(np.asarray(res.column("rid")))
        exp = W.window_map(_ints(t), keys, PRESORT, [col("rid")] + WINDOW)
        for c in res.column_names:
            assert [res.column(c)[int(i)].as_py() for i in order] == exp[c], (keys, c)


# ---- e. fa.transform with a pandas host function ----------------------------------------------------------------------
@pytest.mark.parametrize("name", TYPES)
def test_transform_host_function_once_per_group(engine, name):
    """With num=1 pandas groups the whole table, so keys that the hash would put in different physical partitions
    (uint64 2^63 - 1 and 2^63, which pandas holds as one float64 when the column has NULLs) meet too."""
    t = _table(name, 1000, 8, host_safe=True)
    for keys in KEY_SETS:
        exp = {frozenset(rows) for rows in _groups(t, keys).values()}
        for num in (0, 1):
            calls = []

            def record(df: pd.DataFrame) -> pd.DataFrame:
                calls.append(frozenset(df["rid"].tolist()))
                return df[["rid"]]

            fa.transform(_df(t), record, schema="rid:long", partition=PartitionSpec(by=keys, num=num), engine=engine,
                         as_fugue=True)
            assert len(calls) == len(exp), (keys, num)  # exactly once per group
            assert set(calls) == exp, (keys, num)


# ---- f. fa.take per partition ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", TYPES)
def test_take_per_partition(engine, name):
    t = _table(name, 3000, 9)
    sorts = OrderedDict(v=False)
    for keys in KEY_SETS:
        for na_position in ("first", "last"):
            exp = O.take(t, 2, sorts, na_position, keys).column("rid").to_pylist()
            got = fa.take(_df(t), 2, presort=_presort_str(sorts), na_position=na_position, partition=dict(by=keys),
                          engine=engine, as_fugue=True).as_arrow()
            _types_kept(got, t, t.column_names)
            assert Counter(got.column("rid").to_pylist()) == Counter(exp), (keys, na_position)


# ---- g. the public repartition: raw bits, like hash_pandas_object ------------------------------------------------------
@pytest.mark.parametrize("name", NUMERIC)
def test_public_repartition_hashes_raw_bits(engine, name):
    t = _table(name, 3000, 10)
    bt = B200Table.from_arrow(t, DEV)
    for keys in (["k"], ["k", "kf"]):
        cols = [bt.column(k).cpu().numpy() for k in keys]  # the stored bits, at the storage width
        valid = [None if bt.valid[bt.schema.index_of_key(k)] is None else
                 bt.valid[bt.schema.index_of_key(k)].cpu().numpy() for k in keys]
        for num in (16, K.MAX_PARTITIONS + 976):
            exp = hp.partition_ids(cols, num, valid)
            order, exp_off = hp.stable_partition(exp, num)
            res = engine.repartition(B200DataFrame(bt), PartitionSpec(by=keys, num=num)).native
            assert np.array_equal(res.offsets.cpu().numpy(), exp_off), (keys, num)
            assert np.array_equal(res.column("rid").cpu().numpy(), order), (keys, num)  # stable, too
