"""oracle/sort.py (the reference for the device sort, logical partitions and take) against pandas and plain Python.
Runs without a GPU."""
import functools
import math
from collections import Counter, OrderedDict

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from oracle import sort as O

NEG_NAN = np.array([-0x0007FFFF00000001], dtype=np.int64).view(np.float64)[0]  # sign bit set, with a payload


def _floats(n: int, rng) -> np.ndarray:
    special = np.array([0.0, -0.0, 1.0, -1.0, np.inf, -np.inf, 5e-324, -5e-324, np.nan, NEG_NAN, 2.5])
    return special[rng.integers(0, len(special), n)]


def _table(n: int, seed: int) -> pa.Table:
    rng = np.random.default_rng(seed)
    m = lambda q: rng.random(n) < q  # noqa: E731
    return pa.table({
        "i": pa.array(rng.choice(np.array([-(2**63), 2**63 - 1, 2**63 - 2, -1, 0, 1, 7]), n), mask=m(0.2)),
        "u": pa.array(rng.choice(np.array([0, 1, 2**63, 2**64 - 1, 2**63 - 1], dtype=np.uint64), n), mask=m(0.2)),
        "f": pa.array(_floats(n, rng), mask=m(0.15)),
        "g": pa.array(_floats(n, rng).astype(np.float32), mask=m(0.15)),
        "s": pa.array(list(np.array(["", "b", "a", "é", "Z", "ab"], dtype=object)[rng.integers(0, 6, n)]),
                      mask=m(0.2), type=pa.string()),
        "b": pa.array(rng.random(n) < 0.5, mask=m(0.2)),
        "d": pa.array(rng.integers(-3, 3, n).astype(np.int32), mask=m(0.2)).cast(pa.date32()),
        "t": pa.array(rng.integers(-3, 3, n), mask=m(0.2)).cast(pa.timestamp("us")),
    })


def _py(table: pa.Table, name: str) -> list:
    """Python values under the rule: NaN -> None, -0.0 -> 0.0, dates / timestamps as their storage."""
    a = table.column(name).combine_chunks()
    if pa.types.is_temporal(a.type):
        a = a.view(pa.int32() if a.type.bit_width == 32 else pa.int64())
    out = []
    for x in a.to_pylist():
        if isinstance(x, float):
            x = None if math.isnan(x) else x + 0.0  # -0.0 + 0.0 == 0.0
        out.append(x)
    return out


def _reference_argsort(table: pa.Table, sorts, na_position) -> list:
    cols = {k: _py(table, k) for k in sorts}

    def cmp(a: int, b: int) -> int:
        for k, asc in sorts.items():
            x, y = cols[k][a], cols[k][b]
            if x is None or y is None:
                if x is None and y is None:
                    continue
                first = na_position == "first"
                return (-1 if first else 1) if x is None else (1 if first else -1)
            if x != y:
                return (-1 if x < y else 1) * (1 if asc else -1)
        return 0

    return sorted(range(table.num_rows), key=functools.cmp_to_key(cmp))  # sorted() is stable


def test_issue_example_float_keys():
    t = pa.table({"k": pa.array([0.0, -0.0, 1.0, np.nan, 0.0, NEG_NAN, -1.0, None], type=pa.float64())})
    assert O.argsort(t, OrderedDict(k=True), "last").tolist() == [6, 0, 1, 4, 2, 3, 5, 7]
    assert O.argsort(t, OrderedDict(k=True), "first").tolist() == [3, 5, 7, 6, 0, 1, 4, 2]
    assert O.argsort(t, OrderedDict(k=False), "last").tolist() == [2, 0, 1, 4, 6, 3, 5, 7]
    st = t.take(pa.array(O.argsort(t, OrderedDict(k=True), "last")))
    assert O.logical_offsets(st, ["k"]).tolist() == [0, 1, 4, 5, 8]
    assert O.take(t, 1, OrderedDict(), "last", ["k"]).num_rows == 4


@pytest.mark.parametrize("sorts", [OrderedDict(i=True), OrderedDict(u=False), OrderedDict(f=True), OrderedDict(g=False),
                                   OrderedDict(s=True), OrderedDict(b=False), OrderedDict(d=True), OrderedDict(t=False),
                                   OrderedDict([("s", False), ("f", True)]),
                                   OrderedDict([("b", True), ("i", False), ("u", True), ("g", True)])])
@pytest.mark.parametrize("na_position", ["first", "last"])
def test_argsort_matches_a_comparator_written_from_the_rule(sorts, na_position):
    t = _table(600, 1)
    got = O.argsort(t, sorts, na_position)
    assert got.tolist() == _reference_argsort(t, sorts, na_position)


@pytest.mark.parametrize("na_position", ["first", "last"])
@pytest.mark.parametrize("sorts", [OrderedDict(f=True), OrderedDict(f=False), OrderedDict(x=False),
                                   OrderedDict([("x", True), ("f", False)]), OrderedDict([("s", False), ("x", True)])])
def test_argsort_matches_pandas_stable_sort(sorts, na_position):
    rng = np.random.default_rng(2)
    n = 5000
    f = _floats(n, rng)
    f[rng.random(n) < 0.1] = np.nan
    pdf = pd.DataFrame({"f": f, "x": rng.integers(-50, 50, n),
                        "s": pd.Series(np.array(["a", "b", "é", ""], dtype=object)[rng.integers(0, 4, n)])})
    pdf.loc[rng.random(n) < 0.1, "s"] = None
    t = pa.Table.from_pandas(pdf, preserve_index=False)
    exp = pdf.sort_values(list(sorts), ascending=list(sorts.values()), kind="stable", na_position=na_position).index
    assert O.argsort(t, sorts, na_position).tolist() == exp.tolist()


def test_argsort_is_exact_near_2_63():
    vals = [2**63 - 1, 2**63 - 2, -(2**63), -(2**63) + 1, None, 0]
    t = pa.table({"i": pa.array(vals, type=pa.int64()),
                  "u": pa.array([2**64 - 1, 2**64 - 2, 2**63, 2**63 - 1, None, 0], type=pa.uint64())})
    assert O.argsort(t, OrderedDict(i=True)).tolist() == [2, 3, 5, 1, 0, 4]
    assert O.argsort(t, OrderedDict(u=False), "first").tolist() == [4, 0, 1, 2, 3, 5]


@pytest.mark.parametrize("keys", [["f"], ["g"], ["s"], ["i", "f"], ["b", "d", "s"], ["u", "t"]])
def test_groups_match_pandas_groupby_dropna_false(keys):
    t = _table(2000, 3)
    gid = O.group_ids(t, keys)
    pdf = pd.DataFrame({k: pd.Series(_py(t, k), dtype=object) for k in keys})
    for k in keys:  # None and NaN are one missing value for pandas' grouping
        if pdf[k].map(lambda x: isinstance(x, float)).any():
            pdf[k] = pdf[k].astype(float)
    ng = pdf.groupby(keys, dropna=False, sort=False).ngroup().to_numpy()
    # the same partition of the rows: a bijection between the two numberings
    pairs = set(zip(gid.tolist(), ng.tolist()))
    assert len(pairs) == len(set(gid.tolist())) == len(set(ng.tolist()))
    st = t.take(pa.array(O.argsort(t, OrderedDict((k, True) for k in keys))))
    assert len(O.logical_offsets(st, keys)) - 1 == len(pairs)


@pytest.mark.parametrize("n", [0, 1, 3, 10_000])
@pytest.mark.parametrize("by", [["f"], ["s", "b"]])
def test_take_matches_pandas_groupby_head(n, by):
    t = _table(3000, 4)
    sorts = OrderedDict([("i", False), ("g", True)])
    got = O.take(t, n, sorts, "first", by)
    pdf = pd.DataFrame({k: pd.Series(_py(t, k), dtype=object) for k in t.column_names})
    pdf["f"] = pdf["f"].astype(float)
    pdf["rid"] = np.arange(t.num_rows)
    srt = pdf.iloc[_reference_argsort(t, sorts, "first")]
    exp = srt.groupby(by, dropna=False).head(n)["rid"].tolist()
    rid = pa.array(np.arange(t.num_rows))
    got_rid = O.take(t.append_column("rid", rid), n, sorts, "first", by).column("rid").to_pylist()
    assert got.num_rows == len(exp)
    assert Counter(got_rid) == Counter(exp)


def test_take_without_partition_is_the_sorted_prefix():
    t = _table(500, 5)
    t = t.append_column("rid", pa.array(np.arange(t.num_rows)))
    sorts = OrderedDict([("s", True), ("f", False)])
    order = O.argsort(t, sorts, "last")
    for n in (0, 1, 7, 1000):
        assert O.take(t, n, sorts, "last", []).column("rid").to_pylist() == order[:n].tolist()
