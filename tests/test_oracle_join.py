"""The join oracle (oracle/join.py) against a nested-loop join on small inputs with every special key, and against
pandas ``merge`` (through ``native_engine.join``) on finite data without NULLs.  Runs without a GPU."""
import math
from collections import Counter

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from oracle import join as oj
from oracle import native_engine as ora

INT64_MIN, INT64_MAX = -(2**63), 2**63 - 1
SPECIALS = np.array([0, -1, INT64_MIN, INT64_MAX, 1, 7], dtype=np.int64)


def _nested_loop(pk, pv, bk, bv, outer):
    pairs = []
    for i in range(len(pk)):
        hit = [j for j in range(len(bk)) if pv[i] and bv[j] and pk[i] == bk[j]]
        pairs += [(i, j) for j in hit] or ([(i, -1)] if outer else [])
    return pairs


@pytest.mark.parametrize("seed,np_,nb", [(0, 0, 5), (1, 5, 0), (2, 1, 1), (3, 40, 31), (4, 200, 150), (5, 300, 3)])
@pytest.mark.parametrize("outer", [False, True])
def test_pairs_match_nested_loop(seed, np_, nb, outer):
    rng = np.random.default_rng(seed)
    pk, bk = rng.choice(SPECIALS, np_), rng.choice(SPECIALS, nb)
    pv, bv = (rng.random(np_) > 0.25).astype(np.uint8), (rng.random(nb) > 0.25).astype(np.uint8)
    p, b = oj.join_pairs(pk, pv, bk, bv, outer)
    assert list(zip(p.tolist(), b.tolist())) == _nested_loop(pk, pv, bk, bv, outer)
    cnt = oj.probe_counts(pk, pv, bk, bv, outer)
    assert cnt.tolist() == [sum(1 for x in p if x == i) for i in range(np_)]
    m = oj.matched_build_rows(pk, pv, bk, bv)
    assert m.tolist() == [int(any(pv[i] and bv[j] and pk[i] == bk[j] for i in range(np_))) for j in range(nb)]


def test_pairs_without_validity_and_sorted_output():
    pk = np.array([INT64_MAX, -1, 3, INT64_MIN], dtype=np.int64)
    bk = np.array([3, INT64_MIN, 3, -1, INT64_MAX, 3], dtype=np.int64)
    p, b = oj.join_pairs(pk, None, bk, None, False)
    assert list(zip(p.tolist(), b.tolist())) == [(0, 4), (1, 3), (2, 0), (2, 2), (2, 5), (3, 1)]
    p, b = oj.join_pairs(pk, None, bk, np.zeros(6, np.uint8), True)
    assert list(zip(p.tolist(), b.tolist())) == [(0, -1), (1, -1), (2, -1), (3, -1)]


def test_pairs_millions_of_rows_are_fast():
    rng = np.random.default_rng(9)
    n = 4_000_000
    bk = rng.permutation(n).astype(np.int64)
    pk = rng.integers(0, 2 * n, n)
    p, b = oj.join_pairs(pk, None, bk, None, True)
    assert len(p) == n and np.array_equal(p, np.arange(n))
    hit = b >= 0
    assert np.array_equal(bk[b[hit]], pk[hit]) and np.array_equal(hit, pk < n)


# ---- engine level ---------------------------------------------------------------------------------------
def _nested_rows(left: pa.Table, right: pa.Table, how: str, on):
    """Row-by-row restatement with the rules spelled out: NULL / NaN keys never match, -0.0 == 0.0."""
    def key(r):
        vals = [r[k] for k in on]
        if any(v is None or (isinstance(v, float) and math.isnan(v)) for v in vals):
            return None
        return vals

    lr, rr = left.to_pylist(), right.to_pylist()
    rn = [c for c in right.column_names if c not in on]
    out = []
    hit_r = set()
    for a in lr:
        m = [j for j, b in enumerate(rr) if key(a) is not None and key(a) == key(b)]
        if how in ("semi", "anti"):
            if bool(m) == (how == "semi"):
                out.append(list(a.values()))
            continue
        hit_r |= set(m)
        out += [list(a.values()) + [rr[j][c] for c in rn] for j in m]
        if not m and how in ("left_outer", "full_outer"):
            out.append(list(a.values()) + [None] * len(rn))
    if how in ("right_outer", "full_outer"):
        for j, b in enumerate(rr):
            if j not in hit_r:
                out.append([b[c] if c in on else None for c in left.column_names] + [b[c] for c in rn])
    return Counter(tuple(oj.canon(v) for v in r) for r in out)


def _tables(seed, n1, n2):
    rng = np.random.default_rng(seed)
    fpool = np.array([0.0, -0.0, 1.5, np.nan, -np.inf, np.inf])
    ipool = SPECIALS

    def t(n, tag):
        k = rng.choice(ipool, n)
        f = rng.choice(fpool, n)
        s = rng.choice(np.array(["a", "bb", "", "zz"]), n).tolist()
        return pa.table({"k": pa.array(k, mask=rng.random(n) < 0.2), "f": pa.array(f, mask=rng.random(n) < 0.1),
                         "s": pa.array(s, mask=rng.random(n) < 0.1),
                         tag: pa.array(np.arange(n) + (1000 if tag == "r" else 0))})
    return t(n1, "l"), t(n2, "r")


@pytest.mark.parametrize("how", ["inner", "left_outer", "right_outer", "full_outer", "semi", "anti", "cross"])
@pytest.mark.parametrize("on", [["k"], ["f"], ["s"], ["k", "f"], ["f", "s"]])
def test_rows_match_nested_loop(how, on):
    left, right = _tables(len(on) * 7 + len(how), 60, 45)
    right = right.select([c for c in right.column_names if c in on or c == "r"])
    if how == "cross":
        right = right.rename_columns(["x_" + c for c in right.column_names])
        on = []
    got = oj.join_rows(left, right, how, on)
    assert got == _nested_rows(left, right, how, on) and sum(got.values()) > 0
    assert {len(r) for r in got} == {len(oj.output_names(left, right, how, on))}


def test_rows_special_int64_keys_are_exact_and_right_keys_fill_in():
    left = pa.table({"k": pa.array([INT64_MAX, INT64_MAX - 1, None, -1], pa.int64()), "a": [1, 2, 3, 4]})
    right = pa.table({"k": pa.array([INT64_MAX, INT64_MIN, None, 0], pa.int64()), "b": [10, 20, 30, 40]})
    assert oj.join_rows(left, right, "inner", ["k"]) == Counter({(INT64_MAX, 1, 10): 1})
    assert oj.join_rows(left, right, "right_outer", ["k"]) == Counter(
        {(INT64_MAX, 1, 10): 1, (INT64_MIN, None, 20): 1, (None, None, 30): 1, (0, None, 40): 1})


def test_rows_nan_never_matches_and_negative_zero_does():
    left = pa.table({"k": [float("nan"), -0.0, 2.0], "a": [1, 2, 3]})
    right = pa.table({"k": [float("nan"), 0.0, 2.0], "b": [10, 20, 30]})
    got = oj.join_rows(left, right, "inner", ["k"])
    assert got == Counter({(oj.canon(-0.0), 2, 20): 1, (oj.canon(2.0), 3, 30): 1})
    assert oj.join_rows(left, right, "anti", ["k"]) == Counter({(oj.canon(float("nan")), 1): 1})


@pytest.mark.parametrize("how", ["inner", "left_outer", "right_outer", "full_outer", "semi", "anti"])
def test_rows_match_pandas_on_finite_data(how):
    rng = np.random.default_rng(31)
    n1, n2 = 400, 300
    l = pd.DataFrame({"key": rng.integers(0, 150, n1), "k2": rng.integers(0, 3, n1),
                      "lv": np.round(rng.standard_normal(n1), 3)})
    r = pd.DataFrame({"key": rng.integers(100, 260, n2), "k2": rng.integers(0, 3, n2),
                      "rv": np.round(rng.standard_normal(n2), 3)})
    for on in (["key"], ["key", "k2"]):
        rr = r if on == ["key", "k2"] else r.drop(columns=["k2"])
        exp = ora.join(l, rr, how, on)
        got = oj.join_rows(pa.Table.from_pandas(l, preserve_index=False), pa.Table.from_pandas(rr, preserve_index=False),
                           how, on)
        names = oj.output_names(pa.Table.from_pandas(l), pa.Table.from_pandas(rr), how, on)
        assert names == list(exp.columns)
        want = Counter()
        for row in exp.itertuples(index=False):
            vals = [None if (isinstance(v, float) and math.isnan(v)) else v for v in row]
            vals = [int(v) if c in ("key", "k2") and v is not None else v for c, v in zip(names, vals)]
            want[tuple(oj.canon(float(v)) if c in ("lv", "rv") and v is not None else v
                       for c, v in zip(names, vals))] += 1
        assert got == want
