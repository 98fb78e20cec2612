"""K7 hash join vs the reference's literal truth tables (fugue_test/execution_suite.py:366-543)
and the pandas oracle on random data."""
import numpy as np
import pandas as pd
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import api as fa
from fugue_b200.dataframe import df_eq
from fugue_b200.schema import SchemaError
from oracle import native_engine as ora


@pytest.fixture(scope="module")
def e():
    return fa.make_execution_engine("b200")


def test__join_cross(e):
    a = fa.as_fugue_engine_df(e, [[1, 2], [3, 4]], "a:int,b:int")
    b = fa.as_fugue_engine_df(e, [[6], [7]], "c:int")
    c = fa.join(a, b, how="Cross", engine=e)
    df_eq(c, [[1, 2, 6], [1, 2, 7], [3, 4, 6], [3, 4, 7]], "a:int,b:int,c:int", throw=True)
    b = fa.as_fugue_engine_df(e, [], "c:int")
    df_eq(fa.cross_join(a, b, engine=e), [], "a:int,b:int,c:int", throw=True)


def test__join_inner(e):
    a = fa.as_fugue_engine_df(e, [[1, 2], [3, 4]], "a:int,b:int")
    b = fa.as_fugue_engine_df(e, [[6, 1], [2, 7]], "c:int,a:int")
    c = fa.join(a, b, how="INNER", on=["a"], engine=e)
    df_eq(c, [[1, 2, 6]], "a:int,b:int,c:int", throw=True)
    c = fa.inner_join(b, a, engine=e)
    df_eq(c, [[6, 1, 2]], "c:int,a:int,b:int", throw=True)
    a = fa.as_fugue_engine_df(e, [], "a:int,b:int")
    b = fa.as_fugue_engine_df(e, [], "c:int,a:int")
    df_eq(fa.join(a, b, how="INNER", on=["a"], engine=e), [], "a:int,b:int,c:int", throw=True)


def test_join_multiple(e):
    a = fa.as_fugue_engine_df(e, [[1, 2], [3, 4]], "a:int,b:int")
    b = fa.as_fugue_engine_df(e, [[1, 20], [3, 40]], "a:int,c:int")
    c = fa.as_fugue_engine_df(e, [[1, 200], [3, 400]], "a:int,d:int")
    d = fa.inner_join(a, b, c, engine=e)
    df_eq(d, [[1, 2, 20, 200], [3, 4, 40, 400]], "a:int,b:int,c:int,d:int", throw=True)


def test__join_outer(e):
    a = fa.as_fugue_engine_df(e, [], "a:int,b:int")
    b = fa.as_fugue_engine_df(e, [], "c:str,a:int")
    df_eq(fa.left_outer_join(a, b, engine=e), [], "a:int,b:int,c:str", throw=True)
    a = fa.as_fugue_engine_df(e, [[1, "2"], [3, "4"]], "a:int,b:str")
    b = fa.as_fugue_engine_df(e, [["6", 1], ["2", 7]], "c:str,a:int")
    c = fa.join(a, b, how="left_OUTER", on=["a"], engine=e)
    df_eq(c, [[1, "2", "6"], [3, "4", None]], "a:int,b:str,c:str", throw=True)
    c = fa.join(b, a, how="left_outer", on=["a"], engine=e)
    df_eq(c, [["6", 1, "2"], ["2", 7, None]], "c:str,a:int,b:str", throw=True)
    b = fa.as_fugue_engine_df(e, [[6, 1], [2, 7]], "c:double,a:int")
    c = fa.join(a, b, how="left_OUTER", on=["a"], engine=e)
    df_eq(c, [[1, "2", 6.0], [3, "4", None]], "a:int,b:str,c:double", throw=True)
    b = fa.as_fugue_engine_df(e, [["6", 1], ["2", 7]], "c:str,a:int")
    c = fa.join(a, b, how="right_outer", on=["a"], engine=e)
    df_eq(c, [[1, "2", "6"], [7, None, "2"]], "a:int,b:str,c:str", throw=True)
    c = fa.join(a, b, how="full_outer", on=["a"], engine=e)
    df_eq(c, [[1, "2", "6"], [3, "4", None], [7, None, "2"]], "a:int,b:str,c:str", throw=True)
    # pandas-incompatible cases of the reference (int / bool payloads become NULL, not NaN)
    b = fa.as_fugue_engine_df(e, [[6, 1], [2, 7]], "c:int,a:int")
    c = fa.join(a, b, how="left_OUTER", on=["a"], engine=e)
    df_eq(c, [[1, "2", 6], [3, "4", None]], "a:int,b:str,c:int", throw=True)
    b = fa.as_fugue_engine_df(e, [[True, 1], [False, 7]], "c:bool,a:int")
    c = fa.join(b, a, how="left_outer", on=["a"], engine=e)
    df_eq(c, [[True, 1, "2"], [False, 7, None]], "c:bool,a:int,b:str", throw=True)


def test__join_semi_anti(e):
    a = fa.as_fugue_engine_df(e, [[1, 2], [3, 4]], "a:int,b:int")
    b = fa.as_fugue_engine_df(e, [[6, 1], [2, 7]], "c:int,a:int")
    df_eq(fa.join(a, b, how="semi", on=["a"], engine=e), [[1, 2]], "a:int,b:int", throw=True)
    df_eq(fa.semi_join(b, a, engine=e), [[6, 1]], "c:int,a:int", throw=True)
    df_eq(fa.join(a, b, how="anti", on=["a"], engine=e), [[3, 4]], "a:int,b:int", throw=True)
    df_eq(fa.anti_join(b, a, engine=e), [[2, 7]], "c:int,a:int", throw=True)
    b = fa.as_fugue_engine_df(e, [], "c:int,a:int")
    df_eq(fa.join(a, b, how="semi", on=["a"], engine=e), [], "a:int,b:int", throw=True)
    df_eq(fa.join(a, b, how="anti", on=["a"], engine=e), [[1, 2], [3, 4]], "a:int,b:int", throw=True)


def test__join_with_null_keys(e):
    # SQL will not match null values (two double key columns -> hashed surrogate key + verification)
    a = fa.as_fugue_engine_df(e, [[1, 2, 3], [4, None, 6]], "a:double,b:double,c:int")
    b = fa.as_fugue_engine_df(e, [[1, 2, 33], [4, None, 63]], "a:double,b:double,d:int")
    c = fa.join(a, b, how="INNER", engine=e)
    df_eq(c, [[1, 2, 3, 33]], "a:double,b:double,c:int,d:int", throw=True)


def test_join_errors(e):
    a = fa.as_fugue_engine_df(e, [[1, 2]], "a:int,b:int")
    b = fa.as_fugue_engine_df(e, [[1, 2]], "c:int,d:int")
    with pytest.raises(SchemaError):
        fa.inner_join(a, b, engine=e)
    with pytest.raises(ValueError):
        fa.join(a, a, how="outer", engine=e)
    with pytest.raises(ValueError):
        fa.join(a, a, how="magic", engine=e)
    with pytest.raises(SchemaError):
        fa.cross_join(a, a, engine=e)


@pytest.mark.parametrize("how", ["inner", "left_outer", "right_outer", "full_outer", "semi", "anti"])
def test_random_joins_match_oracle(e, how):
    rng = np.random.default_rng(11)
    n1, n2 = 50_000, 30_000
    l = pd.DataFrame({"key": rng.integers(0, 20_000, n1), "lv": rng.standard_normal(n1)})
    r = pd.DataFrame({"key": rng.integers(10_000, 40_000, n2), "rv": rng.standard_normal(n2)})
    l.loc[rng.integers(0, n1, 500), "key"] = np.nan          # NULL keys on both sides
    r.loc[rng.integers(0, n2, 500), "key"] = np.nan
    ls, rs = "key:double,lv:double", "key:double,rv:double"
    got = fa.join(fa.as_fugue_engine_df(e, l, ls), fa.as_fugue_engine_df(e, r, rs), how=how, engine=e)
    exp = ora.join(l, r, how)
    assert got.count() == len(exp), (got.count(), len(exp))
    df_eq(got, exp.values.tolist() if len(exp) < 200_000 else exp, None if len(exp) >= 200_000 else got.schema,
          throw=True)


def test_string_key_join(e):
    a = fa.as_fugue_engine_df(e, [["x", 1], ["y", 2], [None, 3], ["z", 4]], "k:str,a:int")
    b = fa.as_fugue_engine_df(e, [["y", 10], ["w", 20], ["x", 30], [None, 40], ["x", 50]], "k:str,b:int")
    df_eq(fa.inner_join(a, b, engine=e), [["x", 1, 30], ["x", 1, 50], ["y", 2, 10]], "k:str,a:int,b:int", throw=True)
    df_eq(fa.full_outer_join(a, b, engine=e),
          [["x", 1, 30], ["x", 1, 50], ["y", 2, 10], [None, 3, None], ["z", 4, None], ["w", None, 20],
           [None, None, 40]], "k:str,a:int,b:int", throw=True)


def test_full_size_properties_unique_build_side():
    """BASELINE config 5 shape per GPU (scaled to fit: 50 M x 50 M, unique build side)."""
    from fugue_b200 import kernels as K

    dev = torch.device("cuda", 0)
    n = 50_000_000
    g = torch.Generator(device=dev).manual_seed(2)
    lk = torch.randint(0, n, (n,), dtype=torch.int64, device=dev, generator=g)
    rk = torch.randperm(n, dtype=torch.int64, device=dev, generator=g)
    tab = K.JoinTable(rk, None)
    li, ri = tab.probe(lk, None, outer=False)
    assert li.numel() == n                                   # unique build side: one match per probe row
    assert torch.equal(li, torch.arange(n, device=dev))      # probe-row-major output
    assert torch.equal(rk[ri], lk)                           # every pair really matches
    assert int(tab.status[0]) == 0


@pytest.mark.parametrize("how", ["inner", "left_outer", "full_outer", "semi", "anti"])
def test_radix_join_path_matches_oracle(e, how, monkeypatch):
    """Force the radix (partition-first) path on a mid-size input and compare with pandas."""
    import fugue_b200.join as J

    monkeypatch.setattr(J, "RADIX_JOIN_MIN_ROWS", 1000)
    rng = np.random.default_rng(21)
    n1, n2 = 120_000, 90_000
    l = pd.DataFrame({"key": rng.integers(0, 60_000, n1), "lv": rng.standard_normal(n1), "li": np.arange(n1)})
    r = pd.DataFrame({"key": rng.integers(30_000, 100_000, n2), "rv": rng.standard_normal(n2)})
    l.loc[rng.integers(0, n1, 300), "key"] = np.nan
    r.loc[rng.integers(0, n2, 300), "key"] = np.nan
    got = fa.join(fa.as_fugue_engine_df(e, l, "key:double,lv:double,li:long"),
                  fa.as_fugue_engine_df(e, r, "key:double,rv:double"), how=how, engine=e)
    exp = ora.join(l, r, how)
    assert got.count() == len(exp)
    df_eq(got, exp.values.tolist(), got.schema, throw=True)


def test_radix_join_with_a_hot_key_on_the_build_side(e, monkeypatch):
    """>= 2M rows on both sides takes the radix (region) path; a skewed build side overflows its region of
    the hash table.  The build reports that and is redone with one region: no match may be lost, and each
    match must pair the right rows."""
    from _join_spy import Launches
    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.table import B200Table
    from oracle import join as oj

    launches = Launches(monkeypatch)
    rng = np.random.default_rng(5)
    n = 2_200_000
    bk = rng.integers(0, 50_000, n).astype("int64")
    bk[: n // 8] = 77                       # 12.5 % of the build rows share one key
    pk = rng.integers(0, 60_000, n).astype("int64")
    pk[:3] = 77
    left = B200DataFrame(B200Table("key:long,lv:long", [torch.from_numpy(pk).cuda(), torch.arange(n, device="cuda")]))
    right = B200DataFrame(B200Table("key:long,rv:long", [torch.from_numpy(bk).cuda(), torch.arange(n, device="cuda")]))
    uk, cnt = np.unique(bk, return_counts=True)
    res = e.join(left, right, "inner", ["key"]).native
    assert launches.path() == "fused-fallback", launches.calls
    expect_total = int(np.sum(cnt[np.searchsorted(uk, pk[np.isin(pk, uk)])]))
    assert res.num_rows == expect_total
    # the pairs of the first 1000 probe rows (275 k matches each for the hot key's three), build rows included
    lv, rv = res.column("lv").cpu().numpy(), res.column("rv").cpu().numpy()
    first = lv < 1000
    order = np.lexsort((rv[first], lv[first]))
    exp_l, exp_r = oj.join_pairs(pk[:1000], None, bk, None, False)
    assert np.array_equal(lv[first][order], exp_l) and np.array_equal(rv[first][order], exp_r)
    # semi / anti on the same data
    launches.clear()
    semi = e.join(left, right, "semi", ["key"]).native
    assert launches.path() == "table16-fallback", launches.calls
    assert np.array_equal(np.sort(semi.column("lv").cpu().numpy()), np.flatnonzero(np.isin(pk, uk)))
