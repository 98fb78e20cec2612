"""UPPER, LOWER, SUBSTR, TRIM, REPLACE, CONCAT and || on the H100: the per-entry transform (K12) entry for entry
against oracle/string_build.py, UPPER / LOWER over every scalar code point against pyarrow, a SUBSTR grid
against sqlite3, the deduplication against a Python dict (also with 3-bit hashes), whole engine calls against
oracle/expressions.py, the result cache, and one select over 100 M rows."""
import random
import sqlite3

import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.compute as pc
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from fugue_b200 import strings as ST
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import SelectColumns, col, null, functions as ff
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.partition import PartitionSpec
from fugue_b200.schema import Schema
from fugue_b200.table import B200Table
from oracle import expressions as ox
from oracle import string_build as osb

DEV = torch.device("cuda", 0)
ALPHABET = ["a", "b", "A", "B", " ", "\t", "é", "É", "ß", "ẞ", "İ", "ı", "€", "中", "😀", "𝄞", "Ω", "ω", "K", "-"]
S = col("s")
EXPRS = [ff.upper(S), ff.lower(S), ff.substr(S, 2), ff.substr(S, -3, 2), ff.substr(S, 0, 2), ff.substr(S, 4, -3),
         ff.trim(S), ff.ltrim(S), ff.rtrim(S), ff.trim(S, "a\tß"), ff.ltrim(S, "😀 "), ff.rtrim(S, ""),
         ff.replace(S, "a", "xyz"), ff.replace(S, "aa", "b"), ff.replace(S, "", "q"), ff.replace(S, "ß", ""),
         ff.concat(S, "-", S), ff.concat("<", S, None, ">"), ff.concat_strict(S, "|", S),
         ff.concat_strict(S, None), ff.substr(S, null()), ff.upper(ff.trim(ff.substr(S, 2))),
         ff.lower(ff.concat("Ä", S)), ff.concat(ff.substr(S, null()), "x"), ff.replace(ff.upper(S), "SS", "ß")]


def _words(rng, n, max_len=7, alphabet=ALPHABET):
    lens = rng.integers(0, max_len + 1, n)
    idx = rng.integers(0, len(alphabet), int(lens.sum()))
    out, pos = [], 0
    for k in lens:
        out.append("".join(alphabet[i] for i in idx[pos:pos + k]))
        pos += k
    return out


def _host(offsets, data, valid, n):
    offs = offsets.cpu().numpy()
    raw = data.cpu().numpy().tobytes()
    ok = [True] * n if valid is None else valid.cpu().numpy().astype(bool).tolist()
    return [raw[offs[i]:offs[i + 1]].decode("utf-8") if ok[i] else None for i in range(n)]


def _steps_result(d: pa.Array, e):
    """The transformed dictionary, entry for entry (no deduplication)."""
    _, steps = ST.string_chain(e, {"s"})
    dd = ST.device_dictionary(d, DEV)
    o, dt, v = ST.apply_steps(dd.offsets, dd.data, dd.valid, steps)
    return _host(o, dt, v, len(d))


def _check_entries(d: pa.Array, exprs=EXPRS):
    vals = d.to_pylist()
    for e in exprs:
        assert _steps_result(d, e) == [osb.evaluate(e, v) for v in vals], str(e)


# ---- K12 entry for entry -----------------------------------------------------------------------------------
def test_transform_matches_oracle_entry_for_entry():
    rng = np.random.default_rng(0)
    words = _words(rng, 4000) + ["", " ", "\t", "  a  ", "aaa", "aaaa", "ßß", "İstanbul"]
    _check_entries(pa.array(words))
    _check_entries(pa.array(words, type=pa.large_string()))
    with_nulls = pa.array([None if i % 7 == 3 else w for i, w in enumerate(words)])
    _check_entries(with_nulls)
    _check_entries(with_nulls.slice(5, 700))                                      # offset != 0
    _check_entries(pa.array(words, type=pa.large_string()).slice(1, 300))
    _check_entries(pa.array([], type=pa.string()))
    _check_entries(pa.array(["", ""]))


def test_transform_long_entries():
    rng = np.random.default_rng(1)
    long = ["".join(rng.choice(ALPHABET, int(rng.integers(66_000, 70_000)))) for _ in range(40)]
    long[3] = "a" * 70_000
    _check_entries(pa.array(long), EXPRS[:16] + [ff.substr(S, 65_000, 3), ff.substr(S, -65_537)])


def test_transform_one_million_entries():
    rng = np.random.default_rng(2)
    d = pa.array(_words(rng, 1_000_000, 16))
    assert _steps_result(d, ff.upper(S)) == pc.utf8_upper(d).to_pylist()
    _check_entries(d, [ff.substr(S, 2, 5), ff.trim(S, " a"), ff.replace(S, "a", "ab"),
                       ff.concat_strict(S, "-", S)])


def test_case_mapping_every_code_point():
    cps = [chr(c) for c in range(0x110000) if not 0xD800 <= c <= 0xDFFF]
    assert len(cps) == 1_112_064
    d = pa.array(cps)
    assert _steps_result(d, ff.upper(S)) == pc.utf8_upper(d).to_pylist()
    assert _steps_result(d, ff.lower(S)) == pc.utf8_lower(d).to_pylist()
    one = pa.array(["".join(cps[::7]), "".join(cps[3::5])])  # long mixed entries: the table search mid-entry
    assert _steps_result(one, ff.upper(S)) == pc.utf8_upper(one).to_pylist()
    assert _steps_result(one, ff.lower(S)) == pc.utf8_lower(one).to_pylist()


def test_substr_grid_against_sqlite():
    rng = np.random.default_rng(3)
    words = _words(rng, 300, 10) + ["", "hello", "😀中é", None]
    d = pa.array(words)
    db = sqlite3.connect(":memory:")
    for a in range(-8, 9):
        for b in [None] + list(range(-3, 9)):
            e = ff.substr(S, a) if b is None else ff.substr(S, a, b)
            if b is None:
                want = [db.execute("SELECT substr(?, ?)", (w, a)).fetchone()[0] for w in words]
            else:
                want = [db.execute("SELECT substr(?, ?, ?)", (w, a, b)).fetchone()[0] for w in words]
            assert _steps_result(d, e) == want, (a, b)


# ---- deduplication -----------------------------------------------------------------------------------------
def _check_dedup(vals, bits):
    d = pa.array(vals, type=pa.string())
    dd = ST.device_dictionary(d, DEV)
    new, remap, remap_valid, copy = ST.dedup(dd.offsets, dd.data, dd.valid, bits)
    first = list(dict.fromkeys(v for v in vals if v is not None))
    assert new.to_pylist() == first and new.type == pa.string()
    code = {v: i for i, v in enumerate(first)}
    r = remap.cpu().numpy()[:len(vals)]
    ok = [True] * len(vals) if remap_valid is None else remap_valid.cpu().numpy().astype(bool).tolist()
    assert [int(x) if m else None for x, m in zip(r, ok)] == [code.get(v) for v in vals]
    assert _host(copy.offsets, copy.data, copy.valid, len(first)) == first


@pytest.mark.parametrize("bits", [64, 3])
def test_dedup_first_occurrence(bits):
    rng = np.random.default_rng(4)
    vals = _words(rng, 20_000, 3)
    vals[5] = vals[17] = None
    _check_dedup(vals, bits)
    _check_dedup(["x"], bits)
    _check_dedup([None, None], bits)
    _check_dedup([], bits)


def test_dedup_heavy_duplication():
    rng = np.random.default_rng(5)
    d = pa.array(_words(rng, 1_000_000, 12))
    _, steps = ST.string_chain(ff.substr(S, 1, 1), {"s"})
    r = ST.evaluate(d, DEV, steps)
    vals = [osb.substr(v, 1, 1) for v in d.to_pylist()]
    first = list(dict.fromkeys(vals))
    assert r.dictionary.to_pylist() == first and r.remap_valid is None and r.null_code is None
    code = {v: i for i, v in enumerate(first)}
    assert r.remap.cpu().numpy().tolist() == [code[v] for v in vals]


# ---- the engine ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def e():
    return fa.make_execution_engine("b200")


def _table(rng, n, ndict, null_entries=False):
    entries = list(dict.fromkeys(_words(rng, ndict * 2)))[:ndict]
    entries += [w.upper() for w in entries[:20]] + [" " + w + "\t" for w in entries[:20]]
    if null_entries:
        entries[1] = None
    codes = rng.integers(0, len(entries), n)
    v, k = rng.integers(-5, 5, n), rng.integers(0, 40, n)
    mask = rng.random(n) < 0.15
    s = pa.DictionaryArray.from_arrays(pa.array(codes.astype(np.int32), mask=mask), pa.array(entries))
    t = B200Table.from_arrow(pa.table({"s": s, "v": v, "k": k}), DEV, Schema("s:str,v:long,k:long"))
    strs = np.array(entries, dtype=object)[codes]
    strs[mask] = None
    return B200DataFrame(t), pd.DataFrame({"s": pd.array(strs, dtype="string"), "v": v, "k": k})


def _rows(x):
    if isinstance(x, pa.Table):
        return [tuple(r.values()) for r in x.to_pylist()]
    return [tuple(None if v is pd.NA else (v.item() if hasattr(v, "item") else v) for v in r)
            for r in x.itertuples(index=False)]


def _as_arrow(df):
    return df.as_arrow() if hasattr(df, "as_arrow") else df.native.to_arrow()


@pytest.mark.parametrize("null_entries", [False, True])
def test_select_filter_assign_sql(e, null_entries):
    rng = np.random.default_rng(6)
    df, pdf = _table(rng, 20_000, 300, null_entries)
    for b in EXPRS:
        sel = SelectColumns(S, b.alias("x"), ff.length(b).alias("n"), (b == "A").alias("q"), b.is_null().alias("z"))
        where = b.like("%a%") | (col("v") > 2)
        got = _as_arrow(e.select(df, sel, where=where))
        df2, exprs, _ = osb.lower_exprs(pdf, list(sel.all_cols) + [where])
        want = ox.select(df2, SelectColumns(*exprs[:-1]), where=exprs[-1])
        assert _rows(got) == _rows(want), str(b)
        assert got.schema.field("x").type == pa.string()
        cond = (b != "") & b.not_null()
        got = _as_arrow(e.filter(df, cond))
        df2, (c2,), added = osb.lower_exprs(pdf, [cond])
        assert _rows(got) == _rows(ox.filter_rows(df2, c2).drop(columns=added)), str(b)
    cols = [ff.upper(S).alias("s"), ff.concat(S, "!").alias("w")]
    got = _as_arrow(e.assign(df, cols))
    df2, exprs, added = osb.lower_exprs(pdf, cols)
    assert _rows(got) == _rows(ox.assign(df2, exprs).drop(columns=added))
    got = fa.raw_sql("SELECT s, UPPER(TRIM(s)) AS u, s || '-' || s AS c, SUBSTRING(s, 2, 2) AS m FROM", df,
                     "WHERE LOWER(s) LIKE '%a%' AND REPLACE(s, 'a', '') != ''", engine=e, as_fugue=True).as_arrow()
    sel = SelectColumns(S, ff.upper(ff.trim(S)).alias("u"), ff.concat_strict(S, "-", S).alias("c"),
                        ff.substr(S, 2, 2).alias("m"))
    where = ff.lower(S).like("%a%") & (ff.replace(S, "a", "") != "")
    df2, exprs, _ = osb.lower_exprs(pdf, list(sel.all_cols) + [where])
    assert _rows(got) == _rows(ox.select(df2, SelectColumns(*exprs[:-1]), where=exprs[-1]))


def _groups(pdf, f):
    out = {}
    for s, k in zip(pdf["s"].tolist(), pdf["k"].tolist()):
        out.setdefault(f(None if s is pd.NA else s), []).append((s, k))
    return out


def test_group_by_and_aggregates(e):
    rng = np.random.default_rng(7)
    df, pdf = _table(rng, 50_000, 500, True)
    got = fa.raw_sql("SELECT UPPER(s) AS u, COUNT(*) AS n FROM", df, "GROUP BY UPPER(s)", engine=e,
                     as_fugue=True).as_arrow()
    want = {u: len(r) for u, r in _groups(pdf, osb.upper).items()}
    res = dict(zip(got.column("u").to_pylist(), got.column("n").to_pylist()))
    assert res == want and len(res) == got.num_rows  # case variants merge into one group
    got = fa.raw_sql("SELECT LOWER(s) AS l, COUNT(DISTINCT UPPER(s)) AS d, MAX(TRIM(s)) AS m FROM", df,
                     "GROUP BY LOWER(s)", engine=e, as_fugue=True).as_arrow()
    want = {}
    for l, r in _groups(pdf, osb.lower).items():
        ss = [s for s, _ in r if s is not pd.NA]
        want[l] = (len({osb.upper(s) for s in ss}), max((osb.trim(s) for s in ss), default=None))
    assert {l: (d, m) for l, d, m in zip(*(got.column(c).to_pylist() for c in ("l", "d", "m")))} == want
    got = fa.aggregate(df, "k", engine=e, as_fugue=True, lo=ff.min(ff.upper(S)), hi=ff.max(ff.concat(S, "~")),
                       f=ff.first(ff.lower(S)), c=ff.count(ff.substr(S, 2))).as_arrow()
    vals = {}
    for s, k in zip(pdf["s"].tolist(), pdf["k"].tolist()):
        vals.setdefault(k, []).append(None if s is pd.NA else s)
    for k, lo, hi, f, c in zip(*(got.column(x).to_pylist() for x in ("k", "lo", "hi", "f", "c"))):
        ss = [s for s in vals[k] if s is not None]
        assert lo == (min(osb.upper(s) for s in ss) if ss else None)
        assert hi == max(osb.concat(s, "~") for s in vals[k])  # CONCAT of a NULL row is '~'
        assert f == next((osb.lower(s) for s in vals[k] if s is not None), None)  # FIRST skips NULL
        assert c == sum(osb.substr(s, 2) is not None for s in vals[k])


def test_window_map(e):
    rng = np.random.default_rng(8)
    df, pdf = _table(rng, 6000, 200)
    t = df.native
    rid = torch.arange(t.num_rows, dtype=torch.int64, device=DEV)
    t = B200Table(Schema("rid:long,s:str,k:long"), [rid, t.columns[0], t.columns[2]], [None, t.valid[0], None],
                  {"s": t.dictionaries["s"]})
    cols = [ff.upper(S).alias("u"), ff.max(ff.lower(S)).over().alias("m"),
            ff.min(ff.trim(S)).over(running=True).alias("r")]
    got = fa.transform(B200DataFrame(t), ColumnMap("rid", *cols), schema="rid:long,u:str,m:str,r:str",
                       partition=PartitionSpec(by="k", presort="rid"), engine=e, as_fugue=True).as_arrow()
    svals = [None if s is pd.NA else s for s in pdf["s"].tolist()]
    keys = pdf["k"].tolist()
    mx, run, want = {}, {}, {}
    for r, (s, k) in enumerate(zip(svals, keys)):
        if s is not None:
            mx[k] = max(mx.get(k, osb.lower(s)), osb.lower(s))
    for r, (s, k) in enumerate(zip(svals, keys)):
        if s is not None:
            run[k] = min(run.get(k, osb.trim(s)), osb.trim(s))
        want[r] = (osb.upper(s), mx.get(k), run.get(k))
    assert {r: (u, m, x) for r, u, m, x in zip(*(got.column(c).to_pylist() for c in ("rid", "u", "m", "r")))} == want


def test_result_cache(e):
    rng = np.random.default_rng(9)
    df, _ = _table(rng, 5000, 100)
    sel = SelectColumns(ff.upper(S).alias("u"))
    before = ST.transforms
    a = e.select(df, sel).native.dictionaries["u"]
    assert ST.transforms == before + 1
    uploads = ST.uploads
    b = e.select(df, sel).native.dictionaries["u"]
    e.filter(df, ff.upper(S) == "A")
    e.select(df, SelectColumns(ff.length(ff.upper(S)).alias("n"), ff.upper(S).like("A%").alias("p")))
    assert ST.transforms == before + 1 and ST.uploads == uploads and b is a  # no transform, no upload
    e.select(df, SelectColumns(ff.lower(S).alias("l")))
    assert ST.transforms == before + 2


def test_upper_select_100m_rows(e):
    n = 100_000_000
    rng = np.random.default_rng(10)
    entries = list(dict.fromkeys(_words(rng, 3000, 12)))[:2000]
    d = pa.array(entries)
    g = torch.Generator(device=DEV).manual_seed(10)
    codes = torch.randint(0, len(entries), (n,), dtype=torch.int32, device=DEV, generator=g)
    valid = (torch.rand(n, device=DEV, generator=g) > 0.1).to(torch.uint8)
    t = B200Table(Schema("s:str"), [codes], [valid], {"s": d})
    got = e.select(B200DataFrame(t), SelectColumns(ff.upper(S).alias("u"))).native
    ups = [osb.upper(w) for w in entries]
    first = list(dict.fromkeys(ups))
    assert got.dictionaries["u"].to_pylist() == first
    remap = torch.tensor([first.index(u) for u in ups], dtype=torch.int32, device=DEV)
    assert torch.equal(got.valid[0].bool(), valid.bool())
    keep = valid.bool()
    assert torch.equal(got.columns[0][keep], remap[codes.long()][keep])
