"""K15 regular expressions on the H100: both kernels entry for entry against pyarrow's RE2 (the seeded corpus of
test_regex_cpu.py, sliced, large_string, empty, NULL-entry, over-64 KB and 1 M-entry dictionaries), the engine
(filter with RLIKE / NOT RLIKE, select, assign, GROUP BY REGEXP_EXTRACT, raw_sql, a ColumnMap window map),
composition with UPPER / LIKE / LENGTH / CAST, the caches, and one 100 M-row filter."""
import random

import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.compute as pc
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

import _regex_corpus as RC
from fugue_b200 import api as fa
from fugue_b200 import kernels as K
from fugue_b200 import regex as R
from fugue_b200 import strings as ST
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import SelectColumns, col, functions as ff
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.partition import PartitionSpec
from fugue_b200.schema import Schema
from fugue_b200.table import B200Table

DEV = torch.device("cuda", 0)
S = col("s")


def _host(offsets, data, valid, n):
    offs = offsets.cpu().numpy()
    raw = data.cpu().numpy().tobytes()
    ok = [True] * n if valid is None else valid.cpu().numpy().astype(bool).tolist()
    return [raw[offs[i]:offs[i + 1]].decode("utf-8") if ok[i] else None for i in range(n)]


def dev_match(d, p, full=False):
    dd = ST.device_dictionary(d, DEV)
    out, ok = K.regex_match(dd.offsets, dd.data, dd.valid, R.match_program(p, full))
    return [bool(x) if v else None for x, v in zip(out.cpu().tolist(), ok.cpu().tolist())]


def dev_transform(d, step):
    dd = ST.device_dictionary(d, DEV)
    offs, data, valid = ST.apply_steps(dd.offsets, dd.data, dd.valid, [step])
    return _host(offs, data, valid, len(d))


def _corpus():
    rng = random.Random(15)
    pats = []
    while len(pats) < 200:
        p = RC.random_pattern(rng)
        try:
            R.parse(p)
        except (NotImplementedError, ValueError):
            continue
        pats.append(p)
    return pats, RC.random_strings(rng, 300) + [None]


def _check(d, pats):
    strs = d.to_pylist()
    for p in pats:
        assert dev_match(d, p) == RC.matches(strs, p), p
        assert dev_match(d, p, True) == RC.matches(strs, p, True), p
        for g in range(min(RC.groups_of(p), 8) + 1):
            assert dev_transform(d, ("REGEXP_EXTRACT", p, g)) == RC.extract(strs, p, g), (p, g)
        for glob in (False, True):
            assert dev_transform(d, ("REGEXP_REPLACE", p, "<\\0>", glob)) == RC.replace(strs, p, "<\\0>", glob), p


def test_kernels_match_re2_on_the_corpus():
    pats, strs = _corpus()
    _check(pa.array(strs, pa.string()), pats)


def test_kernels_on_every_dictionary_layout():
    pats, strs = _corpus()
    pats = pats[:40] + [r"\d+", "^$", "x*", r"(a)|b"]
    _check(pa.array(["zz"] * 7 + strs, pa.string()).slice(7), pats)      # offset != 0
    _check(pa.array(strs, pa.large_string()), pats)
    _check(pa.array([], pa.string()), pats)
    _check(pa.array([None, "a", None, ""], pa.string()), pats)
    big = pa.array(["ab1 x" * 20_000, "1" * 70_000, "é" * 40_000 + "a"], pa.string())  # over 64 KB, many matches
    _check(big, [r"\d", "x*", "a|b", r"(\d)(x)?", "é$"])


def test_one_million_entries():
    rng = random.Random(3)
    strs = RC.random_strings(rng, 1_000_000, 14)
    d = pa.array(strs, pa.string())
    for p in [r"^\d{1,2}", r"[\w.]+@\w+", "(a|b|c)x"]:
        assert dev_match(d, p) == RC.matches(strs, p)
        assert dev_transform(d, ("REGEXP_EXTRACT", p, 0)) == RC.extract(strs, p, 0)
    assert dev_transform(d, ("REGEXP_REPLACE", r"\s+", "_", True)) == RC.replace(strs, r"\s+", "_", True)


# ---- the engine ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def e():
    return fa.make_execution_engine("b200")


ENTRIES = ["2024-01-15 x", "ann@mail.org", "bob@site.com", "x7", "", "no digits", "中@文.cn", "1999-12-31",
           "  42 ", "a\nb", "carl@mail.org"]


def _table(n, null_entries=False, seed=0):
    rng = np.random.default_rng(seed)
    entries = list(ENTRIES) + ([None] if null_entries else [])
    codes = rng.integers(0, len(entries), n)
    v, k = rng.integers(-5, 5, n), rng.integers(0, 7, n)
    mask = rng.random(n) < 0.15
    s = pa.DictionaryArray.from_arrays(pa.array(codes.astype(np.int32), mask=mask), pa.array(entries, pa.string()))
    t = B200Table.from_arrow(pa.table({"s": s, "v": v, "k": k}), DEV, Schema("s:str,v:long,k:long"))
    strs = np.array(entries, dtype=object)[codes]
    strs[mask] = None
    return B200DataFrame(t), list(strs), v.tolist(), k.tolist()


def _arrow(x):
    return x.as_arrow() if hasattr(x, "as_arrow") else x.native.to_arrow()


@pytest.mark.parametrize("null_entries", [False, True])
def test_filter_select_assign_sql(e, null_entries):
    df, strs, v, _ = _table(20_000, null_entries, 1)
    hit = RC.matches(strs, r"\d")
    got = _arrow(e.filter(df, S.rlike(r"\d") & (col("v") > 0)))
    assert got.column("s").to_pylist() == [s for s, h, x in zip(strs, hit, v) if h and x > 0]
    got = _arrow(e.filter(df, ~S.rlike(r"\d")))
    assert got.column("s").to_pylist() == [s for s, h in zip(strs, hit) if h is False]
    sel = SelectColumns(S, ff.regexp_full_match(S, r"\w+@\w+\.\w+").alias("f"),
                        ff.regexp_extract(S, r"@(.*)", 1).alias("dom"),
                        ff.regexp_replace(S, r"\d", "#", "g").alias("r"), ff.regexp_replace(S, "o", "0").alias("r1"))
    got = _arrow(e.select(df, sel))
    assert got.column("f").to_pylist() == RC.matches(strs, r"\w+@\w+\.\w+", True)
    assert got.column("dom").to_pylist() == RC.extract(strs, r"@(.*)", 1)
    assert got.column("r").to_pylist() == RC.replace(strs, r"\d", "#", True)
    assert got.column("r1").to_pylist() == RC.replace(strs, "o", "0", False)
    got = _arrow(e.assign(df, [ff.regexp_extract(S, r"\d+").alias("s")]))
    assert got.column("s").to_pylist() == RC.extract(strs, r"\d+", 0)
    got = fa.raw_sql("SELECT s, REGEXP_REPLACE(TRIM(s), '\\d', '<\\0>', 'g') AS r FROM", df,
                     "WHERE s RLIKE '^\\d' AND v > 0", engine=e, as_fugue=True).as_arrow()
    keep = [i for i, (h, x) in enumerate(zip(RC.matches(strs, r"^\d"), v)) if h and x > 0]
    trimmed = [strs[i].strip(" ") for i in keep]
    assert got.column("r").to_pylist() == RC.replace(trimmed, r"\d", "<\\0>", True)


def test_composition(e):
    df, strs, _, _ = _table(10_000, True, 2)
    sel = SelectColumns(ff.upper(ff.regexp_extract(S, r"@(\w+)", 1)).alias("u"),
                        ff.regexp_replace(S, "a", "A", "g").like("%A%").alias("l"),
                        ff.length(ff.regexp_extract(S, r"\d+")).alias("n"),
                        ff.regexp_matches(ff.regexp_replace(S, r"\d", "", "g"), "^-").alias("m"),
                        ff.regexp_extract(S, r"\d+").cast("long").alias("c"))
    with pytest.raises(ValueError):  # '' and "no digits" do not parse as BIGINT; the device says so as Arrow does
        _arrow(e.select(df, sel))
    sel = SelectColumns(*sel.all_cols[:4])
    got = _arrow(e.select(df, sel))
    ext = RC.extract(strs, r"@(\w+)", 1)
    assert got.column("u").to_pylist() == [None if x is None else x.upper() for x in ext]
    rep = RC.replace(strs, "a", "A", True)
    assert got.column("l").to_pylist() == [None if x is None else "A" in x for x in rep]
    num = RC.extract(strs, r"\d+", 0)
    assert got.column("n").to_pylist() == [None if x is None else len(x) for x in num]
    assert got.column("m").to_pylist() == RC.matches(RC.replace(strs, r"\d", "", True), "^-")
    only = B200DataFrame(B200Table.from_arrow(pa.table({"s": pa.array(["7", "  12 x", "x 300"]).dictionary_encode()}),
                                              DEV, Schema("s:str")))
    got = _arrow(e.select(only, SelectColumns(ff.regexp_extract(S, r"\d+").cast("long").alias("c"))))
    assert got.column("c").to_pylist() == [7, 12, 300]


def test_group_by_and_aggregates(e):
    df, strs, _, ks = _table(30_000, True, 3)
    got = fa.raw_sql("SELECT REGEXP_EXTRACT(s, '@(.*)', 1) AS d, COUNT(*) AS n FROM", df,
                     "GROUP BY REGEXP_EXTRACT(s, '@(.*)', 1)", engine=e, as_fugue=True).as_arrow()
    want = {}
    for x in RC.extract(strs, "@(.*)", 1):
        want[x] = want.get(x, 0) + 1
    assert dict(zip(got.column("d").to_pylist(), got.column("n").to_pylist())) == want
    got = fa.aggregate(df, "k", engine=e, as_fugue=True, lo=ff.min(ff.regexp_replace(S, r"\d", "")),
                       c=ff.count_distinct(ff.regexp_extract(S, r"\w"))).as_arrow()
    rep, ext = RC.replace(strs, r"\d", "", False), RC.extract(strs, r"\w", 0)
    for k, lo, c in zip(*(got.column(x).to_pylist() for x in ("k", "lo", "c"))):
        rs = [r for r, kk in zip(rep, ks) if kk == k and r is not None]
        assert lo == (min(rs) if rs else None)
        assert c == len({x for x, kk in zip(ext, ks) if kk == k and x is not None})


def test_window_map(e):
    df, strs, _, ks = _table(6000, False, 4)
    t = df.native
    rid = torch.arange(t.num_rows, dtype=torch.int64, device=DEV)
    t = B200Table(Schema("rid:long,s:str,k:long"), [rid, t.columns[0], t.columns[2]], [None, t.valid[0], None],
                  {"s": t.dictionaries["s"]})
    cols = [ff.regexp_extract(S, r"\d+").alias("x"), ff.sum(ff.regexp_matches(S, r"\d").cast("long")).over().alias("m")]
    got = fa.transform(B200DataFrame(t), ColumnMap("rid", *cols), schema="rid:long,x:str,m:long",
                       partition=PartitionSpec(by="k", presort="rid"), engine=e, as_fugue=True).as_arrow()
    hit, ext = RC.matches(strs, r"\d"), RC.extract(strs, r"\d+", 0)
    tot = {}
    for h, k in zip(hit, ks):
        if h is not None:
            tot[k] = tot.get(k, 0) + int(h)
    want = {r: (ext[r], tot.get(ks[r])) for r in range(len(strs))}
    assert {r: (x, m) for r, x, m in zip(*(got.column(c).to_pylist() for c in ("rid", "x", "m")))} == want


def test_caches(e):
    df, _, _, _ = _table(5000, False, 5)
    sel = SelectColumns(ff.regexp_extract(S, r"\d+").alias("x"))
    before, matches = ST.transforms, ST.regex_matches
    a = e.select(df, sel).native.dictionaries["x"]
    e.filter(df, S.rlike("^a"))
    assert ST.transforms == before + 1 and ST.regex_matches == matches + 1
    b = e.select(df, sel).native.dictionaries["x"]
    e.filter(df, S.rlike("^a"))
    assert ST.transforms == before + 1 and ST.regex_matches == matches + 1 and a is b  # no regex kernel ran


def test_filter_100m_rows(e):
    n = 100_000_000
    rng = random.Random(11)
    entries = list(dict.fromkeys(RC.random_strings(rng, 3000, 12)))[:2000]
    d = pa.array(entries)
    g = torch.Generator(device=DEV).manual_seed(11)
    codes = torch.randint(0, len(entries), (n,), dtype=torch.int32, device=DEV, generator=g)
    valid = (torch.rand(n, device=DEV, generator=g) > 0.1).to(torch.uint8)
    t = B200Table(Schema("s:str"), [codes], [valid], {"s": d})
    got = e.filter(B200DataFrame(t), ff.regexp_matches(S, r"\d.?é|^@")).native
    hit = torch.tensor(RC.matches(entries, r"\d.?é|^@"), dtype=torch.bool, device=DEV)
    keep = valid.bool() & hit[codes.long()]
    assert torch.equal(got.columns[0], codes[keep])
