"""LIKE, LENGTH and string MIN / MAX on the H100: the per-entry kernels (K11) entry for entry against
oracle/strings.py, FB_X_LOOKUP in the expression evaluator (K8) bit for bit against the numpy machine model,
filter / select / assign / SQL against oracle/expressions.py, GROUP BY and window MIN / MAX against direct
restatements over the strings, the dictionary cache, and one filter at 100 M rows."""

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

import _lookup_sim as lsim
from fugue_b200 import api as fa
from fugue_b200 import expr as X
from fugue_b200 import kernels as K
from fugue_b200 import strings as ST
from fugue_b200.colmap import ColumnMap
from fugue_b200.column import SelectColumns, col, functions as ff
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.partition import PartitionSpec
from fugue_b200.schema import Schema
from fugue_b200.table import B200Table, expr_type
from oracle import expressions as ox
from oracle import strings as ostr

DEV = torch.device("cuda", 0)
ALPHABET = ["a", "b", "c", "%", "_", "!", "é", "ß", "€", "中", "😀", "𝄞"]
PATTERNS = [("", None), ("%", None), ("%%", None), ("_", None), ("a%", None), ("%a", None), ("%a%b%", None),
            ("_é%", None), ("%€", None), ("%😀_", None), ("__", None), ("a_%_c", None), ("%中%𝄞%", None),
            ("!%%", "!"), ("%!%", "!"), ("!_%", "!"), ("%!!%", "!"), ("a!_b", "!"), ("%_%_%", None)]


@pytest.fixture(scope="module")
def e():
    return fa.make_execution_engine("b200")


def _words(rng, n, max_len=7, alphabet=ALPHABET):
    lens = rng.integers(0, max_len + 1, n)
    idx = rng.integers(0, len(alphabet), int(lens.sum()))
    out, pos = [], 0
    for k in lens:
        out.append("".join(alphabet[i] for i in idx[pos:pos + k]))
        pos += k
    return out


def _check_entries(d: pa.Array, patterns):
    dd = ST.device_dictionary(d, DEV)
    vals = d.to_pylist()
    got = K.string_length(dd.offsets, dd.data, dd.valid).cpu().numpy()
    assert got.tolist() == [ostr.length(v) or 0 for v in vals]
    for p, esc in patterns:
        m, mv = K.string_like(dd.offsets, dd.data, dd.valid, ST.like_tokens(p, esc))
        want = [ostr.like(v, p, esc) for v in vals]
        assert m.cpu().numpy().tolist() == [int(bool(w)) for w in want], (p, esc)
        assert mv.cpu().numpy().tolist() == [int(v is not None) for v in vals]


# ---- K11 ---------------------------------------------------------------------------------------------------
def test_kernels_match_oracle_entry_for_entry():
    rng = np.random.default_rng(0)
    words = _words(rng, 5000) + ["", "a", "%", "_", "!", "😀", "a😀c", "é€中𝄞"]
    _check_entries(pa.array(words), PATTERNS)
    _check_entries(pa.array(words, type=pa.large_string()), PATTERNS)
    with_nulls = pa.array([None if i % 7 == 3 else w for i, w in enumerate(words)])
    _check_entries(with_nulls, PATTERNS)
    _check_entries(with_nulls.slice(5, 700), PATTERNS)                            # offset != 0
    _check_entries(pa.array(words, type=pa.large_string()).slice(1, 300), PATTERNS[:6])
    _check_entries(pa.array([], type=pa.string()), PATTERNS[:3])
    _check_entries(pa.array(["", ""]), PATTERNS[:4])


def test_kernels_long_entries():
    rng = np.random.default_rng(1)
    long = ["".join(_words(rng, 1, 0)) + "".join(rng.choice(ALPHABET, int(rng.integers(1000, 3000))))
            for _ in range(300)]
    long[7] = "a" * 5000 + "b"
    _check_entries(pa.array(long), PATTERNS + [("%b", None), ("a%a%a%b", None), ("%" + "_" * 1000 + "%", None)])


def test_kernels_one_million_entries():
    rng = np.random.default_rng(2)
    words = _words(rng, 1_000_000, 16)
    _check_entries(pa.array(words), [("%ab%", None), ("a%", None), ("%_é_%", None), ("___", None), ("%!%%", "!")])


# ---- K8 FB_X_LOOKUP against the machine model --------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2047, 2048, 2049, 132 * 3 * 2048 + 3000])
def test_lookup_matches_model(n):
    rng = np.random.default_rng(n)
    entries = _words(rng, 50)
    entries[3] = None
    entries[0] = "a"  # matches 'a%'
    d = pa.array(entries)
    codes = rng.integers(0, 50, n).astype(np.int32)
    valid = (rng.random(n) > 0.3).astype(np.uint8)
    codes[valid == 0] = 0  # NULL rows whose stored code is an entry that matches
    v = rng.integers(-3, 3, n)
    t = B200Table(Schema("s:str,v:long"), [torch.from_numpy(codes).to(DEV), torch.from_numpy(v).to(DEV)],
                  [torch.from_numpy(valid).to(DEV), None], {"s": d})
    for ex in [col("s").like("a%"), ~col("s").like("%b_"), col("s").like("a%") & (col("v") > 0),
               ff.length(col("s")) * 2 + col("v")]:
        prog = X._Program(t)
        cls, _ = prog.compile(ex, top=True)
        prog.output(torch.int64, True)
        outs, outv = prog.run()
        cols = [t.columns[i] if isinstance(i, int) else prog.tables[i][0] for i in prog.cols]
        vals = [t.valid[i] if isinstance(i, int) else prog.tables[i][1] for i in prog.cols]
        types = [expr_type(t.schema.types[i]) if isinstance(i, int) else K.T_I64 for i in prog.cols]
        want, wantv = lsim.run(n, [c.cpu().numpy() for c in cols], [None if m is None else m.cpu().numpy() for m in vals],
                              prog.ins, [K.T_I64], col_types=types)
        assert np.array_equal(outs[0].cpu().numpy(), want[0]), str(ex)
        assert np.array_equal(outv[0].cpu().numpy(), wantv[0]), str(ex)
        if "LIKE" in str(ex) and "v" not in str(ex):
            assert not outv[0].cpu().numpy()[valid == 0].any()


# ---- the engine ----------------------------------------------------------------------------------------------
def _table(rng, n, ndict, null_entries=False, null_key=None):
    """(device frame, pandas frame) of s:str (a dictionary of ``ndict`` entries, one NULL entry with
    ``null_entries``), v:long and k:long; rows with k == null_key have NULL s."""
    entries = list(dict.fromkeys(_words(rng, ndict * 2)))[:ndict]
    if null_entries:
        entries[1] = None
    codes = rng.integers(0, len(entries), n)
    v, k = rng.integers(-5, 5, n), rng.integers(0, 40, n)
    mask = (rng.random(n) < 0.15) | (k == null_key)
    s = pa.DictionaryArray.from_arrays(pa.array(codes.astype(np.int32), mask=mask), pa.array(entries))
    tbl = pa.table({"s": s, "v": v, "k": k})
    t = B200Table.from_arrow(tbl, DEV, Schema("s:str,v:long,k:long"))
    strs = np.array(entries, dtype=object)[codes]
    strs[mask] = None
    pdf = pd.DataFrame({"s": pd.array(strs, dtype="string"), "v": v, "k": k})
    return B200DataFrame(t), pdf


def _rows(x):
    if isinstance(x, pa.Table):
        return [tuple(r.values()) for r in x.to_pylist()]
    return [tuple(None if v is pd.NA else (v.item() if hasattr(v, "item") else v) for v in r)
            for r in x.itertuples(index=False)]


def _as_arrow(df):
    return df.as_arrow() if hasattr(df, "as_arrow") else df.native.to_arrow()


def _oracle_filter(pdf, c):
    df2, (c2,), added = ostr.lower(pdf, [c])
    return ox.filter_rows(df2, c2).drop(columns=added)


def _oracle_select(pdf, sel, where):
    df2, exprs, _ = ostr.lower(pdf, list(sel.all_cols) + [where])
    return ox.select(df2, SelectColumns(*exprs[:-1]), where=exprs[-1])


def _oracle_assign(pdf, cols):
    df2, exprs, added = ostr.lower(pdf, cols)
    return ox.assign(df2, exprs).drop(columns=added)


@pytest.mark.parametrize("null_entries", [False, True])
def test_filter_select_assign_sql(e, null_entries):
    rng = np.random.default_rng(3)
    df, pdf = _table(rng, 20_000, 300, null_entries)
    for p, esc in PATTERNS:
        cond = col("s").like(p, esc)
        for c in (cond, ~cond & (col("v") > 0)):
            got = _as_arrow(e.filter(df, c))
            assert _rows(got) == _rows(_oracle_filter(pdf, c)), str(c)
    sel = SelectColumns(col("s"), ff.length(col("s")).alias("n"), (ff.length(col("s")) * 2 + col("v")).alias("m"),
                        col("s").like("%a%").alias("p"), (~col("s").like("a!_%", "!")).alias("q"))
    got = _as_arrow(e.select(df, sel, where=col("s").like("%b%") | (col("v") > 2)))
    assert _rows(got) == _rows(_oracle_select(pdf, sel, where=col("s").like("%b%") | (col("v") > 2)))
    got = _as_arrow(e.assign(df, [ff.length(col("s")).alias("v"), col("s").like("_%").alias("x")]))
    assert _rows(got) == _rows(_oracle_assign(pdf, [ff.length(col("s")).alias("v"), col("s").like("_%").alias("x")]))
    got = fa.raw_sql("SELECT s, LENGTH(s) AS n FROM", df, "WHERE s LIKE '%a%' AND s NOT LIKE '%!%%' ESCAPE '!'",
                     engine=e, as_fugue=True).as_arrow()
    want = _oracle_select(pdf, SelectColumns(col("s"), ff.length(col("s")).alias("n")),
                     where=col("s").like("%a%") & ~col("s").like("%!%%", "!"))
    assert _rows(got) == _rows(want)


def _group_extremes(pdf, keys):
    """MIN / MAX of the non-NULL strings per group (code-point order; None for an all-NULL group)."""
    out = {}
    for k, g in (pdf.groupby(keys, dropna=False) if keys else [((), pdf)]):
        vals = [x for x in g["s"].tolist() if x is not None and x is not pd.NA]
        out[k if isinstance(k, tuple) else (k,)] = (min(vals) if vals else None, max(vals) if vals else None)
    return out


@pytest.mark.parametrize("n", [30_000, 4_500_000])
def test_group_min_max(e, n):
    rng = np.random.default_rng(4)
    tbl, pdf = _table(rng, n, 5000, null_entries=True, null_key=7)  # group 7: NULL values only
    want = _group_extremes(pdf, ["k"])
    for with_pct in (False, True):
        aggs = dict(lo=ff.min(col("s")), hi=ff.max(col("s")))
        if with_pct:
            aggs["md"] = ff.median(col("v"))
        got = fa.aggregate(tbl, "k", engine=e, as_fugue=True, **aggs).as_arrow()
        res = {(k,): (lo, hi) for k, lo, hi in zip(got.column("k").to_pylist(), got.column("lo").to_pylist(),
                                                 got.column("hi").to_pylist())}
        assert res == want
        assert got.schema.field("lo").type == pa.string()
    got = fa.aggregate(tbl, None, engine=e, as_fugue=True, lo=ff.min(col("s")), hi=ff.max(col("s"))).as_arrow()
    assert (got.column("lo")[0].as_py(), got.column("hi")[0].as_py()) == _group_extremes(pdf, [])[()]
    got = fa.raw_sql("SELECT k, MIN(s) AS lo, MAX(s) AS hi FROM", tbl, "GROUP BY k", engine=e, as_fugue=True).as_arrow()
    assert {(k,): (lo, hi) for k, lo, hi in zip(*(got.column(c).to_pylist() for c in ("k", "lo", "hi")))} == want


def _frame_extremes(part, frame):
    """Per row of one partition (a list of (p, s) in presort order): MIN and MAX of the non-NULL strings of its
    frame - ``None`` the whole partition, "running", ("rows", a, b) or ("range", a, b) on the integer p."""
    out = []
    for i, (p, _) in enumerate(part):
        if frame is None:
            rows = part
        elif frame == "running":
            rows = part[:i + 1]
        elif frame[0] == "rows":
            rows = part[max(0, i + frame[1]):max(0, i + frame[2] + 1)]
        else:
            rows = [r for r in part if p + frame[1] <= r[0] <= p + frame[2]]
        vals = [s for _, s in rows if s is not None]
        out.append((min(vals) if vals else None, max(vals) if vals else None))
    return out


def test_window_min_max(e):
    rng = np.random.default_rng(5)
    n = 6000
    entries = list(dict.fromkeys(_words(rng, 800)))[:400]
    codes = rng.integers(0, len(entries), n)
    mask = rng.random(n) < 0.2
    key = rng.integers(0, 60, n)
    mask[key == 11] = True  # a partition with NULL values only
    p = rng.integers(0, 40, n)
    tbl = pa.table({"rid": np.arange(n), "key": key, "p": p,
                    "s": pa.DictionaryArray.from_arrays(pa.array(codes.astype(np.int32), mask=mask), pa.array(entries))})
    tbl = B200DataFrame(B200Table.from_arrow(tbl, DEV, Schema("rid:long,key:long,p:long,s:str")))
    frames = {"w": None, "r": "running", "m": ("rows", -3, 1), "g": ("range", -5, 0)}
    kw = {"w": {}, "r": {"running": True}, "m": {"rows": (-3, 1)}, "g": {"range": (-5, 0)}}
    cols = []
    for name in frames:
        cols += [ff.min(col("s")).over(**kw[name]).alias(name + "lo"), ff.max(col("s")).over(**kw[name]).alias(name + "hi")]
    out_schema = "rid:long," + ",".join(f"{c.output_name}:str" for c in cols)
    got = fa.transform(tbl, ColumnMap("rid", *cols), schema=out_schema, partition=PartitionSpec(by="key", presort="p"),
                       engine=e, as_fugue=True).as_arrow()
    at = {r: i for i, r in enumerate(got.column("rid").to_pylist())}
    svals = [None if m else entries[c] for c, m in zip(codes, mask)]
    order = np.lexsort((np.arange(n), p, key))  # stable presort inside every partition
    parts = {}
    for r in order:
        parts.setdefault(int(key[r]), []).append(int(r))
    for name, frame in frames.items():
        lo, hi = got.column(name + "lo").to_pylist(), got.column(name + "hi").to_pylist()
        for rows in parts.values():
            want = _frame_extremes([(int(p[r]), svals[r]) for r in rows], frame)
            assert [(lo[at[r]], hi[at[r]]) for r in rows] == want, name


def test_dictionary_cache(e):
    rng = np.random.default_rng(6)
    df, _ = _table(rng, 5000, 100)
    t = df.native
    before = ST.uploads
    e.filter(df, col("s").like("a%"))
    e.select(df, SelectColumns(ff.length(col("s")).alias("n")))
    e.filter(B200DataFrame(t.select(["s", "v"]).rename({"v": "w"})), col("s").like("%b"))
    assert ST.uploads == before + 1
    df2, _ = _table(np.random.default_rng(7), 5000, 100)
    e.filter(df2, col("s").like("a%"))
    assert ST.uploads == before + 2


def test_filter_like_100m_rows(e):
    n = 100_000_000
    rng = np.random.default_rng(8)
    entries = list(dict.fromkeys(_words(rng, 3000, 12)))[:2000]
    d = pa.array(entries)
    match = np.array([ostr.like(w, "%ab%") for w in entries])
    g = torch.Generator(device=DEV).manual_seed(8)
    codes = torch.randint(0, len(entries), (n,), dtype=torch.int32, device=DEV, generator=g)
    valid = (torch.rand(n, device=DEV, generator=g) > 0.1).to(torch.uint8)
    rid = torch.arange(n, dtype=torch.int64, device=DEV)
    t = B200Table(Schema("s:str,rid:long"), [codes, rid], [valid, None], {"s": d})
    got = e.filter(B200DataFrame(t), col("s").like("%ab%")).native
    keep = torch.from_numpy(match).to(DEV)[codes.long()] & valid.bool()
    want = torch.nonzero(keep).squeeze(1)
    assert torch.equal(got.columns[1], want)
    assert torch.equal(got.columns[0], codes[want])
