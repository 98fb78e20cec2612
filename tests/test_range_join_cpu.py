"""Range joins on the CPU (DESIGN §7r): the oracle against SQLite and ``pandas.merge`` + a filter, a numpy model of
``fb_range_join_count`` / ``fb_range_join_emit`` (the MAX-tree walk included) against the oracle, the schema, type,
``how`` and ``closed`` rules, the SQL forms parsed to the engine call, every rejection, and the ``fa.range_join``
plumbing, all before any device work."""
import math
import sqlite3

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest

from fugue_b200 import api as fa
from fugue_b200.dataframe import ArrowDataFrame, DataFrame, as_fugue_df
from fugue_b200.join import get_range_schemas
from fugue_b200.lifecycle import EngineLifecycle
from fugue_b200.schema import Schema, SchemaError
from oracle import range_join as R

_OPS = {"both": ("<=", "<="), "left": ("<=", "<"), "right": ("<", "<="), "neither": ("<", "<")}


def _random_tables(rng, n1, n2, nkeys=1, null=0.1, span=60):
    left = {"t": [None if rng.random() < null else int(v) for v in rng.integers(-5, span + 5, n1)]}
    s = rng.integers(0, span, n2)
    e = s + rng.integers(-3, 12, n2)  # some reversed, some zero-width
    right = {"s": [None if rng.random() < null else int(v) for v in s],
             "e": [None if rng.random() < null else int(v) for v in e]}
    for k in range(nkeys):
        left[f"k{k}"] = [None if rng.random() < null else int(v) for v in rng.integers(0, 4, n1)]
        right[f"k{k}"] = [None if rng.random() < null else int(v) for v in rng.integers(0, 3, n2)]
    return left, right


def _oracle(left, right, on, closed, how):
    lk = list(zip(*[left[k] for k in on])) if on else [()] * len(left["t"])
    rk = list(zip(*[right[k] for k in on])) if on else [()] * len(right["s"])
    lk = [None if any(v is None for v in k) else k for k in lk]
    rk = [None if any(v is None for v in k) else k for k in rk]
    code = lambda v: None if v is None else v + (1 << 63)  # noqa: E731
    return R.match_pairs(lk, [code(v) for v in left["t"]], rk, [code(v) for v in right["s"]],
                         [code(v) for v in right["e"]], closed, how)


@pytest.mark.parametrize("closed", R.CLOSED)
@pytest.mark.parametrize("how", R.HOWS)
@pytest.mark.parametrize("nkeys", [0, 1, 2])
def test_oracle_equals_sqlite(closed, how, nkeys):
    rng = np.random.default_rng(len(closed) * 10 + nkeys + len(how))
    left, right = _random_tables(rng, 300, 200, nkeys)
    on = [f"k{k}" for k in range(nkeys)]
    db = sqlite3.connect(":memory:")
    db.execute(f"CREATE TABLE l (i INTEGER, t INTEGER{''.join(f', {k} INTEGER' for k in on)})")
    db.execute(f"CREATE TABLE r (j INTEGER, s INTEGER, e INTEGER{''.join(f', {k} INTEGER' for k in on)})")
    db.executemany(f"INSERT INTO l VALUES ({', '.join('?' * (2 + nkeys))})",
                   [(i, left["t"][i], *[left[k][i] for k in on]) for i in range(300)])
    db.executemany(f"INSERT INTO r VALUES ({', '.join('?' * (3 + nkeys))})",
                   [(j, right["s"][j], right["e"][j], *[right[k][j] for k in on]) for j in range(200)])
    lo, hi = _OPS[closed]
    cond = " AND ".join([f"l.{k} = r.{k}" for k in on] + [f"r.s {lo} l.t", f"l.t {hi} r.e"])
    if closed == "both":  # SQL's BETWEEN is the closed interval
        cond = " AND ".join([f"l.{k} = r.{k}" for k in on] + ["l.t BETWEEN r.s AND r.e"])
    join = "LEFT JOIN" if how == "left_outer" else "JOIN"
    got = db.execute(f"SELECT l.i, COALESCE(r.j, -1) FROM l {join} r ON {cond} ORDER BY l.i, r.s, r.j").fetchall()
    assert _oracle(left, right, on, closed, how) == [tuple(p) for p in got]


@pytest.mark.parametrize("closed", R.CLOSED)
def test_oracle_equals_pandas_merge_and_filter(closed):
    rng = np.random.default_rng(7)
    n1, n2 = 2000, 500
    left = pd.DataFrame({"k": rng.integers(0, 20, n1), "t": rng.standard_normal(n1).round(1), "i": np.arange(n1)})
    right = pd.DataFrame({"k": rng.integers(0, 20, n2), "s": rng.standard_normal(n2).round(1), "j": np.arange(n2)})
    right["e"] = right["s"] + rng.random(n2).round(1)
    m = left.merge(right, on="k")
    lo, hi = _OPS[closed]
    keep = (m.s <= m.t if lo == "<=" else m.s < m.t) & (m.t <= m.e if hi == "<=" else m.t < m.e)
    exp = m[keep].sort_values(["i", "s", "j"], kind="stable")
    got = R.range_join(pa.Table.from_pandas(left, preserve_index=False),
                       pa.Table.from_pandas(right, preserve_index=False), ["k"], "t", "s", "e", "inner", closed)
    assert got.column("i").to_pylist() == exp.i.tolist() and got.column("j").to_pylist() == exp.j.tolist()


def test_oracle_codes_and_edges():
    """uint64 past 2^63 and the int64 extremes, beyond SQLite's integers: the loop against hand-worked pairs and
    against the numpy level."""
    u = pa.array([0, (1 << 63) - 1, 1 << 63, (1 << 64) - 1], pa.uint64())
    assert R.order_codes(u) == [0, (1 << 63) - 1, 1 << 63, (1 << 64) - 1]
    i = pa.array([-(1 << 63), -1, 0, (1 << 63) - 1], pa.int64())
    assert R.order_codes(i) == [0, (1 << 63) - 1, 1 << 63, (1 << 64) - 1]
    f = R.order_codes(pa.array([-math.inf, -1.0, -0.0, 0.0, 1.0, math.inf, math.nan, None]))
    assert f[0] < f[1] < f[2] == f[3] < f[4] < f[5] and f[6:] == [None, None]
    left = pa.table({"t": pa.array([1 << 63, (1 << 63) - 1, (1 << 64) - 1, 0], pa.uint64())})
    right = pa.table({"s": pa.array([1 << 63, 0, (1 << 64) - 1, 5], pa.uint64()),
                      "e": pa.array([(1 << 64) - 1, (1 << 63) - 1, (1 << 64) - 1, 4], pa.uint64()), "j": [0, 1, 2, 3]})
    got = R.range_join(left, right, [], "t", "s", "e", "left_outer")
    assert list(zip(got.column("t").to_pylist(), got.column("j").to_pylist())) == [
        (1 << 63, 0), ((1 << 63) - 1, 1), ((1 << 64) - 1, 0), ((1 << 64) - 1, 2), (0, 1)]
    got = R.range_join(left, right, [], "t", "s", "e", "left_outer", "neither")  # open ends at the top code
    assert got.column("j").to_pylist() == [None, None, None, None]
    got = R.range_join(left, right, [], "t", "s", "e", "left_outer", "right")
    assert got.column("j").to_pylist() == [None, 1, 0, None]
    rng = np.random.default_rng(8)
    for closed in R.CLOSED:
        for how in R.HOWS:
            lc = rng.integers(0, 40, 300).astype(np.uint64) + np.uint64((1 << 63) - 20)
            sc = rng.integers(0, 40, 200).astype(np.uint64) + np.uint64((1 << 63) - 20)
            ec = sc + rng.integers(0, 6, 200).astype(np.uint64)
            lk, rk = rng.integers(0, 3, 300), rng.integers(0, 3, 200)
            lok, rok = rng.random(300) > 0.1, rng.random(200) > 0.1
            loop = R.match_pairs([(int(k),) if ok else None for k, ok in zip(lk, lok)], [int(c) for c in lc],
                                 [(int(k),) if ok else None for k, ok in zip(rk, rok)], [int(c) for c in sc],
                                 [int(c) for c in ec], closed, how)
            li, ri = R.match_pairs_np(lk, lc, lok, rk, sc, ec, rok, closed, how)
            assert list(zip(li.tolist(), ri.tolist())) == loop


# ---- a numpy model of fb_range_join_count / fb_range_join_emit ---------------------------------------------------
class _Model:
    """The device path step by step: right rows kept and sorted by (key, start), the runs, the MAX tree over the
    end codes (levels as fb_window_tree lays them out), and per left row the binary search plus the walk of
    ``range_prev_hit`` (csrc/fb_join.cu), with a count of the tree nodes it reads."""

    def __init__(self, rk, sc, ec, rok):
        keep = np.flatnonzero(rok & (sc <= ec))
        order = np.lexsort((sc[keep], rk[keep]))
        self.rows = keep[order]
        self.keys, self.starts, self.ends = rk[self.rows], sc[self.rows], ec[self.rows]
        n = len(self.rows)
        heads = np.flatnonzero(np.r_[True, self.keys[1:] != self.keys[:-1]]) if n else np.zeros(0, np.int64)
        self.run_off = np.r_[heads, n]
        self.run_of = {int(self.keys[h]): r for r, h in enumerate(heads)}
        self.levels = [self.ends]
        while len(self.levels[-1]) >= 2:
            lv = self.levels[-1]
            m = len(lv) // 2
            self.levels.append(np.maximum(lv[0:2 * m:2], lv[1:2 * m:2]))
        self.reads = 0

    def node(self, level, m):
        self.reads += 1
        return int(self.levels[level][m])

    def prev_hit(self, s, q, t):
        lo, hi, level, left_levels, b = s, q, 0, [], -1
        while lo < hi:
            if hi & 1 and self.node(level, hi - 1) >= t:
                b = hi - 1
                break
            hi &= ~1
            if lo & 1:
                left_levels.append(level)
                lo += 1
            lo, hi, level = lo >> 1, hi >> 1, level + 1
        if b < 0:
            for level in reversed(left_levels):
                m = (s + (1 << level) - 1) >> level
                if self.node(level, m) >= t:
                    b = m
                    break
            else:
                return -1
        while level > 0:
            b = 2 * b + 1 if self.node(level - 1, 2 * b + 1) >= t else 2 * b
            level -= 1
        return b

    def row(self, key, ok, x, closed):
        """The sorted positions of the row's matches, right to left as the kernel finds them."""
        r = self.run_of.get(int(key)) if ok else None
        if r is None:
            return []
        s, e = int(self.run_off[r]), int(self.run_off[r + 1])
        lo, hi = closed in ("both", "left"), closed in ("both", "right")
        p = s + int(np.searchsorted(self.starts[s:e], x, "right" if lo else "left"))
        if not hi and x == (1 << 64) - 1:
            return []
        t = x if hi else x + 1
        out, q = [], self.prev_hit(s, p, t)
        while q >= 0:
            out.append(q)
            q = self.prev_hit(s, q, t)
        return out

    def pairs(self, lk, lc, lok, closed, how):
        counts = []
        walks = [self.row(k, ok, int(x), closed) for k, x, ok in zip(lk, lc, lok)]
        for w in walks:  # count
            counts.append(len(w) if w or how == "inner" else 1)
        offsets = np.r_[0, np.cumsum(counts)].astype(np.int64)
        li = np.full(offsets[-1], -7, np.int64)
        ri = np.full(offsets[-1], -7, np.int64)
        for i, w in enumerate(walks):  # emit: from the back of the row's slots
            o = offsets[i] + counts[i]
            for q in w:
                o -= 1
                li[o], ri[o] = i, self.rows[q]
            if not w and how == "left_outer":
                li[o - 1], ri[o - 1] = i, -1
        return li, ri


def _model_case(rng, n1, n2, nk, spread, width):
    lk, rk = rng.integers(0, nk + 1, n1), rng.integers(0, nk, n2)
    lc = rng.integers(0, spread, n1).astype(np.uint64)
    sc = rng.integers(0, spread, n2).astype(np.uint64)
    ec = sc + rng.integers(0, width, n2).astype(np.uint64) - np.uint64(1)  # start - 1: reversed
    return lk, lc, rng.random(n1) > 0.05, rk, sc, ec, rng.random(n2) > 0.05


@pytest.mark.parametrize("closed", R.CLOSED)
@pytest.mark.parametrize("how", R.HOWS)
@pytest.mark.parametrize("n1,n2,nk,spread,width", [(500, 300, 3, 200, 30), (400, 1000, 1, 5000, 400),
                                                    (300, 257, 5, 40, 3), (1, 1, 1, 3, 3), (50, 0, 1, 9, 2)])
def test_kernel_model_equals_oracle(closed, how, n1, n2, nk, spread, width):
    rng = np.random.default_rng(n1 + n2 + len(closed) + len(how))
    lk, lc, lok, rk, sc, ec, rok = _model_case(rng, n1, n2, nk, spread, width)
    li, ri = _Model(rk, sc, ec, rok).pairs(lk, lc, lok, closed, how)
    eli, eri = R.match_pairs_np(lk, lc, lok, rk, sc, ec, rok, closed, how)
    assert np.array_equal(li, eli) and np.array_equal(ri, eri)


def test_kernel_model_adversarial_nesting_is_logarithmic():
    """One interval spanning the whole run, then 2^14 short ones after it: a walk back over a prefix maximum reads
    O(run) per row; the tree walk reads O((1 + matches) log run)."""
    n = 1 << 14
    sc = np.r_[0, np.arange(1, n + 1) * 10].astype(np.uint64)
    ec = np.r_[n * 10 + 100, np.arange(1, n + 1) * 10 + 3].astype(np.uint64)
    rk = np.zeros(n + 1, np.int64)
    model = _Model(rk, sc, ec, np.ones(n + 1, bool))
    rng = np.random.default_rng(9)
    lc = rng.integers(0, n * 10, 300).astype(np.uint64)
    li, ri = model.pairs(np.zeros(300, np.int64), lc, np.ones(300, bool), "both", "inner")
    eli, eri = R.match_pairs_np(np.zeros(300, np.int64), lc, np.ones(300, bool), rk, sc, ec, np.ones(n + 1, bool))
    assert np.array_equal(li, eli) and np.array_equal(ri, eri)
    log = int(math.log2(n + 1)) + 1
    assert model.reads <= 300 * 4 * log * 3, model.reads  # <= 2 matches a row, ~4 log n reads a walk


class _DF:
    def __init__(self, expr: str):
        self.schema = Schema(expr)
        self.columns = self.schema.names


def test_schema_rule():
    a, b = _DF("k:long,t:datetime,v:double"), _DF("k:long,s:datetime,e:datetime,w:str")
    on, s = get_range_schemas(a, b, ["k"], "t", "s", "e")
    assert on == ["k"] and str(s) == "k:long,t:datetime,v:double,s:datetime,e:datetime,w:str"
    assert get_range_schemas(a, b, None, "t", "s", "e")[0] == ["k"]  # None: the common columns but at
    assert str(get_range_schemas(a, _DF("p:datetime"), [], "t", "p", "p")[1]) == "k:long,t:datetime,v:double,p:datetime"
    assert get_range_schemas(_DF("t:long"), _DF("s:long"), None, "t", "s", "s")[0] == []
    for args in ((b, [], "t", "s", "e"),                               # k is common but not a key
                 (_DF("k:int,s:datetime,e:datetime"), ["k"], "t", "s", "e"),  # key types differ
                 (_DF("k:long,s:long,e:long"), ["k"], "t", "s", "e"),          # value types differ
                 (_DF("k:long,s:datetime,e:date"), ["k"], "t", "s", "e"),
                 (b, ["k"], "u", "s", "e"), (b, ["k"], "t", "x", "e"), (b, ["k"], "t", "s", "x"),
                 (_DF("k:long,t:datetime,s:datetime,e:datetime"), ["k"], "t", "s", "e")):  # t is common
        with pytest.raises(SchemaError):
            get_range_schemas(a, *args)
    for args in ((["k", "t"], "t", "s", "e"), (["k", "s"], "t", "s", "e"), (["k"], ["t"], "s", "e"),
                 (["k"], "t", None, "e")):
        with pytest.raises(ValueError):
            get_range_schemas(a, b, *args)


def _host_table(cols):
    import torch

    from fugue_b200.dataframe import B200DataFrame
    from fugue_b200.table import B200Table

    schema = Schema(",".join(f"{n}:{t}" for n, t in cols))
    tensors = [torch.tensor([0], dtype=torch.int32) if t == "str" else torch.tensor([1]) for _, t in cols]
    return B200DataFrame(B200Table(schema, tensors, [None] * len(cols),
                                   {n: pa.array(["x"]) for n, t in cols if t == "str"}))


def test_engine_rejections_before_the_device():
    from fugue_b200.dist import DistributedB200Engine
    from fugue_b200.execution_engine import B200ExecutionEngine

    eng = B200ExecutionEngine.__new__(B200ExecutionEngine)
    eng.to_df = lambda df, schema=None: df  # type: ignore
    eng.get_current_parallelism = lambda: 1  # type: ignore
    a, b = _host_table([("k", "long"), ("t", "long")]), _host_table([("k", "long"), ("s", "long"), ("e", "long")])
    for kw in (dict(how="right_outer"), dict(how="full_outer"), dict(how="semi"), dict(how="cross"),
               dict(how=None), dict(closed="open"), dict(closed=None), dict(closed=3)):
        with pytest.raises(ValueError):
            eng.range_join(a, b, on=["k"], at="t", start="s", end="e", **kw)
    sa = _host_table([("k", "long"), ("t", "str")])
    sb = _host_table([("k", "long"), ("s", "str"), ("e", "str")])
    with pytest.raises(ValueError, match="numeric or temporal"):  # string range columns
        eng.range_join(sa, sb, on=["k"], at="t", start="s", end="e")
    ba = _host_table([("k", "long"), ("t", "bool")])
    bb = _host_table([("k", "long"), ("s", "bool"), ("e", "bool")])
    with pytest.raises(ValueError, match="numeric or temporal"):
        eng.range_join(ba, bb, on=["k"], at="t", start="s", end="e")
    with pytest.raises(SchemaError):
        eng.range_join(a, _host_table([("k", "long"), ("s", "int"), ("e", "long")]), on=["k"], at="t", start="s",
                       end="e")
    dist = DistributedB200Engine.__new__(DistributedB200Engine)
    dist._world = 2
    dist.to_df = lambda df, schema=None: (_ for _ in ()).throw(AssertionError("must reject first"))  # type: ignore
    with pytest.raises(NotImplementedError, match="multi-GPU"):
        dist.range_join(None, None, on=["k"], at="t", start="s", end="e")


class _Engine:
    """Records the range and hash join calls the SQL engine makes."""
    is_distributed = False

    def __init__(self):
        self.calls = []

    def to_df(self, df):
        return df

    def range_join(self, df1, df2, **kw):
        self.calls.append((df1, df2, kw))
        return df1

    def join(self, df1, df2, **kw):
        raise AssertionError("a range join must not reach the hash join")


@pytest.mark.parametrize("cond,on,closed", [
    ("a.k = b.k AND a.t BETWEEN b.s AND b.e", ["k"], "both"),
    ("a.t BETWEEN b.s AND b.e AND a.k = b.k", ["k"], "both"),
    ("(a.k = b.k) AND a.t between b.s and b.e", ["k"], "both"),
    ("a.t BETWEEN b.s AND b.e", [], "both"),
    ("a.k = b.k AND b.s <= a.t AND a.t < b.e", ["k"], "left"),
    ("a.k = b.k AND a.t < b.e AND b.s <= a.t", ["k"], "left"),
    ("a.k = b.k AND a.t >= b.s AND b.e > a.t", ["k"], "left"),
    ("b.s < a.t AND a.t <= b.e AND a.k = b.k", ["k"], "right"),
    ("a.t > b.s AND a.t < b.e", [], "neither"),
    ("b.e >= a.t AND b.s <= a.t", [], "both"),
    ("(b.s <= a.t) AND (a.t <= b.e) AND a.k = b.k AND a.j = b.j", ["k", "j"], "both"),
])
def test_sql_forms(cond, on, closed):
    from fugue_b200.sql import B200SQLEngine

    eng = _Engine()
    ta, tb = _DF("k:long,j:long,t:long"), _DF("k:long,j:long,s:long,e:long")
    for kind, how in (("", "inner"), ("INNER ", "inner"), ("LEFT ", "left_outer"), ("LEFT OUTER ", "left_outer")):
        B200SQLEngine(eng).select({"ta": ta, "tb": tb}, f"SELECT * FROM ta AS a {kind}JOIN tb b ON {cond}")
        d1, d2, kw = eng.calls[-1]
        assert d1 is ta and d2 is tb
        assert kw == dict(on=on, at="t", start="s", end="e", how=how, closed=closed)
    # table names, and qualifiers that name no table (raw_sql's generated names): the side the other operand
    # leaves, or FROM order
    B200SQLEngine(eng).select({"ta": ta, "tb": tb}, "SELECT * FROM ta JOIN tb ON tb.s <= ta.t AND ta.t <= tb.e")
    assert eng.calls[-1][2]["closed"] == "both"
    for c in ("x.t BETWEEN y.s AND y.e", "x.t BETWEEN b.s AND b.e", "a.t BETWEEN y.s AND y.e",
              "y.s <= x.t AND x.t < y.e", "b.s <= x.t AND x.t < y.e"):
        B200SQLEngine(eng).select({"ta": ta, "tb": tb}, f"SELECT * FROM ta a JOIN tb b ON x.k = y.k AND {c}")
        assert eng.calls[-1][2]["at"] == "t" and eng.calls[-1][2]["start"] == "s", c


@pytest.mark.parametrize("sql", [
    "SELECT * FROM ta a JOIN tb b ON a.k = b.k AND b.t BETWEEN a.s AND a.e",   # the interval on the left
    "SELECT * FROM ta a JOIN tb b ON a.k = b.k AND b.t >= a.s AND b.t <= a.e",
    "SELECT * FROM ta a JOIN tb b ON a.k = b.k AND a.t >= b.s",                # one inequality
    "SELECT * FROM ta a JOIN tb b ON a.k = b.k AND a.t >= b.s AND a.u <= b.e",  # two left columns
    "SELECT * FROM ta a JOIN tb b ON a.t >= b.s AND a.t >= b.e",               # two lower bounds
    "SELECT * FROM ta a JOIN tb b ON a.t BETWEEN b.s AND b.e AND a.t <= b.e",
    "SELECT * FROM ta a JOIN tb b ON a.t BETWEEN b.s AND b.e AND a.u BETWEEN b.s AND b.e",
    "SELECT * FROM ta a JOIN tb b ON a.t NOT BETWEEN b.s AND b.e",
    "SELECT * FROM ta a JOIN tb b ON a.t BETWEEN b.s - 5 AND b.e",             # arithmetic
    "SELECT * FROM ta a JOIN tb b ON a.t + 1 >= b.s AND a.t <= b.e",
    "SELECT * FROM ta a JOIN tb b ON a.t BETWEEN b.s AND b.e OR a.k = b.k",    # OR
    "SELECT * FROM ta a JOIN tb b ON a.t >= b.s AND a.t <= b.e OR a.k = b.k",
    "SELECT * FROM ta a JOIN tb b ON t BETWEEN s AND e",                       # unqualified
    "SELECT * FROM ta a JOIN tb b ON a.t >= s AND a.t <= b.e",
    "SELECT * FROM ta a JOIN tb b ON a.t BETWEEN a.s AND b.e",
    "SELECT * FROM ta a JOIN tb b ON a.t >= a.s AND a.t <= b.e",
    "SELECT * FROM ta a JOIN tb b ON a.k = b.j AND a.t BETWEEN b.s AND b.e",
    "SELECT * FROM ta a RIGHT JOIN tb b ON a.t BETWEEN b.s AND b.e",
    "SELECT * FROM ta a FULL OUTER JOIN tb b ON b.s <= a.t AND a.t <= b.e",
    "SELECT * FROM ta a LEFT SEMI JOIN tb b ON a.t BETWEEN b.s AND b.e",
    "SELECT * FROM ta a LEFT ANTI JOIN tb b ON a.t BETWEEN b.s AND b.e",
    "SELECT a.t FROM ta a JOIN tb b ON a.t BETWEEN b.s AND b.e",
    "SELECT * FROM ta a JOIN tb b ON a.k = a.k AND a.t BETWEEN b.s AND b.e",  # an equality within one table
    "SELECT * FROM ta a JOIN tb b ON b.k = b.k AND b.s <= a.t AND a.t < b.e",
])
def test_sql_rejections(sql):
    from fugue_b200.sql import B200SQLEngine

    eng = _Engine()
    with pytest.raises(NotImplementedError):
        B200SQLEngine(eng).select({"ta": _DF("k:long,t:long,u:long"), "tb": _DF("k:long,j:long,s:long,e:long")},
                                  sql)
    assert eng.calls == []


def test_plain_join_errors_are_unchanged():
    from fugue_b200.sql import B200SQLEngine

    for cond in ("a.k = b.k AND a.t >= b.s", "a.t BETWEEN b.s - 1 AND b.e", "b.t BETWEEN a.s AND a.e"):
        with pytest.raises(NotImplementedError, match="only equi-joins on equally named columns"):
            B200SQLEngine(_Engine()).select({"ta": _DF("k:long,t:long"), "tb": _DF("k:long,s:long,e:long")},
                                            f"SELECT * FROM ta a JOIN tb b ON {cond}")


class _Recorder(EngineLifecycle):
    """Every engine method records (name, args, kwargs) and returns a fixed frame."""
    is_distributed = False

    def __init__(self):
        self.conf = {}
        self.log = []

    def to_df(self, df, schema=None):
        return as_fugue_df(df, schema)

    def convert_yield_dataframe(self, df, as_local):
        self.log.append(("convert", as_local))
        return df

    def __getattr__(self, name):
        if name.startswith("_"):
            raise AttributeError(name)

        def method(*args, **kwargs):
            self.log.append((name, args, kwargs))
            return ArrowDataFrame([[len(self.log)]], "n:long")

        return method


def test_api_plumbing():
    eng = _Recorder()
    pdf1, pdf2 = pd.DataFrame({"k": [1], "t": [5]}), pd.DataFrame({"k": [1], "s": [4], "e": [6]})
    out = fa.range_join(pdf1, pdf2, on=("k",), at="t", start="s", end="e", engine=eng)
    assert isinstance(out, pd.DataFrame)
    name, (d1, d2), kw = eng.log[0]
    assert name == "range_join" and d1.schema == "k:long,t:long" and d2.schema == "k:long,s:long,e:long"
    assert kw == dict(on=["k"], at="t", start="s", end="e", how="inner", closed="both")
    assert eng.log[1] == ("convert", False)
    out = fa.range_join(pdf1, pdf2, on=None, at="t", start="s", end="e", how="left_outer", closed="left",
                        engine=eng, as_fugue=True, as_local=True)
    assert isinstance(out, DataFrame)
    assert eng.log[2][2] == dict(on=None, at="t", start="s", end="e", how="left_outer", closed="left")
    assert eng.log[3] == ("convert", True)
    assert isinstance(fa.range_join(ArrowDataFrame(pdf1), pdf2, [], "t", "s", "e", engine=eng), DataFrame)


def test_sql_join_keyword_is_not_an_alias():
    """``FROM a LEFT JOIN b`` (no alias, as raw_sql writes it) is a left outer join."""
    from fugue_b200.sql import B200SQLEngine

    eng = _Engine()
    ta, tb = _DF("k:long,t:long"), _DF("k:long,s:long,e:long")
    B200SQLEngine(eng).select({"ta": ta, "tb": tb}, "SELECT * FROM ta LEFT JOIN tb ON ta.t BETWEEN tb.s AND tb.e")
    assert eng.calls[-1][2] == dict(on=[], at="t", start="s", end="e", how="left_outer", closed="both")
    B200SQLEngine(eng).select({"ta": ta, "tb": tb}, "SELECT * FROM ta INNER JOIN tb ON ta.t BETWEEN tb.s AND tb.e")
    assert eng.calls[-1][2]["how"] == "inner"
