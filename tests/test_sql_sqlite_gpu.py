"""SQL joins and SELECT clauses on the H100 against SQLite (the standard library's, >= 3.39 for RIGHT and FULL
joins): each statement runs through the B200 SQL engine on the device and in an in-memory SQLite database loaded
from the same Arrow tables, and the two answers are compared as multisets of rows, or as sequences where the
statement's ORDER BY gives a total order.

a. every join spelling the SQL engine accepts gives SQLite's rows, and the texts it used to read as another join
   raise NotImplementedError;
b. join keys of every type through SQL (uint64 at and above 2^63 against ``oracle/join.py``: SQLite has no such
   integer);
c. every hash-join path reached from SQL: the fused kernel, the join table, the radix path (both sides at
   ``RADIX_JOIN_MIN_ROWS``);
d. range joins (``ON a.k = b.k AND a.t BETWEEN b.s AND b.e`` and the two-inequality forms) with NULL and reversed
   intervals;
e. seeded combinations of WHERE, GROUP BY, HAVING, DISTINCT, ORDER BY and LIMIT over one table with NULLs, one of
   them above ``GROUPBY_PARTITION_MIN_ROWS`` so the partitioned group-by runs.

SQLite's text is written for the engine's output schema: df1's columns, then df2's non-key columns; the keys of a
RIGHT or FULL join are ``COALESCE(a.k, b.k)``, SEMI is ``WHERE EXISTS``, ANTI ``WHERE NOT EXISTS``.  Temporal
columns compare as their storage integers, a bool as 0 / 1, and a device NaN as NULL (SQLite stores a NaN as NULL;
the engine's join never matches a NaN key, as it never matches a NULL).  -0.0 compares equal to 0.0.

Left out, because the two engines differ on purpose:
- integer ``/`` and ``%``: SQLite truncates, the engine divides to a double and takes a floored modulo
  (DESIGN §7e);
- LIKE's case rules: SQLite ignores ASCII case unless ``PRAGMA case_sensitive_like = ON``, which these tests set;
- backslashes in string literals: the engine's ``sql._unquote`` resolves escapes, SQLite keeps the backslash;
- integer overflow: SQLite raises, the engine wraps; the values here keep every sum far from 2^63;
- uint64 values at or above 2^63: SQLite has no such integer (part b compares them with ``oracle/join.py``);
- ordering comparisons of two strings and a NULL inside a string IN list: the engine raises NotImplementedError;
- the float sums are of dyadic values (multiples of 1/4 below 2^20), so every SUM and AVG is exact in both.
"""
import datetime
import sqlite3
from collections import Counter
from typing import Any, Dict, List

import numpy as np
import pyarrow as pa
import pytest

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(sqlite3.sqlite_version_info < (3, 39), reason="needs SQLite >= 3.39")]
torch = pytest.importorskip("torch")

from fugue_b200 import api as fa
from fugue_b200 import join as J
from fugue_b200 import kernels as K
from fugue_b200.dataframe import B200DataFrame
from fugue_b200.schema import SchemaError
from fugue_b200.table import B200Table
from oracle import join as oj

DEV = torch.device("cuda", 0)
_ENGINE: List[Any] = []
HOWS = ["inner", "left_outer", "right_outer", "full_outer", "semi", "anti"]


def _engine():
    if not _ENGINE:
        _ENGINE.append(fa.make_execution_engine("b200"))
    return _ENGINE[0]


def _df(tbl: pa.Table) -> B200DataFrame:
    return B200DataFrame(B200Table.from_arrow(tbl, DEV))


def _device(tables: Dict[str, pa.Table], sql: str) -> pa.Table:
    res = _engine().sql_engine.select({n: _df(t) for n, t in tables.items()}, sql)
    return res.native.to_arrow()


def _storage(c: Any) -> Any:
    """A column as SQLite holds it: temporal values as their storage integers."""
    if pa.types.is_date32(c.type):
        return c.cast(pa.int32())
    if pa.types.is_timestamp(c.type) or pa.types.is_date64(c.type):
        return c.cast(pa.int64())
    return c


def _value(v: Any) -> Any:
    if isinstance(v, float):
        return None if v != v else v + 0.0  # NaN is NULL; -0.0 is 0.0
    return v


def _rows(t: pa.Table) -> List[tuple]:
    cols = [_storage(t.column(i)).to_pylist() for i in range(t.num_columns)]
    return [tuple(_value(v) for v in r) for r in zip(*cols)]


def _connect(tables: Dict[str, pa.Table], index: Any = ()) -> sqlite3.Connection:
    con = sqlite3.connect(":memory:")
    con.execute("PRAGMA case_sensitive_like = ON")
    for name, t in tables.items():
        cols = t.column_names
        con.execute(f"CREATE TABLE {name} ({', '.join(cols)})")
        con.executemany(f"INSERT INTO {name} VALUES ({', '.join('?' * len(cols))})",
                        zip(*[_storage(t[c]).to_pylist() for c in cols]))
    for name, cols in index:
        con.execute(f"CREATE INDEX ix_{name} ON {name} ({', '.join(cols)})")
    return con


def _sqlite(con: sqlite3.Connection, sql: str) -> List[tuple]:
    return [tuple(_value(v) for v in r) for r in con.execute(sql).fetchall()]


def _same(got: List[tuple], want: List[tuple], ordered: bool, what: str) -> None:
    if ordered:
        assert got == want, f"{what}\n got  {got[:5]}\n want {want[:5]}"
    else:
        g, w = Counter(got), Counter(want)
        assert g == w, (f"{what}\n {sum(g.values())} rows, want {sum(w.values())}; extra "
                        f"{list((g - w).items())[:3]}, missing {list((w - g).items())[:3]}")


def _join_sqlite(how: str, keys: List[str], left: pa.Table, right: pa.Table) -> str:
    """SQLite's text of ``ta a <how> JOIN tb b`` on ``keys``, in the engine's output schema."""
    outer_key = how in ("right_outer", "full_outer")
    sel = [f"COALESCE(a.{c}, b.{c})" if c in keys and outer_key else f"a.{c}" for c in left.column_names]
    cond = " AND ".join(f"a.{k} = b.{k}" for k in keys)
    if how in ("semi", "anti"):
        return (f"SELECT {', '.join(sel)} FROM ta a WHERE {'' if how == 'semi' else 'NOT '}EXISTS "
                f"(SELECT 1 FROM tb b WHERE {cond})")
    sel += [f"b.{c}" for c in right.column_names if c not in keys]
    if how == "cross":
        return f"SELECT {', '.join(sel)} FROM ta a CROSS JOIN tb b"
    kw = {"inner": "INNER", "left_outer": "LEFT", "right_outer": "RIGHT", "full_outer": "FULL"}[how]
    return f"SELECT {', '.join(sel)} FROM ta a {kw} JOIN tb b ON {cond}"


def _check_join(left: pa.Table, right: pa.Table, from_text: str, how: str, keys: List[str],
                con: Any = None) -> None:
    con = con or _connect({"ta": left, "tb": right})
    sql = f"SELECT * FROM {from_text}"
    got = _device({"ta": left, "tb": right}, sql)
    _same(_rows(got), _sqlite(con, _join_sqlite(how, keys, left, right)), False, sql)


# ---- a. every accepted join spelling -----------------------------------------------------------------------------
def _spelling_tables(seed: int = 0):
    rng = np.random.default_rng(seed)
    n1, n2 = 300, 200
    left = pa.table({"k": pa.array(rng.integers(0, 40, n1), mask=rng.random(n1) < 0.1),
                     "j": pa.array(np.array(["x", "y", "", "é"])[rng.integers(0, 4, n1)], mask=rng.random(n1) < 0.1),
                     "v": pa.array(rng.integers(-2**20, 2**20, n1) / 4.0, mask=rng.random(n1) < 0.1)})
    right = pa.table({"k": pa.array(rng.integers(20, 60, n2), mask=rng.random(n2) < 0.1),
                      "j": pa.array(np.array(["y", "", "z", "é"])[rng.integers(0, 4, n2)], mask=rng.random(n2) < 0.1),
                      "w": pa.array(rng.integers(-1000, 1000, n2), mask=rng.random(n2) < 0.1)})
    return left, right


SPELLINGS = [
    ("ta JOIN tb ON ta.k = tb.k", "inner", ["k"]),
    ("ta INNER JOIN tb USING (k)", "inner", ["k"]),
    ("ta AS a JOIN tb AS b ON a.k = b.k AND a.j = b.j", "inner", ["k", "j"]),
    ("ta a inner join tb b on b.k = a.k", "inner", ["k"]),
    ("ta LEFT JOIN tb ON ta.k = tb.k", "left_outer", ["k"]),
    ("ta a LEFT OUTER JOIN tb b USING (k, j)", "left_outer", ["k", "j"]),
    ("ta\n  a\n  left\n  outer join tb b\n  on (a.k = b.k)", "left_outer", ["k"]),
    ("ta RIGHT JOIN tb ON tb.k = ta.k", "right_outer", ["k"]),
    ("ta a RIGHT OUTER JOIN tb AS b ON (a.j = b.j) AND (b.k = a.k)", "right_outer", ["j", "k"]),
    ("ta FULL JOIN tb USING (j)", "full_outer", ["j"]),
    ("`ta` a FULL OUTER JOIN `tb` b ON `a`.`k` = `b`.`k`", "full_outer", ["k"]),
    ("ta full outer join tb on ta.k = tb.k and ta.j = tb.j", "full_outer", ["k", "j"]),
    ("ta SEMI JOIN tb ON ta.k = tb.k", "semi", ["k"]),
    ("ta a LEFT SEMI JOIN tb b USING (k, j)", "semi", ["k", "j"]),
    ("ta ANTI JOIN tb b ON ta.k = b.k", "anti", ["k"]),
    ("ta AS a left anti join tb ON a.j = tb.j", "anti", ["j"]),
    ("ta JOIN tb ON k = k", "inner", ["k"]),
    # the texts that used to run another join and now run the one SQLite runs
    ("ta a LEFT JOIN tb b ON a.k = b.k AND a.k = b.k", "left_outer", ["k"]),
    ("ta NATURAL JOIN tb", "inner", ["k", "j"]),
    ("ta NATURAL LEFT JOIN tb", "left_outer", ["k", "j"]),
    ("ta a NATURAL FULL OUTER JOIN tb b", "full_outer", ["k", "j"]),
]


@pytest.mark.parametrize("from_text,how,keys", SPELLINGS)
def test_join_spelling(from_text, how, keys):
    left, right = _spelling_tables()
    common = [c for c in right.column_names if c in left.column_names and c not in keys]
    if common and how not in ("semi", "anti"):  # a column of both tables in the output must be a key
        with pytest.raises(SchemaError):
            _device({"ta": left, "tb": right}, f"SELECT * FROM {from_text}")
    right = right.drop_columns(common)
    _check_join(left, right, from_text, how, keys)


def test_cross_join_spellings():
    rng = np.random.default_rng(1)
    left = pa.table({"x": pa.array(rng.integers(0, 9, 40), mask=rng.random(40) < 0.2), "y": np.arange(40.0)})
    right = pa.table({"z": pa.array(np.array(["p", "", "日本"])[rng.integers(0, 3, 30)], mask=rng.random(30) < 0.2)})
    con = _connect({"ta": left, "tb": right})
    for text in ("ta CROSS JOIN tb", "ta a CROSS JOIN tb b", "ta AS a cross join tb AS b"):
        got = _device({"ta": left, "tb": right}, f"SELECT * FROM {text}")
        _same(_rows(got), _sqlite(con, _join_sqlite("cross", [], left, right)), False, text)


@pytest.mark.parametrize("from_text", [
    "ta OUTER JOIN tb USING (k)",
    "ta CROSS JOIN tb ON ta.k = tb.k",
    "ta JOIN tb ON ta.k = ta.k",
    "ta JOIN tb ON z.k = q.k",
    "ta JOIN tb",
    "ta LEFT JOIN tb",
    "ta NATURAL JOIN tb USING (k)",
])
def test_join_texts_that_used_to_run_another_join(from_text):
    left, right = _spelling_tables()
    with pytest.raises(NotImplementedError):
        _device({"ta": left, "tb": right}, f"SELECT * FROM {from_text}")


def test_raw_sql_dataframes_and_aliases():
    """``fa.raw_sql``'s dataframes have generated names: qualifiers may name them by alias, or by any name."""
    left, right = _spelling_tables(2)
    right = right.drop_columns(["j"])
    con = _connect({"ta": left, "tb": right})
    for pieces, how in ((("SELECT * FROM", left, "LEFT JOIN", right, "ON l.k = r.k"), "left_outer"),
                        (("SELECT * FROM", left, "AS a FULL JOIN", right, "AS b ON a.k = b.k"), "full_outer"),
                        (("SELECT * FROM", left, "a RIGHT JOIN", right, "ON b.k = a.k"), "right_outer")):
        got = fa.raw_sql(*[_df(p) if isinstance(p, pa.Table) else p for p in pieces], engine=_engine(),
                         as_fugue=True).native.to_arrow()
        _same(_rows(got), _sqlite(con, _join_sqlite(how, ["k"], left, right)), False, str(pieces[2:]))


# ---- b. keys of every type ---------------------------------------------------------------------------------------
def _key(name: str, n: int, rng, side: int) -> pa.Array:
    mask = rng.random(n) < 0.08
    if name.startswith("int") or name.startswith("uint"):
        tp = getattr(pa, name)()
        info = np.iinfo(np.dtype(name))
        vals = np.concatenate([[info.min, info.max, 0], rng.integers(max(info.min, -30), 30, n)])[:n]
        return pa.array(vals.astype(name), mask=mask, type=tp)
    if name.startswith("float"):
        pool = np.array([-0.0, 0.0, np.nan, 1.5, -2.25, np.inf, 3.0, 1e30, -7.0], dtype=name)
        return pa.array(pool[rng.integers(0, len(pool), n)], mask=mask)
    if name == "string":
        pool = [["", "a", "é", "日本", "ab", "x" * 20], ["ab", "日本", "", "zz", "é", "b"]][side]
        return pa.array(np.array(pool)[rng.integers(0, len(pool), n)], mask=mask)
    if name == "bool":
        return pa.array(rng.random(n) < 0.5, mask=mask)
    if name == "date32":
        return pa.array(rng.integers(18000, 18040, n).astype("int32"), mask=mask).cast(pa.date32())
    if name == "timestamp_us":
        return pa.array(rng.integers(0, 50, n) * 1_000_003, mask=mask).cast(pa.timestamp("us"))
    if name == "timestamp_ns_utc":
        return pa.array(rng.integers(0, 50, n) * 999_999_937, mask=mask).cast(pa.timestamp("ns", "UTC"))
    raise ValueError(name)


KEY_TYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "float32", "float64", "string", "bool",
             "date32", "timestamp_us", "timestamp_ns_utc"]


@pytest.mark.parametrize("name", KEY_TYPES)
def test_key_types(name):
    rng = np.random.default_rng(KEY_TYPES.index(name))
    n1, n2 = 1500, 900
    left = pa.table({"k": _key(name, n1, rng, 0), "v": np.arange(n1)})
    right = pa.table({"k": _key(name, n2, rng, 1), "w": np.arange(n2) * 2.0})
    con = _connect({"ta": left, "tb": right})
    for how in HOWS:
        kw = {"inner": "", "left_outer": "LEFT ", "right_outer": "RIGHT ", "full_outer": "FULL OUTER ",
              "semi": "LEFT SEMI ", "anti": "LEFT ANTI "}[how]
        _check_join(left, right, f"ta a {kw}JOIN tb b ON a.k = b.k", how, ["k"], con)


@pytest.mark.parametrize("names", [["int64", "string"], ["int32", "float64", "date32"], ["string", "bool", "uint16"]])
def test_multi_column_keys(names):
    """Two and three key columns: a hashed surrogate key whose matches are verified column by column."""
    rng = np.random.default_rng(len(names))
    n1, n2 = 3000, 2000
    keys = [f"k{i}" for i in range(len(names))]
    left = pa.table({**{k: _key(t, n1, rng, 0) for k, t in zip(keys, names)}, "v": np.arange(n1)})
    right = pa.table({**{k: _key(t, n2, rng, 1) for k, t in zip(keys, names)}, "w": np.arange(n2) - 5})
    con = _connect({"ta": left, "tb": right})
    cond = " AND ".join(f"a.{k} = b.{k}" for k in keys)
    for how in HOWS:
        kw = {"inner": "INNER", "left_outer": "LEFT", "right_outer": "RIGHT", "full_outer": "FULL",
              "semi": "SEMI", "anti": "ANTI"}[how]
        _check_join(left, right, f"ta a {kw} JOIN tb b ON {cond}", how, keys, con)
        _check_join(left, right, f"ta {kw} JOIN tb USING ({', '.join(reversed(keys))})", how, keys, con)


def test_uint64_keys_at_and_above_2_63():
    rng = np.random.default_rng(5)
    pool = np.array([0, 1, 2**63 - 1, 2**63, 2**63 + 1, 2**64 - 1, 12345], dtype=np.uint64)
    n1, n2 = 700, 500
    left = pa.table({"k": pa.array(pool[rng.integers(0, 7, n1)], mask=rng.random(n1) < 0.1), "v": np.arange(n1)})
    right = pa.table({"k": pa.array(pool[rng.integers(0, 7, n2)], mask=rng.random(n2) < 0.1), "w": np.arange(n2)})
    for how in HOWS:
        kw = {"inner": "JOIN", "left_outer": "LEFT JOIN", "right_outer": "RIGHT OUTER JOIN",
              "full_outer": "FULL JOIN", "semi": "SEMI JOIN", "anti": "ANTI JOIN"}[how]
        got = _device({"ta": left, "tb": right}, f"SELECT * FROM ta {kw} tb ON ta.k = tb.k")
        assert oj.rows_of(got) == oj.join_rows(left, right, how, ["k"]), how


# ---- c. every hash-join path from SQL ----------------------------------------------------------------------------
@pytest.mark.parametrize("ncols", [2, K.JOIN2_MAX_COLS + 1], ids=["fused", "wide"])
def test_fused_and_join_table_paths(ncols):
    """One int64 key: inner / left outer through the fused kernel (or, with more columns than it takes, the join
    table), right / full / semi / anti through the join table."""
    rng = np.random.default_rng(ncols)
    n1, n2 = 40_000, 30_000
    left = pa.table({"k": pa.array(rng.integers(0, 20_000, n1), mask=rng.random(n1) < 0.05),
                     **{f"v{i}": pa.array(rng.integers(0, 100, n1), mask=rng.random(n1) < 0.1)
                        for i in range(ncols - 1)}})
    right = pa.table({"k": pa.array(rng.integers(10_000, 30_000, n2), mask=rng.random(n2) < 0.05),
                      "w": pa.array(rng.integers(0, 2**20, n2) / 4.0, mask=rng.random(n2) < 0.1)})
    con = _connect({"ta": left, "tb": right}, [("ta", ["k"]), ("tb", ["k"])])
    for how in HOWS:
        kw = {"inner": "", "left_outer": "LEFT ", "right_outer": "RIGHT ", "full_outer": "FULL ",
              "semi": "SEMI ", "anti": "ANTI "}[how]
        _check_join(left, right, f"ta {kw}JOIN tb USING (k)", how, ["k"], con)


def _pairs(got: pa.Table) -> np.ndarray:
    """(left row, right row) of every output row, -1 for a missing side, sorted."""
    li = np.asarray(got["v"].fill_null(-1))
    ri = np.asarray(got["w"].fill_null(-1)) if "w" in got.column_names else np.full(len(li), -1)
    p = np.stack([li, ri], axis=1)
    return p[np.lexsort((p[:, 1], p[:, 0]))]


def test_radix_path():
    """Both sides at RADIX_JOIN_MIN_ROWS: every join type through the radix-partitioned path.  SQLite takes minutes
    over 2 M rows a side, so the rows are compared with ``oracle/join.py``'s numpy join: v and w are the row
    numbers of each side, so an output row is the pair of rows it joins, and its key must be that of its row."""
    n = J.RADIX_JOIN_MIN_ROWS
    rng = np.random.default_rng(9)
    k1 = pa.array(rng.integers(0, 3 * n // 2, n), mask=rng.random(n) < 0.02)
    k2 = pa.array(rng.integers(n // 2, 2 * n, n), mask=rng.random(n) < 0.02)
    left, right = pa.table({"k": k1, "v": np.arange(n)}), pa.table({"k": k2, "w": np.arange(n)})
    kl, vl = np.asarray(k1.fill_null(0)), np.asarray(k1.is_valid())
    kr, vr = np.asarray(k2.fill_null(0)), np.asarray(k2.is_valid())
    nl, nr = np.asarray(k1.fill_null(-1)), np.asarray(k2.fill_null(-1))  # keys with NULL as -1
    lo, ro = oj.join_pairs(kl, vl, kr, vr, outer=True)      # every left row, and its matches
    rr, rl = oj.join_pairs(kr, vr, kl, vl, outer=True)      # every right row, and its matches
    hit = np.zeros(n, bool)
    hit[lo[ro >= 0]] = True
    want = {"inner": (lo[ro >= 0], ro[ro >= 0]), "left_outer": (lo, ro), "right_outer": (rl, rr),
            "full_outer": (np.concatenate([lo, rl[rl < 0]]), np.concatenate([ro, rr[rl < 0]])),
            "semi": (np.flatnonzero(hit), None), "anti": (np.flatnonzero(~hit), None)}
    for how in HOWS:
        kw = {"inner": "INNER", "left_outer": "LEFT OUTER", "right_outer": "RIGHT OUTER",
              "full_outer": "FULL OUTER", "semi": "LEFT SEMI", "anti": "LEFT ANTI"}[how]
        got = _device({"ta": left, "tb": right}, f"SELECT * FROM ta a {kw} JOIN tb b ON a.k = b.k")
        li, ri = want[how]
        p = np.stack([li, np.full(len(li), -1) if ri is None else ri], axis=1)
        assert np.array_equal(_pairs(got), p[np.lexsort((p[:, 1], p[:, 0]))]), how
        key = np.where(np.asarray(got["v"].fill_null(-1)) >= 0, nl[np.asarray(got["v"].fill_null(0))],
                       nr[np.asarray(got["w"].fill_null(0))] if "w" in got.column_names else -1)
        assert np.array_equal(np.asarray(got["k"].fill_null(-1)), key), how


# ---- d. range joins ----------------------------------------------------------------------------------------------
RANGE_FORMS = {  # closed -> (device condition, SQLite condition)
    "both": ("a.t BETWEEN b.s AND b.e", "a.t BETWEEN b.s AND b.e"),
    "left": ("b.s <= a.t AND a.t < b.e", "b.s <= a.t AND a.t < b.e"),
    "right": ("a.t <= b.e AND b.s < a.t", "a.t <= b.e AND b.s < a.t"),
    "neither": ("b.e > a.t AND a.t > b.s", "b.e > a.t AND a.t > b.s"),
}


@pytest.mark.parametrize("closed", list(RANGE_FORMS))
@pytest.mark.parametrize("keyed", [True, False], ids=["keyed", "no_key"])
def test_range_join(closed, keyed):
    rng = np.random.default_rng(len(closed) + keyed)
    n1, n2 = (4000, 600) if keyed else (500, 120)
    s = rng.integers(0, 1000, n2)
    e = s + rng.integers(-20, 60, n2)  # some intervals reversed: they hold nothing
    left = pa.table({"k": pa.array(rng.integers(0, 8, n1), mask=rng.random(n1) < 0.05),
                     "t": pa.array(rng.integers(-10, 1100, n1), mask=rng.random(n1) < 0.05),
                     "v": np.arange(n1)})
    right = pa.table({"k": pa.array(rng.integers(0, 8, n2), mask=rng.random(n2) < 0.05),
                      "s": pa.array(s, mask=rng.random(n2) < 0.05), "e": pa.array(e, mask=rng.random(n2) < 0.05),
                      "w": rng.integers(0, 2**20, n2) / 4.0})
    if not keyed:
        right = right.rename_columns(["kb", "s", "e", "w"])
    con = _connect({"ta": left, "tb": right})
    dev, ref = RANGE_FORMS[closed]
    if keyed:
        dev, ref = f"a.k = b.k AND {dev}", f"{ref} AND b.k = a.k"
    cols = ", ".join([f"a.{c}" for c in left.column_names] +
                     [f"b.{c}" for c in right.column_names if not (keyed and c == "k")])
    for kw in ("", "LEFT "):
        sql = f"SELECT * FROM ta a {kw}JOIN tb b ON {dev}"
        got = _device({"ta": left, "tb": right}, sql)
        _same(_rows(got), _sqlite(con, f"SELECT {cols} FROM ta a {kw}JOIN tb b ON {ref}"), False, sql)


def test_range_join_on_dates():
    rng = np.random.default_rng(21)
    n1, n2 = 2000, 300
    s = rng.integers(18000, 18300, n2)
    left = pa.table({"k": rng.integers(0, 4, n1), "t": pa.array(rng.integers(17990, 18400, n1).astype("int32"),
                                                                mask=rng.random(n1) < 0.05).cast(pa.date32())})
    right = pa.table({"k": rng.integers(0, 4, n2),
                      "s": pa.array(s.astype("int32"), mask=rng.random(n2) < 0.05).cast(pa.date32()),
                      "e": pa.array((s + rng.integers(-5, 40, n2)).astype("int32")).cast(pa.date32())})
    con = _connect({"ta": left, "tb": right})
    for kw in ("INNER ", "LEFT OUTER "):
        sql = f"SELECT * FROM ta a {kw}JOIN tb b ON b.k = a.k AND a.t >= b.s AND a.t < b.e"
        got = _device({"ta": left, "tb": right}, sql)
        _same(_rows(got), _sqlite(con, f"SELECT a.k, a.t, b.s, b.e FROM ta a {kw}JOIN tb b "
                                       f"ON b.k = a.k AND a.t >= b.s AND a.t < b.e"), False, sql)


# ---- e. SELECT clauses in combination ----------------------------------------------------------------------------
def _days(iso: str) -> int:
    return (datetime.date.fromisoformat(iso) - datetime.date(1970, 1, 1)).days


_D0 = _days("2020-12-05")


def _select_table(rng, n: int) -> pa.Table:
    words = np.array(["", "a", "bb", "Bb", "b%", "é", "日本", "abc", "zz"])
    return pa.table({
        "rid": np.arange(n, dtype=np.int64),
        "g1": pa.array(rng.integers(0, 6, n), mask=rng.random(n) < 0.1),
        "g2": pa.array(words[rng.integers(0, 4, n)], mask=rng.random(n) < 0.1),
        "i": pa.array(rng.integers(-50, 51, n), mask=rng.random(n) < 0.15),
        "f": pa.array(rng.integers(-2**20, 2**20, n) / 4.0, mask=rng.random(n) < 0.15),
        "s": pa.array(words[rng.integers(0, len(words), n)], mask=rng.random(n) < 0.1),
        "d": pa.array((_D0 + rng.integers(0, 400, n)).astype("int32"), mask=rng.random(n) < 0.1).cast(pa.date32()),
    })


# (device text, SQLite text) of WHERE atoms; NULL operands make many of them NULL
_ATOMS = [
    ("i > 10", None), ("i <= -5", None), ("f < 0.5", None), ("f >= -1000.25", None), ("i = g1", None),
    ("i <> g1", None), ("i IN (1, 2, 3, NULL)", None), ("i NOT IN (1, 2, NULL)", None), ("g1 IN (0, 2, 5)", None),
    ("g1 NOT IN (1, 3)", None), ("i BETWEEN -10 AND 20", None), ("i NOT BETWEEN -10 AND 20", None),
    ("f BETWEEN -100000.25 AND 1000.5", None), ("i BETWEEN g1 AND 30", None), ("s = 'bb'", None),
    ("s <> ''", None), ("s IS NULL", None), ("f IS NOT NULL", None), ("i IS NULL", None), ("s LIKE 'b%'", None),
    ("s NOT LIKE '%é%'", None), ("g2 LIKE 'B_'", None), ("s IN ('a', 'zz')", None), ("s NOT IN ('', 'bb')", None),
    ("d >= DATE '2021-03-01'", f"d >= {_days('2021-03-01')}"),
    ("d BETWEEN DATE '2021-01-10' AND DATE '2021-06-30'", f"d BETWEEN {_days('2021-01-10')} AND {_days('2021-06-30')}"),
    ("d NOT BETWEEN DATE '2021-01-10' AND DATE '2021-06-30'",
     f"d NOT BETWEEN {_days('2021-01-10')} AND {_days('2021-06-30')}"),
    ("i + g1 > 5", None), ("f * 2 >= i", None), ("i - 3 * g1 < 0", None), ("i > 1000", None),
]


def _atom(rng):
    dev, ref = _ATOMS[rng.integers(0, len(_ATOMS))]
    return dev, ref or dev


def _pred(rng, depth: int = 0):
    r = rng.integers(0, 6 if depth < 2 else 1)
    if r == 0 or depth >= 2:
        return _atom(rng)
    a, b = _pred(rng, depth + 1), _pred(rng, depth + 1)
    if r in (1, 2):
        return f"({a[0]}) AND ({b[0]})", f"({a[1]}) AND ({b[1]})"
    if r in (3, 4):
        return f"({a[0]}) OR ({b[0]})", f"({a[1]}) OR ({b[1]})"
    return f"NOT (({a[0]}) OR ({b[0]}))", f"NOT (({a[1]}) OR ({b[1]}))"


_AGGS = ["COUNT(*) AS c", "COUNT(i) AS ci", "COUNT(s) AS cs", "SUM(i) AS si", "SUM(f) AS sf", "MIN(i) AS mi",
         "MAX(i) AS xi", "MIN(f) AS mf", "MAX(f) AS xf", "AVG(f) AS af", "AVG(i) AS ai", "MIN(s) AS ms",
         "MAX(s) AS xs", "MIN(d) AS md", "MAX(d) AS xd"]
_HAVING = ["COUNT(*) > 3", "SUM(i) > 0", "MAX(f) IS NOT NULL", "AVG(i) < 1", "MIN(s) = ''", "COUNT(i) >= COUNT(f)"]
# (select-list keys, GROUP BY text, output names that order the groups totally)
_KEYS = [("g1", "g1", ["g1"]), ("g2", "g2", ["g2"]), ("g1, g2", "g1, g2", ["g1", "g2"]),
         ("g2, g1", "g1, g2", ["g2", "g1"]), ("g1 + 1 AS ge", "g1 + 1", ["ge"]),
         ("g1 * 2 + i AS ge", "g1 * 2 + i", ["ge"]), ("", "g1", None), ("g2", "g2, g1", None)]


def _order(names: List[str], rng, nulls: bool = True):
    dirs = [" DESC" if rng.random() < 0.5 else "" for _ in names]
    dev = ", ".join(n + d for n, d in zip(names, dirs))
    ref = ", ".join(f"{n}{d}{' NULLS LAST' if nulls else ''}" for n, d in zip(names, dirs))
    return dev, ref


def _statements(seed: int, count: int):
    """(device SQL, SQLite SQL, ordered) over table t."""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < count:
        kind = rng.integers(0, 6)
        w, wr = _pred(rng)
        where = rng.random() < 0.7
        wd, wref = (f" WHERE {w}", f" WHERE {wr}") if where else ("", "")
        if kind == 0:
            out.append((f"SELECT rid, g1, i, f, s, d FROM t{wd}", f"SELECT rid, g1, i, f, s, d FROM t{wref}", False))
        elif kind == 1:
            o, orf = _order(["i", "rid"], rng)
            lim = int(rng.integers(0, 60))
            out.append((f"SELECT rid, i, s, f + i AS x FROM t{wd} ORDER BY {o} LIMIT {lim}",
                        f"SELECT rid, i, s, f + i AS x FROM t{wref} ORDER BY {orf} LIMIT {lim}", True))
        elif kind == 2:
            cols = ["g1", "g2", "s"][:int(rng.integers(1, 4))]
            sel = ", ".join(cols)
            if rng.random() < 0.5:
                o, orf = _order(cols, rng)
                lim = int(rng.integers(1, 20))
                out.append((f"SELECT DISTINCT {sel} FROM t{wd} ORDER BY {o} LIMIT {lim}",
                            f"SELECT DISTINCT {sel} FROM t{wref} ORDER BY {orf} LIMIT {lim}", True))
            else:
                out.append((f"SELECT DISTINCT {sel} FROM t{wd}", f"SELECT DISTINCT {sel} FROM t{wref}", False))
        elif kind == 3:
            aggs = ", ".join(_AGGS[j] for j in sorted(rng.choice(len(_AGGS), int(rng.integers(1, 5)), replace=False)))
            out.append((f"SELECT {aggs} FROM t{wd}", f"SELECT {aggs} FROM t{wref}", False))
        else:
            sel_keys, group, order = _KEYS[rng.integers(0, len(_KEYS))]
            # at most three aggregates: with HAVING's and the hidden keys they stay within one group-by kernel call
            aggs = ", ".join(_AGGS[j] for j in sorted(rng.choice(len(_AGGS), int(rng.integers(1, 4)), replace=False)))
            sel = f"{sel_keys}, {aggs}" if sel_keys else aggs
            having = f" HAVING {_HAVING[rng.integers(0, len(_HAVING))]}" if rng.random() < 0.4 else ""
            dev = f"SELECT {sel} FROM t{wd} GROUP BY {group}{having}"
            ref = f"SELECT {sel} FROM t{wref} GROUP BY {group}{having}"
            if order is not None and rng.random() < 0.5:
                o, orf = _order(order, rng)
                lim = f" LIMIT {int(rng.integers(1, 8))}" if rng.random() < 0.5 else ""
                out.append((f"{dev} ORDER BY {o}{lim}", f"{ref} ORDER BY {orf}{lim}", True))
            else:
                out.append((dev, ref, False))
    return out


def _check_statements(tbl: pa.Table, statements) -> None:
    con = _connect({"t": tbl})
    df = _df(tbl)
    for dev, ref, ordered in statements:
        got = _engine().sql_engine.select({"t": df}, dev).native.to_arrow()
        _same(_rows(got), _sqlite(con, ref), ordered, f"{dev}\n  SQLite: {ref}")


@pytest.mark.parametrize("seed", range(6))
def test_select_clauses(seed):
    rng = np.random.default_rng(100 + seed)
    _check_statements(_select_table(rng, int(rng.integers(1, 5000)) if seed else 1), _statements(seed, 50))


def test_select_clauses_on_the_partitioned_group_by():
    n = K.GROUPBY_PARTITION_MIN_ROWS
    rng = np.random.default_rng(77)
    tbl = pa.table({"g1": pa.array(rng.integers(0, 200_000, n), mask=rng.random(n) < 0.01),
                    "g2": pa.array(rng.integers(0, 3, n)),
                    "i": pa.array(rng.integers(-50, 51, n), mask=rng.random(n) < 0.1),
                    "f": pa.array(rng.integers(-2**20, 2**20, n) / 4.0, mask=rng.random(n) < 0.1)})
    _check_statements(tbl, [
        ("SELECT g1, COUNT(*) AS c, SUM(i) AS si, MIN(f) AS mf, AVG(f) AS af FROM t GROUP BY g1",
         "SELECT g1, COUNT(*) AS c, SUM(i) AS si, MIN(f) AS mf, AVG(f) AS af FROM t GROUP BY g1", False),
        ("SELECT g1, g2, MAX(i) AS xi, SUM(f) AS sf FROM t WHERE i IS NOT NULL OR f > 0 GROUP BY g1, g2 "
         "HAVING COUNT(*) > 20 ORDER BY g1 DESC, g2 LIMIT 500",
         "SELECT g1, g2, MAX(i) AS xi, SUM(f) AS sf FROM t WHERE i IS NOT NULL OR f > 0 GROUP BY g1, g2 "
         "HAVING COUNT(*) > 20 ORDER BY g1 DESC NULLS LAST, g2 NULLS LAST LIMIT 500", True),
    ])
