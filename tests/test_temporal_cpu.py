"""Date and timestamp expressions without a GPU: builders, SQL text, the oracle against independent calendars, and the
compiler's programs run through the numpy machine model (tests/_temporal_sim.py) against the oracle."""
import datetime as dt
import sqlite3

import numpy as np
import pandas as pd
import pyarrow as pa
import pyarrow.compute as pc
import pytest
import torch

import _temporal_sim as tsim
from fugue_b200 import expr as X
from fugue_b200 import kernels as K
from fugue_b200.column import SelectColumns, col, function, functions as f, lit, to_sql
from fugue_b200.schema import Schema
from fugue_b200.sql import _parse_select, _top_level_from
from fugue_b200.table import B200Table, expr_type
from oracle import expressions as OX
from oracle import scalar as OS
from oracle import temporal as OT

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
UNITS = {"D": pa.date32(), "s": pa.timestamp("s"), "ms": pa.timestamp("ms"), "us": pa.timestamp("us"),
         "ns": pa.timestamp("ns", tz="UTC")}
CODE = {"D": K.TU_DAY, "s": K.TU_S, "ms": K.TU_MS, "us": K.TU_US, "ns": K.TU_NS}


def edge_days():
    """Day counts around every calendar rule: the epoch, leap days of 1900 / 2000 / 2100, years -1 .. 1 and 400,
    ISO-week year ends, month ends."""
    out = [0, 1, -1, 2 ** 31 - 1, -(2 ** 31), 146097, -146097, 146096, -146098]
    for y in (1900, 2000, 2100, -1, 0, 1, 400, 1969, 1970, 2018, 2019, 2020, 2021, 2024, 2026):
        for m, d in ((1, 1), (1, 3), (1, 29), (1, 30), (1, 31), (2, 28), (3, 1), (12, 28), (12, 31)):
            out.append(OT.days_of(y, m, d))
        out.append(OT.days_of(y, 3, 1) - 1)  # Feb 28 or 29
    return out


def edge_values(unit):
    per = OT.PER_DAY[unit]
    vals = [I64_MIN, I64_MIN + 1, I64_MAX, I64_MAX - 1]
    for d in edge_days():
        for off in (0, -1, 1, per // 2, per - 1):
            v = d * per + off
            if I64_MIN <= v <= I64_MAX and (unit != "D" or -(2 ** 31) <= v < 2 ** 31):
                vals.append(v)
    return vals


def in_domain(v, unit):
    """Where the calendar results are specified: the year lies within the range of an int32 day count."""
    return -(2 ** 31) <= v // OT.PER_DAY[unit] < 2 ** 31


def table(cols):
    """A host table from {name: (arrow type, int values with None)}."""
    fields, data, valid = [], [], []
    for name, (tp, vals) in cols.items():
        fields.append(pa.field(name, tp))
        npdt = np.int32 if pa.types.is_date32(tp) or tp == pa.int32() else np.int64
        data.append(torch.from_numpy(np.array([0 if v is None else v for v in vals], dtype=npdt)))
        nulls = np.array([v is None for v in vals])
        valid.append(torch.from_numpy((~nulls).astype(np.uint8)) if nulls.any() else None)
    return B200Table(Schema(fields), data, valid)


def frame(cols):
    return (pd.DataFrame({n: pd.array([pd.NA if v is None else v for v in vals], dtype="Int64")
                          for n, (_, vals) in cols.items()}),
            {n: tp for n, (tp, _) in cols.items() if OT.unit_of(tp)})


def run_model(t, exprs):
    """Compile into one program, run the machine model; a list of python values (None = NULL) per expression."""
    prog = X._Program(t)
    meta = []
    for e in exprs:
        cls, _ = prog.compile(e, top=True)
        cls = "i" if cls == "n" else cls
        prog.output({"i": torch.int64, "f": torch.float64, "b": torch.uint8}[cls], True)
        meta.append(cls)
    cols = [t.columns[i].numpy() for i in prog.cols]
    valid = [None if t.valid[i] is None else t.valid[i].numpy() for i in prog.cols]
    outs, outv = tsim.run(t.num_rows, cols, valid, prog.ins, [o[2] for o in prog.outs],
                          col_types=[expr_type(t.schema.types[i]) for i in prog.cols])
    res = []
    for cls, o, v in zip(meta, outs, outv):
        vals = o.astype(bool).tolist() if cls == "b" else o.tolist()
        res.append([x if ok else None for x, ok in zip(vals, v)])
    return res, prog


def run_oracle(cols, exprs):
    df, types = frame(cols)
    named = [e.alias(f"o{i}") for i, e in enumerate(exprs)]
    low_df, low, _ = OT.lower(df, named, types)
    low_df, low, _ = OS.lower(low_df, low)  # CASE, GREATEST / LEAST
    got = OX.select(low_df, SelectColumns(*low))
    return [[None if x is pd.NA else x for x in got[f"o{i}"].tolist()] for i in range(len(exprs))]


# ---- builders, literals, SQL text ----------------------------------------------------------------------------
def test_literals_and_builders():
    s = Schema([pa.field("t", pa.timestamp("ns")), pa.field("d", pa.date32())])
    assert lit(dt.date(2024, 1, 31)).infer_type(s) == pa.date32()
    assert lit(dt.datetime(2024, 1, 31, 12)).infer_type(s) == pa.timestamp("us")
    assert lit(dt.timedelta(days=1)).infer_type(s) == pa.duration("us")
    aware = dt.datetime(2024, 1, 31, 12, tzinfo=dt.timezone(dt.timedelta(hours=2)))
    assert lit(aware).value == dt.datetime(2024, 1, 31, 10)
    assert f.year(col("t")).fingerprint() == f.extract("YEAR", col("t")).fingerprint() == \
        f.date_part("year", col("t")).fingerprint()
    assert f.dayofweek(col("t")).kwargs == {"field": "dow"} and f.dayofyear(col("t")).kwargs == {"field": "doy"}
    assert f.extract("week", col("t")).infer_type(s) == pa.int64()
    assert f.extract("epoch", col("t")).infer_type(s) == pa.float64()
    assert f.date_trunc("month", col("t")).infer_type(s) == pa.timestamp("ns")
    assert f.date_trunc("month", col("d")).infer_type(s) == pa.date32()
    assert f.add_months(col("d"), 1).infer_type(s) == pa.date32()
    assert f.datediff("day", col("d"), col("t")).infer_type(s) == pa.int64()
    assert (col("t") + dt.timedelta(hours=1)).infer_type(s) == pa.timestamp("ns")
    for bad in (lambda: f.extract("fortnight", col("t")), lambda: f.date_trunc("epoch", col("t")),
                lambda: f.datediff("dow", col("t"), col("t")), lambda: f.add_months(col("t"), 1.5)):
        with pytest.raises(ValueError):
            bad()


SQL_FORMS = [
    lit(dt.date(2024, 1, 31)), lit(dt.date(1, 1, 1)), lit(dt.datetime(2024, 1, 31, 12)),
    lit(dt.datetime(1969, 12, 31, 23, 59, 59, 500000)), lit(dt.timedelta(days=7)), lit(dt.timedelta(days=-7)),
    lit(dt.timedelta(days=1, hours=2, minutes=3, seconds=4, microseconds=5)), lit(-dt.timedelta(seconds=1)),
    col("t") >= lit(dt.date(2024, 1, 1)), col("t") + dt.timedelta(hours=36), col("t") - dt.timedelta(days=2),
    f.add_months(col("t"), 3), f.add_months(col("t"), -12), f.add_months(col("t"), col("n") + 1),
    f.datediff("week", col("a"), col("t")), f.date_trunc("quarter", col("t")) == lit(dt.date(2024, 1, 1)),
] + [f.extract(x, col("t")) for x in OT.FIELDS] + [f.date_trunc(p, col("t")) for p in OT.PARTS]


@pytest.mark.parametrize("e", SQL_FORMS, ids=[to_sql(e) for e in SQL_FORMS])
def test_print_parse_is_a_fixed_point(e):
    text = to_sql(e.alias("x"))
    st = _parse_select(text, "tbl", text)
    assert st.columns[0].fingerprint() == e.alias("x").fingerprint(), text
    assert to_sql(st.columns[0]) == text


def test_parser_spellings_and_names():
    sql = ("SELECT YEAR(t) AS y, DATE_PART('dow', t) AS w, t + INTERVAL '3' MONTH AS a, t - INTERVAL '1' YEAR AS b, "
           "INTERVAL '2' MONTH + t AS c, t + INTERVAL '90' MINUTE AS m, EXTRACT(isodow FROM t) AS i, year, day, date, "
           "timestamp, interval FROM tbl WHERE t < TIMESTAMP '2024-06-01 00:00:00'")
    cut = _top_level_from(sql)
    st = _parse_select(sql[7:cut[0]], sql[cut[1]:], sql)
    want = [f.year(col("t")), f.extract("dow", col("t")), f.add_months(col("t"), 3), f.add_months(col("t"), -12),
            f.add_months(col("t"), 2), col("t") + dt.timedelta(minutes=90), f.extract("isodow", col("t")), col("year"),
            col("day"), col("date"), col("timestamp"), col("interval")]
    for got, w in zip(st.columns, want):
        assert got.alias("").fingerprint() == w.fingerprint(), str(got)
    assert st.where.fingerprint() == (col("t") < lit(dt.datetime(2024, 6, 1))).fingerprint()
    for bad in ("DATE '2024-13-01'", "TIMESTAMP '2024-01-01 25:00:00'", "INTERVAL 'x' DAY", "INTERVAL '1' FORTNIGHT",
                "EXTRACT(fortnight FROM t)", "DATE_TRUNC('epoch', t)"):
        with pytest.raises(ValueError):
            _parse_select(bad + " AS x", "tbl", bad)


# ---- the oracle against independent calendars ------------------------------------------------------------------
def test_oracle_matches_python_datetime_over_years_1_to_9999():
    rng = np.random.default_rng(5)
    lo, hi = dt.date(1, 1, 1).toordinal(), dt.date(9999, 12, 31).toordinal()
    ords = list(rng.integers(lo, hi + 1, 20000)) + [lo, hi] + [dt.date(y, 12, 31).toordinal() for y in range(1, 9999, 7)]
    for o in ords:
        d = dt.date.fromordinal(int(o))
        days = int(o) - dt.date(1970, 1, 1).toordinal()
        iso = d.isocalendar()
        got = [OT.extract(x, days, "D") for x in ("year", "month", "day", "isoyear", "week", "isodow", "dow", "doy")]
        assert got == [d.year, d.month, d.day, iso[0], iso[1], iso[2], iso[2] % 7, d.timetuple().tm_yday], d
        assert OT.days_of(d.year, d.month, d.day) == days
        assert OT.date_trunc("week", days, "D") == days - d.weekday()
        assert OT.date_trunc("quarter", days, "D") == \
            dt.date(d.year, (d.month - 1) // 3 * 3 + 1, 1).toordinal() - dt.date(1970, 1, 1).toordinal()


def test_oracle_matches_numpy_pyarrow_pandas_sqlite():
    rng = np.random.default_rng(9)
    us = np.concatenate([rng.integers(-(2 ** 62), 2 ** 62, 3000), rng.integers(-10 ** 15, 4 * 10 ** 15, 3000),
                         np.array(edge_values("us")[4:], dtype=np.int64)])
    us = us[(us > -6 * 10 ** 16) & (us < 2.5 * 10 ** 17)]  # years 68 .. 9892: what pyarrow and pandas can show
    arr = pa.array(us, pa.timestamp("us"))
    pins = {"year": pc.year(arr), "month": pc.month(arr), "day": pc.day(arr), "hour": pc.hour(arr),
            "minute": pc.minute(arr), "second": pc.second(arr), "quarter": pc.quarter(arr), "doy": pc.day_of_year(arr),
            "week": pc.iso_week(arr), "isoyear": pc.iso_year(arr),
            "isodow": pc.day_of_week(arr, count_from_zero=False, week_start=1),
            "dow": pc.day_of_week(arr, count_from_zero=True, week_start=7)}
    for field, want in pins.items():
        assert [OT.extract(field, int(v), "us") for v in us] == want.to_pylist(), field
    for part in ("year", "quarter", "month", "week", "day", "hour", "minute", "second"):
        want = pc.floor_temporal(arr, unit=part, week_starts_monday=True).cast(pa.int64()).to_pylist()
        assert [OT.date_trunc(part, int(v), "us") for v in us] == want, part
    # numpy: unit conversions floor (numpy itself is not exact at the very ends of int64)
    for v in [-(2 ** 62), -1, 0, 1, 10 ** 18, 2 ** 62] + list(rng.integers(-(2 ** 62), 2 ** 62, 200)):
        for a, b in (("ns", "us"), ("us", "ms"), ("ms", "s"), ("us", "D"), ("ns", "D"), ("s", "D")):
            want = np.datetime64(int(v), a).astype(f"datetime64[{b}]").astype(np.int64)
            assert OT.cast(int(v), a, b) == int(want), (v, a, b)
    assert OT.cast(I64_MAX // 1000, "s", "ns") == I64_MAX and OT.cast(-(10 ** 12), "D", "us") == I64_MIN
    # add_months: pandas.DateOffset and dateutil.relativedelta
    from dateutil.relativedelta import relativedelta
    base = pd.Timestamp("1970-01-01")
    for v in list(rng.integers(-10 ** 15, 4 * 10 ** 15, 400)) + [OT.days_of(2024, 1, d) * 86400 * 10 ** 6 + 5 for d in (29, 30, 31)]:
        ts = base + pd.Timedelta(microseconds=int(v))
        for n in (1, -1, 12, -12, 13, -13, 25, 1200, -1200):
            got = OT.add_months(int(v), n, "us")
            assert got == (ts + pd.DateOffset(months=n) - base) // pd.Timedelta(microseconds=1), (ts, n)
            assert got == (ts.to_pydatetime() + relativedelta(months=n) - dt.datetime(1970, 1, 1)) // dt.timedelta(microseconds=1)
    # sqlite strftime
    con = sqlite3.connect(":memory:")
    for v in list(rng.integers(-6 * 10 ** 10, 2 * 10 ** 11, 400)) + [0, -1, 86399, -86400]:
        row = con.execute("SELECT strftime('%Y %m %d %H %M %S %j %w', ?, 'unixepoch')", (int(v),)).fetchone()[0]
        got = [OT.extract(x, int(v), "s") for x in ("year", "month", "day", "hour", "minute", "second", "doy", "dow")]
        assert got == [int(x) for x in row.split()], v
    assert OT.extract("second", -500000, "us") == 59 and OT.extract("year", -500000, "us") == 1969
    assert OT.datediff("week", OT.days_of(2024, 1, 7), "D", OT.days_of(2024, 1, 8), "D") == 1  # Sunday -> Monday
    assert OT.datediff("year", OT.days_of(2023, 12, 31), "D", OT.days_of(2024, 1, 1) * 86400, "s") == 1


# ---- the compiler through the machine model ----------------------------------------------------------------------
@pytest.mark.parametrize("unit", list(UNITS))
def test_every_field_and_part_of_every_unit(unit):
    rng = np.random.default_rng(11)
    vals = [v for v in edge_values(unit) if in_domain(v, unit)]
    span = 2 ** 31 - 1 if unit == "D" else min(2 ** 62, (2 ** 31 - 1) * OT.PER_DAY[unit])
    vals += [int(v) for v in rng.integers(-span, span, 3000)] + [None]
    other = [int(v) for v in rng.integers(-40000, 40000, len(vals))]
    months = [int(v) for v in rng.choice([0, 1, -1, 12, -12, 13, -13, 4800, -4800, 7], len(vals))]
    cols = {"t": (UNITS[unit], vals), "d": (pa.date32(), other), "n": (pa.int64(), months)}
    exprs = [f.extract(x, col("t")) for x in OT.FIELDS] + [f.date_trunc(p, col("t")) for p in OT.PARTS] + \
        [f.datediff(p, col("d"), col("t")) for p in OT.PARTS] + [f.datediff("month", col("t"), col("d"))] + \
        [f.add_months(col("t"), col("n")), f.add_months(col("t"), 1), f.add_months(col("t"), col("n") * 2 - 1),
         function("extract", col("t"), field="YEAR"), f.year(f.add_months(f.date_trunc("month", col("t")), 1))]
    t = table(cols)
    for i in range(0, len(exprs), 6):
        model, _ = run_model(t, exprs[i:i + 6])
        want = run_oracle(cols, exprs[i:i + 6])
        for e, m, w in zip(exprs[i:i + 6], model, want):
            assert m == w, (unit, str(e), [(v, a, b) for v, a, b in zip(vals, m, w) if a != b][:3])


def test_model_never_fails_outside_the_domain():
    for unit in UNITS:
        vals = np.array([v for v in edge_values(unit)], dtype=np.int64)
        for fn, words in ((tsim.ts_part, K.TIME_FIELDS), (tsim.ts_trunc, K.TIME_PARTS), (tsim.ts_index, K.TIME_PARTS)):
            for code in range(len(words)):
                with np.errstate(all="ignore"):
                    assert fn(vals, code, CODE[unit]).shape == vals.shape


LITERALS = [dt.date(2024, 1, 1), dt.datetime(2024, 1, 1), dt.datetime(2024, 1, 1, 12, 0, 0, 500000),
            dt.datetime(1969, 12, 31, 23, 59, 59, 999999), dt.datetime(9999, 12, 31, 23, 59, 59), dt.datetime(1, 1, 1),
            dt.date(1970, 1, 1)]


@pytest.mark.parametrize("unit", list(UNITS))
def test_literal_against_column_in_every_unit(unit):
    per = OT.PER_DAY[unit]
    vals = [None, I64_MIN, I64_MAX, 0, -1, 1] if unit != "D" else [None, -(2 ** 31), 2 ** 31 - 1, 0, -1, 1]
    for l in LITERALS:
        q = OT.literal_us(l) * per // OT.PER_DAY["us"]
        vals += [v for v in (q - 1, q, q + 1, q + 2) if I64_MIN <= v <= I64_MAX and (unit != "D" or abs(v) < 2 ** 31)]
    cols = {"t": (UNITS[unit], vals)}
    t = table(cols)
    for l in LITERALS:
        exprs = [col("t") < lit(l), col("t") <= lit(l), col("t") > lit(l), col("t") >= lit(l), col("t") == lit(l),
                 col("t") != lit(l), lit(l) < col("t"), lit(l) >= col("t")]
        model, prog = run_model(t, exprs)
        assert all(op < K.X_MULSAT_I for op, *_ in prog.ins)  # rescaled on the host: no device instruction
        for e, m, w in zip(exprs, model, run_oracle(cols, exprs)):
            assert m == w, (unit, str(e))
    model, _ = run_model(t, [lit(dt.date(2024, 1, 1)) < lit(dt.datetime(2024, 1, 1, 0, 0, 1)),
                             lit(dt.datetime(2024, 1, 2)) - lit(dt.date(2024, 1, 1)) == lit(dt.timedelta(days=1))])
    assert model == [[True] * len(vals)] * 2


def test_casts_between_temporal_types_saturate_and_floor():
    s_vals = [None, 0, -1, 1, I64_MAX // 10 ** 9, I64_MAX // 10 ** 9 + 1, I64_MIN // 10 ** 9 - 1, I64_MAX, I64_MIN, 86399, -86401]
    cols = {"s": (pa.timestamp("s"), s_vals), "d": (pa.date32(), [None, 0, -1, 1, 2 ** 31 - 1, -(2 ** 31), 19000, 5, 6, 7, 8]),
            "us": (pa.timestamp("us", tz="UTC"), [None, -1, 0, 1, -86400 * 10 ** 6 - 1, I64_MIN, I64_MAX, 5, 6, 7, 86400 * 10 ** 6])}
    exprs = [col("s").cast(pa.timestamp("ns")), col("s").cast(pa.date32()), col("d").cast(pa.timestamp("us")),
             col("d").cast(pa.timestamp("ns")), col("us").cast(pa.date32()), col("us").cast(pa.timestamp("s")),
             col("us").cast(pa.date64()), col("d").cast(pa.timestamp("us")) < col("us"),
             f.date_trunc("day", col("us")).cast(pa.date32()), col("s").cast(pa.timestamp("ns")) > col("us").cast(pa.timestamp("ns"))]
    model, _ = run_model(table(cols), exprs)
    want = run_oracle(cols, exprs)
    for e, m, w in zip(exprs, model, want):
        assert m == w, str(e)
    assert model[0][4:9] == [I64_MAX // 10 ** 9 * 10 ** 9, I64_MAX, I64_MIN, I64_MAX, I64_MIN]
    assert model[4][1] == -1  # 1969-12-31 23:59:59.999999 is the day before the epoch


def test_two_temporal_columns_meet_as_raw_integers():
    """``d > ts``, ``ts - d``, ``ts + 1``: exactly the programs of plain int64 columns."""
    t = table({"d": (pa.date32(), [1, 2]), "ts": (pa.timestamp("us"), [3, 4])})
    p = table({"d": (pa.int32(), [1, 2]), "ts": (pa.int64(), [3, 4])})
    for e in (col("d") > col("ts"), col("ts") - col("d"), col("ts") + 1, f.coalesce(col("d"), col("ts")),
              f.greatest(col("d"), col("ts"), 5), col("ts").cast("long") * 2, col("d").cast(float)):
        a, b = X._Program(t), X._Program(p)
        assert a.compile(e) == b.compile(e) and a.ins == b.ins, str(e)


def test_interval_arithmetic_and_rejections():
    cols = {"d": (pa.date32(), [0, 19000, None]), "s": (pa.timestamp("s"), [0, -5, 7]),
            "z": (pa.timestamp("us", tz="Europe/Paris"), [0, 1, 2]), "u": (pa.duration("us"), [1, 2, 3]),
            "k": (pa.time64("us"), [1, 2, 3]), "n": (pa.int64(), [1, 2, 3])}
    t = table(cols)
    exprs = [col("d") + dt.timedelta(days=2), col("s") - dt.timedelta(hours=1), dt.timedelta(seconds=5) + col("s"),
             col("s") - lit(dt.datetime(1970, 1, 1, 0, 0, 7)), f.coalesce(col("d"), dt.date(2000, 1, 1)),
             f.case([(col("n") > 1, col("s"))], dt.datetime(2000, 1, 1)), col("u") > dt.timedelta(microseconds=1),
             f.greatest(col("d"), dt.date(1980, 1, 1)), col("z") < lit(dt.datetime(1970, 1, 1, 0, 0, 0, 1))]
    model, _ = run_model(t, exprs)
    for e, m, w in zip(exprs, model, run_oracle(cols, exprs)):
        assert m == w, str(e)
    for bad in (col("d") + dt.timedelta(hours=1), col("s") + dt.timedelta(milliseconds=1), col("n") > lit(dt.date(2024, 1, 1)),
                col("s") + lit(dt.date(2024, 1, 1)), f.coalesce(col("s"), dt.datetime(2000, 1, 1, 0, 0, 0, 5)),
                f.year(col("n")), f.add_months(col("d"), col("n") / 2)):
        with pytest.raises(ValueError):
            X._Program(t).compile(bad)
    for bad in (f.year(col("z")), f.date_trunc("day", col("z")), f.add_months(col("z"), 1), f.datediff("day", col("d"), col("z")),
                f.hour(col("k")), f.year(col("u")), function("STRFTIME", col("d"), "%Y"),
                function("INTERVAL_MONTHS", lit(3)) + col("n")):
        with pytest.raises(NotImplementedError):
            X._Program(t).compile(bad)


def _tree(rng, depth):
    """A random int64 / bool tree over the temporal nodes, arithmetic, CASE, COALESCE and Kleene logic."""
    ts = [col("t"), col("d"), col("g")]

    def point():
        x = ts[int(rng.integers(0, 3))]
        r = int(rng.integers(0, 4))
        if r == 0:
            return f.date_trunc(OT.PARTS[int(rng.integers(0, 8))], x)
        if r == 1:
            return f.add_months(x, col("n") if rng.random() < 0.5 else int(rng.integers(-30, 30)))
        return x

    def num(d):
        r = int(rng.integers(0, 7 if d > 0 else 3))
        if r == 0:
            return f.extract(OT.FIELDS[int(rng.integers(0, 12))], point())
        if r == 1:
            return f.datediff(OT.PARTS[int(rng.integers(0, 8))], point(), point())
        if r == 2:
            return col("n")
        if r == 3:
            return num(d - 1) + num(d - 1) * int(rng.integers(-3, 4))
        if r == 4:
            return f.case([(boolean(d - 1), num(d - 1))], num(d - 1))
        if r == 5:
            return f.coalesce(num(d - 1), num(d - 1), 0)
        return num(d - 1) - num(d - 1)

    def boolean(d):
        r = int(rng.integers(0, 5 if d > 0 else 2))
        if r == 0:
            l = dt.datetime(2024, 1, 1) + dt.timedelta(seconds=int(rng.integers(-10 ** 8, 10 ** 8)), microseconds=int(rng.integers(0, 2)) * 500)
            x = point()
            return [x < lit(l), x >= lit(l), lit(l.date()) <= x, x != lit(l)][int(rng.integers(0, 4))]
        if r == 1:
            return num(d) > int(rng.integers(-5, 2030))
        if r == 2:
            return boolean(d - 1) & boolean(d - 1)
        if r == 3:
            return boolean(d - 1) | ~boolean(d - 1)
        return num(d - 1).is_null() | boolean(d - 1)

    return num(depth) if rng.random() < 0.6 else boolean(depth)


def test_random_trees_match_the_oracle():
    rng = np.random.default_rng(2024)
    n = 300
    base = OT.days_of(2024, 1, 1)

    def nulls(vals):
        return [None if rng.random() < 0.15 else int(v) for v in vals]

    cols = {"t": (pa.timestamp("us"), nulls(rng.integers(-3 * 10 ** 15, 3 * 10 ** 15, n))),
            "d": (pa.date32(), nulls(base + rng.integers(-20000, 20000, n))),
            "g": (pa.timestamp("ns", tz="UTC"), nulls(rng.integers(-(2 ** 62), 2 ** 62, n))),
            "n": (pa.int64(), nulls(rng.integers(-40, 40, n)))}
    t = table(cols)
    checked = 0
    while checked < 300:
        e = _tree(rng, int(rng.integers(1, 4)))
        try:
            model, _ = run_model(t, [e])
        except X._OutOfResources:
            continue
        assert model[0] == run_oracle(cols, [e])[0], str(e)
        checked += 1


def test_opcode_numbers_match_the_header():
    """The new opcodes follow FB_X_LEAST_F = 59; the header, the binding and the builders' word lists agree."""
    import os
    import re

    from fugue_b200 import column as C

    text = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "fugue_b200.h")).read()
    num = {m.group(1): int(m.group(2)) for m in re.finditer(r"\b(FB_(?:X|TU|TF|TP)_[A-Z0-9_]+) = (\d+)", text)}
    assert num["FB_X_LEAST_F"] == 59 and K.X_LEAST_F == 59
    for name in ("MULSAT_I", "FLOORDIV_I", "TS_PART", "TS_TRUNC", "TS_INDEX", "TS_ADDMON"):
        assert num["FB_X_" + name] == getattr(K, "X_" + name)
    assert [num["FB_X_" + n] for n in ("MULSAT_I", "FLOORDIV_I", "TS_PART", "TS_TRUNC", "TS_INDEX", "TS_ADDMON")] == list(range(60, 66))
    assert [num["FB_TF_" + w.upper()] for w in K.TIME_FIELDS] == list(range(len(K.TIME_FIELDS))) and num["FB_TF_COUNT"] == 12
    assert [num["FB_TP_" + w.upper()] for w in K.TIME_PARTS] == list(range(len(K.TIME_PARTS))) and num["FB_TP_COUNT"] == 8
    assert [num["FB_TU_" + u] for u in ("DAY", "S", "MS", "US", "NS")] == [K.TU_DAY, K.TU_S, K.TU_MS, K.TU_US, K.TU_NS]
    assert C.TIME_FIELDS == K.TIME_FIELDS and C.TIME_PARTS == K.TIME_PARTS and K.XF_UNIT_SHIFT == 8
