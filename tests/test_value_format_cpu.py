"""Casts to string without a GPU: the K14 format routines through their host export (fb_debug_value_format_host)
against CPython's repr / str and pyarrow's cast / strftime, the dictionary keys, and the compiler's rewrite of casts
inside expressions, run end to end by the K8 machine model (tests/_lookup_sim.py) with K14 on the host."""
import random

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest
import torch

import _lookup_sim as lsim
from test_string_build_cpu import _oracle_evaluate
from fugue_b200 import expr as X
from fugue_b200 import kernels as K
from fugue_b200 import strings as ST
from fugue_b200.column import ColumnExpr, Kind, col, functions as ff, lit
from fugue_b200.schema import Schema
from fugue_b200.table import B200Table
from oracle import strings as ostr

_PER = {"s": 1, "ms": 1000, "us": 10 ** 6, "ns": 10 ** 9}
_TU = {"s": K.TU_S, "ms": K.TU_MS, "us": K.TU_US, "ns": K.TU_NS}


def texts(values: np.ndarray, kind: int, valid=None):
    offs, data = K.value_format_host(values, valid, kind)
    b = data.tobytes()
    return [b[offs[i]:offs[i + 1]].decode() for i in range(len(values))]


def _floats_from_bits(bits):
    return np.array(bits, dtype=np.uint64).view(np.float64)


def _check_repr(xs: np.ndarray):
    got = texts(xs, K.FMT_F64)
    bad = [(x, g) for x, g in zip(xs.tolist(), got) if g != repr(x)]
    assert not bad, bad[:5]


# ---- floats -----------------------------------------------------------------------------------------------
def test_float_edges_equal_repr():
    xs = [0.0, -0.0, float("inf"), -float("inf"), float("nan"), -float("nan"), 5e-324, -5e-324, 2.2250738585072014e-308,
          2.225073858507201e-308, 1.7976931348623157e308, -1.7976931348623157e308, 0.1, 0.2, 0.3, 1 / 3, 2 / 3,
          1e16, 9999999999999998.0, 1e15, 123456789012345.6, 1e-4, 9.999999999999999e-05, 1e-5, 0.00012345, 1.5e-05]
    for k in range(-60, 60):  # 2^53 +- k
        xs.append(float(2 ** 53 + k))
    for e in range(-1074, 1024):  # powers of two and their neighbours
        p = np.float64(2.0) ** e if e > -1075 else 0.0
        xs += [float(p), float(np.nextafter(p, np.inf)), float(np.nextafter(p, -np.inf))]
    for e in range(-324, 309):  # powers of ten and their neighbours
        p = float(f"1e{e}")
        xs += [p, float(np.nextafter(p, np.inf)), float(np.nextafter(p, -np.inf))]
    a = np.array(xs, dtype=np.float64)
    _check_repr(np.concatenate([a, -a]))
    # NaN payloads of both signs are all "nan"
    nans = _floats_from_bits([0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0xFFFFFFFFFFFFFFFF])
    assert texts(nans, K.FMT_F64) == ["nan"] * 4


def test_float32_values_are_written_widened():
    f = np.array([0.1, 1 / 3, 3.4028235e38, 1e-45, 16777217.0], dtype=np.float32)
    assert texts(f.astype(np.float64), K.FMT_F64) == [str(float(x)) for x in f.tolist()]
    assert texts(np.array([np.float32(0.1)], np.float64), K.FMT_F64) == ["0.10000000149011612"]


def test_random_float_bits_equal_repr():
    rng = np.random.default_rng(14)
    bits = rng.integers(0, 2 ** 64, 10 ** 6, dtype=np.uint64, endpoint=False)
    _check_repr(bits.view(np.float64))


def test_random_short_decimals_equal_repr():
    rng = np.random.default_rng(15)
    mant = rng.integers(-10 ** 7, 10 ** 7, 10 ** 6)
    scale = rng.integers(-12, 12, 10 ** 6)
    xs = np.array([float(f"{m}e{s}") for m, s in zip(mant.tolist(), scale.tolist())], dtype=np.float64)
    _check_repr(xs)


# ---- integers and bools -----------------------------------------------------------------------------------
def test_integers_equal_str():
    rng = np.random.default_rng(16)
    i = np.concatenate([np.array([0, 1, -1, 9, 10, -10, 2 ** 63 - 1, -2 ** 63, 10 ** 18, -10 ** 18], np.int64),
                        rng.integers(-2 ** 63, 2 ** 63 - 1, 10 ** 5, dtype=np.int64)])
    assert texts(i, K.FMT_I64) == [str(x) for x in i.tolist()]
    u = np.concatenate([np.array([0, 2 ** 64 - 1, 2 ** 63, 10 ** 19], np.uint64),
                        rng.integers(0, 2 ** 64 - 1, 10 ** 5, dtype=np.uint64)])
    assert texts(u, K.FMT_U64) == [str(x) for x in u.tolist()]
    assert texts(np.array([0, 1, 7], np.int64), K.FMT_BOOL) == ["false", "true", "true"]


def test_null_values_get_no_bytes():
    offs, _ = K.value_format_host(np.array([5, 6, 7], np.int64), np.array([1, 0, 1], np.uint8), K.FMT_I64)
    assert offs.tolist() == [0, 1, 1, 2]


# ---- dates and timestamps ---------------------------------------------------------------------------------
def _arrow_date(vals, tp, st):
    return pc.cast(pa.array(vals, st).view(tp), pa.string()).to_pylist()


def test_date32_equals_arrow():
    rng = random.Random(17)
    lo, hi = -12687428, 11248737  # the days Arrow writes as dates
    vals = [lo - 1, lo, hi, hi + 1, -2 ** 31, 2 ** 31 - 1, 0, -1, -719162, -719163, -800000, 2932896, 2932897, 3000000]
    vals += [rng.randrange(-2 ** 31, 2 ** 31) for _ in range(10 ** 5)]
    vals += [rng.randrange(lo - 10, hi + 10) for _ in range(10 ** 6)]
    got = texts(np.array(vals, np.int64), K.FMT_DATE32)
    assert got[:5] == ["<value out of range: -12687429>", "-32767-01-01", "32767-12-31", "<value out of range: 11248738>",
                       "<value out of range: -2147483648>"]
    assert got == _arrow_date(vals, pa.date32(), pa.int32())


def test_date64_equals_arrow():
    rng = random.Random(18)
    day = 86_400_000
    vals = [-1, 1, -day, -day - 1, 971890963199999, 971890963200000, -1096193779200000, -1096193779200001,
            -2 ** 63, 2 ** 63 - 1]
    vals += [rng.randrange(-2 ** 63, 2 ** 63) for _ in range(10 ** 5)]
    vals += [rng.randrange(-1100000000000000, 1000000000000000) for _ in range(10 ** 6)]
    got = texts(np.array(vals, np.int64), K.FMT_DATE64)
    assert got[:2] == ["1970-01-01", "1970-01-01"]  # Arrow truncates a date64's milliseconds toward 0
    assert got == _arrow_date(vals, pa.date64(), pa.int64())


def _strftime(vals, unit):
    """pyarrow's text, None where pyarrow raises (seconds far beyond year 32767)."""
    out = []
    for k in range(0, len(vals), 4096):
        chunk = vals[k:k + 4096]
        try:
            out += pc.strftime(pa.array(chunk, pa.int64()).view(pa.timestamp(unit)), format="%Y-%m-%d %H:%M:%S").to_pylist()
        except pa.ArrowInvalid:
            out += [_strftime_one(v, unit) for v in chunk]
    return out


def _strftime_one(v, unit):
    try:
        return pc.strftime(pa.array([v], pa.int64()).view(pa.timestamp(unit)), format="%Y-%m-%d %H:%M:%S")[0].as_py()
    except pa.ArrowInvalid:
        return None


@pytest.mark.parametrize("unit", ["s", "ms", "us", "ns"])
def test_timestamps_equal_strftime(unit):
    rng = random.Random(19)
    per = _PER[unit]
    kind = K.FMT_TS + _TU[unit] + (K.FMT_TS_FRAC if per > 1 else 0)
    # milliseconds above 9.1e18 (year 292 million) are left out: there Arrow's hours differ from its own day model
    top = 2 ** 63 - 1 if unit != "ms" else 9 * 10 ** 18
    edges = [0, -1, 1, -per, per - 1, top, -2 ** 63, -2 ** 63 + 1, 86400 * per - 1, -86400 * per]
    vals = edges + [rng.randrange(-2 ** 63, top) for _ in range(10 ** 5)]
    span = min(253402300800, (2 ** 63 - 1) // per - 1)  # years 1 .. 9999, inside int64
    vals += [rng.randrange(-span, span) * per + rng.randrange(per) for _ in range(10 ** 6)]
    got = texts(np.array(vals, np.int64), kind)
    want = _strftime(vals, unit)
    assert want.count(None) < len(vals) // 100
    assert [g for g, w in zip(got, want) if w is not None] == [w for w in want if w is not None]
    if unit == "us":
        assert got[6] == "-28164-12-21 19:59:05.224192" and got[7] == "-28164-12-21 19:59:05.224193"


def test_timestamp_whole_seconds_without_fraction():
    vals = np.array([0, -1000, 1704067200000], np.int64)
    assert texts(vals, K.FMT_TS + K.TU_MS) == ["1970-01-01 00:00:00", "1969-12-31 23:59:59", "2024-01-01 00:00:00"]
    with pytest.raises(Exception, match="unknown format kind"):
        texts(vals, K.FMT_TS + K.TU_S + K.FMT_TS_FRAC)


# ---- dictionary keys --------------------------------------------------------------------------------------
def test_format_keys_canonical():
    f = torch.tensor([0.0, -0.0, float("nan"), -float("nan"), 1.5])
    k = ST._format_keys(f, pa.float32())
    assert k[0] != k[1] and k[2] == k[3] and len(set(k.tolist())) == 4
    d = torch.tensor([0, 1, -1, 86_400_000 - 1, -86_400_000 + 1, 2 ** 62], dtype=torch.int64)
    k = ST._format_keys(d, pa.date64()).tolist()
    assert k[:5] == [0, 0, 0, 0, 0] and k[5] == 2 ** 62  # the day Arrow writes; out of range: the raw value
    assert ST._format_keys(torch.tensor([0, 2, 1], dtype=torch.uint8), pa.bool_()).tolist() == [0, 1, 1]


def test_format_kind_rejects_zones_and_other_types():
    assert ST.format_kind(pa.timestamp("ns", "UTC")) == K.FMT_TS + K.TU_NS
    for tp in (pa.timestamp("us", "Asia/Tokyo"), pa.decimal128(10, 2), pa.duration("s"), pa.time64("us")):
        with pytest.raises(NotImplementedError):
            ST.format_kind(tp)


# ---- the compiler: casts inside expressions, on the machine model ------------------------------------------
def _host_format(values, valid, kind):
    offs, data = K.value_format_host(values.numpy(), None if valid is None else valid.numpy(), kind)
    return torch.from_numpy(offs), torch.from_numpy(data)


def _eval_model(nrows, device, cols, valid, program, out_dtypes, want_valid, col_types=None, out_types=None):
    outs, outv = lsim.run(nrows, [c.numpy() for c in cols], [None if v is None else v.numpy() for v in valid],
                          program, list(out_types), col_types=col_types)
    res = [torch.from_numpy(np.ascontiguousarray(o)).view(dt) for o, dt in zip(outs, out_dtypes)]
    return res, [torch.from_numpy(v.astype(np.uint8)) if w else None for v, w in zip(outv, want_valid)]


def _entry_tables(d, device, *args):
    vals = d.to_pylist()
    valid = None if d.null_count == 0 else torch.tensor([v is not None for v in vals], dtype=torch.uint8)
    if args:
        return torch.tensor([bool(ostr.like(v, args[0], args[1])) for v in vals], dtype=torch.int64), valid
    return torch.tensor([len(v) if v is not None else 0 for v in vals], dtype=torch.int64), valid


def _host_parse(d, device, tp):
    b = [x.encode() for x in d.to_pylist()]
    offs = np.cumsum([0] + [len(x) for x in b]).astype(np.int64)
    v, ok, _ = K.string_parse_host(offs, np.frombuffer(b"".join(b) + b"\0", np.uint8), None, ST.parse_target(tp))
    assert ok.all()
    return ST.ParseResult(torch.from_numpy(v.copy()), None, None)


def _patched(monkeypatch):
    monkeypatch.setattr(K, "eval_expr", _eval_model)
    monkeypatch.setattr(K, "value_format", _host_format)
    monkeypatch.setattr(ST, "like_table", lambda d, dev, p, e: _entry_tables(d, dev, p, e))
    monkeypatch.setattr(ST, "length_table", _entry_tables)
    monkeypatch.setattr(ST, "evaluate", _oracle_evaluate)
    monkeypatch.setattr(ST, "parse_table", _host_parse)


def _table():
    ids = [12, 7, 120, None, 3, 12]
    d = [19723, -1, 0, 19723, None, 0]
    v = [0.5, -0.0, 0.0, float("nan"), 1e16, None]
    valid = lambda xs: torch.tensor([x is not None for x in xs], dtype=torch.uint8)
    t = B200Table(Schema("id:long,d:date,v:double,s:str"),
                  [torch.tensor([x or 0 for x in ids], dtype=torch.int64),
                   torch.tensor([x or 0 for x in d], dtype=torch.int32),
                   torch.tensor([0.0 if x is None else x for x in v], dtype=torch.float64),
                   torch.tensor([0, 1, 0, 1, 0, 1], dtype=torch.int32)],
                  [valid(ids), valid(d), valid(v), None], {"s": pa.array(["a", "b"])})
    return t


def _strings(t, name):
    ci = t.schema.index_of_key(name)
    d = t.dictionaries[name].to_pylist()
    valid = t.valid[ci]
    return [None if valid is not None and not valid[i] else d[int(c)] for i, c in enumerate(t.columns[ci].tolist())]


def test_whole_column_casts(monkeypatch):
    _patched(monkeypatch)
    out = X.project(_table(), [col("id").cast(str), col("d").cast(str), col("v").cast(str).alias("vs")])
    assert _strings(out, "id") == ["12", "7", "120", None, "3", "12"]
    assert _strings(out, "d") == ["2024-01-01", "1969-12-31", "1970-01-01", "2024-01-01", None, "1970-01-01"]
    assert _strings(out, "vs") == ["0.5", "-0.0", "0.0", "nan", "1e+16", None]
    for name in ("id", "d", "vs"):
        entries = out.dictionaries[name].to_pylist()
        assert len(entries) == len(set(entries))


def test_casts_inside_expressions(monkeypatch):
    _patched(monkeypatch)
    t = _table()
    mask = X.predicate_mask(t, col("id").cast(str).like("12%"))
    assert mask.tolist() == [1, 0, 1, 0, 0, 1]
    mask = X.predicate_mask(t, col("d").cast(str) == "2024-01-01")
    assert mask.tolist() == [1, 0, 0, 1, 0, 0]
    out = X.project(t, [ff.length(col("id").cast(str)).alias("n"), ff.concat(col("id").cast(str), "-x").alias("c"),
                        ColumnExpr(Kind.BINARY, "||", [col("id").cast(str), lit("!")]).alias("p"),
                        ff.trim(col("d").cast(str)).cast("date").alias("back")])
    assert out.columns[0].tolist()[:3] == [2, 1, 3] and out.valid[0].tolist()[3] == 0
    assert _strings(out, "c") == ["12-x", "7-x", "120-x", "-x", "3-x", "12-x"]
    assert _strings(out, "p") == ["12!", "7!", "120!", None, "3!", "12!"]
    assert out.columns[3].tolist()[:4] == [19723, -1, 0, 19723] and out.valid[3].tolist()[4] == 0


def test_rejections_stay(monkeypatch):
    _patched(monkeypatch)
    t = _table()
    with pytest.raises(NotImplementedError):  # a string column cast to string, inside an expression
        X.predicate_mask(t, col("s").cast(str).like("a"))
    with pytest.raises(NotImplementedError):  # two string operands in one function
        X.project(t, [ff.concat(col("id").cast(str), col("d").cast(str)).alias("c")])
    with pytest.raises(NotImplementedError):  # a time zone the device has no database for
        tz = B200Table(Schema([pa.field("t", pa.timestamp("us", "Asia/Tokyo"))]), [torch.zeros(2, dtype=torch.int64)])
        X.project(tz, [col("t").cast(str)])
