"""Corpora and the pyarrow expectation for the string casts (K13), shared by the CPU and GPU test files.

``expected(strings, tp)`` is pyarrow's own ``cast(..., safe=False)``, entry by entry: the entries that raise are
found by bisection, so a corpus of millions of valid strings costs a handful of casts."""
import datetime
import fractions
import random
import struct
from typing import List, Optional, Sequence, Tuple

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc

from fugue_b200 import kernels as K

INT_TYPES = [pa.int8(), pa.int16(), pa.int32(), pa.int64(), pa.uint8(), pa.uint16(), pa.uint32(), pa.uint64()]
TS_TYPES = [pa.timestamp(u, tz) for u in ("s", "ms", "us", "ns") for tz in (None, "UTC", "Asia/Tokyo")]
ALL_TYPES = INT_TYPES + [pa.float32(), pa.float64(), pa.bool_(), pa.date32(), pa.date64()] + TS_TYPES


def layout(strings: Sequence[Optional[str]]) -> Tuple[np.ndarray, np.ndarray, Optional[np.ndarray]]:
    """The Arrow layout of a dictionary on the host: (int64 offsets, uint8 data, uint8 validity or None)."""
    raw = [b"" if s is None else s.encode("utf-8", "surrogatepass") for s in strings]
    offs = np.zeros(len(raw) + 1, dtype=np.int64)
    np.cumsum([len(b) for b in raw], out=offs[1:])
    data = np.frombuffer(b"".join(raw), dtype=np.uint8) if offs[-1] else np.zeros(0, dtype=np.uint8)
    valid = None if all(s is not None for s in strings) else np.array([s is not None for s in strings], np.uint8)
    return offs, data, valid


def words(arr: pa.Array) -> np.ndarray:
    """A cast result as the 8-byte words K13 writes (NULL: 0): integers sign- or zero-extended, floats as float64
    bits (a float32 widened), bool 0 / 1, dates and timestamps as their stored count."""
    tp = arr.type
    if pa.types.is_floating(tp):
        v = arr.fill_null(0).to_numpy(zero_copy_only=False).astype(np.float64).view(np.int64)
    elif pa.types.is_boolean(tp):
        v = arr.fill_null(False).to_numpy(zero_copy_only=False).astype(np.int64)
    elif pa.types.is_unsigned_integer(tp):
        v = arr.fill_null(0).to_numpy(zero_copy_only=False).astype(np.uint64).view(np.int64)
    elif pa.types.is_integer(tp):
        v = arr.fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64)
    else:
        store = pa.int32() if pa.types.is_date32(tp) else pa.int64()
        v = arr.view(store).fill_null(0).to_numpy(zero_copy_only=False).astype(np.int64)
    return v


def expected(strings: Sequence[Optional[str]], tp: pa.DataType) -> Tuple[np.ndarray, np.ndarray]:
    """(words, ok) per entry: what pyarrow's cast gives, and whether it parses (NULL entries: not ok)."""
    n = len(strings)
    out = np.zeros(n, dtype=np.int64)
    ok = np.zeros(n, dtype=bool)
    src = pa.array(list(strings), type=pa.string())

    def go(lo: int, hi: int) -> None:
        if lo >= hi:
            return
        try:
            r = pc.cast(src[lo:hi], tp, safe=False)
        except (pa.ArrowInvalid, pa.ArrowNotImplementedError):
            r = None
        if r is None:
            if hi - lo > 1:
                mid = (lo + hi) // 2
                go(lo, mid)
                go(mid, hi)
            return
        out[lo:hi] = words(r)
        ok[lo:hi] = r.is_valid().to_numpy(zero_copy_only=False)

    go(0, n)
    return out, ok


def target_of(tp: pa.DataType) -> int:
    from fugue_b200 import strings as ST
    return ST.parse_target(tp)


def host_parse(strings: Sequence[Optional[str]], tp: pa.DataType) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    offs, data, valid = layout(strings)
    return K.string_parse_host(offs, data, valid, target_of(tp))


# ---- corpora ---------------------------------------------------------------------------------------------------
CORNERS = ["+1", " 1", "1 ", "007", "-0", "0", "1.0", "1e3", "1_000", "", "0x", "0X", "0xff", "0XFF", "0x00ff", "-0x10",
           "0x80", "0x7f", "0xFFFFFFFFFFFFFFFF", "0x8000000000000000", "0x1", "0xg", "128", "-128", "-129", "255", "256",
           "-1", "+.5", "5.", "1.e5", "1E5", "1e+5", "1e0005", "inf", "-inf", "+inf", "Infinity", "-INFINITY", "nan",
           "NaN", "-nan", "+nan", "nan(123)", "nan()", "nan(a_b)", "nan(-)", "infinit", "infx", "3.4028235e38",
           "3.5e38", "1e400", "-1e400", "1.7976931348623159e308", "1.7976931348623157e308", "1e999999999999",
           "1e-999999999999", "4.9e-324", "2.4703282292062327e-324", "2.4703282292062328e-324", "1e-400", "-1e-400",
           "0.1000000000000000055511151231257827", "1.5", " 1.5", "1,5", "0x1p3", "1e", "e5", ".", ".e5", "-.", "+",
           "-", "--1", "+-1", "1..2", "1e5.", "00", "0.", ".5", "1d5", "1.0f", "true", "false", "TRUE", "False",
           "tRuE", "yes", "t", "01", "2", " true", "true ", "2024-02-29", "2024-02-30", "1900-02-29", "2000-02-29",
           "2024-1-2", "20240102", "2024-01-02T00", "2024-01-02 ", "-2024-01-01", "+2024-01-01", "12024-01-01",
           "0000-01-01", "0001-01-01", "9999-12-31", "2024-13-01", "2024-00-10", "2024-04-31", "2024-01-00",
           "2024-01-02T03", "2024-01-02 03:04", "2024-01-02T03:04:05", "2024-01-02T03:04:05.123456",
           "2024-01-02T03:04:05.", "2024-01-02T24:00:00", "2024-01-02T23:59:60", "2024-01-02T3:04",
           "2024-01-02T03:04:05Z", "2024-01-02T03:04:05+01:00", "2024-01-02T03:04:05+0100", "2024-01-02T03:04:05+01",
           "2024-01-02T03Z", "2024-01-02Z", "2024-01-02T03:04:05.1234567", "2024-01-02T03:04:05.000",
           "2024-01-02T03:04:05.123", "2024-01-02T03:04:05.123456789", "2024-01-02T03:04:05.1234567890",
           "2024-01-02T0304", "2024-01-02T03:04:05-23:59", "2024-01-02T03:04:05+24:00", "2024-01-02T03:04:05 +01:00",
           "2024-01-02T03:04:05+1", "2024-01-02T03:04.5", "2024-01-02T", "2024-01-02T03:", "2024-01-02T030405",
           "2024-01-02T03:04:05+01:0", "2024-01-02T03:04:05+01:60", "2024-01-02T03:04:05z", "2024-01-02+01:00",
           "2024-01-02t03", "2024-01-02  03", "2024-01-02T03+0100", "2262-04-11T23:47:16.854775807",
           "2262-04-11T23:47:16.854775808", "1677-09-21T00:12:43.145224192", "1677-09-21T00:12:44",
           "1677-09-21T00:12:43", "2262-04-11T23:47:17", "2262-04-11T23:47:16.854775807-01:00",
           "1677-09-21T00:12:43.145224191-01:00", "1677-09-21T00:12:44+01:00", "1970-01-01", "1969-12-31T23:59:59.999",
           "é", "١", "１"]


def int_corpus() -> List[str]:
    out = []
    for bits in (8, 16, 32, 64):
        for lo, hi in ((-(1 << (bits - 1)), (1 << (bits - 1)) - 1), (0, (1 << bits) - 1)):
            for v in (lo, hi):
                out += [str(v - 1), str(v), str(v + 1)]
        for nd in range(1, bits // 4 + 2):
            for d in ("0", "1", "7", "8", "f", "F"):
                out += ["0x" + d * nd, "0X" + d * nd, "0x" + "0" * (nd - 1) + "1"]
    out += [str(1 << 64), str((1 << 64) + 1), "0" * 30 + "7", "-" + "0" * 30 + "128", "-" + "0" * 40]
    return out


def random_doubles(count: int, seed: int) -> List[str]:
    """repr, %.17g, %.20g and %.40g of random finite double bit patterns."""
    rng = np.random.default_rng(seed)
    bits = rng.integers(0, 1 << 63, count, dtype=np.int64).astype(np.uint64) | \
        (rng.integers(0, 2, count).astype(np.uint64) << np.uint64(63))
    vals = bits.view(np.float64)
    vals = vals[np.isfinite(vals)]
    out: List[str] = []
    for fmt in (repr, "%.17g".__mod__, "%.20g".__mod__, "%.40g".__mod__):
        out.extend(fmt(float(v)) for v in vals)
    return out


def _next_up(x: float) -> float:
    return struct.unpack("<d", struct.pack("<q", struct.unpack("<q", struct.pack("<d", x))[0] + 1))[0]


def _decimal(fr: fractions.Fraction, digits: int) -> str:
    """``fr`` (> 0) as a decimal string, exact when its expansion ends within ``digits`` significant digits."""
    n, d = fr.numerator, fr.denominator
    e = 0
    while n >= d * 10:
        d *= 10
        e += 1
    while n < d:
        n *= 10
        e -= 1
    s = (n * 10 ** (digits - 1)) // d
    return f"{str(s)[0]}.{str(s)[1:]}e{e}"


def halfway_corpus(count: int, seed: int, f32: bool = False) -> List[str]:
    """Exact decimal halfway points between adjacent floats, and the decimals one unit above and below them in
    the last digit: significands of up to 800 digits, most of which go through the undecided path."""
    rng = random.Random(seed)
    out = []
    for _ in range(count):
        if f32:
            b = rng.randrange(1, 0x7F7FFFFF)
            a = struct.unpack("<f", struct.pack("<I", b))[0]
            nxt = struct.unpack("<f", struct.pack("<I", b + 1))[0]
        else:
            b = rng.randrange(1, 0x7FEFFFFFFFFFFFFF)
            a = struct.unpack("<d", struct.pack("<Q", b))[0]
            nxt = _next_up(a)
        mid = (fractions.Fraction(a) + fractions.Fraction(nxt)) / 2
        n, d = mid.numerator, mid.denominator
        k = 0
        while d % 10 and k < 2000:  # d is a power of two: the expansion ends after as many digits as its log2
            d *= 10
            k += 1
        digits = len(str(mid.numerator * 10 ** k // mid.denominator)) + 1
        s = _decimal(mid, digits)
        mant, exp = s.split("e")
        last = int(mant.replace(".", ""))
        width = len(mant) - 1
        for delta in (0, 1, -1):
            v = str(last + delta).rjust(width, "0")
            out.append(f"{v[0]}.{v[1:]}e{exp}")
    return out


def boundary_floats() -> List[str]:
    out = ["4.9406564584124654e-324", "2.4703282292062327e-324", "2.4703282292062328e-324", "2.2250738585072011e-308",
           "2.2250738585072014e-308", "2.2250738585072012e-308", "1.7976931348623157e308", "1.7976931348623158e308",
           "1.7976931348623159e308", "1.40129846e-45", "7.0064923e-46", "7.0064924e-46", "1.1754942e-38",
           "1.17549435e-38", "3.4028234e38", "3.4028235e38", "3.40282357e38", "3.4028236e38", "9007199254740993",
           "9007199254740992", "9007199254740991", "16777217", "16777216", "16777215", "1e22", "1e23", "1e-22",
           "1e-23", "1e10", "1e11", "1e-10", "1e-11", "123456789012345678901234567890"]
    for e in range(-350, 320, 7):
        out += [f"1e{e}", f"9.999999999999999e{e}", f"5e{e}"]
    return out


def all_dates() -> List[str]:
    d = datetime.date(1, 1, 1)
    one = datetime.timedelta(days=1)
    out = []
    while True:
        out.append(d.isoformat())
        if d == datetime.date(9999, 12, 31):
            return out
        d += one


def random_timestamps(count: int, seed: int) -> List[str]:
    rng = random.Random(seed)
    out = []
    for _ in range(count):
        y = rng.choice([rng.randrange(1, 10000), rng.randrange(1670, 2270), rng.randrange(1960, 2040)])
        s = f"{y:04d}-{rng.randrange(1, 13):02d}-{rng.randrange(1, 29):02d}"
        form = rng.randrange(6)
        if form > 0:
            s += rng.choice("T ") + f"{rng.randrange(24):02d}"
        if form > 1:
            s += f":{rng.randrange(60):02d}"
        if form > 2:
            s += f":{rng.randrange(60):02d}"
        if form > 3:
            s += "." + "".join(rng.choice("0123456789") for _ in range(rng.randrange(0, 10)))
        if rng.random() < 0.5:
            s += rng.choice(["Z", f"+{rng.randrange(24):02d}", f"-{rng.randrange(24):02d}{rng.randrange(60):02d}",
                             f"+{rng.randrange(24):02d}:{rng.randrange(60):02d}"])
        out.append(s)
    return out


MUTATION_BYTES = "0123456789+-.eE:T Z" + "abcdfnixyAFINX"


def mutants(valid: Sequence[str], count: int, seed: int) -> List[str]:
    rng = random.Random(seed)
    out = []
    for _ in range(count):
        s = rng.choice(valid)
        k = rng.randrange(len(s) + 1)
        op = rng.randrange(3)
        c = rng.choice(MUTATION_BYTES)
        if op == 0:
            s = s[:k] + c + s[k:]
        elif op == 1 and s:
            k = min(k, len(s) - 1)
            s = s[:k] + s[k + 1:]
        elif s:
            k = min(k, len(s) - 1)
            s = s[:k] + c + s[k + 1:]
        out.append(s)
    return out
