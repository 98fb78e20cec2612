"""One value pool per key type, with the type's edges, for the key-type sweeps (``test_oracle_keys.py`` on the CPU and
``test_key_types_gpu.py`` on the device).

Every pool holds the type's MIN and MAX and the values where a key path goes wrong: 2^15 / 2^31 / 2^63 set the sign
bit of a uint16 / uint32 / uint64's storage; floats have +-0.0, +-inf, the smallest subnormals, a NaN and a negative
NaN with a payload (NULL under DESIGN §7d), and float16 its largest finite value 65504.  Columns are built from their
storage bits through Arrow, never through pandas, which would turn a NaN into a NULL.

``HOST_SAFE`` pools replace the temporal extremes (outside the range of Python's and pandas' date / time types) with
values a pandas host callback can receive.  time64 holds valid times of day only.
"""
import numpy as np
import pyarrow as pa

I8, I16, I32, I64 = (np.iinfo(t) for t in (np.int8, np.int16, np.int32, np.int64))
_TS = np.array([I64.min, I64.max, -1, 0, 1, 10**15], dtype=np.int64)
_TS_HOST = np.array([-(10**9), -1, 0, 1, 10**9], dtype=np.int64)

KEY_TYPES = {
    "int8": (pa.int8(), np.array([I8.min, I8.max, -1, 0, 1, 5], dtype=np.int8)),
    "int16": (pa.int16(), np.array([I16.min, I16.max, -1, 0, 256], dtype=np.int16)),
    "int32": (pa.int32(), np.array([I32.min, I32.max, -1, 0, 65536], dtype=np.int32)),
    "int64": (pa.int64(), np.array([I64.min, I64.max, I64.max - 1, -1, 0, 2**40], dtype=np.int64)),
    "uint8": (pa.uint8(), np.array([0, 1, 127, 128, 255], dtype=np.uint8)),
    "uint16": (pa.uint16(), np.array([0, 1, 2**15 - 1, 2**15, 2**16 - 1], dtype=np.uint16)),
    "uint32": (pa.uint32(), np.array([0, 1, 2**31 - 1, 2**31, 2**32 - 1], dtype=np.uint32)),
    "uint64": (pa.uint64(), np.array([0, 1, 2**63 - 1, 2**63, 2**64 - 2, 2**64 - 1], dtype=np.uint64)),
    # bits: 0, -0, 1, -1, inf, -inf, +-smallest subnormal, NaN, negative NaN with payload, 65504, -65504, 1.5
    "float16": (pa.float16(), np.array([0x0000, 0x8000, 0x3C00, 0xBC00, 0x7C00, 0xFC00, 0x0001, 0x8001, 0x7E00,
                                        0xFE01, 0x7BFF, 0xFBFF, 0x3E00], dtype=np.uint16)),
    "float32": (pa.float32(), np.array([0, 0x80000000, 0x3F800000, 0xBF800000, 0x7F800000, 0xFF800000, 1, 0x80000001,
                                        0x7FC00000, 0xFFC00001, 0x7F7FFFFF, 0xFF7FFFFF], dtype=np.uint32)),
    "float64": (pa.float64(), np.array([0, 1 << 63, 0x3FF0000000000000, 0xBFF0000000000000, 0x7FF0000000000000,
                                        0xFFF0000000000000, 1, (1 << 63) | 1, 0x7FF8000000000000,
                                        0xFFF80000FFFFFFFF, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF],
                                       dtype=np.uint64)),
    "bool": (pa.bool_(), np.array([False, True])),
    # first value "z": the dictionary's code order (first appearance) is not the sorted order
    "string": (pa.string(), np.array(["z", "", "a", "é", "日本", "Z", "ab", "a "], dtype=object)),
    "date32": (pa.date32(), np.array([I32.min, I32.max, -1, 0, 19000], dtype=np.int32)),
    "date64": (pa.date64(), np.array([I64.min, I64.max, -86_400_000, 0, 19000 * 86_400_000], dtype=np.int64)),
    "ts_s": (pa.timestamp("s"), _TS),
    "ts_ms": (pa.timestamp("ms"), _TS),
    "ts_us": (pa.timestamp("us"), _TS),
    "ts_ns": (pa.timestamp("ns"), _TS),
    "ts_tz": (pa.timestamp("us", tz="America/New_York"), _TS),
    "duration": (pa.duration("us"), _TS),
    "time64": (pa.time64("us"), np.array([0, 86_400 * 10**6 - 1, 1, 43_200 * 10**6], dtype=np.int64)),
}
TYPES = list(KEY_TYPES)

HOST_SAFE = {
    "date32": np.array([-700_000, -1, 0, 1, 2_900_000], dtype=np.int32),  # years 53 and 9909
    "date64": np.array([-700_000, -1, 0, 1, 2_900_000], dtype=np.int64) * 86_400_000,
    **{k: _TS_HOST for k in ("ts_s", "ts_ms", "ts_us", "ts_ns", "ts_tz", "duration")},
}


def _storage_type(tp: pa.DataType) -> pa.DataType:
    if pa.types.is_floating(tp):
        return {16: pa.uint16(), 32: pa.uint32(), 64: pa.uint64()}[tp.bit_width]
    if pa.types.is_temporal(tp):
        return pa.int32() if tp.bit_width == 32 else pa.int64()
    return tp


def key_array(name: str, n: int, rng: np.random.Generator, null_rate: float = 0.1, host_safe: bool = False) -> pa.Array:
    """``n`` cells of key type ``name`` drawn from its pool (every pool value appears when ``n`` allows), about
    ``null_rate`` of them NULL."""
    tp, pool = KEY_TYPES[name]
    if host_safe:
        pool = HOST_SAFE.get(name, pool)
    idx = rng.integers(0, len(pool), n)
    idx[: min(n, len(pool))] = np.arange(min(n, len(pool)))
    vals = pool[rng.permutation(idx)]
    mask = rng.random(n) < null_rate if null_rate > 0 else None
    if tp == pa.string():
        return pa.array(list(vals), mask=mask, type=tp)
    if tp == pa.bool_():
        return pa.array(vals, mask=mask, type=tp)
    st = _storage_type(tp)
    return pa.array(vals, mask=mask, type=st).view(tp) if st != tp else pa.array(vals, mask=mask, type=tp)
