"""The boundary the operators' data crosses, against exact references: the validity-bitmap kernels, Arrow ingest and
export, segment copies, and the pipelined host -> device -> host ``fa.transform``.

a. ``K.bits_to_bytes`` / ``K.bytes_to_bits`` against ``np.unpackbits`` / ``np.packbits`` at every bit offset, at odd
   lengths and past the row count one launch grid covers.
b. ``B200Table.from_arrow`` -> ``to_arrow`` on every key type, ``large_string``, an all-NULL column and 0-row tables,
   from chunks sliced at every offset 0-7, with and without a validity buffer: values of valid slots by storage bits.
c. ``K.copy_segments`` against numpy on random plans (every width, several source tables, runs of 0 / 1 / odd /
   several pieces / above the piece cap, odd source offsets, more segments than one grid row), with a sentinel in
   every destination byte no run covers; ``B200Table.compacted()`` against a numpy concatenation.
d. The pipelined transform against the same call on a device table and against the oracle's stable hash partition
   on the normalised keys (DESIGN §7d), on every key type it takes; a spy proves which path produced each result.
"""
from collections import defaultdict

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

from _key_types import KEY_TYPES, TYPES, _storage_type, key_array  # noqa: E402
from fugue_b200 import api as fa  # noqa: E402
from fugue_b200 import kernels as K  # noqa: E402
from fugue_b200 import sort as S  # noqa: E402
from fugue_b200 import streaming  # noqa: E402
from fugue_b200.colmap import ColumnMap  # noqa: E402
from fugue_b200.column import col  # noqa: E402
from fugue_b200.dataframe import B200DataFrame  # noqa: E402
from fugue_b200.partition import PartitionSpec  # noqa: E402
from fugue_b200.schema import Schema  # noqa: E402
from fugue_b200.table import B200Table  # noqa: E402
from oracle import hash_partition as hp  # noqa: E402
from oracle.keys import canonical_rows  # noqa: E402

DEV = torch.device("cuda", 0)


def _sms() -> int:
    return torch.cuda.get_device_properties(DEV).multi_processor_count


@pytest.fixture(scope="module")
def engine():
    return fa.make_execution_engine("b200")


def _bits(a) -> np.ndarray:
    """Storage bits (unsigned, of the type's width) of every slot of a fixed-width Arrow array."""
    if isinstance(a, pa.ChunkedArray):
        a = a.combine_chunks() if a.num_chunks > 0 else pa.array([], type=a.type)
    w = a.type.bit_width // 8
    if len(a) == 0:
        return np.zeros(0, dtype=f"u{w}")
    return np.frombuffer(a.buffers()[1], dtype=f"u{w}", count=a.offset + len(a))[a.offset:]


def _host(t: torch.Tensor) -> np.ndarray:
    a = t.cpu().numpy()
    return a.view(f"u{a.dtype.itemsize}")


# ---- a. validity bitmap kernels ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("length", [0, 1, 7, 8, 9, 255, 257])
def test_bits_to_bytes_every_bit_offset(length):
    rng = np.random.default_rng(length)
    for off in list(range(16)) + [8 * 1000 + 5]:
        nbytes = (off + length + 7) // 8
        bits = rng.integers(0, 256, max(nbytes, 1), dtype=np.uint8)  # exactly the bytes the rows span
        got = K.bits_to_bytes(torch.from_numpy(bits).to(DEV), off, length).cpu().numpy()
        exp = np.unpackbits(bits, bitorder="little")[off:off + length]
        assert got.dtype == np.uint8 and np.array_equal(got, exp), (off, length)


def test_bits_to_bytes_beyond_one_grid():
    """The launch is capped at 16 CTAs per SM x 256 threads: more rows than that take the grid-stride loop."""
    rng = np.random.default_rng(1)
    cap = 16 * _sms() * 256
    for off, length in ((3, 2 * cap + 11), (13, cap + 1)):
        bits = rng.integers(0, 256, (off + length + 7) // 8, dtype=np.uint8)
        got = K.bits_to_bytes(torch.from_numpy(bits).to(DEV), off, length).cpu().numpy()
        assert np.array_equal(got, np.unpackbits(bits, bitorder="little")[off:off + length]), (off, length)


def _check_bytes_to_bits(mask: np.ndarray) -> None:
    d = torch.from_numpy(mask).to(DEV)
    bits, nulls = K.bytes_to_bits(d)
    exp = np.packbits(mask != 0, bitorder="little")  # unused high bits of the last byte are zero
    got = bits.cpu().numpy()
    assert got.shape == exp.shape and np.array_equal(got, exp), len(mask)
    assert int(nulls.item()) == int((mask == 0).sum()), len(mask)


@pytest.mark.parametrize("length", [0, 1, 7, 8, 9, 255, 257, 4099])
def test_bytes_to_bits_tail_and_null_count(length):
    rng = np.random.default_rng(length)
    # any nonzero byte is valid; 1 is what the kernels write, 2 / 0x80 / 0xFF are what other code may hand in
    mask = np.array([0, 1, 2, 0x80, 0xFF], dtype=np.uint8)[rng.integers(0, 5, length)]
    _check_bytes_to_bits(mask)
    if length > 0:
        _check_bytes_to_bits(np.full(length, 0xFF, dtype=np.uint8))  # all valid: tail bits still zero
        _check_bytes_to_bits(np.zeros(length, dtype=np.uint8))


def test_bytes_to_bits_beyond_one_grid():
    """One thread per output byte, capped at 16 CTAs per SM x 256 threads: about 4.4 M rows on 132 SMs."""
    rng = np.random.default_rng(2)
    cap_rows = 16 * _sms() * 256 * 8
    for length in (cap_rows + 3, 2 * cap_rows + 13):
        mask = (rng.random(length) < 0.7).astype(np.uint8) * np.uint8(0x80)
        _check_bytes_to_bits(mask)


# ---- b. from_arrow -> to_arrow ----------------------------------------------------------------------------------------
ROUND_TRIP = TYPES + ["large_string"]


def _pool_array(name: str, n: int, rng, null_rate: float) -> pa.Array:
    if name == "large_string":
        return key_array("string", n, rng, null_rate).cast(pa.large_string())
    return key_array(name, n, rng, null_rate)


def _chunks(name: str, rng, salt: int) -> list:
    """Slices at every offset 0-7 of an array with NULLs, chunks of length 0 and 1, and chunks without a
    validity buffer, in one column.  String chunks each get values of their own, so their dictionaries differ."""
    def base(n, null_rate):
        a = _pool_array(name, n, rng, null_rate)
        if pa.types.is_string(a.type) or pa.types.is_large_string(a.type):
            a = pa.array([None if v is None else f"{v}{salt}.{i % 5}" for i, v in enumerate(a.to_pylist())],
                         type=a.type)
        return a

    with_nulls = base(80, 0.3)
    out = [with_nulls.slice(o, 9 + 3 * o) for o in range(8)]
    out += [with_nulls.slice(4, 0), with_nulls.slice(5, 1), with_nulls.slice(3, 1)]
    plain = base(23, 0.0)
    assert plain.buffers()[0] is None
    out += [plain, plain.slice(3, 11), with_nulls.slice(61, 17)]
    return out


def _check_round_trip(tbl: pa.Table) -> None:
    t = B200Table.from_arrow(tbl, DEV)
    assert t.num_rows == tbl.num_rows
    rt = t.to_arrow()
    assert rt.schema == tbl.schema
    for i, name in enumerate(tbl.column_names):
        src = tbl.column(name)
        tp = src.type
        ok = np.asarray(src.is_valid()) if tbl.num_rows > 0 else np.zeros(0, dtype=bool)
        # the device side: the byte mask and the stored values
        if t.valid[i] is None:
            assert src.null_count == 0, name
        else:
            assert np.array_equal(t.valid[i].cpu().numpy(), ok.astype(np.uint8)), name
        stored = t.columns[i].cpu().numpy()
        if pa.types.is_string(tp) or pa.types.is_large_string(tp):
            d = t.dictionaries[name].to_pylist()
            got_vals = [d[c] for c in stored[ok].tolist()]
            assert got_vals == [v for v in src.to_pylist() if v is not None], name
        elif pa.types.is_boolean(tp):
            assert stored.dtype == np.uint8 and set(np.unique(stored[ok]).tolist()) <= {0, 1}, name
            assert stored[ok].astype(bool).tolist() == [v for v in src.to_pylist() if v is not None], name
        else:
            assert np.array_equal(stored.view(f"u{stored.dtype.itemsize}")[ok], _bits(src)[ok]), name
        # the Arrow side after the round trip
        back = rt.column(name)
        assert back.type == tp and back.null_count == src.null_count, name
        if tbl.num_rows == 0:
            assert len(back) == 0
            continue
        assert np.array_equal(np.asarray(back.is_valid()), ok), name
        if pa.types.is_string(tp) or pa.types.is_large_string(tp) or pa.types.is_boolean(tp):
            assert back.to_pylist() == src.to_pylist(), name
        else:
            assert np.array_equal(_bits(back)[ok], _bits(src)[ok]), name


@pytest.mark.parametrize("name", ROUND_TRIP)
def test_arrow_round_trip_sliced_chunks(name):
    rng = np.random.default_rng([3, ROUND_TRIP.index(name)])
    chunks = _chunks(name, rng, 0)
    n = sum(len(c) for c in chunks)
    tp = chunks[0].type
    tbl = pa.table({
        "c": pa.chunked_array(chunks, type=tp),
        "other": pa.chunked_array(_chunks(name, rng, 1)[::-1], type=tp),  # the same chunks in another order
        "all_null": pa.chunked_array([pa.nulls(n - 7, tp).slice(0), pa.nulls(10, tp).slice(3)], type=tp),
        "rid": pa.array(np.arange(n, dtype=np.int64)),
    })
    _check_round_trip(tbl)
    _check_round_trip(tbl.slice(5, n - 12))  # the table sliced again: every chunk offset moves
    _check_round_trip(pa.table({"c": pa.chunked_array(chunks[3:4], type=tp)}))  # one chunk at offset 3


def test_arrow_round_trip_zero_rows():
    types = [KEY_TYPES[n][0] for n in TYPES] + [pa.large_string()]
    names = [f"c{i}" for i in range(len(types))]
    _check_round_trip(pa.table([pa.array([], type=tp) for tp in types], names=names))
    _check_round_trip(pa.table([pa.chunked_array([], type=tp) for tp in types], names=names))  # no chunks at all
    _check_round_trip(pa.table([pa.chunked_array([pa.array([], type=tp)] * 2, type=tp) for tp in types],
                               names=names))


# ---- c. segment copies ------------------------------------------------------------------------------------------------
WIDTHS = (1, 2, 4, 8)
SENTINEL = 0xA5


def _copy_plan(seed: int, lens: np.ndarray, ntab: int, odd_src: bool = True):
    """Run copy of every width from ``ntab`` source tables; returns (got, expected) destination bytes per width.
    Runs land in the destination in a shuffled order with gaps of 0-3 elements, every byte outside them is the
    sentinel, and every run stays inside its source and its destination."""
    rng = np.random.default_rng(seed)
    nseg = len(lens)
    tab = rng.integers(0, ntab, nseg)
    src_off = rng.integers(0, 400, nseg) * 2 + (rng.random(nseg) < 0.6 if odd_src else 0)  # odd: 8-byte head peel
    tlen = [int(max([0] + list(src_off[tab == s] + lens[tab == s]))) + int(rng.integers(1, 3)) for s in range(ntab)]
    place = rng.permutation(nseg)
    gaps = rng.integers(0, 4, nseg)
    dst_off = np.zeros(nseg, dtype=np.int64)
    pos = int(rng.integers(0, 3))
    for s in place:
        pos += int(gaps[s])
        dst_off[s] = pos
        pos += int(lens[s])
    dlen = pos + int(rng.integers(0, 3))
    srcs = [[rng.integers(0, 256, tlen[s] * w, dtype=np.uint8).view(f"u{w}") for w in WIDTHS] for s in range(ntab)]
    exp = [np.full(dlen * w, SENTINEL, dtype=np.uint8).view(f"u{w}") for w in WIDTHS]
    for sgi in range(nseg):
        a, ln, d = int(src_off[sgi]), int(lens[sgi]), int(dst_off[sgi])
        for c in range(len(WIDTHS)):
            exp[c][d:d + ln] = srcs[tab[sgi]][c][a:a + ln]
    dsrc = [torch.from_numpy(srcs[s][c].view(f"i{WIDTHS[c]}") if WIDTHS[c] > 1 else srcs[s][c]).to(DEV)
            for s in range(ntab) for c in range(len(WIDTHS))]
    ddst = [torch.full((dlen * w,), SENTINEL, dtype=torch.uint8, device=DEV).view(dsrc[c].dtype)
            for c, w in enumerate(WIDTHS)]
    t64 = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).to(DEV)  # noqa: E731
    K.copy_segments(dsrc, ddst, t64(src_off), t64(dst_off), t64(lens),
                    src_table=torch.from_numpy(tab.astype(np.int32)).to(DEV))
    return [_host(d) for d in ddst], exp


def _assert_copies(got, exp):
    for w, g, e in zip(WIDTHS, got, exp):
        assert g.shape == e.shape
        bad = np.flatnonzero(g != e)
        assert bad.size == 0, f"width {w}: {bad.size} elements differ, first at {bad[:5]}"


@pytest.mark.parametrize("seed", range(4))
def test_copy_segments_random_plans(seed):
    rng = np.random.default_rng([10, seed])
    nseg = 300
    kinds = rng.integers(0, 6, nseg)
    lens = np.select([kinds == 0, kinds == 1, kinds == 2, kinds == 3, kinds == 4],
                     [0, 1, 2, rng.integers(0, 500, nseg) * 2 + 1, rng.integers(1, 500, nseg) * 2],
                     rng.integers(8193, 30000, nseg)).astype(np.int64)
    lens[:6] = [0, 1, 2, 3, 8191, 8193]
    _assert_copies(*_copy_plan(seed, lens, ntab=3, odd_src=seed != 3))


def test_copy_segments_piece_cap():
    """Few long runs: every SM gets pieces of 8192 rows, at most 64 per run, so a run above 64 x 8192 rows makes
    pieces loop; with odd and even lengths and source offsets for the 16-byte path's head and tail."""
    lens = np.array([64 * 8192 + 12345, 64 * 8192 + 2, 3 * 8192 + 7, 1, 0, 2], dtype=np.int64)
    _assert_copies(*_copy_plan(20, lens, ntab=2))


def test_copy_segments_beyond_one_grid_row():
    """More than 65535 segments: the CTAs of a column take several segments each."""
    rng = np.random.default_rng(21)
    lens = rng.integers(0, 5, 70_001).astype(np.int64)
    _assert_copies(*_copy_plan(21, lens, ntab=4))


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_compacted_matches_numpy(world):
    rng = np.random.default_rng([22, world])
    nown = 6
    lens = rng.integers(0, 3000, (world, nown)).astype(np.int64)
    lens[:, 2] = 0                        # a partition no rank sent rows to
    lens[0, 4] = 0
    lens[world - 1, 0] = 70_000           # a run of several pieces
    so = np.zeros((world, nown + 1), dtype=np.int64)
    start = 0
    for s in range(world):
        so[s] = start + np.concatenate([[0], np.cumsum(lens[s])])
        start = int(so[s, -1])
    n = start
    cols = [np.arange(n, dtype=np.int64), rng.standard_normal(n), rng.integers(-2**31, 2**31, n).astype(np.int32),
            rng.integers(-2**15, 2**15, n).astype(np.int16), rng.integers(0, 256, n).astype(np.uint8)]
    valid = [None, (rng.random(n) < 0.8).astype(np.uint8), None, (rng.random(n) < 0.5).astype(np.uint8), None]
    t = B200Table("rid:long,x:double,i:int,s:short,b:uint8", [torch.from_numpy(c).to(DEV) for c in cols],
                  [None if v is None else torch.from_numpy(v).to(DEV) for v in valid], partition_keys=["rid"])
    t.segment_offsets = torch.from_numpy(so)
    c = t.compacted()
    order = np.concatenate([np.arange(so[s, j], so[s, j + 1]) for j in range(nown) for s in range(world)]
                           + [np.zeros(0, dtype=np.int64)]).astype(np.int64)
    assert np.array_equal(c.offsets.cpu().numpy(), np.concatenate([[0], np.cumsum(lens.sum(0))]))
    for i in range(len(cols)):
        assert np.array_equal(c.columns[i].cpu().numpy(), cols[i][order]), i
        if valid[i] is None:
            assert c.valid[i] is None
        else:
            assert np.array_equal(c.valid[i].cpu().numpy(), valid[i][order]), i


# ---- d. the pipelined transform ---------------------------------------------------------------------------------------
STREAM_TYPES = [t for t in TYPES if t not in ("bool", "string")]  # the types the pipelined path takes
FLOATS = ("float16", "float32", "float64")
NUMS = (1, 3, 16, 256, 1000, K.MAX_PARTITIONS + 76)
ALL_FUNCS_AT = (3, 256, K.MAX_PARTITIONS + 76)
N = 9000
CUTS = (0, 1, 8, 1003, 1003, 4100, 4101, N)  # chunks of 1, 7, 995, 0, 3097, 1 and 4899 rows, at offset slices


def _key_column(name: str, n: int, rng) -> pa.Array:
    """Every pool value of the type (for floats +-0.0 and NaN payloads), the rest half pool values and half random
    storage bits, so floats also carry random NaN payloads and subnormals, and there are many distinct keys."""
    tp, pool = KEY_TYPES[name]
    st = _storage_type(tp)
    npdt = np.dtype(st.to_pandas_dtype())
    vals = pool.astype(npdt)[rng.integers(0, len(pool), n)]
    vals[: len(pool)] = pool.astype(npdt)
    rnd = rng.integers(0, 256, n * npdt.itemsize, dtype=np.uint8).view(npdt)
    pick = rng.random(n) < 0.5
    pick[: len(pool)] = False
    vals = np.where(pick, rnd, vals)
    a = pa.array(vals, type=st)
    return a.view(tp) if st != tp else a


def _stream_input(keys, seed: int) -> pa.Table:
    rng = np.random.default_rng(seed)
    cols = {"rid": pa.array(np.arange(N, dtype=np.int64))}
    for k, name in keys:
        cols[k] = _key_column(name, N, rng) if name != "int_small" else pa.array(rng.integers(-3, 4, N))
    cols.update(p1=pa.array(rng.integers(0, 256, N).astype(np.uint8)),
                p2=pa.array(rng.integers(-2**15, 2**15, N).astype(np.int16)),
                p4=pa.array(rng.standard_normal(N).astype(np.float32)),
                p8=pa.array(rng.standard_normal(N)))
    tbl = pa.table(cols)
    return pa.concat_tables([tbl.slice(a, b - a) for a, b in zip(CUTS[:-1], CUTS[1:])])


def _normalised(a: pa.ChunkedArray):
    """The key as the logical hash partition hashes it (DESIGN §7d), restated: float bits at the width the device
    uses (float16 widened to float64), -0.0 read as 0.0, NaN as NULL; other types by their storage."""
    bits = _bits(a)
    if not pa.types.is_floating(a.type):
        return bits, None  # hashed zero-extended from their own width, as pandas does
    f = bits.view({16: np.float16, 32: np.float32, 64: np.float64}[a.type.bit_width])
    if a.type == pa.float16():
        f = f.astype(np.float64)
    f = np.where(f == 0, np.zeros_like(f), f)
    return f, ~np.isnan(f)


def _oracle(tbl: pa.Table, keys, num: int):
    cols, valid = zip(*[_normalised(tbl.column(k)) for k in keys])
    pids = hp.partition_ids(list(cols), num, list(valid))
    return hp.stable_partition(pids, num)


def _functions(tbl: pa.Table, keys):
    sch = Schema(tbl.schema)
    key_fields = [tbl.schema.field(k) for k in keys]

    def identity(t: B200Table) -> B200Table:
        return t

    def add_col(t: B200Table) -> B200Table:
        return B200Table(Schema(t.schema, "w:double"), list(t.columns) + [t.column("p8") * 2.0 + 1.0])

    reordered = ["p8", "rid"] + list(reversed(keys)) + ["p1"]

    def drop_reorder(t: B200Table) -> B200Table:
        return t.select(reordered)

    def filter_rows(t: B200Table) -> B200Table:
        return S.take_rows(t, K.compact_indices((t.column("rid") % 3 != 1) & (t.column("p4") < 0.8)))

    def fresh(t: B200Table) -> B200Table:
        return B200Table(Schema("x:long,y:double,z:int"), [t.column("rid") * 7 - 1, t.column("p8") - 0.5,
                                                           t.column("p2").to(torch.int32) * 3])

    cm = ColumnMap(col("rid"), *[col(k) for k in keys], (col("p8") * 2.0).alias("w"), col("p1"))
    return [
        ("identity", identity, sch),
        ("add_col", add_col, Schema(sch, "w:double")),
        ("drop_reorder", drop_reorder, sch.extract(reordered)),
        ("filter", filter_rows, sch),
        ("fresh", fresh, Schema("x:long,y:double,z:int")),
        ("column_map", cm, Schema(pa.schema([pa.field("rid", pa.int64())] + key_fields
                                            + [pa.field("w", pa.float64()), pa.field("p1", pa.uint8())]))),
        # every output an aligned 8-byte column: the map is fused into the scatter on the device table (K4)
        ("column_map_fused", ColumnMap(col("rid"), (col("p8") * 3.0).alias("w")), Schema("rid:long,w:double")),
    ]


def _same_bits(got: pa.Table, exp: pa.Table, what) -> None:
    assert got.schema == exp.schema, what
    for c in exp.column_names:
        g, e = got.column(c), exp.column(c)
        assert g.null_count == 0 and e.null_count == 0, (what, c)
        assert np.array_equal(_bits(g), _bits(e)), (what, c)


def _run_case(engine, monkeypatch, keys, seed: int) -> None:
    tbl = _stream_input(keys, seed)
    names = [k for k, _ in keys]
    rid = np.arange(N)
    spied = []
    real = streaming.streaming_transform

    def spy(*a, **kw):
        r = real(*a, **kw)
        spied.append(r is not None)
        return r

    monkeypatch.setattr(streaming, "streaming_transform", spy)
    canon = canonical_rows(tbl, names)
    for num in NUMS:
        order, offsets = _oracle(tbl, names, num)
        spec = PartitionSpec(by=names, algo="hash", num=num)
        funcs = _functions(tbl, names)
        if num not in ALL_FUNCS_AT:
            funcs = funcs[:1]
        for fname, fn, out_schema in funcs:
            what = (names, num, fname)
            seen = []

            def recorded(t: B200Table, fn=fn):
                seen.append((t.offsets.cpu().numpy(), t.column("rid").cpu().numpy()))
                return fn(t)

            using = fn if isinstance(fn, ColumnMap) else recorded
            ran = len(spied)
            got = fa.transform(tbl, using, schema=out_schema, partition=spec, engine=engine, as_local=True,
                               as_fugue=True).as_arrow()
            assert len(spied) == ran + 1, what
            assert spied[-1] == (num <= K.MAX_PARTITIONS), what  # the pipelined path ran, or declined
            exp = fa.transform(B200DataFrame(B200Table.from_arrow(tbl, DEV)), using, schema=out_schema,
                               partition=spec, engine=engine, as_local=True, as_fugue=True).as_arrow()
            assert len(spied) == ran + 1, what  # a device table never takes the pipelined path
            _same_bits(got, exp, what)
            # inside the function: the oracle's partition, and every canonical key tuple in one partition
            for off, r in seen:
                assert np.array_equal(off, offsets), what
                assert np.array_equal(r, rid[order]), what
                part = np.searchsorted(off, np.arange(N), side="right") - 1
                where = defaultdict(set)
                for row, p in zip(r.tolist(), part.tolist()):
                    where[canon[row]].add(p)
                assert all(len(p) == 1 for p in where.values()), what
            if fname == "identity":
                assert len(seen) == 2, what
                assert np.array_equal(np.asarray(got.column("rid")), rid[order]), what
                for c in tbl.column_names:
                    assert np.array_equal(_bits(got.column(c)), _bits(tbl.column(c))[order]), (what, c)


@pytest.mark.parametrize("name", STREAM_TYPES)
def test_pipelined_transform_one_key(engine, monkeypatch, name):
    _run_case(engine, monkeypatch, [("k", name)], 30 + STREAM_TYPES.index(name))


@pytest.mark.parametrize("name", FLOATS)
def test_pipelined_transform_float_and_int_key(engine, monkeypatch, name):
    _run_case(engine, monkeypatch, [("k", name), ("j", "int_small")], 60 + FLOATS.index(name))
    _run_case(engine, monkeypatch, [("j", "int_small"), ("k", name)], 70 + FLOATS.index(name))


def test_pipelined_transform_two_float_keys(engine, monkeypatch):
    _run_case(engine, monkeypatch, [("k", "float16"), ("g", "float64")], 80)
