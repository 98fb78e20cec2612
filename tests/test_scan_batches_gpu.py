"""The K9 wrappers with more columns than one launch sequence takes (``SCAN_MAX_COLS + 1``): every column's outputs
equal, bit for bit, those of the same column run alone.  Segments include empty ones, and the columns have NULLs."""
from typing import Any, List, Optional, Sequence

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

from fugue_b200 import kernels as K

DEV = torch.device("cuda", 0)
NCOLS = K.SCAN_MAX_COLS + 1
N = 20_000  # several tiles of 2048 rows
OPS = [K.AGG_SUM_F64, K.AGG_SUM_I64, K.AGG_COUNT, K.AGG_MIN_I64, K.AGG_MAX_I64, K.AGG_MIN_F64, K.AGG_MAX_F64]


def _offsets(rng: np.random.Generator) -> torch.Tensor:
    cuts = np.sort(rng.integers(0, N + 1, 300))
    cuts = np.concatenate([[0, 0], cuts, cuts[:20], [N, N]])  # empty segments at the ends and in between
    return torch.from_numpy(np.sort(cuts).astype(np.int64)).to(DEV)


def _f64(rng: np.random.Generator) -> torch.Tensor:
    v = rng.standard_normal(N) * 1e3
    v[rng.integers(0, N, 20)] = np.nan
    v[rng.integers(0, N, 10)] = np.inf
    return torch.from_numpy(v).to(DEV)


def _valid(rng: np.random.Generator, i: int) -> Optional[torch.Tensor]:
    return None if i % 3 == 0 else torch.from_numpy((rng.random(N) > 0.2).astype(np.uint8)).to(DEV)


def _op_columns(rng: np.random.Generator) -> List[Any]:
    cols = []
    for i in range(NCOLS):
        op = OPS[i % len(OPS)]
        if op == K.AGG_COUNT:
            v = None
        elif op in (K.AGG_SUM_I64, K.AGG_MIN_I64, K.AGG_MAX_I64):
            v = torch.from_numpy(rng.integers(-(2 ** 40), 2 ** 40, N)).to(DEV)
        else:
            v = _f64(rng)
        cols.append((op, v, _valid(rng, i)))
    return cols


def _same(batched: Sequence[Any], run_one: Any, items: Sequence[Any]) -> None:
    assert len(batched) == len(items) == NCOLS
    for item, got in zip(items, batched):
        exp = run_one([item])[0]
        assert len(got) == len(exp)
        for g, e in zip(got, exp):
            if e is None:
                assert g is None
                continue
            assert torch.equal(g.view(torch.int64), e.view(torch.int64))


def test_segmented_scan_batches():
    rng = np.random.default_rng(1)
    off, cols = _offsets(rng), _op_columns(rng)
    _same(K.segmented_scan(off, N, cols), lambda c: K.segmented_scan(off, N, c), cols)


@pytest.mark.parametrize("start,end", [(-3, 2), (-2000, 1500), (None, 5), (-5, None)])
def test_window_frame_batches(start, end):
    rng = np.random.default_rng(2)
    off, cols = _offsets(rng), _op_columns(rng)
    _same(K.window_frame(off, N, start, end, cols), lambda c: K.window_frame(off, N, start, end, c), cols)


def test_window_bounded_batches():
    rng = np.random.default_rng(3)
    cols = _op_columns(rng)
    lo = rng.integers(-10, N, N)
    lo_t = torch.from_numpy(lo).to(DEV)
    hi_t = torch.from_numpy(lo + rng.integers(-5, 3000, N)).to(DEV)
    _same(K.window_bounded(lo_t, hi_t, cols), lambda c: K.window_bounded(lo_t, hi_t, c), cols)


def test_segmented_moments_batches():
    rng = np.random.default_rng(4)
    off = _offsets(rng)
    cols = [(_f64(rng), _valid(rng, i)) for i in range(NCOLS)]
    _same(K.segmented_moments(off, N, cols), lambda c: K.segmented_moments(off, N, c), cols)


def test_segmented_shape_moments_batches():
    rng = np.random.default_rng(5)
    off = _offsets(rng)
    cols = [(_f64(rng), _valid(rng, i)) for i in range(NCOLS)]
    _same(K.segmented_shape_moments(off, N, cols), lambda c: K.segmented_shape_moments(off, N, c), cols)


def test_segmented_comoments_batches():
    rng = np.random.default_rng(6)
    off = _offsets(rng)
    pairs = [(_f64(rng), _valid(rng, i), _f64(rng), _valid(rng, i + 1)) for i in range(NCOLS)]
    _same(K.segmented_comoments(off, N, pairs), lambda c: K.segmented_comoments(off, N, c), pairs)
