"""Oracle: the canonical grouping / matching key of an Arrow cell (CPU only, plain Python).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Two cells are in one group, one logical partition, or match in a join (NULLs aside) exactly when their canonical
keys are equal.  The rule is DESIGN §7d, for every key type:

* NULL, and a NaN of either sign and any payload, are ``None``;
* float16 / float32 / float64 values are Python ``float`` with -0.0 read as 0.0;
* signed and unsigned integers are Python ``int`` of their value (uint64 >= 2^63 is a positive int);
* bool is ``bool``, a string is ``str``;
* date32 / date64 / timestamp (any unit, with or without a time zone) / duration / time32 / time64 are the ``int``
  of their storage, so values outside Python's ``datetime`` range are keys like any other.

``oracle/sort.null_and_rank`` states the same classes as (NULL flag, dense rank); ``tests/test_oracle_keys.py`` checks
that the two agree on every key type.
"""
import math
from typing import Hashable, List, Sequence

import numpy as np
import pyarrow as pa


def _plain(a: pa.Array) -> pa.Array:
    """Dictionary arrays decoded; temporal arrays viewed as their integer storage."""
    if pa.types.is_dictionary(a.type):
        a = a.cast(a.type.value_type)
    if pa.types.is_temporal(a.type):
        a = a.view(pa.int32() if a.type.bit_width == 32 else pa.int64())
    return a


def canonical(a) -> List[Hashable]:
    """Canonical key of every cell of an Arrow array (or chunked array)."""
    if isinstance(a, pa.ChunkedArray):
        a = a.combine_chunks()
    a = _plain(a)
    if pa.types.is_floating(a.type):
        vals = np.asarray(a.cast(pa.float64()).fill_null(np.nan).to_numpy(zero_copy_only=False), dtype=np.float64)
        return [None if math.isnan(x) else x + 0.0 for x in vals.tolist()]  # -0.0 + 0.0 == 0.0
    return a.to_pylist()


def canonical_rows(table: pa.Table, names: Sequence[str]) -> List[tuple]:
    """Canonical key tuple of every row over the columns ``names``."""
    cols = [canonical(table.column(n)) for n in names]
    return list(zip(*cols)) if cols else [() for _ in range(table.num_rows)]
