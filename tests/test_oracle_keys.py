"""oracle/keys.py (the canonical key of a cell) against oracle/sort.null_and_rank and the rule of DESIGN §7d, and
oracle/join.join_rows on every key type.  Runs without a GPU."""
from collections import Counter

import numpy as np
import pyarrow as pa
import pytest

from _key_types import KEY_TYPES, TYPES, key_array
from oracle import join as oj
from oracle import sort as O
from oracle.keys import canonical, canonical_rows


@pytest.mark.parametrize("name", TYPES)
def test_canonical_keys_are_the_classes_of_null_and_rank(name):
    """Two cells have equal canonical keys exactly when null_and_rank gives them equal (NULL flag, rank)."""
    a = key_array(name, 600, np.random.default_rng([1, TYPES.index(name)]))
    for arr in (a, a.dictionary_encode() if name == "string" else a):
        keys = canonical(arr)
        null, rank = O.null_and_rank(pa.table({"k": arr}), "k")
        cls = [None if nl else int(r) for nl, r in zip(null.tolist(), rank.tolist())]
        assert [k is None for k in keys] == [c is None for c in cls]
        pairs = set(zip(keys, cls))
        assert len(pairs) == len(set(keys)) == len(set(cls)), name  # one class for one key and the reverse
        for k in keys:
            hash(k)


def test_canonical_key_rule():
    f16 = pa.array(np.array([0x0000, 0x8000, 0x7E00, 0xFE01, 0x7BFF, 0x0001], dtype=np.uint16)).view(pa.float16())
    assert canonical(f16) == [0.0, 0.0, None, None, 65504.0, 2.0**-24]
    assert str(canonical(f16)[1]) == "0.0"  # -0.0 reads as 0.0
    f64 = pa.array([-0.0, float("nan"), None, float("-inf"), 5e-324])
    assert [str(x) for x in canonical(f64)] == ["0.0", "None", "None", "-inf", "5e-324"]
    assert canonical(pa.array([2**63, 2**64 - 1, None], type=pa.uint64())) == [2**63, 2**64 - 1, None]
    assert canonical(pa.array([2**31, 2**32 - 1], type=pa.uint32())) == [2**31, 2**32 - 1]
    assert canonical(pa.array([-(2**63)], type=pa.int64())) == [-(2**63)]
    ts = pa.array(np.array([-(2**63), 2**63 - 1], dtype=np.int64)).view(pa.timestamp("s", tz="America/New_York"))
    assert canonical(ts) == [-(2**63), 2**63 - 1]  # storage: no datetime can hold these
    assert canonical(pa.array(np.array([-(2**31)], dtype=np.int32)).view(pa.date32())) == [-(2**31)]
    assert canonical(pa.array(["b", None, "a"]).dictionary_encode()) == ["b", None, "a"]
    assert canonical_rows(pa.table({"a": [1, None], "b": [-0.0, 2.0]}), ["a", "b"]) == [(1, 0.0), (None, 2.0)]


@pytest.mark.parametrize("name", TYPES)
def test_join_rows_matches_every_key_type_by_its_canonical_key(name):
    """A self-join on a key column gives count^2 rows per non-NULL canonical key; NULL and NaN keys match nothing."""
    a = key_array(name, 300, np.random.default_rng([2, TYPES.index(name)]), host_safe=True)
    t = pa.table({"k": a, "i": pa.array(np.arange(len(a)))})
    counts = Counter(k for k in canonical(a) if k is not None)
    exp = sum(c * c for c in counts.values())
    assert sum(oj.join_rows(t, t.rename_columns(["k", "j"]), "inner", ["k"]).values()) == exp
    semi = sum(oj.join_rows(t, t.select(["k"]), "semi", ["k"]).values())
    assert semi == sum(counts.values())


def test_join_rows_float16_example():
    t = pa.table({"k": pa.array(np.array([0.0, -0.0, np.nan, 1.5, -2.0, 65504.0], dtype=np.float16))})
    assert sum(oj.join_rows(t, t, "inner", ["k"]).values()) == 7  # {0, -0}^2 + 1.5 + -2 + 65504
