"""A spy on the C entry points of the K7 hash join: which path produced a join's result.

``kernels.JoinTable`` (16-byte multimap) and ``kernels.join_fused`` (4-byte slots) each pick among a whole-table,
a region (one table region per hash partition) and a batched region mode, and fall back to the whole table when a
region overflows.  ``Launches`` records every call; ``path()`` and ``batches()`` name the mode of the last build,
the one whose table was kept.  The budgets are the L2 batch sizes of csrc/fb_join.cu: a change to them changes
``batches()`` and fails the tests that assert a batch count.
"""
from typing import Any, List, NamedTuple, Tuple

from fugue_b200 import _lib

# name -> argument positions of (nrows, capacity, num_parts, (partition offset pointers...))
SPIED = {
    "fb_join_build_u64": (2, 5, 6, (9,)),
    "fb_join_probe_count_u64": (2, 5, 6, ()),
    "fb_join_probe_write_u64": (2, 5, 6, ()),
    "fb_join2_build": (2, 5, 6, (9,)),
    "fb_join2_probe": (2, 6, 7, ()),
    "fb_join2_build_probe": (2, 10, 11, (5, 9)),
    "fb_join2_emit": (2, 5, 6, ()),
}
TABLE16 = ("fb_join_build_u64", "fb_join_probe_count_u64", "fb_join_probe_write_u64")
BUILDS = ("fb_join_build_u64", "fb_join2_build", "fb_join2_build_probe")
# bytes of table regions one batch works on, and bytes per slot
BUDGET = {"fb_join_build_u64": (64 << 20, 16), "fb_join2_build": (48 << 20, 4), "fb_join2_build_probe": (24 << 20, 4)}


class Call(NamedTuple):
    name: str
    nrows: int
    capacity: int
    parts: int
    offsets: Tuple[bool, ...]


class Launches:
    def __init__(self, monkeypatch: Any):
        lib = _lib.load()
        self.calls: List[Call] = []
        for name, (n, c, p, offs) in SPIED.items():
            def spy(*a: Any, _real: Any = getattr(lib, name), _name: str = name, _pos: tuple = (n, c, p, offs)) -> int:
                self.calls.append(Call(_name, int(a[_pos[0]]), int(a[_pos[1]]), int(a[_pos[2]]),
                                       tuple(bool(a[o]) for o in _pos[3])))
                return _real(*a)

            monkeypatch.setattr(lib, name, spy)

    def clear(self) -> None:
        self.calls.clear()

    def _kept(self, family: str) -> Tuple[Call, List[Call]]:
        fam = [c for c in self.calls if (c.name in TABLE16) == (family == "table16")]
        builds = [c for c in fam if c.name in BUILDS]
        assert builds, self.calls
        last = builds[-1]
        # every probe / emit after the kept build uses its table geometry
        after = fam[max(i for i, c in enumerate(fam) if c.name in BUILDS) + 1:]
        assert all((c.capacity, c.parts) == (last.capacity, last.parts) for c in after), fam
        return last, builds[:-1]

    def path(self, family: str = None) -> str:
        """The path of the last join since ``clear()``: ``family`` is "table16" or "fused" (default: the family of
        the last build)."""
        if family is None:
            family = "table16" if [c for c in self.calls if c.name in BUILDS][-1].name in TABLE16 else "fused"
        last, earlier = self._kept(family)
        if last.name == "fb_join2_build_probe":
            return "fused-build-probe"
        if last.parts == 0:
            return f"{family}-fallback" if any(b.parts > 0 for b in earlier) else family
        if family == "fused":
            return "fused-region"
        return "table16-batched" if last.offsets[0] else "table16-region"

    def batches(self, family: str = None) -> int:
        """Number of region batches the kept build ran in (1 without partition offsets)."""
        if family is None:
            family = "table16" if [c for c in self.calls if c.name in BUILDS][-1].name in TABLE16 else "fused"
        last, _ = self._kept(family)
        if last.parts == 0 or not all(last.offsets):
            return 1
        budget, slot = BUDGET[last.name]
        per = max(1, budget // (last.capacity // last.parts * slot))
        return -(-last.parts // per)
