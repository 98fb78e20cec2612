"""String functions on dictionary-encoded columns: ``LIKE`` and ``LENGTH``.

A string column is int32 codes on the device plus a dictionary (an Arrow ``string`` / ``large_string``
array) on the host (``table.py``).  LIKE and LENGTH depend on the string alone, so they are evaluated once
per dictionary entry on the device (K11, ``fb_strings.cu``) and the expression evaluator maps every row's
code to its entry's result (``FB_X_LOOKUP``, K8).

The dictionary's Arrow layout (offsets widened to int64, the UTF-8 bytes, a validity byte per entry) is
uploaded once per dictionary object and device.  The copy hangs off the ``pa.Array`` through a weak
reference: tables that share a dictionary object (``select``, ``rename``, filters, derived tables) share
the copy, and it is freed with the dictionary.
"""
import weakref
from typing import Any, Dict, List, Optional, Tuple

import numpy as np
import pyarrow as pa
import torch

from . import kernels as K

_CACHE: Dict[int, Tuple[Any, Dict[torch.device, "DeviceDictionary"]]] = {}
uploads = 0  # dictionaries copied to a device so far (the cache's misses)


class DeviceDictionary:
    """The Arrow layout of a string dictionary in device memory: entry i is
    ``data[offsets[i]:offsets[i + 1]]``; ``valid`` (uint8 per entry) is None when no entry is NULL."""

    def __init__(self, offsets: torch.Tensor, data: torch.Tensor, valid: Optional[torch.Tensor]):
        self.offsets, self.data, self.valid = offsets, data, valid
        self.size = int(offsets.shape[0]) - 1


def _upload(d: pa.Array, device: torch.device) -> DeviceDictionary:
    global uploads
    if not (pa.types.is_string(d.type) or pa.types.is_large_string(d.type)):
        raise NotImplementedError(f"string function on a dictionary of type {d.type}")
    n = len(d)
    bufs = d.buffers()
    if n == 0 or bufs[1] is None:
        offs = np.zeros(n + 1, dtype=np.int64)
    else:
        wide = np.int64 if pa.types.is_large_string(d.type) else np.int32
        offs = np.frombuffer(bufs[1], dtype=wide, count=d.offset + n + 1)[d.offset:].astype(np.int64)
    lo, hi = int(offs[0]), int(offs[-1])
    raw = np.frombuffer(bufs[2], dtype=np.uint8, count=hi)[lo:hi] if hi > lo else np.zeros(0, dtype=np.uint8)
    data = np.zeros(max(hi - lo, 1), dtype=np.uint8)  # at least one byte: a real device pointer
    data[:hi - lo] = raw
    valid = None
    if d.null_count > 0:
        valid = torch.from_numpy(d.is_valid().to_numpy(zero_copy_only=False).astype(np.uint8)).to(device)
    uploads += 1
    return DeviceDictionary(torch.from_numpy(offs - lo).to(device), torch.from_numpy(data).to(device), valid)


def device_dictionary(d: pa.Array, device: torch.device) -> DeviceDictionary:
    """The device copy of dictionary ``d`` on ``device``: uploaded on first use, then cached on ``d``."""
    key = id(d)
    ent = _CACHE.get(key)
    if ent is None or ent[0]() is not d:
        def drop(ref: Any, key: int = key) -> None:
            if key in _CACHE and _CACHE[key][0] is ref:
                del _CACHE[key]

        ent = (weakref.ref(d, drop), {})
        _CACHE[key] = ent
    per_dev = ent[1]
    if device not in per_dev:
        per_dev[device] = _upload(d, device)
    return per_dev[device]


def like_tokens(pattern: str, escape: Optional[str]) -> List[int]:
    """A LIKE pattern as the tokens of ``fb_string_like``: UTF-8 literal bytes, ``LIKE_ONE`` for ``_`` and
    ``LIKE_ANY`` for a run of ``%``; with an ``escape`` character, it makes the next character a literal.
    Raises ValueError for a pattern that ends in a lone escape character, NotImplementedError for a pattern
    of more than ``K.LIKE_MAX_TOKENS`` tokens."""
    toks: List[int] = []
    i = 0
    while i < len(pattern):
        ch = pattern[i]
        if escape is not None and ch == escape:
            if i + 1 == len(pattern):
                raise ValueError(f"LIKE pattern {pattern!r} ends in the escape character {escape!r}")
            toks.extend(pattern[i + 1].encode("utf-8"))
            i += 2
            continue
        if ch == "%":
            if not toks or toks[-1] != K.LIKE_ANY:
                toks.append(K.LIKE_ANY)
        elif ch == "_":
            toks.append(K.LIKE_ONE)
        else:
            toks.extend(ch.encode("utf-8"))
        i += 1
    if len(toks) > K.LIKE_MAX_TOKENS:
        raise NotImplementedError(f"LIKE pattern of {len(toks)} tokens; the device takes {K.LIKE_MAX_TOKENS}")
    return toks


def like_table(d: pa.Array, device: torch.device, pattern: str, escape: Optional[str]
               ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """Per entry of ``d``: 1 where it matches ``pattern``, as the 8-byte table ``FB_X_LOOKUP`` reads (int64),
    and the entry validity (None: no NULL entry)."""
    toks = like_tokens(pattern, escape)
    dd = device_dictionary(d, device)
    out, out_valid = K.string_like(dd.offsets, dd.data, dd.valid, toks)
    return out.to(torch.int64), (out_valid if dd.valid is not None else None)


def length_table(d: pa.Array, device: torch.device) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """Per entry of ``d``: its number of code points (int64), and the entry validity (None: no NULL)."""
    dd = device_dictionary(d, device)
    return K.string_length(dd.offsets, dd.data, dd.valid), dd.valid
