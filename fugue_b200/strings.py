"""String functions on dictionary-encoded columns: ``LIKE`` and ``LENGTH``, and the functions that build
strings (``UPPER LOWER SUBSTR TRIM LTRIM RTRIM REPLACE CONCAT ||``).

A string column is int32 codes on the device plus a dictionary (an Arrow ``string`` / ``large_string``
array) on the host (``table.py``).  LIKE and LENGTH depend on the string alone, so they are evaluated once
per dictionary entry on the device (K11, ``fb_strings.cu``) and the expression evaluator maps every row's
code to its entry's result (``FB_X_LOOKUP``, K8).

The dictionary's Arrow layout (offsets widened to int64, the UTF-8 bytes, a validity byte per entry) is
uploaded once per dictionary object and device.  The copy hangs off the ``pa.Array`` through a weak
reference: tables that share a dictionary object (``select``, ``rename``, filters, derived tables) share
the copy, and it is freed with the dictionary.

A string-building expression over one string column is a function of the entry too (K12, ``fb_strbuild.cu``):
``string_chain`` reads it as the column and a chain of steps, ``evaluate`` runs the steps over the dictionary
on the device (one measure and one write launch per step; intermediate dictionaries stay on the device),
deduplicates the results and returns the new dictionary and the entry -> new code table the rows are mapped
through (``FB_X_LOOKUP``).  Results are cached per (dictionary object, chain) the same way as uploads.

REGEXP_MATCHES / REGEXP_FULL_MATCH are per-entry tables as LIKE is (``regex_table``), and REGEXP_EXTRACT /
REGEXP_REPLACE are chain steps (K15, ``fb_regex.cu``, compiled by ``regex.py``).

A cast of a string to a number, bool, date or timestamp is a function of the entry as well (K13,
``fb_strparse.cu``): ``parse_table`` parses every entry once and returns the per-entry table ``FB_X_LOOKUP`` reads,
cached per (dictionary object, device, target type).  The parse is Arrow's ``cast(safe=False)`` of the entry; the
few floats of more than 19 significant digits the device leaves undecided are re-parsed by pyarrow on the host
(``parse_fallbacks`` counts them).  An entry that does not parse is an error only when a valid row of the table
being evaluated refers to it (``check_referenced``).

A cast of a number, bool, date or timestamp to a string goes the other way (K14, ``fb_format.cu``): ``format_values``
finds the distinct values on the device, formats each once there and returns the codes into the new dictionary.
"""
import weakref
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import pyarrow as pa
import torch

from . import kernels as K
from . import regex as R
from .column import ColumnExpr, Kind, check_call, is_string_build, lit

_CACHE: Dict[int, Tuple[Any, Dict[Any, Any]]] = {}     # dictionary -> {device: DeviceDictionary}
_DERIVED: Dict[int, Tuple[Any, Dict[Any, Any]]] = {}   # dictionary -> {(chain, device): StringResult}
uploads = 0     # dictionaries copied to a device so far (the cache's misses)
transforms = 0  # string expressions evaluated over a dictionary so far (the result cache's misses)
parses = 0      # dictionaries parsed to a type so far (the parse cache's misses)
parse_fallbacks = 0  # entries re-parsed on the host because the device left them undecided


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


def _slot(cache: Dict[int, Tuple[Any, Dict[Any, Any]]], d: pa.Array) -> Dict[Any, Any]:
    """The cache entry of dictionary object ``d``: dropped when ``d`` is freed."""
    key = id(d)
    ent = cache.get(key)
    if ent is None or ent[0]() is not d:
        def drop(ref: Any, key: int = key) -> None:
            if key in cache and cache[key][0] is ref:
                del cache[key]

        ent = (weakref.ref(d, drop), {})
        cache[key] = ent
    return ent[1]


def device_dictionary(d: pa.Array, device: torch.device) -> DeviceDictionary:
    """The device copy of dictionary ``d`` on ``device``: uploaded on first use, then cached on ``d``."""
    per_dev = _slot(_CACHE, d)
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


regex_matches = 0  # dictionaries tested against a regular expression so far (the regex cache's misses)


def regex_table(d: pa.Array, device: torch.device, pattern: str, full: bool
                ) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """Per entry of ``d``: 1 where the regular expression ``pattern`` matches somewhere in it (``full``: matches
    all of it), as the int64 table ``FB_X_LOOKUP`` reads, and the entry validity (None: no NULL entry).  Computed
    on first use (K15), then cached on ``d``, so a repeated call launches nothing."""
    global regex_matches
    per = _slot(_DERIVED, d)
    key = (("REGEX", pattern, full), device)
    if key not in per:
        prog = R.match_program(pattern, full)
        regex_matches += 1
        dd = device_dictionary(d, device)
        out, out_valid = K.regex_match(dd.offsets, dd.data, dd.valid, prog)
        per[key] = (out.to(torch.int64), out_valid if dd.valid is not None else None)
    return per[key]


def length_table(d: pa.Array, device: torch.device) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """Per entry of ``d``: its number of code points (int64), and the entry validity (None: no NULL)."""
    dd = device_dictionary(d, device)
    return K.string_length(dd.offsets, dd.data, dd.valid), dd.valid


# ---- string-building functions ------------------------------------------------------------------------
def _utf8(fn: str, v: str) -> bytes:
    b = v.encode("utf-8")
    if len(b) > K.STR_MAX_LITERAL:
        raise NotImplementedError(f"{fn}: a literal of {len(b)} bytes; the device takes {K.STR_MAX_LITERAL}")
    return b


def _concat_parts(e: ColumnExpr) -> List[ColumnExpr]:
    """The operands of a chain of ``||`` (no alias or cast inside), left to right."""
    out: List[ColumnExpr] = []
    for a in e.args:
        if a.kind == Kind.BINARY and a.head == "||" and a.as_type is None and a.as_name == "":
            out.extend(_concat_parts(a))
        else:
            out.append(a)
    return out


def string_chain(e: ColumnExpr, string_columns: Any) -> Tuple[str, Tuple[Any, ...]]:
    """A string-building expression (``is_string_build``) as (its one string column, its steps), innermost
    step first.  ``string_columns``: the names of the table's string columns.  A step is a hashable tuple:
    ``("UPPER",)``, ``("LOWER",)``, ``("SUBSTR", start, length or None)``, ``("TRIM" / "LTRIM" / "RTRIM",
    characters)``, ``("REPLACE", from, to)``, ``("FORMAT", tokens, null_is_empty)`` for CONCAT / ``||``, or
    ``("REGEXP_EXTRACT", pattern, group)``, ``("REGEXP_REPLACE", pattern, rewrite, global)`` or ``("NULL",)`` (a
    NULL literal argument: every result is NULL).  Literals are UTF-8 bytes; regular expressions stay ``str``.
    Raises NotImplementedError for what the device does not evaluate (two different string operands, numbers
    in a concatenation, a non-literal argument, no string column) and ValueError for a wrong argument count
    or a literal of the wrong type."""

    def operand(x: Any) -> Tuple[str, Tuple[Any, ...]]:
        x = x if isinstance(x, ColumnExpr) else lit(x)
        str_cast = x.as_type is None or pa.types.is_string(x.as_type) or pa.types.is_large_string(x.as_type)
        if x.kind == Kind.NAMED and x.name in string_columns and str_cast:
            return x.name, ()
        if is_string_build(x) and str_cast:
            return chain(x)
        raise NotImplementedError(f"{e}: a string function needs a string expression over one string column, "
                                  f"got {x}")

    def chain(x: ColumnExpr) -> Tuple[str, Tuple[Any, ...]]:
        fn, args = ("||", list(x.args)) if x.kind == Kind.BINARY else check_call(x.head, x.args)
        if fn in ("CONCAT", "||"):
            parts = _concat_parts(x) if fn == "||" else args
            toks: List[int] = []
            base: Any = None
            null = False
            for p in parts:
                if p.kind == Kind.LITERAL and p.as_type is None:
                    if p.value is None:
                        null = True
                    elif isinstance(p.value, str):
                        toks.extend(p.value.encode("utf-8"))
                    else:
                        raise NotImplementedError(f"a number inside a concatenation: {x}")
                    continue
                fp = p.fingerprint()
                if base is None:
                    base = (fp, operand(p))
                elif base[0] != fp:
                    raise NotImplementedError(f"a concatenation of different string expressions (every operand "
                                              f"that is not a literal must be the same): {x}")
                toks.append(K.STR_SELF)
            if base is None:
                raise NotImplementedError(f"a concatenation of literals only (no string column): {x}")
            if len(toks) > K.STR_MAX_TOKENS:
                raise NotImplementedError(f"a concatenation of {len(toks)} tokens; the device takes {K.STR_MAX_TOKENS}")
            name, steps = base[1]
            step = ("NULL",) if (fn == "||" and null) else ("FORMAT", tuple(toks), fn == "CONCAT")
            return name, steps + (step,)
        vals = [a.value for a in args[1:]]  # literals of the types column.SCALARS gives
        name, steps = operand(args[0])
        if any(v is None for v in vals):
            return name, steps + (("NULL",),)
        if fn == "SUBSTR":
            for v in vals:
                if not -(1 << 62) <= v <= 1 << 62:
                    raise NotImplementedError(f"SUBSTR: {v} is outside [-2^62, 2^62]")
            step: Tuple[Any, ...] = ("SUBSTR", vals[0], vals[1] if len(vals) > 1 else None)
        elif fn in ("TRIM", "LTRIM", "RTRIM"):
            step = (fn, _utf8(fn, vals[0]) if vals else b" ")
        elif fn == "REPLACE":
            step = (fn, _utf8(fn, vals[0]), _utf8(fn, vals[1]))
        elif fn == "REGEXP_EXTRACT":
            group = vals[1] if len(vals) > 1 else 0
            R.extract_program(vals[0], group)  # the pattern's and the group's errors, before anything runs
            step = (fn, vals[0], group)
        elif fn == "REGEXP_REPLACE":
            step = (fn, vals[0], vals[1], R.replace_options(vals[2] if len(vals) > 2 else None))
            R.replace_program(*step[1:])
        else:
            step = (fn,)
        return name, steps + (step,)

    return chain(e)


class StringResult:
    """A string expression evaluated over a dictionary: the new ``dictionary`` (distinct entries, in the order
    of their first source entry), ``remap`` (int64: source entry -> new code; a per-entry table for
    ``FB_X_LOOKUP``), ``remap_valid`` (uint8, 0 where the result is NULL; None: no NULL result) and
    ``null_code``: the code of the result for a NULL row (None: NULL), which is not NULL only after a CONCAT."""

    def __init__(self, dictionary: pa.Array, remap: torch.Tensor, remap_valid: Optional[torch.Tensor],
                 null_code: Optional[int]):
        self.dictionary, self.remap, self.remap_valid, self.null_code = dictionary, remap, remap_valid, null_code


_STEP_OPS = {"UPPER": K.STR_UPPER, "LOWER": K.STR_LOWER, "SUBSTR": K.STR_SUBSTR, "TRIM": K.STR_TRIM,
             "LTRIM": K.STR_LTRIM, "RTRIM": K.STR_RTRIM, "REPLACE": K.STR_REPLACE, "FORMAT": K.STR_FORMAT}


def _step_args(step: Tuple[Any, ...]) -> Dict[str, Any]:
    name = step[0]
    if name == "SUBSTR":
        return {"start": step[1], "length": step[2]}
    if name in ("TRIM", "LTRIM", "RTRIM"):
        return {"lits": [step[1]]}
    if name == "REPLACE":
        return {"lits": [step[1], step[2]]}
    if name == "FORMAT":
        return {"tokens": step[1], "null_is_empty": step[2]}
    return {}


def _scan(lengths: torch.Tensor) -> Tuple[torch.Tensor, int]:
    """Offsets of outputs of ``lengths`` bytes (exclusive scan, n + 1 entries) and the total."""
    offs = torch.zeros(int(lengths.shape[0]) + 1, dtype=torch.int64, device=lengths.device)
    torch.cumsum(lengths, 0, out=offs[1:])
    return offs, int(offs[-1].item())


def apply_steps(offsets: torch.Tensor, data: torch.Tensor, valid: Optional[torch.Tensor], steps: Sequence[Any]
                ) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
    """The dictionary (offsets, data, validity) after ``steps``, entry for entry, on the device."""
    for step in steps:
        m = int(offsets.shape[0]) - 1
        if step[0] == "NULL":
            valid = torch.zeros(m, dtype=torch.uint8, device=offsets.device)
            continue
        if step[0] in ("REGEXP_EXTRACT", "REGEXP_REPLACE"):
            prog = R.extract_program(*step[1:]) if step[0] == "REGEXP_EXTRACT" else R.replace_program(*step[1:])
            lengths, out_valid = K.regex_transform(offsets, data, valid, prog)
            new_offsets, total = _scan(lengths)
            new_data = torch.empty(max(total, 1), dtype=torch.uint8, device=offsets.device)
            K.regex_transform(offsets, data, valid, prog, out_offsets=new_offsets, out_data=new_data)
            offsets, data, valid = new_offsets, new_data, out_valid
            continue
        op, kw = _STEP_OPS[step[0]], _step_args(step)
        lengths, out_valid = K.string_transform(op, offsets, data, valid, **kw)
        new_offsets, total = _scan(lengths)
        new_data = torch.empty(max(total, 1), dtype=torch.uint8, device=offsets.device)
        K.string_transform(op, offsets, data, valid, out_offsets=new_offsets, out_data=new_data, **kw)
        offsets, data, valid = new_offsets, new_data, out_valid
    return offsets, data, valid


def dedup(offsets: torch.Tensor, data: torch.Tensor, valid: Optional[torch.Tensor], bits: int = 64
          ) -> Tuple[pa.Array, torch.Tensor, Optional[torch.Tensor], DeviceDictionary]:
    """Distinct non-NULL entries of a device dictionary, in the order of their first entry: (the new dictionary
    as a ``pa.string()`` array, entry -> new code (int64, at least one element), its validity (None: no NULL
    entry), the new dictionary's device copy).  Equal entries are found through a hash of ``bits`` bits, a
    stable radix sort of the (hash, entry) pairs and a byte comparison inside each run of equal hashes."""
    from .sort import _radix_sort_pairs

    dev = offsets.device
    m = int(offsets.shape[0]) - 1
    if valid is not None and bool(valid.all().item()):
        valid = None
    ids = torch.arange(m, dtype=torch.int64, device=dev)
    sh, si = _radix_sort_pairs(K.string_hash(offsets, data, valid, bits), ids.clone())  # sorts in place
    canon = K.string_first_equal(offsets, data, valid, sh, si)
    keep = canon == ids
    if valid is not None:
        keep &= valid.bool()
    code = torch.cumsum(keep, 0) - 1
    remap = code[canon] if m > 0 else torch.zeros(1, dtype=torch.int64, device=dev)
    remap_valid = valid if m > 0 else torch.zeros(1, dtype=torch.uint8, device=dev)
    kept = torch.nonzero(keep).squeeze(1)
    k = int(kept.shape[0])
    new_offsets, total = _scan(offsets[kept + 1] - offsets[kept])
    if total > (1 << 31) - 1:
        raise NotImplementedError(f"a string result of {total} bytes; a pa.string() dictionary holds 2^31 - 1")
    new_data = torch.empty(max(total, 1), dtype=torch.uint8, device=dev)
    K.string_transform(K.STR_COPY, offsets, data, None, src=kept, out_offsets=new_offsets, out_data=new_data)
    host_offsets = new_offsets.cpu().numpy().astype(np.int32)
    host_data = new_data[:total].cpu().numpy()
    d = pa.Array.from_buffers(pa.string(), k, [None, pa.py_buffer(host_offsets), pa.py_buffer(host_data)])
    return d, remap.contiguous(), remap_valid, DeviceDictionary(new_offsets, new_data, None)


def _evaluate(d: pa.Array, device: torch.device, steps: Tuple[Any, ...]) -> StringResult:
    global transforms
    transforms += 1
    dd = device_dictionary(d, device)
    n = dd.size
    offsets, data, valid = dd.offsets, dd.data, dd.valid
    extra = any(s[0] == "FORMAT" and s[2] for s in steps)
    if extra:  # one more entry, NULL: what a NULL row becomes (CONCAT skips NULL operands)
        ones = torch.ones(n, dtype=torch.uint8, device=device)
        offsets = torch.cat([offsets, offsets[-1:]])
        valid = torch.cat([ones if valid is None else valid, torch.zeros(1, dtype=torch.uint8, device=device)])
    offsets, data, valid = apply_steps(offsets, data, valid, steps)
    new, remap, remap_valid, copy = dedup(offsets, data, valid)
    _slot(_CACHE, new)[device] = copy  # the new dictionary's device copy: LIKE / LENGTH of it upload nothing
    null_code = None
    if extra and (remap_valid is None or bool(remap_valid[n].item())):
        null_code = int(remap[n].item())
    return StringResult(new, remap, remap_valid, null_code)


def evaluate(d: pa.Array, device: torch.device, steps: Tuple[Any, ...]) -> StringResult:
    """``steps`` (``string_chain``) over dictionary ``d`` on ``device``: computed on first use, then cached on
    ``d``, so a repeated call launches nothing and returns the same ``StringResult`` (the same ``pa.Array``)."""
    per = _slot(_DERIVED, d)
    key = (steps, device)
    if key not in per:
        per[key] = _evaluate(d, device, steps)
    return per[key]


# ---- casts from strings (K13) -------------------------------------------------------------------------
_INT_TARGETS = {8: (K.PARSE_I8, K.PARSE_U8), 16: (K.PARSE_I16, K.PARSE_U16), 32: (K.PARSE_I32, K.PARSE_U32),
                64: (K.PARSE_I64, K.PARSE_U64)}
_TS_UNITS = {"s": K.TU_S, "ms": K.TU_MS, "us": K.TU_US, "ns": K.TU_NS}


def parse_target(tp: pa.DataType) -> int:
    """The ``fb_string_parse`` target of a cast from a string to ``tp``; NotImplementedError for a type the device
    does not parse to (float16, decimal, binary, nested, time, duration ...)."""
    if pa.types.is_integer(tp):
        return _INT_TARGETS[tp.bit_width][pa.types.is_unsigned_integer(tp)]
    if pa.types.is_float32(tp) or pa.types.is_float64(tp):
        return K.PARSE_F32 if pa.types.is_float32(tp) else K.PARSE_F64
    if pa.types.is_boolean(tp):
        return K.PARSE_BOOL
    if pa.types.is_date32(tp) or pa.types.is_date64(tp):
        return K.PARSE_DATE32 if pa.types.is_date32(tp) else K.PARSE_DATE64
    if pa.types.is_timestamp(tp):
        return K.PARSE_TS + _TS_UNITS[tp.unit] + (K.PARSE_TS_ZONED if tp.tz is not None else 0)
    raise NotImplementedError(f"cast of a string to {tp} has no device implementation")


class StringParseError(ValueError):
    """A string a valid row refers to does not parse as the cast's target type (worded as Arrow words it)."""


def parse_error(entry: Any, tp: pa.DataType) -> StringParseError:
    return StringParseError(f"Failed to parse string: '{entry}' as a scalar of type {tp}")


class ParseResult:
    """A dictionary parsed to one type: ``values`` (int64 per entry, the 8-byte words ``FB_X_LOOKUP`` reads),
    ``valid`` (uint8, 0 for a NULL entry or one that does not parse; None: every entry parsed) and ``bad`` (int64
    device tensor of the entries that do not parse, None if there is none)."""

    def __init__(self, values: torch.Tensor, valid: Optional[torch.Tensor], bad: Optional[torch.Tensor]):
        self.values, self.valid, self.bad = values, valid, bad


def _parse(d: pa.Array, device: torch.device, tp: pa.DataType) -> ParseResult:
    global parses, parse_fallbacks
    target = parse_target(tp)
    parses += 1
    dd = device_dictionary(d, device)
    values, valid, status, first_bad = K.string_parse(dd.offsets, dd.data, dd.valid, target)
    bad = None
    if first_bad is not None:
        undecided = torch.nonzero(status == K.PARSE_UNDECIDED).squeeze(1).cpu().tolist()
        if undecided:
            import pyarrow.compute as pc

            parse_fallbacks += len(undecided)
            for i in undecided:  # a float of more than 19 significant digits: pyarrow rounds it
                try:
                    v = pc.cast(d[i:i + 1], tp, safe=False)
                except (pa.ArrowInvalid, pa.ArrowNotImplementedError):
                    status[i] = K.PARSE_INVALID
                    continue
                word = v.cast(pa.float64()).to_numpy(zero_copy_only=False).view(np.int64)[0]
                values[i] = int(word)
                valid[i] = 1
                status[i] = K.PARSE_OK
        idx = torch.nonzero(status == K.PARSE_INVALID).squeeze(1)
        bad = idx if int(idx.shape[0]) > 0 else None
    if dd.valid is None and bad is None:
        valid = None
    return ParseResult(values, valid, bad)


def parse_table(d: pa.Array, device: torch.device, tp: pa.DataType) -> ParseResult:
    """Every entry of dictionary ``d`` cast to ``tp`` on ``device``: parsed on first use, then cached on ``d``, so
    a repeated call launches nothing and reads nothing back."""
    per = _slot(_DERIVED, d)
    key = (("PARSE", tp), device)
    if key not in per:
        per[key] = _parse(d, device, tp)
    return per[key]


def check_referenced(r: ParseResult, d: pa.Array, tp: pa.DataType, codes: torch.Tensor,
                     code_valid: Optional[torch.Tensor], remap: Optional[torch.Tensor] = None,
                     remap_valid: Optional[torch.Tensor] = None, null_code: Optional[int] = None) -> None:
    """Raise the parse error of the first row that refers to an entry of ``d`` that does not parse.  ``codes`` /
    ``code_valid``: the rows' codes; with ``remap`` they are codes of a source dictionary whose entry ``e`` is entry
    ``remap[e]`` of ``d`` (``remap_valid``: 0 where it is NULL), and a NULL row is entry ``null_code`` (None: NULL).
    Costs nothing when every entry parsed."""
    if r.bad is None:
        return
    dev = codes.device
    bad = torch.zeros(len(d), dtype=torch.bool, device=dev)
    bad[r.bad] = True
    if remap is not None:
        src = bad[remap.clamp(0, max(len(d) - 1, 0))]
        if remap_valid is not None:
            src &= remap_valid.bool()
        src_of = remap
    else:
        src, src_of = bad, None
    c = codes.long()
    inside = (c >= 0) & (c < int(src.shape[0]))
    hit = src[c.clamp(0, max(int(src.shape[0]) - 1, 0))] & inside
    if code_valid is not None:
        hit &= code_valid.bool()
        if null_code is not None and bool(bad[null_code].item()):
            hit |= ~code_valid.bool()
    rows = torch.nonzero(hit)
    if int(rows.shape[0]) == 0:
        return
    row = int(rows[0, 0].item())
    if code_valid is not None and not bool(code_valid[row].item()):
        entry = null_code
    else:
        entry = int(c[row].item())
        if src_of is not None:
            entry = int(src_of[entry].item())
    raise parse_error(d[entry].as_py(), tp)


# ---- casts to strings (K14) ---------------------------------------------------------------------------
formats = 0  # columns whose distinct values were formatted to a dictionary so far
_DAY_MS = 86_400_000
_DAY_RANGE = (-12_687_428, 11_248_737)  # the days Arrow writes as a date (years -32767 .. 32767), fb_format.cuh


def format_kind(tp: pa.DataType) -> int:
    """The ``fb_value_format`` kind of a cast from ``tp`` to string; NotImplementedError for a type the device does
    not format (decimal, time, duration, nested, a timestamp in a time zone other than UTC ...)."""
    if pa.types.is_boolean(tp):
        return K.FMT_BOOL
    if pa.types.is_integer(tp):
        return K.FMT_U64 if tp == pa.uint64() else K.FMT_I64
    if pa.types.is_floating(tp):
        return K.FMT_F64
    if pa.types.is_date32(tp) or pa.types.is_date64(tp):
        return K.FMT_DATE32 if pa.types.is_date32(tp) else K.FMT_DATE64
    if pa.types.is_timestamp(tp):
        if tp.tz is not None and tp.tz.upper() != "UTC":
            raise NotImplementedError(f"cast of a timestamp in time zone {tp.tz} to string (only UTC; there is no "
                                      f"time-zone database on the device)")
        return K.FMT_TS + _TS_UNITS[tp.unit]
    raise NotImplementedError(f"cast of {tp} to string has no device implementation")


def _format_keys(values: torch.Tensor, tp: pa.DataType) -> torch.Tensor:
    """The int64 word whose text is the value's: a float64's bits with every NaN one pattern (-0.0 stays apart from
    0.0), a bool as 0 / 1, a date64 in range truncated to its day (the day Arrow writes), the value otherwise."""
    if values.dtype.is_floating_point:
        v = values.to(torch.float64)
        return torch.where(torch.isnan(v), torch.full_like(v, float("nan")), v).view(torch.int64)
    k = values.to(torch.int64)
    if pa.types.is_boolean(tp):
        return (k != 0).to(torch.int64)
    if pa.types.is_date64(tp):
        floor_day = torch.div(k, _DAY_MS, rounding_mode="floor")
        inside = (floor_day >= _DAY_RANGE[0]) & (floor_day <= _DAY_RANGE[1])
        return torch.where(inside, torch.div(k, _DAY_MS, rounding_mode="trunc") * _DAY_MS, k)
    return k


def format_values(values: torch.Tensor, valid: Optional[torch.Tensor], tp: pa.DataType, device: torch.device
                  ) -> Tuple[torch.Tensor, Optional[torch.Tensor], pa.Array]:
    """``CAST(x AS STRING)`` of a column of arrow type ``tp`` (``values``: its storage, or the 64-bit value K8
    computed for it): (int32 codes, the validity, a ``pa.string()`` dictionary of distinct entries).  The distinct
    values are found on the device over 8-byte keys the text is a function of (``_format_keys``), formatted there
    (K14) and copied to the host once; the dictionary's device copy is registered, so string functions of the result
    upload nothing.  A timestamp column has the unit's fraction digits on every row iff a valid value has a fraction
    of a second."""
    global formats
    kind = format_kind(tp)
    n = int(values.shape[0])
    if n == 0:
        return torch.empty(0, dtype=torch.int32, device=device), valid, pa.array([], type=pa.string())
    keys = _format_keys(values, tp)
    if valid is not None:
        keys = torch.where(valid.bool(), keys, torch.zeros_like(keys))
    uniq, inv = torch.unique(keys, return_inverse=True)
    if kind >= K.FMT_TS and (kind & 7) != K.TU_S:
        per = {K.TU_MS: 1000, K.TU_US: 1_000_000, K.TU_NS: 1_000_000_000}[kind & 7]
        if bool((torch.remainder(uniq, per) != 0).any().item()):  # a NULL row's key is 0: a whole second
            kind |= K.FMT_TS_FRAC
    formats += 1
    offsets, data = K.value_format(uniq, None, kind)
    total = int(offsets[-1].item())
    if total > (1 << 31) - 1:
        raise NotImplementedError(f"a string result of {total} bytes; a pa.string() dictionary holds 2^31 - 1")
    k = int(uniq.shape[0])
    host_offsets = offsets.cpu().numpy().astype(np.int32)
    host_data = data[:total].cpu().numpy()
    d = pa.Array.from_buffers(pa.string(), k, [None, pa.py_buffer(host_offsets), pa.py_buffer(host_data)])
    _slot(_CACHE, d)[device] = DeviceDictionary(offsets, data, None)
    return inv.to(torch.int32).contiguous(), valid, d
