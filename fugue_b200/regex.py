"""Regular expressions of an RE2 subset, compiled on the host for the device (K15, ``csrc/fb_regex.cu``).

``REGEXP_MATCHES`` / ``REGEXP_FULL_MATCH`` / ``REGEXP_EXTRACT`` / ``REGEXP_REPLACE`` follow RE2 as pyarrow runs it:
UTF-8 code points, ``.`` not matching ``\\n``, ASCII-only ``\\d \\w \\s`` (``\\s`` is ``[\\t\\n\\f\\r ]``), ``^`` / ``$``
only at the start / end of the text, leftmost-first alternation and lazy quantifiers.

A pattern is first checked by RE2 itself (pyarrow on a one-NULL array): what RE2 rejects is a ``ValueError`` with
RE2's message.  The parser below then reads the subset the device runs - literals and escaped metacharacters,
``\\t \\n \\r \\f \\v \\a \\xHH \\x{H...}``, ``.``, classes with ranges and ``\\d \\D \\w \\W \\s \\S``, ``(...)``,
``(?:...)``, ``|``, ``* + ? {n} {n,} {n,m}`` greedy or lazy, ``^ $ \\A \\z`` - and raises ``NotImplementedError``
naming anything else RE2 accepts (flags, word boundaries, Unicode and POSIX classes, ``\\Q...\\E``, ``\\C``,
named groups, octal escapes), so the device never answers for a pattern it does not understand.

The program is a position automaton: every instruction that consumes one code point is a position (at most
``REGEX_MAX_STATES`` after counted repetition expands).  For each point a match can be at - after a position, or
where a match starts - the closure lists the positions the empty-width part of the program reaches, in RE2's
leftmost-first priority order (a depth-first walk that visits each instruction once), with the capture slots set
on the way.  Assertions are decided while the closure is built, so each closure has an "at the end of the text"
variant and a start closure also an "at byte 0" one.  ``fb_regex_program`` carries the closures (as bit sets for
the Thompson machine of REGEXP_MATCHES, as ordered lists for the Pike VM of EXTRACT / REPLACE), a per-ASCII-byte
mask of the positions that accept it and a range table for the other code points.
"""
import functools
import re
from typing import Any, List, Optional, Sequence, Tuple

import pyarrow as pa
import pyarrow.compute as pc

from . import _lib

MAX_CP = 0x10FFFF
MAX_STATES = _lib.REGEX_MAX_STATES
MAX_SLOTS = _lib.REGEX_MAX_SLOTS
MATCH, EXTRACT, REPLACE, REPLACE_ALL = range(4)  # fb_regex_op
GROUP = 256  # FB_REGEX_GROUP
_START, _START_AT0 = MAX_STATES, MAX_STATES + 1  # closure rows of a match start (away from byte 0 / at it)

Ranges = Tuple[Tuple[int, int], ...]
_DIGIT: Ranges = ((48, 57),)
_WORD: Ranges = ((48, 57), (65, 90), (95, 95), (97, 122))
_SPACE: Ranges = ((9, 10), (12, 13), (32, 32))
_DOT: Ranges = ((0, 9), (11, MAX_CP))
_ESCAPED = {"t": 9, "n": 10, "r": 13, "f": 12, "v": 11, "a": 7}


def _norm(rs: Sequence[Tuple[int, int]]) -> Ranges:
    out: List[List[int]] = []
    for lo, hi in sorted(rs):
        if out and lo <= out[-1][1] + 1:
            out[-1][1] = max(out[-1][1], hi)
        else:
            out.append([lo, hi])
    return tuple((a, b) for a, b in out)


def _negate(rs: Ranges) -> Ranges:
    out, lo = [], 0
    for a, b in _norm(rs):
        if a > lo:
            out.append((lo, a - 1))
        lo = b + 1
    if lo <= MAX_CP:
        out.append((lo, MAX_CP))
    return tuple(out)


_CLASSES = {"d": _DIGIT, "D": _negate(_DIGIT), "w": _WORD, "W": _negate(_WORD), "s": _SPACE, "S": _negate(_SPACE)}


def _check_re2(pattern: str, rewrite: Optional[str] = None) -> None:
    """ValueError with RE2's message for a pattern (or a rewrite of it) that RE2 rejects."""
    arr = pa.array([None], type=pa.string())
    try:
        if rewrite is None:
            pc.match_substring_regex(arr, pattern=pattern)
        else:
            pc.replace_substring_regex(arr, pattern=pattern, replacement=rewrite)
    except (pa.ArrowInvalid, pa.ArrowNotImplementedError) as ex:
        raise ValueError(f"{ex} (pattern {pattern!r}" + ("" if rewrite is None else f", rewrite {rewrite!r}") + ")") \
            from None


class _Parser:
    """Recursive descent over a pattern RE2 accepted.  Nodes: ("set", ranges), ("cat", items), ("alt", items),
    ("rep", node, min, max or None, greedy), ("cap", group, node), ("bol",), ("eol",)."""

    def __init__(self, pattern: str):
        self.p, self.i, self.groups = pattern, 0, 0

    def unsupported(self, what: str) -> NotImplementedError:
        return NotImplementedError(f"regular expression {self.p!r}: {what} is not supported on the device")

    def peek(self) -> Optional[str]:
        return self.p[self.i] if self.i < len(self.p) else None

    def alt(self) -> Any:
        items = [self.cat()]
        while self.peek() == "|":
            self.i += 1
            items.append(self.cat())
        return items[0] if len(items) == 1 else ("alt", items)

    def cat(self) -> Any:
        items = []
        while self.peek() not in (None, "|", ")"):
            x = self.atom()
            while True:
                rep = self.repeat()
                if rep is None:
                    break
                greedy = self.peek() != "?"
                if not greedy:
                    self.i += 1
                x = ("rep", x, rep[0], rep[1], greedy)
            items.append(x)
        return ("cat", items)

    def repeat(self) -> Optional[Tuple[int, Optional[int]]]:
        c = self.peek()
        if c in ("*", "+", "?"):
            self.i += 1
            return {"*": (0, None), "+": (1, None), "?": (0, 1)}[c]
        m = re.match(r"\{(\d+)(,(\d*))?\}", self.p[self.i:]) if c == "{" else None
        if m is None:  # RE2 reads a '{' that does not start {n}, {n,} or {n,m} as a literal
            return None
        self.i += m.end()
        lo = int(m.group(1))
        return lo, (lo if m.group(2) is None else (int(m.group(3)) if m.group(3) else None))

    def atom(self) -> Any:
        c = self.p[self.i]
        self.i += 1
        if c == "(":
            if self.p.startswith("?:", self.i):
                self.i += 2
                x = self.alt()
            elif self.p.startswith("?P<", self.i) or self.p.startswith("?<", self.i):
                raise self.unsupported("a named group")
            elif self.peek() == "?":
                raise self.unsupported("a flag group such as (?i)")
            else:
                self.groups += 1
                k = self.groups
                x = ("cap", k, self.alt())
            self.i += 1  # ')'
            return x
        if c == "[":
            return ("set", self.cls())
        if c == ".":
            return ("set", _DOT)
        if c == "^":
            return ("bol",)
        if c == "$":
            return ("eol",)
        if c == "\\":
            d = self.p[self.i]
            if d == "A":
                self.i += 1
                return ("bol",)
            if d == "z":
                self.i += 1
                return ("eol",)
            if d in ("b", "B"):
                raise self.unsupported("a word boundary \\b / \\B")
            r = self.escape()
            return ("set", r if isinstance(r, tuple) else ((r, r),))
        return ("set", ((ord(c), ord(c)),))

    def escape(self) -> Any:
        """After a backslash: a class (ranges) or one code point."""
        d = self.p[self.i]
        self.i += 1
        if d in _CLASSES:
            return _CLASSES[d]
        if d in ("p", "P"):
            raise self.unsupported("a Unicode class \\p / \\P")
        if d in ("Q", "E"):
            raise self.unsupported("a quoted run \\Q...\\E")
        if d == "C":
            raise self.unsupported("\\C (any byte)")
        if d in _ESCAPED:
            return _ESCAPED[d]
        if d == "x":
            if self.peek() == "{":
                j = self.p.index("}", self.i)
                v = int(self.p[self.i + 1:j], 16)
                self.i = j + 1
                return v
            v = int(self.p[self.i:self.i + 2], 16)
            self.i += 2
            return v
        if d.isascii() and not d.isalnum():
            return ord(d)
        raise self.unsupported(f"the escape \\{d}")

    def cls(self) -> Ranges:
        neg = self.peek() == "^"
        if neg:
            self.i += 1
        rs: List[Tuple[int, int]] = []
        first = True
        while True:
            if self.peek() == "]" and not first:
                self.i += 1
                break
            first = False
            if re.match(r"\[:\^?[A-Za-z]+:\]", self.p[self.i:]):
                raise self.unsupported("a POSIX class such as [[:alpha:]]")
            lo = self.cls_atom()
            if isinstance(lo, tuple):
                rs.extend(lo)
                continue
            if self.peek() == "-" and self.i + 1 < len(self.p) and self.p[self.i + 1] != "]":
                self.i += 1
                rs.append((lo, self.cls_atom()))
            else:
                rs.append((lo, lo))
        return _negate(_norm(rs)) if neg else _norm(rs)

    def cls_atom(self) -> Any:
        c = self.p[self.i]
        self.i += 1
        return self.escape() if c == "\\" else ord(c)


def _nullable(x: Any) -> bool:
    k = x[0]
    if k == "set":
        return False
    if k in ("bol", "eol"):
        return True
    if k == "cat":
        return all(_nullable(y) for y in x[1])
    if k == "alt":
        return any(_nullable(y) for y in x[1])
    if k == "rep":
        return x[2] == 0 or _nullable(x[1])
    return _nullable(x[2])


def _positions(x: Any) -> int:
    """The positions of the program of x, with counted repetition expanded."""
    k = x[0]
    if k == "set":
        return 1
    if k in ("bol", "eol"):
        return 0
    if k in ("cat", "alt"):
        return sum(_positions(y) for y in x[1])
    if k == "rep":
        return _positions(x[1]) * (x[3] if x[3] is not None else max(x[2], 1))
    return _positions(x[2])


class Regex:
    """A parsed pattern: ``ast`` and ``groups`` (the number of capturing groups)."""

    def __init__(self, pattern: str, ast: Any, groups: int):
        self.pattern, self.ast, self.groups = pattern, ast, groups


@functools.lru_cache(maxsize=256)
def parse(pattern: str) -> Regex:
    """The pattern checked by RE2 (ValueError), read as the device subset (NotImplementedError otherwise) and
    held to the device limits (NotImplementedError naming the limit)."""
    if not isinstance(pattern, str):
        raise NotImplementedError(f"a regular expression must be a string literal, got {pattern!r}")
    _check_re2(pattern)
    p = _Parser(pattern)
    ast = p.alt()
    if p.i != len(pattern):  # RE2 accepted it, so this is a construct the parser does not know
        raise p.unsupported(f"the text at {p.i}")

    def walk(x: Any) -> None:
        if x[0] == "rep":
            if x[3] is None and _nullable(x[1]):
                raise p.unsupported("an unbounded repetition of an expression that can match the empty string")
            walk(x[1])
        elif x[0] in ("cat", "alt"):
            for y in x[1]:
                walk(y)
        elif x[0] == "cap":
            walk(x[2])

    walk(ast)
    n = _positions(ast)
    if n > MAX_STATES:
        raise NotImplementedError(f"regular expression {pattern!r} has {n} positions after counted repetition "
                                  f"expands; the device takes at most {MAX_STATES}")
    return Regex(pattern, ast, p.groups)


class _Program:
    """Thompson instructions: [op, arg, out, out2] with op char (arg: ranges) / split / save (arg: slot) /
    assert (arg: 'bol' / 'eol') / match."""

    def __init__(self) -> None:
        self.ins: List[List[Any]] = []

    def new(self, op: str, arg: Any = None, out: int = -1, out2: int = -1) -> int:
        self.ins.append([op, arg, out, out2])
        return len(self.ins) - 1

    def compile(self, x: Any, k: int) -> int:
        """The entry of x's instructions, which continue at k."""
        kind = x[0]
        if kind == "set":
            return self.new("char", x[1], k)
        if kind in ("bol", "eol"):
            return self.new("assert", kind, k)
        if kind == "cat":
            for y in reversed(x[1]):
                k = self.compile(y, k)
            return k
        if kind == "alt":
            entries = [self.compile(y, k) for y in x[1]]
            e = entries[-1]
            for f in reversed(entries[:-1]):
                e = self.new("split", None, f, e)
            return e
        if kind == "cap":
            end = self.new("save", 2 * x[1] + 1, k)
            return self.new("save", 2 * x[1], self.compile(x[2], end))
        _, y, lo, hi, greedy = x
        if hi is None:
            loop = self.new("split")
            body = self.compile(y, loop)
            self.ins[loop][2:] = [body, k] if greedy else [k, body]
            t = loop
            if lo > 0:  # x{n,}: x{n - 1} then x+
                t = body
                lo -= 1
        else:
            t = k
            for _ in range(hi - lo):  # nested optionals, as RE2 expands x{n,m}: (x(x)?)?
                body = self.compile(y, t)
                t = self.new("split", None, body, k) if greedy else self.new("split", None, k, body)
        for _ in range(lo):
            t = self.compile(y, t)
        return t

    def closure(self, pc: int, at_start: bool, at_end: bool, pos_of: dict) -> List[Tuple[int, int]]:
        """(target, slots set) in priority order: targets are positions or MAX_STATES (the match)."""
        out: List[Tuple[int, int]] = []
        seen = set()
        stack = [(pc, 0)]
        while stack:
            pc, saves = stack.pop()
            if pc in seen:
                continue
            seen.add(pc)
            op, arg, o1, o2 = self.ins[pc]
            if op == "char":
                out.append((pos_of[pc], saves))
            elif op == "match":
                out.append((MAX_STATES, saves))
            elif op == "split":
                stack.append((o2, saves))
                stack.append((o1, saves))
            elif op == "save":
                stack.append((o1, saves | (1 << arg)))
            elif (arg == "bol" and at_start) or (arg == "eol" and at_end):
                stack.append((o1, saves))
        return out


def _build(rx: Regex, full: bool, op: int, slots: Sequence[int], group_pair: int = 0,
           rewrite: Sequence[int] = ()) -> "_lib.RegexProgram":
    ast = ("cat", [("bol",), rx.ast, ("eol",)]) if full else rx.ast
    P = _Program()
    start = P.new("save", 0, P.new("save", 1, P.new("match")))
    P.ins[start][2] = P.compile(ast, P.ins[start][2])
    chars = [pc for pc, ins in enumerate(P.ins) if ins[0] == "char"]
    pos_of = {pc: i for i, pc in enumerate(chars)}
    local = {s: i for i, s in enumerate(slots)}

    prog = _lib.RegexProgram()
    prog.npos, prog.nslots, prog.op, prog.group_pair = len(chars), len(slots), op, group_pair
    for p, pc in enumerate(chars):
        for lo, hi in P.ins[pc][1]:
            for b in range(lo, min(hi, 127) + 1):
                prog.ascii[b] |= 1 << p
    cuts = sorted({128} | {c for pc in chars for lo, hi in P.ins[pc][1] for c in (lo, hi + 1) if 128 < c <= MAX_CP})
    los: List[int] = []
    masks: List[int] = []
    for c in cuts:
        m = 0
        for p, pc in enumerate(chars):
            if any(lo <= c <= hi for lo, hi in P.ins[pc][1]):
                m |= 1 << p
        if not masks or masks[-1] != m:
            los.append(c)
            masks.append(m)
    if len(los) > _lib.REGEX_MAX_RANGES:
        raise NotImplementedError(f"regular expression {rx.pattern!r} needs {len(los)} code-point ranges; the device "
                                  f"takes at most {_lib.REGEX_MAX_RANGES}")
    prog.nranges = len(los)
    for r, (lo, m) in enumerate(zip(los, masks)):
        prog.range_lo[r], prog.range_mask[r] = lo, m

    rows = [(p, P.ins[pc][2], False) for p, pc in enumerate(chars)] + [(_START, start, False),
                                                                       (_START_AT0, start, True)]
    lists = {}
    for row, pc, at0 in rows:
        for end in (0, 1):
            lists[2 * row + end] = P.closure(pc, at0, bool(end), pos_of)
    e = 0
    for c in range(_lib.REGEX_MAX_CLOSURES):
        prog.cl_off[c] = e
        for target, saves in lists.get(c, ()):
            prog.ent_target[e] = target
            prog.ent_save[e] = sum(1 << i for s, i in local.items() if (saves >> s) & 1)
            if target == MAX_STATES:
                prog.cl_accept[c] = 1
            else:
                prog.cl_mask[c] |= 1 << target
            e += 1
    prog.cl_off[_lib.REGEX_MAX_CLOSURES] = e
    prog.restart = int(bool(lists[2 * _START] or lists[2 * _START + 1]))
    if len(rewrite) > _lib.REGEX_MAX_REWRITE:
        raise NotImplementedError(f"a rewrite of {len(rewrite)} tokens; the device takes {_lib.REGEX_MAX_REWRITE}")
    prog.nrewrite = len(rewrite)
    for t, tok in enumerate(rewrite):
        prog.rewrite[t] = tok
    return prog


@functools.lru_cache(maxsize=256)
def match_program(pattern: str, full: bool) -> "_lib.RegexProgram":
    """REGEXP_MATCHES (``full``: REGEXP_FULL_MATCH, the pattern anchored as ``\\A(?:p)\\z``)."""
    return _build(parse(pattern), full, MATCH, ())


def check_group(pattern: str, group: int) -> None:
    rx = parse(pattern)
    if isinstance(group, bool) or not isinstance(group, int) or not 0 <= group <= rx.groups:
        raise ValueError(f"REGEXP_EXTRACT: group {group!r} of {pattern!r}, which has {rx.groups} group(s)")


@functools.lru_cache(maxsize=256)
def extract_program(pattern: str, group: int) -> "_lib.RegexProgram":
    """REGEXP_EXTRACT: the text of group ``group`` (0: the whole match) of the leftmost match."""
    check_group(pattern, group)
    return _build(parse(pattern), False, EXTRACT, (2 * group, 2 * group + 1))


def rewrite_tokens(pattern: str, rewrite: str) -> Tuple[List[int], List[int]]:
    """A REGEXP_REPLACE rewrite as (tokens, the groups it names besides 0): UTF-8 bytes, and ``GROUP + k`` for
    ``\\k``.  ``\\\\`` is a backslash; RE2's check of the rewrite comes first (ValueError)."""
    rx = parse(pattern)
    if not isinstance(rewrite, str):
        raise NotImplementedError(f"REGEXP_REPLACE needs a string literal rewrite, got {rewrite!r}")
    _check_re2(pattern, rewrite)
    groups: List[int] = []
    toks: List[int] = []
    i = 0
    while i < len(rewrite):
        c = rewrite[i]
        if c == "\\" and i + 1 < len(rewrite) and rewrite[i + 1].isdigit():
            k = int(rewrite[i + 1])
            if k > rx.groups:
                raise ValueError(f"REGEXP_REPLACE: the rewrite {rewrite!r} names group {k}; {pattern!r} has "
                                 f"{rx.groups}")
            if k > 0 and k not in groups:
                groups.append(k)
            toks.append(GROUP + (0 if k == 0 else 1 + groups.index(k)))
            i += 2
            continue
        if c == "\\" and i + 1 < len(rewrite) and rewrite[i + 1] == "\\":
            toks.append(ord("\\"))
            i += 2
            continue
        if c == "\\":
            raise ValueError(f"REGEXP_REPLACE: invalid rewrite {rewrite!r}")
        toks.extend(c.encode("utf-8"))
        i += 1
    if 2 * (1 + len(groups)) > MAX_SLOTS:
        raise NotImplementedError(f"REGEXP_REPLACE: the rewrite {rewrite!r} names {len(groups)} groups besides \\0; "
                                  f"the device tracks at most {MAX_SLOTS // 2 - 1}")
    return toks, groups


@functools.lru_cache(maxsize=256)
def replace_program(pattern: str, rewrite: str, global_: bool) -> "_lib.RegexProgram":
    """REGEXP_REPLACE: the first match (``global_``: every match) replaced by ``rewrite``."""
    toks, groups = rewrite_tokens(pattern, rewrite)
    slots = [0, 1] + [s for k in groups for s in (2 * k, 2 * k + 1)]
    return _build(parse(pattern), False, REPLACE_ALL if global_ else REPLACE, slots, 0, toks)


def replace_options(options: Optional[str]) -> bool:
    """Whether REGEXP_REPLACE's options ask for every match: None / '' (the first) or 'g'."""
    if options in (None, ""):
        return False
    if options == "g":
        return True
    raise NotImplementedError(f"REGEXP_REPLACE options {options!r}: only 'g' is supported")
