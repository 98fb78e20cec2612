"""Regular-expression test corpus and reference: seeded patterns from the device subset's grammar, strings over an
alphabet with multi-byte code points, newlines, vertical tabs and spaces, and the four functions as pyarrow (RE2)
computes them.  pyarrow is the authority the device follows; REGEXP_EXTRACT is restated through
``replace_substring_regex``: a lazy prefix finds the leftmost start and an extra group makes group g group g + 1."""
import random
from typing import List, Optional

import pyarrow as pa
import pyarrow.compute as pc

ALPHABET = ["a", "b", "c", "x", "1", "7", "-", ".", " ", "\n", "\v", "\t", "é", "中", "😀", "@", "_", "A"]
_LITERALS = ["a", "b", "c", "x", "1", "-", "é", "中", "😀", "@", "_", "A", "\\.", "\\-", "\\n", "\\t", "\\v",
             "\\x41", "\\x{4E2D}", "\\*"]
_CLASSES = [".", "\\d", "\\w", "\\s", "\\D", "\\W", "\\S", "[a-c]", "[^a]", "[\\d.]", "[^\\s@]", "[é-中]",
            "[^\\w\\n]", "[a\\-]", "[]a]"]

# the cases of the semantics the device must share with RE2, verbatim
SEMANTIC_CASES = [  # (function, string, pattern, extra, expected)
    ("matches", "a\vb", r"a\sb", None, False),
    ("matches", "b\n", r"b$", None, False),
    ("replace_all", "aaa", "^a", "#", "#aa"),
    ("extract", "ab", "a|ab", 0, "a"),
    ("extract", "aaa", "(a*?)(a*)", 1, ""),
    ("extract", "aaa", "(a*?)(a*)", 2, "aaa"),
    ("replace_all", "2024-01-15 x 7", "x*", "-", "-2-0-2-4---0-1---1-5- - -7-"),
    ("matches", "\n", ".", None, False),
    ("matches", "中", "^.$", None, True),
]


def random_pattern(rng: random.Random, depth: int = 0) -> str:
    """A pattern of the device subset (it may still be over a device limit)."""
    parts = []
    for _ in range(rng.randint(1, 3)):
        r = rng.random()
        if r < 0.3:
            atom = rng.choice(_LITERALS)
        elif r < 0.6:
            atom = rng.choice(_CLASSES)
        elif r < 0.75 and depth < 2:
            inner = "|".join(random_pattern(rng, depth + 1) for _ in range(rng.randint(1, 3)))
            atom = ("(" if rng.random() < 0.7 else "(?:") + inner + ")"
        elif r < 0.85:
            atom = rng.choice(["^", "$", "\\A", "\\z"])
            parts.append(atom)
            continue
        else:
            atom = rng.choice(_LITERALS) + rng.choice(_LITERALS)
        if rng.random() < 0.45:
            q = rng.choice(["*", "+", "?", "{2}", "{1,3}", "{0,2}", "{2,}"])
            atom += q + ("?" if rng.random() < 0.3 else "")
        parts.append(atom)
    return "".join(parts)


def random_strings(rng: random.Random, n: int, max_len: int = 10) -> List[str]:
    out = [""]
    while len(out) < n:
        out.append("".join(rng.choice(ALPHABET) for _ in range(rng.randint(0, max_len))))
    return out


def _arr(strs: List[Optional[str]]) -> pa.Array:
    return pa.array(strs, type=pa.string())


def matches(strs: List[Optional[str]], p: str, full: bool = False) -> List[Optional[bool]]:
    return pc.match_substring_regex(_arr(strs), pattern=f"\\A(?:{p})\\z" if full else p).to_pylist()


def replace(strs: List[Optional[str]], p: str, rewrite: str, global_: bool) -> List[Optional[str]]:
    kw = {} if global_ else {"max_replacements": 1}
    return pc.replace_substring_regex(_arr(strs), pattern=p, replacement=rewrite, **kw).to_pylist()


def extract(strs: List[Optional[str]], p: str, g: int) -> List[Optional[str]]:
    assert g <= 8
    hit = matches(strs, p)
    got = pc.replace_substring_regex(_arr(strs), pattern=f"\\A(?s:.*?)((?:{p}))(?s:.*)\\z",
                                     replacement="\\" + str(g + 1), max_replacements=1).to_pylist()
    return [None if h is None else (x if h else "") for h, x in zip(hit, got)]


def groups_of(p: str) -> int:
    from fugue_b200 import regex

    return regex.parse(p).groups
