"""K15 regular expressions without a GPU: the compiled programs run through the kernels' own per-entry code on the
CPU (``fb_debug_regex_host``) against pyarrow's RE2 on a seeded corpus, the semantic cases RE2 and Python differ on,
the builders and the SQL parser, every error rule and limit, and compiled K8 programs on the machine model."""
import random

import numpy as np
import pandas as pd
import pyarrow as pa
import pytest
import torch

import _regex_corpus as RC
from fugue_b200 import kernels as K
from fugue_b200 import regex as R
from fugue_b200 import strings as ST
from fugue_b200.column import col, functions as ff, null, to_sql
from fugue_b200.sql import _parse_select

N_PATTERNS = 400


def parse_expr(text):
    return _parse_select("*", "t WHERE " + text, "SELECT * FROM t WHERE " + text).where


def _layout(strs):
    arr = pa.array(strs, type=pa.string())
    b = arr.buffers()
    offs = np.frombuffer(b[1], dtype=np.int32, count=len(arr) + 1).astype(np.int64)
    data = np.frombuffer(b[2], dtype=np.uint8).copy() if b[2] is not None and offs[-1] > 0 else np.zeros(1, np.uint8)
    valid = None if arr.null_count == 0 else arr.is_valid().to_numpy(zero_copy_only=False).astype(np.uint8)
    return offs, data, valid


def run(strs, prog):
    """The kernels' per-entry code over ``strs`` on the CPU: bools for a match program, strings otherwise."""
    offs, data, valid = _layout(strs)
    out, ok, res = K.regex_host(offs, data, valid, prog)
    if res is None:
        return [bool(x) if v else None for x, v in zip(out, ok)]
    o, buf = res
    return [bytes(buf[o[i]:o[i + 1]]).decode("utf-8") if ok[i] else None for i in range(len(strs))]


def _corpus():
    rng = random.Random(15)
    pats = []
    while len(pats) < N_PATTERNS:
        p = RC.random_pattern(rng)
        try:
            R.parse(p)
        except (NotImplementedError, ValueError):
            continue
        pats.append(p)
    return pats, RC.random_strings(rng, 60) + [None]


PATTERNS, STRINGS = _corpus()


def test_corpus_matches_and_full_matches_follow_re2():
    for p in PATTERNS:
        assert run(STRINGS, R.match_program(p, False)) == RC.matches(STRINGS, p), p
        assert run(STRINGS, R.match_program(p, True)) == RC.matches(STRINGS, p, full=True), p


def test_corpus_extract_follows_re2():
    for p in PATTERNS:
        for g in range(min(RC.groups_of(p), 8) + 1):
            assert run(STRINGS, R.extract_program(p, g)) == RC.extract(STRINGS, p, g), (p, g)


def test_corpus_replace_follows_re2():
    for p in PATTERNS:
        rewrites = ["<\\0>", "#"] + (["[\\1|\\\\]"] if RC.groups_of(p) >= 1 else [])
        for rw in rewrites:
            for glob in (False, True):
                assert run(STRINGS, R.replace_program(p, rw, glob)) == RC.replace(STRINGS, p, rw, glob), (p, rw, glob)


@pytest.mark.parametrize("case", RC.SEMANTIC_CASES, ids=lambda c: f"{c[0]}-{c[2]}")
def test_semantic_cases(case):
    fn, s, p, extra, want = case
    ref = {"matches": lambda: RC.matches([s], p)[0], "extract": lambda: RC.extract([s], p, extra)[0],
           "replace_all": lambda: RC.replace([s], p, extra, True)[0]}[fn]()
    assert ref == want  # pyarrow itself
    prog = {"matches": lambda: R.match_program(p, False), "extract": lambda: R.extract_program(p, extra),
            "replace_all": lambda: R.replace_program(p, extra, True)}[fn]()
    assert run([s], prog)[0] == want


def test_long_entry_and_many_matches():
    s = ("ab1 " * 20_000) + "é"
    assert run([s], R.replace_program("\\d", "<\\0>", True)) == RC.replace([s], "\\d", "<\\0>", True)
    assert run([s], R.extract_program("(\\d) é", 1)) == ["1"]
    assert run([s], R.match_program("é$", False)) == [True]


# ---- builders and SQL -------------------------------------------------------------------------------------------
S = col("s")
BUILT = [ff.regexp_matches(S, r"^\d+$"), ff.regexp_full_match(S, "a|b'c"), ff.regexp_extract(S, "@(.*)", 1),
         ff.regexp_extract(S, r"\w+"), ff.regexp_replace(S, r"(a)\.", r"\1-\\", "g"), ff.regexp_replace(S, "x", "y"),
         S.rlike("[^a]"), ~S.rlike("a"), ff.upper(ff.regexp_extract(ff.trim(S), "b+")),
         ff.regexp_matches(ff.regexp_replace(S, "a", "b"), "b") & (col("v") > 0), ff.regexp_matches(S, null())]


@pytest.mark.parametrize("e", BUILT, ids=str)
def test_to_sql_parse_fixed_point(e):
    text = to_sql(e)
    assert parse_expr(text).fingerprint() == e.fingerprint(), text


def test_sql_spellings():
    assert parse_expr(r"REGEXP_LIKE(s, '^\d')").fingerprint() == ff.regexp_matches(S, r"^\d").fingerprint()
    assert parse_expr(r"s RLIKE '\d'").fingerprint() == S.rlike(r"\d").fingerprint()
    assert parse_expr(r"s NOT RLIKE '\d'").fingerprint() == (~S.rlike(r"\d")).fingerprint()
    assert parse_expr("REGEXP_EXTRACT(s, 'a', 0)").fingerprint() == ff.regexp_extract(S, "a").fingerprint()
    assert parse_expr("REGEXP_MATCHES(s, 'it''s')").args[1].value == "it's"
    st = _parse_select("s rlike", "t", "SELECT s rlike FROM t")  # an implicit alias named rlike
    assert [c.output_name for c in st.columns] == ["rlike"]


def test_types():
    from fugue_b200.schema import Schema

    sch = Schema("s:str,v:long")
    assert ff.regexp_matches(S, "a").infer_type(sch) == pa.bool_()
    assert ff.regexp_full_match(S, "a").infer_type(sch) == pa.bool_()
    assert ff.regexp_extract(S, "a").infer_type(sch) == pa.string()
    assert ff.regexp_replace(S, "a", "b").infer_type(sch) == pa.string()


# ---- errors -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [r"(a)\1", "(?=a)", "a++", "a{1001}", "a**", "(", "[a"])
def test_re2_rejects_is_value_error(p):
    with pytest.raises(ValueError):
        ff.regexp_matches(S, p)


@pytest.mark.parametrize("p,what", [("(?i)a", "flag"), (r"\bx", "word boundary"), (r"\pL", "Unicode"),
                                    (r"\p{Greek}", "Unicode"), ("[[:alpha:]]", "POSIX"), (r"\Q.\E", "quoted"),
                                    (r"\C", "any byte"), ("(?P<n>a)", "named"), ("(a*)*", "empty"),
                                    (r"\101", "escape")])
def test_outside_the_subset_is_not_implemented(p, what):
    with pytest.raises(NotImplementedError, match=what):
        ff.regexp_matches(S, p)


def test_limits():
    ff.regexp_matches(S, "a{64}")
    with pytest.raises(NotImplementedError, match="positions"):
        ff.regexp_matches(S, "a{65}")
    with pytest.raises(NotImplementedError, match="positions"):
        ff.regexp_matches(S, "(ab){1,40}")
    with pytest.raises(NotImplementedError, match="groups"):
        ff.regexp_replace(S, "(a)(b)(c)(d)", r"\1\2\3\4")
    ff.regexp_replace(S, "(a)(b)(c)(d)", r"\1\2\3\0")


def test_argument_errors():
    with pytest.raises(NotImplementedError):
        ff.regexp_matches(S, col("p"))
    with pytest.raises(NotImplementedError):
        ff.regexp_replace(S, "a", col("r"))
    with pytest.raises(NotImplementedError):
        ff.regexp_extract(S, "a", col("g"))
    with pytest.raises(ValueError):
        ff.regexp_extract(S, "(a)", 2)
    with pytest.raises(ValueError):
        ff.regexp_replace(S, "(a)", r"\2")
    with pytest.raises(NotImplementedError):
        ff.regexp_replace(S, "a", "b", "gi")
    with pytest.raises(ValueError):
        parse_expr("REGEXP_EXTRACT(s)")
    ff.regexp_extract(S, "a", null())
    ff.regexp_replace(S, null(), "b")


# ---- compiled K8 programs on the machine model ------------------------------------------------------------------
def test_compiled_programs_on_the_machine_model(monkeypatch):
    """The K8 programs of the bool functions (and their combination with other terms) run by the numpy machine
    model, with per-entry tables made by the kernels' host code, against pyarrow row by row."""
    import test_strings_cpu as TS

    def regex_table(d, device, pattern, full):
        vals = run(d.to_pylist(), R.match_program(pattern, full))
        return (torch.tensor([bool(v) for v in vals], dtype=torch.int64),
                None if d.null_count == 0 else torch.tensor([v is not None for v in vals], dtype=torch.uint8))

    monkeypatch.setattr(ST, "regex_table", regex_table)
    rng = np.random.default_rng(3)
    for null_entries in (False, True):
        t, pdf = TS._random_table(rng, 2000, 40, null_entries)
        rows = [None if x is pd.NA else x for x in pdf["s"].tolist()]
        v = pdf["v"].tolist()
        for p in [r"^\w", "é|中", "a.?b", r"\d*$", "^$"]:
            for full in (False, True):
                e = ff.regexp_full_match(col("s"), p) if full else ff.regexp_matches(col("s"), p)
                want = RC.matches(rows, p, full)
                _, got = TS._run_model(t, e)
                assert got == want, (p, full)
                _, got = TS._run_model(t, e & (col("v") > 0))
                assert got == [None if w is None and x > 0 else (False if x <= 0 else w) for w, x in zip(want, v)]
                _, got = TS._run_model(t, ~col("s").rlike(p) if not full else ~e)
                assert got == [None if w is None else not w for w in want]
