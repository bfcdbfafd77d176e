"""CPU tests of the string predicates: the oracle (tests/string_match_oracle.py) against the reference's known answers
(tests/golden/string_match_kats.json), against brute force and against pyarrow.compute; the regex-subset mapping of
str_contains on every known-answer pattern and its refusals; the declared symbols and the header / Rust parity.
tests/test_gpu_string_match.py holds the device against this oracle."""
import json
import os
import random
import re

import numpy as np
import pytest

import string_match_oracle as so

ROOT = os.path.dirname(os.path.dirname(__file__))
KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "string_match_kats.json")))
ALPHABET = ["a", "b", "\n", "é", "€", "😀", "%", "_"]


def oracle_of(case):
    """the oracle's answer to a known-answer case, or "refused" for a regex outside the device subset"""
    import polars_b200 as plb
    col, pat = case["col"], case["pattern"]
    op = case["op"]
    if op == "like":
        return so.like(col, pat, negate=case["negate"])
    if op == "contains":
        return so.contains(col, pat)
    if op in ("starts_with", "ends_with"):
        return getattr(so, op)(col, pat)
    try:
        kind, p, flags, esc = plb.regex_to_device(pat)
    except plb.B200Error as e:
        assert e.status == 4
        return "refused"
    return mapped_oracle(col, kind, p, flags, esc)


def mapped_oracle(col, kind, p, flags, esc):
    """the oracle of the device call a regex maps to"""
    import polars_b200 as plb
    if kind == "like":
        return so.like(col, p, no_newline=bool(flags & plb.LIKE_NO_NEWLINE), escape=esc, open_start=bool(flags & plb.LIKE_OPEN_START),
                       open_end=bool(flags & plb.LIKE_OPEN_END))
    return getattr(so, kind)(col, p)


@pytest.mark.parametrize("case", KATS, ids=[f"{i}:{c['op']}:{c['src'].rsplit(':', 1)[-1]}" for i, c in enumerate(KATS)])
def test_oracle_known_answers(case):
    got = oracle_of(case)
    assert got == ("refused" if case["expected"] is None else case["expected"]), case["src"]


@pytest.mark.parametrize("case", [c for c in KATS if c["op"] == "regex" and c["expected"] is not None], ids=lambda c: c["pattern"])
def test_regex_mapping_on_known_answers(case):
    """the mapped call and the subset's own regex semantics give the reference's answer"""
    assert so.regex_search(case["col"], case["pattern"]) == case["expected"]


def rand_text(rng, max_len=6):
    return "".join(rng.choice(ALPHABET) for _ in range(rng.randrange(max_len + 1)))


def test_like_oracle_equals_brute_force():
    """the recursive matcher against Python's re over the same decoded characters (re is only a cross-check here:
    '%' -> (?:.*) and '_' -> '.', DOTALL unless no_newline, \\A ... \\Z anchors)"""
    rng = random.Random(7)
    for _ in range(3000):
        toks = [rng.choice([("lit", rng.choice(ALPHABET[:6])), ("any",), ("star",)]) for _ in range(rng.randrange(5))]
        text = rand_text(rng)
        nn, o0, o1 = rng.random() < 0.5, rng.random() < 0.3, rng.random() < 0.3
        rx = "".join(re.escape(t[1]) if t[0] == "lit" else "." if t[0] == "any" else ".*" for t in toks)
        rx = ("" if o0 else r"\A") + rx + ("" if o1 else r"\Z")
        want = re.search(rx, text, 0 if nn else re.S) is not None
        assert so.like_match(text.encode(), toks, nn, o0, o1) == want, (toks, text, nn, o0, o1)


def test_like_escape_and_utf8():
    assert so.like(["a%b", "axb", "a_b"], "a\\%b", escape="\\") == [True, False, False]
    assert so.like(["a\\b", "ab"], "a\\\\b", escape="\\") == [True, False]
    assert so.like(["é", "ab", "😀", ""], "_") == [True, False, True, False]
    assert so.like(["a\nb"], "a%b") == [True] and so.like(["a\nb"], "a%b", no_newline=True) == [False]
    assert so.like(["a\nb"], "a_b", no_newline=True) == [False]
    with pytest.raises(ValueError):
        so.like(["x"], "a\\b", escape="\\")


def test_predicate_oracles_equal_brute_force():
    rng = random.Random(3)
    for _ in range(500):
        col = [None if rng.random() < 0.1 else bytes(rng.choice(b"ab\x00\xff") for _ in range(rng.randrange(6))) for _ in range(8)]
        pat = bytes(rng.choice(b"ab\x00\xff") for _ in range(rng.randrange(4)))
        for x, c, s, e in zip(col, so.contains(col, pat), so.starts_with(col, pat), so.ends_with(col, pat)):
            if x is None:
                assert c is s is e is None
                continue
            at = [i for i in range(len(x) - len(pat) + 1) if x[i:i + len(pat)] == pat]      # every match position, by slicing
            assert c == bool(at) and s == (0 in at) and e == (len(x) - len(pat) in at)
        other = [bytes(rng.choice(b"ab\x00") for _ in range(rng.randrange(4))) for _ in range(8)]
        for op in so.CMPS:
            for x, y, r in zip(col, other, so.compare(op, col, other)):
                assert r is None if x is None else r == so.CMPS[op](x, y)
    assert so.compare("lt", [b"a", b"a\x00"], [b"a\x00", b"b"]) == [True, True]
    assert so.compare("eq", [None, b"x"], None, missing=True) == [True, False]
    assert so.compare("ne", [None, b"x"], None, missing=True) == [False, True]
    assert so.compare("eq", [None, b"x"], None) == [None, None]


def test_oracle_against_pyarrow():
    pa = pytest.importorskip("pyarrow")
    pc = pytest.importorskip("pyarrow.compute")
    rng = random.Random(11)
    for _ in range(200):
        col = [None if rng.random() < 0.1 else rand_text(rng) for _ in range(12)]
        arr = pa.array(col, pa.large_string())
        pat = rand_text(rng, 3)
        assert so.starts_with(col, pat) == pc.starts_with(arr, pattern=pat).to_pylist()
        assert so.ends_with(col, pat) == pc.ends_with(arr, pattern=pat).to_pylist()
        assert so.contains(col, pat) == pc.match_substring(arr, pattern=pat).to_pylist()
        assert so.compare("eq", col, pat) == pc.equal(arr, pa.scalar(pat, pa.large_string())).to_pylist()
        assert so.compare("lt", col, pat) == pc.less(arr, pa.scalar(pat, pa.large_string())).to_pylist()
        other = [rand_text(rng, 3) for _ in col]
        assert so.compare("le", col, other) == pc.less_equal(arr, pa.array(other, pa.large_string())).to_pylist()
        lp = "".join(rng.choice(["a", "é", "\n", "%", "_"]) for _ in range(rng.randrange(4)))
        assert so.like(col, lp) == pc.match_like(arr, pattern=lp).to_pylist(), lp


def test_numpy_oracle_equals_list_oracle():
    rng = np.random.default_rng(5)
    rows = rng.integers(0, 3, size=(400, 6), dtype=np.uint8) + ord("a")
    offs = np.arange(401, dtype=np.int64) * 6
    m = so.np_rows(rows.ravel(), offs, 6)
    col = [bytes(r) for r in rows]
    for nd in (b"", b"a", b"ab", b"abc", b"aaaaaa", b"aaaaaaa"):
        assert so.np_contains(m, nd).tolist() == so.contains(col, nd)
        assert so.np_starts_with(m, nd).tolist() == so.starts_with(col, nd)
    other = rng.integers(0, 3, size=(400, 6), dtype=np.uint8) + ord("a")
    for op in so.CMPS:
        assert so.np_compare(op, rows, other).tolist() == so.compare(op, col, [bytes(r) for r in other])


REFUSED = [r"^\S+$", "(not_valid_regex", "a+", "a?", "a|b", "[ab]", "a{2}", r"\d", r"\bword", "(?i)abc", "a*", ".+", "x$y", "a^", r"\<"]


@pytest.mark.parametrize("pattern", REFUSED)
def test_regex_subset_refusals(pattern):
    import polars_b200 as plb
    with pytest.raises(plb.B200Error) as e:
        plb.regex_to_device(pattern)
    assert e.value.status == 4


@pytest.mark.parametrize("pattern,expected", [
    ("green", ("contains", b"green", 0, None)),
    ("^PROMO", ("starts_with", b"PROMO", 0, None)),
    ("BRASS$", ("ends_with", b"BRASS", 0, None)),
    (r"\*\.\$", ("contains", b"*.$", 0, None)),
    ("special.*requests", ("like", b"special%requests", 2 | 4 | 8, "\\")),
    (".*Customer.*Complaints.*", ("like", b"%Customer%Complaints%", 2 | 4 | 8, "\\")),
    ("(?s)^a.c$", ("like", b"a_c", 0, "\\")),
    ("^abc$", ("like", b"abc", 2, "\\")),
    ("50%_off.", ("like", b"50\\%\\_off_", 2 | 4 | 8, "\\")),
])
def test_regex_subset_mapping(pattern, expected):
    import polars_b200 as plb
    assert plb.regex_to_device(pattern) == expected


def test_regex_mapping_equals_subset_semantics():
    """random subset regexes: the oracle of the mapped call equals the subset's regex meaning, Rust's `$` included"""
    import polars_b200 as plb
    rng = random.Random(13)
    texts = [None, "", "\n", "a\n", "ab\nc", "%_a", "éa", "a.b", "cab", "b\na"]
    pieces = ["a", "b", ".", ".*", r"\.", "%", "_", "é", r"\$"]
    for _ in range(600):
        p = ("(?s)" if rng.random() < 0.3 else "") + ("^" if rng.random() < 0.3 else "")
        p += "".join(rng.choice(pieces) for _ in range(rng.randrange(4))) + ("$" if rng.random() < 0.3 else "")
        kind, pat, flags, esc = plb.regex_to_device(p)
        assert mapped_oracle(texts, kind, pat, flags, esc) == so.regex_search(texts, p), p
    # the regex crate's $ is the end of the text only (Python's re would also match before a final "\n")
    assert so.regex_search(["ab\n", "ab"], "ab$") == [False, True]


def test_declared_symbols_and_rust_parity():
    import polars_b200 as plb
    for name in ("bl_string_compare", "bl_string_match", "bl_string_filter"):
        assert hasattr(plb.lib(), name)
    header = open(os.path.join(ROOT, "include", "polars_b200.h")).read()
    assert "enum { BL_STR_STARTS_WITH = 0, BL_STR_ENDS_WITH = 1, BL_STR_CONTAINS = 2, BL_STR_LIKE = 3 };" in header
    assert "enum { BL_STR_NEGATE = 1, BL_LIKE_NO_NEWLINE = 2, BL_LIKE_OPEN_START = 4, BL_LIKE_OPEN_END = 8 };" in header
    assert "bl_status bl_string_filter(const bl_string_column* chunks, int32_t n_chunks, const bl_column* mask, int32_t out_location, bl_string_column* out);" in header
    rs = open(os.path.join(ROOT, "integration", "polars_b200_sys.rs")).read()
    assert "pub fn bl_string_compare(op: i32, lhs: *const BlStringColumn, n_lhs_chunks: i32, rhs: *const BlStringColumn, n_rhs_chunks: i32, missing: i32, out_location: i32, out: *mut BlColumn) -> i32;" in rs
    assert "pub fn bl_string_match(kind: i32, flags: i32, escape: i32, col: *const BlStringColumn, n_chunks: i32, pattern: *const BlStringColumn, n_pattern_chunks: i32, out_location: i32, out: *mut BlColumn) -> i32;" in rs
    assert "pub fn bl_string_filter(" in rs and "pub const BL_LIKE_OPEN_END: i32 = 8;" in rs
    assert plb.STR_KINDS == {"starts_with": 0, "ends_with": 1, "contains": 2, "like": 3}
    assert (plb.STR_NEGATE, plb.LIKE_NO_NEWLINE, plb.LIKE_OPEN_START, plb.LIKE_OPEN_END) == (1, 2, 4, 8)
