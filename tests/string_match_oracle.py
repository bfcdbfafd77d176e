"""Exact reference semantics of the string predicates (bl_string_compare, bl_string_match, bl_string_filter), restated on
Python bytes, plus a numpy form for large fixed-width inputs.

Values are bytes or None (null); a result is a list of True / False / None.
  compare      unsigned byte order with a proper prefix first — Python's bytes order (polars-compute comparisons/binary.rs)
  starts_with / ends_with / contains   byte predicates; the empty pattern matches every non-null row
  like         ^(?s)<pattern>$ of polars-sql's visit_like over DECODED characters: '%' any run, '_' exactly one character,
               by a direct recursive matcher (no `re`); no_newline: neither matches '\\n'; open_start / open_end: the match
               may begin / end anywhere (a regex search without ^ / $)
  regex_search the device regex subset (polars_b200.regex_to_device) with the regex crate's meaning, for the mapping tests"""
from functools import lru_cache

import numpy as np

CMPS = {"eq": lambda a, b: a == b, "ne": lambda a, b: a != b, "lt": lambda a, b: a < b, "le": lambda a, b: a <= b,
        "gt": lambda a, b: a > b, "ge": lambda a, b: a >= b}


def enc(v):
    return None if v is None else (v.encode() if isinstance(v, str) else bytes(v))


def _rhs(other, n):
    if isinstance(other, list):
        assert len(other) == n
        return [enc(v) for v in other]
    return [enc(other)] * n


def compare(op: str, col, other, missing: bool = False) -> list:
    a, b = [enc(v) for v in col], _rhs(other, len(col))
    out = []
    for x, y in zip(a, b):
        if x is None or y is None:
            if missing:
                out.append((x is None and y is None) == (op == "eq"))
            else:
                out.append(None)
        else:
            out.append(CMPS[op](x, y))
    return out


def _pred(col, pattern, fn, negate=False) -> list:
    a, p = [enc(v) for v in col], _rhs(pattern, len(col))
    return [None if x is None or y is None else fn(x, y) != negate for x, y in zip(a, p)]


def starts_with(col, pattern, negate=False) -> list:
    return _pred(col, pattern, lambda x, y: x.startswith(y), negate)


def ends_with(col, pattern, negate=False) -> list:
    return _pred(col, pattern, lambda x, y: x.endswith(y), negate)


def contains(col, pattern, negate=False) -> list:
    return _pred(col, pattern, lambda x, y: y in x, negate)


def like_tokens(pattern: bytes, escape=None) -> list:
    """('lit', char) | ('any',) | ('star',) over the decoded pattern; a bad escape raises ValueError"""
    s, toks, i = pattern.decode(), [], 0
    esc = None if escape is None else (escape if isinstance(escape, str) else chr(escape))
    while i < len(s):
        c = s[i]
        if esc is not None and c == esc:
            if i + 1 >= len(s) or s[i + 1] not in ("%", "_", esc):
                raise ValueError("bad escape")
            toks.append(("lit", s[i + 1]))
            i += 2
            continue
        toks.append(("star",) if c == "%" else ("any",) if c == "_" else ("lit", c))
        i += 1
    return toks


def like_match(text: bytes, toks, no_newline=False, open_start=False, open_end=False) -> bool:
    t = text.decode()
    toks = tuple(toks)

    @lru_cache(maxsize=None)
    def m(i, j):      # does t[i:] match toks[j:]?
        if j == len(toks):
            return i == len(t) or open_end
        k = toks[j]
        if k[0] == "star":
            return m(i, j + 1) or (i < len(t) and not (no_newline and t[i] == "\n") and m(i + 1, j))
        if i == len(t):
            return False
        if k[0] == "any":
            return not (no_newline and t[i] == "\n") and m(i + 1, j + 1)
        return t[i] == k[1] and m(i + 1, j + 1)

    starts = range(len(t) + 1) if open_start else (0,)
    return any(m(i, 0) for i in starts)


def like(col, pattern, negate=False, no_newline=False, escape=None, open_start=False, open_end=False) -> list:
    p = enc(pattern)
    if p is None:
        return [None] * len(col)
    toks = like_tokens(p, escape)
    return [None if x is None else like_match(x, toks, no_newline, open_start, open_end) != negate for x in (enc(v) for v in col)]


def regex_search(col, pattern: str) -> list:
    """str.contains(pattern, literal=False) for a regex of the device subset, in the regex crate's meaning ($ only at the
    end of the text, '.' one character, '\\n' only under (?s)).  Written against the subset's grammar, not `re`."""
    s = pattern
    dotall = s.startswith("(?s)")
    s = s[4:] if dotall else s
    a0 = s.startswith("^")
    s = s[1:] if a0 else s
    toks, i, a1 = [], 0, False
    while i < len(s):
        if s[i] == "\\":
            toks.append(("lit", s[i + 1])); i += 2
        elif s[i] == "." and s[i + 1:i + 2] == "*":
            toks.append(("star",)); i += 2
        elif s[i] == ".":
            toks.append(("any",)); i += 1
        elif s[i] == "$" and i == len(s) - 1:
            a1 = True; i += 1
        else:
            toks.append(("lit", s[i])); i += 1
    return [None if x is None else like_match(x, toks, not dotall, not a0, not a1) for x in (enc(v) for v in col)]


def filter_rows(col, mask) -> list:
    return [enc(v) for v, k in zip(col, mask) if k]


# ---------------------------------------------------------------------------- numpy form (fixed-width rows)
def np_rows(data: np.ndarray, offsets: np.ndarray, width: int) -> np.ndarray:
    """rows of exactly `width` bytes as an (n, width) uint8 matrix"""
    n = offsets.size - 1
    assert np.all(np.diff(offsets) == width)
    return data[offsets[0]:offsets[0] + n * width].reshape(n, width)


def np_contains(rows: np.ndarray, needle: bytes) -> np.ndarray:
    n, w = rows.shape
    m = len(needle)
    if m == 0:
        return np.ones(n, bool)
    if m > w:
        return np.zeros(n, bool)
    nd = np.frombuffer(needle, np.uint8)
    hit = np.zeros(n, bool)
    for i in range(w - m + 1):
        hit |= np.all(rows[:, i:i + m] == nd, axis=1)
    return hit


def np_starts_with(rows: np.ndarray, prefix: bytes) -> np.ndarray:
    m = len(prefix)
    if m > rows.shape[1]:
        return np.zeros(rows.shape[0], bool)
    return np.all(rows[:, :m] == np.frombuffer(prefix, np.uint8), axis=1)


def np_compare(op: str, a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """equal-width rows (n, w) compared in byte order: the first differing byte decides"""
    diff = a != b
    first = np.where(diff.any(axis=1), diff.argmax(axis=1), a.shape[1])
    idx = np.minimum(first, a.shape[1] - 1)
    av, bv = a[np.arange(a.shape[0]), idx].astype(np.int16), b[np.arange(b.shape[0]), idx].astype(np.int16)
    c = np.where(first == a.shape[1], 0, np.sign(av - bv))
    return {"eq": c == 0, "ne": c != 0, "lt": c < 0, "le": c <= 0, "gt": c > 0, "ge": c >= 0}[op]
