"""Plain-Python restatement of DataFrame.unique and the is_unique / is_duplicated / is_first_distinct / is_last_distinct
masks (polars-core/src/frame/mod.rs:2317-2442, polars-ops/src/series/ops/is_unique.rs, is_first_distinct.rs,
is_last_distinct.rs).

One dict from the canonical row key to [first row, last row, count], filled in row order; the kept ids and the four
masks are read off it.  A row key is the tuple of its columns' canonical values: a null is a value of its own, floats
compare by total equality (-0.0 == +0.0, every NaN equal), strings and binary by bytes.  `np_table` is the same table
computed with numpy, for inputs too large for the dict."""
import math

import numpy as np

KEEP = ("first", "last", "any", "none")
KINDS = ("first", "last", "unique", "duplicated")


def canon(v):
    if v is None:
        return ("null",)
    if isinstance(v, (float, np.floating)):
        return ("nan",) if math.isnan(v) else ("f", float(v) + 0.0)      # + 0.0 turns -0.0 into +0.0
    if isinstance(v, str):
        return ("b", v.encode())
    if isinstance(v, (bytes, bytearray)):
        return ("b", bytes(v))
    if isinstance(v, (bool, np.bool_)):
        return ("t", bool(v))
    return ("i", int(v))


def table(cols):
    """cols: one list of values per key column (None = null) -> (row keys, {key: [first, last, count]})"""
    n = len(cols[0]) if cols else 0
    keys = [tuple(canon(c[i]) for c in cols) for i in range(n)]
    t = {}
    for i, k in enumerate(keys):
        e = t.get(k)
        if e is None:
            t[k] = [i, i, 1]
        else:
            e[1] = i
            e[2] += 1
    return keys, t


def masks(cols):
    """kind -> one bool per row"""
    keys, t = table(cols)
    return {"first": [t[k][0] == i for i, k in enumerate(keys)], "last": [t[k][1] == i for i, k in enumerate(keys)],
            "unique": [t[k][2] == 1 for k in keys], "duplicated": [t[k][2] > 1 for k in keys]}


def arg_unique(cols, keep):
    """the kept rows as ascending row ids"""
    if keep not in KEEP:
        raise ValueError(keep)
    m = masks(cols)["first" if keep in ("first", "any") else "last" if keep == "last" else "unique"]
    return [i for i, b in enumerate(m) if b]


def _np_codes(values, valid):
    """one column (a numpy array, or a list of str / bytes / None) -> int64 class ids (equal ids <=> equal canonical values; nulls share one id of their own)"""
    if not isinstance(values, np.ndarray):      # str / bytes lists stay Python objects: numpy's bytes strip trailing NULs
        d = {}
        values = np.fromiter((d.setdefault(canon(x), len(d)) for x in values), dtype=np.int64, count=len(values))
    v = values
    if v.dtype.kind == "f":
        with np.errstate(invalid="ignore"):      # signalling NaN payloads
            f = v.astype(np.float64) + 0.0
        bits = f.view(np.uint64).copy()
        bits[np.isnan(f)] = np.uint64(0x7FF8000000000000)
        v = bits
    elif v.dtype.kind == "b":
        v = v.astype(np.uint8)
    codes = np.unique(v, return_inverse=True)[1].astype(np.int64).reshape(-1)
    if valid is not None:
        codes = np.where(np.asarray(valid, bool), codes, codes.max(initial=-1) + 1)
    return codes


def np_group_ids(cols):
    """cols: (values, valid | None) per key column -> int64 group id per row, 0 .. G - 1"""
    g = None
    for values, valid in cols:
        c = _np_codes(values, valid)
        g = c if g is None else np.unique(g * (int(c.max(initial=0)) + 1) + c, return_inverse=True)[1].astype(np.int64).reshape(-1)
    return np.unique(g, return_inverse=True)[1].astype(np.int64).reshape(-1)


def np_masks(cols):
    """the four masks of numpy key columns, derived from the same (first, last, count) table"""
    g = np_group_ids(cols)
    n = g.size
    if n == 0:
        e = np.zeros(0, bool)
        return {k: e for k in KINDS}
    _, first, count = np.unique(g, return_index=True, return_counts=True)
    last = n - 1 - np.unique(g[::-1], return_index=True)[1]
    rows = np.arange(n)
    return {"first": first[g] == rows, "last": last[g] == rows, "unique": count[g] == 1, "duplicated": count[g] > 1}


def np_arg_unique(cols, keep):
    m = np_masks(cols)["first" if keep in ("first", "any") else "last" if keep == "last" else "unique"]
    return np.flatnonzero(m).astype(np.uint32)
