"""Plain-Python restatement of the reference's window functions (mapping_strategy "group_to_rows") and cumulative functions.

- partitions: groups in first-occurrence order (a null key is its own group, floats -0 == +0 and NaN == NaN), each group's
  rows ascending (GroupsIdx), or stably sorted by one order_by key (update_groups_sort_by, polars-expr/src/expressions/
  sortby.rs:57-100: total order with NaN greatest, `descending` reverses it, nulls placed by `nulls_last` alone);
- the det_* scans of polars-ops/src/series/ops/cum_agg.rs with Rust integer wrapping and the f32 -> f64 sum (:14-53),
  min_ignore_nan / max_ignore_nan (polars-utils/src/min_max.rs:33-48, floats :87-108), cum_count (:428-466) and shift;
- aggregations broadcast to the rows of their group (the per-group values come from the quantile oracle and the reducers
  restated here for the kinds the GPU tests use).
Values are Python numbers (floats keep their sign of zero and NaN), None for null."""
from __future__ import annotations

import functools
import math

import numpy as np

from quantile_oracle import quantile_of

INT_BITS = {"int8": (8, True), "int16": (16, True), "int32": (32, True), "int64": (64, True),
            "uint8": (8, False), "uint16": (16, False), "uint32": (32, False), "uint64": (64, False)}


def wrap(x: int, dtype: str) -> int:
    bits, signed = INT_BITS[dtype]
    x &= (1 << bits) - 1
    return x - (1 << bits) if signed and x >> (bits - 1) else x


def scan_dtype(kind: str, dtype: str) -> str:
    """Output dtype of a cumulative kind / shift (cum_agg.rs:261-333)"""
    small = dtype in ("int8", "int16", "uint8", "uint16")
    if kind == "cum_sum":
        return "uint32" if dtype == "bool" else "int64" if small else dtype
    if kind == "cum_prod":
        return "int64" if dtype == "bool" or small or dtype in ("int32", "uint32") else dtype
    if kind == "cum_count":
        return "uint32"
    return dtype


def _canon(v):
    if v is None:
        return ("null",)
    if isinstance(v, float):
        if v != v:
            return ("nan",)
        return ("v", v + 0.0)
    return ("v", v)


def groups(key_cols, n: int):
    """key_cols: list of per-row value lists -> row lists of the groups in first-occurrence order (rows ascending)"""
    if not key_cols:
        return [list(range(n))] if n else []
    at, out = {}, []
    for r in range(n):
        k = tuple(_canon(c[r]) for c in key_cols)
        if k not in at:
            at[k] = len(out)
            out.append([])
        out[at[k]].append(r)
    return out


def _tot_cmp(a, b) -> int:
    """total order: NaN greatest and equal to NaN, -0.0 == +0.0"""
    an = isinstance(a, float) and a != a
    bn = isinstance(b, float) and b != b
    if an or bn:
        return (an > bn) - (an < bn)
    return (a > b) - (a < b)


def sort_group(rows, key, descending: bool, nulls_last: bool):
    """stable sort of one group's rows by key[row] (sort_by: ties keep row order)"""
    def cmp(i, j):
        a, b = key[i], key[j]
        if a is None or b is None:
            if a is None and b is None:
                return 0
            return (1 if nulls_last else -1) if a is None else (-1 if nulls_last else 1)
        c = _tot_cmp(a, b)
        return -c if descending else c
    return sorted(rows, key=functools.cmp_to_key(cmp))


def partition_order(key_cols, n: int, order=None, descending=False, nulls_last=False):
    g = groups(key_cols, n)
    if order is not None:
        g = [sort_group(rows, order, descending, nulls_last) for rows in g]
    return g


def min_ignore_nan(s, v):
    if isinstance(v, float) and v != v:
        return s
    if isinstance(s, float) and s != s:
        return v
    return s if s < v else v       # equal: the later value


def max_ignore_nan(s, v):
    if isinstance(v, float) and v != v:
        return s
    if isinstance(s, float) and s != s:
        return v
    return v if s < v else s       # equal: the earlier value


def cum_seq(kind: str, vals, dtype: str):
    """One partition's values in scan order (None = null) -> outputs in the same order"""
    odt = scan_dtype(kind, dtype)
    out = []
    if kind == "cum_count":
        c = 0
        for v in vals:
            c += v is not None
            out.append(c)
        return out
    is_float = dtype.startswith("float")
    if kind == "cum_sum":
        s = 0.0 if is_float else 0
    elif kind == "cum_prod":
        s = np.float32(1.0) if dtype == "float32" else 1.0 if is_float else 1
    else:
        s = float("nan") if is_float else None
    for v in vals:
        if v is None:
            out.append(None)
            continue
        if dtype == "bool":
            v = int(v)
        if kind == "cum_sum":
            s = s + float(v) if is_float else wrap(s + v, odt)      # Float32: the f64 state of det_sum_to_f64
            out.append(float(np.float32(s)) if dtype == "float32" else s)
        elif kind == "cum_prod":
            if dtype == "float32":
                s = np.float32(s) * np.float32(v)
                out.append(float(s))
            else:
                s = s * float(v) if is_float else wrap(s * v, odt)
                out.append(s)
        else:
            fn = min_ignore_nan if kind == "cum_min" else max_ignore_nan
            s = v if s is None else fn(s, v)
            out.append(s)
    return out


def agg_value(kind: str, vals, dtype: str, q=None, method=None):
    """One group's aggregation over its values in fold order (None = null) -> value or None"""
    name, _, dd = kind.partition(":")
    valid = [v for v in vals if v is not None]
    if name == "len":
        return len(vals)
    if name == "count":
        return len(valid)
    if name == "n_unique":
        return len({_canon(v) for v in vals})
    if name in ("first", "last"):
        return (vals[0] if name == "first" else vals[-1]) if vals else None
    if not valid:
        return 0 if name == "sum" and not dtype.startswith("float") else (0.0 if name == "sum" else None)
    if name == "sum":
        return math.fsum(valid) if dtype.startswith("float") else wrap(sum(valid), "int64" if dtype in ("int8", "int16", "uint8", "uint16") else dtype)
    if name == "min":
        return functools.reduce(min_ignore_nan, valid)
    if name == "max":
        return functools.reduce(max_ignore_nan, valid)
    if name == "mean":
        return math.fsum(valid) / len(valid)
    if name in ("var", "std"):
        ddof = int(dd) if dd else 1
        if len(valid) <= ddof:
            return None
        m = math.fsum(valid) / len(valid)
        r = math.fsum((x - m) ** 2 for x in valid) / (len(valid) - ddof)
        return math.sqrt(r) if name == "std" else r
    if name in ("median", "quantile"):
        return quantile_of([0 if v is None else v for v in vals], [v is not None for v in vals], 0.5 if name == "median" else q,
                           "linear" if name == "median" else method)
    raise ValueError(kind)


def over(ops, key_cols, n: int, order=None, descending=False, nulls_last=False):
    """ops: [(kind, values list | None, dtype, options)] -> one output list per op (row order, None = null)"""
    part = partition_order(key_cols, n, order, descending, nulls_last)
    outs = []
    for kind, vals, dtype, opts in ops:
        res = [None] * n
        for rows in part:
            seq = [vals[r] for r in rows] if vals is not None else [0] * len(rows)
            if kind.startswith("cum_"):
                rev = bool(opts.get("reverse", False))
                r_rows = rows[::-1] if rev else rows
                got = cum_seq(kind, [vals[r] for r in r_rows], dtype)
                for r, x in zip(r_rows, got):
                    res[r] = x
            elif kind == "shift":
                k = int(opts.get("periods", 1))
                for i, r in enumerate(rows):
                    j = i - k
                    res[r] = seq[j] if 0 <= j < len(rows) else None
            else:
                q = method = None
                if kind.startswith("quantile:"):
                    _, qs, method = (kind.split(":") + ["nearest"])[:3]
                    q = float(qs)
                a = agg_value(kind, seq, dtype, q, method)
                for r in rows:
                    res[r] = a
        outs.append(res)
    return outs
