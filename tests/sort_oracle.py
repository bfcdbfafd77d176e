"""Plain-Python restatement of the reference's multi-column arg_sort, the checker of bl_arg_sort / bl_sort.

Order (polars-utils/src/sort.rs:113-128, reorder_cmp): nulls compare equal to each other and sit first or last by
`nulls_last` alone; values compare in their total order (floats by tot_cmp, polars-utils/src/total_ord.rs: NaN == NaN
and greater than every other value, -0.0 == +0.0), reversed by `descending`.  Columns are compared in order and ties
fall back to the row index: the stable order, which the reference returns for a single column (arg_sort.rs:118-185) and
with maintain_order (arg_sort_multiple.rs:66-75).  `limit` keeps the first rows (frame/mod.rs:1482-1486).
O(n log n) Python comparisons: meant for small inputs."""
from __future__ import annotations

import functools
import math

import numpy as np


def _tot_cmp(a, b) -> int:
    if isinstance(a, float) and math.isnan(a):
        return 0 if (isinstance(b, float) and math.isnan(b)) else 1
    if isinstance(b, float) and math.isnan(b):
        return -1
    return (a > b) - (a < b)          # -0.0 == +0.0 here already


def _reorder_cmp(a, b, descending: bool, nulls_last: bool) -> int:
    if a is None and b is None:
        return 0
    if a is None:
        return 1 if nulls_last else -1
    if b is None:
        return -1 if nulls_last else 1
    c = _tot_cmp(a, b)
    return -c if descending else c


def _broadcast(v, n: int, what: str):
    if isinstance(v, (bool, np.bool_)):
        return [bool(v)] * n
    v = [bool(x) for x in v]
    if len(v) != n:
        raise ValueError(f"the length of `{what}` ({len(v)}) does not match the length of `by` ({n})")
    return v


def arg_sort(cols, valids=None, descending=False, nulls_last=False, limit=None) -> np.ndarray:
    """cols: key columns (sequences / numpy arrays of one length); valids: per column a bool array or None.
    -> the uint32 permutation, truncated to `limit`."""
    k = len(cols)
    valids = valids if valids is not None else [None] * k
    desc, nl = _broadcast(descending, k, "descending"), _broadcast(nulls_last, k, "nulls_last")
    n = len(cols[0]) if k else 0
    rows = []
    for c, v in zip(cols, valids):
        vals = [x.item() if hasattr(x, "item") else x for x in c]
        rows.append([None if (v is not None and not v[i]) or vals[i] is None else vals[i] for i in range(n)])

    def cmp(i, j):
        for c in range(k):
            r = _reorder_cmp(rows[c][i], rows[c][j], desc[c], nl[c])
            if r:
                return r
        return (i > j) - (i < j)

    order = sorted(range(n), key=functools.cmp_to_key(cmp))
    if limit is not None and limit >= 0:
        order = order[:limit]
    return np.array(order, dtype=np.uint32)


def numpy_sort_keys(col, valid, descending: bool, nulls_last: bool):
    """The same order as numpy keys for np.lexsort (least significant first): (value key, null rank) of one column.
    Floats: -0.0 -> +0.0 and every NaN -> +inf-above (rank by np.unique), then negated for descending."""
    a = np.asarray(col)
    valid = np.ones(a.shape, bool) if valid is None else np.asarray(valid, bool)
    if a.dtype.kind == "f":
        x = np.where(a == 0, 0.0, a).astype(np.float64)
        nan = np.isnan(x)
        _, rank = np.unique(np.where(nan, 0.0, x), return_inverse=True)
        key = np.where(nan, rank.max(initial=0) + 1, rank).astype(np.int64)
    elif a.dtype == np.bool_:
        key = a.astype(np.int64)
    else:
        _, key = np.unique(a, return_inverse=True)       # dense rank: exact for every integer dtype incl. uint64
        key = key.astype(np.int64)
    key = np.where(valid, -key if descending else key, 0)
    null_rank = np.where(valid, 0, 1) if nulls_last else np.where(valid, 1, 0)
    return key, null_rank


def numpy_arg_sort(cols, valids=None, descending=False, nulls_last=False, limit=None) -> np.ndarray:
    """Vectorised equivalent of arg_sort for large inputs: np.lexsort (stable) over the transformed keys."""
    k = len(cols)
    valids = valids if valids is not None else [None] * k
    desc, nl = _broadcast(descending, k, "descending"), _broadcast(nulls_last, k, "nulls_last")
    keys = []
    for c in reversed(range(k)):          # lexsort: last key is the primary one
        key, null_rank = numpy_sort_keys(cols[c], valids[c], desc[c], nl[c])
        keys += [key, null_rank]
    n = len(cols[0])
    order = np.lexsort(keys) if n else np.zeros(0, np.int64)
    if limit is not None and limit >= 0:
        order = order[:limit]
    return order.astype(np.uint32)
