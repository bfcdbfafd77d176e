"""Pure-Python restatement of the reference's rank (polars-ops/src/series/ops/rank.rs:61-188), per partition, with the
order_by tie rule of ORDINAL and this library's RANDOM tie key.  Values are Python lists with None for a null: ints,
floats (NaN, -0.0 and infinities allowed), bools or bytes.  No numpy in the rule itself, so it is readable next to rank.rs;
`rank_np` is a vectorised restatement for large inputs, checked against `rank` on CPU (tests/test_rank.py)."""
from __future__ import annotations

import math

import numpy as np

METHODS = ["average", "min", "max", "dense", "ordinal", "random"]
M32 = 0xFFFFFFFF


def total_key(v):
    """A sort key whose order is the reference's total order (reorder_cmp / tot_cmp): NaN == NaN and greatest,
    -0.0 == +0.0; bytes unsigned with a proper prefix first; False < True."""
    if isinstance(v, float):
        return (1, 0.0) if math.isnan(v) else (0, v + 0.0)
    if isinstance(v, bool):
        return (0, int(v))
    return (0, v)


def fmix32(h: int) -> int:
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & M32
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & M32
    h ^= h >> 16
    return h


def random_key(row: int, seed: int) -> int:
    """RANDOM's tie key of a row (the header's bl_rank): fmix32(fmix32(row ^ seed_lo) + seed_hi)"""
    return fmix32(((fmix32((row & M32) ^ (seed & M32)) + (seed >> 32)) & M32))


def order_ranks(keys, descending=False, nulls_last=False):
    """The position of every row in the stable sort of an order_by column with its flags (nulls placed by nulls_last only)"""
    n = len(keys)
    valid = [i for i in range(n) if keys[i] is not None]
    nulls = [i for i in range(n) if keys[i] is None]
    valid = sorted(valid, key=lambda i: total_key(keys[i]), reverse=descending)      # Python's reverse sort stays stable
    order = valid + nulls if nulls_last else nulls + valid
    pos = [0] * n
    for p, i in enumerate(order):
        pos[i] = p
    return pos


def rank_partition(values, rows, method, descending=False, tie=None):
    """{row: rank} for the rows of one partition (in row order).  tie: row -> secondary key (ORDINAL's order_by position,
    RANDOM's random_key); None keeps row order."""
    nn = [r for r in rows if values[r] is not None]
    if tie is not None:
        nn = sorted(nn, key=tie)
    # the stable arg_sort with nulls last (rank.rs:101-107), sliced to the non-null rows
    idx = sorted(nn, key=lambda r: total_key(values[r]), reverse=descending)
    out = {}
    if method in ("ordinal", "random"):
        for p, r in enumerate(idx):
            out[r] = p + 1
        return out
    # tie runs: consecutive sorted values that are not equal under tot_eq (rank.rs:117-123)
    s = 0
    dense = 0
    while s < len(idx):
        e = s + 1
        while e < len(idx) and total_key(values[idx[e]]) == total_key(values[idx[s]]):
            e += 1
        dense += 1
        for r in idx[s:e]:
            out[r] = {"average": 0.5 * ((s + 1) + e), "min": s + 1, "max": e, "dense": dense}[method]
        s = e
    return out


def rank(values, method, descending=False, parts=None, order=None, seed=0):
    """Ranks of every row (None for a null value).  parts: a partition label per row (None: one partition; any hashable,
    None included, is its own label); order: ORDINAL's order_by position per row (order_ranks)."""
    n = len(values)
    groups = {}
    for r in range(n):
        groups.setdefault(parts[r] if parts is not None else 0, []).append(r)
    tie = None
    if method == "ordinal" and order is not None:
        tie = lambda r: order[r]      # noqa: E731
    if method == "random":
        tie = lambda r: random_key(r, seed)      # noqa: E731
    out = [None] * n
    for rows in groups.values():
        for r, k in rank_partition(values, rows, method, descending, tie).items():
            out[r] = k
    return out


def brute(values, method, descending=False):
    """The definitions: min = 1 + #{v_j < v_i}, max = #{v_j <= v_i}, dense = 1 + #distinct{v_j < v_i}, average = (min + max) / 2,
    under the total order (reversed when descending); nulls give None.  ORDINAL / RANDOM are not defined this way."""
    keys = [None if v is None else total_key(v) for v in values]
    lt = (lambda a, b: a > b) if descending else (lambda a, b: a < b)
    out = []
    for k in keys:
        if k is None:
            out.append(None)
            continue
        others = [j for j in keys if j is not None]
        mn = 1 + sum(lt(j, k) for j in others)
        mx = sum(lt(j, k) or j == k for j in others)
        dn = 1 + len({j for j in others if lt(j, k)})
        out.append({"min": mn, "max": mx, "dense": dn, "average": (mn + mx) / 2}[method])
    return out


def rank_np(x: np.ndarray, valid, method, descending=False, gid=None, tie=None):
    """A numpy restatement of `rank` for large inputs: x numeric, valid a bool mask or None, gid int partition labels or None,
    tie a secondary int key (ORDINAL's order position or RANDOM's key) or None.  Returns (ranks, valid): ranks uint32 or
    float64 with 0 in null slots."""
    n = len(x)
    valid = np.ones(n, bool) if valid is None else np.asarray(valid, bool)
    g = np.zeros(n, np.int64) if gid is None else np.asarray(gid, np.int64)
    isnan = np.isnan(x) if x.dtype.kind == "f" else np.zeros(n, bool)
    if x.dtype.kind == "f":
        v = x.astype(np.float64) + 0.0
        v[isnan] = 0.0
        cls = isnan.astype(np.int64)      # NaN after every number
    elif x.dtype.kind == "u":
        v, cls = x.astype(np.uint64), np.zeros(n, np.int64)
    else:
        v, cls = x.astype(np.int64), np.zeros(n, np.int64)
    if descending:
        cls = -cls
        v = -v if v.dtype.kind == "f" else ~v      # ~v reverses the integer order without overflow
    tk = np.arange(n) if tie is None else np.asarray(tie)
    # lexsort: last key is primary.  Order: partition, null last, value class, value, tie key, row.
    perm = np.lexsort((np.arange(n), tk, v, cls, ~valid, g))
    out = np.zeros(n, np.float64 if method == "average" else np.uint32)
    gs, vs, cs, oks = g[perm], v[perm], cls[perm], valid[perm]
    seg_head = np.ones(n, bool)
    seg_head[1:] = gs[1:] != gs[:-1]
    run_head = seg_head.copy()
    run_head[1:] |= (vs[1:] != vs[:-1]) | (cs[1:] != cs[:-1]) | (oks[1:] != oks[:-1])
    pos = np.arange(n)
    S = np.maximum.accumulate(np.where(seg_head, pos, 0))
    s = np.maximum.accumulate(np.where(run_head, pos, 0))
    run_id = np.cumsum(run_head) - 1
    starts = np.nonzero(run_head)[0]
    ends = np.append(starts[1:], n)
    e = ends[run_id]
    if method in ("ordinal", "random"):
        r = pos - S + 1
    elif method == "min":
        r = s - S + 1
    elif method == "max":
        r = e - S
    elif method == "dense":
        r = run_id - run_id[S] + 1
    else:
        r = 0.5 * ((s - S + 1).astype(np.float64) + (e - S).astype(np.float64))
    out[perm] = np.where(oks, r, 0)
    return out, valid
