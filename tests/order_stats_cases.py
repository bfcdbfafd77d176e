"""Builders, exact references and CPU restatements of the plan choices of the order statistics built on the stable sort:
bl_top_k (top_k.cu), bl_rank (rank.cu) and bl_rolling_quantile(_by) (rolling_quantile.cu).

References (tests/test_order_stats_cases.py checks them against sort_oracle, rank_oracle and rolling_quantile_oracle):
- topk_ref: np.lexsort over the sort keys and the row index; the first k rows, ascending.
- rank_ref: lexsort by (partition, nulls last, value), run and partition heads, the five methods in closed form.
- rq_ref: an exact per-window selection (np.sort of each window's valid values) with the f64 index arithmetic
  of k_rq_out; rq_monotone: the closed form of a column whose values never decrease along the rows.

Restatements (each GPU test asserts what its input reaches through them):
- topk_plan: op_top_k's host loop (AND / OR, varying digits, per-step histogram, bucket, need, count, list or
  streaming, tie step or final mark) with the launch counts of every k_topk_pass flavour.
- rank_plan: which of start / seg_pos / seg_run / valid_bm rank_one allocates, whether k_rank_starts runs, and the
  tile count against the grid min(ntiles, 8 SM).
- rq_plan / rq_edges: the wavelet matrix's level count L, its k_wm_count launches (L, plus 1 with nulls) and where every
  window's s and e fall among the 224-position blocks and 1792-position tiles.
"""
from __future__ import annotations

import math
from collections import Counter

import numpy as np

import sort_oracle

TK_LIST_DIV = 32            # top_k.cu: candidate sets of at most n / TK_LIST_DIV rows run over a row-id list
F_TILE = 4096               # filter.cu: mask_first / mask_rows count the set bits per tile of F_TILE rows
SELECT_DIV = 8              # sort.cu SORT_SELECT_DIV: a sort with limit <= n / 8 selects first (4- and 8-byte keys)
RK_TILE = 2048              # rank.cu: positions per k_rank_heads / k_rank_starts / k_rank_out tile
RK_WARP = 256               # positions per warp (8 bitmap words)
BV_BITS, BV_TILE = 224, 1792      # rolling_quantile.cu: bitvector block and tile
QMETHODS = ["nearest", "lower", "higher", "midpoint", "linear", "equiprobable"]
RANK_METHODS = ["average", "min", "max", "dense", "ordinal"]


def grid_cap(sm: int) -> int:
    """the CTA cap of rank.cu's three kernels: 8 per SM"""
    return 8 * sm


# ================================================================================================ keys
def value_key(x, dtype: str) -> np.ndarray:
    """sort_value_key (sort_keys.cuh) as uint64: integers with the sign bit flipped, floats canonical (-0 -> +0, one
    NaN) and mapped to an order-preserving unsigned key, Bool 0 / 1"""
    a = np.asarray(x)
    if dtype == "bool":
        return a.astype(np.uint64)
    if dtype.startswith("int"):
        w = a.dtype.itemsize
        return a.view(f"u{w}").astype(np.uint64) ^ np.uint64(1 << (8 * w - 1))
    if dtype.startswith("uint"):
        return a.astype(np.uint64)
    if dtype == "float32":
        z = a + np.float32(0)
        u = np.where(np.isnan(z), np.uint32(0x7FC00000), z.view(np.uint32)).astype(np.uint64)
        return np.where(u >> np.uint64(31), ~u & np.uint64(0xFFFFFFFF), u | np.uint64(0x80000000))
    z = a + 0.0
    u = np.where(np.isnan(z), np.uint64(0x7FF8000000000000), z.view(np.uint64)).astype(np.uint64)
    return np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))


def _wide(dtype: str) -> bool:
    return dtype in ("int64", "uint64", "float64")


def bits_for(v: int) -> int:
    """common.cuh bits_for: the bits of v, at least 1 and at most 32"""
    b = 1
    while b < 32 and (v >> b):
        b += 1
    return b


# ================================================================================================ top_k
def topk_ref(cols, valids, k, desc=False, nl=False) -> np.ndarray:
    """the first k rows of the stable order (lexsort with the row index last), as ascending uint32 row ids"""
    return np.sort(sort_oracle.numpy_arg_sort(cols, valids, desc, nl, limit=k)).astype(np.uint32)


def topk_parts(cols, valids, dtypes, desc, nl):
    """op_top_k's key parts, most significant first: (kind, key uint64 per row, rows its AND / OR reduces, top shift)"""
    k = len(cols)
    desc = [desc] * k if isinstance(desc, bool) else list(desc)
    nl = [nl] * k if isinstance(nl, bool) else list(nl)
    n = len(cols[0])
    parts = []
    for c, v, dt, d, l in zip(cols, valids, dtypes, desc, nl):
        ok = np.ones(n, bool) if v is None else np.asarray(v, bool)
        if v is not None:
            parts.append(("nulls", ((~ok).astype(np.uint64) ^ np.uint64(0 if l else 1)), np.ones(n, bool), 0))
        width = np.uint64(2**64 - 1) if _wide(dt) else np.uint64(0xFFFFFFFF)
        key = value_key(c, dt)
        if d:
            key = ~key & width
        parts.append(("value", np.where(ok, key, np.uint64(0)), ok, 56 if _wide(dt) else 24))
    return parts


def topk_digits(parts, n):
    """(part, shift) of every digit a pass looks at, most significant first: the varying key digits, then every digit
    of the row index (bits_for(n - 1) bits); and the number of key digits"""
    digits = []
    for p, (_, key, rows, top) in enumerate(parts):
        if rows.any():
            a = np.bitwise_and.reduce(key[rows])
            o = np.bitwise_or.reduce(key[rows])
            vary = int(a ^ o)
        else:
            vary = 0      # AND not in OR: no row reduced
        for sh in range(top, -1, -8):
            if (vary >> sh) & 0xFF:
                digits.append((p, sh))
    nk = len(digits)
    row_bits = bits_for(n - 1)
    for sh in range((row_bits - 1) // 8 * 8, -1, -8):
        digits.append((len(parts), sh))
    return digits, nk


def topk_plan(cols, valids, dtypes, k, desc=False, nl=False, list_div=TK_LIST_DIV):
    """op_top_k's host loop.  Returns a dict: launches (Counter of the kernel names the launch profile shows), steps
    (per pass: part, shift, list or streaming, rows it runs over, whether it appends a list, bucket b, need and count
    after it), row_digits (digits of the row index), tie (need at the tie step or None) and ids (the selected rows)."""
    n = len(cols[0])
    out = {"launches": Counter(), "steps": [], "row_digits": (bits_for(max(n - 1, 0)) + 7) // 8, "tie": None}
    if k >= n:
        out["launches"]["iota"] += 1 if n else 0
        out["ids"] = np.arange(n, dtype=np.uint32)
        return out
    if k == 0:
        out["ids"] = np.zeros(0, np.uint32)
        return out
    list_max = n // list_div
    parts = topk_parts(cols, valids, dtypes, desc, nl)
    out["launches"]["topk_andor"] = len(parts)
    digits, nk = topk_digits(parts, n)
    keys = [p[1] for p in parts] + [np.arange(n, dtype=np.uint64)]
    cand = np.ones(n, bool)
    sel = np.zeros(n, bool)
    listed, m, need, count = False, n, k, n
    L = out["launches"]
    for di in range(len(digits) + 1):
        if di >= nk and not listed and count > list_max:
            if count == n:      # nothing narrowed the rows: rows 0 .. need
                L["iota"] += 1
                out["ids"] = np.arange(need, dtype=np.uint32)
                return out
            L["topk_tie"] += 1
            L["mask_first"] += 1
            L["k3_tile_counts"] += 2      # mask_first's tile offsets, then op_mask_rows'
            L["mask_rows"] += 1
            out["tie"] = need
            sel[np.flatnonzero(cand)[:need]] = True
            out["ids"] = np.flatnonzero(sel).astype(np.uint32)
            return out
        p, sh = digits[di]
        list_out = count <= list_max and count < m
        L["topk_pass_list" if listed else "topk_pass"] += 1
        d = ((keys[p] >> np.uint64(sh)) & np.uint64(0xFF)).astype(np.int64)
        h = np.bincount(d[cand], minlength=256)
        below, b = 0, 0
        while below + h[b] < need:
            below += h[b]
            b += 1
        sel |= cand & (d < b)
        cand &= d == b
        step = {"part": p, "shift": sh, "list": listed, "rows": m, "appends": list_out, "b": b}
        if list_out:
            listed, m = True, count
        need -= below
        count = int(h[b])
        step.update(need=need, count=count)
        out["steps"].append(step)
        if count == need:
            break
    L["topk_mark_list" if listed else "topk_mark"] += 1
    L["k3_tile_counts"] += 1
    L["mask_rows"] += 1
    sel |= cand
    out["ids"] = np.flatnonzero(sel).astype(np.uint32)
    return out


def topk_msd_brute(cols, valids, dtypes, k, desc=False, nl=False):
    """brute-force MSD select: the k-th row of the full stable order fixes the bucket of every digit; after each digit
    the candidates are the rows whose digits so far equal that row's, and `need` is k minus the rows below them.
    Returns [(part, shift, b, need, count)] over the digits topk_plan visits, for the same digit list."""
    n = len(cols[0])
    parts = topk_parts(cols, valids, dtypes, desc, nl)
    digits, _ = topk_digits(parts, n)
    keys = [p[1] for p in parts] + [np.arange(n, dtype=np.uint64)]
    order = np.lexsort([np.arange(n)] + [keys[p] for p in reversed(range(len(parts)))])
    pivot = order[k - 1]
    less, eq = np.zeros(n, bool), np.ones(n, bool)
    res = []
    for p, sh in digits:
        d = ((keys[p] >> np.uint64(sh)) & np.uint64(0xFF)).astype(np.int64)
        less |= eq & (d < d[pivot])
        eq &= d == d[pivot]
        res.append((p, sh, int(d[pivot]), k - int(less.sum()), int(eq.sum())))
    return res


# ================================================================================================ rank
def rank_ref(x, valid, method, desc=False, gid=None):
    """ranks (uint32, or float64 for average; 0 in null slots): stable lexsort by (partition, nulls last, value), run
    heads where the value, the validity or the partition changes, partition heads where the partition changes; with
    S the partition's first position, s / e the run's first / end position and R the run number:
    ordinal = i - S + 1, min = s - S + 1, max = e - S, dense = R - R(S) + 1, average = (min + max) / 2"""
    n = len(x)
    key, null_rank = sort_oracle.numpy_sort_keys(x, valid, desc, True)
    g = np.zeros(n, np.int64) if gid is None else np.asarray(gid, np.int64)
    perm = np.lexsort((np.arange(n), key, null_rank, g))
    gs, ks, ns = g[perm], key[perm], null_rank[perm]
    seg = np.r_[True, gs[1:] != gs[:-1]]
    run = seg | np.r_[True, (ks[1:] != ks[:-1]) | (ns[1:] != ns[:-1])]
    pos = np.arange(n)
    S = np.maximum.accumulate(np.where(seg, pos, 0))
    s = np.maximum.accumulate(np.where(run, pos, 0))
    R = np.cumsum(run) - 1
    heads = np.flatnonzero(run)
    e = np.r_[heads[1:], n][R]
    r = {"ordinal": pos - S + 1, "min": s - S + 1, "max": e - S, "dense": R - R[S] + 1}.get(method)
    if method == "average":
        r = 0.5 * ((s - S + 1).astype(np.float64) + (e - S).astype(np.float64))
    ok = ns == 0
    out = np.zeros(n, np.float64 if method == "average" else np.uint32)
    out[perm] = np.where(ok, r, 0)
    return out


def rank_plan(n, method, partitioned, nulls, sm):
    """rank_one's buffers and launches for one op over n rows"""
    runs = method in ("average", "min", "max", "dense")
    start = runs and method != "dense"
    ntiles = -(-n // RK_TILE)
    grid = min(ntiles, grid_cap(sm))
    return {"start": start, "seg_pos": partitioned, "seg_run": partitioned and method == "dense", "valid_bm": nulls,
            "rank_starts": start or partitioned, "ntiles": ntiles, "grid": grid, "rounds": -(-ntiles // grid) if grid else 0}


def rank_launches(plans):
    """the rank kernels' launch counts over several ops"""
    c = Counter()
    for p in plans:
        c["rank_heads"] += 1
        c["rank_out"] += 1
        c["rank_starts"] += int(p["rank_starts"])
    return c


def first_row_ids(gid):
    """partition_ids (window.cu, op_group_first_ids): every row's partition named by the partition's first row, so the
    sort puts partitions in the order of their first rows"""
    g = np.asarray(gid)
    _, first, inv = np.unique(g, return_index=True, return_inverse=True)
    return first[inv.reshape(-1)]


def rank_heads(x, valid, gid=None, desc=False):
    """the run heads and partition heads k_rank_heads sees: positions in the device's sort by (first-row partition id,
    nulls last, value), stable"""
    n = len(x)
    key, null_rank = sort_oracle.numpy_sort_keys(x, valid, desc, True)
    g = np.zeros(n, np.int64) if gid is None else first_row_ids(gid)
    perm = np.lexsort((np.arange(n), key, null_rank, g))
    gs, ks, ns = g[perm], key[perm], null_rank[perm]
    seg = np.r_[True, gs[1:] != gs[:-1]]
    run = seg | np.r_[True, (ks[1:] != ks[:-1]) | (ns[1:] != ns[:-1])]
    return np.flatnonzero(run), np.flatnonzero(seg)


def head_places(heads):
    """where head positions fall inside k_rank_heads' layout: lane 0 / 31 of a word, first / last word of a warp's 8,
    first / last position of a tile (2048)"""
    h = np.asarray(heads, np.int64)
    return {"lane0": int((h % 32 == 0).sum()), "lane31": int((h % 32 == 31).sum()),
            "warp_first": int((h % RK_WARP == 0).sum()), "warp_last": int((h % RK_WARP == RK_WARP - 1).sum()),
            "tile_first": int((h % RK_TILE == 0).sum()), "tile_last": int((h % RK_TILE == RK_TILE - 1).sum())}


def labels_from_heads(n, heads):
    """one label per sorted position: the number of heads at or before it (position 0 is always a head)"""
    lab = np.zeros(n, np.int64)
    h = np.asarray([x for x in heads if 0 < x < n], np.int64)
    lab[h] = 1
    return np.cumsum(lab)


# ================================================================================================ rolling quantile
def rq_levels(n: int) -> int:
    """wm_build's L: the least L >= 1 with 2^L >= n"""
    L = 1
    while (1 << L) < n:
        L += 1
    return L


def rq_plan(n: int, nulls: bool):
    """the matrix one value column builds: L levels, k_wm_count / k_wm_split launches (one per level, plus the null
    bitvector), tiles per bitvector (n / 1792 + 1: the last holds position n)"""
    L = rq_levels(n)
    return {"L": L, "wm_count": L + int(nulls), "tiles": n // BV_TILE + 1}


def fixed_bounds(n, w, center=False):
    """the window [s, e) of every position of one partition (det_offsets / det_offsets_center, as op_rolling_quantile)"""
    L, R = w - 1, 1
    if center:
        R = w // 2 + (w & 1)
        L = w - R
    i = np.arange(n, dtype=np.int64)
    return np.maximum(i - min(L, n), 0), np.minimum(i + min(R, n), n)


def rq_edges(s, e, n):
    """how many windows start / end on a 224-position block edge, a 1792-position tile edge, and end at n on a tile edge"""
    s, e = np.asarray(s), np.asarray(e)
    return {"s_block": int(((s % BV_BITS == 0) & (s > 0)).sum()), "e_block": int(((e % BV_BITS == 0) & (e < n)).sum()),
            "s_tile": int(((s % BV_TILE == 0) & (s > 0)).sum()), "e_tile": int(((e % BV_TILE == 0) & (e < n)).sum()),
            "e_n_on_tile": int(((e == n) & (n % BV_TILE == 0)).sum())}


def q_index(m: int, q: float, method: str):
    """k_rq_out's (lo, hi) for m valid values, in f64: round half away from zero, ceil, floor, the EQUIPROBABLE clamp"""
    fi = (float(m) - 1.0) * q
    if method == "nearest":
        lo = math.floor(fi + 0.5) if fi >= 0 else 0
    elif method == "higher":
        lo = math.ceil(fi)
    elif method == "equiprobable":
        lo = int(max(math.ceil(float(m) * q) - 1.0, 0.0))
    else:
        lo = math.floor(fi)
    return min(lo, m - 1), math.ceil(fi), fi


def q_finish(x, y, lo, hi, fi, method, T):
    """the method's arithmetic in T (FinishLinear): y is read only when hi != lo"""
    if method not in ("midpoint", "linear") or hi == lo:
        return T(x)
    with np.errstate(all="ignore"):
        if method == "midpoint":
            return T((T(x) + T(y)) / T(2))
        return T(T(fi - float(lo)) * (T(y) - T(x)) + T(x))


def rq_windows(x, valid, T, s, e):
    """every window's valid values as T, ordered (np.sort: an exact selection of every rank at once)"""
    x = np.asarray(x)
    ok = np.ones(len(x), bool) if valid is None else np.asarray(valid, bool)
    return [np.sort(x[a:b][ok[a:b]].astype(T)) for a, b in zip(s, e)]


def rq_pick(wins, T, q, method, min_samples):
    """the quantile of every window of rq_windows; null below max(min_samples, 1) valid values.  Returns (values as T,
    validity)."""
    vals = np.zeros(len(wins), T)
    good = np.zeros(len(wins), bool)
    for i, w in enumerate(wins):
        m = len(w)
        if m == 0 or m < min_samples:
            continue
        lo, hi, fi = q_index(m, q, method)
        vals[i] = q_finish(w[lo], w[hi] if hi < m else w[lo], lo, hi, fi, method, T)
        good[i] = True
    return vals, good


def rq_ref(x, valid, T, q, method, s, e, min_samples):
    """every position's quantile over the valid values of [s, e)"""
    return rq_pick(rq_windows(x, valid, T, s, e), T, q, method, min_samples)


def rq_monotone(v_at, q, method, s, e, T, xp=np):
    """the closed form over a column with no nulls whose value at row r is v_at(r), never decreasing: the k-th
    smallest of [s, e) is v_at(s + k).  xp: numpy or torch (s, e int64 arrays / tensors)."""
    m = e - s
    mf = m.to(xp.float64) if xp is not np else m.astype(np.float64)
    fi = (mf - 1.0) * q
    if method == "nearest":
        lo = xp.floor(fi + 0.5)
    elif method == "higher":
        lo = xp.ceil(fi)
    elif method == "equiprobable":
        lo = xp.clamp(xp.ceil(mf * q) - 1.0, min=0.0) if xp is not np else np.maximum(np.ceil(mf * q) - 1.0, 0.0)
    else:
        lo = xp.floor(fi)
    to_i = (lambda t: t.to(xp.int64)) if xp is not np else (lambda t: t.astype(np.int64))
    lo = xp.minimum(to_i(lo), m - 1)
    hi = to_i(xp.ceil(fi))
    x = v_at(s + lo)
    if method not in ("midpoint", "linear"):
        return x
    y = v_at(s + xp.minimum(hi, m - 1))
    if method == "midpoint":
        z = (x + y) / 2
    else:
        fr = fi - (lo.to(xp.float64) if xp is not np else lo.astype(np.float64))
        z = (fr.to(x.dtype) if xp is not np else fr.astype(x.dtype)) * (y - x) + x
    return xp.where(hi != lo, z, x)
