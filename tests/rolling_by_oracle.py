"""CPU restatement of the reference's time-based rolling windows (rolling_*_by) and of the decomposition bl_rolling_by uses.

- `ref_windows`: group_by_values_iter_lookbehind (polars-time/src/windows/group_by.rs:247-326) literally, with its duplicate
  fast path and the i64 wrapping of t - P (Duration::add_*, duration.rs:929-1045).
- `bs_windows`: the closed-form bounds k_rollby_bounds computes by binary search.
- `decompose`: the window reduction of k_rollby_out with the block / sub-block sizes as parameters, over any associative
  combine (tests use tuple concatenation, which shows every window comes out as exactly its positions, in order).
- `window_values`: the reference's rows and windows (min_samples on the window length, nulls included; by-null rows null),
  for the kinds' exact window values of rolling_oracle.
"""
from __future__ import annotations

import numpy as np

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
CLOSED = ("right", "left", "both", "none")


def wrap64(x: int) -> int:
    return (x + (1 << 63)) % (1 << 64) - (1 << 63)


def _entry(t, lb, closed):
    return t > lb if closed in ("right", "none") else t >= lb


def _exit(t, ub, closed):
    return t <= ub if closed in ("right", "both") else t < ub


def ref_windows(times, P, closed):
    """(start, end) per position of one sorted segment, as the reference's iterator yields them (start_offset = 0)."""
    out = []
    start = end = 0
    last = times[0] if times else None
    for i, t in enumerate(times):
        if t == last and i > 0:
            out.append((start, end))
            continue
        last = t
        lb = wrap64(t - P)
        while start < i and not _entry(times[start], lb, closed):
            start += 1
        if _exit(t, t, closed):
            end = i
        else:
            end = max(end, start)
        while end < len(times) and _exit(times[end], t, closed):
            end += 1
        out.append((start, end))
    return out


def _first(times, lo, hi, pred):
    while lo < hi:
        m = (lo + hi) // 2
        if pred(times[m]):
            hi = m
        else:
            lo = m + 1
    return lo


def bs_windows(times, P, closed):
    """The bounds of k_rollby_bounds: binary searches inside the segment (see its comment)."""
    n = len(times)
    thr = I64_MIN + P
    incl = closed in ("left", "both")
    out = []
    for p, t in enumerate(times):
        lb = wrap64(t - P)
        if t < thr:
            s = _first(times, 0, p + 1, lambda u: u >= t)
        else:
            s = _first(times, 0, p + 1, (lambda u: u >= lb) if incl else (lambda u: u > lb))
            if times[0] < thr:
                x = _first(times, 0, p, lambda u: u >= thr)
                tw = times[x - 1]
                s = max(s, _first(times, 0, x, lambda u: u >= tw))
        if closed in ("right", "both"):
            e = _first(times, p + 1, n, lambda u: u > t)
        else:
            e = _first(times, 0, p + 1, lambda u: u >= t)
        out.append((s, e))
    return out


def decompose(s, e, seg, n, B, SUB, lift, combine):
    """Window [s, e) (non-empty, inside one segment) as k_rollby_out reduces it: across blocks of B through prefix / suffix /
    table; inside one block through the same structure over sub-blocks of SUB (k_rollby_out's shared-memory form and
    window_global's fold give the same runs)."""
    def head(p):
        return p == 0 or seg[p - 1] != seg[p]

    def end(q):      # q is one past a position: a segment end
        return q == n or seg[q] != seg[q - 1]

    def pre(p, size):      # from max(block start, segment head) to p
        a = p
        while a % size and not head(a):
            a -= 1
        return fold(a, p + 1)

    def suf(p, size):      # from p to min(block end, segment end)
        b = p + 1
        while b % size and not end(b):
            b += 1
        return fold(p, b)

    def fold(a, b):
        st = None
        for q in range(a, b):
            st = lift(q) if st is None else combine(st, lift(q))
        return st

    def table(l, r, size):      # the disjoint sparse table over the totals of blocks l..r of `size` positions
        tot = lambda k: fold(k * size, min(n, (k + 1) * size))
        if l == r:
            return tot(l)
        k = (l ^ r).bit_length() - 1
        g = 1 << k
        left = fold(l * size, (l // g + 1) * g * size)      # the suffix of l inside its group of 2^k blocks
        right = fold((r // g) * g * size, min(n, (r + 1) * size))
        return combine(left, right)

    bs, be = s // B, (e - 1) // B
    if bs < be:
        st = suf(s, B)
        if be - bs > 1:
            st = combine(st, table(bs + 1, be - 1, B))
        return combine(st, pre(e - 1, B))
    sl, sr = s // SUB, (e - 1) // SUB
    if sl < sr:
        st = suf(s, SUB)
        if sr - sl > 1:
            st = combine(st, table(sl + 1, sr - 1, SUB))
        return combine(st, pre(e - 1, SUB))
    if s % SUB == 0 or head(s):
        return pre(e - 1, SUB)
    if e % SUB == 0 or end(e):
        return suf(s, SUB)
    return fold(s, e)


def order_of(by, by_valid, parts):
    """The position order: partitions in first-occurrence order, times ascending (stable), null times last."""
    n = len(by)
    gid = {}
    g = [gid.setdefault(k, len(gid)) for k in (zip(*parts) if parts else [()] * n)]
    perm = sorted(range(n), key=lambda r: (g[r], not by_valid[r], by[r] if by_valid[r] else 0, r))
    return perm, [g[r] for r in perm]


def windows_of(by, by_valid, parts, P, closed):
    """Row -> (start, end) of its window in the position order (None: null `by`), plus that order."""
    perm, seg = order_of(by, by_valid, parts)
    win = [None] * len(by)
    lo = 0
    while lo < len(perm):
        hi = lo
        while hi < len(perm) and seg[hi] == seg[lo]:
            hi += 1
        valid = [p for p in range(lo, hi) if by_valid[perm[p]]]
        ts = [int(by[perm[p]]) for p in valid]
        if ts:
            for k, (s, e) in enumerate(ref_windows(ts, P, closed)):
                win[perm[valid[k]]] = (lo + s, lo + e)
        lo = hi
    return win, perm


def window_values(values, valid, by, by_valid, P, closed, min_samples, parts=()):
    """Per row: None when the output is null before the kind's own rule (a null `by`, or a window of fewer than
    min_samples rows, nulls included), else the window's non-null values in position order."""
    win, perm = windows_of(by, by_valid, parts, P, closed)
    out = []
    for r in range(len(by)):
        w = win[r]
        if w is None or w[1] - w[0] < min_samples:
            out.append(None)
        else:
            out.append([values[perm[p]] for p in range(w[0], w[1]) if valid[perm[p]]])
    return out


def numpy_sum_by(values, times, P, closed):
    """Integer rolling_sum_by of a sorted, non-null, unpartitioned column: searchsorted bounds and wrapping int64 prefix
    sums (a restatement for large sizes; no wrapping of t - P: the caller keeps times far from i64::MIN)."""
    t = np.asarray(times, dtype=np.int64)
    lb = t - np.int64(P)
    s = np.searchsorted(t, lb, side="left" if closed in ("left", "both") else "right")
    e = np.searchsorted(t, t, side="right" if closed in ("right", "both") else "left")
    c = np.concatenate([[0], np.cumsum(np.asarray(values, dtype=np.int64))])
    return c[e] - c[s], s, e


def replay_by(kind, dtype, values, valid, by, by_valid, P, closed, min_samples, ddof=1, parts=()):
    """The reference's window machines (rolling_oracle.SumWindow / MomentWindow) driven over the time-based windows, as
    rolling_apply_agg_window does (rolling_kernels/shared.rs:109-204): a window of fewer than min_samples rows is null and
    `update` is not called for it.  One machine per partition.  Float SUM / MEAN / VAR / STD; None for a null output."""
    import rolling_oracle as ro
    win, perm = windows_of(by, by_valid, parts, P, closed)
    _, seg = order_of(by, by_valid, parts)
    T = np.float32 if dtype == "float32" else float
    vals = [T(values[r]) if valid[r] else None for r in perm]
    out = [None] * len(by)
    machine, cur = None, None
    for p, r in enumerate(perm):
        if seg[p] != cur:
            cur = seg[p]
            if kind == "rolling_sum":
                machine = ro.SumWindow(vals, T, True)
            elif kind == "rolling_mean":
                machine = ro.SumWindow(vals, float, True)
            else:
                machine = ro.MomentWindow(vals, ddof)
            machine.start = machine.end = p
        w = win[r]
        if w is None or w[1] - w[0] < min_samples:
            continue
        machine.update(*w)
        cnt = machine.count()
        if kind == "rolling_sum":
            v = machine.get_sum(T)
        elif kind == "rolling_mean":
            v = None if cnt == 0 else machine.get_sum(T) / T(cnt)
        else:
            v = machine.get()
            if v is not None:
                v = T(v)
                if kind == "rolling_std":
                    v = T(np.sqrt(v)) if T is np.float32 else float(np.sqrt(v))
        out[r] = v if v is not None and cnt >= min_samples else None
    return out
