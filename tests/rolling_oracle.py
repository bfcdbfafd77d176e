"""A literal Python restatement of the reference's fixed-window rolling machinery (polars-compute/src/rolling).

Values are lists with None for a null.  `dtype` is the value dtype after the reference's casts ("float32", "float64" or an
integer dtype name); integer sums wrap in that dtype.  Float32 arithmetic is numpy float32, Float64 is Python float.
Also: the exact evaluator (fractions) the GPU bound checks compare against, and the van Herk decomposition the device uses.
"""
from __future__ import annotations

import math
from collections import deque
from fractions import Fraction

import numpy as np

INT_BITS = {"int32": (32, True), "uint32": (32, False), "int64": (64, True), "uint64": (64, False)}


def wrap(v: int, dtype: str) -> int:
    bits, signed = INT_BITS[dtype]
    v &= (1 << bits) - 1
    return v - (1 << bits) if signed and v >> (bits - 1) else v


def det_offsets(i, w, n):                      # rolling/mod.rs:72-77
    if w == 0:
        return i, i
    return max(i - (w - 1), 0), i + 1


def det_offsets_center(i, w, n):               # rolling/mod.rs:78-87
    if w == 0:
        return i, i
    right = -(-w // 2)
    return max(i - (w - right), 0), min(n, i + right)


def _isfinite(x):
    return math.isfinite(float(x))


class SumWindow:
    """rolling/sum.rs: Kahan add / sub of finite values in the accumulator type K, non-finite counters, reset."""

    def __init__(self, vals, K, is_float):
        self.vals, self.K, self.is_float = vals, K, is_float
        self.start = self.end = 0
        self.reset()

    def reset(self):
        self.sum = self.K(0)
        self.err_add = self.K(0)
        self.err_sub = self.K(0)
        self.nf = self.pinf = self.ninf = self.null_count = 0

    def add(self, v):
        if self.is_float:
            if _isfinite(v):
                y = self.K(v) - self.err_add
                ns = self.sum + y
                self.err_add = (ns - self.sum) - y
                self.sum = ns
            else:
                self.nf += 1
                self.pinf += v > 0
                self.ninf += v < 0
        else:
            self.sum += v

    def sub(self, v):
        if self.is_float:
            if _isfinite(v):
                y = self.K(type(v)(0) - v) - self.err_sub
                ns = self.sum + y
                self.err_sub = (ns - self.sum) - y
                self.sum = ns
            else:
                self.nf -= 1
                self.pinf -= v > 0
                self.ninf -= v < 0
        else:
            self.sum -= v

    def update(self, s, e):
        if s >= self.end:
            self.reset()
            self.start = self.end = s
        for i in range(self.start, s):
            if self.vals[i] is None:
                self.null_count -= 1
            else:
                self.sub(self.vals[i])
        for i in range(self.end, e):
            if self.vals[i] is None:
                self.null_count += 1
            else:
                self.add(self.vals[i])
        self.start, self.end = s, e

    def get_sum(self, T):
        if self.nf == 0:
            return T(self.sum)
        if self.nf == self.pinf:
            return T(math.inf)
        if self.nf == self.ninf:
            return T(-math.inf)
        return T(math.nan)

    def count(self):
        return (self.end - self.start) - self.null_count


class ArgMinMaxWindow:
    """rolling/arg_min_max.rs: the monotonic deque; a new value pops the tail only when strictly better."""

    def __init__(self, vals, is_max):
        self.vals, self.is_max = vals, is_max
        self.idx = deque()
        self.nonnull = 0
        self.start = self.end = 0

    def better(self, a, b):                      # MinPropagateNan / MaxPropagateNan is_better (min_max.rs:155-186)
        an, bn = a != a, b != b
        if self.is_max:                          # nan_max_lt(b, a): NaN is the greatest
            return (an and not bn) or (not an and not bn and b < a)
        return (an and not bn) or (not an and not bn and a < b)      # nan_min_lt(a, b): NaN is the least

    def update(self, s, e):
        while self.idx and self.idx[0] < s:
            self.idx.popleft()
        for i in range(self.start, min(s, self.end)):
            self.nonnull -= self.vals[i] is not None
        for i in range(max(s, self.end), e):
            if self.vals[i] is not None:
                while self.idx and self.better(self.vals[i], self.vals[self.idx[-1]]):
                    self.idx.pop()
                self.idx.append(i)
                self.nonnull += 1
        self.start, self.end = s, e

    def get(self):
        return self.vals[self.idx[0]] if self.idx else None

    def count(self):
        return self.nonnull


class VarState:
    """polars-compute/src/moment.rs:90-129"""

    def __init__(self, weight=0.0, mean=0.0, dp=0.0):
        self.weight, self.mean, self.dp = weight, mean, dp

    def copy(self):
        return VarState(self.weight, self.mean, self.dp)

    def insert_one(self, x):
        nw = self.weight + 1.0
        dm = x - self.mean
        nm = self.mean + dm / nw
        self.dp += (x - nm) * dm
        self.weight, self.mean = nw, nm
        if self.weight == 0.0:
            self.mean = self.dp = 0.0

    def combine(self, o):
        if o.weight == 0.0:
            return
        nw = self.weight + o.weight
        frac = o.weight / nw
        dm = o.mean - self.mean
        nm = self.mean + dm * frac
        self.dp += o.dp + o.weight * (o.mean - nm) * dm
        self.weight, self.mean = nw, nm
        if self.weight == 0.0:
            self.mean = self.dp = 0.0

    def finalize(self, ddof):
        if self.weight <= ddof:
            return None
        var = self.dp / (self.weight - ddof)
        return 0.0 if var < 0.0 else var


class MomentWindow:
    """rolling/moment.rs: a queue of two stacks (front: suffix states, back: values + agg_back) with flip."""

    def __init__(self, vals, ddof):
        self.vals, self.ddof = vals, ddof
        self.start = self.end = 0
        self.reset()

    def reset(self):
        self.nf = self.null_count = 0
        self.front, self.back = [], []
        self.agg_back = VarState()

    def push(self, v):
        x = float(v)
        if math.isfinite(x):
            self.back.append(x)
            self.agg_back.insert_one(x)
        else:
            self.back.append(0.0)
            self.agg_back.insert_one(0.0)
            self.nf += 1

    def pop(self, v):
        if not self.front:
            agg = VarState()
            while self.back:
                agg.insert_one(self.back.pop())
                self.front.append(agg.copy())
            self.agg_back = VarState()
        self.front.pop()
        self.nf -= not math.isfinite(float(v))

    def update(self, s, e):
        if s >= self.end:
            self.reset()
            self.start = self.end = s
        for i in range(self.start, s):
            if self.vals[i] is None:
                self.null_count -= 1
            else:
                self.pop(self.vals[i])
        for i in range(self.end, e):
            if self.vals[i] is None:
                self.null_count += 1
            else:
                self.push(self.vals[i])
        self.start, self.end = s, e

    def get(self):
        st = self.agg_back.copy()
        if self.front:
            st.combine(self.front[-1])
        v = st.finalize(self.ddof)
        if v is None:
            return None
        return math.nan if self.nf > 0 else v

    def count(self):
        return (self.end - self.start) - self.null_count


def out_dtype(kind, dtype):
    if kind == "rolling_sum":
        return "uint32" if dtype == "bool" else ("int64" if dtype in ("int8", "int16", "uint8", "uint16") else dtype)
    if kind in ("rolling_min", "rolling_max"):
        return dtype
    return "float32" if dtype == "float32" else "float64"


def rolling(kind, values, dtype, window_size, min_samples=None, center=False, ddof=1, counts=False):
    """One partition, the nulls path (rolling_apply_agg_window, nulls/mod.rs:46-98); the no-nulls path gives the same
    values and validity.  Returns a list with None for a null output (counts: also the non-null count of every window,
    which is what is_valid compares with min_samples)."""
    if min_samples is None:
        min_samples = window_size
    assert 0 <= min_samples <= window_size
    n = len(values)
    offs = det_offsets_center if center else det_offsets
    is_float = dtype in ("float32", "float64")
    if kind == "rolling_sum":
        if dtype == "bool":
            vals, odt = [None if v is None else int(bool(v)) for v in values], "uint32"
        else:
            odt = out_dtype(kind, dtype)
            vals = [None if v is None else (np.float32(v) if dtype == "float32" else float(v) if is_float else int(v)) for v in values]
        K = np.float32 if dtype == "float32" else float if is_float else int
        win = SumWindow(vals, K, is_float)
    elif kind == "rolling_mean":
        T = np.float32 if dtype == "float32" else float
        vals = [None if v is None else T(v) for v in values]
        win = SumWindow(vals, float, True)
    elif kind in ("rolling_min", "rolling_max"):
        vals = [None if v is None else (np.float32(v) if dtype == "float32" else float(v) if is_float else int(v)) for v in values]
        win = ArgMinMaxWindow(vals, kind == "rolling_max")
    else:
        T = np.float32 if dtype == "float32" else float
        vals = [None if v is None else T(v) for v in values]
        win = MomentWindow(vals, ddof)
    out, cnts = [], []
    for i in range(n):
        s, e = offs(i, window_size, n)
        win.update(s, e)
        cnt = win.count()
        cnts.append(cnt)
        if kind == "rolling_sum":
            v = win.get_sum(K) if is_float else wrap(win.sum, odt)
        elif kind == "rolling_mean":
            v = None if cnt == 0 else win.get_sum(T) / T(cnt)
        elif kind in ("rolling_min", "rolling_max"):
            v = win.get()
        else:
            v = win.get()
            if v is not None:
                v = T(v)
                if kind == "rolling_std":
                    v = T(np.sqrt(v)) if T is np.float32 else math.sqrt(v)
        out.append(v if v is not None and cnt >= min_samples else None)
    return (out, cnts) if counts else out


def partition_order(groups, order=None):
    """rows of each partition (first-occurrence order of the groups), stably sorted by `order` (ascending) inside it"""
    first = {}
    for r, g in enumerate(groups):
        first.setdefault(g, []).append(r)
    parts = list(first.values())
    if order is not None:
        parts = [sorted(p, key=lambda r: order[r]) for p in parts]
    return parts


def rolling_over(kind, values, dtype, groups, order=None, **kw):
    """rolling_*(...).over(groups, order_by=order): each partition rolled in partition order, results back to the rows"""
    out = [None] * len(values)
    for rows in partition_order(groups, order):
        res = rolling(kind, [values[r] for r in rows], dtype, **kw)
        for r, v in zip(rows, res):
            out[r] = v
    return out


# ---------------------------------------------------------------------------------------------------- exact evaluator
def exact_windows(values, window_size, center=False, segments=None):
    """for every position: the list of non-null values of its window (segments: [(lo, hi)], default the whole list)"""
    n = len(values)
    segments = segments or [(0, n)]
    offs = det_offsets_center if center else det_offsets
    res = [None] * n
    for lo, hi in segments:
        for i in range(lo, hi):
            s, e = offs(i - lo, window_size, hi - lo)
            res[i] = [v for v in values[lo + s: lo + e] if v is not None]
    return res


def exact_moments(xs):
    """(k, sum, M2) of the window exactly: every float is an integer over a power of two, so with one common scale the sums
    of x and x^2 are exact big integers and M2 = (k sum x^2 - (sum x)^2) / k"""
    ratios = [float(x).as_integer_ratio() for x in xs]
    e = max((d.bit_length() - 1 for _, d in ratios), default=0)
    ints = [m << (e - (d.bit_length() - 1)) for m, d in ratios]
    k, s1 = len(ints), sum(ints)
    s2 = sum(i * i for i in ints)
    return k, Fraction(s1, 1 << e), (Fraction(k * s2 - s1 * s1, k << (2 * e)) if k else Fraction(0))


def exact_sum(xs):
    return exact_moments(xs)[1]


def exact_var(xs, ddof):
    k, _, m2 = exact_moments(xs)
    return None if k <= ddof else m2 / (k - ddof)


U64 = 2.0 ** -53


def sum_bound(xs, u_out):
    """the header's SUM bound against the exact window value"""
    k = len(xs)
    return 1.01 * max(k - 1, 0) * U64 * math.fsum(abs(float(x)) for x in xs) + u_out * abs(float(exact_sum(xs)))


def mean_bound(xs, u_out):
    k = len(xs)
    s = exact_sum(xs)
    return (1.01 * max(k - 1, 0) * U64 * math.fsum(abs(float(x)) for x in xs) + u_out * abs(float(s))) / k + 2 * u_out * abs(float(s / k))


def var_bound(xs, ddof, u_out):
    """the header's VAR bound: 4.04 (k + 2) u M2 (1 + k mean^2 / M2)^(1/2) / (k - ddof) + u_o |exact|"""
    k, s, m2 = exact_moments(xs)
    m2f, mean = float(m2), float(s / k)
    kappa = math.sqrt(1 + k * mean * mean / m2f) if m2f > 0 else 1.0
    return 4.04 * (k + 2) * U64 * m2f * kappa / (k - ddof) + u_out * float(m2 / (k - ddof))


# ---------------------------------------------------------------------------------------------------- the device's decomposition
def decomposed(values, window_size, center, segments, lift, combine, empty):
    """van Herk / Gil-Werman as the device evaluates it: blocks of B = min(w, n) positions from position 0, prefixes
    restarted at block starts and segment heads, suffixes at block ends and segment ends; the window of position i is
    suffix[s] (+) prefix[l] when it spans two blocks, else prefix[l] when s == max(block start, segment head), else suffix[s]."""
    n = len(values)
    if n == 0:
        return []
    B = min(window_size, n)
    seg_of = [0] * n
    for k, (lo, hi) in enumerate(segments):
        for p in range(lo, hi):
            seg_of[p] = k
    lifted = [empty if v is None else lift(v) for v in values]
    pre, suf = [None] * n, [None] * n
    for p in range(n):
        head = p % B == 0 or seg_of[p] != seg_of[p - 1]
        pre[p] = lifted[p] if head else combine(pre[p - 1], lifted[p])
    for p in range(n - 1, -1, -1):
        tail = (p + 1) % B == 0 or p == n - 1 or seg_of[p] != seg_of[p + 1]
        suf[p] = lifted[p] if tail else combine(lifted[p], suf[p + 1])
    right = -(-window_size // 2)
    L, R = (window_size - right, right) if center else (window_size - 1, 1)
    out = []
    for i in range(n):
        lo, hi = segments[seg_of[i]]
        s, l = max(i - L, lo), min(i + R, hi) - 1
        b = l - l % B
        if s < b:
            out.append(combine(suf[s], pre[l]))
        elif s == max(b, lo):
            out.append(pre[l])
        else:
            out.append(suf[s])
    return out
