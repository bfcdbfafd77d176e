"""Reference restatements of the rolling quantile (bl_rolling_quantile / bl_rolling_quantile_by).

- window_quantile / rolling_quantile / rolling_quantile_over / rolling_quantile_by: per window, as the reference's
  QuantileWindow::get_agg / QuantileUpdate::quantile compute it (polars-compute/src/rolling/no_nulls/quantile.rs:55-105,
  nulls/quantile.rs:52-106, quantile_filter.rs:559-567, 610-671): the window's non-null values sorted by tot_cmp, the index
  in f64, the arithmetic in numpy float32 / float64 scalars.
- WaveletMatrix / numpy_rolling_quantile: the device's structure in numpy, built level by level, with the descent
  vectorised over all positions.  It is the fast reference where sorting every window is too slow.
"""
import math

import numpy as np

import rolling_oracle as ro
from rolling_by_oracle import window_values

METHODS = ["nearest", "lower", "higher", "midpoint", "linear", "equiprobable"]


def out_type(dtype: str):
    """to_float: Float32 stays Float32, every other numeric dtype becomes Float64"""
    return np.float32 if dtype == "float32" else np.float64


def tot_key(x):
    """tot_cmp as a sort key: NaN greatest, -0.0 == +0.0"""
    x = float(x)
    return (1, 0.0) if x != x else (0, x + 0.0)


def round_half_away(x: float) -> int:
    """f64::round of a non-negative x"""
    r = math.floor(x)
    return r + 1 if x - r >= 0.5 else r


def indices(m: int, q: float, method: str):
    """(lo, hi) of the method for m valid values; hi is None when only lo is read"""
    fi = (float(m) - 1.0) * q
    if method == "nearest":
        return min(round_half_away(fi), m - 1), None
    if method == "lower":
        return min(math.floor(fi), m - 1), None
    if method == "higher":
        return min(math.ceil(fi), m - 1), None
    if method == "equiprobable":
        return int(max(math.ceil(float(m) * q) - 1.0, 0.0)), None
    lo, hi = min(math.floor(fi), m - 1), math.ceil(fi)
    return lo, (hi if hi != lo else None)


def window_quantile(win, q: float, method: str, T):
    """the quantile of one window's non-null values (already converted to T); None for an empty window"""
    m = len(win)
    if m == 0:
        return None
    srt = sorted(win, key=tot_key)
    lo, hi = indices(m, q, method)
    x = T(srt[lo])
    if hi is None:
        return x
    y = T(srt[hi])
    with np.errstate(all="ignore"):
        if method == "midpoint":
            return T((x + y) / T(2))
        fi = (float(m) - 1.0) * q
        return T(T(fi - float(lo)) * (y - x) + x)      # no lo == hi guard: inf, inf -> NaN


def _to_T(values, valid, T):
    return [T(float(v)) if ok else None for v, ok in zip(values, valid)]


def rolling_quantile(values, valid, dtype, q, method, window_size, min_samples=None, center=False):
    """one partition: None where the window's non-null count is below max(min_samples, 1)"""
    T = out_type(dtype)
    ms = window_size if min_samples is None else min_samples
    vals = _to_T(values, valid, T)
    out = []
    for win in ro.exact_windows(vals, window_size, center):
        out.append(window_quantile(win, q, method, T) if len(win) >= max(ms, 1) else None)
    return out


def rolling_quantile_over(values, valid, dtype, groups, order=None, **kw):
    """rolling_quantile(...).over(groups, order_by=order): each partition in partition order, results back to the rows"""
    out = [None] * len(values)
    for rows in ro.partition_order(groups, order):
        res = rolling_quantile([values[r] for r in rows], [valid[r] for r in rows], dtype, **kw)
        for r, v in zip(rows, res):
            out[r] = v
    return out


def rolling_quantile_by(values, valid, dtype, by, by_valid, P, closed, q, method, min_samples=1, parts=()):
    """time windows: None for a null `by`, a window of fewer than min_samples rows, or fewer than max(min_samples, 1)
    non-null values (rolling_kernels/shared.rs:109-204, then is_valid)"""
    T = out_type(dtype)
    vals = _to_T(values, valid, T)
    wins = window_values(vals, valid, by, by_valid, P, closed, min_samples, parts)
    return [None if w is None or len(w) < max(min_samples, 1) else window_quantile(w, q, method, T) for w in wins]


# ---------------------------------------------------------------------------------------------------- wavelet matrix
def stable_ranks(values, valid):
    """rank of every row in the stable total order, nulls last (op_arg_sort with BL_SORT_NULLS_LAST)"""
    v = np.asarray(values)
    valid = np.asarray(valid, dtype=bool)
    if v.dtype.kind == "f":
        v = np.where(np.isnan(v), np.inf, v + 0.0)      # NaN above +inf below; ties broken by the NaN flag
        nan = np.isnan(np.asarray(values)).astype(np.int8)
        order = np.lexsort((np.arange(len(v)), v, nan, ~valid))
    else:
        order = np.lexsort((np.arange(len(v)), v, ~valid))
    ranks = np.empty(len(v), dtype=np.int64)
    ranks[order] = np.arange(len(v))
    return ranks, order


class WaveletMatrix:
    """levels[l]: the prefix count of zeros of level l's bits (rank0 at any position); Z[l]: its zero total"""

    def __init__(self, A):
        A = np.asarray(A, dtype=np.int64)
        n = len(A)
        self.L = max(1, int(n - 1).bit_length())
        self.levels, self.Z = [], []
        cur = A
        for l in range(self.L):
            b = ((cur >> (self.L - 1 - l)) & 1).astype(bool)
            self.levels.append(np.concatenate([[0], np.cumsum(~b)]).astype(np.int64))
            self.Z.append(int((~b).sum()))
            cur = np.concatenate([cur[~b], cur[b]])

    def kth(self, s, e, k):
        """the k-th smallest (0-based) of A[s:e] for arrays s, e, k"""
        s, e, k = (np.asarray(x, dtype=np.int64).copy() for x in (s, e, k))
        v = np.zeros_like(s)
        for l in range(self.L):
            zs, ze = self.levels[l][s], self.levels[l][e]
            z = ze - zs
            go0 = k < z
            s = np.where(go0, zs, self.Z[l] + s - zs)
            e = np.where(go0, ze, self.Z[l] + e - ze)
            k = np.where(go0, k, k - z)
            v |= (~go0).astype(np.int64) << (self.L - 1 - l)
        return v


def numpy_rolling_quantile(values, valid, dtype, q, method, s, e, min_samples, live=None):
    """every position of a column whose positions are its rows: window [s, e); live = False where the output is null
    beforehand (a time window below min_samples rows or a null `by`).  Returns (out values as T, validity)."""
    T = out_type(dtype)
    valid = np.ones(len(values), dtype=bool) if valid is None else np.asarray(valid, dtype=bool)
    ranks, order = stable_ranks(values, valid)
    V = np.asarray(values)[order].astype(T)      # integers: numpy's int -> float64 rounds to nearest, as the device's cast
    wm = WaveletMatrix(ranks)
    s = np.asarray(s, dtype=np.int64)
    e = np.asarray(e, dtype=np.int64)
    cv = np.concatenate([[0], np.cumsum(valid)])
    m = cv[e] - cv[s]
    ok = (m >= max(min_samples, 1)) & (True if live is None else np.asarray(live, dtype=bool))
    mm = np.where(ok, m, 1)
    fi = (mm.astype(np.float64) - 1.0) * q
    fl = np.floor(fi).astype(np.int64)
    ce = np.ceil(fi).astype(np.int64)
    if method == "nearest":
        lo = np.minimum(np.where(fi - fl >= 0.5, fl + 1, fl), mm - 1)
    elif method == "higher":
        lo = np.minimum(ce, mm - 1)
    elif method == "equiprobable":
        lo = np.maximum(np.ceil(mm.astype(np.float64) * q) - 1.0, 0.0).astype(np.int64)
    else:
        lo = np.minimum(fl, mm - 1)
    x = V[wm.kth(np.where(ok, s, 0), np.where(ok, e, 1), np.where(ok, lo, 0))]
    if method in ("midpoint", "linear"):
        two = ok & (ce != lo)
        y = V[wm.kth(np.where(two, s, 0), np.where(two, e, 1), np.where(two, ce, 0))]
        with np.errstate(all="ignore"):
            if method == "midpoint":
                z = (x + y) / T(2)
            else:
                z = (fi - lo.astype(np.float64)).astype(T) * (y - x) + x
        x = np.where(two, z, x)
    return np.where(ok, x, T(0)).astype(T), ok
