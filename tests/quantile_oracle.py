"""Plain-Python restatement of the reference's per-group median / quantile over GroupsIdx (the CPU oracle of
BL_AGG_MEDIAN / BL_AGG_QUANTILE).

Reference: agg_quantile_generic / agg_median_generic (polars-core/src/frame/group_by/aggregations/mod.rs:297-408),
quantile_idx / linear_interpol / midpoint_interpol and generic_quantiles (chunked_array/ops/aggregate/quantile.rs:21-65,
:179-234), QuantileMethod (polars-compute/src/rolling/mod.rs:40-48).  Values go to f64 first; a Float32 column's result is
cast back to f32 (round to nearest); integer columns give Float64.  The value order is tot_cmp: NaN greatest, -0.0 == +0.0.
"""
from __future__ import annotations

import math

import numpy as np

METHODS = ("nearest", "lower", "higher", "midpoint", "linear", "equiprobable")


def rust_round(x: float) -> float:
    """f64::round: half away from zero (Python's round() and numpy's round half to even)"""
    f = math.floor(abs(x))
    r = f + 1.0 if abs(x) - f >= 0.5 else f
    return math.copysign(r, x)


def _tot_key(v: float):
    return (1, 0.0) if math.isnan(v) else (0, v + 0.0)


def quantile_idx(q: float, length: int, nulls: int, method: str):
    """quantile.rs:21-48 -> (idx, float_idx, top_idx)"""
    m = float(length - nulls)
    float_idx = (m - 1.0) * q + float(nulls)
    if method == "nearest":
        idx = int(rust_round(float_idx))
        return idx, 0.0, idx
    if method == "equiprobable":
        idx = int(max(math.ceil(m * q) - 1.0, 0.0)) + nulls
        return idx, 0.0, idx
    idx = int(math.ceil(float_idx)) if method == "higher" else int(float_idx)
    idx = min(max(idx, 0), length - 1)
    return idx, float_idx, int(math.ceil(float_idx))


def quantile_of(values, valid, q: float, method: str):
    """One group: `values` (Python numbers), `valid` (bools or None) -> float or None (generic_quantiles, quantile.rs:179-234)"""
    vals = [float(v) for v, ok in zip(values, valid if valid is not None else [True] * len(values)) if ok]
    nulls = len(values) - len(vals)
    if not vals:
        return None
    srt = [None] * nulls + sorted(vals, key=_tot_key)      # ca.sort(false): nulls first
    idx, float_idx, top = quantile_idx(q, len(srt), nulls, method)
    lower = srt[idx]
    if idx == top or method not in ("midpoint", "linear"):
        return lower
    upper = srt[idx + 1]
    if lower == upper:
        return lower
    if method == "midpoint":
        return (lower + upper) / 2.0
    return (float_idx - float(idx)) * (upper - lower) + lower


def group_tuples(keys):
    """GroupsIdx: groups in first-occurrence order, each group's rows ascending.  keys: a list of hashable per-row keys"""
    groups, order = {}, []
    for r, k in enumerate(keys):
        if isinstance(k, float) and math.isnan(k):
            k = ("nan",)
        elif isinstance(k, float) and k == 0.0:
            k = 0.0
        if k not in groups:
            groups[k] = []
            order.append(k)
        groups[k].append(r)
    return [groups[k] for k in order]


def group_quantile(keys, values: np.ndarray, valid, q: float, method: str = "nearest"):
    """Per-group quantile -> (numpy results in first-occurrence group order, validity).  Float32 in -> float32 out."""
    if not 0.0 <= q <= 1.0:
        raise ValueError("quantile should be between 0.0 and 1.0")
    if method not in METHODS:
        raise ValueError(f"unknown method {method}")
    out_dt = np.float32 if values.dtype == np.float32 else np.float64
    vl = values.tolist()
    res, ok = [], []
    for rows in group_tuples(keys):
        r = quantile_of([vl[i] for i in rows], None if valid is None else [bool(valid[i]) for i in rows], q, method)
        ok.append(r is not None)
        res.append(0.0 if r is None else r)
    return np.array(res, np.float64).astype(out_dt), np.array(ok, bool)


def group_median(keys, values, valid):
    return group_quantile(keys, values, valid, 0.5, "linear")


def numpy_group_quantile(gid: np.ndarray, values: np.ndarray, valid, q, method: str, n_groups: int):
    """Vectorised restatement for large inputs: gid = group id per row (0..n_groups-1).  One lexsort of (value, null-first,
    group), then the same index rule per group with numpy arithmetic in f64.  np.round is half-to-even, so nearest adds 1
    to floor(x) where x - floor(x) >= 0.5 (an exact subtraction), as rust_round does.  q may be a list: one sort, a
    (results, validity) pair per quantile."""
    n = values.shape[0]
    v = values.astype(np.float64)
    ok = np.ones(n, bool) if valid is None else np.asarray(valid, bool)
    # total order key: NaN greatest, -0.0 == +0.0 (the value itself otherwise); nulls first inside a group
    nan = np.isnan(v)
    order = np.lexsort((np.where(nan, 0.0, v + 0.0), nan, ok, gid))
    sv = v[order]
    counts = np.bincount(gid, minlength=n_groups).astype(np.int64)
    nulls = np.bincount(gid, weights=(~ok).astype(np.float64), minlength=n_groups).astype(np.int64)
    starts = np.concatenate(([0], np.cumsum(counts)[:-1]))
    out_dt = np.float32 if values.dtype == np.float32 else np.float64
    if isinstance(q, (list, tuple)):
        return [_numpy_picks(sv, n, counts, nulls, starts, qq, method, n_groups, out_dt) for qq in q]
    return _numpy_picks(sv, n, counts, nulls, starts, q, method, n_groups, out_dt)


def _numpy_picks(sv, n, counts, nulls, starts, q, method, n_groups, out_dt):
    m = (counts - nulls).astype(np.float64)
    has = m > 0
    float_idx = (m - 1.0) * q + nulls.astype(np.float64)
    if method == "nearest":
        fl = np.floor(float_idx)
        idx = (fl + (float_idx - fl >= 0.5)).astype(np.int64)
        top = idx
    elif method == "equiprobable":
        idx = np.maximum(np.ceil(m * q) - 1.0, 0.0).astype(np.int64) + nulls
        top = idx
    else:
        idx = (np.ceil(float_idx) if method == "higher" else np.trunc(float_idx)).astype(np.int64)
        idx = np.clip(idx, 0, np.maximum(counts - 1, 0))
        top = np.ceil(float_idx).astype(np.int64)
    safe = np.where(has, starts + idx, 0)
    lower = sv[np.minimum(safe, n - 1)] if n else np.zeros(n_groups)
    res = lower.copy()
    if method in ("midpoint", "linear"):
        interp = has & (idx != top)
        up_pos = np.minimum(np.where(interp, starts + idx + 1, 0), max(n - 1, 0))
        upper = sv[up_pos] if n else np.zeros(n_groups)
        with np.errstate(invalid="ignore"):
            if method == "midpoint":
                val = (lower + upper) / 2.0
            else:
                val = (float_idx - idx.astype(np.float64)) * (upper - lower) + lower
        res = np.where(interp & (lower != upper), val, lower)
    return np.where(has, res, 0.0).astype(out_dt), has
