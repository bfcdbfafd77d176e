"""CPU oracle of the asof join (bl_join_asof), in two independent forms.

`cursor_asof` / `cursor_asof_by` restate the reference literally (paths relative to crates/polars-ops/src/frame/join/asof):
the three cursor states (mod.rs:47-200), join_asof_impl with its all-null early exit and the tolerance filter
(default.rs:12-145), and one cursor per right group with `by` keys (groups.rs:39-160).  Values are numpy scalars of the key
dtype, so float differences round in that dtype; integer differences are exact (abs_diff).

`rule_asof` is the per-row rule the device computes (include/polars_b200.h, bl_join_asof), vectorised with searchsorted over
total-order keys.  It is only valid under the precondition, which `precondition_ok` checks.

A side is a list of values with None for a null (small inputs) or a (numpy values, valid | None) pair (rule_asof).
"""
from __future__ import annotations

import numpy as np

BACKWARD, FORWARD, NEAREST = "backward", "forward", "nearest"


# ---------------------------------------------------------------------------------------------------- scalar semantics
def _is_float(x) -> bool:
    return isinstance(x, (float, np.floating))


def tot_key(x):
    """tot_cmp (polars-utils/src/total_ord.rs): NaN greatest and equal to itself, -0.0 == +0.0"""
    if _is_float(x):
        return (1, 0.0) if x != x else (0, float(x))
    return (0, int(x))


def abs_diff(a, b):
    """polars-utils/src/abs_diff.rs: integers exact (unsigned), floats `a > b ? a - b : b - a` in their own dtype"""
    if _is_float(a):
        with np.errstate(invalid="ignore"):
            return a - b if a > b else b - a
    return abs(int(a) - int(b))


def _tot_cmp(a, b) -> int:
    ka, kb = tot_key(a), tot_key(b)
    return (ka > kb) - (ka < kb)


# ---------------------------------------------------------------------------------------------------- the cursors
class Forward:
    def __init__(self, allow_eq):
        self.scan, self.allow_eq = 0, allow_eq

    def next(self, l, right):
        while self.scan < len(right):
            r = right[self.scan]
            if r is not None:
                c = _tot_cmp(r, l)              # ge_allow_eq(right_val, left_val)
                if c > 0 or (c == 0 and self.allow_eq):
                    return self.scan
            self.scan += 1
        return None


class Backward:
    def __init__(self, allow_eq):
        self.best, self.scan, self.allow_eq = None, 0, allow_eq

    def next(self, l, right):
        while self.scan < len(right):
            r = right[self.scan]
            if r is not None:
                c = _tot_cmp(r, l)              # lt_allow_eq(right_val, left_val)
                if c < 0 or (c == 0 and self.allow_eq):
                    self.best = self.scan
                else:
                    break
            self.scan += 1
        return self.best


class Nearest:
    def __init__(self, allow_eq):
        self.smaller, self.upper, self.allow_eq = None, 0, allow_eq

    def next(self, l, right):
        n = len(right)
        while self.upper < n:
            r = right[self.upper]
            if r is None:
                self.upper += 1
                continue
            if r > l:
                break
            self.upper += 1
        if self.allow_eq and self.upper > 0:
            r = right[self.upper - 1]
            if r is not None and r == l:
                return self.upper - 1

        def eq_opt(a, b):                       # Option<T> == Option<T>
            return (a is None and b is None) or (a is not None and b is not None and a == b)
        while self.upper + 1 < n and eq_opt(right[self.upper + 1], right[self.upper]):
            self.upper += 1
        cursor = self.smaller if self.smaller is not None else 0
        while cursor < self.upper:
            r = right[cursor]
            if r is None:
                cursor += 1
                continue
            if r >= l:
                break
            self.smaller = cursor
            cursor += 1

        def get(i):
            return right[i] if (i is not None and i < n) else None
        lo, hi = get(self.smaller), get(self.upper)
        if lo is None and hi is None:
            return None
        if hi is None:
            return self.smaller
        if lo is None:
            return self.upper
        return self.upper if abs_diff(l, hi) <= abs_diff(l, lo) else self.smaller


STATES = {BACKWARD: Backward, FORWARD: Forward, NEAREST: Nearest}


def _filter(tol):
    if tol is None:
        return lambda l, r: True
    at = abs_diff(tol, type(tol)(0))
    return lambda l, r: abs_diff(l, r) <= at


def cursor_asof(left, right, strategy, allow_eq=True, tol=None):
    """join_asof_impl (default.rs:12-69): -> list of right row indices / None"""
    if all(v is None for v in left) or all(v is None for v in right):
        return [None] * len(left)
    st, keep = STATES[strategy](allow_eq), _filter(tol)
    out = []
    for l in left:
        j = None if l is None else st.next(l, right)
        out.append(j if (j is not None and keep(l, right[j])) else None)
    return out


def _group_key(vals):
    """one row's `by` values -> a hashable key with floats canonicalised (-0 == +0, NaN == NaN); None when any is null"""
    if any(v is None for v in vals):
        return None
    return tuple(("nan",) if (_is_float(v) and v != v) else (float(v) + 0.0 if _is_float(v) else v) for v in vals)


def cursor_asof_by(left, right, left_by, right_by, strategy, allow_eq=True, tol=None):
    """asof_join_by_* + asof_in_group (groups.rs:39-160): left_by / right_by are lists of per-row tuples of `by` values"""
    groups = {}
    for j, k in enumerate(map(_group_key, right_by)):
        if k is not None:
            groups.setdefault(k, []).append(j)
    states, keep, out = {}, _filter(tol), []
    for l, lk in zip(left, map(_group_key, left_by)):
        if lk is None or l is None or lk not in groups:
            out.append(None)
            continue
        idxs = groups[lk]
        st = states.setdefault(lk, STATES[strategy](allow_eq))
        j = st.next(l, [right[i] for i in idxs])
        out.append(idxs[j] if (j is not None and keep(l, right[idxs[j]])) else None)
    return out


# ---------------------------------------------------------------------------------------------------- the per-row rule
def precondition_ok(left, right) -> bool:
    """non-null left values non-decreasing; right nulls first, then non-decreasing (total order)"""
    lv = [tot_key(v) for v in left if v is not None]
    if any(a > b for a, b in zip(lv, lv[1:])):
        return False
    z = 0
    while z < len(right) and right[z] is None:
        z += 1
    if any(v is None for v in right[z:]):
        return False
    rv = [tot_key(v) for v in right[z:]]
    return not any(a > b for a, b in zip(rv, rv[1:]))


def total_keys(values: np.ndarray) -> np.ndarray:
    """uint64 keys whose order is tot_cmp's (the device's AsofNum::key)"""
    v = np.asarray(values)
    if v.dtype.kind == "f":
        w = v.astype(np.float64) + 0.0
        bits = np.where(np.isnan(w), np.float64(np.nan), w).view(np.uint64)
        return np.where(bits >> np.uint64(63), ~bits, bits | np.uint64(1 << 63))
    if v.dtype.kind == "i":
        return v.astype(np.int64).view(np.uint64) ^ np.uint64(1 << 63)
    return v.astype(np.uint64)


def _diff(a, b):
    """abs_diff elementwise: floats in their dtype, integers exact as uint64"""
    if a.dtype.kind == "f":
        with np.errstate(invalid="ignore"):
            return np.where(a > b, a - b, b - a)
    ai, bi = a.astype(np.int64) if a.dtype.kind == "i" else a.astype(np.uint64), b.astype(np.int64) if b.dtype.kind == "i" else b.astype(np.uint64)
    au, bu = ai.view(np.uint64) if ai.dtype == np.int64 else ai, bi.view(np.uint64) if bi.dtype == np.int64 else bi
    return np.where(ai > bi, au - bu, bu - au)


def rule_segment(lv, rv, strategy, allow_eq, tol):
    """lv: non-null left values; rv: a sorted, null-free right segment -> positions in rv (-1 = none)"""
    n = len(rv)
    if n == 0 or len(lv) == 0:
        return np.full(len(lv), -1, np.int64)
    lk, rk = total_keys(lv), total_keys(rv)
    fl = rv.dtype.kind == "f"
    if strategy == BACKWARD:
        j = np.searchsorted(rk, lk, side="right" if allow_eq else "left") - 1
    elif strategy == FORWARD:
        j = np.searchsorted(rk, lk, side="left" if allow_eq else "right")
        j = np.where(j < n, j, -1)
    else:
        U = np.searchsorted(rk, lk, side="right")
        if fl:
            U = np.where((U < n) & np.isnan(rv[np.minimum(U, n - 1)]), n, U)
        prev = rv[np.maximum(U - 1, 0)]
        exact = (U > 0) & (prev == lv) if allow_eq else np.zeros(len(lv), bool)
        Ue = np.where(U < n, np.searchsorted(rk, rk[np.minimum(U, n - 1)], side="right") - 1, U)
        lb = np.minimum(np.searchsorted(rk, lk, side="left"), Ue)
        lb_ok = lb < Ue
        if fl:
            lb_ok &= ~np.isnan(rv[np.minimum(lb, n - 1)])
        L = np.where(lb_ok, lb - 1, Ue - 1)
        hasL, hasU = L >= 0, Ue < n
        dU = _diff(lv, rv[np.minimum(Ue, n - 1)])
        dL = _diff(lv, rv[np.maximum(L, 0)])
        with np.errstate(invalid="ignore"):
            both = np.where(dU <= dL, Ue, L)
        j = np.where(hasL & hasU, both, np.where(hasU, Ue, np.where(hasL, L, -1)))
        j = np.where(exact, U - 1, j)
    j = np.asarray(j, np.int64)
    if tol is not None:
        at = _diff(np.array([tol], rv.dtype), np.zeros(1, rv.dtype))[0]
        d = _diff(lv, rv[np.clip(j, 0, n - 1)])
        with np.errstate(invalid="ignore"):
            j = np.where((j >= 0) & (d <= at), j, -1)
    return j


def rule_asof(left, right, strategy, allow_eq=True, tol=None, left_groups=None, right_groups=None):
    """The per-row rule: left / right = (values, valid | None); *_groups: int64 group ids (-1 = null `by` key) or None.
    -> (uint32 index, bool valid)"""
    lv, lvalid = left
    rv, rvalid = right
    nl = len(lv)
    lvalid = np.ones(nl, bool) if lvalid is None else np.asarray(lvalid, bool)
    rvalid = np.ones(len(rv), bool) if rvalid is None else np.asarray(rvalid, bool)
    out = np.full(nl, -1, np.int64)
    if left_groups is None:
        z = int(np.argmax(rvalid)) if rvalid.any() else len(rv)
        rows = np.nonzero(lvalid)[0]
        j = rule_segment(lv[rows], rv[z:], strategy, allow_eq, tol)
        out[rows] = np.where(j >= 0, j + z, -1)
    else:
        rorder = np.argsort(right_groups, kind="stable")
        rgs = right_groups[rorder]
        lsel = np.nonzero((left_groups >= 0) & lvalid)[0]
        lorder = lsel[np.argsort(left_groups[lsel], kind="stable")]
        lgs = left_groups[lorder]
        for g in np.unique(lgs):
            seg = rorder[np.searchsorted(rgs, g, "left"):np.searchsorted(rgs, g, "right")]
            seg = seg[rvalid[seg]]
            if len(seg) == 0:
                continue
            rows = lorder[np.searchsorted(lgs, g, "left"):np.searchsorted(lgs, g, "right")]
            j = rule_segment(lv[rows], rv[seg], strategy, allow_eq, tol)
            out[rows] = np.where(j >= 0, seg[np.maximum(j, 0)], -1)
    valid = out >= 0
    return np.where(valid, out, 0xFFFFFFFF).astype(np.uint32), valid


def rule_lists(left, right, strategy, allow_eq=True, tol=None, dtype=None):
    """rule_asof on None-lists -> list of indices / None"""
    dt = np.dtype(dtype) if dtype is not None else np.asarray([v for v in left + right if v is not None] or [0]).dtype
    lv = np.array([0 if v is None else v for v in left], dt)
    rv = np.array([0 if v is None else v for v in right], dt)
    idx, valid = rule_asof((lv, np.array([v is not None for v in left], bool)), (rv, np.array([v is not None for v in right], bool)), strategy, allow_eq, tol)
    return [int(i) if ok else None for i, ok in zip(idx, valid)]
