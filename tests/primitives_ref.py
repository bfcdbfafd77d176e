"""Plain numpy / Python-int restatements of the streaming primitives K1 (elementwise arithmetic), K2 (compare),
K3 (filter), K4 (gather) and K6 (hash partition), plus the extreme-value inputs their tests use.

Test infrastructure only.  Except for the K6 partition function, nothing here calls oracle/, so the GPU results are
checked against a second, independent statement of each rule (tests/test_primitives_reference.py checks the two
statements against each other on the CPU).

Conventions: a validity is a numpy bool array (True = valid) or None (no nulls); a scalar operand is a numpy scalar of
the column's dtype.  Values in null slots are unspecified: compare them with `valid_equal`, which ignores them.

Rules restated:
  * integers are computed exactly and wrapped mod 2^w; floor division and modulo follow Python's floor semantics, so
    MIN // -1 wraps to MIN and MIN % -1 == 0.  For floordiv / mod only, an array divisor of 0 gives a null row and a
    scalar divisor of 0 makes every row null.  Integer true division is float64(a) / float64(b) (never null: division
    by 0 gives inf or NaN); with a scalar right-hand side it is float64(a) * (1.0 / float64(c)).
  * floats use one IEEE operation per source operation in the column's own dtype (no contraction, no flush to zero):
    sub with a scalar right-hand side is a + (-c); floordiv / mod / truediv with a scalar right-hand side multiply by
    the reciprocal: floor(a * (1/c)), a - c * floor(a * (1/c)), a * (1/c).
  * comparisons use the total order: NaN == NaN and NaN is the largest value; -0.0 == 0.0.  Nulls propagate, except
    for eq / ne with missing=True, where null == null and the result is never null.
  * filter keeps the rows whose mask bit is set and valid; gather is `take`, where a null index (a null slot or
    IDX_NULL) gives a null row holding 0.
  * K6 sends a row to hash_to_partition(dirty_hash(key_bits(key)), P); a null key goes to partition 0.
"""
from __future__ import annotations

import numpy as np

IDX_NULL = 0xFFFFFFFF
INT_DTYPES = ("int64", "int32", "uint64", "uint32")
FLOAT_DTYPES = ("float64", "float32")
DTYPES = INT_DTYPES + FLOAT_DTYPES
OPS = ("add", "sub", "mul", "floordiv", "mod", "truediv")
CMPS = ("eq", "ne", "lt", "le", "gt", "ge")
_UNSIGNED = {np.dtype("int64"): np.uint64, np.dtype("int32"): np.uint32, np.dtype("uint64"): np.uint64, np.dtype("uint32"): np.uint32,
             np.dtype("float64"): np.uint64, np.dtype("float32"): np.uint32}


def _and(a, b):
    if a is None:
        return None if b is None else np.asarray(b, bool)
    return np.asarray(a, bool) if b is None else (np.asarray(a, bool) & np.asarray(b, bool))


# ------------------------------------------------------------------ K1 elementwise
def int_exact(op: str, a: int, b: int, dtype) -> tuple[int | float, bool]:
    """One integer operation on Python ints, wrapped to the dtype's width -> (value, valid).  truediv -> a float."""
    dt = np.dtype(dtype)
    if op == "truediv":
        fa, fb = np.float64(a), np.float64(b)
        with np.errstate(all="ignore"):
            return float(fa / fb), True
    if op in ("floordiv", "mod") and b == 0:
        return 0, False
    r = {"add": lambda: a + b, "sub": lambda: a - b, "mul": lambda: a * b, "floordiv": lambda: a // b, "mod": lambda: a % b}[op]()
    w = 8 * dt.itemsize
    r &= (1 << w) - 1
    if dt.kind == "i" and r >= 1 << (w - 1):
        r -= 1 << w
    return r, True


def _int_floor_divmod(a: np.ndarray, b: np.ndarray, dt: np.dtype):
    """Vectorised floor division and modulo with the exact-then-wrap result; (0, 0) where b == 0."""
    zero = b == 0
    neg1 = (b == -1) if dt.kind == "i" else np.zeros(b.shape, bool)
    safe = np.where(zero | neg1, np.ones(1, dt), b)
    with np.errstate(all="ignore"):
        q = np.floor_divide(a, safe)
        r = np.remainder(a, safe)
    # x // -1 == -x (which wraps MIN to MIN) and x % -1 == 0
    q = np.where(neg1, (np.zeros(1, _UNSIGNED[dt]) - a.view(_UNSIGNED[dt])).view(dt), q)
    r = np.where(neg1, np.zeros(1, dt), r)
    return np.where(zero, np.zeros(1, dt), q).astype(dt), np.where(zero, np.zeros(1, dt), r).astype(dt)


def arith(op: str, lhs, rhs, lhs_valid=None, rhs_valid=None):
    """K1: lhs (op) rhs with at most one numpy scalar side -> (values, valid|None)."""
    l_scalar, r_scalar = np.ndim(lhs) == 0, np.ndim(rhs) == 0
    assert not (l_scalar and r_scalar)
    dt = np.asarray(rhs if l_scalar else lhs).dtype
    n = np.asarray(rhs if l_scalar else lhs).size
    a = np.full(n, lhs, dt) if l_scalar else np.asarray(lhs, dt)
    b = np.full(n, rhs, dt) if r_scalar else np.asarray(rhs, dt)
    valid = _and(None if l_scalar else lhs_valid, None if r_scalar else rhs_valid)
    if dt.kind == "f":
        with np.errstate(all="ignore"):
            if op == "add":
                out = a + b
            elif op == "sub":
                out = a + (-b) if r_scalar else a - b
            elif op == "mul":
                out = a * b
            else:
                inv = dt.type(1) / dt.type(rhs) if r_scalar else None
                q = a * inv if r_scalar else a / b
                if op == "truediv":
                    out = q
                elif op == "floordiv":
                    out = np.floor(q)
                else:
                    out = a - b * np.floor(q)
        return out.astype(dt), valid
    if op == "truediv":
        fa, fb = a.astype(np.float64), b.astype(np.float64)
        with np.errstate(all="ignore"):
            out = fa * (np.float64(1.0) / np.float64(rhs)) if r_scalar else fa / fb
        return out, valid
    if op in ("add", "sub", "mul"):
        u = _UNSIGNED[dt]
        ua, ub = a.view(u), b.view(u)
        out = (ua + ub) if op == "add" else (ua - ub) if op == "sub" else (ua * ub)
        return out.view(dt), valid
    q, r = _int_floor_divmod(a, b, dt)
    return (q if op == "floordiv" else r), _and(valid, b != 0)


# ------------------------------------------------------------------ K2 compare
def _tot_ge(a, b):
    if a.dtype.kind == "f":
        return np.isnan(a) | (a >= b)
    return a >= b


def _tot_eq(a, b):
    if a.dtype.kind == "f":
        return np.where(np.isnan(a), np.isnan(b), a == b)
    return a == b


def compare(op: str, lhs, rhs, lhs_valid=None, rhs_valid=None, missing: bool = False):
    """K2: lhs (op) rhs in the total order; rhs may be a numpy scalar -> (bool values, valid|None)."""
    a = np.asarray(lhs)
    n = a.size
    r_scalar = np.ndim(rhs) == 0
    b = np.full(n, rhs, a.dtype) if r_scalar else np.asarray(rhs, a.dtype)
    with np.errstate(invalid="ignore"):
        r = {"eq": lambda: _tot_eq(a, b), "ne": lambda: ~_tot_eq(a, b), "lt": lambda: ~_tot_ge(a, b), "le": lambda: _tot_ge(b, a),
             "gt": lambda: ~_tot_ge(b, a), "ge": lambda: _tot_ge(a, b)}[op]()
    rv = None if r_scalar else rhs_valid
    if missing and op in ("eq", "ne"):
        va = np.ones(n, bool) if lhs_valid is None else np.asarray(lhs_valid, bool)
        vb = np.ones(n, bool) if rv is None else np.asarray(rv, bool)
        both = va & vb
        alt = (va == vb) if op == "eq" else (va != vb)
        return np.where(both, r, alt), None
    return r, _and(lhs_valid, rv)


# ------------------------------------------------------------------ K3 filter, K4 gather
def filter(values, valid, mask, mask_valid=None):
    """K3: the rows whose mask slot is true and valid -> (values, valid|None)."""
    keep = np.asarray(mask, bool) if mask_valid is None else (np.asarray(mask, bool) & np.asarray(mask_valid, bool))
    return np.asarray(values)[keep], (None if valid is None else np.asarray(valid, bool)[keep])


def gather(values, valid, idx, idx_valid=None):
    """K4: take(values, idx); a null index slot or IDX_NULL gives a null row holding 0 -> (values, valid|None)."""
    values, idx = np.asarray(values), np.asarray(idx, np.uint32)
    null = idx == np.uint32(IDX_NULL)
    if idx_valid is not None:
        null |= ~np.asarray(idx_valid, bool)
    safe = np.where(null, 0, idx).astype(np.int64)
    out = np.where(null, np.zeros(1, values.dtype), values[safe] if values.size else np.zeros(idx.size, values.dtype))
    ov = ~null if valid is None else (~null & np.asarray(valid, bool)[safe])
    return out.astype(values.dtype), (None if (valid is None and not null.any()) else ov)


# ------------------------------------------------------------------ K6 hash partition
def partition_of(keys, valid, n_partitions: int) -> np.ndarray:
    """K6: the partition of every row.  The hash functions come from the oracle, whose KAT pins them to the reference."""
    import oracle
    p = oracle.hash_to_partition(oracle.dirty_hash(oracle.key_bits(np.asarray(keys))), n_partitions).astype(np.int64)
    if valid is not None:
        p[~np.asarray(valid, bool)] = 0
    return p


def partition_offsets(parts: np.ndarray, n_partitions: int) -> np.ndarray:
    """Start of every partition's range in the output, and the total at the end (n_partitions + 1 entries)."""
    return np.concatenate([[0], np.cumsum(np.bincount(parts, minlength=n_partitions))]).astype(np.int64)


# ------------------------------------------------------------------ comparison helpers
def valid_equal(got, got_valid, exp, exp_valid) -> str | None:
    """None when the validities agree and every valid slot holds the same bits (any NaN equals any NaN); otherwise a
    short description of the first difference."""
    got, exp = np.asarray(got), np.asarray(exp)
    if got.dtype != exp.dtype:
        return f"dtype {got.dtype} != {exp.dtype}"
    if got.shape != exp.shape:
        return f"length {got.shape} != {exp.shape}"
    gv = np.ones(got.shape, bool) if got_valid is None else np.asarray(got_valid, bool)
    ev = np.ones(exp.shape, bool) if exp_valid is None else np.asarray(exp_valid, bool)
    if not np.array_equal(gv, ev):
        i = int(np.nonzero(gv != ev)[0][0])
        return f"validity differs at row {i}: got {gv[i]} expected {ev[i]} ({int((gv != ev).sum())} rows)"
    if exp.dtype == np.bool_:
        bad = ev & (got != exp)
    else:
        u = _UNSIGNED[exp.dtype]
        bad = ev & (got.view(u) != exp.view(u))
        if exp.dtype.kind == "f":
            bad &= ~(np.isnan(got) & np.isnan(exp))
    if bad.any():
        i = int(np.nonzero(bad)[0][0])
        return f"{int(bad.sum())} values differ, first at row {i}: got {got[i]!r} expected {exp[i]!r}"
    return None


# ------------------------------------------------------------------ inputs
def float_specials(dtype) -> np.ndarray:
    """±0, ±inf, NaNs with different payloads and signs, the smallest and largest subnormals and normals."""
    dt = np.dtype(dtype)
    u = _UNSIGNED[dt]
    if dt.itemsize == 8:
        bits = [0x0, 1 << 63, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001,
                0x7FFFFFFFFFFFFFFF, 0x7FF4000000000123, 0x1, 0x800FFFFFFFFFFFFF, 0x0010000000000000, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF]
    else:
        bits = [0x0, 1 << 31, 0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FFFFFFF, 0x7FA00123, 0x1, 0x807FFFFF,
                0x00800000, 0x7F7FFFFF, 0xFF7FFFFF]
    return np.array(bits, u).view(dt)


def int_specials(dtype) -> np.ndarray:
    info = np.iinfo(np.dtype(dtype))
    vals = [info.min, info.max, 0, 1, 2, 7, info.max - 1, info.max // 2, info.max // 2 + 1]
    if info.min < 0:
        vals += [-1, -2, -7, info.min + 1, info.min // 2]
    return np.array(vals, np.dtype(dtype))


def scalars(dtype) -> list:
    """The special scalar right- / left-hand sides: {3, -3, 0, 0.1, subnormal, inf, NaN} for floats (plus -0.0 and
    -inf), {0, ±1, min, max, 7} for integers."""
    dt = np.dtype(dtype)
    if dt.kind == "f":
        tiny = np.array([1], _UNSIGNED[dt]).view(dt)[0]
        return [dt.type(v) for v in (3.0, -3.0, 0.0, -0.0, 0.1, tiny, np.inf, -np.inf, np.nan)]
    info = np.iinfo(dt)
    vals = [0, 1, info.max, info.min, 7] + ([-1] if info.min < 0 else [])
    return [dt.type(v) for v in dict.fromkeys(vals)]


def column(rng, dtype, n: int, divisor: bool = False) -> np.ndarray:
    """Values over the dtype's whole range with the specials at the front.  Integers: uniform over [min, max]; with
    divisor=True a quarter of the rows are small divisors (|d| <= 9) and every 13th row is 0, so quotients are
    non-trivial and division by zero is exercised, and the specials are rotated so that row 0 holds -1 (a signed
    column's row 0 holds MIN: MIN // -1).  Floats: a third random bit patterns (NaN payloads, ±inf, ±0, subnormals),
    the rest normal values of mixed sign and magnitude."""
    dt = np.dtype(dtype)
    if dt.kind == "f":
        u = _UNSIGNED[dt]
        v = (rng.normal(0, 1, n) * np.exp2(rng.integers(-30, 31, n))).astype(dt)
        bits = rng.integers(0, np.iinfo(u).max, n, dtype=u, endpoint=True).view(dt)
        pick = rng.random(n) < 1 / 3
        v[pick] = bits[pick]
        sp = float_specials(dt)
    else:
        info = np.iinfo(dt)
        v = rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)
        if divisor:
            small = rng.random(n) < 0.25
            v[small] = rng.integers(-9 if info.min < 0 else 0, 10, int(small.sum())).astype(dt)
            v[::13] = 0
        sp = int_specials(dt)
        if divisor and info.min < 0:
            sp = np.roll(sp, -int(np.nonzero(sp == -1)[0][0]))
    k = min(n, sp.size)
    v[:k] = sp[:k]
    return v


def validity(rng, n: int, null_frac: float = 0.15) -> np.ndarray:
    return rng.random(n) >= null_frac
