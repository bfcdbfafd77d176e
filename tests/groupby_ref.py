"""Exact restatement of the fused group_by aggregations (K5: sum, mean, min, max, count, len) in numpy and Python, plus
the input generators its tests use.

Test infrastructure only.  Nothing here calls oracle/: tests/test_groupby_reference.py checks this statement against
the oracle on the CPU, and tests/test_gpu_groupby_plans.py checks every K5 plan against it.

Groups
  * rows group on canonical key bits: every NaN is one key and -0.0 == 0.0; null keys form one group;
  * with maintain_order the groups come in first-occurrence order, and each output key is the key at the group's first
    row; unordered results are compared after `canonical_order` (null group last, then by canonical bits).
Integers and counts (exact)
  * len counts rows, count counts non-null values;
  * integer sum wraps to the output dtype: 8/16-bit inputs give Int64, Int32 / UInt32 wrap at 32 bits, Int64 / UInt64 at
    64 bits; min / max are exact in the input dtype;
  * a group without a non-null value: sum = 0, mean / min / max are null.
Float min / max
  * NaN is ignored and an all-NaN group gives NaN; the sign of a zero result is not pinned (C fmin and Rust f64::min
    leave it unspecified), so any zero matches any zero.  Float32 results are exact.
Float sum / mean (and the mean of an integer column)
  * any NaN, or +inf together with -inf, gives NaN; otherwise a group holding an infinity gives that infinity;
  * otherwise the reference value is e = fl(exact sum) (math.fsum, or an exact vectorised sum when the group is
    exact-summable, see below) and S = sum of |x|.  For m summands any order of pairwise f64 additions - atomics in no
    fixed order, warp-shuffle trees, CTA-private partial sums - lands within (m - 1) * 2^-53 * S of the exact sum;
    rounding an Int64 / UInt64 summand to f64 adds 2^-53 * S, and rounding the reference's own value another 2^-53 * S:
    B = (m + 1) * 2^-53 * S bounds |got - e|;
  * exact-summable groups: every summand is an integer multiple of some q = 2^-s and S < 2^53 * q.  Then every partial
    sum of every order is exact, B = 0 and sum / mean must match bit for bit (the sign of a zero sum is not pinned);
  * a Float32 output is the f64 result rounded once: add 2^-24 * |e| and half an f32 subnormal ulp (2^-150);
  * mean = sum / count: the bound divides by the count and adds one rounding of the quotient.
  The sign of a zero sum is not pinned either: the device accumulator starts at +0.0, the reference's single-row sum
  returns the value itself.
"""
from __future__ import annotations

import math

import numpy as np

from primitives_ref import column, float_specials, int_specials, valid_equal, validity  # noqa: F401  (re-exported)

U = 2.0 ** -53
VALUE_DTYPES = ("int64", "uint64", "int32", "uint32", "float64", "float32")
SMALL_DTYPES = ("int8", "int16", "uint8", "uint16")
KINDS = ("sum", "mean", "min", "max", "count", "len")
_UNS = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


# ------------------------------------------------------------------ groups
def key_bits(keys) -> np.ndarray:
    """Canonical key bits as uint64: one NaN, -0.0 -> 0.0; integers as their zero-extended bit pattern."""
    k = np.asarray(keys)
    u = _UNS[k.dtype.itemsize]
    if k.dtype.kind == "f":
        with np.errstate(invalid="ignore"):
            c = np.where(k == 0, np.zeros(1, k.dtype), k)
        bits = c.view(u).copy()
        bits[np.isnan(k)] = np.array([np.nan], k.dtype).view(u)[0]
        return bits.astype(np.uint64)
    return k.view(u).astype(np.uint64)


class Groups:
    """gid: group of every row; first: first row of every group; order: rows sorted by group (ascending rows inside a
    group); offsets: group g owns order[offsets[g]:offsets[g + 1]]; null: the null group's index or -1."""

    def __init__(self, gid, first, null):
        self.gid, self.first, self.null = gid, first, null
        self.G = first.size
        self.order = np.argsort(gid, kind="stable")
        self.size = np.bincount(gid, minlength=self.G).astype(np.int64)
        self.offsets = np.concatenate([[0], np.cumsum(self.size)]).astype(np.int64)


def _from_codes(codes: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """codes (int64 per row, equal codes = one group) -> (gid per row, first row per group), groups in first-occurrence
    order."""
    _, first, inv = np.unique(codes, return_index=True, return_inverse=True)
    inv = np.asarray(inv).reshape(-1)
    rank_of = np.argsort(first, kind="stable")
    rank = np.empty(rank_of.size, np.int64)
    rank[rank_of] = np.arange(rank_of.size)
    return rank[inv], first[rank_of]


def group(keys, key_valid=None, maintain_order: bool = True) -> Groups:
    """One key column.  Unordered: null group last, the others by canonical bits (`canonical_order`)."""
    bits = key_bits(keys)
    n = bits.size
    kv = np.ones(n, bool) if key_valid is None else np.asarray(key_valid, bool)
    if n == 0:
        return Groups(np.zeros(0, np.int64), np.zeros(0, np.int64), -1)
    rows = np.nonzero(kv)[0]
    _, first_v, inv = np.unique(bits[kv], return_index=True, return_inverse=True)
    first = rows[first_v]
    gid = np.empty(n, np.int64)
    gid[rows] = np.asarray(inv).reshape(-1)
    if rows.size < n:                                   # the null group: after the others (the canonical unordered order)
        gid[~kv] = first.size
        first = np.append(first, np.nonzero(~kv)[0][0])
    if maintain_order:
        rank_of = np.argsort(first, kind="stable")
        rank = np.empty(rank_of.size, np.int64)
        rank[rank_of] = np.arange(rank_of.size)
        gid, first = rank[gid], first[rank_of]
    null = int(gid[np.nonzero(~kv)[0][0]]) if (~kv).any() else -1
    return Groups(gid, first.astype(np.int64), null)


def group_multi(keys_list, valids_list) -> Groups:
    """Several key columns: two rows are one group iff every column has the same (validity, canonical bits); groups
    in first-occurrence order."""
    n = np.asarray(keys_list[0]).size
    codes = np.zeros(n, np.int64)
    for k, v in zip(keys_list, valids_list):
        g = group(k, v, maintain_order=False)
        combined = codes * np.int64(g.G + 1) + g.gid
        _, codes = np.unique(combined, return_inverse=True)
        codes = np.asarray(codes).reshape(-1).astype(np.int64)
    if n == 0:
        return Groups(np.zeros(0, np.int64), np.zeros(0, np.int64), -1)
    gid, first = _from_codes(codes)
    return Groups(gid, first.astype(np.int64), -1)


def out_keys(keys, key_valid, g: Groups):
    """Output key column: the key at every group's first row."""
    k = np.asarray(keys)
    return k[g.first], (None if key_valid is None else np.asarray(key_valid, bool)[g.first])


def canonical_order(keys, key_valid) -> np.ndarray:
    """Permutation that puts a group_by result into the unordered reference order (null group last, then by bits)."""
    bits = key_bits(keys)
    kv = np.ones(bits.size, bool) if key_valid is None else np.asarray(key_valid, bool)
    return np.lexsort((np.where(kv, bits, np.uint64(0)), ~kv))


# ------------------------------------------------------------------ aggregations
def kahan32(exp: "FloatExpect") -> "FloatExpect":
    """The bound of a Float32 sum computed as a Kahan sum in f32 (the reference's polars-utils/src/kahan_sum.rs, which
    the oracle and the deterministic device path follow): (2 eps + 2 m eps^2) S with eps = 2^-24, plus subnormal slop.
    It replaces the bound of an f64 sum rounded once."""
    eps = 2.0 ** -24
    tol = (2 * eps + 2 * exp.m * eps * eps) * exp.S + 2.0 ** -149
    return FloatExpect(exp.kind, exp.dtype, exp.e, np.where(exp.special, 0.0, tol), exp.valid)


def sum_out_dtype(dtype) -> np.dtype:
    dt = np.dtype(dtype)
    return np.dtype(np.int64) if dt.name in SMALL_DTYPES else dt


def out_dtype(kind: str, dtype) -> np.dtype:
    dt = np.dtype(dtype) if dtype is not None else None
    if kind in ("len", "count"):
        return np.dtype(np.uint32)
    if kind == "sum":
        return sum_out_dtype(dt)
    if kind == "mean":
        return np.dtype(np.float32) if dt == np.float32 else np.dtype(np.float64)
    return dt


class FloatExpect:
    """Expected float sum / mean: value `e` (f64 per group), the bound `tol` on |got - e| (0 = must match exactly),
    the validity, and the output dtype."""

    def __init__(self, kind, dtype, e, tol, valid):
        self.kind, self.dtype, self.e, self.tol, self.valid = kind, np.dtype(dtype), e, tol, valid


def _sorted(values, valid, g: Groups):
    v = np.asarray(values)[g.order]
    ok = np.ones(v.size, bool) if valid is None else np.asarray(valid, bool)[g.order]
    return v, ok


def _reduceat(fn, x, g: Groups):
    if g.G == 0:
        return x[:0]
    return fn.reduceat(x, g.offsets[:-1])


def _quantum(x: np.ndarray) -> np.ndarray:
    """Value of the lowest set mantissa bit of every finite f64 (inf for 0)."""
    m, e = np.frexp(x)
    k = np.abs(m * 2.0 ** 53).astype(np.int64)
    low = k & -k
    with np.errstate(over="ignore"):
        q = np.ldexp(low.astype(np.float64), e - 53)
    return np.where(x == 0, np.inf, q)


def _exact_sums(x: np.ndarray, g: Groups, fsum_limit: int):
    """Per-group fl(exact sum) of the finite f64 array x (already ordered by group, zeros for excluded rows), with
    S = sum |x| (rounded up) and an `exact` flag per group (exact-summable: every order gives the exact sum)."""
    m_rows = g.size
    s_fast = _reduceat(np.add, x, g)
    with np.errstate(over="ignore"):
        S = _reduceat(np.add, np.abs(x), g) * (1.0 + 2.0 * U * m_rows.astype(np.float64))
    q = _reduceat(np.minimum, _quantum(x), g)
    with np.errstate(over="ignore", invalid="ignore"):
        exact = (m_rows <= 1) | (S < np.ldexp(1.0, 53) * q) | (S == 0)
    e = s_fast.copy()
    slow = np.nonzero(~exact)[0]
    rows = int(m_rows[slow].sum())
    assert rows <= fsum_limit, f"{rows} rows of float sums need math.fsum (limit {fsum_limit}): use exact-summable values"
    xl = x.tolist()
    for gi in slow.tolist():
        e[gi] = math.fsum(xl[g.offsets[gi]:g.offsets[gi + 1]])
    return e, S, exact


def _int_exact_sum(v: np.ndarray, ok: np.ndarray, g: Groups):
    """Per-group fl(exact integer sum) of an integer array (no wrapping), and S = sum |x| as f64 (rounded up)."""
    dt = v.dtype
    if dt.itemsize == 8:
        if dt.kind == "u":
            hi = (v >> np.uint64(32)).astype(np.int64)
            lo = (v & np.uint64(0xFFFFFFFF)).astype(np.int64)
        else:
            hi = v >> np.int64(32)
            lo = (v & np.int64(0xFFFFFFFF))
        hi = np.where(ok, hi, 0)
        lo = np.where(ok, lo, 0)
        e = _reduceat(np.add, hi, g).astype(np.float64) * 2.0 ** 32 + _reduceat(np.add, lo, g).astype(np.float64)
    else:
        e = _reduceat(np.add, np.where(ok, v.astype(np.int64), 0), g).astype(np.float64)
    a = np.where(ok, np.abs(v.astype(np.float64)), 0.0)
    S = _reduceat(np.add, a, g) * (1.0 + 2.0 * U * g.size.astype(np.float64))
    fits = _reduceat(np.maximum, a, g) <= 2.0 ** 53 if g.G else np.zeros(0, bool)
    exact = fits & (S < 2.0 ** 53)
    return e, S, exact


def _float_sum_expect(kind, values, valid, g: Groups, fsum_limit: int) -> FloatExpect:
    v, ok = _sorted(values, valid, g)
    dt = v.dtype
    odt = out_dtype(kind, dt)
    cnt = _reduceat(np.add, ok.astype(np.int64), g)
    if dt.kind == "f":
        with np.errstate(invalid="ignore"):
            x = v.astype(np.float64)
        nan = _reduceat(np.logical_or, ok & np.isnan(x), g)
        pinf = _reduceat(np.logical_or, ok & (x == np.inf), g)
        ninf = _reduceat(np.logical_or, ok & (x == -np.inf), g)
        fin = np.where(ok & np.isfinite(x), x, 0.0)
        e, S, exact = _exact_sums(fin, g, fsum_limit)
        m = _reduceat(np.add, (fin != 0).astype(np.int64), g).astype(np.float64)
        B = np.where(exact, 0.0, (m + 1.0) * U * S)
        special = np.where(nan | (pinf & ninf), np.nan, np.where(pinf, np.inf, np.where(ninf, -np.inf, 0.0)))
        is_special = nan | pinf | ninf
    else:
        e, S, exact = _int_exact_sum(v, ok, g)
        m = cnt.astype(np.float64)
        B = np.where(exact, 0.0, (m + 1.0) * U * S)
        special = np.zeros(g.G)
        is_special = np.zeros(g.G, bool)
    with np.errstate(invalid="ignore", divide="ignore"):
        if kind == "sum":
            val, tol, vld = e, B, np.ones(g.G, bool)
        else:
            c = np.maximum(cnt, 1).astype(np.float64)
            val = e / c
            tol = np.where(B == 0, 0.0, (B + U * (2.0 * np.abs(e) + B)) / c)
            vld = cnt > 0
        if odt == np.float32:
            tol = np.where(tol == 0, 0.0, tol + 2.0 ** -24 * (np.abs(val) + tol) + 2.0 ** -150)
    val = np.where(is_special, special, val)
    tol = np.where(is_special, 0.0, tol)
    fe = FloatExpect(kind, odt, val, tol, vld)
    fe.S, fe.m, fe.special = S, m, is_special
    return fe


def aggregate(kind: str, values, valid, g: Groups, fsum_limit: int = 1_500_000):
    """One aggregation -> (values, valid|None) for exact kinds, or a FloatExpect for float sums and every mean."""
    if kind == "len":
        return g.size.astype(np.uint32), None
    v, ok = _sorted(values, valid, g)
    dt = v.dtype
    cnt = _reduceat(np.add, ok.astype(np.int64), g)
    if kind == "count":
        return cnt.astype(np.uint32), None
    if kind == "mean" or (kind == "sum" and dt.kind == "f"):
        return _float_sum_expect(kind, values, valid, g, fsum_limit)
    has = cnt > 0
    if kind == "sum":
        odt = sum_out_dtype(dt)
        u = _UNS[odt.itemsize]
        x = np.where(ok, v.astype(odt), np.zeros(1, odt)).view(u).astype(np.uint64)
        s = _reduceat(np.add, x, g) if g.G else np.zeros(0, np.uint64)
        return (s & np.uint64((1 << (8 * odt.itemsize)) - 1)).astype(u).view(odt), None
    if kind in ("min", "max"):
        if dt.kind == "f":
            # NaN never enters the fold: np.fmin / np.fmax (like glibc fmin) return NaN for a signalling NaN operand
            num = ok & ~np.isnan(v)
            x = np.where(num, v, np.array([np.inf if kind == "min" else -np.inf], dt))
            r = _reduceat(np.minimum if kind == "min" else np.maximum, x, g)
            r = np.where(_reduceat(np.add, num.astype(np.int64), g) > 0, r, np.array([np.nan], dt))   # all NaN -> NaN
        else:
            info = np.iinfo(dt)
            x = np.where(ok, v, np.array([info.max if kind == "min" else info.min], dt))
            r = _reduceat(np.minimum if kind == "min" else np.maximum, x, g)
        return r.astype(dt), (None if has.all() else has)
    raise ValueError(kind)


# ------------------------------------------------------------------ comparison
def check(got, got_valid, exp) -> str | None:
    """None when `got` matches the expectation; otherwise a short description of the first difference.  Exact kinds:
    validity and bits (any NaN equals any NaN, any zero equals any zero).  FloatExpect: NaN / inf exactly, the rest
    within the bound."""
    got = np.asarray(got)
    if isinstance(exp, FloatExpect):
        if got.dtype != exp.dtype:
            return f"dtype {got.dtype} != {exp.dtype}"
        if got.shape != exp.e.shape:
            return f"length {got.shape} != {exp.e.shape}"
        gv = np.ones(got.shape, bool) if got_valid is None else np.asarray(got_valid, bool)
        if not np.array_equal(gv, exp.valid):
            i = int(np.nonzero(gv != exp.valid)[0][0])
            return f"validity differs at group {i}: got {gv[i]} expected {exp.valid[i]}"
        with np.errstate(invalid="ignore"):
            g64 = got.astype(np.float64)
        e = exp.e
        exact_cmp = exp.tol == 0
        with np.errstate(invalid="ignore", over="ignore"):
            ev = e.astype(exp.dtype).astype(np.float64)    # the expected value in the output dtype
            ok = np.where(np.isnan(e), np.isnan(g64),
                          np.where(exact_cmp, g64 == ev, np.abs(g64 - e) <= exp.tol))
        bad = exp.valid & ~ok
        if bad.any():
            i = int(np.nonzero(bad)[0][0])
            return (f"{int(bad.sum())} groups outside the bound, first {i}: got {got[i]!r} expected {e[i]!r} "
                    f"(tolerance {exp.tol[i]:.3g}, off by {abs(g64[i] - e[i]):.3g})")
        return None
    ev, evalid = exp
    ev = np.asarray(ev)
    if ev.dtype.kind == "f" and got.dtype == ev.dtype and got.shape == ev.shape:
        # any zero equals any zero
        z = (got == 0) & (ev == 0)
        got = np.where(z, ev, got)
    if ev.dtype.kind in "iu" and ev.dtype.itemsize < 4:
        if got.dtype != ev.dtype:
            return f"dtype {got.dtype} != {ev.dtype}"
        got, ev = got.astype(np.int32), ev.astype(np.int32)
    return valid_equal(got, got_valid, ev, evalid)


# ------------------------------------------------------------------ inputs
def capped(x: np.ndarray, max_exp: int) -> np.ndarray:
    """Finite values with |x| >= 2^max_exp get their exponent lowered to max_exp (sign and mantissa kept)."""
    x = np.asarray(x)
    with np.errstate(invalid="ignore"):
        m, e = np.frexp(x.astype(np.float64))
    big = np.isfinite(x) & (e > max_exp)
    out = x.copy()
    out[big] = np.ldexp(m[big], max_exp).astype(x.dtype)
    return out


def sum_cap_exp(dtype, max_group_rows: int) -> int:
    """Per-value exponent cap so that S <= 2^1000 (f64 outputs) or S < FLT_MAX / 2 (f32 outputs) per group."""
    rows_bits = max(1, int(max_group_rows - 1).bit_length())
    return (1000 if np.dtype(dtype) == np.float64 else 126) - rows_bits


def sum_column(rng, dtype, n: int, exact: bool = False, max_group_rows: int = 1 << 22) -> np.ndarray:
    """Values for sum / mean.  Floats: the full-range generator with the magnitude cap, or (exact=True) exact-summable
    values: integers times 2^-s (31 significant bits for f64, 24 for f32) of mixed sign, so a group of up to 2^22 rows
    sums exactly in any order.  Integers: the full-range generator."""
    dt = np.dtype(dtype)
    if dt.kind != "f":
        return column(rng, dt, n)
    if exact:
        bits = 30 if dt == np.float64 else 23
        return np.ldexp(rng.integers(-(1 << bits), 1 << bits, n).astype(np.float64), -20).astype(dt)
    return capped(column(rng, dt, n), sum_cap_exp(dt, max_group_rows))


SPECIAL_GROUPS = ("all_nan", "all_null", "inf_pair", "subnormal", "cancel", "extremes", "singleton")
SPECIAL_ROWS = {"all_nan": 3, "all_null": 3, "inf_pair": 3, "subnormal": 4, "cancel": 9, "extremes": 4, "singleton": 1}


def fill_special(rng, name: str, dtype, for_sum: bool):
    """Values (and validity) of one dedicated group.  Integers have no NaN / inf / subnormal groups: those become a
    wrapping group (MAX repeated) and a MIN group."""
    dt = np.dtype(dtype)
    k = SPECIAL_ROWS[name]
    valid = np.ones(k, bool)
    if name == "all_null":
        return np.zeros(k, dt), np.zeros(k, bool)
    if dt.kind == "f":
        u = _UNS[dt.itemsize]
        sp = float_specials(dt)
        if name == "all_nan":
            v = sp[[4, 5, 6]]
        elif name == "inf_pair":
            v = np.array([np.inf, -np.inf, 1.0], dt)
        elif name == "subnormal":
            v = np.array([1, 3, 0x1234, 7], u).view(dt)
            v[1] = -v[1]
        elif name == "cancel":
            big = rng.normal(0, 1, 4) * 2.0 ** 30
            tiny = 2.0 ** -40 if dt == np.float64 else 2.0 ** -20
            v = np.array([big[0], -big[0], big[1], big[2], -big[1], big[3], -big[2], -big[3], tiny], dt)
        elif name == "extremes":
            v = np.array([np.finfo(dt).min, np.finfo(dt).max, np.finfo(dt).max, np.finfo(dt).min], dt)
        else:
            v = np.array([rng.normal() * 2.0 ** 20], dt)
        if for_sum:
            v = capped(v, sum_cap_exp(dt, 1 << 22))
        return v, valid
    info = np.iinfo(dt)
    if name == "all_nan":
        v = np.array([info.max] * k, dt)
    elif name == "inf_pair":
        v = np.array([info.min] * k, dt)
    elif name == "subnormal":
        v = np.array([1, 0, 1, 0], dt)
    elif name == "cancel":
        x = rng.integers(info.min // 2, info.max // 2, 4, dtype=dt, endpoint=True)
        neg = (np.zeros(1, _UNS[dt.itemsize]) - x.view(_UNS[dt.itemsize])).view(dt)
        v = np.concatenate([x, neg, np.array([1], dt)])
    elif name == "extremes":
        v = np.array([info.min, info.max, info.max, info.min], dt)
    else:
        v = rng.integers(info.min, info.max, 1, dtype=dt, endpoint=True)
    return v, valid


def _distinct_keys(rng, dtype, count: int) -> np.ndarray:
    """`count` distinct canonical keys of the dtype (no NaN, no -0.0), the dtype's specials first."""
    dt = np.dtype(dtype)
    if dt.kind == "f":
        sp = float_specials(dt)
        sp = sp[~np.isnan(sp) & (sp != 0)]          # the NaN and zero groups get keys of their own (Case)
    else:
        sp = int_specials(dt)
    cand = [sp]
    have = 0
    while have < count + sp.size:
        if dt.kind == "f":
            u = _UNS[dt.itemsize]
            c = rng.integers(0, np.iinfo(u).max, 2 * count + 64, dtype=u, endpoint=True).view(dt)
            c = c[~np.isnan(c) & (c != 0)]
        elif dt.itemsize <= 2:
            info = np.iinfo(dt)
            c = rng.permutation(np.arange(info.min, info.max + 1)).astype(dt)      # every value once
        else:
            info = np.iinfo(dt)
            c = rng.integers(info.min, info.max, min(2 * count + 64, 1 << 26), dtype=dt, endpoint=True)
        cand.append(c)
        have += c.size
        if dt.kind != "f" and dt.itemsize <= 2:
            break
    allk = np.concatenate(cand)
    _, idx = np.unique(key_bits(allk), return_index=True)
    idx.sort()                      # specials first, then in generation order
    out = allk[idx]
    assert out.size >= count, f"{dt}: only {out.size} distinct keys, {count} wanted"
    return out[:count]


class Case:
    """Rows of one group_by test: key column (+ validity) and the rows of every dedicated group.

    Layout: one big group (`big` rows), `singletons` one-row groups, `groups` further groups over `rest` rows drawn
    uniformly (or Zipf(`zipf`) when set), the dedicated groups of SPECIAL_GROUPS, and a null-key group (`null_rows`),
    shuffled.  Float keys of the NaN group carry different NaN payloads and the zero group mixes -0.0 and 0.0."""

    def __init__(self, rng, key_dtype, *, big=0, singletons=0, groups=0, rest=0, null_rows=0, specials=True, zipf=None,
                 big_key=None, shuffle=True):
        kd = np.dtype(key_dtype)
        sizes = []
        if big:
            sizes.append(np.full(1, big))
        sizes.append(np.ones(singletons, np.int64))
        if specials:
            sizes.append(np.array([SPECIAL_ROWS[s] for s in SPECIAL_GROUPS]))
        n_fixed = int(sum(s.size for s in sizes))
        labels_fixed = np.repeat(np.arange(n_fixed), np.concatenate(sizes).astype(np.int64)) if n_fixed else np.zeros(0, np.int64)
        if groups and rest:
            if zipf:
                r = (rng.zipf(zipf, rest) - 1) % groups
            else:
                r = rng.integers(0, groups, rest)
            labels = np.concatenate([labels_fixed, n_fixed + r])
        else:
            labels = labels_fixed
        n_labels = n_fixed + (groups if rest else 0)
        # the null group
        labels = np.concatenate([labels, np.full(null_rows, -1)])
        perm = rng.permutation(labels.size) if shuffle else np.arange(labels.size)
        labels = labels[perm]
        self.n = labels.size
        keys_of = _distinct_keys(rng, kd, n_labels)
        if big and big_key is not None:
            hit = np.nonzero(key_bits(keys_of) == key_bits(np.array([big_key], kd))[0])[0]
            if hit.size:
                keys_of[[0, hit[0]]] = keys_of[[hit[0], 0]]
            else:
                keys_of[0] = big_key
        valid_rows = labels >= 0
        keys = keys_of[np.where(valid_rows, labels, 0)] if n_labels else np.zeros(self.n, kd)
        if kd.kind == "f" and rest and groups >= 2:
            # two more labels' rows get alternative encodings of NaN / zero: every NaN payload is one group, -0.0 == 0.0
            sp = float_specials(kd)
            nans = sp[np.isnan(sp)]
            lab_nan, lab_zero = n_labels - 1, n_labels - 2
            rn = np.nonzero(labels == lab_nan)[0]
            keys[rn] = nans[rng.integers(0, nans.size, rn.size)]
            rz = np.nonzero(labels == lab_zero)[0]
            keys[rz] = np.where(rng.random(rz.size) < 0.5, kd.type(0.0), kd.type(-0.0))
        self.keys = keys
        self.key_valid = None if null_rows == 0 else valid_rows
        self.labels = labels
        self.special_rows = {}
        if specials:
            base = 1 if big else 0
            base += singletons
            for i, s in enumerate(SPECIAL_GROUPS):
                self.special_rows[s] = np.nonzero(labels == base + i)[0]

    def values(self, rng, dtype, *, for_sum: bool = False, exact: bool = False, nullable: bool = False, null_frac: float = 0.15):
        """A value column over the case's rows: the full-range generator (magnitude-capped / exact-summable for sum and
        mean), nulls when `nullable`, and the dedicated groups' patterns."""
        dt = np.dtype(dtype)
        if dt.name in SMALL_DTYPES:
            info = np.iinfo(dt)
            v = rng.integers(info.min, info.max, self.n, dtype=dt, endpoint=True)
            k = min(self.n, 2)
            v[:k] = [info.min, info.max][:k]
        elif for_sum:
            v = sum_column(rng, dt, self.n, exact=exact)
        else:
            v = column(rng, dt, self.n)
        valid = validity(rng, self.n, null_frac) if nullable else None
        for s, rows in self.special_rows.items():
            if s == "all_null" and not nullable:
                continue
            if dt.name in SMALL_DTYPES:
                if s == "all_null":
                    valid[rows] = False
                continue
            sv, svalid = fill_special(rng, s, dt, for_sum)
            v[rows] = sv[: rows.size]
            if valid is not None:
                valid[rows] = svalid[: rows.size]
        return v, valid


def expect(case_keys, key_valid, aggs, maintain_order: bool, fsum_limit: int = 1_500_000, g: Groups | None = None):
    """aggs: [(kind, values | None, valid | None)] -> ((keys, key_valid), [expectation per aggregation], groups)."""
    if g is None:
        g = group(case_keys, key_valid, maintain_order)
    ko = out_keys(case_keys, key_valid, g)
    outs = [aggregate(kind, v, m, g, fsum_limit) if kind != "len" else aggregate("len", None, None, g) for kind, v, m in aggs]
    return ko, outs, g
