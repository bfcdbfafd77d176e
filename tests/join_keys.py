"""Join-key columns over the full range of every key dtype the hash join accepts, for the GPU join tests and for the
brute-force checks of the oracle they are compared with.

Every column comes with the values hash joins get wrong: MIN, MAX, 0 and -1; UInt64 2^63 (= i64::MIN, the empty-slot
marker of the WIDE table) and 2^64 - 1; UInt32 values >= 2^31; NaNs with several payloads and both signs, -0.0 and
+0.0, +-inf and subnormals.  Keys compare as the reference compares them: NaN equals NaN, -0.0 equals +0.0, integers by
value.  `canon` states that equality in plain Python and `canon_bits` in numpy; neither uses the oracle.
"""
from __future__ import annotations

import numpy as np

DTYPES = ("int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64")
INT_DTYPES = DTYPES[:8]

_NAN64 = [0x7FF8000000000000, 0xFFF8000000000000, 0x7FF0000000000001, 0x7FF4000000000ABC, 0xFFFFFFFFFFFFFFFF, 0xFFF0000000000001]
_NAN32 = [0x7FC00000, 0xFFC00000, 0x7F800001, 0x7FA00ABC, 0xFFFFFFFF, 0xFF800001]


def specials(dtype) -> np.ndarray:
    """The planted values of `dtype`.  Float NaNs come with several payloads (quiet, signalling, negative), so a column
    holding all of them has several bit patterns for one key."""
    dt = np.dtype(dtype)
    if dt.kind == "f":
        u = np.dtype(f"u{dt.itemsize}")
        nans = np.array(_NAN64 if dt.itemsize == 8 else _NAN32, dtype=u).view(dt)
        fi = np.finfo(dt)
        sub = fi.smallest_subnormal
        vals = [0.0, -0.0, np.inf, -np.inf, sub, -sub, fi.smallest_normal - sub, -(fi.smallest_normal - sub),
                fi.smallest_normal, fi.max, -fi.max, 1.0, -1.0]
        return np.concatenate([nans, np.array(vals, dtype=dt)])
    info = np.iinfo(dt)
    vals = {info.min, info.max, 0, 1, info.max - 1}
    if dt.kind == "i":
        vals |= {-1, info.min + 1}
    else:
        half = (info.max + 1) // 2                  # 2^(bits - 1): UInt64 2^63 is the bit pattern of i64::MIN
        vals |= {half, half - 1, half + 1}
    return np.array(sorted(vals), dtype=dt)


def canon_bits(values) -> np.ndarray:
    """uint64 per value, equal iff the keys are equal: NaNs collapse to one pattern, -0.0 to +0.0, integers keep their
    bit pattern (zero-extended)."""
    v = np.ascontiguousarray(values)
    if v.dtype.kind == "f":
        bits = v.view(np.dtype(f"u{v.dtype.itemsize}")).astype(np.uint64)
        bits = np.where(v == 0, np.uint64(0), bits)
        return np.where(np.isnan(v), np.uint64(0x7FF8000000000000), bits)
    return v.view(np.dtype(f"u{v.dtype.itemsize}")).astype(np.uint64)


def canon(values, valid=None) -> list:
    """Python key per row: None for a null row, "nan" for any NaN, a float (-0.0 == 0.0) or an int otherwise."""
    v = np.asarray(values)
    out = []
    for i, x in enumerate(v.tolist()):
        if valid is not None and not valid[i]:
            out.append(None)
        elif isinstance(x, float) and x != x:
            out.append("nan")
        else:
            out.append(x)
    return out


def _random(rng, dt: np.dtype, n: int) -> np.ndarray:
    if dt.kind == "f":                      # random bit patterns: every exponent, NaN payloads and subnormals included
        u = np.dtype(f"u{dt.itemsize}")
        return rng.integers(0, np.iinfo(u).max, n, dtype=u, endpoint=True).view(dt)
    info = np.iinfo(dt)
    return rng.integers(info.min, info.max, n, dtype=dt, endpoint=True)


def dense_run(rng, dtype, n: int, span: int) -> np.ndarray:
    """n distinct integers from a contiguous run of `span` values that holds both of its ends: the run is centred on
    zero for signed dtypes and ends at the dtype's MAX (2^64 - 1 for UInt64) for unsigned ones.  Not shuffled."""
    dt = np.dtype(dtype)
    info = np.iinfo(dt)
    assert 2 <= n <= span <= int(info.max) - int(info.min) + 1
    off = np.concatenate([[0, span - 1], 1 + rng.permutation(span - 2)[: n - 2]]).astype(np.uint64)
    if dt.kind == "i":
        lo = -(span // 2)
        return (np.int64(lo) + off.astype(np.int64)).astype(dt)
    lo = int(info.max) - span + 1
    return (np.uint64(lo) + off).astype(dt)


def distinct(rng, dtype, n: int, dense: int | None = None) -> np.ndarray:
    """n keys, pairwise different after canonicalisation, in random order.  Without `dense` they span the dtype's range
    and hold every special of `dtype` that fits (one NaN and one zero: they are one key each); with `dense` they come
    from dense_run(span=dense)."""
    dt = np.dtype(dtype)
    if dense is not None:
        out = dense_run(rng, dt, n, dense)
    else:
        sp = specials(dt)
        cand = np.concatenate([sp, _random(rng, dt, n + n // 4 + 64)])
        _, first = np.unique(canon_bits(cand), return_index=True)
        first.sort()                                 # specials first, so each one is kept
        if first.size < n:
            assert dt.itemsize <= 2, (dtype, n)     # 8 / 16-bit dtypes: take the whole range
            cand = np.arange(int(np.iinfo(dt).min), int(np.iinfo(dt).max) + 1).astype(dt)
            first = np.arange(cand.size)
            assert cand.size >= n, (dtype, n)
        out = cand[first[:n]]
    return out[rng.permutation(out.size)]


def keys(rng, dtype, n: int, dups: str = "unique", k: int = 2, nulls: float | int = 0, dense: int | None = None):
    """A key column of n rows -> (values, valid | None).

    dups: "unique" (every key once), "k" (every key k times), "runs" (each key 1..k times, uniformly), "hot" (one key k
    times, the others once).  nulls: a fraction of rows (float) or an exact number of rows (int) without a value; a null
    row keeps a random value underneath.  dense: draw the distinct keys from dense_run(span=dense)."""
    dt = np.dtype(dtype)
    if dups == "unique":
        vals = distinct(rng, dt, n, dense)
    elif dups == "k":
        d = distinct(rng, dt, -(-n // k), dense)
        vals = np.repeat(d, k)[:n]
    elif dups == "runs":
        lens = rng.integers(1, k + 1, n)             # more runs than needed; cut at n rows
        m = int(np.searchsorted(np.cumsum(lens), n)) + 1
        d = distinct(rng, dt, m, dense)
        vals = np.repeat(d, lens[:m])[:n]
    elif dups == "hot":
        d = distinct(rng, dt, n - k + 1, dense)
        vals = np.concatenate([np.repeat(d[:1], k), d[1:]])
    else:
        raise ValueError(dups)
    vals = vals[rng.permutation(n)]
    return vals, null_mask(rng, n, nulls)


def probe(rng, build_values, n: int, hit: float = 0.6, nulls: float | int = 0, dense_edges: bool = False):
    """A probe column of n rows -> (values, valid | None): a `hit` fraction drawn from build_values, the rest full-range
    values and every special of the dtype with every payload (most of them miss).  dense_edges: also the values just
    outside the build keys' [min, max] and the dtype's extremes, where the offset from the minimum wraps."""
    b = np.asarray(build_values)
    dt = b.dtype
    nh = int(n * hit) if b.size else 0
    extra = [specials(dt)]
    if dense_edges and b.size:
        info = np.iinfo(dt)
        lo, hi = int(b.min()), int(b.max())
        extra.append(np.array([x for x in (lo - 1, lo - 2, hi + 1, hi + 2, info.min, info.max) if info.min <= x <= info.max], dtype=dt))
    extra = np.concatenate(extra)
    miss = _random(rng, dt, max(n - nh - extra.size, 0))
    vals = np.concatenate([b[rng.integers(0, b.size, nh)] if nh else b[:0], extra, miss])[:n]
    vals = vals[rng.permutation(vals.size)]
    return vals, null_mask(rng, vals.size, nulls)


def null_mask(rng, n: int, nulls):
    if isinstance(nulls, (int, np.integer)) and not isinstance(nulls, bool):
        if nulls <= 0:
            return None
        valid = np.ones(n, bool)
        valid[rng.choice(n, min(int(nulls), n), replace=False)] = False
        return valid
    if nulls <= 0:
        return None
    return rng.random(n) >= nulls
