"""Inputs and plain restatements shared by the sort-family plan tests (tests/test_gpu_sort_plans.py) and their CPU
cross-checks (tests/test_sort_cases.py): full-range key columns written as bit patterns, GroupsIdx in numpy, a dense
rank of byte strings from Python's sorted(), the window rule of the small-group quantile kernel, and the rounds of
the string-rank refinement."""
from __future__ import annotations

import numpy as np

NP = {"int8": np.int8, "int16": np.int16, "int32": np.int32, "int64": np.int64, "uint8": np.uint8, "uint16": np.uint16,
      "uint32": np.uint32, "uint64": np.uint64, "float32": np.float32, "float64": np.float64, "bool": np.bool_}
KEY_DTYPES = list(NP)

QS_H = 2048          # k_quantile_small: window of QS_H group starts, at most 2 * QS_H keys


def f64_bits(*u) -> np.ndarray:
    return np.array(u, np.uint64).view(np.float64)


def f32_bits(*u) -> np.ndarray:
    return np.array(u, np.uint32).view(np.float32)


# quiet NaN, sign-set NaN, quiet and signalling NaN payloads of both signs, ±0.0, ±inf, the smallest and largest
# subnormals, the smallest normal, ±max finite, ±1
F64_SPECIAL = f64_bits(0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8000000000001, 0xFFFFFFFFFFFFFFFF, 0x7FF0000000000001,
                       0xFFF0000000000001, 0x7FF4000000000000, 0x0000000000000000, 0x8000000000000000, 0x7FF0000000000000,
                       0xFFF0000000000000, 0x0000000000000001, 0x8000000000000001, 0x000FFFFFFFFFFFFF, 0x800FFFFFFFFFFFFF,
                       0x0010000000000000, 0x7FEFFFFFFFFFFFFF, 0xFFEFFFFFFFFFFFFF, 0x3FF0000000000000, 0xBFF0000000000000)
F32_SPECIAL = f32_bits(0x7FC00000, 0xFFC00000, 0x7FC00001, 0xFFFFFFFF, 0x7F800001, 0xFF800001, 0x7FA00000, 0x00000000,
                       0x80000000, 0x7F800000, 0xFF800000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00800000,
                       0x7F7FFFFF, 0xFF7FFFFF, 0x3F800000, 0xBF800000)


def int_pool(dt) -> np.ndarray:
    """MIN, MAX and their neighbours, 0 / ±1, the values around 2^31, 2^32, 2^53 and 2^63 that the dtype holds"""
    info = np.iinfo(dt)
    cand = [info.min, info.min + 1, -1, 0, 1, 2, info.max - 1, info.max]
    for p in (7, 8, 15, 16, 31, 32, 53, 63):
        cand += [(1 << p) - 1, 1 << p, (1 << p) + 1, -(1 << p), -(1 << p) - 1]
    return np.array(sorted({int(c) for c in cand if info.min <= c <= info.max}), dtype=dt)


def full_range_column(rng, dt: str, n: int) -> np.ndarray:
    """n values of dtype dt over its whole range: Int8 / UInt8 / Bool take every value (n >= 256), the other dtypes mix the
    special pool with random bit patterns (floats: any NaN payload, subnormals, both zeros and infinities)."""
    t = NP[dt]
    if dt == "bool":
        return rng.random(n) < 0.5
    if dt in ("int8", "uint8"):
        return rng.permutation(np.resize(np.arange(256, dtype=np.uint8).view(t), n))
    bits = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[np.dtype(t).itemsize]
    rand = rng.integers(0, np.iinfo(bits).max, n, dtype=bits, endpoint=True).view(t)
    pool = F64_SPECIAL if dt == "float64" else F32_SPECIAL if dt == "float32" else int_pool(t)
    out = np.where(rng.random(n) < 0.5, rng.choice(pool, n), rand).astype(t)
    out[: pool.size] = pool[: n]                      # every special value at least once
    return out


def groups_idx(keys) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """GroupsIdx (first, offsets, all) in numpy: groups in first-occurrence order, each group's rows ascending"""
    keys = np.asarray(keys)
    n = keys.size
    _, first, inv = np.unique(keys, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")
    rank = np.empty(first.size, np.int64)
    rank[order] = np.arange(first.size)
    gid = rank[inv.reshape(-1)]
    all_ = np.argsort(gid, kind="stable").astype(np.uint32)
    offsets = np.zeros(first.size + 1, np.uint32)
    np.cumsum(np.bincount(gid, minlength=first.size), out=offsets[1:])
    return first[order].astype(np.uint32), offsets, all_ if n else np.zeros(0, np.uint32)


def keys_with_group_sizes(rng, sizes) -> np.ndarray:
    """int64 keys whose groups, in first-occurrence order, have the given sizes; the rows of different groups are
    interleaved (the first row of each group comes in group order, the rest are shuffled behind them)"""
    sizes = np.asarray(sizes, np.int64)
    rest = rng.permutation(np.repeat(np.arange(sizes.size), sizes - 1))
    return np.concatenate([np.arange(sizes.size), rest]).astype(np.int64)


def small_windows(sizes, h: int = QS_H) -> list[tuple[int, int]]:
    """The groups k_quantile_small takes, window by window: (groups, keys) of window b, which holds the groups whose start
    offset lies in [b*h, (b+1)*h) except a last one of more than h rows (the large-group plan's)."""
    off = np.concatenate([[0], np.cumsum(np.asarray(sizes, np.int64))])
    n = int(off[-1])
    out = []
    for b in range((n + h - 1) // h):
        g0 = int(np.searchsorted(off, b * h, "left"))
        g1 = int(np.searchsorted(off, min(n, (b + 1) * h), "left"))
        if g1 > g0 and off[g1] - off[g1 - 1] > h:
            g1 -= 1
        out.append((max(g1 - g0, 0), int(off[g1] - off[g0]) if g1 > g0 else 0))
    return out


def window_layout(rng) -> tuple[list[int], dict]:
    """Group sizes (in first-occurrence order) that give k_quantile_small each window shape it has to handle ->
    (sizes, {shape: (window, (groups, keys))}), the expected small_windows() entry of each shape's window."""
    h = QS_H
    sizes = [1] * h                                   # W0: h singletons, local ids up to h - 1 beside the 0xFFFF padding
    sizes += [h - 1, h]                               # W1: a group starting exactly at the window start; the last group
    #                                                   starts at the window's last row and has h rows: 2h - 1 keys
    sizes += [h + 1]                                  # W2: next to it a group of h + 1 rows starting in W2: dropped (large)
    #                                                   W3: no group starts in it (the large group covers it)
    sizes += [1, h]                                   # W4: 1 + h = h + 1 keys, padded to a 2h-key network
    sizes += [5000]                                   # W5, W6: a large group, then a window it covers
    sizes += [int(s) for s in rng.integers(1, 60, 200)]
    pad = -sum(sizes) % h
    if pad:
        sizes.append(pad)                             # ends exactly at a window start
    at = sum(sizes) // h
    sizes += [h, h + 1]                               # a group of h rows filling a window, then h + 1 rows from the next start
    sizes += [int(s) for s in rng.integers(1, 9, 300)]  # a ragged last window
    shapes = {"singletons": (0, (h, h)), "start_at_window_start_2h_minus_1_keys": (1, (2, 2 * h - 1)),
              "large_last_group_dropped": (2, (0, 0)), "empty_after_large_group": (3, (0, 0)), "h_plus_1_keys": (4, (2, h + 1)),
              "h_rows_at_window_start": (at, (1, h)), "large_group_at_window_start": (at + 1, (0, 0))}
    return sizes, shapes


def dense_rank_bytes(values, descending: bool = False) -> tuple[np.ndarray, np.ndarray]:
    """Dense 1-based rank of bytes / None in unsigned byte order (Python's bytes comparison: a proper prefix first) from
    sorted() over the distinct values -> (uint32 ranks, 0 where null; validity)"""
    distinct = sorted({v for v in values if v is not None}, reverse=descending)
    rank = {v: i + 1 for i, v in enumerate(distinct)}
    r = np.fromiter((0 if v is None else rank[v] for v in values), np.uint32, count=len(values))
    return r, np.fromiter((v is not None for v in values), bool, count=len(values))


def refinement_rounds(values) -> tuple[int, int]:
    """Rounds of the string-rank refinement over the distinct values (the MSD loop of string_rank.cu): the key of round r
    is (bytes [7r, 7r + 7), min(len - 7r, 8)); buckets of one member drop out.  -> (rounds, rounds in which every active
    value had the same key, so nothing was sorted)"""
    buckets = [sorted({v for v in values if v is not None})]
    buckets = [b for b in buckets if len(b) > 1]
    rounds = skipped = 0
    while buckets:
        r = rounds * 7

        def key(v):
            return v[r:r + 7], min(max(len(v) - r, 0), 8)
        if len({key(v) for b in buckets for v in b}) == 1:
            skipped += 1
        else:
            split = []
            for b in buckets:
                parts = {}
                for v in b:
                    parts.setdefault(key(v), []).append(v)
                split += [p for p in parts.values() if len(p) > 1]
            buckets = split
        rounds += 1
    return rounds, skipped


def radix_passes(keys) -> int:
    """8-bit digits in which the unsigned keys differ: the passes of the radix sort over them"""
    k = np.asarray(keys)
    if k.size < 2:
        return 0
    vary = int(np.bitwise_and.reduce(k)) ^ int(np.bitwise_or.reduce(k))
    return sum(1 for d in range(k.dtype.itemsize) if (vary >> (8 * d)) & 0xFF)
