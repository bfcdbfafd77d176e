"""Inputs, exact numpy references and branch restatements shared by the window-family plan tests
(tests/test_gpu_window_plans.py) and their CPU cross-checks (tests/test_window_cases.py).

- Builders: partition ids whose segment heads sit where the kernels change behaviour (look-back windows, warp lanes,
  tile edges, block and sub-block edges), periodic times for rolling_*_by.
- References that stay exact at 1e7 - 1e8 rows: integer scans and window sums by uint64 prefix differences (wrapping is
  then exact), counts by prefix sums of the validity, min / max by segmented accumulate or a sparse table (two lookups per
  window), float sums and means of exactly summable values (integers times 2^-k, sums far below 2^53) by int64 prefix
  sums.  On such values every bracketing of the float sum is exact, so the parallel plans compare with ==.
- Restatements of the branch each position takes inside one kernel, which the launch profile cannot show: window_state
  (rolling.cu), window_global and k_rollby_out's staged selection (rolling_by.cu) with the sparse-table level they read,
  and the tiles of k_over_scan that hold a segment head (window.cu).  A GPU test asserts that its input reaches every
  branch it claims, so a shape that stops reaching one fails instead of passing silently.
"""
from __future__ import annotations

import numpy as np

# window.cu
OS_THREADS, OS_ITEMS = 256, 8
OS_TILE = OS_THREADS * OS_ITEMS          # 2048 positions per k_over_scan tile
OS_WARP_SPAN = 32 * OS_ITEMS             # 256 consecutive positions per warp: 8 rounds of 32 lanes
OS_LOOKBACK = 32 * OS_TILE               # one look-back window: 32 predecessor tiles, 65 536 positions
# rolling.cu / rolling.cuh
RT_TILE, RT_MAX_B = 1024, 128            # k_roll_tile: outputs per CTA, largest block of the one-pass plan
RS_TILE = 2048                           # k_roll_scan: positions per tile
# rolling_by.cu
RB_B, RB_SUB, RB_HALO = 1024, 32, 128    # blocks, staged sub-blocks, the small-window plan's halo

U32 = np.uint64(0xFFFFFFFF)


def grid_threads(sm: int) -> int:
    """threads of a grid-stride launch at its cap: grid_for(n, 256) = 8 SM x 256, grid_for(G, 128, 16) = 16 SM x 128 and
    grid_for(G, 64, 32) = 32 SM x 64 all come to 2048 SM threads (270 336 at 132 SMs)"""
    return sm * 2048


def scan_wave(sm: int) -> int:
    """positions k_over_scan covers with one wave of its min(tiles, 8 SM) CTAs"""
    return 8 * sm * OS_TILE


# ---------------------------------------------------------------------------------------------------- builders
def gid_from_heads(heads: np.ndarray) -> np.ndarray:
    """Int64 partition ids, one run per segment, ascending: the partition order of such ids is the rows themselves"""
    h = np.asarray(heads, bool).copy()
    h[0] = True
    return np.cumsum(h, dtype=np.int64) - 1


def heads_at(n: int, at) -> np.ndarray:
    h = np.zeros(n, bool)
    h[0] = True
    at = np.asarray([a for a in at if 0 <= a < n], np.int64)
    h[at] = True
    return h


def tile_edge_heads(n: int, tile: int) -> np.ndarray:
    """heads on every lane-0 and lane-31 position of every warp round of tile `tile` (so also its first and last position)"""
    base = tile * OS_TILE
    offs = np.arange(0, OS_TILE, 32)
    return heads_at(n, np.concatenate([base + offs, base + offs + 31]))


def alternating_heads(n: int, a: int = 1, b: int = OS_TILE + 1) -> np.ndarray:
    """segments of a, b, a, b, ... positions"""
    at, p, k = [], 0, 0
    while p < n:
        at.append(p)
        p += a if k % 2 == 0 else b
        k += 1
    return heads_at(n, at)


def scan_heads(gid, reverse: bool) -> np.ndarray:
    """heads in k_over_scan's logical order (reverse: position n - 1 - i): where the id changes from the previous element"""
    g = np.asarray(gid)[::-1] if reverse else np.asarray(gid)
    h = np.ones(len(g), bool)
    h[1:] = g[1:] != g[:-1]
    return h


def exact_floats(rng, n: int, dtype, scale_bits: int = 4, lim: int = 1 << 10):
    """(values, integer numerators): k * 2^-scale_bits with |k| <= lim, exact in Float32 and Float64"""
    k = rng.integers(-lim, lim + 1, n).astype(np.int64)
    return (k.astype(np.float64) / (1 << scale_bits)).astype(dtype), k


# ---------------------------------------------------------------------------------------------------- scans
def seg_start(heads: np.ndarray) -> np.ndarray:
    """index of the segment head of every position"""
    idx = np.where(heads, np.arange(len(heads)), 0)
    return np.maximum.accumulate(idx)


def _prefix_diff_u64(u: np.ndarray, heads: np.ndarray) -> np.ndarray:
    c = np.cumsum(u, dtype=np.uint64)
    ce = np.concatenate([np.zeros(1, np.uint64), c])
    return c - ce[seg_start(heads)]


def _as_u64(x: np.ndarray) -> np.ndarray:
    x = np.asarray(x)
    if x.dtype == np.bool_:
        return x.astype(np.uint64)
    if x.dtype.kind == "i":
        return x.astype(np.int64).view(np.uint64)
    return x.astype(np.uint64)


def cum_ref(kind: str, x, valid, gid, reverse: bool, dtype: str, frac=None):
    """Exact segmented cum_* in row order (positions = rows: gid None or runs of ascending ids).
    x: the values (Bool as numpy bool); valid: bool array or None; frac: for float cum_sum the integer numerators of
    exact_floats (x = frac / 16).  -> output values (0 where the output is null)"""
    n = len(x)
    valid = np.ones(n, bool) if valid is None else np.asarray(valid, bool)
    xs, vs = (x[::-1], valid[::-1]) if reverse else (x, valid)
    heads = scan_heads(np.zeros(n, np.int64) if gid is None else gid, reverse)
    if kind == "cum_count":
        out = _prefix_diff_u64(vs.astype(np.uint64), heads).astype(np.uint32)
    elif kind == "cum_sum" and dtype.startswith("float"):
        f = frac[::-1] if reverse else frac
        s = _prefix_diff_u64(np.where(vs, f, 0).astype(np.int64).view(np.uint64), heads).view(np.int64)
        out = (s.astype(np.float64) / 16.0).astype(dtype)
    elif kind == "cum_sum":
        s = _prefix_diff_u64(np.where(vs, _as_u64(xs), np.uint64(0)), heads)
        odt = {"bool": np.uint32, "int32": np.int32, "uint32": np.uint32, "int64": np.int64, "uint64": np.uint64}[dtype]
        out = s.astype(np.uint32).view(np.int32).astype(odt) if dtype == "int32" else s.astype(odt) if odt != np.int64 else s.view(np.int64)
    else:
        starts = np.flatnonzero(heads)
        ends = np.append(starts[1:], n)
        if kind == "cum_prod":
            u = np.where(vs, _as_u64(xs), np.uint64(1))
            out = np.empty(n, np.uint64)
            for a, b in zip(starts, ends):
                out[a:b] = np.multiply.accumulate(u[a:b], dtype=np.uint64)
            out = out.view(np.int64) if dtype in ("int32", "int64", "bool") else out
        else:
            fn = np.minimum if kind == "cum_min" else np.maximum
            if xs.dtype.kind == "f":
                ident = np.inf if kind == "cum_min" else -np.inf
            else:
                info = np.iinfo(xs.dtype)
                ident = info.max if kind == "cum_min" else info.min
            u = np.where(vs, xs, xs.dtype.type(ident))
            out = np.empty(n, xs.dtype)
            for a, b in zip(starts, ends):
                out[a:b] = fn.accumulate(u[a:b])
    out = np.where(vs, out, out.dtype.type(0)) if kind != "cum_count" else out
    return out[::-1].copy() if reverse else out


# ---------------------------------------------------------------------------------------------------- windows
def fixed_bounds(n: int, w: int, center: bool, gid=None):
    """(s, e, lo, hi) per position: the window [i - L, i + R) clipped to its segment [lo, hi) (positions = rows)"""
    if center:
        R = w // 2 + (w & 1)
        L = w - R
    else:
        L, R = w - 1, 1
    L, R = min(L, n), min(R, n)
    i = np.arange(n, dtype=np.int64)
    if gid is None:
        lo, hi = np.zeros(n, np.int64), np.full(n, n, np.int64)
    else:
        heads = scan_heads(gid, False)
        lo = seg_start(heads)
        ends = np.append(np.flatnonzero(heads)[1:], n)
        hi = ends[np.cumsum(heads) - 1]
    return np.maximum(i - L, lo), np.minimum(i + R, hi), lo, hi


def by_bounds(t, P: int, closed: str, gid=None):
    """(s, e) of rolling_*_by for times ascending inside each segment (positions = rows, no null `by`), by searchsorted
    on (segment, time) composite keys; times stay far from the Int64 limits"""
    t = np.asarray(t, np.int64)
    if gid is not None:
        span = int(t.max() - t.min()) + 2 * P + 2
        key = np.asarray(gid, np.int64) * span + (t - t.min() + P + 1)
    else:
        key = t
    s = np.searchsorted(key, key - P, side="left" if closed in ("left", "both") else "right")
    e = np.searchsorted(key, key, side="right" if closed in ("right", "both") else "left")
    return s.astype(np.int64), e.astype(np.int64)


def window_sum_u64(u: np.ndarray, s: np.ndarray, e: np.ndarray) -> np.ndarray:
    c = np.concatenate([np.zeros(1, np.uint64), np.cumsum(u, dtype=np.uint64)])
    return c[e] - c[s]


def window_count(valid, s, e):
    c = np.concatenate([[0], np.cumsum(np.asarray(valid, np.int64))])
    return c[e] - c[s]


class SparseTable:
    """min or max over any [s, e) of an array in two lookups; levels of 2^k, O(n log n) memory"""

    def __init__(self, x: np.ndarray, is_max: bool):
        self.fn = np.maximum if is_max else np.minimum
        self.lv = [np.asarray(x)]
        k = 1
        while (1 << k) <= len(x):
            p = self.lv[-1]
            h = 1 << (k - 1)
            self.lv.append(self.fn(p[:-h], p[h:]))
            k += 1

    def query(self, s: np.ndarray, e: np.ndarray) -> np.ndarray:
        """e > s everywhere"""
        ln = e - s
        k = np.floor(np.log2(np.maximum(ln, 1))).astype(np.int64)
        out = np.empty(len(s), self.lv[0].dtype)
        for lev in np.unique(k):
            m = k == lev
            a = self.lv[lev]
            out[m] = self.fn(a[s[m]], a[e[m] - (1 << lev)])
        return out


def window_minmax(x, valid, s, e, is_max: bool):
    """(value, count of non-null) per window; value undefined where the count is 0"""
    x = np.asarray(x)
    if x.dtype.kind == "f":
        ident = -np.inf if is_max else np.inf
    else:
        info = np.iinfo(x.dtype)
        ident = info.min if is_max else info.max
    u = np.where(valid, x, x.dtype.type(ident)) if valid is not None else x
    cnt = window_count(np.ones(len(x), bool) if valid is None else valid, s, e)
    val = np.zeros(len(s), x.dtype)
    ne = e > s
    val[ne] = SparseTable(u, is_max).query(s[ne], e[ne])
    return val, cnt


def rolling_ref(kind: str, x, valid, s, e, min_samples: int, frac=None, dtype=None):
    """Exact rolling_* over windows [s, e) for sum / mean / min / max.  -> (values, valid).  frac: integer numerators of
    exact_floats values (x = frac / 16) for float sum / mean."""
    n = len(x)
    v = np.ones(n, bool) if valid is None else np.asarray(valid, bool)
    cnt = window_count(v, s, e)
    dtype = dtype or (str(np.asarray(x).dtype) if np.asarray(x).dtype != np.bool_ else "bool")
    if kind in ("rolling_min", "rolling_max"):
        val, _ = window_minmax(x, v, s, e, kind == "rolling_max")
        return val, (cnt > 0) & (cnt >= min_samples)
    if dtype.startswith("float"):
        sm = window_sum_u64(np.where(v, frac, 0).astype(np.int64).view(np.uint64), s, e).view(np.int64).astype(np.float64) / 16.0
        if kind == "rolling_sum":
            return sm.astype(dtype), cnt >= min_samples
        T = np.float32 if dtype == "float32" else np.float64
        with np.errstate(invalid="ignore", divide="ignore"):
            mean = T(1) * sm.astype(T) / cnt.astype(T)
        return mean, (cnt > 0) & (cnt >= min_samples)
    assert kind == "rolling_sum"
    sm = window_sum_u64(np.where(v, _as_u64(x), np.uint64(0)), s, e)
    if dtype in ("bool", "uint32"):
        out = sm.astype(np.uint32)
    elif dtype == "int32":
        out = sm.astype(np.uint32).view(np.int32)
    elif dtype == "int64":
        out = sm.view(np.int64)
    else:
        out = sm
    return out, cnt >= min_samples


# ---------------------------------------------------------------------------------------------------- branches
TWO, PRE, SUF = 0, 1, 2
STATE_NAMES = {TWO: "two blocks", PRE: "prefix", SUF: "suffix"}


def window_state_branch(s, e, lo, B: int) -> np.ndarray:
    """the branch of window_state (rolling.cu) for every position: TWO (suffix[s] + prefix[l]), PRE or SUF"""
    l = e - 1
    b = l - l % B
    return np.where(s < b, TWO, np.where(s == np.maximum(b, lo), PRE, SUF))


def tile_staging(n: int, L: int, R: int, B: int):
    """k_roll_tile's staged range per CTA: (A, len, last) with last = min(n - 1, o1 - 2 + R), the last position an output
    window of the CTA reaches"""
    o0 = np.arange(0, n, RT_TILE, dtype=np.int64)
    o1 = np.minimum(n, o0 + RT_TILE)
    A = np.maximum(o0 - L, 0) // B * B
    last = np.minimum(n - 1, o1 - 2 + R)
    ln = np.minimum(n, (last // B + 1) * B) - A
    return A, ln, last


def segment_flags(n: int, gid=None):
    """(head, end): head[p] = p starts a segment, end[q] for q in [0, n] = q is one past a segment's last position"""
    if gid is None:
        head = np.zeros(n, bool)
        head[0] = True
    else:
        head = scan_heads(gid, False)
    end = np.zeros(n + 1, bool)
    end[n] = True
    end[1:n] = head[1:]
    return head, end


def rollby_tile_plan(s, e) -> bool:
    """ByPlan's choice: the one-pass small-window plan when no window is wider than RB_HALO (null-`by` rows: s = e)"""
    return int(np.max(np.asarray(e) - np.asarray(s), initial=0)) <= RB_HALO


def rollby_branch(s, e, n: int, tile: bool, gid=None):
    """The branch k_rollby_out takes for every window [s, e) (rows with e > s; positions = rows).
    -> dict name -> bool mask, and `level`: the sparse-table level k read by a cross-level lookup (-1 elsewhere).
    In the stage: 'stage_cross' (Q[l] + P[r] across sub-blocks; 'stage_l_eq_r' / 'stage_k' for the middle), 'stage_P',
    'stage_Q_sub' (r ends a sub-block), 'stage_Q_len' (r is the stage's last position), 'stage_Q_seg' (r ends a segment),
    'stage_fold'.  Outside it: the tile plan's 'tile_fold_global'; the general plan's window_global 'g_adjacent', 'g_l_eq_r',
    'g_k', 'g_pre_block', 'g_pre_head', 'g_suf_block', 'g_suf_n', 'g_suf_seg', 'g_fold'."""
    s = np.asarray(s, np.int64)
    e = np.asarray(e, np.int64)
    i = np.arange(len(s), dtype=np.int64)
    head, end = segment_flags(n, gid)
    o0 = i // RB_B * RB_B
    A = np.maximum(0, o0 - RB_HALO) if tile else o0
    ln = np.minimum(n, o0 + RB_B + RB_HALO if tile else o0 + RB_B) - A
    ne = e > s
    ins = ne & (s >= A) & (e <= A + ln)
    l, r = s - A, e - 1 - A
    sl, sr = l // RB_SUB, r // RB_SUB
    m = {}
    cross = ins & (sl < sr)
    m["stage_cross"] = cross
    m["stage_l_eq_r"] = cross & (sr - sl == 2)
    m["stage_k"] = cross & (sr - sl > 2)
    one = ins & ~cross
    sc = np.clip(s, 0, n - 1)
    ec = np.clip(e, 0, n)
    m["stage_P"] = one & ((l % RB_SUB == 0) | head[sc])
    rest = one & ~m["stage_P"]
    sub_end = r % RB_SUB == RB_SUB - 1
    m["stage_Q_sub"] = rest & sub_end
    m["stage_Q_len"] = rest & ~sub_end & (r == ln - 1)
    m["stage_Q_seg"] = rest & ~sub_end & (r != ln - 1) & end[ec]
    m["stage_fold"] = rest & ~sub_end & (r != ln - 1) & ~end[ec]
    out = ne & ~ins
    level = np.full(len(s), -1, np.int64)
    if tile:
        m["tile_fold_global"] = out
    else:
        bs, be = s // RB_B, (e - 1) // RB_B
        cr = out & (bs < be)
        m["g_adjacent"] = cr & (be - bs == 1)
        m["g_l_eq_r"] = cr & (be - bs == 2)
        m["g_k"] = cr & (be - bs > 2)
        lk, rk = bs + 1, be - 1
        x = np.where(m["g_k"], lk ^ rk, 1)
        level = np.where(m["g_k"], np.floor(np.log2(np.maximum(x, 1))).astype(np.int64), -1)
        one = out & (bs == be)
        m["g_pre_block"] = one & (s % RB_B == 0)
        m["g_pre_head"] = one & (s % RB_B != 0) & head[sc]
        pre = m["g_pre_block"] | m["g_pre_head"]
        m["g_suf_block"] = one & ~pre & (e % RB_B == 0)
        m["g_suf_n"] = one & ~pre & (e % RB_B != 0) & (e == n)
        m["g_suf_seg"] = one & ~pre & (e % RB_B != 0) & (e != n) & end[ec]
        m["g_fold"] = one & ~pre & (e % RB_B != 0) & (e != n) & ~end[ec]
    m["level"] = level
    return m


def sparse_levels(n: int) -> int:
    """K of ByPlan: the smallest K with 2^K >= nb blocks of RB_B"""
    nb = (n + RB_B - 1) // RB_B
    K = 0
    while (1 << K) < nb:
        K += 1
    return K


def head_tiles(gid, reverse: bool) -> np.ndarray:
    """the k_over_scan tiles (in scan order) that hold a segment head other than position 0"""
    h = scan_heads(gid, reverse)
    h[0] = False
    return np.unique(np.flatnonzero(h) // OS_TILE)


def head_lanes(gid, reverse: bool) -> dict:
    """where the segment heads sit in their warp round and tile: counts of lane 0, lane 31, tile-first, tile-last"""
    h = np.flatnonzero(scan_heads(gid, reverse))
    h = h[h > 0]
    return {"lane0": int(np.sum(h % 32 == 0)), "lane31": int(np.sum(h % 32 == 31)),
            "tile_first": int(np.sum(h % OS_TILE == 0)), "tile_last": int(np.sum(h % OS_TILE == OS_TILE - 1))}


def longest_segment_after_head_tile(gid, reverse: bool) -> int:
    """the length of the longest segment that starts in a tile which holds a head: the segments a look-back might have to
    walk more than one 32-tile window for"""
    h = scan_heads(gid, reverse)
    st = np.flatnonzero(h)
    ln = np.diff(np.append(st, len(h)))
    return int(ln.max())


# ---------------------------------------------------------------------------------------------------- brute force
def reduce_by_state_branch(s, e, lo, B: int, n: int, hi):
    """window_state evaluated with position-list states (concatenation): which positions each branch's combination covers.
    The prefix of p starts at max(block start, segment head); the suffix of p ends at min(block end, segment end)."""
    out = []
    br = window_state_branch(s, e, lo, B)
    for i in range(len(s)):
        l = e[i] - 1
        b = l - l % B
        pre = list(range(max(b, lo[i]), l + 1))
        sblk_end = min((s[i] // B + 1) * B, hi[i])
        suf = list(range(s[i], sblk_end))
        out.append(suf + pre if br[i] == TWO else pre if br[i] == PRE else suf)
    return out


def reduce_by_rollby_branch(s, e, n: int, tile: bool, gid=None):
    """rollby_branch evaluated with position-list states: the positions each chosen combination covers (None: empty).
    Staged sub-blocks are aligned at the stage start A, global blocks at 0; a prefix restarts at a segment head, a suffix
    stops at a segment end or at the end of what holds it (the stage, or the column)."""
    m = rollby_branch(s, e, n, tile, gid)
    head, end = segment_flags(n, gid)

    def pre(p, size, base):
        a = p
        while (a - base) % size and not head[a]:
            a -= 1
        return list(range(a, p + 1))

    def suf(p, size, base, limit):
        b = p + 1
        while (b - base) % size and not end[b] and b < limit:
            b += 1
        return list(range(p, b))

    res = []
    for i in range(len(s)):
        a, b = int(s[i]), int(e[i])
        if b <= a:
            res.append(None)
            continue
        o0 = i // RB_B * RB_B
        A = max(0, o0 - RB_HALO) if tile else o0
        stop = min(n, o0 + RB_B + RB_HALO if tile else o0 + RB_B)
        if m["stage_cross"][i]:
            sl, sr = (a - A) // RB_SUB, (b - 1 - A) // RB_SUB
            res.append(suf(a, RB_SUB, A, stop) + list(range(A + (sl + 1) * RB_SUB, A + sr * RB_SUB)) + pre(b - 1, RB_SUB, A))
        elif m["stage_P"][i]:
            res.append(pre(b - 1, RB_SUB, A))
        elif m["stage_Q_sub"][i] or m["stage_Q_len"][i] or m["stage_Q_seg"][i]:
            res.append(suf(a, RB_SUB, A, stop))
        elif m["stage_fold"][i] or (tile and m["tile_fold_global"][i]):
            res.append(list(range(a, b)))
        else:
            bs, be = a // RB_B, (b - 1) // RB_B
            if bs < be:
                res.append(suf(a, RB_B, 0, n) + list(range((bs + 1) * RB_B, be * RB_B)) + pre(b - 1, RB_B, 0))
            elif m["g_pre_block"][i] or m["g_pre_head"][i]:
                res.append(pre(b - 1, RB_B, 0))
            elif m["g_suf_block"][i] or m["g_suf_n"][i] or m["g_suf_seg"][i]:
                res.append(suf(a, RB_B, 0, n))
            else:
                res.append(list(range(a, b)))
    return res
