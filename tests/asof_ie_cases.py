"""Inputs and numpy restatements shared by the asof / inequality-join plan tests (tests/test_gpu_join_asof_ie_plans.py)
and their CPU cross-checks (tests/test_asof_ie_cases.py): the asof `by` rule over every group at once, the right windows
k_asof_search stages per tile, the inequality join's per-row pair counts from a y-domain restatement and its brute force
on sampled rows, and a CPU restatement of the string hash (strings.cu: str_hash_bytes) with inputs that collide in it."""
from __future__ import annotations

import numpy as np

import asof_oracle as ao

AS_ITEMS, AS_THREADS = 8, 256
AS_TILE = AS_ITEMS * AS_THREADS          # left rows per k_asof_search CTA
AS_WIN_BYTES = 16384                     # right window staged in shared memory
TS_THREADS = 1024                        # k_asof_tiles_sorted: one CTA
IE_CROWS = 256                           # left rows per k_ie_count CTA
IE_WSLOTS, IE_WARPS = 512, 8             # output slots per k_ie_emit warp, warps per CTA


def grid_threads(sm: int) -> int:
    """threads of a grid_for(n, 256) launch at its cap: 8 CTAs per SM x 256 threads"""
    return sm * 8 * 256


def tiles_per_thread(nl: int) -> int:
    """`per` of k_asof_tiles_sorted: tiles each of its 1024 threads checks"""
    ntiles = (nl + AS_TILE - 1) // AS_TILE
    return (ntiles + TS_THREADS - 1) // TS_THREADS


def tree_levels(m: int) -> int:
    """levels of the two-predicate merge-sort tree: the smallest L with 2^(L-1) >= m"""
    L = 1
    while (1 << (L - 1)) < m:
        L += 1
    return L


# ---------------------------------------------------------------------------------------------------- asof: windows
def tile_windows(left, right):
    """The right window [wlo, whi) k_asof_search computes for every tile of the left side (no `by`): blo / bhi bound the
    tile's smallest / largest non-null key in the non-null right rows [z, e), widened by one on each side and clipped to
    [z, e).  left / right = (values, valid | None).  -> list of (wlo, whi) per tile, (0, 0) for a tile without keys."""
    lv, lvalid = left
    rv, rvalid = right
    lvalid = np.ones(len(lv), bool) if lvalid is None else lvalid
    rvalid = np.ones(len(rv), bool) if rvalid is None else rvalid
    z, e = (int(np.argmax(rvalid)) if rvalid.any() else len(rv)), len(rv)
    rk, lk = ao.total_keys(rv[z:]), ao.total_keys(lv)
    out = []
    for t in range(0, len(lv), AS_TILE):
        k = lk[t:t + AS_TILE][lvalid[t:t + AS_TILE]]
        if k.size == 0 or z >= e:
            out.append((0, 0))
            continue
        blo = z + int(np.searchsorted(rk, k.min(), "left"))
        bhi = z + int(np.searchsorted(rk, k.max(), "right"))
        out.append((max(z, blo - 1), min(e, bhi + 1)))
    return out


def staged(window, itemsize: int) -> bool:
    """whether k_asof_search reads that window from shared memory"""
    return window[1] > window[0] and (window[1] - window[0]) * itemsize <= AS_WIN_BYTES


# ---------------------------------------------------------------------------------------------------- asof: `by`
def rule_asof_by(left, right, strategy, allow_eq=True, tol=None, left_groups=None, right_groups=None):
    """The per-row rule with `by` over all groups at once: right rows sorted by (group, row), each left row searches its
    group's non-null rows through (group, dense rank of the total-order key) composite keys, so no per-group loop.  Only
    valid when every group's right rows are nulls first, then sorted.  left / right = (values, valid | None); *_groups:
    int64 group ids, -1 for a null `by` key.  -> (uint32 index, bool valid)"""
    lv, lvalid = left
    rv, rvalid = right
    nl, nr = len(lv), len(rv)
    lvalid = np.ones(nl, bool) if lvalid is None else np.asarray(lvalid, bool)
    rvalid = np.ones(nr, bool) if rvalid is None else np.asarray(rvalid, bool)
    lg, rg = np.asarray(left_groups, np.int64), np.asarray(right_groups, np.int64)
    rsel = np.nonzero((rg >= 0) & rvalid)[0]
    rsel = rsel[np.argsort(rg[rsel], kind="stable")]
    lrows = np.nonzero((lg >= 0) & lvalid)[0]
    out = np.full(nl, -1, np.int64)
    if len(rsel) and len(lrows):
        keys = np.concatenate([ao.total_keys(rv[rsel]), ao.total_keys(lv[lrows])])
        _, rank = np.unique(keys, return_inverse=True)
        rank = rank.reshape(-1).astype(np.int64)
        span = int(rank.max()) + 1
        rk = rg[rsel] * span + rank[:len(rsel)]
        lk = lg[lrows] * span + rank[len(rsel):]
        g = lg[lrows]
        z = np.searchsorted(rg[rsel], g, "left")
        e = np.searchsorted(rg[rsel], g, "right")
        r = rv[rsel]
        x = lv[lrows]
        n = len(r)
        fl = r.dtype.kind == "f"

        def at(p):
            return r[np.clip(p, 0, n - 1)]
        if strategy == ao.BACKWARD:
            j = np.searchsorted(rk, lk, "right" if allow_eq else "left") - 1
            j = np.where(j >= z, j, -1)
        elif strategy == ao.FORWARD:
            j = np.searchsorted(rk, lk, "left" if allow_eq else "right")
            j = np.where(j < e, j, -1)
        else:
            U = np.searchsorted(rk, lk, "right")
            if fl:
                U = np.where((U < e) & np.isnan(at(U)), e, U)
            exact = (U > z) & (at(U - 1) == x) if allow_eq else np.zeros(len(x), bool)
            Ue = np.where(U < e, np.searchsorted(rk, rk[np.clip(U, 0, n - 1)], "right") - 1, U)
            lb = np.minimum(np.searchsorted(rk, lk, "left"), Ue)
            lb_ok = lb < Ue
            if fl:
                lb_ok &= ~np.isnan(at(lb))
            L = np.where(lb_ok, lb - 1, Ue - 1)
            hasL, hasU = L >= z, Ue < e
            with np.errstate(invalid="ignore"):
                both = np.where(ao._diff(x, at(Ue)) <= ao._diff(x, at(L)), Ue, L)
            j = np.where(hasL & hasU, both, np.where(hasU, Ue, np.where(hasL, L, -1)))
            j = np.where(exact, U - 1, j)
        if tol is not None:
            t = ao._diff(np.array([tol], r.dtype), np.zeros(1, r.dtype))[0]
            with np.errstate(invalid="ignore"):
                j = np.where((j >= 0) & (ao._diff(x, at(j)) <= t), j, -1)
        out[lrows] = np.where(j >= 0, rsel[np.clip(j, 0, n - 1)], -1)
    valid = out >= 0
    return np.where(valid, out, 0xFFFFFFFF).astype(np.uint32), valid


def kernel_group_order(left_groups, right_groups, left_valid=None):
    """The order the `by` plan's stable sorts give the rows of each side: a group's id is the first row holding it in
    left ‖ right, so groups come in the order they first appear there, and rows without a group (a null `by` key; on the
    left also a null `on` value) come last.  k_asof_segments walks the right rows in this order, k_asof_left_groups the
    left rows.  *_groups: int64 group ids, -1 for a null `by` key.  -> (left rows, right rows) in that order"""
    lg, rg = np.asarray(left_groups, np.int64), np.asarray(right_groups, np.int64)
    g = np.concatenate([lg, rg])
    n, nl = len(g), len(lg)
    ids, first = np.unique(g, return_index=True)
    key = first[np.searchsorted(ids, g)]
    key[g < 0] = n
    if left_valid is not None:
        key[:nl][~np.asarray(left_valid, bool)] = n
    return np.argsort(key[:nl], kind="stable"), np.argsort(key[nl:], kind="stable")


def by_sides(rng, nl, nr, n_groups, dtype="int64", lnull=0.02, bynull=0.02, right_null_groups=0, one_side=0):
    """Random `by` inputs: left `on` sorted globally with lnull nulls; right rows in random group order, each group nulls
    first then sorted; group ids 0 .. n_groups - 1 (n_groups = nl: one per left row); bynull of the `by` keys null on both
    sides (-1); the first right_null_groups groups have only null right rows; `one_side` groups appear on the left only
    and as many on the right only.  -> (L, R, left groups, right groups) with L / R = (values, valid)"""
    lv = np.sort(rng.integers(0, 4 * (nl + nr) + 8, nl)).astype(dtype)
    lg = rng.integers(0, n_groups, nl).astype(np.int64)
    rg = rng.integers(0, n_groups, nr).astype(np.int64)
    if one_side:
        lg[rng.random(nl) < 0.05] = n_groups + rng.integers(0, one_side, 1)[0]
        rg[rng.random(nr) < 0.05] = n_groups + one_side + rng.integers(0, one_side, 1)[0]
    rvals = rng.integers(0, 4 * (nl + nr) + 8, nr)
    rvalid = rng.random(nr) >= 0.02
    rvalid[np.isin(rg, np.arange(right_null_groups))] = False
    # each group's values, nulls first then ascending, go to the group's rows in row order
    order = np.lexsort((rvals, rvalid, rg))
    srt = np.argsort(rg, kind="stable")
    rv = np.empty(nr, np.int64)
    rva = np.empty(nr, bool)
    rv[srt] = rvals[order]
    rva[srt] = rvalid[order]
    lg[rng.random(nl) < bynull] = -1
    rg[rng.random(nr) < bynull] = -1
    lvalid = rng.random(nl) >= lnull
    return (lv, lvalid), (rv.astype(dtype), rva), lg, rg


def groups_as_by(g) -> np.ndarray:
    """group ids -> (int64 `by` column, validity)"""
    return np.where(g >= 0, g, 0).astype(np.int64), g >= 0


# ---------------------------------------------------------------------------------------------------- inequality join
IE_OP = {"<": np.less, "<=": np.less_equal, ">": np.greater, ">=": np.greater_equal}


def ie_keys(values) -> np.ndarray:
    return ao.total_keys(values)


def ie_range(sorted_keys, k, op):
    """[a, b) of an ascending key array whose keys r satisfy `k op r`"""
    if op == "<":
        return np.searchsorted(sorted_keys, k, "right"), np.full(len(k), len(sorted_keys))
    if op == "<=":
        return np.searchsorted(sorted_keys, k, "left"), np.full(len(k), len(sorted_keys))
    if op == ">":
        return np.zeros(len(k), np.int64), np.searchsorted(sorted_keys, k, "left")
    return np.zeros(len(k), np.int64), np.searchsorted(sorted_keys, k, "right")


def ie_counts(left, right, ops) -> np.ndarray:
    """Exact pair count of every left row (0 for a row with a null predicate value).  One predicate: one searchsorted.
    Two predicates: the live right rows split by their y value (few distinct values); per y value, a searchsorted of the
    left x keys in that value's sorted x keys; a cumulative sum over the y values in total order; each left row takes the
    y values its second predicate accepts, which are a prefix or a suffix.  left / right: one (values, valid | None) per
    predicate."""
    nl, nr = len(left[0][0]), len(right[0][0])
    lok = np.ones(nl, bool)
    rok = np.ones(nr, bool)
    for (_, lm), (_, rm) in zip(left, right):
        if lm is not None:
            lok &= lm
        if rm is not None:
            rok &= rm
    lx = ie_keys(left[0][0])
    rx = ie_keys(right[0][0])[rok]
    if len(ops) == 1:
        a, b = ie_range(np.sort(rx), lx, ops[0])
        return np.where(lok, b - a, 0).astype(np.int64)
    ry = ie_keys(right[1][0])[rok]
    ly = ie_keys(left[1][0])
    yvals, cls = np.unique(ry, return_inverse=True)
    cls = cls.reshape(-1)
    per = np.zeros((nl, len(yvals) + 1), np.int64)
    for c in range(len(yvals)):
        xs = np.sort(rx[cls == c])
        a, b = ie_range(xs, lx, ops[0])
        per[:, c + 1] = b - a
    cum = np.cumsum(per, axis=1)
    c0, c1 = ie_range(yvals, ly, ops[1])
    return np.where(lok, cum[np.arange(nl), c1] - cum[np.arange(nl), c0], 0).astype(np.int64)


def ie_brute_rows(left, right, ops, rows) -> list:
    """numpy brute force over every right row for the given left rows -> one sorted array of right rows per left row"""
    nr = len(right[0][0])
    rok = np.ones(nr, bool)
    for _, rm in right:
        if rm is not None:
            rok &= rm
    rkeys = [ie_keys(v) for v, _ in right]
    lkeys = [ie_keys(v) for v, _ in left]
    out = []
    for i in rows:
        m = rok.copy()
        for k, op in enumerate(ops):
            lm = left[k][1]
            if lm is not None and not lm[i]:
                m[:] = False
            m &= IE_OP[op](lkeys[k][i], rkeys[k])
        out.append(np.nonzero(m)[0])
    return out


# ---------------------------------------------------------------------------------------------------- string hash
M64 = (1 << 64) - 1
GOLD = 0x9E3779B97F4A7C15
SEEDS = [(0x2545F4914F6CDD1D * k) & M64 for k in (1, 2, 3, 4)]      # op_string_codes' four attempts


def str_mix(h: int, w: int) -> int:
    h = ((h ^ w) * 0xFF51AFD7ED558CCD) & M64
    return h ^ (h >> 29)


def str_hash_bytes(b: bytes, seed: int) -> int:
    """strings.cu str_hash_bytes: 8-byte little-endian words, a tail word xor-ed with a constant, then a final mix"""
    n = len(b)
    h = seed ^ ((n * GOLD) & M64)
    i = 0
    while i + 8 <= n:
        h = str_mix(h, int.from_bytes(b[i:i + 8], "little"))
        i += 8
    if i < n:
        h = str_mix(h, int.from_bytes(b[i:], "little") ^ 0xC4CEB9FE1A85EC53)
    h ^= h >> 33
    h = (h * 0xC4CEB9FE1A85EC53) & M64
    return h ^ (h >> 33)


def colliding_pair(seed: int, tag: bytes = b"") -> tuple[bytes, bytes]:
    """Two distinct 16-byte ASCII values with one hash under `seed`.  After the first word the states are mix(h0, a1) and
    mix(h0, b1); the second word is xor-ed into the state before the multiply, so b2 = a2 ^ mix(h0, a1) ^ mix(h0, b1)
    gives equal states from then on.  b1 is searched until that difference has no byte with its top bit set."""
    h0 = seed ^ ((16 * GOLD) & M64)
    a = b"collide:" + (b"A" + tag + b"-------")[:8]
    a1, a2 = int.from_bytes(a[:8], "little"), int.from_bytes(a[8:], "little")
    for k in range(1 << 20):
        b1 = int.from_bytes(b"B%07d" % k, "little")
        d = str_mix(h0, a1) ^ str_mix(h0, b1)
        if d & 0x8080808080808080 == 0:
            b = b1.to_bytes(8, "little") + (a2 ^ d).to_bytes(8, "little")
            return a, b
    raise AssertionError("no ASCII collision found")


# ---------------------------------------------------------------------------------------------------- asof: window case
WIN_WIDTHS = (2048, 2049, 4096, 4097)      # the staging limit of 8-byte keys and of 4-byte keys, and one past each
RUN_AT, RUN_LEN = 20_100, 3000             # grid index and length of a run of equal right values


def window_case(rng, dtype):
    """A left / right pair whose tiles have the right windows k_asof_search has to get right, for every key dtype.
    Right: 100 leading nulls, low extremes (integer MIN, MIN + 1; float -inf, -1e30), a strictly increasing grid with
    one run of RUN_LEN equal values at grid index RUN_AT, high extremes (integer MAX - 1; float 1e30, +inf, then 50 NaNs).
    Grid value j sits at 2j units; left keys take every unit between a tile's end points, so about half of them lie
    exactly halfway between two right keys (nearest's tie).  Left tiles (AS_TILE rows, 1 % nulls inside):
      0  the low extremes and grid 0 .. 300: the window is clipped at z
      1-4  windows of exactly WIN_WIDTHS entries
      5  only nulls
      6  keys up to one unit below the run: the window ends one entry into the run, which goes on past it
      7  keys on the run and just above it
      8  (partial) keys above the grid and the extremes (integer MAX, float NaN): the window is clipped at e
    Floats: zeros become -0.0 on the right and on every other left row.  -> (L, R) as (values, valid)"""
    dt = np.dtype(dtype)
    n_grid = 26_000
    units = np.concatenate([2 * np.arange(RUN_AT), np.full(RUN_LEN, 2 * RUN_AT), 2 * np.arange(RUN_AT + 1, n_grid)])
    if dt.kind == "f":
        lo_x, hi_x = [-np.inf, -1e30], [1e30, np.inf]

        def val(u):
            return (-20_000.0 + 0.5 * np.asarray(u, np.float64)).astype(dt)
    else:
        info = np.iinfo(dt)
        lo_x, hi_x = [info.min, info.min + 1], [info.max - 1]

        def val(u):
            return (np.asarray(u, np.uint64) + np.uint64(int(info.min) + 4 & ((1 << 64) - 1))).astype(np.uint64).view(np.int64).astype(dt) \
                if dt.itemsize == 8 else (np.asarray(u, np.int64) + int(info.min) + 4).astype(dt)
    z = 100
    nan_tail = 50 if dt.kind == "f" else 0
    rv = np.concatenate([np.zeros(z, dt), np.array(lo_x, dt), val(units), np.array(hi_x, dt), np.full(nan_tail, np.nan, dt) if nan_tail else np.zeros(0, dt)])
    rvalid = np.arange(len(rv)) >= z

    def pos(j):                                          # right row of grid index j (outside the run)
        return z + len(lo_x) + j + (RUN_LEN - 1 if j > RUN_AT else 0)
    assert all(rv[pos(j)] == val(2 * j) for j in (0, 5, RUN_AT - 1, RUN_AT + 1, n_grid - 1))

    def tile_between(j0, j1, n=AS_TILE):
        u = np.sort(rng.integers(2 * j0, 2 * j1 + 1, n))
        u[0], u[-1] = 2 * j0, 2 * j1
        return val(u)
    tiles = [np.concatenate([np.array(lo_x, dt), tile_between(0, 300, AS_TILE - len(lo_x))])]
    starts = (1000, 4000, 8000, 13000)
    for a, w in zip(starts, WIN_WIDTHS):
        tiles.append(tile_between(a, a + w - 3))         # window [pos(a) - 1, pos(a + w - 3) + 2)
    tiles.append(np.zeros(AS_TILE, dt))
    u6 = np.sort(rng.integers(2 * (RUN_AT - 300), 2 * RUN_AT, AS_TILE))
    u6[-1] = 2 * RUN_AT - 1
    tiles.append(val(u6))
    tiles.append(val(np.sort(rng.integers(2 * RUN_AT, 2 * RUN_AT + 4, AS_TILE))))
    top = [np.nan] * 7 if dt.kind == "f" else [np.iinfo(dt).max] * 7
    tiles.append(np.concatenate([tile_between(RUN_AT + 10, n_grid - 1, 993), np.array(hi_x, dt), np.array(top, dt)]))
    lv = np.concatenate(tiles)
    lvalid = rng.random(len(lv)) >= 0.01
    lvalid[5 * AS_TILE:6 * AS_TILE] = False
    for t in range(len(tiles)):                          # keep each tile's end points
        if t != 5:
            lvalid[t * AS_TILE] = lvalid[min((t + 1) * AS_TILE, len(lv)) - 1] = True
    if dt.kind == "f":
        rv[rv == 0] = -0.0
        zl = np.nonzero(lv == 0)[0]
        lv[zl[::2]] = -0.0
    return (lv, lvalid), (rv, rvalid)


# ---------------------------------------------------------------------------------------------------- inequality join case
Y_POOL = np.array([-np.inf, -1e300, -7.5, -1.0, 0.0] + [float(v) for v in range(1, 58)] + [np.inf, np.nan])      # 64 y values


def ie_wide_case(rng, m, ops):
    """Two predicates over m live right rows: x Int64 over its full range, y Float64 from Y_POOL (64 values in total
    order: -inf .. +inf, NaN), the two lowest and the two highest y values rare (m / 4096 rows each).  m / 10 more right
    rows are not live: half with a null x, half with a null y (5 % of each column).  Left (5 % nulls per column):
      narrow rows (4096): any y; x at or next to one of the 64 right x values at the end its operator selects, so the
          x-range is a few rows at the edge of the x-order
      wide rows (1024): x anywhere (MIN and MAX included), y at the extreme whose operator accepts only the rare y
          values, so the x-range is long and spans the high levels of the tree
    -> (left, right) with one (values, valid) per predicate"""
    op1, op2 = ops
    k = m // 10
    nr = m + k
    i64 = np.iinfo(np.int64)
    rx = rng.integers(i64.min, i64.max, nr, dtype=np.int64, endpoint=True)
    w = np.ones(64)
    w[[0, 1, 62, 63]] = 60 / 4096
    w /= w.sum()
    ry = Y_POOL[rng.choice(64, nr, p=w)]
    dead = rng.permutation(nr)[:k]
    rxv, ryv = np.ones(nr, bool), np.ones(nr, bool)
    rxv[dead[: k // 2]] = False
    ryv[dead[k // 2:]] = False
    live_x = np.sort(rx[rxv & ryv])
    n_narrow, n_wide = 4096, 1024
    t = rng.integers(0, 64, n_narrow)
    edge = live_x[m - 1 - t] if op1 in ("<", "<=") else live_x[t]
    nudge = rng.integers(-1, 2, n_narrow)
    lx_n = np.where((edge > i64.min) & (edge < i64.max), edge + nudge, edge)
    ly_n = Y_POOL[rng.integers(0, 64, n_narrow)]
    lx_w = rng.integers(i64.min, i64.max, n_wide, dtype=np.int64, endpoint=True)
    lx_w[:4] = (i64.min, i64.max, live_x[0], live_x[-1])
    ly_w = Y_POOL[rng.choice([62, 63], n_wide)] if op2 in ("<", "<=") else Y_POOL[rng.choice([0, 1], n_wide)]
    order = rng.permutation(n_narrow + n_wide)
    lx = np.concatenate([lx_n, lx_w])[order]
    ly = np.concatenate([ly_n, ly_w])[order]
    nl = len(lx)
    left = [(lx, rng.random(nl) >= 0.05), (ly, rng.random(nl) >= 0.05)]
    return left, [(rx, rxv), (ry, ryv)]
