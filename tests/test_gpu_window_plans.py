"""GPU tests of the window family -- bl_over (window.cu), bl_rolling (rolling.cu) and bl_rolling_by (rolling_by.cu), which
share rolling.cuh -- on every plan, past their grid caps and past 2^31 rows, against exact references
(tests/window_cases.py; tests/test_window_cases.py checks those against the plain-Python oracles on CPU).

Integer results, counts, validity, min / max and float sums and means of exactly summable values are compared with ==.
Deterministic mode is compared bit for bit with the reference's sequential replay (window_oracle / rolling_oracle /
rolling_by_oracle) on sampled partitions.  Which branch a position takes inside a kernel does not show in the launch
profile, so every test that claims a branch computes it from its input with a CPU restatement (window_cases) and asserts
a count > 0 for it.

Caps.  SM = device_info()["sm_count"]; the values in brackets are for SM = 132 (an H100 SXM).
  k_over_scan             grid min(tiles, 8 SM) [1056] CTAs of one 2048-position tile each: 8 SM x 2048 [2 162 688]
                          positions per wave; a look-back reads 32 predecessor tiles at a time [65 536 positions].
  grid-stride kernels     256 threads x 8 SM CTAs = 2048 SM [270 336] positions per sweep: k_over_shift,
                          k_over_inverse, k_over_seg_ids, k_over_row_ordinal, k_roll_out, k_rollby_bounds.
  k_over_fold             grid_for(G, 128, 16): 2048 SM [270 336] segments per sweep.
  k_roll_fold_sum / _var  grid_for(G, 64, 32): 2048 SM [270 336] segments per sweep.
  k_roll_tile             1024 outputs per CTA, B <= 128, at most 1024 + 3 B [1408] staged positions.
  k_roll_scan             one CTA per span = B max(1, 2048 / B) positions (whole blocks; several 2048-position tiles
                          once B > 2048).
  k_rollby_out            1024 outputs per CTA; the small-window plan stages a halo of 128 on each side; 32-position
                          sub-blocks with a table over them; the general plan's sparse table has ceil(log2(nb)) levels
                          over blocks of 1024.
Branches no input can reach: window_global's single-block `e == n` and segment-end suffixes (a window outside the
general plan's stage lies wholly behind its row's block, so it ends at the start of a run of equal times, never at a
segment end or at n).
"""
import ctypes as C
import math
import zlib

import numpy as np
import pytest

import rolling_by_oracle as rbo
import rolling_oracle as ro
import window_cases as wc

pytestmark = pytest.mark.gpu

CUM = {"int32": ["cum_sum", "cum_prod", "cum_min", "cum_max", "cum_count"], "uint64": ["cum_sum", "cum_prod", "cum_min", "cum_max"],
       "float32": ["cum_sum", "cum_min", "cum_max"], "float64": ["cum_sum", "cum_min", "cum_max"], "bool": ["cum_sum", "cum_count"]}


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as m
    m.init()
    m.set_deterministic(False)
    return m


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


@pytest.fixture(scope="module")
def G(sm):
    return wc.grid_threads(sm)


def full(m, n):
    return np.ones(n, bool) if m is None else m


def profiled(plb, fn):
    plb.profile_reset()
    plb.profile_enable(True)
    try:
        out = fn()
        plb.sync()
        prof = plb.profile()
    finally:
        plb.profile_enable(False)
    return out, {k: int(v.get("launches", 0)) for k, v in prof.items()}


def check(res, vals, ok, what):
    gv, gm = res
    gm = full(gm, len(gv))
    assert gv.dtype == vals.dtype, f"{what}: dtype {gv.dtype}, expected {vals.dtype}"
    assert np.array_equal(gm, ok), f"{what}: validity differs at {np.flatnonzero(gm != ok)[:8]}"
    bad = np.flatnonzero((gv != vals) & ok)
    assert bad.size == 0, f"{what}: {bad.size} values differ, first at {bad[:6]}: got {gv[bad[:4]]}, expected {vals[bad[:4]]}"


def mirrored(gid):
    """the same segment lengths in the opposite order, as ascending runs"""
    return gid.max() - gid[::-1]


def col(x, valid):
    return x if valid is None else (x, valid)


# =========================================================================================== bl_over: k_over_scan
def scan_values(rng, dtype, n, nulls):
    frac = None
    if dtype == "bool":
        x = rng.random(n) < 0.5
    elif dtype.startswith("float"):
        x, frac = wc.exact_floats(rng, n, dtype)
    elif dtype == "int32":
        x = rng.integers(-2**31, 2**31, n).astype(np.int32) | 1      # odd: products do not collapse to 0
    else:
        x = rng.integers(0, 2**64, n, dtype=np.uint64) | np.uint64(1)
    valid = rng.random(n) >= 0.1 if nulls else None
    return x, frac, valid


def scan_shape(name, sm):
    W = wc.scan_wave(sm)
    if name == "long_behind_one":
        n = 1 + 3 * wc.OS_LOOKBACK + 4097
        return n, wc.gid_from_heads(wc.heads_at(n, [1]))
    if name == "tile_edges":
        n = 6 * wc.OS_TILE + 100
        return n, wc.gid_from_heads(wc.tile_edge_heads(n, 3))
    if name == "alternating":
        return W // 2 + 5, wc.gid_from_heads(wc.alternating_heads(W // 2 + 5))
    k, d = {"wave-1": (1, -1), "wave": (1, 0), "wave+1": (1, 1), "2wave-1": (2, -1), "2wave+1": (2, 1)}[name]
    return k * W + d, None


def run_scans(plb, rng, n, gid, nulls, what):
    cols, ops, meta = {}, [], []
    for dt, kinds in CUM.items():
        cols[dt] = scan_values(rng, dt, n, nulls)
        x, _, valid = cols[dt]
        for kind in kinds:
            for rev in (False, True):
                ops.append((kind, col(x, valid), {"reverse": rev}))
                meta.append((dt, kind, rev))
    outs = plb.over(ops, partition_by=[gid] if gid is not None else [])
    for (dt, kind, rev), res in zip(meta, outs):
        x, frac, valid = cols[dt]
        exp = wc.cum_ref(kind, x, valid, gid, rev, dt, frac)
        ok = np.ones(n, bool) if kind == "cum_count" or valid is None else valid
        check(res, exp, ok, f"{what} {dt} {kind} reverse={rev}")


@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("mirror", [False, True])
@pytest.mark.parametrize("shape", ["long_behind_one", "tile_edges", "alternating"])
def test_over_scan_segment_shapes(plb, sm, shape, mirror, nulls):
    """Segmented scans (partition_by ids in ascending runs, so the partition order is the rows).  mirror: the same shape
    reversed, so that the reverse scans meet it in the order the forward scans meet the original.
    long_behind_one: a one-row segment, then one segment over more than 3 look-back windows; the look-back of its later
    tiles MAY walk past one window of 32 tiles (that depends on scheduling, so this input makes it possible, no more).
    tile_edges: heads on every lane-0 / lane-31 position of every warp round of one tile.  alternating: 1-row and
    2049-row segments, a head in nearly every tile."""
    rng = np.random.default_rng(zlib.crc32(f"{shape}-{mirror}-{nulls}".encode()))
    n, gid = scan_shape(shape, sm)
    if mirror:
        gid = mirrored(gid)
    if shape == "long_behind_one":
        assert 0 in wc.head_tiles(gid, mirror) and wc.longest_segment_after_head_tile(gid, mirror) > 3 * wc.OS_LOOKBACK
    elif shape == "tile_edges":
        assert all(v > 0 for v in wc.head_lanes(gid, mirror).values()), wc.head_lanes(gid, mirror)
    else:
        # 2050-position periods drift by 2 a tile: all but one tile in 1024 hold a head
        assert len(wc.head_tiles(gid, mirror)) >= 0.99 * ((n - 1) // wc.OS_TILE)
    run_scans(plb, rng, n, gid, nulls, shape)


@pytest.mark.parametrize("shape", ["wave-1", "wave", "wave+1", "2wave-1", "2wave+1"])
def test_over_scan_whole_column_at_wave_edges(plb, sm, shape):
    """one segment, no partition: n at k 8 SM 2048 and +- 1 (k_over_scan's grid stops growing at 8 SM CTAs)"""
    rng = np.random.default_rng(len(shape))
    n, _ = scan_shape(shape, sm)
    run_scans(plb, rng, n, None, shape.endswith("1"), shape)


# =========================================================================================== bl_over: shift, aggregations
def partition_order(gid, key=None, key_rank=None):
    """rows in the partition order: groups in first-occurrence order, rows ascending or by key_rank (stable)"""
    ug, first, inv = np.unique(gid, return_index=True, return_inverse=True)
    rank = np.empty(len(ug), np.int64)
    rank[np.argsort(first)] = np.arange(len(ug))
    grank = rank[inv.reshape(-1)]
    n = len(gid)
    perm = np.lexsort((np.arange(n), grank)) if key_rank is None else np.lexsort((np.arange(n), key_rank, grank))
    return perm, grank[perm]


def test_shift_with_partitions_and_order_past_the_grid(plb, G):
    """k_over_shift / k_over_inverse / k_over_seg_ids at n > 3 G: periods 0, +-1, +- the segment length (7) and +- 8"""
    rng = np.random.default_rng(41)
    L = 7
    ng = 3 * G // L + 1000
    n = ng * L
    assert n > 3 * G
    gid = rng.permutation(np.repeat(np.arange(ng, dtype=np.int64), L))
    key = rng.permutation(n).astype(np.int64)
    x = rng.integers(-2**62, 2**62, n)
    valid = rng.random(n) >= 0.1
    periods = [0, 1, -1, L, -L, L + 1, -(L + 1)]
    outs = plb.over([("shift", (x, valid), {"periods": p}) for p in periods], partition_by=[gid], order_by=key)
    perm, seg = partition_order(gid, key_rank=key)
    inv = np.empty(n, np.int64)
    inv[perm] = np.arange(n)
    for p, res in zip(periods, outs):
        q = inv - p
        qc = np.clip(q, 0, n - 1)
        ok = (q >= 0) & (q < n) & (seg[qc] == seg[inv]) & valid[perm[qc]]
        check(res, np.where(ok, x[perm[qc]], 0), ok, f"shift {p}")


def group_refs(gid, x, valid, order_rank=None):
    """per-row broadcasts of sum / min / max / count / first / last / median of each row's group (x small integers)"""
    n = len(gid)
    ug, inv = np.unique(gid, return_inverse=True)
    inv = inv.reshape(-1)
    ng = len(ug)
    xv = np.where(valid, x, 0)
    s = np.zeros(ng, np.int64)
    np.add.at(s, inv, xv)
    cnt = np.bincount(inv, weights=valid, minlength=ng).astype(np.int64)
    mn = np.full(ng, np.iinfo(np.int64).max)
    mx = np.full(ng, np.iinfo(np.int64).min)
    np.minimum.at(mn, inv[valid], x[valid])
    np.maximum.at(mx, inv[valid], x[valid])
    seq = np.lexsort((np.arange(n), inv)) if order_rank is None else np.lexsort((np.arange(n), order_rank, inv))
    g_sorted = inv[seq]
    starts = np.searchsorted(g_sorted, np.arange(ng), "left")
    ends = np.searchsorted(g_sorted, np.arange(ng), "right")
    first, last = seq[starts], seq[ends - 1]
    vs = np.lexsort((x, inv))
    vs = vs[valid[vs]]
    gv = inv[vs]
    vst = np.searchsorted(gv, np.arange(ng), "left")
    c = cnt
    med = np.zeros(ng)
    has = c > 0
    a = x[vs[np.minimum(vst + (c - 1) // 2, len(vs) - 1)]].astype(np.float64)
    b = x[vs[np.minimum(vst + c // 2, len(vs) - 1)]].astype(np.float64)
    med[has] = ((a + b) / 2)[has]
    return {"sum": (s[inv], np.ones(n, bool)), "count": (cnt[inv].astype(np.uint32), np.ones(n, bool)),
            "min": (np.where(has, mn, 0)[inv], has[inv]), "max": (np.where(has, mx, 0)[inv], has[inv]),
            "first": (np.where(valid[first], x[first], 0)[inv], valid[first][inv]),
            "last": (np.where(valid[last], x[last], 0)[inv], valid[last][inv]),
            "median": (med[inv], has[inv])}


def test_aggregations_past_the_grid_on_every_plan(plb, G):
    """G + 17 partitions: the fused K5 plan (sum / min / max / count), GroupsIdx (first / last / median, and
    deterministic mode) and the order_by fold, each broadcast back through k_over_row_ordinal"""
    rng = np.random.default_rng(43)
    ng = G + 17
    gid = rng.permutation(np.concatenate([np.repeat(np.arange(ng), 4), rng.integers(0, ng, 1001)])).astype(np.int64) * 7 - 3
    n = len(gid)
    x = rng.integers(-1000, 1000, n).astype(np.int64)
    valid = rng.random(n) >= 0.05
    c = (x, valid)
    ref = group_refs(gid, x, valid)
    kinds = ["sum", "min", "max", "count"]
    for k, res in zip(kinds, plb.over([(k, c) for k in kinds], partition_by=[gid])):
        check(res, *ref[k], f"K5 {k}")
    kinds = ["first", "last", "median", "sum"]
    for k, res in zip(kinds, plb.over([(k, c) for k in kinds], partition_by=[gid])):
        check(res, *ref[k], f"GroupsIdx {k}")
    f, frac = wc.exact_floats(rng, n, "float64")
    plb.set_deterministic(True)
    try:
        (gs, gm), (ga, am) = plb.over([("sum", (f, valid)), ("mean", (f, valid))], partition_by=[gid])
    finally:
        plb.set_deterministic(False)
    fr = group_refs(gid, frac, valid)
    cnt = fr["count"][0].astype(np.float64)
    check((gs, gm), fr["sum"][0] / 16.0, np.ones(n, bool), "deterministic sum")
    with np.errstate(invalid="ignore", divide="ignore"):
        check((ga, am), (fr["sum"][0] / 16.0) / cnt, cnt > 0, "deterministic mean")
    key = rng.integers(0, 50, n).astype(np.int64)      # ties: the fold keeps row order among equal keys
    ref = group_refs(gid, x, valid, order_rank=key)
    kinds = ["first", "last", "sum", "min", "max"]
    for k, res in zip(kinds, plb.over([(k, c) for k in kinds], partition_by=[gid], order_by=key)):
        check(res, *ref[k], f"order_by fold {k}")


# =========================================================================================== deterministic mode
def contiguous_groups(rng, ng):
    """ng ascending runs of 2 to 5 rows"""
    return np.repeat(np.arange(ng, dtype=np.int64), rng.integers(2, 6, ng))


@pytest.mark.parametrize("which", ["G-1", "G+1", "3G"])
def test_deterministic_past_the_fold_grids(plb, G, which):
    """k_over_fold, k_roll_fold_sum and k_roll_fold_var loop over partitions once G exceeds 2048 SM threads: exact
    values on every row, and bit for bit with the reference's sequential machines on sampled partitions"""
    rng = np.random.default_rng(len(which) + 47)
    ng = {"G-1": G - 1, "G+1": G + 1, "3G": 3 * G}[which]
    gid = contiguous_groups(rng, ng)
    n = len(gid)
    valid = rng.random(n) >= 0.1
    f64, frac = wc.exact_floats(rng, n, "float64")
    f32 = f64.astype(np.float32)
    ex = rng.integers(-1, 2, n)
    p = np.where(rng.random(n) < 0.5, -1.0, 1.0) * np.exp2(ex)      # +-2^-1, +-1, +-2: products exact
    noisy = rng.standard_normal(n) * 1e3
    t = np.cumsum(rng.integers(0, 3, n)).astype(np.int64)
    plb.set_deterministic(True)
    try:
        scans = plb.over([("cum_sum", (f64, valid), {}), ("cum_sum", (f32, valid), {"reverse": True}), ("cum_prod", (p, valid), {})],
                         partition_by=[gid])
        rolls = plb.rolling([("rolling_sum", (f64, valid), {"window_size": 3, "min_samples": 1}),
                             ("rolling_mean", (f64, valid), {"window_size": 3, "min_samples": 1}),
                             ("rolling_var", (noisy, valid), {"window_size": 3, "min_samples": 2}),
                             ("rolling_std", (noisy, valid), {"window_size": 3, "min_samples": 2})], partition_by=[gid])
        bys = plb.rolling_by([("rolling_sum", (f64, valid), {"window_size": 3}), ("rolling_mean", (f64, valid), {"window_size": 3}),
                              ("rolling_var", (noisy, valid), {"window_size": 3})], t, partition_by=[gid])
    finally:
        plb.set_deterministic(False)
    check(scans[0], wc.cum_ref("cum_sum", f64, valid, gid, False, "float64", frac), valid, "det cum_sum f64")
    check(scans[1], wc.cum_ref("cum_sum", f32, valid, gid, True, "float32", frac), valid, "det cum_sum f32 reverse")
    heads = wc.scan_heads(gid, False)
    e_sum = wc._prefix_diff_u64(np.where(valid, ex, 0).astype(np.int64).view(np.uint64), heads).view(np.int64)
    neg = wc._prefix_diff_u64((valid & (p < 0)).astype(np.uint64), heads) % np.uint64(2)
    check(scans[2], np.where(valid, np.where(neg == 1, -1.0, 1.0) * np.exp2(e_sum), 0.0), valid, "det cum_prod")
    s, e, _, _ = wc.fixed_bounds(n, 3, False, gid)
    for k, res in zip(("rolling_sum", "rolling_mean"), rolls[:2]):
        check(res, *wc.rolling_ref(k, f64, valid, s, e, 1, frac, "float64"), f"det {k}")
    sb, eb = wc.by_bounds(t, 3, "right", gid)
    for k, res in zip(("rolling_sum", "rolling_mean"), bys[:2]):
        v, ok = wc.rolling_ref(k, f64, valid, sb, eb, 0 if k == "rolling_sum" else 1, frac, "float64")
        check(res, v, ok, f"det {k}_by")
    starts = np.flatnonzero(heads)
    ends = np.append(starts[1:], n)
    pick = rng.choice(len(starts), 300, replace=False)
    pick = np.concatenate([pick, [0, len(starts) - 1]])
    for g in pick:
        a, b = starts[g], ends[g]
        vals = [float(noisy[r]) if valid[r] else None for r in range(a, b)]
        for k, (gv, gm) in zip(("rolling_var", "rolling_std"), rolls[2:]):
            exp = ro.rolling(k, vals, "float64", 3, 2)
            got = [float(gv[r]) if full(gm, n)[r] else None for r in range(a, b)]
            assert got == exp, (k, g, got, exp)
        exp = rbo.replay_by("rolling_var", "float64", [0.0 if v is None else v for v in vals], list(valid[a:b]), t[a:b].tolist(), [True] * (b - a),
                            3, "right", 1)
        gv, gm = bys[2]
        got = [float(gv[r]) if full(gm, n)[r] else None for r in range(a, b)]
        assert got == exp, ("rolling_var_by", g, got, exp)


# =========================================================================================== order_by at scale
ORDER_CASES = [(n, kk) for n in (2**16 - 1, 2**16) for kk in ("int64", "float64", "string")] + [(n, kk) for n in (2**24 - 1, 2**24) for kk in ("int64", "float64")]


@pytest.mark.parametrize("n,key_kind", ORDER_CASES)
def test_order_by_at_scale(plb, n, key_kind):
    """over and rolling with order_by on top of the arg sort of (group id, key): sizes around 2^16 and 2^24 change the
    number of radix passes; ascending / descending and nulls first / last alternate over the cases"""
    i = ORDER_CASES.index((n, key_kind))
    descending, nulls_last = bool(i & 1), bool(i & 2)
    rng = np.random.default_rng(i + 53)
    gid = rng.integers(0, 1000, n).astype(np.int64)
    k = rng.integers(0, 5000, n)
    kvalid = rng.random(n) >= 0.05
    if key_kind == "int64":
        key = (k - 2500).astype(np.int64)
        okey = (key, kvalid)
    elif key_kind == "float64":
        key = (k - 2500.5) / 8.0
        okey = (key, kvalid)
    else:
        okey = plb.StringColumn([b"k%05d" % v if ok else None for v, ok in zip(k.tolist(), kvalid.tolist())])
    x = rng.integers(-10**12, 10**12, n).astype(np.int64)
    (cs, cm), (rs, rm) = plb.over([("cum_sum", x, {})], partition_by=[gid], order_by=okey, descending=descending, nulls_last=nulls_last) + \
        plb.rolling([("rolling_sum", x, {"window_size": 5, "min_samples": 1})], partition_by=[gid], order_by=okey, descending=descending,
                    nulls_last=nulls_last)
    kr = np.where(kvalid, -k if descending else k, 0)
    nullflag = np.where(kvalid, 0, 1 if nulls_last else -1)
    ug, inv = np.unique(gid, return_inverse=True)
    perm, seg = partition_order(gid, key_rank=nullflag * 10**6 + kr)
    xs = x[perm]
    heads = np.ones(n, bool)
    heads[1:] = seg[1:] != seg[:-1]
    cum = wc._prefix_diff_u64(xs.view(np.uint64), heads).view(np.int64)
    exp = np.empty(n, np.int64)
    exp[perm] = cum
    check((cs, cm), exp, np.ones(n, bool), "over cum_sum order_by")
    lo = wc.seg_start(heads)
    pos = np.arange(n)
    s = np.maximum(pos - 4, lo)
    w = wc.window_sum_u64(xs.view(np.uint64), s, pos + 1).view(np.int64)
    exp[perm] = w
    check((rs, rm), exp, np.ones(n, bool), "rolling_sum order_by")


# =========================================================================================== bl_rolling
ROLL_DTYPES = ("int32", "uint64", "bool", "int64", "float64", "float32")


def rolling_columns(rng, n):
    cols = {}
    for dt in ROLL_DTYPES:
        frac = None
        if dt == "bool":
            x = rng.random(n) < 0.5
        elif dt.startswith("float"):
            x, frac = wc.exact_floats(rng, n, dt)
        elif dt == "uint64":
            x = rng.integers(0, 2**64, n, dtype=np.uint64)
        else:
            x = rng.integers(np.iinfo(dt).min, np.iinfo(dt).max, n, dtype=dt, endpoint=True)
        cols[dt] = (x, frac, rng.random(n) >= 0.1)
    return cols


def roll_kinds(dt):
    if dt == "bool":
        return ["rolling_sum"]
    if dt.startswith("float"):
        return ["rolling_sum", "rolling_mean", "rolling_min", "rolling_max"]
    if dt == "int64":
        return ["rolling_min", "rolling_max"]
    return ["rolling_sum"]


def run_rolling(plb, rng, n, w, gid, centers, what):
    cols = rolling_columns(rng, n)
    ops, meta = [], []
    ms = min(w, 2)
    for dt, (x, frac, valid) in cols.items():
        for kind in roll_kinds(dt):
            for center in centers:
                ops.append((kind, (x, valid), {"window_size": w, "min_samples": ms, "center": center}))
                meta.append((dt, kind, center))
    outs, prof = profiled(plb, lambda: plb.rolling(ops, partition_by=[gid] if gid is not None else []))
    for (dt, kind, center), res in zip(meta, outs):
        x, frac, valid = cols[dt]
        s, e, _, _ = wc.fixed_bounds(n, w, center, gid)
        v, ok = wc.rolling_ref(kind, x, valid, s, e, ms, frac, dt)
        check(res, v, ok, f"{what} {dt} {kind} center={center}")
    return prof


def tile_heads(n, w, center, rng):
    """segment heads on block starts / ends, CTA output edges and the halo's first / last staged position of every CTA"""
    R = w // 2 + (w & 1) if center else 1
    L = w - R if center else w - 1
    at = []
    for c, o0 in enumerate(range(0, n, wc.RT_TILE)):
        o1 = min(n, o0 + wc.RT_TILE)
        A = max(o0 - L, 0) // w * w
        last = min(n - 1, o1 - 2 + R)
        pick = [o0, o1 - 1, A, A + 1, last, last + 1, (o0 // w + 1) * w, (o0 // w + 1) * w - 1, o0 + 517 // w * w][c % 9]
        at.append(pick)
    at += list(rng.integers(0, n, n // 700))
    return wc.heads_at(n, at)


@pytest.mark.parametrize("center", [False, True])
@pytest.mark.parametrize("B", [1, 2, 3, 31, 127, 128])
def test_rolling_tile_plan(plb, sm, B, center):
    """k_roll_tile (B = w <= 128) over more than one wave of 1024-output CTAs, with and without partitions"""
    rng = np.random.default_rng(B * 2 + center)
    n = 3 * sm * wc.RT_TILE + 777
    gid = wc.gid_from_heads(tile_heads(n, B, center, rng))
    s, e, lo, _ = wc.fixed_bounds(n, B, center, gid)
    br = np.bincount(wc.window_state_branch(s, e, lo, B), minlength=3)
    want = {wc.PRE} | ({wc.TWO} if B > 1 else set()) | ({wc.SUF} if center and B > 2 else set())
    assert all(br[k] > 0 for k in want), br
    R = B // 2 + (B & 1) if center else 1
    _, _, last = wc.tile_staging(n, B - R if center else B - 1, R, B)
    if (wc.RT_TILE - 2 + R) % B == 0:      # the last output's window ends on the first position of a staged block
        assert np.sum((last[:-1] % B) == 0) > 0
    for g in (gid, None):
        prof = run_rolling(plb, rng, n, B, g, (center,), f"tile B={B} partitions={g is not None}")
        assert prof.get("rolling_tile", 0) > 0 and "rolling_prefix" not in prof, prof


@pytest.mark.parametrize("B", [129, 1023, 1024, 1025, 2047, 2048, 2049, 4096, 4097])
def test_rolling_three_pass_plan(plb, B):
    """k_roll_scan + k_roll_out (B > 128): span = B max(1, 2048 / B) takes its several-blocks, one-block and
    more-than-a-tile forms, and the last CTA of both scans is partial"""
    rng = np.random.default_rng(B)
    span = B * max(1, wc.RS_TILE // B)
    n = 37 * span + span // 2 + 5
    at = list(rng.integers(0, n, n // (3 * B) + 1)) + [k * B for k in range(1, n // B, 7)] + [k * B - 1 for k in range(2, n // B, 5)]
    gid = wc.gid_from_heads(wc.heads_at(n, at))
    for center in (False, True):
        s, e, lo, _ = wc.fixed_bounds(n, B, center, gid)
        br = np.bincount(wc.window_state_branch(s, e, lo, B), minlength=3)
        assert br[wc.TWO] > 0 and br[wc.PRE] > 0 and (br[wc.SUF] > 0 or not center), br
    for g in (gid, None):
        prof = run_rolling(plb, rng, n, B, g, (False, True), f"three-pass B={B} partitions={g is not None}")
        assert prof.get("rolling_prefix", 0) > 0 and prof.get("rolling_out", 0) > 0 and "rolling_tile" not in prof, prof


# =========================================================================================== bl_rolling_by
def by_ops(rng, n, P, closed="right"):
    """int64 sums (wrapping), int32 max and exactly summable float64 means, with nulls"""
    x = rng.integers(-2**63, 2**63, n, dtype=np.int64)
    y = rng.integers(-2**31, 2**31, n).astype(np.int32)
    f, frac = wc.exact_floats(rng, n, "float64")
    valid = rng.random(n) >= 0.1
    ops = [("rolling_sum", (x, valid), {"window_size": P, "closed": closed, "min_samples": 0}),
           ("rolling_max", (y, valid), {"window_size": P, "closed": closed, "min_samples": 1}),
           ("rolling_mean", (f, valid), {"window_size": P, "closed": closed, "min_samples": 1})]
    return ops, (x, y, f, frac, valid)


def check_by(outs, data, s, e, what, out_ok=None):
    x, y, f, frac, valid = data
    for (kind, v, fr, dt, ms), res in zip((("rolling_sum", x, None, "int64", 0), ("rolling_max", y, None, "int32", 1),
                                          ("rolling_mean", f, frac, "float64", 1)), outs):
        val, ok = wc.rolling_ref(kind, v, valid, s, e, ms, fr, dt)
        ok &= (e - s) >= ms
        if out_ok is not None:
            ok &= out_ok
        check(res, val, ok, f"{what} {kind}")


@pytest.mark.parametrize("nb", [1, 2, 3, 4, 5] + [x for k in range(3, 13) for x in (2**k, 2**k + 1)])
def test_rolling_by_sparse_table_levels(plb, nb):
    """nb blocks of 1024 (the last one partial): every level count K = ceil(log2 nb).  Whole-prefix windows read levels
    1 .. log2(nb - 2) of the table, windows of 3 blocks level 0; windows of exactly 1, 2 and 3 blocks"""
    rng = np.random.default_rng(nb)
    n = nb * wc.RB_B - 7 if nb > 1 else 1000
    t = np.arange(n, dtype=np.int64)
    Ps = (n, 1024, 2048, 3072)
    bounds = [wc.by_bounds(t, P, "right") for P in Ps]
    ms = [wc.rollby_branch(s, e, n, False) for s, e in bounds]
    levels = set()
    for m in ms:
        levels |= set(np.unique(m["level"][m["level"] >= 0]).tolist())
    reach = set(range(int(math.log2(nb - 2)) + 1)) if nb >= 5 else {1} if nb == 4 else set()
    assert levels == reach, (levels, reach)
    assert nb < 3 or ms[0]["g_l_eq_r"].sum() > 0
    assert nb < 2 or ms[0]["g_adjacent"].sum() > 0
    for P, (s, e) in zip(Ps, bounds):
        ops, data = by_ops(rng, n, P)
        outs, prof = profiled(plb, lambda: plb.rolling_by(ops, t))
        assert prof.get("rolling_by_out", 0) > 0 and (prof.get("rolling_by_sparse", 0) > 0) == (wc.sparse_levels(n) > 0), prof
        check_by(outs, data, s, e, f"nb={nb} P={P}")


def test_rolling_by_plan_switch(plb):
    """W = 128 runs the one-pass small-window plan, W = 129 the general plan"""
    rng = np.random.default_rng(59)
    n = 200_003
    t = np.arange(n, dtype=np.int64)
    for P, plan, other in ((128, "rolling_by_tile", "rolling_by_out"), (129, "rolling_by_out", "rolling_by_tile")):
        ops, data = by_ops(rng, n, P)
        outs, prof = profiled(plb, lambda: plb.rolling_by(ops, t))
        assert plan in prof and other not in prof, prof
        check_by(outs, data, *wc.by_bounds(t, P, "right"), f"P={P}")


def zoo(tile: bool):
    """(times, segment ids, P), positions = rows (ascending ids, ascending times).  Each test segment is a rising run of
    times, then a run of 1500 equal times, then 700 rising ones: with closed left / none, the window of a row in the run is
    [first time >= T - P, run start), wholly behind the row's own block.  The segments place that window on a block start,
    a segment head, a block end, or neither (fillers between them set the alignment).  With `tile`, P = 100 and the run
    is longer than the halo; only left / none windows stay narrow there (a right / both window of a row in the run holds
    the whole run)."""
    P = 100 if tile else 300
    ts, gs = [], []
    pos = 0

    def add(times):
        nonlocal pos
        ts.append(np.asarray(times, np.int64))
        gs.append(np.full(len(times), len(gs), np.int64))
        pos += len(times)

    def fill_to(mod):      # a filler segment so that the next one starts at pos % 1024 == mod
        add(np.arange((mod - pos) % 1024 + 1024))

    def test_segment(pre):      # the run's times are pre + 5, so its window is [pos + pre + 5 - P, pos + pre)
        # with `tile`, the times after the run jump by more than P, so no window holds the run: every window stays at
        # most P wide and the small-window plan runs
        after = pre + 5 + (P + 1 if tile else 1)
        add(np.concatenate([np.arange(pre), np.full(1500, pre + 5), after + np.arange(700)]))

    fill_to(0)
    test_segment(1024 + 100)                 # run start on a block start: the window ends on a block end
    fill_to(0)
    test_segment(1024 + P - 5)               # the window starts on a block start (closed left) ...
    fill_to(0)
    test_segment(1024 + P - 6)               # ... and with closed none (times > T - P)
    fill_to(100)
    test_segment((P - 5) // 2)               # the window starts on the segment head (mid-block)
    fill_to(100)
    test_segment(600)                        # neither: a fold
    fill_to(500)
    add(np.arange(3000))                     # a segment across blocks for the null-`by` tail
    return np.concatenate(ts), np.concatenate(gs), P


@pytest.mark.parametrize("tile,closed", [(False, "left"), (False, "none"), (False, "right"), (False, "both"), (True, "left"), (True, "none")])
def test_rolling_by_branch_zoo(plb, tile, closed):
    """window_global's single-block prefix (block start, segment head), block-end suffix and fold, or the tile plan's
    fold_global behind a run longer than the halo; a null-`by` tail in a segment that crosses a block boundary; and a
    last window inside one sub-block that ends on the stage's last position (n % 32 != 0), on values where only the
    staged suffix Q[l] gives the exact sum"""
    rng = np.random.default_rng(61 + tile + 2 * len(closed))
    t, gid, P = zoo(tile)
    bvalid = np.ones(len(t), bool)
    bvalid[-40:] = False      # the tail of the last segment: null `by`, sorted last, across a block boundary
    n0 = len(t)
    pad = (20 - (n0 + 4)) % 32      # n % 32 == 20: the stage's last sub-block is partial
    end = np.concatenate([np.arange(-(pad + 1), 0), [10, 11, 12]])      # a head, then three rows in (9, 12]
    t = np.concatenate([t, end]).astype(np.int64)
    gid = np.concatenate([gid, np.full(len(end), gid.max() + 1)])
    bvalid = np.concatenate([bvalid, np.ones(len(end), bool)])
    n = len(t)
    assert n % 32 == 20
    tk = np.where(bvalid, t, 10**12)      # null times count as +inf (nulls last in each segment)
    s, e = wc.by_bounds(tk, P, closed, gid)
    s, e = np.where(bvalid, s, 0), np.where(bvalid, e, 0)
    assert wc.rollby_tile_plan(s, e) == tile
    m = wc.rollby_branch(s, e, n, tile, gid)
    if closed in ("left", "none"):
        want = ["tile_fold_global"] if tile else ["g_pre_block", "g_pre_head", "g_suf_block", "g_fold"]
        assert all(m[k].sum() > 0 for k in want), {k: int(m[k].sum()) for k in want}
    x = rng.integers(-2**63, 2**63, n, dtype=np.int64)
    y = rng.integers(-2**31, 2**31, n).astype(np.int32)
    f, frac = wc.exact_floats(rng, n, "float64")
    f4, frac4 = f.copy(), frac.copy()
    f4[-3:] = [1.0, 2.0**53, -2.0**53]
    frac4[-3:] = [16, 2**57, -2**57]
    valid = rng.random(n) >= 0.1
    valid[-3:] = True
    s3, e3 = wc.by_bounds(tk, 3, "right", gid)
    s3, e3 = np.where(bvalid, s3, 0), np.where(bvalid, e3, 0)
    tile3 = wc.rollby_tile_plan(s3, e3)
    m3 = wc.rollby_branch(s3, e3, n, tile3, gid)
    assert m3["stage_Q_len"][-1], "the last window must end on the stage's last position"
    ops = [("rolling_sum", (x, valid), {"window_size": P, "closed": closed, "min_samples": 0}),
           ("rolling_max", (y, valid), {"window_size": P, "closed": closed, "min_samples": 1}),
           ("rolling_mean", (f, valid), {"window_size": P, "closed": closed, "min_samples": 1})]
    outs, prof = profiled(plb, lambda: plb.rolling_by(ops, (t, bvalid), partition_by=[gid]))
    plan, other = ("rolling_by_tile", "rolling_by_out") if tile else ("rolling_by_out", "rolling_by_tile")
    assert plan in prof and other not in prof, prof
    check_by(outs, (x, y, f, frac, valid), s, e, f"zoo tile={tile} {closed}", out_ok=bvalid)
    [out4], prof = profiled(plb, lambda: plb.rolling_by([("rolling_sum", (f4, valid), {"window_size": 3, "closed": "right", "min_samples": 0})],
                                                        (t, bvalid), partition_by=[gid]))
    assert ("rolling_by_tile" if tile3 else "rolling_by_out") in prof, prof
    v, ok = wc.rolling_ref("rolling_sum", f4, valid, s3, e3, 0, frac4, "float64")
    assert v[-1] == 1.0
    check(out4, v, ok & bvalid, "the last window's sum")


@pytest.mark.parametrize("tile", [True, False])
def test_rolling_by_last_window_on_the_stage_end(plb, tile):
    """A whole column (no partition, so no segment ids to stop at): the last window lies inside one sub-block, starts
    mid-sub-block and ends on the stage's last position (n % 32 == 20).  Its values 1, 2^53, -2^53 sum to exactly 1 only
    as the staged suffix Q[l] = 1 + (2^53 - 2^53); a left-to-right fold gives 0.  `tile`: every window holds at most 3
    rows; else a run of 300 equal times makes the general plan run."""
    rng = np.random.default_rng(73 + tile)
    n = 5 * wc.RB_B + 20
    t = np.arange(n, dtype=np.int64) * 10
    if not tile:
        t[100:400] = t[100]
    t[-3:] = t[-4] + 100 + np.arange(3)
    s, e = wc.by_bounds(t, 3, "right")
    assert wc.rollby_tile_plan(s, e) == tile
    m = wc.rollby_branch(s, e, n, tile)
    assert m["stage_Q_len"][-1] and e[-1] - s[-1] == 3 and (s[-1] - (n - 1) // wc.RB_B * wc.RB_B) % wc.RB_SUB != 0
    f, frac = wc.exact_floats(rng, n, "float64")
    f[-3:] = [1.0, 2.0**53, -2.0**53]
    frac[-3:] = [16, 2**57, -2**57]
    outs, prof = profiled(plb, lambda: plb.rolling_by([("rolling_sum", f, {"window_size": 3})], t))
    assert ("rolling_by_tile" if tile else "rolling_by_out") in prof, prof
    v, ok = wc.rolling_ref("rolling_sum", f, None, s, e, 0, frac, "float64")
    assert v[-1] == 1.0
    check(outs[0], v, ok, f"last window tile={tile}")


def test_rolling_by_in_stage_sub_block_windows(plb):
    """windows inside the staged tile across 2, 3 and 2^k sub-blocks and inside one sub-block touching either edge or
    neither, with partitions: times = positions, widths 1 .. 500"""
    rng = np.random.default_rng(67)
    n = 300_017
    gid = wc.gid_from_heads(rng.random(n) < 1 / 2000)
    t = np.arange(n, dtype=np.int64)
    for P, tile in ((1, True), (20, True), (33, True), (65, True), (100, True), (200, False), (500, False)):
        s, e = wc.by_bounds(t, P, "right", gid)
        assert wc.rollby_tile_plan(s, e) == tile
        m = wc.rollby_branch(s, e, n, tile, gid)
        if P >= 33:
            assert m["stage_cross"].sum() > 0 and (P < 65 or m["stage_l_eq_r"].sum() > 0)
        if P >= 200:
            assert m["stage_k"].sum() > 0
        if P == 20:
            assert m["stage_P"].sum() > 0 and m["stage_Q_sub"].sum() > 0 and m["stage_fold"].sum() > 0 and m["stage_Q_seg"].sum() > 0
        ops, data = by_ops(rng, n, P)
        outs = plb.rolling_by(ops, t, partition_by=[gid])
        check_by(outs, data, s, e, f"P={P}")


def test_rolling_by_unsorted_without_partitions(plb):
    """times out of order, no nulls, no partitions: only the descent count says a sort is needed"""
    rng = np.random.default_rng(71)
    n = 100_000
    t = rng.integers(0, 30_000, n).astype(np.int64)
    order = np.argsort(t, kind="stable")
    ts = t[order]
    for closed in ("right", "left", "both", "none"):
        ops, data = by_ops(rng, n, 500, closed)
        outs = plb.rolling_by(ops, t)
        s, e = wc.by_bounds(ts, 500, closed)
        x, y, f, frac, valid = data
        for (kind, v, fr, dt, ms), res in zip((("rolling_sum", x, None, "int64", 0), ("rolling_max", y, None, "int32", 1),
                                              ("rolling_mean", f, frac, "float64", 1)), outs):
            val, ok = wc.rolling_ref(kind, v[order], valid[order], s, e, ms, None if fr is None else fr[order], dt)
            ev, eo = np.empty_like(val), np.empty(n, bool)
            ev[order], eo[order] = val, ok
            check(res, ev, eo, f"unsorted {closed} {kind}")


# =========================================================================================== past 2^31 rows
N_BIG = 2**31 + 2**20 + 33


class _Dev:
    """a device buffer as a torch tensor, without a copy"""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3}


def need(plb, nbytes):
    free = plb.device_info()["hbm_free"]
    if free < nbytes:
        pytest.skip(f"needs {nbytes / 2**30:.0f} GiB of free device memory, {free / 2**30:.0f} GiB free")


def dev_view(torch, out, n, typestr):
    return torch.as_tensor(_Dev(out.values_ptr, n, typestr), device="cuda")


def valid_bits(torch, out, lo, hi):
    """the validity bits of rows [lo, hi) of a device output (lo a multiple of 8)"""
    if not out.validity_ptr:
        return None
    b = torch.as_tensor(_Dev(out.validity_ptr, (hi - lo + 7) // 8, "|u1"), device="cuda") if lo == 0 else \
        torch.as_tensor(_Dev(out.validity_ptr + lo // 8, (hi - lo + 7) // 8, "|u1"), device="cuda")
    bits = (b.unsqueeze(1) >> torch.arange(8, device="cuda", dtype=torch.uint8)) & 1
    return bits.reshape(-1)[: hi - lo].bool()


CHUNK = 1 << 28


def periodic_i32(torch, n, period, base):
    x = torch.empty(n, dtype=torch.int32, device="cuda")
    for off in range(0, n, CHUNK):
        m = min(CHUNK, n - off)
        x[off:off + m] = (torch.arange(off, off + m, device="cuda", dtype=torch.int64) % period + base).to(torch.int32)
    return x


def periodic_bits(torch, n, period):
    """a bitmap with bit i set iff i % period != 0"""
    nbytes = (n + 7) // 8 + 64
    out = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    w = torch.tensor([1 << k for k in range(8)], device="cuda", dtype=torch.int64)
    for off in range(0, nbytes, CHUNK // 8):
        m = min(CHUNK // 8, nbytes - off)
        i = torch.arange(off * 8, (off + m) * 8, device="cuda", dtype=torch.int64).reshape(m, 8)
        out[off:off + m] = ((i % period != 0).to(torch.int64) * w).sum(1).to(torch.uint8)
    return out


def wrap32(v):
    return ((v + 2**31) % 2**32 - 2**31).to(torch_mod().int32)


def torch_mod():
    import torch
    return torch


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("no CUDA device for torch")
    return t


def test_past_2_31_cum_sum_int32(plb, torch):
    """cum_sum of Int32 x_i = 1 000 003 + i % 3 over 2^31 + 2^20 + 33 rows (no sort): wrapping prefix sums, forward and
    reverse, against the closed form S(i) = (i + 1) c + 3 q + r (r - 1) / 2, q = (i + 1) // 3, r = (i + 1) % 3"""
    n, c = N_BIG, 1_000_003
    need(plb, 3 * 4 * n + (2 << 30))
    x = periodic_i32(torch, n, 3, c)
    torch.cuda.synchronize()
    xc = plb.Column(x.data_ptr(), dtype=np.int32, length=n, location=plb.DEVICE)

    def S(i):      # sum of x[0 .. i - 1]
        q, r = i // 3, i % 3
        return i * c + 3 * q + r * (r - 1) // 2
    total = S(torch.tensor(n, dtype=torch.int64))
    for rev in (False, True):
        [out] = plb.over([("cum_sum", xc, {"reverse": rev})], location=plb.DEVICE)
        plb.sync()
        try:
            assert out.length == n and not out.validity_ptr
            got = dev_view(torch, out, n, "<i4")
            for off in range(0, n, CHUNK):
                m = min(CHUNK, n - off)
                i = torch.arange(off, off + m, device="cuda", dtype=torch.int64)
                exp = (total - S(i)) if rev else S(i + 1)
                assert torch.equal(got[off:off + m], wrap32(exp)), (rev, off)
            del got
        finally:
            out.free()
    del x
    torch.cuda.empty_cache()


def test_past_2_31_cum_count_and_shift(plb, torch):
    """cum_count of a Bool column whose validity is i % 5 != 0 (count = i - i // 5), and shift of an Int32 i % 7 column
    by +-(2^31 + 5)"""
    n = N_BIG
    need(plb, 3 * 4 * n + (2 << 30))
    bits = periodic_bits(torch, n, 5)
    ones = torch.full(((n + 7) // 8 + 64,), 255, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    bc = plb.Column(ones.data_ptr(), bits.data_ptr(), dtype=np.bool_, length=n, location=plb.DEVICE, null_count=-1)
    [out] = plb.over([("cum_count", bc, {})], location=plb.DEVICE)
    plb.sync()
    try:
        got = dev_view(torch, out, n, "<u4")
        for off in range(0, n, CHUNK):
            m = min(CHUNK, n - off)
            i = torch.arange(off, off + m, device="cuda", dtype=torch.int64)
            assert torch.equal(got[off:off + m].to(torch.int64) & 0xFFFFFFFF, i - i // 5), off
        del got
    finally:
        out.free()
    del bits, ones
    x = periodic_i32(torch, n, 7, 0)
    torch.cuda.synchronize()
    xc = plb.Column(x.data_ptr(), dtype=np.int32, length=n, location=plb.DEVICE)
    for p in (2**31 + 5, -(2**31 + 5)):
        [out] = plb.over([("shift", xc, {"periods": p})], location=plb.DEVICE)
        plb.sync()
        try:
            got = dev_view(torch, out, n, "<i4")
            for off in range(0, n, CHUNK):
                m = min(CHUNK, n - off)
                i = torch.arange(off, off + m, device="cuda", dtype=torch.int64)
                q = i - p
                ok = (q >= 0) & (q < n)
                assert torch.equal(valid_bits(torch, out, off, off + m), ok), (p, off)
                assert torch.equal(got[off:off + m], torch.where(ok, q % 7, 0).to(torch.int32)), (p, off)
            del got
        finally:
            out.free()
    del x
    torch.cuda.empty_cache()


def test_past_2_31_rolling_sum_bool_tile(plb, torch):
    """rolling_sum of a Bool column (bit i set iff i % 3 != 0... written as the complement count) with w = 128, center, on
    the tile plan: the window [i - 64, i + 64) clipped to [0, n) holds (b - a) - (ceil(b / 3) - ceil(a / 3)) set bits"""
    n = N_BIG
    need(plb, 4 * n + (2 << 30))
    bits = periodic_bits(torch, n, 3)
    torch.cuda.synchronize()
    bc = plb.Column(bits.data_ptr(), dtype=np.bool_, length=n, location=plb.DEVICE)
    outs, prof = profiled(plb, lambda: plb.rolling([("rolling_sum", bc, {"window_size": 128, "min_samples": 1, "center": True})], location=plb.DEVICE))
    [out] = outs
    assert prof.get("rolling_tile", 0) == 1, prof
    try:
        got = dev_view(torch, out, n, "<u4")
        for off in range(0, n, CHUNK):
            m = min(CHUNK, n - off)
            i = torch.arange(off, off + m, device="cuda", dtype=torch.int64)
            a, b = torch.clamp(i - 64, min=0), torch.clamp(i + 64, max=n)
            exp = (b - a) - ((b + 2) // 3 - (a + 2) // 3)
            assert torch.equal(got[off:off + m].to(torch.int64) & 0xFFFFFFFF, exp), off
            vb = valid_bits(torch, out, off, off + m)
            assert vb is None or bool(vb.all()), off
        del got
    finally:
        out.free()
    del bits
    torch.cuda.empty_cache()


def test_past_2_31_rolling_sum_by_tile(plb, torch):
    """rolling_sum_by of Int32 x_i = i % 5 by the Int32 time i // 2 with P = 3 (six rows a window, the tile plan, no sort):
    the window of row i is [max(0, 2 (t - 2)), min(n, 2 (t + 1))), t = i // 2"""
    n = N_BIG
    need(plb, 5 * 4 * n + (3 << 30))
    x = periodic_i32(torch, n, 5, 0)
    t = torch.empty(n, dtype=torch.int32, device="cuda")
    for off in range(0, n, CHUNK):
        m = min(CHUNK, n - off)
        t[off:off + m] = (torch.arange(off, off + m, device="cuda", dtype=torch.int64) // 2).to(torch.int32)
    torch.cuda.synchronize()
    xc = plb.Column(x.data_ptr(), dtype=np.int32, length=n, location=plb.DEVICE)
    tc = plb.Column(t.data_ptr(), dtype=np.int32, length=n, location=plb.DEVICE)
    outs, prof = profiled(plb, lambda: plb.rolling_by([("rolling_sum", xc, {"window_size": 3})], tc, location=plb.DEVICE))
    [out] = outs
    assert prof.get("rolling_by_tile", 0) == 1 and "rolling_by_out" not in prof, prof

    def F(k):      # sum of x[0 .. k - 1]
        q, r = k // 5, k % 5
        return 10 * q + r * (r - 1) // 2
    try:
        got = dev_view(torch, out, n, "<i4")
        for off in range(0, n, CHUNK):
            m = min(CHUNK, n - off)
            i = torch.arange(off, off + m, device="cuda", dtype=torch.int64)
            tt = i // 2
            a, b = torch.clamp(2 * (tt - 2), min=0), torch.clamp(2 * (tt + 1), max=n)
            assert torch.equal(got[off:off + m].to(torch.int64), F(b) - F(a)), off
        del got
    finally:
        out.free()
    del x, t
    torch.cuda.empty_cache()


def test_2_32_rows_are_refused(plb, torch):
    """a column header of 2^32 rows (a device header over a small buffer: nothing is read) is refused by all three"""
    buf = torch.zeros(64, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    big = plb.Column(buf.data_ptr(), dtype=np.int64, length=2**32, location=plb.DEVICE)
    for call in (lambda: plb.over([("cum_sum", big, {})]), lambda: plb.rolling([("rolling_sum", big, {"window_size": 2})]),
                 lambda: plb.rolling_by([("rolling_sum", big, {"window_size": 2})], big)):
        with pytest.raises(plb.B200Error, match=r"2\^32 - 1 rows") as e:
            call()
        assert e.value.status == 4
    del buf
