"""GPU tests of the rolling windows (bl_rolling).  Results are compared with tests/rolling_oracle.py: validity, integer SUM,
MIN / MAX and every non-finite class bit for bit; finite float SUM / MEAN / VAR / STD under the header's bound against the
exact window value; float results bit for bit in deterministic mode.  Window sizes straddle the scan tile (2048 positions)
so that blocks span CTA tiles, several blocks share one tile, and a window covers the whole column."""
import math
import struct
from fractions import Fraction

import numpy as np
import pytest

import rolling_oracle as ro

pytestmark = pytest.mark.gpu
TILE = 2048
KINDS = ["rolling_sum", "rolling_mean", "rolling_min", "rolling_max", "rolling_var", "rolling_std"]
U = {"float32": 2.0 ** -24, "float64": 2.0 ** -53}


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as plb
    plb.init()
    plb.set_deterministic(False)
    return plb


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


def values(rng, dtype, n, nulls, finite=False):
    if dtype == "bool":
        x = rng.random(n) < 0.5
    elif dtype.startswith("float"):
        x = (rng.standard_normal(n) * 1e3).astype(dtype)
        if not finite:
            sp = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, np.finfo(dtype).tiny / 4], dtype)
            at = rng.random(n) < 0.02
            x[at] = sp[rng.integers(0, len(sp), at.sum())]
    else:
        info = np.iinfo(dtype)
        x = rng.integers(info.min, info.max, n, dtype=dtype, endpoint=True)
        at = rng.random(n) < 0.05
        x[at] = rng.choice(np.array([info.min, info.max, info.max // 2 + 1, 0], dtype), at.sum())
    valid = rng.random(n) >= 0.2 if nulls else None
    return x, valid


def as_list(x, valid):
    out = x.tolist()
    if x.dtype.kind == "f":
        out = [float(v) for v in out]
    if valid is not None:
        out = [v if ok else None for v, ok in zip(out, valid)]
    return out


def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, float) or isinstance(b, float):
        return struct.pack("<d", float(a)) == struct.pack("<d", float(b)) or (a != a and b != b)
    return int(a) == int(b)


class Windows:
    """row -> the non-null values of its window in partition order, computed when asked"""

    def __init__(self, xs, parts, w, center):
        self.xs, self.w, self.center = xs, w, center
        self.at = {r: (rows, k) for rows in parts for k, r in enumerate(rows)}

    def __getitem__(self, r):
        rows, k = self.at[r]
        offs = ro.det_offsets_center if self.center else ro.det_offsets
        s, e = offs(k, self.w, len(rows))
        return [self.xs[q] for q in rows[s:e] if self.xs[q] is not None]


def within_bound(kind, dtype, a, b, win, ddof):
    u_out = U["float32" if dtype == "float32" else "float64"]
    if not math.isfinite(b) or any(not math.isfinite(float(v)) for v in win):
        return (a != a) if b != b else a == b      # the class must agree
    xs = [float(v) for v in win]
    k = len(xs)
    if kind == "rolling_sum":
        return abs(a - math.fsum(xs)) <= ro.sum_bound(xs, u_out) + U["float64"] * abs(b)
    if kind == "rolling_mean":
        return abs(a - math.fsum(xs) / k) <= ro.mean_bound(xs, u_out) + U["float64"] * abs(b)
    # VAR / STD: the header's bound against the exact variance (big-integer moments, tests/rolling_oracle.py)
    ex = ro.exact_var(xs, ddof)
    vb = ro.var_bound(xs, ddof, u_out)
    if kind == "rolling_var":
        return abs(Fraction(a) - ex) <= Fraction(vb)
    return abs(a - math.sqrt(ex)) <= math.sqrt(vb) + u_out * math.sqrt(ex)      # |sqrt(x) - sqrt(y)| <= sqrt(|x - y|)


def check(kind, dtype, got, exp, wins, ddof, exact_floats=False):
    gv, gm = got
    assert gv.dtype == np.dtype(ro.out_dtype(kind, dtype)), (kind, dtype, gv.dtype)
    gl = as_list(gv, gm)
    # a large window costs O(w) per row for the bound: its finite rows are sampled (every validity bit and non-finite class
    # is still checked on every row)
    stride = 1 if wins.w <= 64 else max(1, len(gl) // (48 if kind in ("rolling_var", "rolling_std") else 300))
    bad = []
    for r, (a, b) in enumerate(zip(gl, exp)):
        if same(a, b):
            continue
        if (a is None) == (b is None) and not exact_floats and gv.dtype.kind == "f" and kind != "rolling_min" and kind != "rolling_max":
            if math.isfinite(b) and math.isfinite(a) and r % stride:
                continue
            if within_bound(kind, dtype, a, b, wins[r], ddof):
                continue
        bad.append((r, a, b))
    assert not bad, f"{kind} {dtype}: {len(bad)} rows differ, first {bad[:5]}"


def run(plb, x, valid, dtype, w, center, kinds, keys=(), order=None, ms_set=None, ddof=1, exact_floats=False):
    n = len(x)
    col = (x, valid) if valid is not None else x
    ops, meta = [], []
    for kind in kinds:
        for ms in sorted(ms_set if ms_set is not None else {0, 1, w}):
            opts = {"window_size": w, "min_samples": ms, "center": center}
            if kind in ("rolling_var", "rolling_std"):
                opts["ddof"] = ddof
            ops.append((kind, col, opts))
            meta.append((kind, ms))
    got = plb.rolling(ops, partition_by=list(keys), order_by=order)
    xs = as_list(x, valid)
    kl = [k.tolist() for k in keys]
    groups = list(zip(*kl)) if kl else [0] * n
    parts = ro.partition_order(groups, order.tolist() if order is not None else None)
    wins = Windows(xs, parts, w, center)
    rdt = "int64" if dtype in ("int8", "int16", "uint8", "uint16") else dtype
    for (kind, ms), g in zip(meta, got):
        d = rdt if kind not in ("rolling_min", "rolling_max") else dtype
        exp = ro.rolling_over(kind, xs, d, groups, order.tolist() if order is not None else None, window_size=w, min_samples=ms,
                              center=center, ddof=ddof)
        check(kind, dtype, g, exp, wins, ddof, exact_floats)


N = 3 * TILE + 77
SMALL_MAX = 128      # B <= 128 runs the one-pass shared-memory plan (k_roll_tile), larger B the three-pass plan
WS = [1, 2, 7, SMALL_MAX - 1, SMALL_MAX, SMALL_MAX + 1, TILE - 1, TILE, TILE + 1, 3 * TILE, N + 5]


@pytest.mark.parametrize("dtype", ["int8", "int32", "uint32", "int64", "uint64", "float32", "float64", "bool"])
@pytest.mark.parametrize("w", WS)
@pytest.mark.parametrize("center", [False, True])
def test_whole_column_grid(plb, dtype, w, center):
    rng = np.random.default_rng(WS.index(w) * 31 + len(dtype) + center)
    kinds = ["rolling_sum"] if dtype == "bool" else KINDS
    for nulls in (False, True):
        x, valid = values(rng, dtype, N, nulls)
        run(plb, x, valid, dtype, w, center, kinds)


@pytest.mark.parametrize("dtype", ["int16", "uint64", "float32", "float64"])
@pytest.mark.parametrize("shape", ["partitioned", "ordered"])
@pytest.mark.parametrize("w", [1, 3, 20, SMALL_MAX, SMALL_MAX + 1, TILE + 3])
def test_partitioned_forms(plb, dtype, shape, w):
    """partitions shorter than w, one-row partitions, partitions crossing tile boundaries"""
    rng = np.random.default_rng(w + len(shape) + len(dtype))
    n = 2 * TILE + 333
    x, valid = values(rng, dtype, n, True)
    g = rng.integers(0, 40, n)
    g[::101] = 1000 + np.arange(len(g[::101]))      # one-row partitions
    g[rng.random(n) < 0.3] = 7                        # one partition crossing tiles
    order = rng.integers(0, 50, n) if shape == "ordered" else None
    for center in (False, True):
        run(plb, x, valid, dtype, w, center, KINDS, keys=[g], order=order, ms_set={0, 1})


def test_heads_on_tile_boundaries_and_string_keys(plb):
    n = 4 * TILE + 9
    rng = np.random.default_rng(3)
    x = rng.integers(-1 << 40, 1 << 40, n).astype(np.int64)
    g = np.repeat(np.arange((n + TILE - 1) // TILE), TILE)[:n]      # segment heads exactly on the scan tiles
    run(plb, x, None, "int64", 5, False, ["rolling_sum", "rolling_max"], keys=[g], ms_set={0, 5})
    words = ["a", "bb", None, "", "ccc"]
    s = [words[i] for i in rng.integers(0, len(words), n)]
    got = plb.rolling([("rolling_sum", x, {"window_size": 4})], partition_by=[plb.StringColumn(s)])
    exp = ro.rolling_over("rolling_sum", x.tolist(), "int64", s, None, window_size=4)
    assert all(same(a, b) for a, b in zip(as_list(*got[0]), exp))


def test_million_small_partitions(plb):
    n = 3_000_000
    rng = np.random.default_rng(11)
    g = rng.integers(0, 1_000_000, n)
    x = rng.integers(-1 << 62, 1 << 62, n, dtype=np.int64)
    vals, valid = plb.rolling([("rolling_max", x, {"window_size": 3, "min_samples": 1})], partition_by=[g])[0]
    o = np.argsort(g, kind="stable")
    xs, gs = x[o], g[o]
    best = xs.copy()
    for k in (1, 2):
        same_seg = np.zeros(n, bool)
        same_seg[k:] = gs[k:] == gs[:-k]
        prev = np.empty_like(xs)
        prev[k:] = xs[:-k]
        best = np.where(same_seg, np.maximum(best, prev), best)
    want = np.empty_like(x)
    want[o] = best
    assert np.array_equal(vals, want) and (valid is None or valid.all())


def test_over_2e7_rows_against_numpy(plb):
    """rolling_sum(5) / rolling_mean(5) .over(g) on 2e7 rows against a numpy restatement independent of bl_over"""
    n, w = 20_000_000, 5
    rng = np.random.default_rng(17)
    g = rng.integers(0, 10_000, n)
    x = rng.integers(-1000, 1000, n).astype(np.int64)
    s, m = plb.rolling([("rolling_sum", x, {"window_size": w, "min_samples": 1}), ("rolling_mean", x, {"window_size": w, "min_samples": 1})],
                       partition_by=[g])
    o = np.argsort(g, kind="stable")
    xs, gs = x[o], g[o]
    head = np.ones(n, bool)
    head[1:] = gs[1:] != gs[:-1]
    start = np.maximum.accumulate(np.where(head, np.arange(n), 0))
    P = np.concatenate([[0], np.cumsum(xs)])
    i = np.arange(n)
    lo = np.maximum(i - (w - 1), start)
    ws = P[i + 1] - P[lo]
    want = np.empty(n, np.int64)
    want[o] = ws
    assert np.array_equal(s[0], want)
    cnt = np.empty(n, np.int64)
    cnt[o] = i + 1 - lo
    assert np.array_equal(m[0], want / cnt)      # sums of small integers are exact, so is the mean's one division


def test_deterministic_floats_bit_identical(plb):
    rng = np.random.default_rng(23)
    n = 2 * TILE + 50
    plb.set_deterministic(True)
    try:
        for dtype in ("float32", "float64"):
            x, valid = values(rng, dtype, n, True)
            g = rng.integers(0, 6, n)
            for w, center in ((1, False), (4, True), (37, False), (TILE + 1, True)):
                run(plb, x, valid, dtype, w, center, ["rolling_sum", "rolling_mean", "rolling_var", "rolling_std"], ms_set={0, min(2, w)}, exact_floats=True)
                run(plb, x, valid, dtype, w, center, ["rolling_sum", "rolling_mean", "rolling_var", "rolling_std"], keys=[g], ms_set={1}, ddof=0,
                    exact_floats=True)
        x = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
        run(plb, x, None, "int64", 9, False, ["rolling_mean", "rolling_std"], ms_set={1}, exact_floats=True)
    finally:
        plb.set_deterministic(False)


def test_finite_float_bound_large_window(plb):
    rng = np.random.default_rng(29)
    n = 5 * TILE
    for dtype in ("float32", "float64"):
        x, _ = values(rng, dtype, n, False, finite=True)
        x += np.asarray(1e4, dtype)      # an offset mean: the variance bound's condition factor
        run(plb, x, None, dtype, 2 * TILE + 17, False, ["rolling_sum", "rolling_mean", "rolling_var", "rolling_std"], ms_set={1})


def _plan_kernels(plb, fn):
    plb.profile_reset()
    plb.profile_enable(True)
    fn()
    prof = plb.profile()
    plb.profile_enable(False)
    return {k for k in prof if k.startswith("rolling_") or k.startswith("sort_") or k.startswith("over_")}


def test_profile_shows_the_plan(plb):
    x = np.arange(100_000, dtype=np.float64)
    g = np.arange(100_000) % 7
    assert _plan_kernels(plb, lambda: plb.rolling_agg("rolling_mean", x, SMALL_MAX)) == {"rolling_tile"}
    assert _plan_kernels(plb, lambda: plb.rolling_agg("rolling_mean", x, SMALL_MAX + 1)) == {"rolling_prefix", "rolling_suffix", "rolling_out"}
    k = _plan_kernels(plb, lambda: plb.rolling([("rolling_max", x, {"window_size": 20})], partition_by=[g]))
    assert "rolling_tile" in k and "rolling_prefix" not in k
    plb.set_deterministic(True)
    try:
        k = _plan_kernels(plb, lambda: plb.rolling_agg("rolling_mean", x, 20))
    finally:
        plb.set_deterministic(False)
    assert k == {"rolling_fold"}, k


@pytest.mark.parametrize("w", [5, SMALL_MAX + 72])
def test_whole_column_launch_wraps_the_grid(plb, sm, w):
    """more rows than the output grid covers in one sweep (sm_count x 8 CTAs x 256 threads), on both plans"""
    n = sm * 8 * 256 * 3 + 1001
    rng = np.random.default_rng(w)
    x = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
    valid = rng.random(n) >= 0.1
    vals, ok = plb.rolling([("rolling_sum", (x, valid), {"window_size": w, "min_samples": w - 2})])[0]
    xv = np.where(valid, x, 0).view(np.uint64)
    c = np.concatenate([np.zeros(1, np.uint64), np.cumsum(xv, dtype=np.uint64)])
    cnt = np.concatenate([[0], np.cumsum(valid)])
    i = np.arange(n)
    lo = np.maximum(i - (w - 1), 0)
    want_ok = cnt[i + 1] - cnt[lo] >= w - 2
    assert np.array_equal(ok, want_ok)
    assert np.array_equal(vals[want_ok], (c[i + 1] - c[lo]).view(np.int64)[want_ok])


def test_single_row_and_empty(plb):
    one = plb.rolling_agg("rolling_sum", np.array([5], np.int32), 3, min_samples=1)
    assert one[0].tolist() == [5]
    empty = plb.rolling([("rolling_mean", np.array([], np.int8), {"window_size": 2}), ("rolling_max", np.array([], np.uint16), {"window_size": 2})])
    assert len(empty[0][0]) == 0 and empty[0][0].dtype == np.float64 and empty[1][0].dtype == np.uint16


def test_device_inputs_and_outputs(plb):
    rng = np.random.default_rng(12)
    n = 3 * TILE
    x = rng.integers(-9, 9, n).astype(np.int32)
    m = rng.random(n) > 0.3
    g = rng.integers(0, 4, n)
    dx, dg = plb.to_device(x, m), plb.to_device(g)
    ops = [("rolling_sum", dx, {"window_size": 4, "min_samples": 2}), ("rolling_std", dx, {"window_size": 9, "center": True})]
    hops = [("rolling_sum", (x, m), {"window_size": 4, "min_samples": 2}), ("rolling_std", (x, m), {"window_size": 9, "center": True})]
    outs = plb.rolling(ops, partition_by=[dg], location=plb.DEVICE)
    host = plb.rolling(hops, partition_by=[g])
    for d, h in zip(outs, host):
        dv, dm = d.to_numpy()
        assert np.array_equal(dm, h[1])
        assert np.array_equal(dv[h[1]], h[0][h[1]])


def test_errors(plb):
    import ctypes as C
    B = plb.B200Error
    with pytest.raises(B, match="UNSUPPORTED"):
        plb.rolling_agg("rolling_min", np.array([True, False]), 2)
    with pytest.raises(B, match="INVALID"):
        plb.rolling([("rolling_sum", np.arange(3), {"window_size": 2}), ("rolling_sum", np.arange(4), {"window_size": 2})])
    with pytest.raises(B, match="INVALID"):
        plb.rolling([("rolling_sum", np.arange(3), {"window_size": 2})], partition_by=[np.arange(4)])
    with pytest.raises(B, match="UNSUPPORTED"):
        plb.rolling([("rolling_sum", np.arange(3), {"window_size": 2})], partition_by=[np.array([True, False, True])])
    x = plb.Column(np.arange(3))
    st = x.struct()
    outs = (plb.BlColumn * 1)()

    def call(kind=40, center=0, ws=2, ms=1, ddof=1, reserved=0, key=None):
        op = (plb.BlRollingOp * 1)(plb.BlRollingOp(kind, center, ws, ms, ddof, reserved, C.pointer(st)))
        return plb.lib().bl_rolling(C.byref(key) if key is not None else None, 1 if key is not None else 0, None, op, 1, plb.HOST, outs)
    assert call(kind=99) == 1
    assert call(ms=3) == 1
    assert call(ws=-1, ms=0) == 1
    assert call(ms=-1) == 1
    assert call(ddof=256) == 1
    assert call(ddof=-1) == 1
    assert call(reserved=1) == 1
    assert call(center=2) == 1
    assert call(ws=0, ms=0) == 4
    assert call(key=plb.BlSortKey(C.pointer(st), None, 0, 1)) == 1      # partition flags must be 0


def test_plugin_entries(plb):
    """_polars_plugin_bl_rolling_* through the expression-plugin ABI: input 0 the values, then the partition keys"""
    pa = pytest.importorskip("pyarrow")
    from test_gpu_plugin_abi import Caller
    caller = Caller(plb.lib())
    rng = np.random.default_rng(13)
    n = 3 * TILE + 21
    x = rng.integers(-1000, 1000, n).astype(np.int64)
    valid = rng.random(n) >= 0.15
    g1 = rng.integers(0, 7, n)
    xs = as_list(x, valid)
    X = pa.array(x, mask=~valid)
    cases = [
        ("rolling_sum", {"window_size": 3}, [g1], dict(window_size=3), pa.int64()),
        ("rolling_max", {"window_size": 5, "min_samples": 1, "center": True}, [], dict(window_size=5, min_samples=1, center=True), pa.int64()),
        ("rolling_var", {"window_size": 4, "min_samples": 2, "ddof": 0}, [g1], dict(window_size=4, min_samples=2, ddof=0), pa.float64()),
        # rolling_sum(3, min_samples=None) as Polars' signature passes it: None means window_size
        ("rolling_sum", {"window_size": 3, "min_samples": None, "center": False}, [], dict(window_size=3, min_samples=3), pa.int64()),
    ]
    for entry, kwargs, keys, opts, typ in cases:
        inputs = [("x", [X.slice(0, 1000), X.slice(1000)])] + [(f"k{i}", [pa.array(k)]) for i, k in enumerate(keys)]
        out = caller.call(entry, inputs, kwargs)
        assert out.type == typ, (entry, out.type)
        groups = list(zip(*[k.tolist() for k in keys])) if keys else [0] * n
        exp = ro.rolling_over(entry, xs, "int64", groups, None, **opts)
        got = out.to_pylist()
        if entry == "rolling_var":
            assert all((a is None) == (b is None) and (a is None or abs(a - b) <= 1e-9 * max(1.0, abs(b))) for a, b in zip(got, exp))
        else:
            assert got == exp, (entry, next(i for i, (a, b) in enumerate(zip(got, exp)) if a != b))
    with pytest.raises(Exception):
        caller.call("rolling_sum", [("x", [X])], {"min_samples": 1})      # window_size is required
