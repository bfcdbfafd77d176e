"""GPU tests of the time-based rolling windows (bl_rolling_by) against tests/rolling_by_oracle.py: validity, integer SUM,
MIN / MAX and non-finite classes bit for bit; finite float SUM / MEAN / VAR / STD under the header's bounds against the
exact window value.  Widths cross the 32-position sub-blocks, the 1024-position blocks and the sparse table."""
import ctypes as C
import json
import math
import os
import zlib
from fractions import Fraction

import numpy as np
import pytest

import rolling_oracle as ro
from rolling_by_oracle import CLOSED, I64_MIN, numpy_sum_by, replay_by, window_values

pytestmark = pytest.mark.gpu
KINDS = ["rolling_sum", "rolling_mean", "rolling_min", "rolling_max", "rolling_var", "rolling_std"]
U = {"float32": 2.0 ** -24, "float64": 2.0 ** -53}


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as plb
    plb.init()
    plb.set_deterministic(False)
    return plb


def expected(kind, dtype, win, ddof, ms):
    """the reference's value of a window's non-null values (None: null); floats as Python floats of the exact value.
    is_valid: fewer than min_samples non-null values is null (rolling/sum.rs:219-221, moment.rs:321-323)"""
    if win is None or len(win) < ms:
        return None
    fl = dtype.startswith("float")
    if kind == "rolling_sum":
        if not fl:
            return ro.wrap(sum(int(v) for v in win), ro.out_dtype(kind, dtype))
    if kind in ("rolling_min", "rolling_max"):
        if not win:
            return None
        if any(v != v for v in win):
            return float("nan")
        best = win[0]
        for v in win[1:]:
            if (v > best) if kind == "rolling_max" else (v < best):
                best = v
        return best
    xs = [float(v) for v in win]
    nf = [x for x in xs if not math.isfinite(x)]
    if kind in ("rolling_sum", "rolling_mean"):
        if kind == "rolling_mean" and not xs:
            return None
        if nf:
            v = math.inf if all(x == math.inf for x in nf) else -math.inf if all(x == -math.inf for x in nf) else math.nan
        else:
            v = float(ro.exact_sum(xs))
        return v if kind == "rolling_sum" or not math.isfinite(v) else v / len(xs)
    if len(xs) <= ddof:
        return None
    if nf:
        return math.nan
    var = ro.exact_var(xs, ddof)
    return float(var) if kind == "rolling_var" else math.sqrt(float(var))


def ok_value(kind, dtype, a, b, win, ddof):
    if b is None or a is None:
        return a is None and b is None
    if isinstance(b, int) or kind in ("rolling_min", "rolling_max") and not isinstance(b, float):
        return int(a) == int(b)
    if b != b or not math.isfinite(b):
        return (a != a) if b != b else a == b
    if kind in ("rolling_min", "rolling_max"):
        return float(a) == b and math.copysign(1, float(a)) == math.copysign(1, b)
    xs = [float(v) for v in win]
    u_out = U["float32" if dtype == "float32" else "float64"]
    if kind == "rolling_sum":
        return abs(a - b) <= ro.sum_bound(xs, u_out) + U["float64"] * abs(b)
    if kind == "rolling_mean":
        return abs(a - b) <= ro.mean_bound(xs, u_out) + U["float64"] * abs(b)
    k, s, m2 = ro.exact_moments(xs)      # the header's VAR bound: 8.08 (k + 4) u M2 kappa / (k - ddof) + u_o |exact|
    m2f, mean = float(m2), float(s / k)
    kappa = math.sqrt(1 + k * mean * mean / m2f) if m2f > 0 else 1.0
    vb = 8.08 * (k + 4) * U["float64"] * m2f * kappa / (k - ddof) + u_out * float(m2 / (k - ddof))
    ex = ro.exact_var(xs, ddof)
    if kind == "rolling_var":
        return abs(Fraction(float(a)) - ex) <= Fraction(vb)
    return abs(a - math.sqrt(ex)) <= math.sqrt(vb) + u_out * math.sqrt(ex)


def full(m, n):
    """an output validity (None: no nulls) as a bool array"""
    return np.ones(n, bool) if m is None else m


def make(rng, dtype, n, nulls):
    if dtype == "bool":
        x = rng.random(n) < 0.5
    elif dtype.startswith("float"):
        x = (rng.standard_normal(n) * 1e3).astype(dtype)
        at = rng.random(n) < 0.01
        x[at] = np.array([np.nan, np.inf, -np.inf, -0.0], dtype)[rng.integers(0, 4, at.sum())]
    else:
        info = np.iinfo(dtype)
        x = rng.integers(info.min, info.max, n, dtype=dtype, endpoint=True)
    valid = rng.random(n) >= 0.15 if nulls else np.ones(n, bool)
    return x, valid


def check_all(plb, x, valid, dtype, by, by_valid, P, closed, kinds, ms_set, parts=(), ddof=1):
    n = len(x)
    col = (x, valid) if not valid.all() else x
    bcol = (by, by_valid) if not by_valid.all() else by
    ops, meta = [], []
    for kind in kinds:
        for ms in ms_set:
            opts = {"window_size": int(P), "min_samples": ms, "closed": closed}
            if kind in ("rolling_var", "rolling_std"):
                opts["ddof"] = ddof
            ops.append((kind, col, opts))
            meta.append((kind, ms))
    outs = plb.rolling_by(ops, bcol, partition_by=list(parts))
    xl = [float(v) if dtype.startswith("float") else int(v) for v in x.tolist()]
    bl = [int(v) for v in by.tolist()]
    pl = [list(p.tolist()) for p in parts]
    cache = {}
    for (kind, ms), (gv, gm) in zip(meta, outs):
        assert gv.dtype == np.dtype(ro.out_dtype(kind, dtype)), (kind, dtype, gv.dtype)
        gm = full(gm, n)
        if ms not in cache:
            cache[ms] = window_values(xl, list(valid), bl, list(by_valid), int(P), closed, ms, pl)
        wins = cache[ms]
        bad = []
        for r in range(n):
            a = None if not gm[r] else (float(gv[r]) if gv.dtype.kind == "f" else int(gv[r]))
            b = expected(kind, dtype, wins[r], ddof, ms)
            if not ok_value(kind, dtype, a, b, wins[r], ddof):
                bad.append((r, a, b))
        assert not bad, f"{kind} {dtype} ms={ms} closed={closed}: {len(bad)} rows differ, first {bad[:4]}"


@pytest.mark.parametrize("closed", CLOSED)
@pytest.mark.parametrize("dtype", ["float64", "float32", "int64", "int32"])
def test_kinds_sorted_and_shuffled(plb, dtype, closed):
    rng = np.random.default_rng(zlib.crc32(f"{dtype}-{closed}".encode()))
    n = 2600
    kinds = KINDS if dtype.startswith("float") else ["rolling_sum", "rolling_min", "rolling_max", "rolling_mean"]
    # sorted times with heavy duplicate runs; P gives windows from a handful to ~1100 positions
    t = np.cumsum(rng.integers(0, 3, n)).astype(np.int64) - 1000
    for P in (1, 31, 33, 700):
        x, valid = make(rng, dtype, n, True)
        check_all(plb, x, valid, dtype, t, np.ones(n, bool), P, closed, kinds, (0, 1, 40))
    # shuffled times with null `by`
    x, valid = make(rng, dtype, n, True)
    tb = rng.permutation(t)
    bv = rng.random(n) >= 0.1
    check_all(plb, x, valid, dtype, tb, bv, 64, closed, kinds, (0, 2))


@pytest.mark.parametrize("by_dtype", ["int32", "int64", "uint32", "uint64"])
def test_by_dtypes_and_partitions(plb, by_dtype):
    rng = np.random.default_rng(5)
    n = 3000
    t = rng.integers(0, 400, n).astype(by_dtype)
    g = rng.integers(0, 7, n).astype(np.int32)
    x, valid = make(rng, "float64", n, True)
    check_all(plb, x, valid, "float64", t, np.ones(n, bool), 50, "right", ["rolling_sum", "rolling_max", "rolling_var"], (0, 1), parts=(g,))


def test_times_near_i64_limits(plb):
    rng = np.random.default_rng(9)
    n = 1500
    t = np.sort(np.concatenate([I64_MIN + rng.integers(0, 40, n // 2), np.iinfo(np.int64).max - rng.integers(0, 40, n - n // 2)])).astype(np.int64)
    x, valid = make(rng, "int64", n, False)
    for closed in CLOSED:
        check_all(plb, x, valid, "int64", t, np.ones(n, bool), 20, closed, ["rolling_sum", "rolling_min"], (0,))


def test_long_duplicate_run_behind_left_window(plb):
    # a run of 3000 equal times: each left / none window of the run ends before it, behind the row's own block
    n = 4200
    t = np.concatenate([np.arange(600), np.full(3000, 600), 601 + np.arange(600)]).astype(np.int64)
    rng = np.random.default_rng(3)
    x, valid = make(rng, "int64", n, True)
    for closed in CLOSED:
        check_all(plb, x, valid, "int64", t, np.ones(n, bool), 300, closed, ["rolling_sum", "rolling_max"], (0, 5))


def test_equals_fixed_window_on_arange(plb):
    rng = np.random.default_rng(11)
    n = 50_000
    x = rng.integers(-10**6, 10**6, n).astype(np.int64)
    for w in (1, 20, 1023, 1025, 5000):
        got = plb.rolling_by([(k, x, {"window_size": f"{w}i", "min_samples": 1}) for k in ("rolling_sum", "rolling_min", "rolling_max")], np.arange(n))
        ref = plb.rolling([(k, x, {"window_size": w, "min_samples": 1}) for k in ("rolling_sum", "rolling_min", "rolling_max")])
        for (a, am), (b, bm) in zip(got, ref):
            am, bm = full(am, n), full(bm, n)
            assert np.array_equal(am, bm) and np.array_equal(a[am], b[bm]), w


def test_large_against_numpy(plb):
    rng = np.random.default_rng(13)
    n = 20_000_000
    t = np.cumsum(rng.exponential(1000.0, n)).astype(np.int64)
    x = rng.integers(-10**9, 10**9, n).astype(np.int64)
    for P, closed in ((30_000, "right"), (5_000_000, "left")):
        got, gm = plb.rolling_agg_by("rolling_sum", x, t, P, min_samples=0, closed=closed)
        exp, s, e = numpy_sum_by(x, t, P, closed)
        assert full(gm, n).all() and np.array_equal(got, exp)


def test_many_small_partitions(plb):
    rng = np.random.default_rng(17)
    n = 3_000_000
    g = rng.integers(0, 1_000_000, n).astype(np.int64)
    t = rng.integers(0, 100, n).astype(np.int64)
    x = rng.integers(-1000, 1000, n).astype(np.int64)
    got, gm = plb.rolling_by([("rolling_sum", x, {"window_size": "10i", "min_samples": 0})], t, partition_by=[g])[0]
    order = np.lexsort((t, g))
    gs, ts, xs = g[order], t[order], x[order]
    key = gs * 1000 + ts
    s = np.searchsorted(key, key - 10, side="right")
    e = np.searchsorted(key, key, side="right")
    c = np.concatenate([[0], np.cumsum(xs)])
    exp = np.empty(n, np.int64)
    exp[order] = c[e] - c[s]
    assert full(gm, n).all() and np.array_equal(got, exp)


@pytest.mark.parametrize("closed", CLOSED)
@pytest.mark.parametrize("dtype", ["float64", "float32"])
def test_deterministic_bit_for_bit(plb, dtype, closed):
    # no two rows of a partition share a time; nulls in the values and in `by`; min_samples 3 makes the update skip run
    rng = np.random.default_rng(zlib.crc32(f"det-{dtype}-{closed}".encode()))
    n = 2500
    t = rng.permutation(rng.choice(10**6, n, replace=False)).astype(np.int64)
    bv = rng.random(n) >= 0.05
    x, valid = make(rng, dtype, n, True)
    g = rng.integers(0, 3, n)
    xl = [float(v) for v in x.tolist()]
    for parts in ((), (g,)):
        ops, meta = [], []
        for kind in ("rolling_sum", "rolling_mean", "rolling_var", "rolling_std"):
            for ms in (0, 3):
                opts = {"window_size": 4000, "min_samples": ms, "closed": closed}
                ops.append((kind, (x, valid), opts))
                meta.append((kind, ms))
        plb.set_deterministic(True)
        try:
            outs = plb.rolling_by(ops, (t, bv), partition_by=list(parts))
        finally:
            plb.set_deterministic(False)
        for (kind, ms), (gv, gm) in zip(meta, outs):
            gm = full(gm, n)
            exp = replay_by(kind, dtype, xl, list(valid), t.tolist(), list(bv), 4000, closed, ms, 1, [p.tolist() for p in parts])
            for r in range(n):
                e = exp[r]
                assert bool(gm[r]) == (e is not None), (kind, ms, r)
                if e is not None:
                    a = gv[r]
                    assert np.array([a]).view(np.uint8).tobytes() == np.array([e], dtype=gv.dtype).view(np.uint8).tobytes() or (a != a and e != e), (kind, ms, r, a, e)


@pytest.mark.parametrize("dtype", ["int8", "int16", "uint8", "uint16", "uint32", "uint64", "bool"])
def test_value_dtypes(plb, dtype):
    # small integers: SUM widens to Int64 and MIN / MAX narrow back; VAR / STD / MEAN over integers in f64; Bool: SUM only
    rng = np.random.default_rng(zlib.crc32(dtype.encode()))
    n = 2200
    t = np.cumsum(rng.integers(0, 3, n)).astype(np.int64)
    kinds = ["rolling_sum"] if dtype == "bool" else KINDS
    for closed in ("right", "left"):
        x, valid = make(rng, dtype, n, True)
        check_all(plb, x, valid, dtype, rng.permutation(t), np.ones(n, bool), 40, closed, kinds, (0, 3))


def plan_of(plb, fn):
    plb.profile_enable(True)
    plb.profile_reset()
    try:
        out = fn()
        prof = plb.profile()
    finally:
        plb.profile_enable(False)
    return out, prof


def test_wide_float_windows_across_the_table(plb):
    # sizes from sm_count: several CTA waves of 1024-position blocks; windows of ~20 000 positions cross ~20 blocks, so the
    # sparse table's middle runs carry float SUM / MEAN and VAR states.  Values are multiples of 1/8, so the exact window
    # moments come from integer prefix sums; the header's bounds are checked on every row.
    sm = plb.device_info()["sm_count"]
    rng = np.random.default_rng(23)
    n = sm * 1024 * 3 + 517
    t = np.cumsum(rng.integers(1, 3, n)).astype(np.int64)
    k = rng.integers(-(1 << 20), 1 << 20, n)
    x = k / 8.0
    P = 30_000
    (gs, gm), (gv, vm), (gd, dm) = plan_of(plb, lambda: plb.rolling_by([("rolling_sum", x, {"window_size": P}), ("rolling_mean", x, {"window_size": P}),
                                                                        ("rolling_var", x, {"window_size": P})], t))[0]
    s = np.searchsorted(t, t - P, side="right")
    e = np.arange(1, n + 1)
    c1 = np.concatenate([[0], np.cumsum(k)])
    c2 = np.concatenate([[0], np.cumsum(k * k)])
    cnt = e - s
    s1 = (c1[e] - c1[s]).astype(np.float64)
    s2 = [int(a) for a in (c2[e] - c2[s])]
    m2 = np.array([float(Fraction(int(c) * b - int(a) * int(a), int(c) * 64)) for a, b, c in zip(c1[e] - c1[s], s2, cnt)])
    sa = np.concatenate([[0], np.cumsum(np.abs(x))])
    absum = sa[e] - sa[s]
    u = 2.0 ** -53
    assert full(gm, n).all() and np.all(np.abs(gs - s1 / 8) <= 1.01 * (cnt - 1) * u * absum + u * np.abs(s1 / 8))
    assert np.all(np.abs(gv - s1 / 8 / cnt) <= (1.01 * (cnt - 1) * u * absum + u * np.abs(s1 / 8)) / cnt + 3 * u * np.abs(s1 / 8 / cnt))
    mean = s1 / 8 / cnt
    ok = cnt > 1
    kappa = np.sqrt(1 + cnt * mean * mean / np.where(m2 > 0, m2, 1))
    exact = m2 / np.maximum(cnt - 1, 1)
    bound = 8.08 * (cnt + 4) * u * m2 * kappa / np.maximum(cnt - 1, 1) + u * exact
    assert np.array_equal(full(dm, n), ok) and np.all(np.abs(gd[ok] - exact[ok]) <= bound[ok])


def test_plan_choice(plb):
    # the largest window W chooses the plan: W <= 128 the one-pass tile kernel, wider the scans, table and output kernel
    n = 100_000
    x = np.arange(n, dtype=np.int64)
    for P, plan, other in ((128, "rolling_by_tile", "rolling_by_out"), (129, "rolling_by_out", "rolling_by_tile")):
        (got, _), prof = plan_of(plb, lambda: plb.rolling_agg_by("rolling_sum", x, np.arange(n), P))
        assert plan in prof and other not in prof, (P, sorted(prof))
        ref = plb.rolling_agg("rolling_sum", x, P, min_samples=1)[0]
        assert np.array_equal(got, ref)


def kat_cases():
    with open(os.path.join(os.path.dirname(__file__), "golden", "rolling_by_kats.json")) as f:
        return json.load(f)


def test_kats_on_device(plb):
    for c in kat_cases():
        x = np.array(c["values"], dtype=c["dtype"])
        by = np.array([0 if v is None else v for v in c["by"]], dtype=c["by_dtype"])
        bv = np.array([v is not None for v in c["by"]])
        parts = [np.unique(np.array(p), return_inverse=True)[1] for p in c["parts"]]
        opts = {"window_size": c["window_size"], "min_samples": c["min_samples"], "closed": c["closed"]}
        if c["kind"] in ("rolling_var", "rolling_std"):
            opts["ddof"] = c["ddof"]
        call = lambda: plb.rolling_by([(c["kind"], x, opts)], (by, bv) if not bv.all() else by, partition_by=parts)[0]
        if c.get("error"):
            with pytest.raises(plb.B200Error):
                call()
            continue
        gv, gm = call()
        got = [v.item() if ok else None for v, ok in zip(gv, full(gm, len(x)))]
        assert got == c["expected"], (c["src"], got)


def test_c_abi_errors(plb):
    B = plb.B200Error
    with pytest.raises(B, match="INVALID"):
        plb.rolling_agg_by("rolling_sum", np.arange(3), np.array([1, 2 ** 63, 3], dtype=np.uint64), 2)
    with pytest.raises(B, match="INVALID"):
        plb.rolling_agg_by("rolling_sum", np.arange(3), np.arange(3, dtype=np.float64), 2)
    with pytest.raises(B, match="INVALID"):
        plb.rolling_agg_by("rolling_sum", np.arange(3), np.arange(4), 2)
    with pytest.raises(B, match="UNSUPPORTED"):
        plb.rolling_by([("rolling_sum", np.arange(3), {"window_size": 2})], np.arange(3), partition_by=[np.array([True, False, True])])
    x = plb.Column(np.arange(3))
    st = x.struct()
    b = plb.Column(np.arange(3))
    bst = b.struct()
    xb = plb.Column(np.array([True, False, True]))
    xbst = xb.struct()
    outs = (plb.BlColumn * 1)()

    def call(kind=40, closed=0, ws=2, ms=1, ddof=1, reserved=0, values=st, by=bst, key=None, n_ops=1):
        op = (plb.BlRollingByOp * 1)(plb.BlRollingByOp(kind, closed, ws, ms, ddof, reserved, C.pointer(values) if values is not None else None))
        return plb.lib().bl_rolling_by(C.byref(key) if key is not None else None, 1 if key is not None else 0, C.byref(by) if by is not None else None,
                                       op, n_ops, plb.HOST, outs)
    assert call() == 0
    plb.lib().bl_column_free(C.byref(outs[0]))
    assert call(kind=99) == 1
    assert call(closed=4) == 1
    assert call(closed=-1) == 1
    assert call(ws=0) == 1
    assert call(ws=-5) == 1
    assert call(ms=-1) == 1
    assert call(ddof=256) == 1
    assert call(reserved=1) == 1
    assert call(values=None) == 1
    assert call(by=None) == 1
    assert call(n_ops=0) == 1
    assert call(kind=42, values=xbst) == 4      # Bool MIN
    assert call(kind=43, values=xbst) == 4      # Bool MAX
    assert call(key=plb.BlSortKey(C.pointer(st), None, 0, 1)) == 1      # partition flags must be 0


def test_plugin_entries(plb):
    """_polars_plugin_bl_rolling_*_by through the expression-plugin ABI: the values, the `by` column, then partition keys"""
    pa = pytest.importorskip("pyarrow")
    from test_gpu_plugin_abi import Caller
    caller = Caller(plb.lib())
    rng = np.random.default_rng(29)
    n = 5000
    x = rng.integers(-1000, 1000, n).astype(np.int64)
    valid = rng.random(n) >= 0.15
    t = rng.integers(0, 3000, n).astype(np.int64)
    g = rng.integers(0, 5, n).astype(np.int64)
    X = pa.array(x, mask=~valid)
    xl = [int(v) for v in x.tolist()]
    cases = [      # entry, kwargs, keys, (P, closed, min_samples, ddof), output type
        ("rolling_sum_by", {"window_size": 20}, [], (20, "right", 0, 1), pa.int64()),      # min_samples default 0
        ("rolling_max_by", {"window_size": 20, "closed": "left"}, [g], (20, "left", 1, 1), pa.int64()),      # default 1
        ("rolling_mean_by", {"window_size": 50, "min_samples": None, "closed": 2}, [g], (50, "both", 1, 1), pa.float64()),
        ("rolling_var_by", {"window_size": 30, "min_samples": 2, "ddof": 0, "closed": "none"}, [], (30, "none", 2, 0), pa.float64()),
        ("rolling_std_by", {"window_size": 300, "closed": "right"}, [], (300, "right", 1, 1), pa.float64()),
        ("rolling_min_by", {"window_size": 7}, [g], (7, "right", 1, 1), pa.int64()),
    ]
    for entry, kwargs, keys, (P, closed, ms, ddof), typ in cases:
        inputs = [("x", [X.slice(0, 1700), X.slice(1700)]), ("t", [pa.array(t)])] + [(f"k{i}", [pa.array(k)]) for i, k in enumerate(keys)]
        out = caller.call(entry, inputs, kwargs)
        assert out.type == typ, (entry, out.type)
        kind = entry[:-3]
        wins = window_values(xl, list(valid), t.tolist(), [True] * n, P, closed, ms, [k.tolist() for k in keys])
        for r, a in enumerate(out.to_pylist()):
            b = expected(kind, "int64", wins[r], ddof, ms)
            assert ok_value(kind, "int64", a, b, wins[r], ddof), (entry, r, a, b)
    X3 = [("x", [pa.array([1, 2, 3])]), ("t", [pa.array([0, 1, 2])])]
    for bad in ({"min_samples": 1}, {"window_size": 2, "closed": "middle"}, {"window_size": 2, "closed": 7}, {"window_size": 2, "closed": True},
                {"window_size": 2.5}, {"window_size": float(2 ** 60)}, {"window_size": 0}):
        with pytest.raises(RuntimeError):
            caller.call("rolling_sum_by", X3, bad)
