"""GPU tests of the rolling quantile (bl_rolling_quantile / bl_rolling_quantile_by) against tests/rolling_quantile_oracle.py:
every method and quantile bit for bit (with -0.0 / +0.0 and NaN payloads canonicalised, which the reference leaves open),
every value dtype at its extremes, null patterns, min_samples, center, partitions and order_by, every `closed` with
duplicate, null and shuffled times, sizes past the grids of the build and query kernels up to 25 levels, several ops on
one matrix, device output, the C ABI's errors and the plugin entries."""
import ctypes as C

import numpy as np
import pytest

import rolling_oracle as ro
import rolling_quantile_oracle as rq

pytestmark = pytest.mark.gpu
QS = [0.0, 0.1, 0.25, 0.3, 0.5, 0.75, 0.9, 1.0]
DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]
BV_TILE = 1792      # positions per CTA of the build kernels


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as plb
    plb.init()
    return plb


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


def canon(v, T):
    """values with -0.0 -> +0.0 and every NaN one NaN, as integer bits"""
    with np.errstate(invalid="ignore"):
        v = np.asarray(v, dtype=T) + T(0)
    v = np.where(np.isnan(v), T(np.nan), v).astype(T)
    return v.view(np.uint32 if T is np.float32 else np.uint64)


def assert_matches(got, exp, T, what=""):
    """got: (values, validity or None) from the device; exp: oracle list (None = null)"""
    gv, gm = got
    assert gv.dtype == T, what
    ev = np.array([T(0) if e is None else e for e in exp], dtype=T)
    em = np.array([e is not None for e in exp], dtype=bool)
    gmask = np.ones(len(gv), bool) if gm is None else np.asarray(gm, bool)
    assert np.array_equal(gmask, em), (what, np.nonzero(gmask != em)[0][:10])
    bad = np.nonzero(canon(np.where(em, gv, T(0)), T) != canon(ev, T))[0]
    assert bad.size == 0, (what, bad[:10], gv[bad[:5]], ev[bad[:5]])


def assert_np(got, exp_vals, exp_ok, T, what=""):
    gv, gm = got
    gmask = np.ones(len(gv), bool) if gm is None else np.asarray(gm, bool)
    assert np.array_equal(gmask, exp_ok), what
    bad = np.nonzero(canon(np.where(exp_ok, gv, T(0)), T) != canon(np.where(exp_ok, exp_vals, T(0)), T))[0]
    assert bad.size == 0, (what, bad[:10], gv[bad[:5]], exp_vals[bad[:5]])


def run(plb, col, q, method, w, ms=None, center=False, **kw):
    return plb.rolling_quantile([(col, {"quantile": q, "interpolation": method, "window_size": w, "min_samples": ms, "center": center})], **kw)[0]


def pyvals(x):
    return [float(v) for v in x.tolist()] if x.dtype.kind == "f" else [int(v) for v in x.tolist()]


def float_pool(rng, ft, n):
    info = np.finfo(ft)
    pool = np.array([0.0, -0.0, np.inf, -np.inf, info.max, -info.max, info.tiny, info.smallest_subnormal, -info.smallest_subnormal,
                     1.5, -1.5, 3.0, 3.0, 2.0], ft)
    x = rng.choice(pool, n)
    it = np.uint32 if np.dtype(ft).itemsize == 4 else np.uint64
    nan_bits = (np.array([0x7FC00000, 0xFFC00001, 0x7F800001], np.uint32) if it is np.uint32 else
                np.array([0x7FF8000000000000, 0xFFF8000000000001, 0x7FF0000000000001], np.uint64))
    at = rng.random(n) < 0.08
    x[at] = rng.choice(nan_bits, int(at.sum())).astype(it).view(ft)
    return x


def extremes(rng, dtype, n):
    if dtype.startswith("float"):
        return float_pool(rng, np.dtype(dtype).type, n)
    info = np.iinfo(dtype)
    pool = np.array([info.min, info.min + 1, 0, 1, info.max // 3, info.max - 1, info.max], dtype)
    if dtype in ("int64", "uint64"):      # beyond 2^53: neighbours that round to one f64
        pool = np.concatenate([pool, np.array([2 ** 53 + 1, 2 ** 53 + 3, 2 ** 60 + 5], dtype)])
    return rng.choice(pool, n)


# ------------------------------------------------------------------------------------------------ known answers
def test_known_answers(plb):
    import json
    import os
    kats = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rolling_quantile_kats.json")))
    for c in kats:
        vals = np.array([0.0 if v is None else v for v in c["values"]])
        valid = np.array([v is not None for v in c["values"]])
        col = (vals, valid) if not valid.all() else vals
        opts = {"quantile": c["quantile"], "interpolation": c["method"], "window_size": c["window_size"], "min_samples": c["min_samples"]}
        if "by" in c:
            got = plb.rolling_quantile_by([(col, dict(opts, closed=c["closed"]))], np.array(c["by"], np.int64))[0]
        else:
            got = plb.rolling_quantile([(col, dict(opts, center=c["center"]))])[0]
        assert_matches(got, c["expected"], np.float64, c["src"])


# ------------------------------------------------------------------------------------------------ methods, dtypes, nulls
@pytest.mark.parametrize("method", rq.METHODS)
def test_every_method_and_quantile(plb, method):
    rng = np.random.default_rng(1)
    n = 257
    x = float_pool(rng, np.float64, n)
    valid = rng.random(n) > 0.15
    for q in QS:
        for w, ms, center in ((1, 1, False), (2, 0, False), (7, 1, True), (7, 7, False), (40, 3, True), (300, 1, False)):
            got = run(plb, (x, valid), q, method, w, ms, center)
            exp = rq.rolling_quantile(pyvals(x), list(valid), "float64", q, method, w, ms, center)
            assert_matches(got, exp, np.float64, (q, w, ms, center))


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_at_its_extremes(plb, dtype):
    rng = np.random.default_rng(2)
    n = 600
    x = extremes(rng, dtype, n)
    valid = rng.random(n) > 0.1
    T = rq.out_type(dtype)
    for method in rq.METHODS:
        for q, w in ((0.3, 5), (0.5, 4), (0.9, 33)):
            got = run(plb, (x, valid), q, method, w, 1)
            exp = rq.rolling_quantile(pyvals(x), list(valid), dtype, q, method, w, 1)
            assert_matches(got, exp, T, (dtype, method, q, w))


def test_linear_inf_inf_is_nan_and_float32_arithmetic(plb):
    x = np.array([np.inf, np.inf, np.inf, 1.0, 2.0])
    got = run(plb, x, 0.5, "linear", 2)
    assert np.isnan(got[0][1]) and np.isnan(got[0][2])
    f = np.array([1.0, 1.1, 1.7, -3.3, 1e-3], np.float32)
    for method in ("linear", "midpoint"):
        for q in (0.3, 0.7):
            got = run(plb, f, q, method, 3, 1)
            exp = rq.rolling_quantile(pyvals(f), [True] * 5, "float32", q, method, 3, 1)
            assert_matches(got, exp, np.float32, (method, q))


@pytest.mark.parametrize("pattern", ["none", "all", "runs", "alternating"])
def test_null_patterns(plb, pattern):
    rng = np.random.default_rng(3)
    n = 500
    x = rng.normal(size=n)
    valid = {"none": np.ones(n, bool), "all": np.zeros(n, bool), "runs": (np.arange(n) // 37) % 2 == 0,
             "alternating": np.arange(n) % 2 == 0}[pattern]
    for method in rq.METHODS:
        for w, ms in ((1, 0), (1, 1), (8, 0), (8, 1), (8, 8), (n + 5, 1)):
            got = run(plb, (x, valid), 0.25, method, w, ms, center=w == 8)
            exp = rq.rolling_quantile(pyvals(x), list(valid), "float64", 0.25, method, w, ms, w == 8)
            assert_matches(got, exp, np.float64, (pattern, method, w, ms))


# ------------------------------------------------------------------------------------------------ partitions, order_by
@pytest.mark.parametrize("descending", [False, True])
def test_partitions_and_order_by(plb, descending):
    rng = np.random.default_rng(4)
    n = 3000
    x = rng.integers(-50, 50, n).astype(np.int32)
    valid = rng.random(n) > 0.2
    g = rng.integers(0, 40, n)
    t = rng.permutation(n).astype(np.int64)
    order = (-t if descending else t).tolist()
    for method in ("nearest", "linear", "midpoint"):
        for w, center in ((5, False), (6, True), (200, False)):
            got = plb.rolling_quantile([((x, valid), {"quantile": 0.4, "interpolation": method, "window_size": w, "min_samples": 1, "center": center})],
                                       partition_by=[g], order_by=t, descending=descending)[0]
            exp = rq.rolling_quantile_over(pyvals(x), list(valid), "int32", g.tolist(), order, q=0.4, method=method, window_size=w,
                                           min_samples=1, center=center)
            assert_matches(got, exp, np.float64, (method, w, center))
    got = plb.rolling_quantile([(x, {"quantile": 0.5, "window_size": 3})], partition_by=[g])[0]      # partitions alone
    exp = rq.rolling_quantile_over(pyvals(x), [True] * n, "int32", g.tolist(), None, q=0.5, method="nearest", window_size=3)
    assert_matches(got, exp, np.float64, "partitions")


# ------------------------------------------------------------------------------------------------ time windows
@pytest.mark.parametrize("closed", ["right", "left", "both", "none"])
def test_time_windows(plb, closed):
    rng = np.random.default_rng(5)
    n = 1500
    x = rng.normal(size=n).astype(np.float32)
    valid = rng.random(n) > 0.1
    t = np.sort(rng.integers(0, 400, n)).astype(np.int64)      # duplicate times
    for shuffled in (False, True):
        tt = t if not shuffled else rng.permutation(t)
        tv = np.ones(n, bool) if not shuffled else rng.random(n) > 0.05
        by = (tt, tv) if not tv.all() else tt
        for method in ("lower", "linear", "equiprobable"):
            for P, ms in ((1, 1), (7, 0), (7, 3), (1000, 1)):
                got = plb.rolling_quantile_by([((x, valid), {"quantile": 0.6, "interpolation": method, "window_size": P, "min_samples": ms,
                                                             "closed": closed})], by)[0]
                exp = rq.rolling_quantile_by(pyvals(x), list(valid), "float32", tt.tolist(), list(tv), P, closed, 0.6, method, ms)
                assert_matches(got, exp, np.float32, (shuffled, method, P, ms))
    g = rng.integers(0, 5, n)
    got = plb.rolling_quantile_by([((x, valid), {"quantile": 0.5, "interpolation": "linear", "window_size": 9, "closed": closed})], t, partition_by=[g])[0]
    exp = rq.rolling_quantile_by(pyvals(x), list(valid), "float32", t.tolist(), [True] * n, 9, closed, 0.5, "linear", 1, parts=(g.tolist(),))
    assert_matches(got, exp, np.float32, "partitioned")


def test_date_and_datetime_by(plb):
    rng = np.random.default_rng(6)
    n = 400
    x = rng.integers(0, 1000, n).astype(np.int64)
    days = np.sort(rng.integers(18000, 18100, n))
    d = days.astype("datetime64[D]")
    got = plb.rolling_median_agg_by(x, d, "3d")
    us = (days * 86_400_000_000).tolist()
    exp = rq.rolling_quantile_by(pyvals(x), [True] * n, "int64", us, [True] * n, 3 * 86_400_000_000, "right", 0.5, "linear", 1)
    assert_matches(got, exp, np.float64, "date")
    ns = np.sort(rng.integers(0, 10 ** 12, n))
    got = plb.rolling_quantile_agg_by(x, ns.astype("datetime64[ns]"), 0.2, "90s", "higher", closed="left")
    exp = rq.rolling_quantile_by(pyvals(x), [True] * n, "int64", ns.tolist(), [True] * n, 90 * 10 ** 9, "left", 0.2, "higher", 1)
    assert_matches(got, exp, np.float64, "datetime ns")


# ------------------------------------------------------------------------------------------------ sizes
def test_sizes_past_the_grids(plb, sm):
    # the query kernel's grid is capped at 8 CTAs of 256 per SM; the build kernels run one CTA per 1792 positions
    rng = np.random.default_rng(7)
    for n in (BV_TILE - 1, BV_TILE, BV_TILE + 1, 224 * 37, sm * 8 * 256 * 3 + 37):
        x = rng.integers(-1000, 1000, n).astype(np.int64)
        valid = rng.random(n) > 0.05
        for method, q, w, center in (("linear", 0.5, 20, False), ("nearest", 0.9, 1001, True), ("midpoint", 0.3, 3, False)):
            bounds = np.array([(ro.det_offsets_center if center else ro.det_offsets)(i, w, n) for i in range(n)]) if n < 20000 else None
            if bounds is None:
                i = np.arange(n)
                if center:
                    r = w // 2 + (w & 1)
                    s, e = np.maximum(i - (w - r), 0), np.minimum(i + r, n)
                else:
                    s, e = np.maximum(i - w + 1, 0), i + 1
            else:
                s, e = bounds[:, 0], bounds[:, 1]
            ev, ok = rq.numpy_rolling_quantile(x, valid, "int64", q, method, s, e, 1)
            assert_np(run(plb, (x, valid), q, method, w, 1, center), ev, ok, np.float64, (n, method))


def test_twenty_five_levels(plb):
    n = 2 ** 24 + 1
    rng = np.random.default_rng(8)
    x = rng.normal(size=n)
    i = np.arange(n)
    w = 77
    ev, ok = rq.numpy_rolling_quantile(x, None, "float64", 0.37, "linear", np.maximum(i - w + 1, 0), i + 1, w)
    assert_np(run(plb, x, 0.37, "linear", w), ev, ok, np.float64, "2^24 + 1")


def test_ascending_column_closed_form(plb):
    n = 2 ** 25
    x = np.arange(n, dtype=np.float64)
    i = np.arange(n)
    for w, method in ((1000, "linear"), (2 ** 20, "lower")):
        s = np.maximum(i - w + 1, 0)
        m = (i - s + 1).astype(np.float64)
        fi = (m - 1.0) * 0.3
        lo = np.floor(fi)
        exp = (s + lo) + ((fi - lo) * 1.0 if method == "linear" else 0.0)
        got = run(plb, x, 0.3, method, w, 1)
        assert got[1] is None or got[1].all()
        assert np.array_equal(got[0], exp), method


# ------------------------------------------------------------------------------------------------ call forms
def test_several_ops_share_one_matrix(plb):
    rng = np.random.default_rng(9)
    n = 20_000
    x = rng.normal(size=n)
    valid = rng.random(n) > 0.1
    col = (x, valid)
    ops = [(col, {"quantile": q, "interpolation": m, "window_size": w, "min_samples": 1, "center": c})
           for q, m, w, c in ((0.25, "linear", 10, False), (0.5, "linear", 10, False), (0.75, "nearest", 99, True), (0.1, "lower", 5, False))]
    plb.profile_enable(True)
    plb.profile_reset()
    together = plb.rolling_quantile(ops)
    launches = plb.profile()
    plb.profile_enable(False)
    assert launches["rolling_quantile_ranks"]["launches"] == 1      # one build for four ops
    for op, got in zip(ops, together):
        alone = plb.rolling_quantile([op])[0]
        assert np.array_equal(got[0], alone[0]) and np.array_equal(got[1], alone[1])
        dev = plb.rolling_quantile([op], location=plb.DEVICE)[0]
        assert dev.location == plb.DEVICE
        dv, dm = dev.to_numpy()
        assert np.array_equal(dv, alone[0]) and np.array_equal(dm, alone[1])
    t = np.sort(rng.integers(0, 10 ** 6, n))
    byops = [(col, {"quantile": q, "interpolation": "linear", "window_size": P}) for q, P in ((0.5, 100), (0.9, 100), (0.5, 5000))]
    for op, got in zip(byops, plb.rolling_quantile_by(byops, t)):
        alone = plb.rolling_quantile_by([op], t)[0]
        assert np.array_equal(got[0], alone[0]) and np.array_equal(got[1], alone[1])


def test_header_errors(plb):
    L = plb.lib()
    x = np.arange(10, dtype=np.int64)
    st = plb.Column(x).struct()
    bst = plb.Column(np.ones(10, bool)).struct()
    short = plb.Column(x[:5]).struct()
    outs = (plb.BlColumn * 2)()
    INVALID, UNSUPPORTED = 1, 4

    def fixed(ops, parts=None, n_parts=0):
        arr = (plb.BlRollingQuantileOp * len(ops))(*ops)
        return L.bl_rolling_quantile(parts, C.c_int32(n_parts), None, arr, C.c_int32(len(ops)), C.c_int32(plb.HOST), outs)

    def by(ops, b=st):
        arr = (plb.BlRollingQuantileByOp * len(ops))(*ops)
        return L.bl_rolling_quantile_by(None, C.c_int32(0), C.byref(b) if b is not None else None, arr, C.c_int32(len(ops)), C.c_int32(plb.HOST), outs)

    F = plb.BlRollingQuantileOp
    B = plb.BlRollingQuantileByOp
    p = C.pointer(st)
    assert fixed([F(0.5, 4, 0, 3, 1, p)]) == 0
    for q in (-0.1, 1.5, float("nan")):
        assert fixed([F(q, 4, 0, 3, 1, p)]) == INVALID
        assert by([B(q, 4, 0, 3, 1, p)]) == INVALID
    assert fixed([F(0.5, 6, 0, 3, 1, p)]) == INVALID and fixed([F(0.5, -1, 0, 3, 1, p)]) == INVALID
    assert fixed([F(0.5, 4, 2, 3, 1, p)]) == INVALID                      # center
    assert fixed([F(0.5, 4, 0, 3, 4, p)]) == INVALID                      # min_samples > window_size
    assert fixed([F(0.5, 4, 0, -1, 0, p)]) == INVALID
    assert fixed([F(0.5, 4, 0, 0, 0, p)]) == UNSUPPORTED
    assert fixed([F(0.5, 4, 0, 3, 1, None)]) == INVALID
    assert fixed([F(0.5, 4, 0, 3, 1, C.pointer(bst))]) == UNSUPPORTED
    assert fixed([F(0.5, 4, 0, 3, 1, p), F(0.5, 4, 0, 3, 1, C.pointer(short))]) == INVALID
    skey = plb.BlSortKey(C.pointer(short), None, 0, 0)
    assert fixed([F(0.5, 4, 0, 3, 1, p)], (plb.BlSortKey * 1)(skey), 1) == INVALID
    assert by([B(0.5, 4, 0, 3, 1, p)]) == 0
    assert by([B(0.5, 6, 0, 3, 1, p)]) == INVALID
    assert by([B(0.5, 4, 4, 3, 1, p)]) == INVALID                         # closed
    assert by([B(0.5, 4, 0, 0, 1, p)]) == INVALID                         # P <= 0
    assert by([B(0.5, 4, 0, 3, -1, p)]) == INVALID
    assert by([B(0.5, 4, 0, 3, 1, p)], None) == INVALID
    assert by([B(0.5, 4, 0, 3, 1, p)], plb.Column(x.astype(np.float64)).struct()) == INVALID      # `by` dtype
    assert by([B(0.5, 4, 0, 3, 1, p)], short) == INVALID
    assert by([B(0.5, 4, 0, 3, 1, C.pointer(bst))]) == UNSUPPORTED
    # more rows than the row limits: a length-only descriptor is rejected before anything is read
    big = plb.BlColumn(3, plb.HOST, 2 ** 32, 0, 0, st.values, None, None)
    assert fixed([F(0.5, 4, 0, 3, 1, C.pointer(big))]) == UNSUPPORTED
    assert by([B(0.5, 4, 0, 3, 1, C.pointer(big))], big) == UNSUPPORTED
    big31 = plb.BlColumn(3, plb.HOST, 2 ** 31, 0, 0, st.values, None, None)
    b31key = plb.BlSortKey(C.pointer(big31), None, 0, 0)
    assert fixed([F(0.5, 4, 0, 3, 1, C.pointer(big31))], (plb.BlSortKey * 1)(b31key), 1) == UNSUPPORTED


def test_plugin_entries(plb):
    import pyarrow as pa
    from test_gpu_plugin_abi import Caller
    caller = Caller(plb.lib())
    rng = np.random.default_rng(10)
    n = 2000
    x = rng.integers(0, 50, n)
    xm = rng.random(n) < 0.1
    g = rng.integers(0, 7, n)
    t = np.sort(rng.integers(0, 5000, n)).astype(np.int64)
    X = pa.array(x, mask=xm)
    vals, valid = x.tolist(), (~xm).tolist()
    out = caller.call("rolling_quantile", [("x", [X.slice(0, 700), X.slice(700)]), ("g", [pa.array(g)])],
                      kwargs={"quantile": 0.3, "method": "higher", "window_size": 6, "min_samples": 2})
    assert out.type == pa.float64()
    exp = rq.rolling_quantile_over(vals, valid, "int64", g.tolist(), None, q=0.3, method="higher", window_size=6, min_samples=2)
    assert out.to_pylist() == [None if e is None else float(e) for e in exp]
    out = caller.call("rolling_median", [("x", [X])], kwargs={"window_size": 5, "center": True})
    exp = rq.rolling_quantile(vals, valid, "int64", 0.5, "linear", 5, 5, True)
    assert out.to_pylist() == [None if e is None else float(e) for e in exp]
    out = caller.call("rolling_quantile_by", [("x", [X]), ("t", [pa.array(t)])], kwargs={"quantile": 0.8, "method": "midpoint", "window_size": 40, "closed": "both"})
    exp = rq.rolling_quantile_by(vals, valid, "int64", t.tolist(), [True] * n, 40, "both", 0.8, "midpoint", 1)
    assert out.to_pylist() == [None if e is None else float(e) for e in exp]
    out = caller.call("rolling_median_by", [("x", [X]), ("t", [pa.array(t)]), ("g", [pa.array(g)])], kwargs={"window_size": 40})
    exp = rq.rolling_quantile_by(vals, valid, "int64", t.tolist(), [True] * n, 40, "right", 0.5, "linear", 1, parts=(g.tolist(),))
    assert out.to_pylist() == [None if e is None else float(e) for e in exp]
    with pytest.raises(RuntimeError, match="quantile"):
        caller.call("rolling_quantile", [("x", [X])], kwargs={"window_size": 3})
    with pytest.raises(RuntimeError, match="method"):
        caller.call("rolling_quantile", [("x", [X])], kwargs={"quantile": 0.5, "method": "cubic", "window_size": 3})
