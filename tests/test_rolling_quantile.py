"""CPU tests (-m "not gpu") of the rolling quantile's references, binding and plugin entries: the per-window oracle against
the reference's known answers and a brute force, the numpy wavelet matrix against the oracle at the level-count edges,
the binding's argument errors (raised before the library is called) and the plugin symbols and schemas."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

import rolling_oracle as ro
import rolling_quantile_oracle as rq

HERE = os.path.dirname(os.path.abspath(__file__))
KATS = json.load(open(os.path.join(HERE, "golden", "rolling_quantile_kats.json")))


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return (math.isnan(a) and math.isnan(b)) or a == b


@pytest.mark.parametrize("case", KATS, ids=[f"{i}-{c['src'].split('/')[-1].split(' ')[0]}" for i, c in enumerate(KATS)])
def test_oracle_known_answers(case):
    vals = [0.0 if v is None else v for v in case["values"]]
    valid = [v is not None for v in case["values"]]
    if "by" in case:
        got = rq.rolling_quantile_by(vals, valid, "float64", case["by"], [True] * len(vals), case["window_size"], case["closed"],
                                     case["quantile"], case["method"], case["min_samples"])
    else:
        got = rq.rolling_quantile(vals, valid, "float64", case["quantile"], case["method"], case["window_size"], case["min_samples"], case["center"])
    assert all(_same(None if g is None else float(g), x) for g, x in zip(got, case["expected"])), (got, case["expected"])


@pytest.mark.parametrize("method", ["lower", "higher", "linear", "midpoint", "nearest"])
def test_oracle_against_numpy_quantile(method):
    # numpy's quantile over each window of NaN-free floats: the same picks (nearest where (m - 1) q is not a half: numpy
    # rounds half to even), and within a few ulps for the interpolations (its arithmetic differs)
    rng = np.random.default_rng(1)
    x = rng.normal(size=60)
    for w in (1, 2, 5, 8):
        for q in (0.0, 0.1, 0.25, 0.5, 0.9, 1.0):
            got = rq.rolling_quantile(x, [True] * len(x), "float64", q, method, w, 1)
            for i, g in enumerate(got):
                win = x[max(0, i - w + 1): i + 1]
                fi = (len(win) - 1) * q
                if method == "nearest" and fi - math.floor(fi) == 0.5:
                    continue
                want = np.quantile(win, q, method=method if method != "midpoint" else "midpoint")
                if method in ("lower", "higher", "nearest"):
                    assert g == want
                else:
                    assert abs(g - want) <= 4e-16 * max(1.0, abs(want))


def test_oracle_rules():
    T = np.float64
    assert math.isnan(rq.window_quantile([math.inf, math.inf], 0.5, "linear", T))      # no lo == hi guard
    assert rq.window_quantile([math.inf, math.inf], 0.5, "midpoint", T) == math.inf
    assert math.isnan(rq.window_quantile([1.0, math.nan], 1.0, "lower", T))             # NaN is the greatest
    assert rq.window_quantile([math.nan, 2.0, 1.0], 0.5, "lower", T) == 2.0
    assert rq.window_quantile([1.0, 2.0, 3.0, 4.0], 0.5, "equiprobable", T) == 2.0      # ceil(4 * 0.5) - 1 = 1
    assert rq.window_quantile([1.0, 2.0, 3.0], 0.25, "nearest", T) == 2.0              # round(0.5) = 1, half away from zero
    f = rq.window_quantile([np.float32(1.0), np.float32(1.1)], 0.3, "linear", np.float32)
    assert isinstance(f, np.float32) and f == np.float32(np.float32(0.3) * (np.float32(1.1) - np.float32(1.0)) + np.float32(1.0))
    assert rq.rolling_quantile([1.0, 2.0], [False, False], "float64", 0.5, "linear", 2, 0) == [None, None]      # all null: null


def _wm_vs_oracle(x, valid, dtype, w, ms, center=False):
    n = len(x)
    L = ro.det_offsets_center if center else ro.det_offsets
    bounds = [L(i, w, n) for i in range(n)]
    s, e = [b[0] for b in bounds], [b[1] for b in bounds]
    for method in rq.METHODS:
        for q in (0.0, 0.3, 0.5, 1.0):
            want = rq.rolling_quantile(list(x), list(valid), dtype, q, method, w, ms, center)
            got, ok = rq.numpy_rolling_quantile(x, valid, dtype, q, method, s, e, ms)
            for i in range(n):
                assert (want[i] is None) == (not ok[i]), (method, q, i)
                if ok[i]:
                    a, b = float(got[i]), float(want[i])
                    assert (math.isnan(a) and math.isnan(b)) or a == b, (method, q, i, a, b)


@pytest.mark.parametrize("n", [1, 2, 3, 7, 8, 9, 31, 32, 33, 255, 256, 257])
def test_wavelet_matrix_level_edges(n):
    # L = 1, and n = 2^k - 1, 2^k, 2^k + 1 around each level count
    rng = np.random.default_rng(n)
    x = rng.integers(-5, 5, n).astype(np.float64)
    x[rng.random(n) < 0.1] = np.nan
    valid = rng.random(n) > 0.2
    assert rq.WaveletMatrix(np.arange(n)).L == max(1, (n - 1).bit_length())
    _wm_vs_oracle(x, valid, "float64", min(5, n), 1, center=n % 2 == 1)


def test_wavelet_matrix_all_null_and_one_value():
    _wm_vs_oracle(np.zeros(9), np.zeros(9, dtype=bool), "float64", 3, 0)
    _wm_vs_oracle(np.full(9, 2.5), np.ones(9, dtype=bool), "float64", 4, 1)
    _wm_vs_oracle(np.array([7.0]), np.array([True]), "float64", 1, 1)


def test_wavelet_matrix_int_and_float32():
    rng = np.random.default_rng(5)
    big = rng.integers(2 ** 62, 2 ** 63 - 1, 40, dtype=np.int64)
    _wm_vs_oracle(big, np.ones(40, dtype=bool), "int64", 6, 2)
    f = rng.normal(size=40).astype(np.float32)
    _wm_vs_oracle(f, rng.random(40) > 0.3, "float32", 7, 1, center=True)


@pytest.mark.parametrize("method", rq.METHODS)
def test_limits_equal_rolling_min_max(method):
    # q = 0 / 1 give rolling_min / rolling_max on NaN-free columns, as the reference's own limit tests check
    rng = np.random.default_rng(3)
    x = list(rng.normal(size=50))
    valid = list(rng.random(50) > 0.3)
    vals = [v if ok else None for v, ok in zip(x, valid)]
    for q, kind in ((0.0, "rolling_min"), (1.0, "rolling_max")):
        want = ro.rolling(kind, vals, "float64", 4, min_samples=1)
        got = rq.rolling_quantile(x, valid, "float64", q, method, 4, 1)
        assert [None if g is None else float(g) for g in got] == want


def test_binding_argument_errors():
    import polars_b200 as plb
    x = np.arange(5.0)
    bad = [
        ([(x, {"window_size": 2})], "needs a quantile"),
        ([(x, {"quantile": 0.5})], "needs a window_size"),
        ([(x, {"quantile": 1.5, "window_size": 2})], "quantile must be"),
        ([(x, {"quantile": float("nan"), "window_size": 2})], "quantile must be"),
        ([(x, {"quantile": True, "window_size": 2})], "quantile must be"),
        ([(x, {"quantile": 0.5, "window_size": 2, "interpolation": "cubic"})], "unknown interpolation"),
        ([(x, {"quantile": 0.5, "window_size": 0})], "at least 1"),
        ([(x, {"quantile": 0.5, "window_size": 2, "min_samples": 3})], "min_samples"),
        ([(x, {"quantile": 0.5, "window_size": 2.0})], "integer"),
        ([(x, {"quantile": 0.5, "window_size": 2, "ddof": 1})], "takes no option"),
        ([(None, {"quantile": 0.5, "window_size": 2})], "needs a value column"),
        ([(x, 0.5, 2)], "(column, options)"),
        ([], "at least one operation"),
    ]
    for ops, msg in bad:
        with pytest.raises(ValueError, match=msg.replace("(", r"\(").replace(")", r"\)")):
            plb.rolling_quantile(ops)
    t = np.arange(5, dtype=np.int64)
    for opts, msg in (({"quantile": 0.5, "window_size": "2i", "closed": "middle"}, "closed"),
                      ({"quantile": 0.5, "window_size": "2i", "min_samples": -1}, "min_samples"),
                      ({"quantile": 0.5, "window_size": "2s"}, "'i' units"),
                      ({"quantile": 0.5, "window_size": 2, "center": True}, "takes no option")):
        with pytest.raises(ValueError, match=msg):
            plb.rolling_quantile_by([(x, opts)], t)


@pytest.mark.parametrize("entry", ["rolling_quantile", "rolling_median", "rolling_quantile_by", "rolling_median_by"])
def test_plugin_symbols_and_schemas(entry):
    # Float32 stays Float32, every other numeric dtype gives Float64
    from test_over import ArrowSchema
    import polars_b200 as plb
    lib = plb.lib()
    assert hasattr(lib, f"_polars_plugin_bl_{entry}")
    fn = getattr(lib, f"_polars_plugin_field_bl_{entry}")
    for fmt_in, fmt_out in ((b"l", b"g"), (b"c", b"g"), (b"L", b"g"), (b"i", b"g"), (b"f", b"f"), (b"g", b"g")):
        fields = (ArrowSchema * 2)()
        fields[0].format, fields[0].name = fmt_in, b"x"
        fields[1].format, fields[1].name = b"l", b"t"
        out = ArrowSchema()
        fn(fields, C.c_size_t(2), C.byref(out), None, C.c_size_t(0))
        assert out.format == fmt_out, (fmt_in, out.format)
        C.CFUNCTYPE(None, C.POINTER(ArrowSchema))(out.release)(C.byref(out))
