"""CPU tests (-m "not gpu") of the per-group median / quantile: the plain-Python oracle against the reference's known
answers (tests/golden/quantile_kats.json) and against numpy, the C ABI / plugin symbols, and the Python kind parsing."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest

import quantile_oracle as qo
from test_cabi_cpu import declared_symbols

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NP = {"int8": np.int8, "int16": np.int16, "int32": np.int32, "int64": np.int64, "uint8": np.uint8, "uint16": np.uint16, "uint32": np.uint32,
      "uint64": np.uint64, "float32": np.float32, "float64": np.float64}


def quantile_kats():
    with open(os.path.join(ROOT, "tests", "golden", "quantile_kats.json")) as f:
        return json.load(f)["quantile"]


def kat_column(case):
    vals = case["values"]
    valid = np.array([v is not None for v in vals], bool)
    return np.array([0 if v is None else v for v in vals], dtype=NP[case["dtype"]]), (None if valid.all() else valid)


def kat_q_method(case):
    return (0.5, "linear") if case["kind"] == "median" else (case["q"], case["method"])


def check_kat_result(case, got, ok):
    exp_dt = np.float32 if case["dtype"] == "float32" else np.float64
    assert got.dtype == exp_dt, case["cite"]
    for g, v, e in zip(got.tolist(), ok.tolist(), case["expect"]):
        assert v == (e is not None), case["cite"]
        if e is None:
            continue
        if case.get("approx"):
            assert abs(g - e) < 1e-7, case["cite"]
        else:
            assert g == exp_dt(e), f"{case['cite']}: {g!r} != {e!r}"


@pytest.mark.parametrize("case", quantile_kats(), ids=lambda c: c["cite"][-70:])
def test_oracle_matches_reference_kats(case):
    vals, valid = kat_column(case)
    q, m = kat_q_method(case)
    got, ok = qo.group_quantile(case["keys"], vals, valid, q, m)
    check_kat_result(case, got, ok)


def test_rust_round_is_half_away_from_zero():
    assert [qo.rust_round(x) for x in (0.5, 1.5, 2.5, -0.5, -2.5, 0.49999999999999994, 2.4999999999999996)] == [1.0, 2.0, 3.0, -1.0, -3.0, 0.0, 2.0]
    assert round(2.5) == 2 and np.round(2.5) == 2.0      # why the oracle does not use them


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("method", ["lower", "higher", "midpoint", "linear", "nearest"])
def test_oracle_agrees_with_numpy(seed, method):
    rng = np.random.default_rng(seed)
    n_groups = 1 + seed * 3
    for _ in range(n_groups):
        size = int(rng.integers(1, 40))
        x = rng.normal(size=size) if seed % 2 else rng.integers(-50, 50, size).astype(np.float64)
        for q in (0.0, 0.1, 0.25, 0.5, 0.6, 0.9, 1.0):
            got, ok = qo.group_quantile([0] * size, x, None, q, method)
            fi = (size - 1) * q
            if method == "nearest" and abs(fi - math.floor(fi) - 0.5) < 1e-9:
                continue          # numpy's nearest rounds half to even
            exp = np.quantile(x, q, method=method)
            assert ok[0] and math.isclose(got[0], exp, rel_tol=1e-12, abs_tol=1e-12), (method, q, got[0], exp)


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("method", qo.METHODS)
def test_vectorised_restatement_agrees_with_oracle(seed, method):
    rng = np.random.default_rng(100 + seed)
    n = 600
    gid = rng.integers(0, 25, n)
    vals = rng.choice(np.array([0.0, -0.0, 1.5, -2.0, np.nan, np.inf, -np.inf, 3.0]), n)
    some = rng.random(n) < 0.4
    vals[some] = rng.normal(size=int(some.sum()))
    valid = rng.random(n) > 0.3
    valid[gid == 3] = False                      # one all-null group
    first = {}
    for g in gid.tolist():
        first.setdefault(g, len(first))
    dense = np.array([first[g] for g in gid.tolist()])
    for q in (0.0, 0.25, 0.5, 0.9, 1.0):
        a, av = qo.group_quantile(dense.tolist(), vals, valid, q, method)
        b, bv = qo.numpy_group_quantile(dense, vals, valid, q, method, len(first))
        assert np.array_equal(av, bv)
        assert np.array_equal(np.where(av, a, 0.0), np.where(bv, b, 0.0), equal_nan=True), (q, method)


def test_oracle_special_floats():
    x = np.array([np.inf, np.inf, -np.inf, np.inf, np.nan, 1.0, -0.0, 0.0])
    keys = [0, 0, 1, 1, 2, 2, 3, 3]
    got, ok = qo.group_quantile(keys, x, None, 0.5, "linear")
    assert got[0] == np.inf                      # lower == upper: inf, not inf - inf
    assert np.isnan(got[1])                      # -inf + 0.5 * (inf - -inf)
    assert np.isnan(got[2]) and got[3] == 0.0    # NaN is the greatest value; the midpoint of 1 and NaN is NaN
    got, _ = qo.group_quantile(keys, x, None, 0.0, "lower")
    assert got[2] == 1.0
    f32 = np.array([1.0, 2.0, 2.0000002], np.float32)
    got, _ = qo.group_quantile([0, 0, 0], f32, None, 0.75, "linear")
    assert got.dtype == np.float32 and got[0] == np.float32(0.5 * (np.float64(np.float32(2.0000002)) - 2.0) + 2.0)


def test_oracle_rejects_bad_quantile():
    with pytest.raises(ValueError):
        qo.group_quantile([0], np.array([1.0]), None, 1.5)
    with pytest.raises(ValueError):
        qo.group_quantile([0], np.array([1.0]), None, float("nan"))


def test_header_and_library_export_quantile():
    import polars_b200 as plb
    syms = declared_symbols()
    assert "bl_groupby_agg_params" in syms
    hdr = open(os.path.join(ROOT, "include", "polars_b200.h")).read()
    assert "BL_AGG_MEDIAN = 11" in hdr and "BL_AGG_QUANTILE = 12" in hdr
    for i, m in enumerate(qo.METHODS):
        assert f"BL_QUANTILE_{m.upper()} = {i}" in hdr
        assert plb.QUANTILE_METHODS[m] == i
    assert C.sizeof(plb.BlAggParam) == 16
    lib = plb.lib()
    for s in ("bl_groupby_agg_params", "_polars_plugin_bl_group_median", "_polars_plugin_field_bl_group_median",
              "_polars_plugin_bl_group_quantile", "_polars_plugin_field_bl_group_quantile"):
        assert hasattr(lib, s), s
    rs = open(os.path.join(ROOT, "integration", "polars_b200_sys.rs")).read()
    assert "pub struct BlAggParam { pub quantile: f64, pub method: i32, pub reserved: i32 }" in rs


@pytest.mark.parametrize("name", ["group_median", "group_quantile"])
@pytest.mark.parametrize("value_type,expect", [("int64", b"g"), ("int8", b"g"), ("uint32", b"g"), ("float64", b"g"), ("float32", b"f")])
def test_plugin_field_reports_float_output(name, value_type, expect):
    # the field function needs no device
    import polars_b200 as plb
    import pyarrow as pa
    from test_gpu_plugin_abi import ArrowSchema
    lib = plb.lib()
    fn = getattr(lib, f"_polars_plugin_field_bl_{name}")
    fn.restype = None
    fields = (ArrowSchema * 3)()
    pa.field("k", pa.int64())._export_to_c(C.addressof(fields[0]))
    pa.field("k2", pa.int32())._export_to_c(C.addressof(fields[1]))
    pa.field("v", getattr(pa, value_type)())._export_to_c(C.addressof(fields[2]))
    out = ArrowSchema()
    fn(fields, C.c_size_t(3), C.byref(out), None, C.c_size_t(0))
    assert out.format == b"+s" and out.n_children == 3
    kids = [out.children[i].contents for i in range(3)]
    assert [k.name for k in kids] == [b"key", b"key_1", b"agg"]
    assert [k.format for k in kids] == [b"l", b"i", expect]


def test_python_kind_parsing():
    import polars_b200 as plb
    assert plb.AGGS["median"] == 11 and plb._agg_kind("median") == 11
    assert plb._agg_kind("quantile:0.9") == 12 and plb._agg_kind("quantile:0.25:linear") == 12
    assert plb._agg_param("quantile:0.9") == (0.9, 0)                  # Polars' default method is nearest
    assert plb._agg_param("quantile:0.25:linear") == (0.25, 4)
    assert plb._agg_param("quantile:1:equiprobable") == (1.0, 5)
    assert plb._agg_param("median") is None and plb._agg_param("var:0") is None
    with pytest.raises(ValueError, match="unknown quantile method"):
        plb._agg_param("quantile:0.5:cubic")
    with pytest.raises(ValueError):
        plb._agg_param("quantile")
    assert plb._agg_kind("var:0") == 8 and plb._agg_kind("std") == 9 | (1 << 16)      # the other kinds are unchanged
