"""GPU tests of bl_arg_sort / bl_sort: the reference's known answers, bit-exact permutations against the oracle
(tests/sort_oracle.py) and numpy over every key dtype, direction and null placement, the radix-pass edge cases, limits,
payload gathers and the plugin entry."""
import ctypes as C

import numpy as np
import pytest

import sort_oracle
from test_sort import NP, expected_payload_ok, kat_columns, sort_kats

pytestmark = pytest.mark.gpu

DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64", "bool"]


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as plb
    plb.init()
    return plb


def cols_arg(cols, valids):
    return [(c, v) if v is not None else c for c, v in zip(cols, valids)]


def random_column(rng, dt, n, null_frac=0.15):
    if dt == "bool":
        c = rng.random(n) < 0.5
    elif dt.startswith("float"):
        c = rng.normal(size=n).astype(NP[dt])
        c[rng.random(n) < 0.05] = np.nan
        c[rng.random(n) < 0.05] = -0.0
        c[rng.random(n) < 0.05] = 0.0
        c[rng.random(n) < 0.02] = np.inf
        c[rng.random(n) < 0.02] = -np.inf
        if n:
            c[rng.random(n) < 0.2] = c[0]                                                    # ties
    else:
        info = np.iinfo(NP[dt])
        c = rng.integers(info.min, info.max, n, dtype=NP[dt], endpoint=True)
        c[rng.random(n) < 0.3] = c[0] if n else 0                                            # ties
    valid = rng.random(n) > null_frac if null_frac else None
    return c, valid


@pytest.mark.parametrize("case", sort_kats(), ids=lambda c: c["cite"][-60:])
def test_reference_kats(plb, case):
    cols, valids = kat_columns(case["by"], case["dtypes"])
    if "expect_error" in case:
        with pytest.raises(ValueError, match=case["expect_error"]):
            plb.arg_sort(cols_arg(cols, valids), case["descending"], case["nulls_last"], case.get("limit"))
        return
    idx = plb.arg_sort(cols_arg(cols, valids), case["descending"], case["nulls_last"], case.get("limit"))
    if "expect_idx" in case:
        assert idx.tolist() == case["expect_idx"]
    if "payload" in case:
        pcols, pvalids = kat_columns(case["payload"], case["payload_dtypes"])
        outs = plb.sort(cols_arg(cols, valids), cols_arg(pcols, pvalids), case["descending"], case["nulls_last"], case.get("limit"))
        for (v, m), exp in zip(outs, case["expect_payload"]):
            assert expected_payload_ok(v, m, exp), (v, m, exp)


@pytest.mark.parametrize("dt", DTYPES)
def test_every_dtype_direction_and_null_placement(plb, dt):
    rng = np.random.default_rng(DTYPES.index(dt))
    for n in (0, 1, 7, 4095, 4096, 4097, 100_003):
        c, valid = random_column(rng, dt, n)
        for nv in (None, valid):
            for desc in (False, True):
                for nl in (False, True):
                    got = plb.arg_sort([(c, nv) if nv is not None else c], desc, nl)
                    exp = sort_oracle.numpy_arg_sort([c], [nv], desc, nl) if n > 5000 else sort_oracle.arg_sort([c], [nv], desc, nl)
                    assert np.array_equal(got, exp), (dt, n, nv is not None, desc, nl)


def test_special_columns(plb):
    n = 5000
    rng = np.random.default_rng(7)
    cases = [(np.zeros(n), np.zeros(n, bool)),                                  # all null
             (np.full(n, np.nan), None), (np.full(n, np.nan, np.float32), rng.random(n) < 0.5),   # all NaN
             (np.full(n, 42, np.int64), None), (np.full(n, -3, np.int8), rng.random(n) < 0.5),    # constant
             (np.arange(n, dtype=np.int64), None), (np.arange(n, dtype=np.float64)[::-1].copy(), None)]   # already sorted / reversed
    for c, v in cases:
        for desc in (False, True):
            for nl in (False, True):
                got = plb.arg_sort([(c, v) if v is not None else c], desc, nl)
                assert np.array_equal(got, sort_oracle.numpy_arg_sort([c], [v], desc, nl)), (c.dtype, v is not None, desc, nl)


def test_varying_bits_cross_digit_boundaries(plb):
    """keys whose varying bits sit in one digit, straddle the boundary to the next, then the one after; skipped digits
    in the middle (bits 0-3 and 40-47 vary, 8-39 constant); and negative values (sign-bit digit varies)"""
    rng = np.random.default_rng(11)
    n = 50_000
    base = np.int64(0x1234_5678_9A00)
    for span in (8, 9, 16, 17, 24, 25, 40, 63):
        c = base + rng.integers(0, 1 << span, n, dtype=np.int64) if span < 63 else rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
        for desc in (False, True):
            assert np.array_equal(plb.arg_sort([c], desc), sort_oracle.numpy_arg_sort([c], None, desc)), span
        u = (c & 0xFFFFFFFF).astype(np.uint32)
        assert np.array_equal(plb.arg_sort([u]), sort_oracle.numpy_arg_sort([u])), span
    gaps = (rng.integers(0, 16, n, dtype=np.int64) | (rng.integers(0, 256, n, dtype=np.int64) << 40)) + (np.int64(0x55) << 16)
    assert np.array_equal(plb.arg_sort([gaps]), sort_oracle.numpy_arg_sort([gaps]))
    neg = rng.integers(-300, 300, n).astype(np.int16)
    assert np.array_equal(plb.arg_sort([neg], True, True), sort_oracle.numpy_arg_sort([neg], None, True, True))


@pytest.mark.parametrize("k", [2, 3])
def test_several_key_columns_mixed_flags(plb, k):
    rng = np.random.default_rng(20 + k)
    for n in (7, 4097, 100_003):
        for trial in range(4):
            dts = [DTYPES[i] for i in rng.integers(0, len(DTYPES), k)]
            cols, valids = zip(*[random_column(rng, dt, n, 0.1 * (trial % 3)) for dt in dts])
            for i, dt in enumerate(dts):          # few distinct values so later columns break ties
                if dt != "bool":
                    cols[i][:] = cols[i][rng.integers(0, min(n, 5), n)]
            desc = [bool(x) for x in rng.random(k) < 0.5]
            nl = [bool(x) for x in rng.random(k) < 0.5]
            got = plb.arg_sort(cols_arg(cols, valids), desc, nl)
            exp = sort_oracle.arg_sort(cols, list(valids), desc, nl) if n < 5000 else sort_oracle.numpy_arg_sort(cols, list(valids), desc, nl)
            assert np.array_equal(got, exp), (dts, desc, nl, n)


def test_limits(plb):
    rng = np.random.default_rng(3)
    n = 10_000
    a, av = rng.integers(0, 50, n).astype(np.int32), rng.random(n) > 0.1
    b = rng.normal(size=n)
    full = sort_oracle.numpy_arg_sort([a, b], [av, None], [True, False], True)
    for limit in (0, 1, 333, n, n + 10):
        got = plb.arg_sort([(a, av), b], [True, False], True, limit=limit)
        assert np.array_equal(got, full[:limit]), limit
        outs = plb.sort([(a, av), b], [b, (a.astype(np.int64), av)], [True, False], True, limit=limit)
        assert np.array_equal(outs[0][0], b[full[:limit]])


def test_sort_payload_columns_with_validity(plb):
    rng = np.random.default_rng(5)
    n = 100_003
    key, kv = rng.integers(0, 1000, n).astype(np.int64), rng.random(n) > 0.05
    p1, p1v = rng.normal(size=n), rng.random(n) > 0.3
    p2 = rng.integers(-5, 5, n).astype(np.int32)
    p3 = rng.integers(0, 10, n).astype(np.uint64)
    perm = sort_oracle.numpy_arg_sort([key], [kv], True, False)
    outs = plb.sort([(key, kv)], [(p1, p1v), p2, p3, (key, kv)], descending=True)
    (g1, m1), (g2, m2), (g3, m3), (g4, m4) = outs
    assert np.array_equal(g1[m1], p1[perm][p1v[perm]]) and np.array_equal(m1, p1v[perm])
    assert np.array_equal(g2, p2[perm]) and m2 is None
    assert np.array_equal(g3, p3[perm]) and m3 is None
    assert np.array_equal(m4, kv[perm]) and np.array_equal(g4[m4], key[perm][kv[perm]])
    # device-resident inputs and outputs
    dk = plb.to_device(key, kv)
    dp = plb.to_device(p2)
    [o] = plb.sort([dk], [dp], descending=True, location=plb.DEVICE)
    assert np.array_equal(o.to_numpy()[0], p2[perm])
    idx = plb.arg_sort([dk], descending=True, location=plb.DEVICE)
    assert idx.length == n and np.array_equal(idx.to_numpy()[0], perm)


def test_errors(plb):
    with pytest.raises(plb.B200Error) as e:
        plb.arg_sort([np.arange(5), np.arange(4)])
    assert e.value.status == 1
    with pytest.raises(plb.B200Error) as e:
        plb.sort([np.arange(5)], [np.arange(5, dtype=np.int16)])
    assert e.value.status == 4
    with pytest.raises(plb.B200Error) as e:
        plb.sort([np.arange(5)], [np.arange(4)])
    assert e.value.status == 1
    lib = plb.lib()
    out = plb.BlColumn()
    assert lib.bl_arg_sort(None, C.c_int32(0), None, C.c_int64(-1), C.c_int32(plb.HOST), C.byref(out)) == 1


@pytest.mark.parametrize("dt", ["int64", "uint32"])
def test_large_against_numpy(plb, dt):
    """2e7 rows: one u64-key and one u32-key sort against numpy's stable argsort"""
    rng = np.random.default_rng(99)
    n = 20_000_000
    c = rng.integers(0, np.iinfo(NP[dt]).max, n, dtype=NP[dt])
    c[::7] = c[3]
    dc = plb.to_device(c)
    got = plb.arg_sort([dc], location=plb.DEVICE).to_numpy()[0]
    assert np.array_equal(got, np.argsort(c, kind="stable").astype(np.uint32))


def test_plugin_arg_sort(plb):
    import pyarrow as pa
    from test_gpu_plugin_abi import Caller
    caller = Caller(plb.lib())
    a = pa.array([3, None, 1, 3, 2, None], pa.int64())
    b = pa.array([1.0, 2.0, float("nan"), 0.5, 2.0, 1.0])
    out = caller.call("arg_sort", [("a", [a.slice(0, 2), a.slice(2)]), ("b", [b])])
    assert out.type == pa.uint32() and out.to_pylist() == [5, 1, 2, 4, 3, 0]          # nulls tie: column b breaks it
    out = caller.call("arg_sort", [("a", [a]), ("b", [b])], kwargs={"descending": True, "nulls_last": True})
    assert out.to_pylist() == [0, 3, 4, 2, 1, 5]
    # int bitmask: column 1 descending only; column 0 nulls last
    out = caller.call("arg_sort", [("a", [a]), ("b", [b])], kwargs={"descending": 2, "nulls_last": 1})
    assert out.to_pylist() == [2, 4, 0, 3, 1, 5]
    exp = sort_oracle.arg_sort([np.array([3, 0, 1, 3, 2, 0]), np.asarray(b)], [np.array([1, 0, 1, 1, 1, 0], bool), None], [False, True], [True, False])
    assert exp.tolist() == [2, 4, 0, 3, 1, 5]


def test_null_rows_do_not_add_passes(plb):
    """the AND/OR digit test looks at valid rows only: nullable Int64 in [0, 1e6) takes the same 3 value passes as without
    nulls, plus the 1-bit null-rank pass; an all-null column needs no value pass"""
    rng = np.random.default_rng(8)
    n = 200_000
    c, v = rng.integers(0, 1_000_000, n).astype(np.int64), rng.random(n) > 0.1

    def passes(cols, desc=False, nl=False):
        plb.profile_reset()
        plb.profile_enable(True)
        try:
            got = plb.arg_sort(cols, desc, nl)
            plb.sync()
            return got, int(plb.profile().get("sort_scatter", {}).get("launches", 0))
        finally:
            plb.profile_enable(False)
    for desc in (False, True):
        for nl in (False, True):
            got, p = passes([(c, v)], desc, nl)
            assert np.array_equal(got, sort_oracle.numpy_arg_sort([c], [v], desc, nl))
            assert p == 4, (desc, nl, p)
    got, p = passes([c])
    assert p == 3 and np.array_equal(got, np.argsort(c, kind="stable"))
    z = np.full(n, 7, np.int64)
    got, p = passes([(z, np.zeros(n, bool))])
    assert p == 0 and np.array_equal(got, np.arange(n))


class _FakeSeries:
    """the slice of pl.Series that polars_b200.engine's Sort UDF touches, over numpy"""
    _DT = {np.dtype("int64"): "Int64", np.dtype("float64"): "Float64", np.dtype("int32"): "Int32", np.dtype("int8"): "Int8",
           np.dtype("bool"): "Boolean", np.dtype("object"): "String"}

    def __init__(self, name, values=None, valid=None):
        if values is None:
            name, values = "", name
        self.name, self.values = name, np.asarray(values)
        self.valid = None if valid is None else np.asarray(valid, bool)

    @property
    def dtype(self):
        return self._DT[self.values.dtype]

    def null_count(self):
        return 0 if self.valid is None else int((~self.valid).sum())

    def is_null(self):
        return _FakeSeries(self.name, np.zeros(len(self.values), bool) if self.valid is None else ~self.valid)

    def fill_null(self, v):
        vals = self.values.copy()
        if self.valid is not None:
            vals[~self.valid] = v
        return _FakeSeries(self.name, vals)

    def to_numpy(self):
        return self.values

    def set(self, mask, value):
        assert value is None
        return _FakeSeries(self.name, self.values, ~np.asarray(mask.values, bool))


class _FakeFrame:
    def __init__(self, series):
        self.cols = {s.name: s for s in series}

    @property
    def columns(self):
        return list(self.cols)

    @property
    def schema(self):
        return {c: s.dtype for c, s in self.cols.items()}

    def rechunk(self):
        return self

    def get_column(self, c):
        return self.cols[c]

    def select(self, names):
        return _FakeFrame([self.cols[c] for c in names])

    def __getitem__(self, idx):
        i = np.asarray(idx.values, np.int64)
        return _FakeFrame([_FakeSeries(s.name, s.values[i], None if s.valid is None else s.valid[i]) for s in self.cols.values()])


def test_engine_sort_udf_on_the_device(plb, monkeypatch):
    """the B2 Sort UDF end to end with a numpy stand-in for the few polars calls it makes (no Polars wheel here): numeric
    columns come back through K4, String / Boolean / Int8 columns through the stand-in's take of the same permutation"""
    import sys
    import types
    from polars_b200 import engine
    from test_sort import SchemaTraverser, expr_ir, make
    fake = types.ModuleType("polars")
    fake.Series = _FakeSeries
    fake.DataFrame = lambda series: _FakeFrame(series)
    monkeypatch.setitem(sys.modules, "polars", fake)
    rng = np.random.default_rng(9)
    n = 3000
    g = rng.integers(-2, 3, n).astype(np.int8)
    a, av = rng.integers(0, 40, n).astype(np.int64), rng.random(n) > 0.2
    b, bv = rng.normal(size=n), rng.random(n) > 0.3
    f = rng.random(n) < 0.5
    s = np.array([f"s{i % 17}" for i in range(n)], dtype=object)
    frame = _FakeFrame([_FakeSeries("g", g), _FakeSeries("a", a, av), _FakeSeries("b", b, bv), _FakeSeries("f", f), _FakeSeries("s", s)])
    exprs = {0: make("Column", name="g"), 1: make("Column", name="a")}
    nodes = {40: make("DataFrameScan", df=frame, projection=None, selection=None),
             41: make("Sort", input=40, by_column=[expr_ir(0, "g"), expr_ir(1, "a")], sort_options=(True, [False, True], [True, False]), slice=(0, 2500, None))}
    nt = SchemaTraverser(nodes, exprs, 41, frame.schema)
    engine.execute_with_b200(nt, raise_on_fail=True)
    out = nt.udf()
    perm = sort_oracle.numpy_arg_sort([g, a], [None, av], [True, False], [False, True], 2500)
    assert out.columns == ["g", "a", "b", "f", "s"]
    assert np.array_equal(out.get_column("g").values, g[perm])
    oa = out.get_column("a")
    assert np.array_equal(oa.valid, av[perm]) and np.array_equal(oa.values[oa.valid], a[perm][av[perm]])
    ob = out.get_column("b")
    assert np.array_equal(ob.valid, bv[perm]) and np.array_equal(ob.values[ob.valid], b[perm][bv[perm]])
    assert np.array_equal(out.get_column("f").values, f[perm]) and np.array_equal(out.get_column("s").values, s[perm])
