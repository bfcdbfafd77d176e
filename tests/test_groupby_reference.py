"""CPU checks of tests/groupby_ref.py, the exact restatement of the fused group_by aggregations, against the C oracle on
the same full-range inputs, and a self-test showing its float bound catches one lost, doubled or f32-rounded summand in
a group of 2^20 rows."""
import math

import numpy as np
import pytest

import groupby_ref as ref

KEY_DTYPES = ("int64", "uint64", "int32", "uint32", "float64", "float32", "int16", "uint8")


@pytest.fixture(scope="module")
def oracle():
    import oracle as o
    return o


def _case(seed, key_dtype, nullable):
    rng = np.random.default_rng(seed)
    narrow = np.dtype(key_dtype).itemsize == 1          # 256 keys: fewer groups
    case = ref.Case(rng, key_dtype, big=3000, singletons=60 if narrow else 200, groups=100 if narrow else 150, rest=6000,
                    null_rows=40 if nullable else 0)
    cols = []
    for dt in ref.VALUE_DTYPES + ref.SMALL_DTYPES:
        s = case.values(rng, dt, for_sum=True, nullable=nullable)
        mm = s if np.dtype(dt).kind != "f" else case.values(rng, dt, nullable=nullable)
        if np.dtype(dt).kind == "f":
            mm = (_quiet(mm[0]), mm[1])
        cols.append((dt, s, mm))
    return case, cols


def _quiet(x):
    """Signalling NaNs made quiet.  The oracle's fmin / fmax (glibc) return NaN for a signalling NaN operand, so the fold
    restarts after one; the reference's f64::min / f32::min ignore every NaN, as the device and groupby_ref do."""
    u = np.uint64 if x.dtype == np.float64 else np.uint32
    q = u(1 << 51) if x.dtype == np.float64 else u(1 << 22)
    b = x.view(u).copy()
    nan = np.isnan(x)
    b[nan] |= q
    return b.view(x.dtype)


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("key_dtype", KEY_DTYPES)
def test_restatement_matches_oracle(oracle, key_dtype, nullable):
    case, cols = _case(len(key_dtype) * 7 + nullable, key_dtype, nullable)
    for maintain_order in (True, False):
        for dt, s, mm in cols:
            aggs = [("sum", *s), ("mean", *s), ("min", *mm), ("max", *mm), ("count", *mm), ("len", None, None)]
            (k, kv), exps, g = ref.expect(case.keys, case.key_valid, aggs, maintain_order)
            ok_, okv, oouts, _ = oracle.group_by_agg(case.keys, case.key_valid, aggs, 4, maintain_order)
            if not maintain_order:
                o = ref.canonical_order(ok_, okv)
                ok_, okv = ok_[o], (None if okv is None else okv[o])
                oouts = [(v[o], None if m is None else m[o]) for v, m in oouts]
            err = ref.check(ok_, okv, (k, kv))
            assert err is None, (dt, maintain_order, "keys", err)
            for (kind, _, _), exp, (ov, om) in zip(aggs, exps, oouts):
                if kind == "sum" and np.dtype(dt) == np.float32:
                    exp = ref.kahan32(exp)     # the oracle sums Float32 in f32 (oracle.c kahanf_add)
                err = ref.check(ov, om, exp)
                assert err is None, (key_dtype, dt, kind, maintain_order, err)


def test_dedicated_groups_are_present():
    rng = np.random.default_rng(3)
    case = ref.Case(rng, "float64", big=100, singletons=5, groups=10, rest=100, null_rows=3)
    v, m = case.values(rng, "float64", for_sum=True, nullable=True)
    g = ref.group(case.keys, case.key_valid, True)
    for name, rows in case.special_rows.items():
        assert rows.size == ref.SPECIAL_ROWS[name]
        assert np.unique(g.gid[rows]).size == 1, name          # every dedicated group is one group of its own
        assert np.sum(g.gid == g.gid[rows[0]]) == rows.size, name
    (k, kv), (s, mean, mn), _ = ref.expect(case.keys, case.key_valid, [("sum", v, m), ("mean", v, m), ("min", v, m)], True)
    gid = {n: int(g.gid[r[0]]) for n, r in case.special_rows.items()}
    assert np.isnan(s.e[gid["all_nan"]]) and np.isnan(s.e[gid["inf_pair"]]) and np.isnan(mn[0][gid["all_nan"]])
    assert not mean.valid[gid["all_null"]] and s.e[gid["all_null"]] == 0 and not mn[1][gid["all_null"]]
    assert s.e[gid["subnormal"]] != 0 and s.tol[gid["subnormal"]] == 0      # exact: a flush to zero is visible
    assert kv is not None and not kv.all()                                   # the null key group


def test_float_bound_self_test(oracle):
    """One group of 2^20 rows: the exact result and the oracle's Kahan sum pass; dropping one row, doubling one row and
    rounding every summand through f32 each fail.

    Exact-summable values (the GPU tests' large float cases) have a bound of 0, so every perturbation fails.  Values with
    full 53-bit mantissas, uniform in [0, 100), have the bound (m + 1) 2^-53 S, about 2^-33 S here: a lost or doubled
    row (about 2^-20 S) is 8000 times larger.  Rounding each of them through f32 is not: the errors are unbiased and
    add up to about 2^-36 S, inside the bound of any f64 summation order.  That perturbation is shown on a group of 64
    rows instead, where it is 2^15 times the bound."""
    rng = np.random.default_rng(11)
    n = 1 << 20
    key = np.zeros(n, np.int64)
    g = ref.group(key)
    for exact in (True, False):
        x = ref.sum_column(rng, "float64", n, exact=True) if exact else rng.uniform(0, 100, n)
        exp = ref.aggregate("sum", x, None, g)
        assert (exp.tol == 0).all() == exact

        def fails(got):
            return ref.check(np.array([got]), None, exp) is not None

        assert not fails(exp.e[0])
        _, _, oouts, _ = oracle.group_by_agg(key, None, [("sum", x, None)], 4, True)
        assert not fails(oouts[0][0][0]), "the oracle's Kahan sum must pass"
        i = int(np.argsort(np.abs(x))[n // 2])      # a row of typical size
        assert fails(exp.e[0] - x[i]), "dropping one row must fail"
        assert fails(exp.e[0] + x[i]), "doubling one row must fail"
        if exact:
            f32 = np.sum(x.astype(np.float32).astype(np.float64))       # exact-summable: numpy's order is as good as any
            assert fails(f32), "rounding every summand through f32 must fail"
    small = ref.group(np.zeros(64, np.int64))
    x = rng.uniform(0, 100, 64)
    exp = ref.aggregate("sum", x, None, small)
    assert ref.check(np.array([math.fsum(x.tolist())]), None, exp) is None
    assert ref.check(np.array([math.fsum(x.astype(np.float32).astype(np.float64).tolist())]), None, exp) is not None
    # mean: the same perturbations divided by the count
    x = ref.sum_column(rng, "float64", n, exact=True)
    exp = ref.aggregate("mean", x, None, g)
    s = float(np.sum(x))
    i = n // 3
    assert ref.check(np.array([s / n]), None, exp) is None
    assert ref.check(np.array([(s - x[i]) / n]), None, exp) is not None


def test_float32_output_rules():
    """Float32 sum: the f64 sum rounded once; a value one f32 ulp away fails when the group is exact-summable."""
    rng = np.random.default_rng(5)
    g = ref.group(np.zeros(1000, np.int64))
    x = ref.sum_column(rng, "float32", 1000, exact=True)
    exp = ref.aggregate("sum", x, None, g)
    assert exp.dtype == np.float32 and exp.tol[0] == 0
    good = np.array([np.float32(np.sum(x.astype(np.float64)))])
    assert ref.check(good, None, exp) is None
    assert ref.check(np.nextafter(good, np.float32(np.inf)), None, exp) is not None


def test_integer_sum_wraps():
    g = ref.group(np.zeros(4, np.int64))
    for dt, want in (("int64", -2), ("uint64", (1 << 64) - 2), ("int32", -2), ("uint32", (1 << 32) - 2), ("int8", 2 * 127 + 2 * -128), ("uint16", 4 * 65535)):
        info = np.iinfo(dt)
        x = np.array([info.max, info.max, info.min, info.min] if dt in ("int8",) else [info.max] * 4 if dt == "uint16" else [info.max, info.max, 0, 0], dt)
        v, _ = ref.aggregate("sum", x, None, g)
        assert v.dtype == ref.sum_out_dtype(dt)
        assert int(v[0]) == want, (dt, v)
