"""CPU checks of tests/primitives_ref.py: the numpy restatements of K1-K4 agree with the C oracle, and the vectorised
integer rules agree with exact Python-int arithmetic, on the extreme-value inputs the GPU tests use.  A disagreement
here is a bug in one of the two statements, found before any GPU time is spent."""
import numpy as np
import pytest

import oracle
import primitives_ref as ref


def _check(what, got, got_valid, exp, exp_valid):
    err = ref.valid_equal(got, got_valid, exp, exp_valid)
    assert err is None, f"{what}: {err}"


@pytest.mark.parametrize("dtype", ref.DTYPES)
def test_arith_matches_oracle(dtype):
    rng = np.random.default_rng(11)
    n = 3001
    a, b = ref.column(rng, dtype, n), ref.column(rng, dtype, n, divisor=True)
    av, bv = ref.validity(rng, n), ref.validity(rng, n)
    for op in ref.OPS:
        for lv, rv in ((av, bv), (None, None)):
            _check((op, "aa"), *ref.arith(op, a, b, lv, rv), *oracle.arith(op, a, b, lv, rv))
            for s in ref.scalars(dtype):
                _check((op, "as", s), *ref.arith(op, a, s, lv, None), *oracle.arith(op, a, s, lv, None))
                _check((op, "sa", s), *ref.arith(op, s, b, None, rv), *oracle.arith(op, s, b, None, rv))


@pytest.mark.parametrize("dtype", ref.INT_DTYPES)
def test_int_vectorised_matches_python_ints(dtype):
    # every pair of specials (min, max, 0, ±1, ...) through the vectorised rule and through exact Python ints
    sp = ref.int_specials(dtype)
    a, b = np.repeat(sp, sp.size), np.tile(sp, sp.size)
    for op in ref.OPS:
        got, gv = ref.arith(op, a, b)
        gv = np.ones(a.size, bool) if gv is None else gv
        for i in range(a.size):
            e, ev = ref.int_exact(op, int(a[i]), int(b[i]), dtype)
            assert gv[i] == ev, (op, a[i], b[i])
            if ev:
                if op == "truediv":
                    assert (got[i] == e) or (np.isnan(got[i]) and e != e), (op, a[i], b[i], got[i], e)
                else:
                    assert int(got[i]) == e, (op, a[i], b[i], got[i], e)
    info = np.iinfo(np.dtype(dtype))
    if info.min < 0:
        q, _ = ref.arith("floordiv", np.array([info.min], dtype), np.array([-1], dtype))
        r, _ = ref.arith("mod", np.array([info.min], dtype), np.array([-1], dtype))
        assert q[0] == info.min and r[0] == 0
    q, qv = ref.arith("floordiv", np.array([5, 6], dtype), np.dtype(dtype).type(0))
    assert qv is not None and not qv.any(), "a scalar divisor of 0 makes every row null"
    t, tv = ref.arith("truediv", np.array([5, 0], dtype), np.array([0, 0], dtype))
    assert tv is None and np.isinf(t[0]) and np.isnan(t[1]), "integer true division by 0 is IEEE, never null"


@pytest.mark.parametrize("dtype", ref.DTYPES)
def test_compare_matches_oracle(dtype):
    rng = np.random.default_rng(12)
    n = 3001
    a, b = ref.column(rng, dtype, n), ref.column(rng, dtype, n)
    eq = rng.random(n) < 1 / 3
    b[eq] = a[eq]
    av, bv = ref.validity(rng, n), ref.validity(rng, n)
    for op in ref.CMPS:
        for lv, rv in ((av, bv), (None, bv), (None, None)):
            _check((op, "aa"), *ref.compare(op, a, b, lv, rv), *oracle.compare(op, a, b, lv, rv))
            if op in ("eq", "ne"):
                _check((op, "missing"), *ref.compare(op, a, b, lv, rv, missing=True), *oracle.compare(op, a, b, lv, rv, missing=True))
        for s in ref.scalars(dtype):
            a2 = a.copy()
            a2[::3] = s
            _check((op, "scalar", s), *ref.compare(op, a2, s, av), *oracle.compare(op, a2, s, av))
            if op in ("eq", "ne"):
                _check((op, "scalar missing", s), *ref.compare(op, a2, s, av, missing=True), *oracle.compare(op, a2, s, av, missing=True))


def test_float_total_order_specials():
    for dt in ref.FLOAT_DTYPES:
        nan, z, nz, inf = (np.dtype(dt).type(v) for v in (np.nan, 0.0, -0.0, np.inf))
        a = np.array([nan, nan, z, nz, inf], dt)
        b = np.array([nan, inf, nz, z, nan], dt)
        assert ref.compare("eq", a, b)[0].tolist() == [True, False, True, True, False]
        assert ref.compare("gt", a, b)[0].tolist() == [False, True, False, False, False]
        assert ref.compare("lt", a, b)[0].tolist() == [False, False, False, False, True]


@pytest.mark.parametrize("dtype", ref.DTYPES)
def test_filter_matches_oracle(dtype):
    rng = np.random.default_rng(13)
    for n in (0, 1, 33, 4097):
        v = ref.column(rng, dtype, n)
        valid, mask, mvalid = ref.validity(rng, n), rng.random(n) < 0.5, ref.validity(rng, n)
        for vv, mv in ((valid, mvalid), (None, None), (valid, None)):
            _check(("filter", n), *ref.filter(v, vv, mask, mv), *oracle.filter(v, vv, mask, mv))


@pytest.mark.parametrize("dtype", ref.DTYPES)
def test_gather_matches_oracle(dtype):
    rng = np.random.default_rng(14)
    n, m = 1000, 4097
    v = ref.column(rng, dtype, n)
    valid = ref.validity(rng, n)
    idx = rng.integers(0, n, m).astype(np.uint32)
    ivalid = ref.validity(rng, m)
    for vv in (valid, None):
        _check("bitmap", *ref.gather(v, vv, idx, ivalid), *oracle.gather(v, vv, idx, ivalid))
        # the oracle has no sentinel: the same nulls as a bitmap over an in-range index
        sent = idx.copy()
        sent[~ivalid] = ref.IDX_NULL
        e, ev = oracle.gather(v, vv, np.where(ivalid, idx, 0).astype(np.uint32), ivalid)
        _check("sentinel", *ref.gather(v, vv, sent), e, ev)
    g, gv = ref.gather(v, None, idx)
    assert gv is None and np.array_equal(g.view(np.uint8), v[idx].view(np.uint8))


def test_partition_of_reproduces_reference_kat(kats):
    vecs = kats["hash"][0]["vectors"]
    keys = np.array([int(x["key_u64"]) for x in vecs], np.uint64)
    for p in (1, 2, 3, 7, 8, 16):
        parts = ref.partition_of(keys, None, p)
        assert parts.tolist() == [x["part"][str(p)] for x in vecs], p
        offs = ref.partition_offsets(parts, p)
        assert offs[0] == 0 and offs[-1] == keys.size and np.all(np.diff(offs) >= 0)
    valid = np.arange(keys.size) % 3 != 0
    assert (ref.partition_of(keys, valid, 17)[~valid] == 0).all(), "a null key goes to partition 0"


def test_partition_canonicalises_float_keys():
    for dt in ref.FLOAT_DTYPES:
        sp = ref.float_specials(dt)
        parts = ref.partition_of(sp, None, 64)
        nan = np.isnan(sp)
        assert len(set(parts[nan].tolist())) == 1, "every NaN bit pattern hashes alike"
        assert parts[0] == parts[1], "-0.0 and 0.0 hash alike"
