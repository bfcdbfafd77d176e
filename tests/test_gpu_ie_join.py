"""GPU tests of the inequality join (bl_ie_join): every result is compared with the brute-force rule (tests/ie_join_oracle.py,
or its numpy form below for larger inputs) as an exact multiset of (left row, right row | null) pairs, and every result is
checked for left rows ascending.  Covered: the reference's known answers, every dtype for both predicates (mixed and
8/16-bit), every operator and operator pair for inner and left joins, nulls, NaN, +-0, +-inf and integer extremes, one huge
tie run, empty and all-null sides, right sizes around powers of two, a skewed output, the right flip and payload gathers,
device inputs and outputs, repeatability, the error cases, and point-in-interval / single-predicate joins at scale."""
import itertools
import json
import os

import numpy as np
import pytest

import ie_join_oracle as io

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NULL = 0xFFFFFFFF
OPS = io.OPS
NUMERIC = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as plb
    plb.init()
    return plb


def np_key(a):
    """uint64 keys whose order is the total order of the values (NaN greatest, -0.0 == +0.0)"""
    a = np.asarray(a)
    if a.dtype.kind == "f":
        v = a.astype(np.float64) + 0.0
        v = np.where(np.isnan(v), np.nan, v)
        u = v.view(np.uint64)
        return np.where(u >> np.uint64(63), ~u, u | np.uint64(1 << 63))
    if a.dtype.kind == "i":
        return a.astype(np.int64).view(np.uint64) ^ np.uint64(1 << 63)
    return a.astype(np.uint64)


def np_expect(left, right, ops, how):
    """brute force on numpy columns (values, valid|None): sorted pair codes li * (nr + 1) + (ri | nr)"""
    nl, nr = len(left[0][0]), len(right[0][0])
    mask = np.ones((nl, nr), bool)
    for (lv, lm), (rv, rm), op in zip(left, right, ops):
        a, b = np_key(lv)[:, None], np_key(rv)[None, :]
        mask &= {"<": a < b, "<=": a <= b, ">": a > b, ">=": a >= b}[op]
        if lm is not None:
            mask &= lm[:, None]
        if rm is not None:
            mask &= rm[None, :]
    li, ri = np.nonzero(mask)
    codes = li.astype(np.int64) * (nr + 1) + ri
    if how == "left":
        un = np.nonzero(~mask.any(axis=1))[0]
        codes = np.concatenate([codes, un.astype(np.int64) * (nr + 1) + nr])
    return np.sort(codes)


def got_codes(res, nr):
    (li, lv), (ri, rv) = res
    assert li.dtype == np.uint32 and ri.dtype == np.uint32 and lv is None
    assert np.all(np.diff(li.astype(np.int64)) >= 0), "left rows must come ascending"
    r = ri.astype(np.int64)
    if rv is not None:
        assert np.all(ri[~rv] == NULL), "a null slot must hold BL_IDX_NULL"
        r = np.where(rv, r, nr)
    return np.sort(li.astype(np.int64) * (nr + 1) + r)


def run(plb, left, right, ops, how="inner"):
    return plb.ie_join([plb.Column(v, m) for v, m in left], [plb.Column(v, m) for v, m in right], list(ops), how)


def check(plb, left, right, ops, how="inner"):
    res = run(plb, left, right, ops, how)
    got = got_codes(res, len(right[0][0]))
    exp = np_expect(left, right, ops, how)
    assert np.array_equal(got, exp), f"{ops} {how}: {len(got)} pairs, expected {len(exp)}"
    return res


def col(values, dtype):
    valid = np.array([v is not None for v in values], bool)
    vals = np.array([0 if v is None else v for v in values], dtype=dtype)
    return vals, (None if valid.all() else valid)


def rand_col(rng, n, dtype, null_frac=0.0, span=None):
    dt = np.dtype(dtype)
    if dt.kind == "f":
        v = (rng.integers(-(span or 20), span or 20, n) / 2).astype(dt)
    else:
        info = np.iinfo(dt)
        lo, hi = (max(info.min, -(span or 20)), min(info.max, span or 20)) if span is not False else (info.min, info.max)
        v = rng.integers(lo, hi, n, dtype=np.int64 if dt.kind == "i" or dt.itemsize < 8 else np.uint64, endpoint=True).astype(dt)
    m = rng.random(n) >= null_frac if null_frac else None
    return v, m


# ---------------------------------------------------------------------------- known answers
def kats():
    with open(os.path.join(ROOT, "tests", "golden", "ie_join_kats.json")) as f:
        return json.load(f)["ie_join"]


@pytest.mark.parametrize("k", kats(), ids=lambda k: k["cite"].split("(")[-1].rstrip(")"))
def test_known_answers(plb, k):
    left = [col(c, d) for c, d in zip(k["left"], k["dtypes"])]
    right = [col(c, d) for c, d in zip(k["right"], k["dtypes"])]
    (li, lv), (ri, rv) = run(plb, left, right, k["ops"], k["how"])
    lv = np.ones(len(li), bool) if lv is None else lv
    rv = np.ones(len(ri), bool) if rv is None else rv
    got = io.as_multiset([(int(a) if va else None, int(b) if vb else None) for a, va, b, vb in zip(li, lv, ri, rv)])
    assert got == io.as_multiset([tuple(p) for p in k["expect"]])


# ---------------------------------------------------------------------------- operators, dtypes, special values
@pytest.mark.parametrize("how", ["inner", "left"])
@pytest.mark.parametrize("op", OPS)
def test_single_operator(plb, op, how):
    rng = np.random.default_rng(1)
    for dt in ("int32", "float64"):
        check(plb, [rand_col(rng, 300, dt, 0.1)], [rand_col(rng, 200, dt, 0.1)], [op], how)


@pytest.mark.parametrize("how", ["inner", "left"])
@pytest.mark.parametrize("op1,op2", list(itertools.product(OPS, OPS)))
def test_operator_pairs(plb, op1, op2, how):
    rng = np.random.default_rng(2)
    for n_l, n_r in ((200, 150), (37, 300)):
        check(plb, [rand_col(rng, n_l, "int64", 0.1), rand_col(rng, n_l, "float32", 0.1)],
              [rand_col(rng, n_r, "int64", 0.1), rand_col(rng, n_r, "float32", 0.1)], [op1, op2], how)


@pytest.mark.parametrize("dx", NUMERIC)
def test_dtypes(plb, dx):
    rng = np.random.default_rng(3)
    dy = NUMERIC[(NUMERIC.index(dx) + 3) % len(NUMERIC)]
    left = [rand_col(rng, 250, dx, 0.05), rand_col(rng, 250, dy, 0.05)]
    right = [rand_col(rng, 180, dx, 0.05), rand_col(rng, 180, dy, 0.05)]
    for ops in ((">=", "<"), ("<", ">=")):
        check(plb, left, right, ops, "left")
    check(plb, left[:1], right[:1], ["<="], "inner")
    # the full value range of the dtype (extremes included)
    full_l, full_r = rand_col(rng, 200, dx, span=False), rand_col(rng, 200, dx, span=False)
    if np.dtype(dx).kind != "f":
        info = np.iinfo(dx)
        full_l[0][:4] = [info.min, info.max, 0, info.min]
        full_r[0][:4] = [info.max, info.min, 0, info.max]
    check(plb, [full_l], [full_r], [">"], "left")


@pytest.mark.parametrize("dt", ["float32", "float64"])
def test_float_specials(plb, dt):
    specials = [np.nan, -0.0, 0.0, np.inf, -np.inf, -1.0, 1.0, 2.0]
    rng = np.random.default_rng(4)
    lv = np.array(rng.choice(specials, 120), dt)
    rv = np.array(rng.choice(specials, 90), dt)
    ly = np.array(rng.choice(specials, 120), dt)
    ry = np.array(rng.choice(specials, 90), dt)
    lm, rm = rng.random(120) > 0.1, rng.random(90) > 0.1
    for op1, op2 in itertools.product(OPS, OPS):
        check(plb, [(lv, lm), (ly, None)], [(rv, None), (ry, rm)], [op1, op2], "left")
    for op in OPS:
        check(plb, [(lv, lm)], [(rv, rm)], [op], "inner")


def test_all_equal_keys(plb):
    n = 3000
    z = np.zeros(n, np.int64)
    for ops in (["<="], [">="], ["<"], ["<=", ">="], ["<", "<="], [">=", ">"]):
        k = len(ops)
        check(plb, [(z[:50], None)] * k, [(z, None)] * k, ops, "left")


def test_empty_and_all_null(plb):
    e = np.zeros(0, np.int32)
    v = np.arange(10, dtype=np.int32)
    nulls = np.zeros(10, bool)
    for how in ("inner", "left"):
        for ops in (["<"], ["<", ">="]):
            k = len(ops)
            check(plb, [(e, None)] * k, [(v, None)] * k, ops, how)
            check(plb, [(v, None)] * k, [(e, None)] * k, ops, how)
            check(plb, [(e, None)] * k, [(e, None)] * k, ops, how)
            check(plb, [(v, nulls)] * k, [(v, None)] * k, ops, how)
            check(plb, [(v, None)] * k, [(v, nulls)] * k, ops, how)
    # two predicates: a right row is live only when both of its columns are valid
    m1, m2 = np.arange(10) % 2 == 0, np.arange(10) % 2 == 1
    check(plb, [(v, None), (v, None)], [(v, m1), (v, m2)], ["<=", ">="], "left")


@pytest.mark.parametrize("nr", [1, 2, 3, 31, 32, 33, 63, 64, 65, 127, 128, 129, 255, 256, 257, 1023, 1024, 1025, 4095, 4096, 4097])
def test_tree_block_edges(plb, nr):
    rng = np.random.default_rng(nr)
    left = [rand_col(rng, 97, "int32", 0.05, 50), rand_col(rng, 97, "int32", 0.05, 50)]
    right = [rand_col(rng, nr, "int32", 0.05, 50), rand_col(rng, nr, "int32", 0.05, 50)]
    for ops in (("<", ">"), (">=", "<="), ("<=", "<")):
        check(plb, left, right, ops, "left")


def test_skewed_output(plb):
    # one left row matches every right row; every other left row matches none
    nr, nl = 200_000, 5000
    lx = np.ones(nl, np.int64)
    lx[1234] = -1
    zeros, ones = np.zeros(nr, np.int64), np.ones(nl, np.int64)
    for ops in (["<"], ["<", ">"]):
        k = len(ops)
        left, right = [(lx, None), (ones, None)][:k], [(zeros, None), (zeros, None)][:k]
        for how in ("inner", "left"):
            li = check(plb, left, right, ops, how)[0][0]
            assert np.count_nonzero(li == 1234) == nr


# ---------------------------------------------------------------------------- binding: flip, payloads, device, repeatability
def test_right_flip(plb):
    rng = np.random.default_rng(5)
    left = [rand_col(rng, 120, "int64", 0.1), rand_col(rng, 120, "float64", 0.1)]
    right = [rand_col(rng, 90, "int64", 0.1), rand_col(rng, 90, "float64", 0.1)]
    for ops in (["<", ">="], [">"]):
        k = len(ops)
        (li, lv), (ri, rv) = run(plb, left[:k], right[:k], ops, "right")
        assert rv is None and np.all(np.diff(ri.astype(np.int64)) >= 0)
        lv = np.ones(len(li), bool) if lv is None else lv
        got = io.as_multiset([(int(a) if va else None, int(b)) for a, va, b in zip(li, lv, ri)])
        L = [[None if (m is not None and not m[i]) else v[i].item() for i in range(len(v))] for v, m in left[:k]]
        R = [[None if (m is not None and not m[i]) else v[i].item() for i in range(len(v))] for v, m in right[:k]]
        assert got == io.as_multiset(io.brute(L, R, ops, "right"))


def test_payloads(plb):
    rng = np.random.default_rng(6)
    lx, rx = rand_col(rng, 80, "int32")[0], rand_col(rng, 60, "int32")[0]
    lpay = np.arange(80, dtype=np.int64) * 10
    rpay = np.arange(60, dtype=np.float64) / 4
    rstr = plb.StringColumn([f"r{i}" if i % 7 else None for i in range(60)])
    li, ri = plb.ie_join(lx, rx, "<=", "left")
    (lout,), (rout, sout) = plb.ie_join(lx, rx, "<=", "left", left_cols=[lpay], right_cols=[rpay, rstr])
    rvalid = np.ones(len(ri[0]), bool) if ri[1] is None else ri[1]
    assert np.array_equal(lout[0], lpay[li[0]])
    assert np.array_equal(rout[1] if rout[1] is not None else np.ones(len(rvalid), bool), rvalid)
    assert np.array_equal(rout[0][rvalid], rpay[ri[0][rvalid]])
    exp_s = [f"r{j}".encode() if (ok and j % 7) else None for j, ok in zip(ri[0], rvalid)]
    assert list(sout) == exp_s


def test_device_inputs_and_outputs(plb):
    rng = np.random.default_rng(7)
    lx, ly = rand_col(rng, 500, "int64", 0.1), rand_col(rng, 500, "float64", 0.1)
    rx, ry = rand_col(rng, 400, "int64", 0.1), rand_col(rng, 400, "float64", 0.1)
    host = run(plb, [lx, ly], [rx, ry], ["<", ">="], "left")
    dev = plb.ie_join([plb.to_device(*lx), plb.to_device(*ly)], [plb.to_device(*rx), plb.to_device(*ry)], ["<", ">="], "left", location=plb.DEVICE)
    assert all(isinstance(d, plb.OutColumn) and d.location == plb.DEVICE for d in dev)
    (dli, _), (dri, drv) = dev[0].to_numpy(), dev[1].to_numpy()
    assert np.array_equal(dli, host[0][0]) and np.array_equal(dri, host[1][0])
    assert (drv is None and host[1][1] is None) or np.array_equal(drv, host[1][1])


def test_repeatable_bytes(plb):
    rng = np.random.default_rng(8)
    left = [rand_col(rng, 3000, "float32", 0.05, 30), rand_col(rng, 3000, "int16", 0.05, 30)]
    right = [rand_col(rng, 2000, "float32", 0.05, 30), rand_col(rng, 2000, "int16", 0.05, 30)]
    a = run(plb, left, right, [">=", "<"], "left")
    b = run(plb, left, right, [">=", "<"], "left")
    assert np.array_equal(a[0][0], b[0][0]) and np.array_equal(a[1][0], b[1][0]) and np.array_equal(a[1][1], b[1][1])


def test_errors(plb):
    i64, f64 = np.arange(4, dtype=np.int64), np.arange(4, dtype=np.float64)
    with pytest.raises(plb.ComputeError):
        plb.ie_join(i64, f64, "<")
    with pytest.raises(plb.B200Error) as e:
        plb.ie_join(np.array([True, False]), np.array([True]), "<")
    assert e.value.status == 4
    with pytest.raises(plb.B200Error) as e:
        plb.ie_join([i64, i64[:3]], [i64, i64], ["<", "<"])
    assert e.value.status == 1
    # the C ABI rejects what the binding would refuse up front
    import ctypes as C
    cols = (plb.BlColumn * 2)(plb.Column(i64).struct(), plb.Column(i64).struct())
    out_l, out_r = plb.BlColumn(), plb.BlColumn()
    ops = (C.c_int32 * 2)(0, 9)
    L = plb.lib()
    assert L.bl_ie_join(cols, cols, ops, 3, 0, 0, C.byref(out_l), C.byref(out_r)) == 1
    assert L.bl_ie_join(cols, cols, ops, 2, 0, 0, C.byref(out_l), C.byref(out_r)) == 1
    assert L.bl_ie_join(cols, cols, (C.c_int32 * 1)(0), 1, 2, 0, C.byref(out_l), C.byref(out_r)) == 1
    assert L.bl_ie_join(None, cols, (C.c_int32 * 1)(0), 1, 0, 0, C.byref(out_l), C.byref(out_r)) == 1


# ---------------------------------------------------------------------------- at scale
def test_point_in_interval_1e7(plb):
    rng = np.random.default_rng(9)
    n_int, n_pt = 1_000_000, 10_000_000
    gaps, lens = rng.integers(1, 100, n_int), rng.integers(1, 100, n_int)
    starts = (np.cumsum(gaps + lens) - lens).astype(np.int64)
    ends = starts + lens
    perm = rng.permutation(n_int)
    st, en = starts[perm], ends[perm]
    t = rng.integers(0, int(ends[-1]) + 100, n_pt).astype(np.int64)
    dev = plb.ie_join([plb.to_device(t), plb.to_device(t)], [plb.to_device(st), plb.to_device(en)], [">=", "<"], "inner", location=plb.DEVICE)
    (li, _), (ri, _) = dev[0].to_numpy(), dev[1].to_numpy()
    k = np.searchsorted(starts, t, "right") - 1
    hit = (k >= 0) & (t < ends[np.maximum(k, 0)])
    inv = np.empty(n_int, np.int64)
    inv[perm] = np.arange(n_int)
    assert np.array_equal(li, np.nonzero(hit)[0].astype(np.uint32))
    assert np.array_equal(ri, inv[k[hit]].astype(np.uint32))


def test_single_predicate_2e8_pairs(plb):
    rng = np.random.default_rng(10)
    nl, nr = 20_000, 20_000
    l = rng.integers(0, 10**6, nl).astype(np.int64)
    r = rng.integers(0, 10**6, nr).astype(np.int64)
    dev = plb.ie_join(plb.to_device(l), plb.to_device(r), "<", "inner", location=plb.DEVICE)
    (li, _), (ri, _) = dev[0].to_numpy(), dev[1].to_numpy()
    rs = np.sort(r)
    exp_cnt = nr - np.searchsorted(rs, l, "right")
    assert li.size == exp_cnt.sum() and li.size > 1.5e8
    assert np.all(np.diff(li.astype(np.int64)) >= 0)
    assert np.array_equal(np.bincount(li, minlength=nl), exp_cnt)
    starts = np.concatenate([[0], np.cumsum(exp_cnt)])
    for i in np.random.default_rng(11).choice(nl, 20, replace=False):
        got = np.sort(ri[starts[i]:starts[i + 1]])
        assert np.array_equal(got, np.nonzero(r > l[i])[0].astype(np.uint32))
