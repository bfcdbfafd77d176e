"""GPU tests of the asof join (bl_join_asof): every index column is compared bit for bit, index and validity, with the
oracle (tests/asof_oracle.py: the reference's cursors for small inputs, the per-row rule for large ones) over the reference's
known answers, every key dtype, strategy and option, the NaN quirks, integer extremes, degenerate shapes, shared-memory and
global-memory windows, `by` keys of every kind, the error cases, device inputs and outputs, payloads and 2e7 rows."""
import numpy as np
import pytest

import asof_oracle as ao
from test_join_asof import asof_kats, kat_payload, same

pytestmark = pytest.mark.gpu
STRATS = ("backward", "forward", "nearest")
NULL = 0xFFFFFFFF


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as plb
    plb.init()
    return plb


def as_list(res):
    vals, valid = res
    assert vals.dtype == np.uint32
    if valid is not None:
        assert np.all(vals[~valid] == NULL), "a null slot must hold BL_IDX_NULL"
    return [None if (valid is not None and not valid[i]) else int(vals[i]) for i in range(len(vals))]


def check_bits(res, exp_idx, exp_valid):
    vals, valid = res
    valid = np.ones(len(vals), bool) if valid is None else valid
    assert np.array_equal(valid, exp_valid), f"validity differs at {np.nonzero(valid != exp_valid)[0][:10]}"
    assert np.array_equal(vals, exp_idx), f"index differs at {np.nonzero(vals != exp_idx)[0][:10]}"


def col(values, dtype):
    dt = np.dtype(dtype)
    valid = np.array([v is not None for v in values], bool)
    arr = np.array([0 if v is None else v for v in values], dt)
    return (arr, valid) if not valid.all() else arr


def by_col(plb, values, dtype=None):
    if values and any(isinstance(v, str) for v in values):
        return plb.StringColumn(values)
    kind = dtype or ("float64" if any(isinstance(v, float) for v in values) else "int64")
    return col(values, kind)


@pytest.mark.parametrize("case", asof_kats(), ids=lambda c: c["cite"][-70:])
def test_reference_kats(plb, case):
    dt = case["dtype"]
    lb = [by_col(plb, c, case["by_dtype"]) for c in case["left_by"]] if case["left_by"] else None
    rb = [by_col(plb, c, case["by_dtype"]) for c in case["right_by"]] if case["right_by"] else None
    res = plb.join_asof(col(case["left"], dt), col(case["right"], dt), case["strategy"], case["tol"], case["allow_eq"], lb, rb)
    got = as_list(res)
    assert same(kat_payload(case, got), case["expect"])


def random_sides(rng, dtype, nl, nr, pool, lnull=0.15, rnull=0.3):
    """sorted (total order) random sides with heavy duplicates; left nulls anywhere, right nulls first"""
    def side(n):
        v = rng.choice(pool, n).astype(dtype)
        return v[np.argsort(ao.total_keys(v), kind="stable")]
    lv, rv = side(nl), side(nr)
    lvalid = rng.random(nl) >= lnull
    k = int(rng.integers(0, max(int(nr * rnull), 0) + 1)) if nr else 0
    rvalid = np.arange(nr) >= k
    return (lv, lvalid), (rv, rvalid)


def pool_for(dtype):
    dt = np.dtype(dtype)
    if dt.kind == "f":
        return np.array([-np.inf, -7.5, -1.0, -0.0, 0.0, 0.5, 1.0, 1.5, 2.0, 3.0, 1e30, np.inf, np.nan], dt)
    info = np.iinfo(dt)
    base = [0, 1, 2, 3, 5, 8, 13, 21, 34, 55]
    if dt.kind == "i":
        base += [-1, -5, -34]
    return np.array(base + [info.min, info.min + 1, info.max - 1, info.max], dt)


def as_oracle_lists(side):
    v, ok = side
    return [x if o else None for x, o in zip(v, ok)]


DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"]


@pytest.mark.parametrize("dtype", DTYPES)
def test_every_dtype_strategy_and_option(plb, dtype):
    rng = np.random.default_rng(DTYPES.index(dtype))
    pool = pool_for(dtype)
    for trial in range(6):
        nl, nr = int(rng.integers(0, 3000)), int(rng.integers(0, 700))
        L, R = random_sides(rng, dtype, nl, nr, pool)
        left, right = as_oracle_lists(L), as_oracle_lists(R)
        for strategy in STRATS:
            for allow_eq in (False, True):
                for tol in (None, pool[int(rng.integers(0, len(pool)))], pool[1]):
                    exp = ao.cursor_asof(left, right, strategy, allow_eq, tol)
                    got = as_list(plb.join_asof(L, R, strategy, None if tol is None else np.array([tol], dtype), allow_eq))
                    assert got == exp, (dtype, trial, strategy, allow_eq, tol)


def test_nan_quirks(plb):
    r = np.array([0.0, 5.0, np.nan])
    assert as_list(plb.join_asof(np.array([6.0]), r, "nearest")) == [2]
    assert as_list(plb.join_asof(np.array([5.0]), r, "nearest")) == [0]
    for dt in ("float32", "float64"):
        for s in ("backward", "nearest"):
            got = as_list(plb.join_asof(np.array([0.0, 6.0, np.nan, np.nan], dt), np.array([0.0, 5.0, 10.0, 42.0], dt), s))
            assert got == [0, 1, 3, 3]


@pytest.mark.parametrize("dtype", ["int64", "uint64", "int32", "uint32"])
def test_integer_extremes_do_not_overflow(plb, dtype):
    info = np.iinfo(dtype)
    right = np.array([info.min, info.min + 1, 0 if dtype[0] == "i" else 1, info.max - 1, info.max], dtype)
    left = np.array([info.min, info.min, 0 if dtype[0] == "i" else 1, info.max - 2, info.max, info.max], dtype)
    lst_l, lst_r = list(left), list(right)
    for strategy in STRATS:
        for allow_eq in (False, True):
            for tol in (None, np.array([info.max], dtype), np.array([1], dtype), np.array([info.min if dtype[0] == "i" else 0], dtype)):
                exp = ao.cursor_asof(lst_l, lst_r, strategy, allow_eq, None if tol is None else tol[0])
                assert as_list(plb.join_asof(left, right, strategy, tol, allow_eq)) == exp, (strategy, allow_eq, tol)


@pytest.mark.parametrize("dtype", ["int8", "uint8", "int16", "uint16"])
def test_small_int_key_takes_an_int32_tolerance(plb, dtype):
    """the tolerance of an 8/16-bit key is an Int32, as the reference extracts it: 200 on an Int8 key, or a negative one"""
    info = np.iinfo(dtype)
    right = np.array(sorted({info.min, info.min + 3, 0, 5, info.max - 7, info.max}), dtype)
    left = np.array(sorted([info.min, info.min + 1, 0, 2, 3, info.max - 1, info.max]), dtype)
    for strategy in STRATS:
        for tol in (200, -3, 0, 70000):
            exp = ao.cursor_asof(list(left), list(right), strategy, True, np.int32(tol))
            assert as_list(plb.join_asof(left, right, strategy, tol)) == exp, (strategy, tol)
            assert as_list(plb.join_asof(left, right, strategy, np.array([tol], np.int32))) == exp


def test_empty_left_returns_at_once(plb):
    """an empty left side is answered without looking at the right side: the reference's answer is empty whatever it holds"""
    assert as_list(plb.join_asof(np.zeros(0, np.int64), np.array([3, 1, 2], np.int64))) == []


def test_degenerate_shapes(plb):
    e = np.zeros(0, np.int64)
    one = np.array([3], np.int64)
    nulls = (np.zeros(4, np.int64), np.zeros(4, bool))
    for strategy in STRATS:
        assert as_list(plb.join_asof(e, one, strategy)) == []
        assert as_list(plb.join_asof(one, e, strategy)) == [None]
        assert as_list(plb.join_asof(nulls, one, strategy)) == [None] * 4
        assert as_list(plb.join_asof(one, nulls, strategy)) == [None]
        assert as_list(plb.join_asof(one, one, strategy)) == [0]
        assert as_list(plb.join_asof(one, one, strategy, allow_exact_matches=False)) == [None]


@pytest.mark.parametrize("shape", ["sparse", "dense"])
def test_window_in_and_out_of_shared_memory(plb, shape):
    """sparse: the right side far larger than the left, so a tile's window does not fit in shared memory; dense: many left
    rows per right row"""
    rng = np.random.default_rng(5)
    if shape == "sparse":
        nl, nr, hi = 20_000, 2_000_000, 10**9
    else:
        nl, nr, hi = 300_000, 3_000, 10**6
    lv = np.sort(rng.integers(0, hi, nl)).astype(np.int64)
    rv = np.sort(rng.integers(0, hi, nr)).astype(np.int64)
    for strategy in STRATS:
        for tol in (None, 1000):
            idx, valid = ao.rule_asof((lv, None), (rv, None), strategy, True, tol)
            check_bits(plb.join_asof(lv, rv, strategy, tol), idx, valid)


def test_by_int32(plb):
    rng = np.random.default_rng(8)
    nl, nr = 5000, 2000
    L, R = random_sides(rng, "int64", nl, nr, pool_for("int64")[:13], rnull=0)
    lg, rg = rng.integers(0, 5, nl).astype(np.int32), rng.integers(1, 7, nr).astype(np.int32)      # groups on one side only
    lgv, rgv = rng.random(nl) > 0.1, rng.random(nr) > 0.1
    left, right = as_oracle_lists(L), as_oracle_lists(R)
    lb = [(int(g),) if ok else (None,) for g, ok in zip(lg, lgv)]
    rb = [(int(g),) if ok else (None,) for g, ok in zip(rg, rgv)]
    for strategy in STRATS:
        for allow_eq in (False, True):
            exp = ao.cursor_asof_by(left, right, lb, rb, strategy, allow_eq)
            got = as_list(plb.join_asof(L, R, strategy, None, allow_eq, [(lg, lgv)], [(rg, rgv)]))
            assert got == exp, (strategy, allow_eq)


def test_by_float64_canonicalised(plb):
    lb = np.array([-0.0, 0.0, np.nan, 1.0, np.nan, -0.0])
    rb = np.array([0.0, np.nan, -0.0, np.nan, 2.0])
    lv = np.array([1, 2, 3, 4, 5, 6], np.int64)
    rv = np.array([0, 1, 2, 3, 4], np.int64)
    exp = ao.cursor_asof_by(list(lv), list(rv), [(x,) for x in lb], [(x,) for x in rb], "backward")
    assert as_list(plb.join_asof(lv, rv, "backward", left_by=[lb], right_by=[rb])) == exp
    assert exp == [0, 2, 3, None, 3, 2]


def test_by_strings_host_device_chunked_sliced(plb):
    rng = np.random.default_rng(9)
    syms = ["A", "B", "", "CC", None, "é"]
    nl, nr = 400, 150
    L, R = random_sides(rng, "float64", nl, nr, pool_for("float64"), rnull=0)
    ls = [syms[i] for i in rng.integers(0, len(syms), nl)]
    rs = [syms[i] for i in rng.integers(0, len(syms), nr)]
    exp = ao.cursor_asof_by(as_oracle_lists(L), as_oracle_lists(R), [(s,) for s in ls], [(s,) for s in rs], "nearest")
    host = plb.StringColumn(ls), plb.StringColumn(rs)
    dev = plb.DeviceStringColumn(host[0]), plb.DeviceStringColumn(host[1])
    chunked = [plb.StringColumn(ls[:100]), plb.StringColumn(ls[100:])], [plb.StringColumn(rs[:7]), plb.StringColumn(rs[7:])]
    sliced = plb.StringColumn(["pad", "pad"] + ls, offset=2), plb.StringColumn(["x"] + rs + ["y"], offset=1, length=nr)
    for lb, rb in (host, dev, chunked, sliced):
        assert as_list(plb.join_asof(L, R, "nearest", left_by=[lb], right_by=[rb])) == exp


def test_by_several_mixed_columns(plb):
    rng = np.random.default_rng(10)
    nl, nr = 3000, 1000
    L, R = random_sides(rng, "int32", nl, nr, pool_for("int32"), rnull=0)
    a_l, a_r = rng.integers(0, 3, nl).astype(np.int8), rng.integers(0, 3, nr).astype(np.int8)
    b_l, b_r = rng.choice([0.0, -0.0, 1.5], nl), rng.choice([0.0, -0.0, 1.5], nr)
    s = ["x", "y"]
    c_l, c_r = [s[i] for i in rng.integers(0, 2, nl)], [s[i] for i in rng.integers(0, 2, nr)]
    d_lv, d_rv = rng.random(nl) > 0.05, rng.random(nr) > 0.05
    d_l, d_r = rng.integers(0, 2, nl).astype(np.uint64) << np.uint64(40), rng.integers(0, 2, nr).astype(np.uint64) << np.uint64(40)
    lb = [(a_l[i], b_l[i], c_l[i], d_l[i] if d_lv[i] else None) for i in range(nl)]
    rb = [(a_r[i], b_r[i], c_r[i], d_r[i] if d_rv[i] else None) for i in range(nr)]
    for strategy in STRATS:
        exp = ao.cursor_asof_by(as_oracle_lists(L), as_oracle_lists(R), lb, rb, strategy, True, np.int32(7))
        got = as_list(plb.join_asof(L, R, strategy, 7, True, [a_l, b_l, plb.StringColumn(c_l), (d_l, d_lv)], [a_r, b_r, plb.StringColumn(c_r), (d_r, d_rv)]))
        assert got == exp, strategy


def test_by_left_sorted_only_within_groups(plb):
    """the global check fails, the per-group check passes: same answer as the cursors"""
    rng = np.random.default_rng(12)
    nl, nr = 20_000, 4_000
    lg = np.sort(rng.integers(0, 50, nl)).astype(np.int64)            # grouped, each group time-sorted
    lv = np.concatenate([np.sort(rng.integers(0, 10_000, int((lg == g).sum()))) for g in range(50)]).astype(np.int64)
    rg = rng.integers(0, 50, nr).astype(np.int64)
    rv = np.sort(rng.integers(0, 10_000, nr)).astype(np.int64)
    assert (np.diff(lv) < 0).any()
    for strategy in STRATS:
        exp = ao.cursor_asof_by(list(lv), list(rv), [(g,) for g in lg], [(g,) for g in rg], strategy)
        assert as_list(plb.join_asof(lv, rv, strategy, None, True, [lg], [rg])) == exp
    # unsorted within a group -> UNSUPPORTED, naming the left side
    bad = lv.copy()
    i = int(np.nonzero(lg == lg[0])[0][-1])
    bad[0], bad[i] = bad[i] + 1, 0
    with pytest.raises(plb.B200Error, match="left") as e:
        plb.join_asof(bad, rv, "backward", left_by=[lg], right_by=[rg])
    assert e.value.status == 4


def test_errors(plb):
    i64, f64 = np.array([1, 2], np.int64), np.array([1.0, 2.0])
    with pytest.raises(plb.ComputeError):
        plb.join_asof(i64, f64)
    with pytest.raises(plb.ComputeError):
        plb.join_asof(i64, i64, left_by=[plb.StringColumn(["a", "b"])], right_by=[i64])
    with pytest.raises(plb.ComputeError):
        plb.join_asof(i64, i64, left_by=[i64.astype(np.int32)], right_by=[i64])

    def status(**kw):
        with pytest.raises(plb.B200Error) as e:
            plb.join_asof(**kw)
        return e.value.status
    assert status(left_on=i64, right_on=i64, tolerance=np.array([1, 2], np.int64)) == 1
    assert status(left_on=i64, right_on=i64, tolerance=np.array([1], np.int32)) == 1
    assert status(left_on=i64, right_on=i64, tolerance=(np.array([1], np.int64), np.array([False]))) == 1
    assert status(left_on=i64, right_on=i64, left_by=[np.array([1, 2, 3])], right_by=[i64]) == 1
    assert status(left_on=np.array([True, False]), right_on=np.array([True, False])) == 4
    assert status(left_on=i64, right_on=i64, left_by=[np.array([True, False])], right_by=[np.array([True, False])]) == 4
    with pytest.raises(plb.B200Error, match="left") as e:
        plb.join_asof(np.array([2, 1], np.int64), i64)
    assert e.value.status == 4
    with pytest.raises(plb.B200Error, match="right") as e:
        plb.join_asof(i64, np.array([2, 1], np.int64))
    assert e.value.status == 4
    with pytest.raises(plb.B200Error, match="right"):
        plb.join_asof(i64, (np.array([1, 0, 3], np.int64), np.array([True, False, True])))        # a null after a value
    with pytest.raises(plb.B200Error, match="right"):
        plb.join_asof(i64, i64[::-1].copy(), left_by=[np.zeros(2, np.int64)], right_by=[np.zeros(2, np.int64)])
    # an unsorted left side split over tiles: the cross-tile check
    lv = np.arange(10_000, dtype=np.int64)
    lv[4096:] -= 3000      # tile 2 starts below the largest key of tile 1
    with pytest.raises(plb.B200Error, match="left"):
        plb.join_asof(lv, i64)
    import ctypes as C
    out = plb.BlColumn()
    l = plb.Column(i64).struct()
    assert plb.lib().bl_join_asof(C.byref(l), C.byref(l), None, None, C.c_int32(0), C.c_int32(3), C.c_int32(1), None, C.c_int32(0), C.byref(out)) == 1
    assert plb.lib().bl_join_asof(C.byref(l), C.byref(l), None, None, C.c_int32(1), C.c_int32(0), C.c_int32(1), None, C.c_int32(0), C.byref(out)) == 1
    k = plb.BlSortKey(C.pointer(l), None, 0, 1)
    ka = (plb.BlSortKey * 1)(k)
    assert plb.lib().bl_join_asof(C.byref(l), C.byref(l), ka, ka, C.c_int32(1), C.c_int32(0), C.c_int32(1), None, C.c_int32(0), C.byref(out)) == 1


def test_device_inputs_outputs_and_payloads(plb):
    rng = np.random.default_rng(13)
    L, R = random_sides(rng, "float32", 5000, 800, pool_for("float32"))
    idx, valid = ao.rule_asof(L, R, "nearest", True, np.float32(2.0))
    dl, dr = plb.to_device(*L), plb.to_device(*R)
    out = plb.join_asof(dl, dr, "nearest", np.float32(2.0), location=plb.DEVICE)
    assert out.location == plb.DEVICE
    check_bits(out.to_numpy(), idx, valid)
    pay = rng.integers(0, 10**9, 800).astype(np.int64)
    names = [f"r{i}" if i % 7 else None for i in range(800)]
    (gi, gv), ((p, pv), s) = plb.join_asof(L, R, "nearest", 2.0, right_cols=[pay, plb.StringColumn(names)])
    check_bits((gi, gv), idx, valid)
    pv = np.ones(len(p), bool) if pv is None else pv
    assert np.array_equal(pv, valid) and np.array_equal(p[valid], pay[idx[valid]])
    assert s == [names[j].encode() if ok and names[j] is not None else None for j, ok in zip(idx, valid)]
    d_idx, (d_p, d_s) = plb.join_asof(dl, dr, "nearest", 2.0, right_cols=[pay, plb.StringColumn(names)], location=plb.DEVICE)
    assert isinstance(d_s, plb.DeviceStringColumn) and d_p.location == plb.DEVICE
    check_bits(d_idx.to_numpy(), idx, valid)


@pytest.mark.parametrize("by", [False, True])
def test_large(plb, by):
    rng = np.random.default_rng(14)
    nl, nr = 20_000_000, 2_000_000
    lv = np.sort(rng.integers(0, 10**12, nl)).astype(np.int64)
    rv = np.sort(rng.integers(0, 10**12, nr)).astype(np.int64)
    lvalid = rng.random(nl) > 0.01
    lg = rg = None
    if by:
        lg, rg = rng.integers(0, 1000, nl).astype(np.int64), rng.integers(0, 1000, nr).astype(np.int64)
    for strategy, tol in (("backward", None), ("nearest", 10**6)):
        idx, valid = ao.rule_asof((lv, lvalid), (rv, None), strategy, True, tol, lg, rg)
        got = plb.join_asof((lv, lvalid), rv, strategy, tol, True, [lg] if by else None, [rg] if by else None)
        check_bits(got, idx, valid)
