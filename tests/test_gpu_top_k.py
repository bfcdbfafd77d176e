"""GPU tests of top-k selection (top_k.cu: k_topk_pass, op_mask_rows) and of the selection plan inside sorts with a limit.

bl_top_k must return exactly the checker's row ids: the first k rows of the stable order (sort_oracle; numpy_arg_sort at
large sizes, which tests/test_top_k.py and tests/test_sort_cases.py check against the plain oracle), in ascending row order.
top_k / bottom_k / top_k_by / bottom_k_by and the plugin entries must equal the payload at arg_sort(..., limit=k).  The
launch profile shows which plan ran: streaming passes ("topk_pass") over all rows while a candidate set holds more than
n / 32 rows, list passes ("topk_pass_list") after it, and in a sort with a limit the selection ("topk_andor" first) runs for limit <= n / SELECT_DIV.

Caps.  SM = device_info()["sm_count"]; k_topk_pass and k_mask_rows use grid_for(.., 8 per SM): their grid-stride loops
run again past 8*SM*256 rows (k_topk_pass) and 8*SM*128 words = 8*SM*4096 rows (k_mask_rows); N_BIG = 3*8*SM*4096 + 77
runs both several times, ragged."""
import ctypes as C

import numpy as np
import pytest

import sort_cases as sc
import sort_oracle
from test_top_k import KATS, checker_ids, kat_matches, kat_plan

pytestmark = pytest.mark.gpu

DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64", "bool"]
INVALID, UNSUPPORTED = 1, 4
SELECT_DIV = 8      # sort.cu SORT_SELECT_DIV: a sort with limit <= n / SELECT_DIV selects first


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as m
    m.init()
    return m


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


def profiled(plb, fn):
    plb.profile_reset()
    plb.profile_enable(True)
    try:
        out = fn()
        plb.sync()
        prof = plb.profile()
    finally:
        plb.profile_enable(False)
    return out, {k: int(v.get("launches", 0)) for k, v in prof.items()}


def arg(cols, valids):
    return [(c, v) if v is not None else c for c, v in zip(cols, valids)]


def expected_ids(cols, valids, k, desc, nl):
    return np.sort(sort_oracle.numpy_arg_sort(cols, valids, desc, nl, limit=k)).astype(np.uint32)


def check(plb, cols, valids, k, desc=False, nl=False):
    got = plb.arg_top_k(arg(cols, valids), k, desc, nl)
    exp = expected_ids(cols, valids, k, desc, nl)
    assert got.dtype == np.uint32 and np.array_equal(got, exp), (k, desc, nl, got[:20], exp[:20])
    return got


# ------------------------------------------------------------------------------------------------ known answers
@pytest.mark.parametrize("case", KATS, ids=[f"{i}-{c['op']}" for i, c in enumerate(KATS)])
def test_known_answers(plb, case):
    keys, desc, nl, payload = kat_plan(case)
    frame, dts = case["frame"], case["dtypes"]

    def dev_col(name):
        vals = frame[name]
        if dts[name] == "str":
            return plb.StringColumn(vals)
        valid = np.array([v is not None for v in vals], bool)
        a = np.array([0 if v is None else v for v in vals], dtype=sc.NP[dts[name]] if dts[name] != "bool" else bool)
        return (a, valid) if not valid.all() else a

    k = case["k"]
    by = [dev_col(b) for b in keys]
    ids = plb.arg_top_k(by, k, desc, nl)
    cols = [frame[b] for b in keys]
    assert np.array_equal(ids, checker_ids(cols, [[v is not None for v in c] for c in cols], k, desc, nl))
    order = plb.arg_sort(by, descending=desc, nulls_last=nl, limit=k)
    assert np.array_equal(np.sort(order), ids)
    got = {p: [frame[p][i] for i in order] for p in payload}
    assert kat_matches(case, got), (case["src"], got)
    # the bindings that materialise values (numeric payloads of 4 / 8 bytes and strings)
    if case["op"] in ("top_k_by", "bottom_k_by") and all(dts[p] in ("int64", "float64", "str") for p in payload):
        fn = plb.top_k_by if case["op"] == "top_k_by" else plb.bottom_k_by
        outs = fn([dev_col(p) for p in payload], by if len(by) > 1 else by[0], k, reverse=case["reverse"])
        for p, o in zip(payload, outs):
            vals = o if dts[p] == "str" else [None if (o[1] is not None and not o[1][i]) else o[0][i].item() for i in range(len(o[0]))]
            if dts[p] == "str":
                vals = [None if v is None else v.decode() for v in vals]
            assert vals == got[p], (case["src"], p)


# ------------------------------------------------------------------------------------------------ key dtypes
@pytest.mark.parametrize("dt", DTYPES)
def test_every_dtype_full_range(plb, sm, dt):
    rng = np.random.default_rng(DTYPES.index(dt))
    n = 8 * sm * 256 + 333
    col = sc.full_range_column(rng, dt, n)
    for desc in (False, True):
        for k in (1, 17, 1000, n // 100, n // 3, n - 1):
            check(plb, [col], [None], k, desc)


@pytest.mark.parametrize("dt", ["int32", "float64", "uint16", "bool"])
def test_null_patterns(plb, dt):
    rng = np.random.default_rng(5)
    n = 50_000
    col = sc.full_range_column(rng, dt, n)
    for valid in (rng.random(n) < 0.9, np.zeros(n, bool), np.ones(n, bool), np.arange(n) % 2 == 0, np.arange(n) >= n - 10):
        for desc in (False, True):
            for nl in (False, True):
                for k in (1, 9, int(valid.sum()), max(int((~valid).sum()), 1), n // 2):
                    check(plb, [col], [valid], k, desc, nl)


def test_string_and_binary_keys(plb):
    rng = np.random.default_rng(9)
    n = 20_000
    words = [bytes(rng.integers(0, 256, int(rng.integers(0, 6)), dtype=np.uint8)) for _ in range(700)] + [b"", b"\x00", b"\xff\xff"]
    vals = [None if rng.random() < 0.1 else words[int(i)] for i in rng.integers(0, len(words), n)]
    rank, valid = sc.dense_rank_bytes(vals)
    other = rng.integers(0, 3, n).astype(np.int32)
    for desc in (False, True):
        for nl in (False, True):
            for k in (1, 50, 5000):
                got = plb.arg_top_k([plb.StringColumn(vals), other], k, [desc, not desc], nl)
                exp = expected_ids([rank, other], [valid, None], k, [desc, not desc], nl)
                assert np.array_equal(got, exp)
    texts = [None if v is None else v.hex() for v in vals]
    rank_t, valid_t = sc.dense_rank_bytes([None if t is None else t.encode() for t in texts])
    got = plb.arg_top_k(plb.StringColumn(texts), 300, True, True)
    assert np.array_equal(got, expected_ids([rank_t], [valid_t], 300, True, True))
    order = sort_oracle.numpy_arg_sort([rank_t], [valid_t], True, True, limit=3)
    assert plb.top_k(plb.StringColumn(texts), 3) == [texts[i].encode() for i in order]


def test_several_columns_mixed_flags(plb):
    rng = np.random.default_rng(13)
    n = 300_000
    a = rng.integers(0, 5, n).astype(np.int16)
    b = rng.normal(size=n).round(1)
    c = rng.integers(-2**40, 2**40, n)
    va, vb = rng.random(n) < 0.95, rng.random(n) < 0.9
    for desc, nl in (([True, False, True], [False, True, True]), ([False, True, False], [True, False, False])):
        for k in (1, 100, 20_000, n - 3):
            check(plb, [a, b, c], [va, vb, None], k, desc, nl)


def test_k_edges_and_ties(plb):
    rng = np.random.default_rng(17)
    n = 100_003
    x = rng.integers(0, 50, n).astype(np.int64)
    for k in (0, 1, n - 1, n, n + 7):
        for desc in (False, True):
            got = check(plb, [x], [None], k, desc)
            assert got.size == min(k, n)
    # k cutting a tie run: the run of the smallest value is entered part way
    srt = np.sort(x)
    first = int(np.searchsorted(srt, srt[0], side="right"))
    for k in (first - 1, first, first + 1, first + 1234):
        check(plb, [x], [None], k)
    # all keys equal: only the row-index digits decide
    eq = np.full(n, 7, np.int64)
    for k in (1, 255, 256, 257, 65_537, n - 1):
        got, prof = profiled(plb, lambda: plb.arg_top_k(eq, k))
        assert np.array_equal(got, np.arange(k, dtype=np.uint32))
    # keys that differ only in the last digit of the last column
    y = np.full(n, 2**40, np.int64) + rng.integers(0, 256, n)
    z = np.zeros(n, np.int32)
    for k in (1, 500, n // 2):
        check(plb, [z, y], [None, None], k, [False, True], False)


def test_compaction_threshold_both_sides(plb):
    """the first digit's bucket holds more (streaming to the end) or fewer (list passes) than n / 32 rows"""
    rng = np.random.default_rng(19)
    n = 1 << 20
    # a top byte over 4 values: every bucket has ~n / 4 rows > n / 32, the next byte spreads them
    wide = (rng.integers(0, 4, n).astype(np.uint32) << 24) | rng.integers(0, 1 << 24, n).astype(np.uint32)
    # a top byte over all 256 values: every bucket ~n / 256 < n / 32
    narrow = rng.integers(0, 2**32, n, dtype=np.uint64).astype(np.uint32)
    for col, list_expected in ((narrow, True), (wide, False)):
        for k in (10, 1000):
            got, prof = profiled(plb, lambda: plb.arg_top_k(col, k))
            assert np.array_equal(got, expected_ids([col], [None], k, False, False))
            assert prof.get("topk_pass", 0) >= 1
            if list_expected:
                assert prof.get("topk_pass_list", 0) >= 1
            else:
                assert prof.get("topk_pass", 0) >= 2      # the second digit ran over all rows
    # constant digits cost no pass: keys equal but in the last byte take one AND / OR read, a pass over the last byte,
    # then one streaming pass over the first row-index digit that builds the list (every bucket holds ~n / 256 rows)
    same = np.full(n, 0x01020300, np.uint32) | rng.integers(0, 256, n).astype(np.uint32)
    got, prof = profiled(plb, lambda: plb.arg_top_k(same, 12345))
    assert np.array_equal(got, expected_ids([same], [None], 12345, False, False))
    assert prof.get("topk_andor", 0) == 1 and prof.get("topk_pass", 0) == 2 and prof.get("topk_pass_list", 0) >= 1


def test_tie_step(plb):
    """a tie run too large for a list takes one streaming pass and the first `need` of its rows by tile counts; keys that
    never narrow the rows (all equal) need no pass at all"""
    rng = np.random.default_rng(21)
    n = 1 << 20
    two = rng.integers(0, 2, n).astype(np.int64) * 1000 - 7      # two values: the first bucket holds ~n / 2 rows
    for k in (1, 1000, n // 3, n // 2 + 5):
        for desc in (False, True):
            got, prof = profiled(plb, lambda: plb.arg_top_k(two, k, desc))
            assert np.array_equal(got, expected_ids([two], [None], k, desc, False)), (k, desc)
            if k < int((two == (two.max() if desc else two.min())).sum()):
                assert prof.get("topk_tie", 0) == 1 and prof.get("mask_first", 0) == 1, prof
    valid = rng.random(n) < 0.5
    got, prof = profiled(plb, lambda: plb.arg_top_k((two, valid), 777, False, True))
    assert np.array_equal(got, expected_ids([two], [valid], 777, False, True))
    eq = np.full(n, 5, np.int32)
    got, prof = profiled(plb, lambda: plb.arg_top_k(eq, 4321))
    assert np.array_equal(got, np.arange(4321, dtype=np.uint32))
    assert prof.get("topk_pass", 0) == 0 and prof.get("topk_tie", 0) == 0


def test_sizes_past_the_grids(plb, sm):
    rng = np.random.default_rng(23)
    n = 3 * 8 * sm * 4096 + 77
    x = rng.normal(size=n)
    for k in (3, n // 1000, n // 7, n - 5):
        check(plb, [x], [None], k, True)


def test_device_inputs_and_outputs(plb):
    rng = np.random.default_rng(29)
    n = 200_001
    x = rng.integers(-10**9, 10**9, n)
    valid = rng.random(n) < 0.9
    d = plb.to_device(x, valid)
    out = plb.arg_top_k(d, 5000, True, True, location=plb.DEVICE)
    ids, _ = plb.gather([plb.to_device(np.arange(n, dtype=np.int64))], out, check_bounds=True)[0]
    assert np.array_equal(ids.astype(np.uint32), expected_ids([x], [valid], 5000, True, True))


def test_top_k_bottom_k_values(plb):
    rng = np.random.default_rng(31)
    n = 100_000
    x = rng.normal(size=n)
    valid = rng.random(n) < 0.97
    for fn, desc in ((plb.top_k, True), (plb.bottom_k, False)):
        for k in (5, int(valid.sum()), n, n + 10):      # past the valid count: padded with the nulls
            (v, vm), = [fn((x, valid), k)]
            order = sort_oracle.numpy_arg_sort([x], [valid], desc, True, limit=k)
            vm = np.ones(v.size, bool) if vm is None else vm      # no null among the rows taken
            assert np.array_equal(v[vm], x[order][valid[order]])
            assert np.array_equal(vm, valid[order])
            assert vm[: int(valid.sum())].all() and not vm[int(valid.sum()):].any()


# ------------------------------------------------------------------------------------------------ the limit plan
@pytest.mark.parametrize("dt", ["int32", "int64", "float32", "float64", "uint64", "int16", "bool"])
def test_limit_plan_same_bytes(plb, sm, dt):
    rng = np.random.default_rng(37)
    n = 3 * 8 * sm * 256 + 77
    key = sc.full_range_column(rng, dt, n)
    valid = rng.random(n) < 0.9
    second = rng.integers(0, 7, n).astype(np.int64)
    selectable = dt not in ("int16", "bool")
    for limit in (0, 1, 100, n // SELECT_DIV, n // SELECT_DIV + 1, n // 10):
        for desc in (False, True):
            exp = sort_oracle.numpy_arg_sort([key, second], [valid, None], [desc, False], [True, False], limit=limit)
            got, prof = profiled(plb, lambda: plb.arg_sort([(key, valid), second], [desc, False], [True, False], limit=limit))
            assert np.array_equal(got, exp), (limit, desc)
            took = prof.get("topk_andor", 0) > 0
            assert took == (selectable and 0 < limit <= n // SELECT_DIV), (limit, prof)
            (p, _), = plb.sort([(key, valid), second], [np.arange(n, dtype=np.int64)], [desc, False], [True, False], limit=limit)
            assert np.array_equal(p, exp.astype(np.int64))


def test_limit_plan_string_keys(plb):
    rng = np.random.default_rng(41)
    n = 100_000
    vals = [None if rng.random() < 0.05 else ("w%d" % int(i)).encode() for i in rng.integers(0, 5000, n)]
    rank, valid = sc.dense_rank_bytes(vals)
    x = rng.integers(0, 3, n).astype(np.int32)
    for limit in (7, n // SELECT_DIV, n // SELECT_DIV + 1, n // 2):
        got, prof = profiled(plb, lambda: plb.arg_sort([plb.StringColumn(vals), x], [True, False], True, limit=limit))
        assert np.array_equal(got, sort_oracle.numpy_arg_sort([rank, x], [valid, None], [True, False], True, limit=limit))
        assert (prof.get("topk_andor", 0) > 0) == (limit <= n // SELECT_DIV)


# ------------------------------------------------------------------------------------------------ C ABI errors
def test_header_errors(plb):
    L = plb.lib()
    x = np.arange(10, dtype=np.int64)
    st = plb.Column(x).struct()
    out = plb.BlColumn()

    def call(keys, k=3):
        arr = (plb.BlSortKey * max(len(keys), 1))(*keys)
        return L.bl_top_k(arr if keys else None, C.c_int32(len(keys)), C.c_int64(k), C.c_int32(plb.HOST), C.byref(out))

    key = plb.BlSortKey(C.pointer(st), None, 0, 0)
    assert call([key], -1) == INVALID
    assert call([]) == INVALID
    short = plb.Column(x[:5]).struct()
    assert call([key, plb.BlSortKey(C.pointer(short), None, 0, 0)]) == INVALID
    assert call([plb.BlSortKey(None, None, 0, 0)]) == INVALID
    sc_ = plb.StringColumn(["a"] * 10)
    sst = sc_.struct()
    assert call([plb.BlSortKey(C.pointer(st), C.pointer(sst), 1, 0)]) == INVALID
    assert L.bl_top_k(C.byref(key), C.c_int32(1), C.c_int64(3), C.c_int32(plb.HOST), None) == INVALID
    bad = plb.Column(x).struct()
    bad.dtype = 77
    assert call([plb.BlSortKey(C.pointer(bad), None, 0, 0)]) == UNSUPPORTED      # every dtype the ABI defines is sortable
    big = plb.BlColumn()
    C.memmove(C.byref(big), C.byref(st), C.sizeof(st))
    big.length = 1 << 32
    assert call([plb.BlSortKey(C.pointer(big), None, 0, 0)]) == UNSUPPORTED
    assert call([key], 0) == 0 and out.length == 0


# ------------------------------------------------------------------------------------------------ plugin ABI
def test_plugin_entries(plb):
    import pyarrow as pa
    from test_gpu_plugin_abi import Caller
    caller = Caller(plb.lib())
    rng = np.random.default_rng(43)
    n = 5000
    a = rng.integers(0, 30, n)
    am = rng.random(n) < 0.1
    b = rng.normal(size=n)
    A, B = pa.array(a, mask=am), pa.array(b)
    for name, top in (("top_k_idx", True), ("bottom_k_idx", False)):
        for reverse in (False, True, 1, 2):
            rev = [bool(reverse & 1), bool(reverse & 2)] if not isinstance(reverse, bool) else [reverse, reverse]
            desc = [(not r) if top else r for r in rev]
            for k in (0, 1, 40, n + 1):
                out = caller.call(name, [("a", [A.slice(0, 1000), A.slice(1000)]), ("b", [B])], kwargs={"k": k, "reverse": reverse})
                exp = sort_oracle.numpy_arg_sort([a, b], [~am, None], desc, True, limit=k)
                assert out.type == pa.uint32()
                assert out.to_pylist() == exp.tolist(), (name, reverse, k)
    with pytest.raises(RuntimeError, match="k"):
        caller.call("top_k_idx", [("a", [A])])
    with pytest.raises(RuntimeError, match="k"):
        caller.call("top_k_idx", [("a", [A])], kwargs={"k": -2})
