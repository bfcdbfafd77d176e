"""GPU tests of unique (unique.cu: the K5 table with first rows and lengths, k_uniq_last, k_uniq_mark, op_mask_rows).

bl_unique must return exactly the oracle's row ids (tests/unique_oracle.py; its numpy form at large sizes, which
tests/test_unique.py checks against the dict form) for every keep strategy, and bl_unique_mask exactly its four masks.
The launch profile shows which passes ran: "uniq_last" for the LAST kinds only, one "uniq_mark" per call.

Caps.  SM = device_info()["sm_count"]; k_uniq_mark and k_uniq_last use grid_for(.., 16 per SM) CTAs of 256 threads and
k_mask_rows 16 per SM tiles of 4096 rows: N_BIG = 3 * 16 * SM * 4096 + 77 runs every grid-stride loop several times,
with a ragged tail."""
import ctypes as C

import numpy as np
import pytest

import sort_cases as sc
import unique_oracle as uo
from test_unique import KATS

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED = 1, 4
KEEP_KIND = {"first": "first", "any": "first", "last": "last", "none": "unique"}
DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64", "bool"]


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


def mask_fns(plb):
    return {"first": plb.is_first_distinct, "last": plb.is_last_distinct, "unique": plb.is_unique, "duplicated": plb.is_duplicated}


def check(plb, keys, np_cols, keeps=("first", "last", "any", "none")):
    """every mask and every keep strategy of the device keys `keys` against the numpy oracle over np_cols"""
    m = uo.np_masks(np_cols)
    for kind, fn in mask_fns(plb).items():
        got = fn(keys)
        assert got.dtype == np.bool_ and np.array_equal(got, m[kind]), kind
    for keep in keeps:
        got = plb.arg_unique(keys, keep)
        assert got.dtype == np.uint32 and np.array_equal(got, np.flatnonzero(m[KEEP_KIND[keep]])), keep
    return m


def arg(values, valid):
    return values if valid is None else (values, valid)


# ------------------------------------------------------------------------------------------------ known answers
def kat_column(plb, case, name):
    vals, dt = case["frame"][name], case["dtypes"][name]
    pre = case.get("prefix", {}).get(name, [])
    if dt == "str":
        return plb.StringColumn(pre + vals, offset=len(pre))
    full = pre + vals
    valid = np.array([v is not None for v in full], bool)
    np_dt = {"int64": np.int64, "float64": np.float64, "bool": np.bool_}[dt]
    values = np.array([(False if dt == "bool" else 0) if v is None else v for v in full], dtype=np_dt)
    return plb.Column(values, None if valid.all() else valid, offset=len(pre))


@pytest.mark.parametrize("case", KATS, ids=[f"{i}:{c['src'].rsplit('/', 1)[-1]}" for i, c in enumerate(KATS)])
def test_known_answers(plb, case):
    frame = case["frame"]
    if case["op"] == "mask":
        got = mask_fns(plb)[case["kind"]]([kat_column(plb, case, c) for c in case["keys"]])
        assert got.tolist() == case["expected"], case["src"]
        return
    subset = list(frame) if case["subset"] is None else case["subset"]
    ids = plb.arg_unique([kat_column(plb, case, c) for c in subset], case["keep"]).tolist()
    assert ids == uo.arg_unique([frame[c] for c in subset], case["keep"]), case["src"]
    if case.get("slice"):
        ids = ids[case["slice"][0]:case["slice"][0] + case["slice"][1]]
    got = {c: [frame[c][i] for i in ids] for c in frame}
    exp = case["expected"]
    if case["order"] == "pinned":
        assert all(all(uo.canon(a) == uo.canon(b) for a, b in zip(got[c], exp[c])) and len(got[c]) == len(exp[c]) for c in frame), case["src"]
    else:
        key = lambda c: sorted(uo.canon(v) for v in c)
        assert all(key(got[c]) == key(exp[c]) for c in frame), case["src"]


# ------------------------------------------------------------------------------------------------ key dtypes
@pytest.mark.parametrize("dt", DTYPES)
def test_every_dtype_full_range(plb, sm, dt):
    """full-range bit patterns (Int64 MIN = the table's empty key, UInt64 max, NaN payloads, both zeros) drawn with repeats"""
    rng = np.random.default_rng(DTYPES.index(dt))
    n = 16 * sm * 256 + 333
    pool = sc.full_range_column(rng, dt, 4000)
    col = rng.choice(pool, n)
    col[: pool.size] = pool
    for valid in (None, rng.random(n) < 0.8):
        check(plb, [arg(col, valid)], [(col, valid)])


def test_kept_rows_keep_their_bytes(plb):
    """-0.0 == +0.0 and every NaN is one key, but the gathered row is the kept row's own bytes"""
    for dt, ut in ((np.float64, np.uint64), (np.float32, np.uint32)):
        x = np.array([0.0, -0.0, np.nan, -np.nan, 1.0, -0.0, 0.0], dt)
        x[2:4] = np.array([0x7FF8000000000001, 0xFFF8000000000002] if dt is np.float64 else [0x7FC00001, 0xFFC00002], ut).view(dt)
        for keep, rows in (("first", [0, 2, 4]), ("last", [3, 4, 6]), ("any", [0, 2, 4]), ("none", [4])):
            (v, _), = plb.unique([x], keep=keep)
            assert np.array_equal(v.view(ut), x[rows].view(ut)), (dt, keep)
    (v, _), = plb.unique([np.array([0.0, -0.0])], keep="first")
    assert v.view(np.uint64).tolist() == [0]
    (v, _), = plb.unique([np.array([0.0, -0.0])], keep="last")
    assert v.view(np.uint64).tolist() == [0x8000000000000000]


def test_boolean_keys_at_bit_offsets(plb):
    rng = np.random.default_rng(3)
    n = 5000
    for off in (0, 1, 3, 31, 32, 33):
        b = rng.random(n + off) < 0.5
        valid = rng.random(n + off) < 0.7
        for v in (None, valid):
            key = plb.Column(b, v, offset=off)
            check(plb, [key], [(b[off:], None if v is None else v[off:])])
            other = rng.integers(0, 3, n).astype(np.int32)
            check(plb, [plb.Column(b, v, offset=off), other], [(b[off:], None if v is None else v[off:]), (other, None)])


def test_string_and_binary_keys(plb):
    rng = np.random.default_rng(9)
    n = 20_000
    words = [bytes(rng.integers(0, 256, int(rng.integers(0, 6)), dtype=np.uint8)) for _ in range(700)] + [b"", b"\x00", b"a\x00", b"a"]
    vals = [None if rng.random() < 0.1 else words[int(i)] for i in rng.integers(0, len(words), n)]
    check(plb, [plb.StringColumn(vals)], [(vals, None)])
    texts = [None if v is None else v.hex() for v in vals]
    check(plb, [plb.StringColumn(texts)], [(texts, None)])
    dev = plb.DeviceStringColumn(plb.StringColumn(vals))
    check(plb, [dev], [(vals, None)], keeps=("last",))
    # two chunks of one column
    check(plb, [[plb.StringColumn(vals[:777]), plb.StringColumn(vals[777:])]], [(vals, None)], keeps=("first",))


def test_multi_column_keys(plb):
    rng = np.random.default_rng(13)
    n = 300_000
    # three full-range 64-bit columns: op_pack_keys replaces them by group ids before they fit one word
    pools = [sc.full_range_column(rng, dt, 60) for dt in ("int64", "uint64", "float64")]
    cols = [rng.choice(p, n) for p in pools]
    valids = [None, rng.random(n) < 0.9, None]
    check(plb, [arg(c, v) for c, v in zip(cols, valids)], list(zip(cols, valids)))
    # a string, a Boolean and an Int32 column
    words = [None, "", "x", "y\x00", "zz"]
    s = [words[i] for i in rng.integers(0, len(words), n)]
    b = rng.random(n) < 0.5
    bv = rng.random(n) < 0.9
    i32 = rng.integers(-3, 3, n).astype(np.int32)
    check(plb, [plb.StringColumn(s), (b, bv), i32], [(s, None), (b, bv), (i32, None)])
    # small integers beside wide ones
    i8 = rng.integers(-128, 128, n).astype(np.int8)
    u16 = rng.integers(0, 4, n).astype(np.uint16)
    check(plb, [i8, u16, cols[0]], [(i8, None), (u16, None), (cols[0], None)])


# ------------------------------------------------------------------------------------------------ sizes and distributions
def test_sizes(plb, sm):
    rng = np.random.default_rng(17)
    n_big = 3 * 16 * sm * 4096 + 77
    for n in (0, 1, 2, 31, 32, 33, 63, 65, 1000, 16 * sm * 256 + 31):
        x = rng.integers(0, max(n // 3, 1), n).astype(np.int64)
        valid = rng.random(n) < 0.9
        check(plb, [x], [(x, None)])
        check(plb, [(x, valid)], [(x, valid)])
    x = rng.integers(0, n_big // 2, n_big).astype(np.int64)
    check(plb, [plb.to_device(x)], [(x, None)])


def test_all_null_keys(plb):
    for n in (1, 3, 33, 100_000):
        for dt in (np.int64, np.float32, np.int16):
            x = np.zeros(n, dt)
            valid = np.zeros(n, bool)
            m = check(plb, [(x, valid)], [(x, valid)])
            assert np.flatnonzero(m["first"]).tolist() == [0] and np.flatnonzero(m["last"]).tolist() == [n - 1]
        check(plb, [plb.StringColumn([None] * n)], [([None] * n, None)])
        b = np.zeros(n, bool)
        check(plb, [(b, b)], [(b, b)])


@pytest.mark.parametrize("distinct", [1, 2])
def test_few_keys_over_many_rows(plb, distinct):
    """1 and 2 keys over 2^24 rows: the heavy-hitter and shared-memory K5 plans, and k_uniq_last's one atomic per warp"""
    rng = np.random.default_rng(19 + distinct)
    n = 1 << 24
    x = (rng.integers(0, distinct, n).astype(np.int64) - 1) * 0x7FFFFFFFFFFF
    d = plb.to_device(x)
    check(plb, [d], [(x, None)])
    valid = rng.random(n) < 0.5
    dv = plb.to_device(x, valid)
    check(plb, [dv], [(x, valid)], keeps=("last", "none"))


def test_zipf_sorted_and_distinct(plb):
    rng = np.random.default_rng(23)
    n = 1 << 24
    z = rng.zipf(1.1, n).astype(np.int64)
    check(plb, [plb.to_device(z)], [(z, None)])
    alld = rng.permutation(n).astype(np.int64) * 7919 - 10**12
    check(plb, [plb.to_device(alld)], [(alld, None)])
    runs = np.repeat(np.arange(n // 16, dtype=np.int64), 16)[:n - 5]
    check(plb, [plb.to_device(runs)], [(runs, None)], keeps=("first", "last"))


def test_overflow_redo(plb, sm):
    """The sample reads rows i * n / 65536: they hold 4 keys, every other row a key of its own.  The sampled estimate is far
    too small, the one-shot build overflows and is redone into a larger table before the mark pass reads it."""
    rng = np.random.default_rng(29)
    n = 1 << 22
    x = (np.arange(n, dtype=np.int64) + 1000) * 3
    x[:: n // 65536] = rng.integers(0, 4, 65536)
    for keep in ("first", "last", "none"):
        got, prof = profiled(plb, lambda: plb.arg_unique(x, keep))
        assert np.array_equal(got, uo.np_arg_unique([(x, None)], keep)), keep
        assert prof.get("k5_table_init", 0) >= 2, prof
    check(plb, [x], [(x, None)])


def test_launch_profile(plb):
    rng = np.random.default_rng(31)
    x = rng.integers(0, 1000, 100_000)
    x[:10] = 10**6 + np.arange(10)      # keys of their own: every keep strategy keeps rows
    for kind, fn in mask_fns(plb).items():
        _, prof = profiled(plb, lambda: fn(x))
        assert prof.get("uniq_mark", 0) == 1 and prof.get("uniq_last", 0) == (kind == "last"), (kind, prof)
    for keep in ("first", "last", "any", "none"):
        _, prof = profiled(plb, lambda: plb.arg_unique(x, keep))
        assert prof.get("uniq_mark", 0) == 1 and prof.get("uniq_last", 0) == (keep == "last"), (keep, prof)
        assert prof.get("mask_rows", 0) == 1


# ------------------------------------------------------------------------------------------------ device paths
def test_device_inputs_and_outputs(plb):
    rng = np.random.default_rng(37)
    n = 200_001
    x = rng.integers(-50, 50, n)
    valid = rng.random(n) < 0.9
    d = plb.to_device(x, valid)
    m = uo.np_masks([(x, valid)])
    for keep in ("first", "last", "none"):
        out = plb.arg_unique(d, keep, location=plb.DEVICE)
        (ids, _), = plb.gather([plb.to_device(np.arange(n, dtype=np.int64))], out, check_bounds=True)
        assert np.array_equal(ids, np.flatnonzero(m[KEEP_KIND[keep]]))
    out = plb.is_duplicated(d, location=plb.DEVICE)
    got, _ = out.to_numpy()
    assert np.array_equal(got, m["duplicated"])


def test_unique_payloads(plb):
    rng = np.random.default_rng(41)
    n = 100_000
    k = rng.integers(0, 500, n).astype(np.int32)
    f = rng.normal(size=n)
    fv = rng.random(n) < 0.9
    words = ["w%d" % i for i in range(300)] + [None, ""]
    s = [words[i] for i in rng.integers(0, len(words), n)]
    for keep in ("first", "last", "any", "none"):
        ids = uo.np_arg_unique([(k, None)], keep)
        (gk, _), (gf, gfv), gs = plb.unique([k, (f, fv), plb.StringColumn(s)], subset=[0], keep=keep)
        assert np.array_equal(gk, k[ids]) and np.array_equal(gf.view(np.uint64), f[ids].view(np.uint64))
        assert np.array_equal(np.ones(ids.size, bool) if gfv is None else gfv, fv[ids])
        assert gs == [None if s[i] is None else s[i].encode() for i in ids]
        # subset None: every column is the key, strings included
        ids2 = uo.np_arg_unique([(k, None), (s, None)], keep)
        (gk2, _), gs2 = plb.unique([k, plb.StringColumn(s)], keep=keep)
        assert np.array_equal(gk2, k[ids2]) and gs2 == [None if s[i] is None else s[i].encode() for i in ids2]
    d = plb.unique([plb.to_device(k)], keep="last", location=plb.DEVICE)[0]
    assert np.array_equal(d.to_numpy()[0], k[uo.np_arg_unique([(k, None)], "last")])


# ------------------------------------------------------------------------------------------------ C ABI errors
def test_header_errors(plb):
    L = plb.lib()
    x = np.arange(10, dtype=np.int64)
    st = plb.Column(x).struct()
    out = plb.BlColumn()

    def call(keys, keep=0, mask=False, out_ptr=True):
        arr = (plb.BlSortKey * max(len(keys), 1))(*keys)
        fn = L.bl_unique_mask if mask else L.bl_unique
        return fn(arr if keys else None, C.c_int32(len(keys)), C.c_int32(keep), C.c_int32(plb.HOST), C.byref(out) if out_ptr else None)

    key = plb.BlSortKey(C.pointer(st), None, 0, 0)
    for mask in (False, True):
        assert call([key], -1, mask) == INVALID
        assert call([key], 4, mask) == INVALID
        assert call([], 0, mask) == INVALID
        assert call([key], 0, mask, out_ptr=False) == INVALID
        short = plb.Column(x[:5]).struct()
        assert call([key, plb.BlSortKey(C.pointer(short), None, 0, 0)], 0, mask) == INVALID
        assert call([plb.BlSortKey(None, None, 0, 0)], 0, mask) == INVALID
        sst = plb.StringColumn(["a"] * 10).struct()
        assert call([plb.BlSortKey(C.pointer(st), C.pointer(sst), 1, 0)], 0, mask) == INVALID
        assert call([plb.BlSortKey(None, C.pointer(sst), 0, 0)], 0, mask) == INVALID      # a string key without chunks
        assert call([plb.BlSortKey(C.pointer(st), None, 0, 1)], 0, mask) == INVALID       # flags != 0
        bad = plb.Column(x).struct()
        bad.dtype = 77
        assert call([plb.BlSortKey(C.pointer(bad), None, 0, 0)], 0, mask) == UNSUPPORTED
        big = plb.BlColumn()
        C.memmove(C.byref(big), C.byref(st), C.sizeof(st))
        big.length = (1 << 32) - 1
        assert call([plb.BlSortKey(C.pointer(big), None, 0, 0)], 0, mask) == UNSUPPORTED      # before any upload
        empty = plb.Column(x[:0]).struct()
        assert call([plb.BlSortKey(C.pointer(empty), None, 0, 0)], 1, mask) == 0 and out.length == 0


# ------------------------------------------------------------------------------------------------ plugin ABI
def test_plugin_entries(plb):
    import pyarrow as pa
    from test_gpu_plugin_abi import Caller
    caller = Caller(plb.lib())
    rng = np.random.default_rng(43)
    n = 5000
    a = rng.integers(0, 30, n)
    am = rng.random(n) < 0.1
    b = rng.integers(0, 2, n).astype(bool)
    A, B = pa.array(a, mask=am), pa.array(b)
    cols = [(a, ~am), (b, None)]
    m = uo.np_masks(cols)
    for keep in ("first", "last", "any", "none", None):
        out = caller.call("arg_unique", [("a", [A.slice(0, 1000), A.slice(1000)]), ("b", [B])], kwargs={"keep": keep} if keep else None)
        assert out.type == pa.uint32()
        assert out.to_pylist() == np.flatnonzero(m[KEEP_KIND[keep or "first"]]).tolist(), keep
    for name, kind in (("is_unique", "unique"), ("is_duplicated", "duplicated"), ("is_first_distinct", "first"), ("is_last_distinct", "last")):
        out = caller.call(name, [("a", [A]), ("b", [B])])
        assert out.type == pa.bool_() and out.null_count == 0
        assert out.to_pylist() == m[kind].tolist(), name
    with pytest.raises(RuntimeError, match=r"`keep` must be one of \{'first', 'last', 'any', 'none'\}, got fist"):
        caller.call("arg_unique", [("a", [A])], kwargs={"keep": "fist"})
