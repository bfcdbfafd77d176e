"""GPU tests of rank (bl_rank).  Every method is compared byte for byte with tests/rank_oracle.py (its pure-Python rule for
small inputs, its numpy restatement for large ones), AVERAGE included, and RANDOM against the oracle's copy of the tie key
as well as by its contract: a permutation of each run, the same bytes for the same seed, and a chi-square test of its
uniformity.  Sizes derive from sm_count so that the grid-stride loops of the three rank kernels take several tiles of
2048 positions per CTA."""
import ctypes as C
import os

import numpy as np
import pytest

import rank_oracle as ro

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE = 2048
INTS = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64"]
KINDS = INTS + ["float32", "float64", "bool"]


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as plb
    plb.init()
    return plb


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


def expected(exp, method):
    """oracle list (None = null) -> (values with 0 in null slots, validity or None) as the device returns them"""
    dt = np.float64 if method == "average" else np.uint32
    vals = np.array([0 if e is None else e for e in exp], dt)
    valid = np.array([e is not None for e in exp], bool)
    return vals, (None if valid.all() else valid)


def assert_same(got, exp, what=""):
    gv, gm = got
    ev, em = exp
    assert gv.dtype == ev.dtype, what
    assert gv.tobytes() == ev.tobytes(), (what, gv[:20], ev[:20])
    assert (gm is None and em is None) or (gm is not None and em is not None and np.array_equal(gm, em)), what


def pylist(x, valid):
    if x.dtype.kind == "f":
        out = [float(v) for v in x.tolist()]
    elif x.dtype.kind == "b":
        out = [bool(v) for v in x.tolist()]
    else:
        out = [int(v) for v in x.tolist()]
    return out if valid is None else [v if ok else None for v, ok in zip(out, valid)]


def extremes(rng, dtype, n):
    if dtype == "bool":
        return rng.random(n) < 0.5
    if dtype.startswith("float"):
        ft = np.dtype(dtype)
        it = np.uint32 if ft.itemsize == 4 else np.uint64
        info = np.finfo(ft)
        pool = np.array([0.0, -0.0, np.inf, -np.inf, info.max, -info.max, info.tiny, -info.tiny, info.smallest_subnormal,
                         -info.smallest_subnormal, 1.5, -1.5, 3.0], ft)
        x = rng.choice(pool, n)
        # NaNs with payloads and either sign: every one is the same value
        nan_bits = (np.array([0x7FC00000, 0xFFC00001, 0x7F800001, 0xFFFFFFFF], np.uint32) if ft.itemsize == 4 else
                    np.array([0x7FF8000000000000, 0xFFF8000000000001, 0x7FF0000000000001, 0xFFFFFFFFFFFFFFFF], np.uint64))
        at = rng.random(n) < 0.1
        x[at] = rng.choice(nan_bits, int(at.sum())).astype(it).view(ft)
        return x
    info = np.iinfo(dtype)
    pool = np.array([info.min, info.min + 1, 0, 1, info.max // 2, info.max - 1, info.max], dtype)
    return rng.choice(pool, n)


def run1(plb, col, method, descending=False, seed=0, **kw):
    return plb.rank([(col, {"method": method, "descending": descending, "seed": seed})], **kw)[0]


# ------------------------------------------------------------------------------------------------ known answers
def test_known_answers(plb):
    import json
    kats = json.load(open(os.path.join(ROOT, "tests", "golden", "rank_kats.json")))
    np_dt = {"int32": np.int32, "int64": np.int64, "uint32": np.uint32, "float64": np.float64}
    for c in kats:
        vals = c["values"]
        valid = np.array([v is not None for v in vals], bool)
        if c["dtype"] == "str":
            col = plb.StringColumn(vals)
        else:
            col = (np.array([0 if v is None else v for v in vals], np_dt[c["dtype"]]), valid)
        parts = ()
        if c["parts"] is not None:
            parts = [plb.StringColumn(c["parts"]) if isinstance(c["parts"][0], str) else np.array(c["parts"], np.int64)]
        got = plb.rank([(col, {"method": c["method"], "descending": c["descending"], "seed": 1})], partition_by=parts)[0]
        if c["expected"] is not None:
            assert_same(got, expected(c["expected"], c["method"]), c["src"])
        else:
            for rows, total in c["random_runs"]:
                assert int(got[0][rows].sum()) == total and len(set(got[0][rows].tolist())) == len(rows), c["src"]


# ------------------------------------------------------------------------------------------------ dtypes and methods
@pytest.mark.parametrize("method", ro.METHODS)
@pytest.mark.parametrize("dtype", KINDS)
def test_every_dtype_at_its_extremes(plb, sm, dtype, method):
    rng = np.random.default_rng(KINDS.index(dtype) * 10 + ro.METHODS.index(method))
    n = 3 * TILE + 17
    x = extremes(rng, dtype, n)
    valid = rng.random(n) >= 0.15
    for desc in (False, True):
        seed = int(rng.integers(0, 2**63))
        got = run1(plb, (x, valid), method, desc, seed)
        exp = ro.rank(pylist(x, valid), method, desc, seed=seed)
        assert_same(got, expected(exp, method), (dtype, method, desc))


@pytest.mark.parametrize("method", ro.METHODS)
def test_strings_and_binary(plb, method):
    rng = np.random.default_rng(3)
    pool = [b"", b"\x00", b"\x00\x00", b"\xff", b"\xff\x00", b"a", b"ab", b"abc", b"abcdefghijklmnop", b"abcdefghijklmnoq",
            b"abcdefghijklmno", "é".encode(), b"b"]
    n = 2 * TILE + 5
    vals = [None if rng.random() < 0.1 else pool[int(rng.integers(0, len(pool)))] for _ in range(n)]
    g = rng.integers(0, 4, n)
    for desc in (False, True):
        for parts in (None, g):
            got = plb.rank([(plb.StringColumn(vals), {"method": method, "descending": desc, "seed": 9})],
                           partition_by=() if parts is None else [parts])[0]
            exp = ro.rank(vals, method, desc, None if parts is None else g.tolist(), seed=9)
            assert_same(got, expected(exp, method), (method, desc, parts is None))
    # chunked and on the device: the same answer
    sc = [plb.StringColumn(vals[:1000]), plb.StringColumn(vals[1000:])]
    got = plb.rank([(sc, {"method": method, "seed": 9})])[0]
    assert_same(got, expected(ro.rank(vals, method, seed=9), method), "chunks")
    dev = plb.DeviceStringColumn(plb.StringColumn(vals))
    assert_same(plb.rank([(dev, {"method": method, "seed": 9})])[0], expected(ro.rank(vals, method, seed=9), method), "device")


@pytest.mark.parametrize("method", ro.METHODS)
def test_null_patterns(plb, method):
    rng = np.random.default_rng(11)
    n = TILE + 100
    x = rng.integers(0, 50, n).astype(np.int64)
    g = rng.integers(0, 5, n)
    allnull_part = g == 3
    for valid in (None, rng.random(n) >= 0.3, np.zeros(n, bool), ~allnull_part):
        got = plb.rank([((x, valid), {"method": method, "seed": 4})], partition_by=[g])[0]
        exp = ro.rank(pylist(x, valid), method, parts=g.tolist(), seed=4)
        assert_same(got, expected(exp, method), method)
        got = plb.rank([((x, valid), {"method": method, "seed": 4})])[0]
        assert_same(got, expected(ro.rank(pylist(x, valid), method, seed=4), method), method)


@pytest.mark.parametrize("n", [0, 1, 2])
@pytest.mark.parametrize("method", ro.METHODS)
def test_tiny_columns(plb, n, method):
    for valid in (None, np.zeros(n, bool), np.arange(n) == 0):
        x = np.array([7, 7][:n], np.int32)
        got = plb.rank([((x, valid), {"method": method, "seed": 1})], partition_by=[np.arange(n, dtype=np.int64)])[0]
        assert_same(got, expected(ro.rank(pylist(x, valid), method, parts=list(range(n)), seed=1), method), (n, method))
        got = plb.rank_column((x, valid), method, seed=1)
        assert_same(got, expected(ro.rank(pylist(x, valid), method, seed=1), method), (n, method))
    out = plb.rank_column(np.zeros(0, np.float32), method)
    assert out[0].dtype == (np.float64 if method == "average" else np.uint32) and out[0].size == 0


# ------------------------------------------------------------------------------------------------ partitions and order_by
@pytest.mark.parametrize("method", ro.METHODS)
def test_partition_shapes(plb, method):
    rng = np.random.default_rng(21)
    n = 4 * TILE + 3
    x = rng.integers(-3, 4, n).astype(np.int64)
    valid = rng.random(n) >= 0.1
    shapes = {
        "one_row_each": np.arange(n, dtype=np.int64),
        "few_large": rng.integers(0, 3, n).astype(np.int64),
        "sorted_blocks": np.repeat(np.arange(7), n // 7 + 1)[:n].astype(np.int32),
    }
    for name, g in shapes.items():
        got = plb.rank([((x, valid), {"method": method, "seed": 5})], partition_by=[g])[0]
        exp = ro.rank(pylist(x, valid), method, parts=g.tolist(), seed=5)
        assert_same(got, expected(exp, method), name)
    # a null partition key is its own partition; string keys; two key columns
    gk = rng.integers(0, 4, n)
    gvalid = rng.random(n) >= 0.2
    got = plb.rank([((x, valid), {"method": method, "seed": 5})], partition_by=[(gk, gvalid)])[0]
    labels = [int(k) if ok else None for k, ok in zip(gk, gvalid)]
    assert_same(got, expected(ro.rank(pylist(x, valid), method, parts=labels, seed=5), method), "null key")
    sk = [None if rng.random() < 0.1 else ["", "a", "ab", "\x00"][int(k)] for k in gk]
    g2 = rng.integers(0, 2, n).astype(np.int8)
    got = plb.rank([((x, valid), {"method": method, "seed": 5})], partition_by=[plb.StringColumn(sk), g2])[0]
    labels = list(zip(sk, g2.tolist()))
    assert_same(got, expected(ro.rank(pylist(x, valid), method, parts=labels, seed=5), method), "string keys")


@pytest.mark.parametrize("flags", [(False, False), (True, False), (False, True), (True, True)])
def test_order_by_breaks_ordinal_ties(plb, flags):
    desc_o, nl = flags
    rng = np.random.default_rng(31)
    n = 3 * TILE + 9
    x = rng.integers(0, 6, n).astype(np.int64)
    valid = rng.random(n) >= 0.1
    g = rng.integers(0, 9, n)
    ok = rng.integers(-5, 5, n).astype(np.int64)
    ovalid = rng.random(n) >= 0.1
    okeys = pylist(ok, ovalid)
    pos = ro.order_ranks(okeys, desc_o, nl)
    for desc in (False, True):
        for parts in ((), [g]):
            labels = g.tolist() if parts else None
            res = plb.rank([((x, valid), {"method": m, "descending": desc, "seed": 2}) for m in ro.METHODS], partition_by=parts,
                           order_by=(ok, ovalid), descending=desc_o, nulls_last=nl)
            for m, got in zip(ro.METHODS, res):
                exp = ro.rank(pylist(x, valid), m, desc, labels, order=pos if m == "ordinal" else None, seed=2)
                assert_same(got, expected(exp, m), (m, desc, bool(parts), flags))
    # a string order_by key
    sk = [None if not o else ["b", "", "a\x00", "a", "\xff"][int(v) % 5] for v, o in zip(ok, ovalid)]
    spos = ro.order_ranks([None if s is None else s.encode() for s in sk], desc_o, nl)
    got = plb.rank([((x, valid), {"method": "ordinal"})], partition_by=[g], order_by=plb.StringColumn(sk), descending=desc_o, nulls_last=nl)[0]
    assert_same(got, expected(ro.rank(pylist(x, valid), "ordinal", parts=g.tolist(), order=spos), "ordinal"), "string order_by")


# ------------------------------------------------------------------------------------------------ sizes and long runs
@pytest.mark.parametrize("method", ro.METHODS)
def test_sizes_around_the_tile_and_past_the_grid(plb, sm, method):
    rng = np.random.default_rng(41)
    grid_tiles = sm * 8
    for n in (31, 32, 33, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, grid_tiles * TILE - 1, grid_tiles * TILE + 1, 2 * grid_tiles * TILE + TILE + 5):
        x = rng.integers(0, max(n // 3, 2), n).astype(np.int32)
        valid = rng.random(n) >= 0.05
        seed = int(rng.integers(0, 2**63))
        tie = np.array([ro.random_key(r, seed) for r in range(n)], np.int64) if method == "random" and n < 100_000 else None
        if method == "random" and tie is None:
            r = np.arange(n, dtype=np.uint64)
            tie = _random_keys_np(r, seed)
        got = run1(plb, (x, valid), method, False, seed)
        exp = ro.rank_np(x, valid, method, False, None, tie)
        assert_same(got, (exp[0], None if exp[1].all() else exp[1]), (n, method))
        if n > 100_000:
            g = rng.integers(0, n // 50, n)
            got = plb.rank([((x, valid), {"method": method, "seed": seed})], partition_by=[g])[0]
            exp = ro.rank_np(x, valid, method, False, g, tie)
            assert_same(got, (exp[0], None if exp[1].all() else exp[1]), (n, method, "partitioned"))


def _random_keys_np(r, seed):
    def fmix(h):
        h = h ^ (h >> np.uint64(16)); h = (h * np.uint64(0x85EBCA6B)) & np.uint64(0xFFFFFFFF)
        h = h ^ (h >> np.uint64(13)); h = (h * np.uint64(0xC2B2AE35)) & np.uint64(0xFFFFFFFF)
        return h ^ (h >> np.uint64(16))
    lo, hi = np.uint64(seed & 0xFFFFFFFF), np.uint64(seed >> 32)
    return fmix((fmix((r & np.uint64(0xFFFFFFFF)) ^ lo) + hi) & np.uint64(0xFFFFFFFF)).astype(np.int64)


def test_random_keys_np_matches_oracle():
    seed = 0xDEADBEEF12345678
    assert _random_keys_np(np.arange(1000, dtype=np.uint64), seed).tolist() == [ro.random_key(r, seed) for r in range(1000)]


@pytest.mark.parametrize("method", ro.METHODS)
def test_one_run_across_many_tiles_and_alternating_runs(plb, method):
    n = 4_000_003
    x = np.full(n, 5, np.int64)
    vals, valid = run1(plb, x, method, seed=3)
    assert valid is None
    if method == "average":
        assert np.all(vals == 0.5 * (1 + n))
    elif method in ("min", "dense"):
        assert np.all(vals == 1)
    elif method == "max":
        assert np.all(vals == n)
    elif method == "ordinal":
        assert np.array_equal(vals, np.arange(1, n + 1, dtype=np.uint32))
    else:
        assert np.array_equal(np.sort(vals), np.arange(1, n + 1, dtype=np.uint32))
    alt = (np.arange(n) % 2).astype(np.uint8)
    got = run1(plb, alt, method, seed=3)
    tie = _random_keys_np(np.arange(n, dtype=np.uint64), 3) if method == "random" else None
    exp = ro.rank_np(alt, None, method, False, None, tie)
    assert_same(got, (exp[0], None), method)


# ------------------------------------------------------------------------------------------------ call forms
def test_device_output_and_several_ops(plb):
    rng = np.random.default_rng(51)
    n = 5 * TILE + 1
    x = rng.normal(size=n).round(1)
    valid = rng.random(n) >= 0.1
    g = rng.integers(0, 30, n)
    ops = [((x, valid), {"method": m, "descending": d, "seed": 77}) for m in ro.METHODS for d in (False, True)]
    together = plb.rank(ops, partition_by=[g])
    for op, got in zip(ops, together):
        alone = plb.rank([op], partition_by=[g])[0]
        assert_same(got, alone, op[1])
        dev = plb.rank([op], partition_by=[g], location=plb.DEVICE)[0]
        assert dev.location == plb.DEVICE
        assert_same(dev.to_numpy(), alone, op[1])
    # device-resident inputs
    xd = plb.to_device(x, valid)
    assert_same(plb.rank([(xd, {"method": "dense"})])[0], expected(ro.rank(pylist(x, valid), "dense"), "dense"), "device input")


# ------------------------------------------------------------------------------------------------ RANDOM
def test_random_contract(plb):
    rng = np.random.default_rng(61)
    n = 50_000
    x = rng.integers(0, 100, n).astype(np.int64)
    a = run1(plb, x, "random", seed=123)[0]
    b = run1(plb, x, "random", seed=123)[0]
    c = run1(plb, x, "random", seed=124)[0]
    assert a.tobytes() == b.tobytes() and a.tobytes() != c.tobytes()
    mn = run1(plb, x, "min")[0].astype(np.int64)
    mx = run1(plb, x, "max")[0].astype(np.int64)
    for v in np.unique(x):
        rows = x == v
        assert np.array_equal(np.sort(a[rows]), np.arange(mn[rows][0], mx[rows][0] + 1))
    # a drawn seed gives a valid answer too
    d = plb.rank_column(x, "random")[0]
    assert np.array_equal(np.sort(d), np.sort(a))


def test_random_is_uniform(plb):
    from scipy.stats import chisquare
    m = 60_000
    x = np.zeros(3 * m, np.int64)
    g = np.repeat(np.arange(m), 3)
    r = plb.rank([(x, {"method": "random", "seed": 2024})], partition_by=[g])[0][0].reshape(m, 3).astype(np.int64)
    assert np.array_equal(np.sort(r, axis=1), np.tile([1, 2, 3], (m, 1)))
    code = r[:, 0] * 9 + r[:, 1] * 3 + r[:, 2]
    _, counts = np.unique(code, return_counts=True)
    assert counts.size == 6
    assert chisquare(counts).pvalue > 1e-4, counts


# ------------------------------------------------------------------------------------------------ errors
def test_header_errors(plb):
    L = plb.lib()
    x = np.arange(10, dtype=np.int64)
    col = plb.Column(x)
    st = col.struct()
    key = plb.BlSortKey(C.pointer(st), None, 0, 0)
    outs = (plb.BlColumn * 2)()

    def call(ops, parts=None, n_parts=0, order=None):
        arr = (plb.BlRankOp * len(ops))(*ops)
        return L.bl_rank(parts, C.c_int32(n_parts), order, arr, C.c_int32(len(ops)), C.c_int32(plb.HOST), outs)

    INVALID, UNSUPPORTED = 1, 4
    assert call([plb.BlRankOp(6, 0, 0, C.pointer(key))]) == INVALID
    assert call([plb.BlRankOp(-1, 0, 0, C.pointer(key))]) == INVALID
    assert call([plb.BlRankOp(0, 0, 0, None)]) == INVALID
    bad = plb.BlSortKey(C.pointer(st), None, 0, 1)
    assert call([plb.BlRankOp(0, 0, 0, C.pointer(bad))]) == INVALID
    neither = plb.BlSortKey(None, None, 0, 0)
    assert call([plb.BlRankOp(0, 0, 0, C.pointer(neither))]) == INVALID
    short = plb.Column(x[:5]).struct()
    skey = plb.BlSortKey(C.pointer(short), None, 0, 0)
    assert call([plb.BlRankOp(0, 0, 0, C.pointer(key)), plb.BlRankOp(0, 0, 0, C.pointer(skey))]) == INVALID
    assert call([plb.BlRankOp(0, 0, 0, C.pointer(key))], (plb.BlSortKey * 1)(skey), 1) == INVALID      # partition length
    assert call([plb.BlRankOp(0, 0, 0, C.pointer(key))], (plb.BlSortKey * 1)(bad), 1) == INVALID       # partition flags
    assert call([plb.BlRankOp(0, 0, 0, C.pointer(key))], None, 1) == INVALID
    bst = plb.Column(np.ones(10, bool)).struct()
    bkey = plb.BlSortKey(C.pointer(bst), None, 0, 0)
    assert call([plb.BlRankOp(0, 0, 0, C.pointer(key))], (plb.BlSortKey * 1)(bkey), 1) == UNSUPPORTED
    okey = plb.BlSortKey(C.pointer(st), None, 0, 4)
    assert call([plb.BlRankOp(4, 0, 0, C.pointer(key))], None, 0, C.pointer(okey)) == INVALID          # order_by flags
    with pytest.raises(plb.B200Error, match="UNSUPPORTED"):
        plb.rank([(x, {})], partition_by=[np.ones(10, bool)])
    # more rows than the row limits: a length-only descriptor is rejected before anything is read
    big = plb.BlColumn(3, plb.HOST, 2**32, 0, 0, st.values, None, None)
    bigkey = plb.BlSortKey(C.pointer(big), None, 0, 0)
    assert call([plb.BlRankOp(0, 0, 0, C.pointer(bigkey))]) == UNSUPPORTED
    big31 = plb.BlColumn(3, plb.HOST, 2**31, 0, 0, st.values, None, None)
    b31key = plb.BlSortKey(C.pointer(big31), None, 0, 0)
    assert call([plb.BlRankOp(4, 0, 0, C.pointer(b31key))], (plb.BlSortKey * 1)(b31key), 1) == UNSUPPORTED


# ------------------------------------------------------------------------------------------------ plugin ABI
def test_plugin_entries(plb):
    import pyarrow as pa
    from test_gpu_plugin_abi import Caller
    caller = Caller(plb.lib())
    rng = np.random.default_rng(71)
    n = 3000
    x = rng.integers(0, 20, n)
    xm = rng.random(n) < 0.1
    g = rng.integers(0, 7, n)
    X = pa.array(x, mask=xm)
    vals = [None if m else int(v) for v, m in zip(x, xm)]
    for m in ro.METHODS:
        for desc in (False, True):
            kw = {"descending": desc, "seed": 99}
            out = caller.call(f"rank_{m}", [("x", [X.slice(0, 1000), X.slice(1000)]), ("g", [pa.array(g)])], kwargs=kw)
            exp = ro.rank(vals, m, desc, g.tolist(), seed=99)
            assert out.type == (pa.float64() if m == "average" else pa.uint32())
            assert out.to_pylist() == exp, (m, desc)
            out = caller.call(f"rank_{m}", [("x", [X])], kwargs=kw)
            assert out.to_pylist() == ro.rank(vals, m, desc, seed=99), (m, desc)
    out = caller.call("rank_random", [("x", [X])])      # a drawn seed
    assert sorted(v for v in out.to_pylist() if v is not None) == sorted(v for v in ro.rank(vals, "ordinal") if v is not None)
    with pytest.raises(RuntimeError, match="seed"):
        caller.call("rank_random", [("x", [X])], kwargs={"seed": 1.5})
