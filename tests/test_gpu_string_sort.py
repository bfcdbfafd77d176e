"""GPU tests of sorting by string keys (bl_arg_sort_keys, bl_string_rank): every permutation and rank is compared bit for
bit with the oracle (tests/sort_oracle.py, the dense rank of test_string_sort.py) over the reference's known answers, the
byte-order edge cases, the column shapes, sliced and chunked inputs, mixed keys and flags, and 2e7 rows."""
import numpy as np
import pytest

import sort_oracle
from test_string_sort import as_bytes, check_sorted_frame, dense_rank, edge_strings, kat_frame, string_sort_kats

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as plb
    plb.init()
    return plb


def oracle_sort(cols, descending=False, nulls_last=False, limit=None):
    """cols: bytes / None lists or (numpy, valid) pairs"""
    vals, valids = [], []
    for c in cols:
        if isinstance(c, tuple):
            vals.append(c[0]); valids.append(c[1])
        else:
            vals.append(c); valids.append(None)
    return sort_oracle.arg_sort(vals, valids, descending, nulls_last, limit)


def numpy_sort(cols, descending=False, nulls_last=False, limit=None):
    """the same order from np.lexsort; string columns become object arrays with a validity"""
    vals, valids = [], []
    for c in cols:
        if isinstance(c, tuple):
            vals.append(c[0]); valids.append(c[1])
        else:
            valids.append(np.array([v is not None for v in c], bool))
            vals.append(np.array([b"" if v is None else v for v in c] + [b""], dtype=object)[:-1])
    return sort_oracle.numpy_arg_sort(vals, valids, descending, nulls_last, limit)


def to_key(plb, c):
    return plb.StringColumn(c) if isinstance(c, list) else c


def check_all_flags(plb, vals, desc_list=(False, True), nl_list=(False, True), big=False):
    s = plb.StringColumn(vals)
    for desc in desc_list:
        for nl in nl_list:
            got = plb.arg_sort([s], desc, nl)
            exp = numpy_sort([vals], desc, nl) if big else oracle_sort([vals], desc, nl)
            assert np.array_equal(got, exp), (len(vals), desc, nl)
    if vals:
        for desc in (False, True):
            (r, valid), nd = plb.string_rank(s, desc)
            exp = dense_rank(vals, desc)
            got = [None if (valid is not None and not valid[i]) else int(r[i]) for i in range(len(vals))]
            assert got == exp and nd == len({v for v in vals if v is not None}), (len(vals), desc)


@pytest.mark.parametrize("case", string_sort_kats(), ids=lambda c: c["cite"][-60:])
def test_reference_kats(plb, case):
    frame = kat_frame(case)
    by = [plb.StringColumn(frame[b][0]) if frame[b][2] == "str" else ((frame[b][0], frame[b][1]) if frame[b][1] is not None else frame[b][0]) for b in case["by"]]
    idx = plb.arg_sort(by, case["descending"], case["nulls_last"])
    check_sorted_frame(frame, idx, case["expect"])


def test_byte_order_edge_cases(plb):
    rng = np.random.default_rng(1)
    pool = edge_strings()
    check_all_flags(plb, pool)
    check_all_flags(plb, pool[::-1] + [None] + pool)
    vals = [pool[i] if rng.random() > 0.1 else None for i in rng.integers(0, len(pool), 3000)]
    check_all_flags(plb, vals)


def test_every_length_around_the_chunk_boundaries(plb):
    """every length 0-64 of several fill bytes, so strings end at each position of a 7-byte chunk and continue past it"""
    vals = [bytes([f]) * k for f in (0x00, 0x41, 0x7F, 0x80, 0xFF) for k in range(65)]
    vals += [b"p" * k + bytes([f]) for f in (0x00, 0xFF) for k in range(65)]
    rng = np.random.default_rng(2)
    check_all_flags(plb, [vals[i] for i in rng.permutation(len(vals))])


def test_long_shared_prefix(plb):
    rng = np.random.default_rng(3)
    prefix = bytes(rng.integers(0, 256, 2048, dtype=np.uint8))
    tails = [bytes(rng.integers(0, 256, int(k), dtype=np.uint8)) for k in rng.integers(0, 12, 1000)]
    vals = [prefix + t for t in tails] + [prefix[:100], prefix]
    check_all_flags(plb, vals)


def test_column_shapes(plb):
    rng = np.random.default_rng(4)
    check_all_flags(plb, [b"same"] * 5000)
    check_all_flags(plb, [b"%08d" % i for i in rng.permutation(5000)])
    check_all_flags(plb, [None] * 100)
    check_all_flags(plb, [b"x"])
    check_all_flags(plb, [None])
    assert plb.arg_sort([plb.StringColumn([])]).size == 0
    (r, _), nd = plb.string_rank(plb.StringColumn([None] * 70))
    assert nd == 0
    _, nd = plb.string_rank(plb.StringColumn([]))
    assert nd == 0


def test_sliced_and_chunked_inputs(plb):
    rng = np.random.default_rng(5)
    pool = edge_strings()
    full = [pool[i] if rng.random() > 0.2 else None for i in rng.integers(0, len(pool), 300)]
    for off in (0, 1, 3, 31, 33):
        for ln in (0, 1, 100, 300 - 33):
            sl = full[off:off + ln]
            s = plb.StringColumn(full, offset=off, length=len(sl))
            for desc in (False, True):
                for nl in (False, True):
                    assert np.array_equal(plb.arg_sort([s], desc, nl), oracle_sort([sl], desc, nl)), (off, ln, desc, nl)
            (r, v), nd = plb.string_rank(s)
            assert [None if (v is not None and not v[i]) else int(r[i]) for i in range(len(sl))] == dense_rank(sl)
    # chunks, two of them sliced, one without nulls
    parts = [(full, 7, 50), ([b"zz", b"a"], 0, 2), (full, 101, 99)]
    chunks = [plb.StringColumn(c, offset=o, length=ln) for c, o, ln in parts]
    cat = sum((c[o:o + ln] for c, o, ln in parts), [])
    for desc in (False, True):
        for nl in (False, True):
            assert np.array_equal(plb.arg_sort([chunks], desc, nl), oracle_sort([cat], desc, nl))
    dev = plb.DeviceStringColumn(chunks)
    assert np.array_equal(plb.arg_sort([dev], True, True), oracle_sort([cat], True, True))


@pytest.mark.parametrize("k", [2, 3])
def test_mixed_keys_flags_and_limit(plb, k):
    rng = np.random.default_rng(10 + k)
    words = [b"", b"a", b"ab", b"b", b"\xff", None]
    for n in (7, 1000, 50_000):
        for trial in range(4):
            cols = [[words[i] for i in rng.integers(0, len(words), n)]]
            kinds = ["int64", "float64", "bool", "str"]
            for _ in range(k - 1):
                kind = kinds[rng.integers(0, 4)]
                valid = rng.random(n) > 0.1
                if kind == "str":
                    cols.append([words[i] for i in rng.integers(0, len(words), n)])
                elif kind == "bool":
                    cols.append((rng.random(n) < 0.5, valid))
                elif kind == "int64":
                    cols.append((rng.integers(-3, 3, n).astype(np.int64), valid))
                else:
                    cols.append((rng.choice(np.array([0.0, -0.0, np.nan, 1.5, -np.inf]), n), valid))
            order = rng.permutation(k)
            cols = [cols[i] for i in order]
            desc = [bool(x) for x in rng.random(k) < 0.5]
            nl = [bool(x) for x in rng.random(k) < 0.5]
            limit = [None, 0, 5, n // 2][trial]
            got = plb.arg_sort([to_key(plb, c) for c in cols], desc, nl, limit)
            exp = numpy_sort(cols, desc, nl, limit) if n > 2000 else oracle_sort(cols, desc, nl, limit)
            assert np.array_equal(got, exp), (n, trial, desc, nl, limit)


def test_ties_keep_row_order(plb):
    vals = [b"b", b"a", b"b", None, b"a", None, b"b"]
    assert plb.arg_sort([plb.StringColumn(vals)]).tolist() == [3, 5, 1, 4, 0, 2, 6]
    assert plb.arg_sort([plb.StringColumn(vals)], True, True).tolist() == [0, 2, 6, 1, 4, 3, 5]


def test_sort_payloads_and_string_gather(plb):
    rng = np.random.default_rng(6)
    n = 10_000
    key = [b"k%03d" % i if i % 17 else None for i in rng.integers(0, 300, n)]
    x, xv = rng.integers(-100, 100, n).astype(np.int64), rng.random(n) > 0.1
    f = rng.normal(size=n)
    s = plb.StringColumn(key)
    for limit in (None, 10):
        perm = numpy_sort([key], True, False, limit)
        (gx, gxv), (gf, _) = plb.sort([s], [(x, xv), f], True, False, limit)
        assert np.array_equal(gxv, xv[perm]) and np.array_equal(gx[gxv], x[perm][xv[perm]]) and np.array_equal(gf, f[perm])
        idx = plb.arg_sort([s], True, False, limit, location=plb.DEVICE)
        assert plb.string_gather(s, idx) == [key[i] for i in perm]


def test_device_inputs_and_outputs(plb):
    rng = np.random.default_rng(7)
    vals = [b"v%d" % i if i % 5 else None for i in rng.integers(0, 500, 20_000)]
    dev = plb.DeviceStringColumn(plb.StringColumn(vals))
    num = plb.to_device(rng.integers(0, 3, len(vals)).astype(np.int64))
    out = plb.arg_sort([dev, num], [False, True], True, location=plb.DEVICE)
    assert out.location == plb.DEVICE
    exp = numpy_sort([vals, (num.to_numpy()[0], None)], [False, True], True)
    assert np.array_equal(out.to_numpy()[0], exp)
    rk, nd = plb.string_rank(dev, True, location=plb.DEVICE)
    r, v = rk.to_numpy()
    assert [None if not v[i] else int(r[i]) for i in range(len(vals))] == dense_rank(vals, True) and nd == len({x for x in vals if x is not None})
    enc, nd2 = plb.string_encode(dev)
    assert nd2 == nd


def test_errors(plb):
    import ctypes as C
    a, b = plb.StringColumn([b"a", b"b"]), plb.StringColumn([b"a"])
    with pytest.raises(plb.B200Error, match="differ in length"):
        plb.arg_sort([a, b])
    with pytest.raises(plb.B200Error, match="differ in length"):
        plb.arg_sort([a, np.arange(3)])
    col = plb.Column(np.arange(2))
    st, sst = col.struct(), a.struct()
    out = plb.BlColumn()
    for d in (plb.BlSortKey(C.pointer(st), C.pointer(sst), 1, 0), plb.BlSortKey(None, None, 0, 0)):
        arr = (plb.BlSortKey * 1)(d)
        assert plb.lib().bl_arg_sort_keys(arr, C.c_int32(1), C.c_int64(-1), C.c_int32(plb.HOST), C.byref(out)) == 1
        assert b"exactly one" in plb.lib().bl_last_error()


def test_twenty_million_rows(plb):
    rng = np.random.default_rng(8)
    V, n = 1_000_000, 20_000_000
    lens = rng.integers(1, 16, V)
    offs = np.zeros(V + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    data = rng.integers(0x61, 0x65, int(offs[-1]), dtype=np.uint8)
    vocab = plb.StringColumn(offsets=offs, data=data)
    words = np.array([data[offs[i]:offs[i + 1]].tobytes() for i in range(V)] + [b""], dtype=object)[:-1]
    _, vrank = np.unique(words, return_inverse=True)
    idx, valid = rng.integers(0, V, n).astype(np.uint32), rng.random(n) >= 0.05
    dev = plb.string_gather(vocab, (idx, valid), location=plb.DEVICE)
    keys = vrank[idx].astype(np.int64)
    for desc, nl in ((False, False), (True, True)):
        got = plb.arg_sort([dev], desc, nl)
        assert np.array_equal(got, sort_oracle.numpy_arg_sort([keys], [valid], desc, nl)), (desc, nl)
    (r, v), nd = plb.string_rank(dev)
    assert nd == len(np.unique(vrank[idx[valid]]))
    dense = np.unique(vrank[idx[valid]], return_inverse=True)[1] + 1
    assert np.array_equal(v, valid) and np.array_equal(r[valid], dense)
