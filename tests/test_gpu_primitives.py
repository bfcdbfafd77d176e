"""GPU tests of the streaming kernels K1 (elementwise), K2 (compare), K3 (filter), K4 (gather) and K6 (hash partition)
against the numpy restatements in tests/primitives_ref.py, over the full value range of every dtype and past every grid
cap of the launch code.  Values and validity must match bit for bit (any NaN equals any NaN).

Sizes.  The caps are written for SM = device_info()["sm_count"] (132 on an H100 SXM):
  K1 k_arith          grid_for(n / VN / 4 + 1, 256): <= 8*SM CTAs of 256 threads, one 16-byte vector (VN elements) per
                      thread-step; the 4-deep unrolled loop covers every thread from n = 4 * 8*SM*256 * VN = 8192*SM*VN
                      (32768*SM rows for 4-byte types).  k_int_true_div grid-strides past 8*SM*256 = 2048*SM rows.
  K2 k_compare        grid_for(n / VN + 1, 256) -> <= 64*SM warps of 32*VN rows per step; the unrolled loop covers
                      every warp from n = 4 * 64*SM * 32*VN = 8192*SM*VN rows (32768*SM for 4-byte types).
     k_compare64      (8-byte scalar rhs) 64 rows per warp-step: from 4 * 64*SM * 64 = 16384*SM rows.
  K3 k_compact        min(tiles, 8*SM) CTAs of 4096-row tiles: the tile loop strides past 8*SM*4096 = 32768*SM rows.
     k_scan_u64       one CTA of 1024 threads: the carry between chunks runs past 1024 tiles = 4 194 304 rows.
     k_mask_tile_counts  grid_for(tiles * 128, 128, 16): one tile per CTA up to 16*SM CTAs, past 65536*SM rows.
  K4 k_gather         grid_for((m + 3) / 4, 256): 4 rows per thread, the grid-stride loop past 4 * 8*SM*256 = 8192*SM.
     G_MAX_COLS = 8   columns per launch: 11 columns take two batches.
  K6 k_part_scatter   min(tiles, 8*SM) CTAs of 2048-row tiles: the tile loop strides past 16384*SM rows; the cross-tile
                      cursor reservation runs from the second tile (2049 rows).
N_BIG = max(32768*SM, 1024*4096) + 4097 crosses all of these except the K3 tile-count loop, with a ragged tail
(4097 = one 4096-row K3 tile and one row); N_HUGE = 65536*SM + 4097 crosses that one too.
"""
import numpy as np
import pytest

import primitives_ref as ref

pytestmark = pytest.mark.gpu

EDGE = [
    0,                   # empty: no launch, empty outputs
    1,                   # one row: the scalar tails, one partial validity word
    31, 32, 33,          # one K2 tail ballot word short of / exactly / one past 32 rows
    63, 64, 65,          # one k_compare64 warp-step of 64 rows; K4 rows 64 = 16 full quads
    127, 128, 129,       # one k_compare warp-step of 32 lanes x 4 four-byte rows
    2047, 2048, 2049,    # one K6 tile of 2048 rows; 2049 needs a second tile and the cursor
    4095, 4096, 4097,    # one K3 tile of 4096 rows; 4097 needs a second tile and the scan
]
SIZES = EDGE + ["N_BIG"]


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as m
    m.init()
    return m


@pytest.fixture(scope="module")
def sizes(plb):
    sm = plb.device_info()["sm_count"]
    return {"N_BIG": max(32768 * sm, 1024 * 4096) + 4097, "N_HUGE": 65536 * sm + 4097}


def _n(sizes, size):
    return sizes[size] if isinstance(size, str) else size


def _check(what, got, exp):
    err = ref.valid_equal(got[0], got[1], exp[0], exp[1])
    assert err is None, f"{what}: {err}"


def _status(plb, fn):
    with pytest.raises(plb.B200Error) as e:
        fn()
    return e.value.status


# ------------------------------------------------------------------ K1 elementwise
@pytest.mark.parametrize("dtype", ref.DTYPES)
@pytest.mark.parametrize("size", SIZES)
def test_k1_array_array(plb, sizes, dtype, size):
    n = _n(sizes, size)
    rng = np.random.default_rng(100 + n)
    a, b = ref.column(rng, dtype, n), ref.column(rng, dtype, n, divisor=True)
    av, bv = ref.validity(rng, n), ref.validity(rng, n)
    for op in ref.OPS:
        for lv, rv in ((av, bv), (None, None)):
            _check((op, n, lv is None), plb.elementwise(op, (a, lv), (b, rv)), ref.arith(op, a, b, lv, rv))


@pytest.mark.parametrize("dtype", ref.DTYPES)
def test_k1_scalar_forms(plb, sizes, dtype):
    # every special scalar on either side, nullable and not; then past the grid cap with two of them
    rng = np.random.default_rng(7)
    dt = np.dtype(dtype)
    for n in (2, 33, 4097, 20_011, sizes["N_BIG"]):
        a, b = ref.column(rng, dtype, n), ref.column(rng, dtype, n, divisor=True)
        av, bv = ref.validity(rng, n), ref.validity(rng, n)
        specials = ref.scalars(dtype) if n < sizes["N_BIG"] else [dt.type(7), dt.type(np.nan) if dt.kind == "f" else dt.type(-1 if dt.kind == "i" else 0)]
        for s in specials:
            sc = np.array([s], dt)
            for op in ref.OPS:
                for lv, rv in ((av, bv), (None, None)):
                    _check((op, "as", s, n), plb.elementwise(op, (a, lv), sc), ref.arith(op, a, s, lv, None))
                    _check((op, "sa", s, n), plb.elementwise(op, sc, (b, rv)), ref.arith(op, s, b, None, rv))


def test_k1_null_scalar_and_unsupported(plb):
    a = np.arange(100, dtype=np.int64)
    for op in ref.OPS:
        v, valid = plb.elementwise(op, a, (np.array([3], np.int64), np.array([False])))
        assert valid is not None and not valid.any(), op
        assert v.dtype == (np.float64 if op == "truediv" else np.int64)
    for dt in ("int8", "int16", "bool"):
        x = np.ones(10, dt)
        for op in ref.OPS:
            assert _status(plb, lambda: plb.elementwise(op, x, x)) == 4, (dt, op)
        for op in ref.CMPS:
            assert _status(plb, lambda: plb.compare(op, x, x)) == 4, (dt, op)


# ------------------------------------------------------------------ K2 compare
@pytest.mark.parametrize("dtype", ref.DTYPES)
@pytest.mark.parametrize("size", SIZES)
def test_k2_compare(plb, sizes, dtype, size):
    n = _n(sizes, size)
    rng = np.random.default_rng(200 + n)
    dt = np.dtype(dtype)
    a, b = ref.column(rng, dtype, n), ref.column(rng, dtype, n)
    eq = rng.random(n) < 1 / 3                 # b == a in a third of the rows: the le / ge boundaries
    b[eq] = a[eq]
    av, bv = ref.validity(rng, n), ref.validity(rng, n)
    for op in ref.CMPS:
        for lv, rv in ((av, bv), (None, None)):
            _check((op, n), plb.compare(op, (a, lv), (b, rv)), ref.compare(op, a, b, lv, rv))
        if op in ("eq", "ne"):
            for lv, rv in ((av, bv), (None, bv)):
                _check((op, "missing", n), plb.compare(op, (a, lv), (b, rv), missing=True), ref.compare(op, a, b, lv, rv, missing=True))
    for s in ref.scalars(dtype):
        a2 = a.copy()
        a2[::3] = s                            # rows equal to the scalar
        sc = np.array([s], dt)
        for op in ref.CMPS:
            _check((op, "scalar", s, n), plb.compare(op, (a2, av), sc), ref.compare(op, a2, s, av))
            if op in ("eq", "ne"):
                _check((op, "scalar missing", s, n), plb.compare(op, (a2, av), sc, missing=True), ref.compare(op, a2, s, av, missing=True))
        if size != "N_BIG":
            for op in ref.CMPS:
                _check((op, "scalar non-null", s, n), plb.compare(op, a2, sc), ref.compare(op, a2, s))


def test_k2_null_scalar(plb):
    a = np.arange(100, dtype=np.float64)
    for op in ref.CMPS:
        v, valid = plb.compare(op, a, (np.array([3.0]), np.array([False])))
        assert valid is not None and not valid.any(), op
    assert _status(plb, lambda: plb.compare("eq", a, (np.array([3.0]), np.array([False])), missing=True)) == 4


# ------------------------------------------------------------------ K3 filter
_F_SPECS = [(ref.DTYPES[i % 6], i % 3 != 1) for i in range(19)]       # 19 columns of 4- and 8-byte widths, 13 nullable
_cache = {}


def _columns(specs, n, seed):
    """seeded columns (values, valid|None), kept for the next call with the same shape"""
    key = (tuple(specs), n, seed)
    if key not in _cache:
        _cache.clear()
        rng = np.random.default_rng(seed)
        _cache[key] = [(ref.column(rng, dt, n), ref.validity(rng, n) if nullable else None) for dt, nullable in specs]
    return _cache[key]


@pytest.mark.parametrize("sel", [0.0, 0.001, 0.5, 1.0])
@pytest.mark.parametrize("size", SIZES)
def test_k3_filter_many_columns(plb, sizes, size, sel):
    n = _n(sizes, size)
    cols = _columns(_F_SPECS, n, 300)
    rng = np.random.default_rng(301 + n)
    mask = rng.random(n) < sel
    masks = [(mask, ref.validity(rng, n, 0.1))] + ([(mask, None)] if sel in (0.0, 1.0) else [])
    for m, mv in masks:
        outs = plb.filter(cols, (m, mv))
        assert len(outs) == len(cols)
        for i, ((v, valid), got) in enumerate(zip(cols, outs)):
            _check(("filter col", i, n, sel, mv is None), got, ref.filter(v, valid, m, mv))


@pytest.mark.parametrize("sel", [0.001, 0.5])
def test_k3_filter_huge_one_column(plb, sizes, sel):
    # N_HUGE: more than 16*SM tiles, so the tile-count kernel grid-strides as well
    n = sizes["N_HUGE"]
    rng = np.random.default_rng(302)
    v = rng.integers(0, 2**32, n, dtype=np.uint32)
    valid, mask, mv = ref.validity(rng, n), rng.random(n) < sel, ref.validity(rng, n, 0.1)
    [got] = plb.filter([(v, valid)], (mask, mv))
    _check(("huge", sel), got, ref.filter(v, valid, mask, mv))


@pytest.mark.parametrize("dtype", ["float32", "int32", "uint32"])
def test_k3_filter_cmp_four_byte_nullable(plb, sizes, dtype):
    dt = np.dtype(dtype)
    rng = np.random.default_rng(303)
    for n in (4097, 100_003, sizes["N_BIG"]):
        x, xv = ref.column(rng, dtype, n), ref.validity(rng, n)
        other = rng.integers(-2**63, 2**63 - 1, n, dtype=np.int64)
        specials = ref.scalars(dtype) if n < sizes["N_BIG"] else ref.scalars(dtype)[-2:]
        for s in specials:
            x2 = x.copy()
            x2[::5] = s
            for op in ref.CMPS:
                outs = plb.filter_cmp([(x2, xv), other], 0, op, np.array([s], dt))
                r, rvalid = ref.compare(op, x2, s, xv)
                keep = r & rvalid
                _check((op, s, n, "pred"), outs[0], (x2[keep], None))
                _check((op, s, n, "other"), outs[1], (other[keep], None))


# ------------------------------------------------------------------ K4 gather
_G_SPECS = [(ref.DTYPES[i % 6], i % 2 == 0) for i in range(11)]       # 11 columns: two batches of G_MAX_COLS = 8


@pytest.mark.parametrize("nulls", ["none", "bitmap", "sentinel", "both"])
@pytest.mark.parametrize("size", SIZES)
def test_k4_gather_many_columns(plb, sizes, size, nulls):
    m = _n(sizes, size)
    n_src = 5003
    cols = _columns(_G_SPECS, n_src, 400)
    rng = np.random.default_rng(401 + m)
    idx = rng.integers(0, n_src, m).astype(np.uint32)
    ivalid = None
    if nulls in ("sentinel", "both"):
        idx[rng.random(m) < 0.1] = ref.IDX_NULL
    if nulls in ("bitmap", "both"):
        ivalid = ref.validity(rng, m)
        idx[~ivalid & (rng.random(m) < 0.5)] = n_src + 17      # out of range under a null slot: not an error
    for check in (True, False):
        outs = plb.gather(cols, (idx, ivalid), check_bounds=check)
        for i, ((v, valid), got) in enumerate(zip(cols, outs)):
            exp = ref.gather(v, valid, idx, ivalid)
            _check(("gather col", i, m, nulls, check), got, exp)
            if nulls == "none" and valid is None:
                assert got[1] is None


def test_k4_bounds(plb):
    v = np.arange(1000, dtype=np.int64)
    w = np.arange(500, dtype=np.float32)
    for bad in (1000, 4000, 0xFFFFFFFE):
        idx = np.array([0, 999, bad, 5], np.uint32)
        with pytest.raises(plb.OutOfBoundsError):
            plb.gather([v], idx)
        # hidden by a null slot: gathered as null, no error
        got = plb.gather([v], (idx, np.array([True, True, False, True])))[0]
        _check(("hidden", bad), got, ref.gather(v, None, idx, np.array([True, True, False, True])))
    # the shortest column bounds the index
    with pytest.raises(plb.OutOfBoundsError):
        plb.gather([v, w], np.array([0, 500], np.uint32))
    # the sentinel without a bitmap is a null, with or without the bounds check
    idx = np.array([0, ref.IDX_NULL, 999, ref.IDX_NULL], np.uint32)
    for check in (True, False):
        _check(("sentinel", check), plb.gather([v], idx, check_bounds=check)[0], ref.gather(v, None, idx))


# ------------------------------------------------------------------ K6 hash partition
_P_DTYPES = ["int64", "uint64", "int32", "uint32", "float64", "float32"]
_PAYLOAD_DTYPES = ["int64", "float32", "uint64", "int32", "float64", "uint32", "int64"]


def _check_partition(plb, key, kvalid, P, what):
    n = key.size
    rng = np.random.default_rng(n + P)
    rowid = np.arange(n, dtype=np.uint32)
    payload = [rowid] + [ref.column(rng, dt, n) for dt in _PAYLOAD_DTYPES]      # 8 payload columns, one of them the row id
    (ko, kov), pouts, offs = plb.hash_partition((key, kvalid), payload, P)
    parts = ref.partition_of(key, kvalid, P)
    assert np.array_equal(offs, ref.partition_offsets(parts, P)), (what, P, "offsets")
    got_rows = pouts[0][0]
    # row order inside a partition is unspecified: compare the sorted row ids of every partition's range
    seg = np.repeat(np.arange(P), np.diff(offs))
    order = np.lexsort((got_rows, seg))
    assert np.array_equal(got_rows[order], np.argsort(parts, kind="stable").astype(np.uint32)), (what, P, "row ids")
    src = got_rows.astype(np.int64)
    _check((what, P, "key"), (ko, kov), (key[src], None if kvalid is None else kvalid[src]))
    for j, (p, (po, pov)) in enumerate(zip(payload, pouts)):
        assert pov is None
        _check((what, P, "payload", j), (po, None), (p[src], None))


@pytest.mark.parametrize("nullable", [False, True])
@pytest.mark.parametrize("dtype", _P_DTYPES)
def test_k6_hash_partition(plb, sizes, dtype, nullable):
    for size in SIZES:
        n = _n(sizes, size)
        rng = np.random.default_rng(500 + n)
        key = ref.column(rng, dtype, n)
        if np.dtype(dtype).kind == "f" and n > 64:
            sp = ref.float_specials(dtype)
            key[rng.integers(0, n, n // 16)] = sp[rng.integers(0, sp.size, n // 16)]      # ±0 and NaNs all over
        kvalid = ref.validity(rng, n) if nullable else None
        for P in ((1, 2, 3, 17, 63, 64) if size != "N_BIG" else (3, 64)):
            _check_partition(plb, key, kvalid, P, (dtype, n, nullable))


def test_k6_rejections(plb):
    key = np.arange(100, dtype=np.int64)
    p = np.zeros(100, np.int64)
    assert _status(plb, lambda: plb.hash_partition(key, [p] * 9, 4)) == 4
    assert _status(plb, lambda: plb.hash_partition(key, [(p, np.arange(100) % 2 == 0)], 4)) == 4
    for P in (0, 65):
        assert _status(plb, lambda: plb.hash_partition(key, [p], P)) == 1
    _, pouts, offs = plb.hash_partition(key, [p] * 8, 64)     # the most payload columns it takes
    assert len(pouts) == 8 and offs[-1] == 100


# ------------------------------------------------------------------ device-resident views
# import_column borrows a device view when its values are 16-byte aligned and its validity starts on a 4-byte aligned
# byte, and borrows the bitmap itself only when the length is a multiple of 32; otherwise it copies.
VIEWS = {
    "aligned": (64, 8192),      # values and bitmap borrowed
    "ragged": (64, 8013),       # values borrowed, bitmap copied (its last word would reach past the view)
    "unaligned": (3, 8013),     # copied
}


class _Views:
    """numpy columns uploaded once with to_device, passed back as Column views at an offset"""

    def __init__(self, plb, off, length):
        self.plb, self.off, self.len, self.keep = plb, off, length, []

    def __call__(self, values, valid=None):
        d = self.plb.to_device(values, valid)
        self.keep.append(d)
        col = self.plb.Column(d.values_ptr, d.validity_ptr if valid is not None else None, dtype=values.dtype, length=self.len, offset=self.off,
                              location=self.plb.DEVICE)
        sl = slice(self.off, self.off + self.len)
        return col, values[sl], (None if valid is None else valid[sl])


def _bitmap_copies(plb, fn):
    plb.profile_enable(True)
    plb.profile_reset()
    try:
        fn()
        return plb.profile().get("bitmap_copy", {}).get("launches", 0)
    finally:
        plb.profile_enable(False)


@pytest.mark.parametrize("view", list(VIEWS))
def test_device_views(plb, view):
    off, length = VIEWS[view]
    n = off + length + 100
    rng = np.random.default_rng(600)
    V = _Views(plb, off, length)
    base = {dt: (ref.column(rng, dt, n), ref.validity(rng, n)) for dt in ref.DTYPES}
    ab = {dt: (ref.column(rng, dt, n, divisor=True), ref.validity(rng, n)) for dt in ref.DTYPES}
    probe = V(*base["int64"])[0]
    copies = _bitmap_copies(plb, lambda: plb.elementwise("add", probe, np.array([1], np.int64)))
    assert copies == (0 if view == "aligned" else 1), (view, copies)      # the bitmap is borrowed only when aligned
    for dt in ref.DTYPES:
        ca, a, av = V(*base[dt])
        cb, b, bv = V(*ab[dt])
        for op in ref.OPS:                                                                   # K1
            _check(("k1", dt, op), plb.elementwise(op, ca, cb), ref.arith(op, a, b, av, bv))
            s = np.dtype(dt).type(3)
            _check(("k1 scalar", dt, op), plb.elementwise(op, ca, np.array([s])), ref.arith(op, a, s, av, None))
        for op in ref.CMPS:                                                                  # K2
            _check(("k2", dt, op), plb.compare(op, ca, cb), ref.compare(op, a, b, av, bv))
            _check(("k2 scalar", dt, op), plb.compare(op, ca, np.array([a[7]])), ref.compare(op, a, a[7], av))
    cols = [V(*base[dt]) for dt in ref.DTYPES]                                               # K3
    cm, m, mv = V(rng.random(n) < 0.5, ref.validity(rng, n))
    for (_, v, valid), got in zip(cols, plb.filter([c for c, _, _ in cols], cm)):
        _check(("k3", v.dtype), got, ref.filter(v, valid, m, mv))
    idx_all = rng.integers(0, length, n).astype(np.uint32)                                  # K4
    idx_all[::11] = ref.IDX_NULL
    ci, idx, ivalid = V(idx_all, ref.validity(rng, n))
    for (_, v, valid), got in zip(cols, plb.gather([c for c, _, _ in cols], ci)):
        _check(("k4", v.dtype), got, ref.gather(v, valid, idx, ivalid))
    for dt in ("int64", "float32"):                                                          # K6
        ck, k, kv = V(*base[dt])
        cp, p, _ = V(np.arange(n, dtype=np.int64))
        (ko, kov), [(po, _)], offs = plb.hash_partition(ck, [cp], 17)
        parts = ref.partition_of(k, kv, 17)
        assert np.array_equal(offs, ref.partition_offsets(parts, 17))
        src = (po - off).astype(np.int64)
        seg = np.repeat(np.arange(17), np.diff(offs))
        assert np.array_equal(src[np.lexsort((src, seg))], np.argsort(parts, kind="stable")), ("k6", dt)
        _check(("k6 key", dt), (ko, kov), (k[src], kv[src]))
