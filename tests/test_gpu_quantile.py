"""GPU tests (-m gpu) of the per-group median / quantile (BL_AGG_MEDIAN, BL_AGG_QUANTILE): every result is bit-identical to
the plain-Python oracle (tests/quantile_oracle.py), up to the sign of a zero and the payload of a NaN, which the reference
does not pin.  The two device plans (small groups sorted in shared memory, large groups through the radix sort) are also
compared with each other byte for byte through BL_QUANTILE_GLOBAL=1."""
import ctypes as C

import numpy as np
import pyarrow as pa
import pytest

import quantile_oracle as qo
from test_gpu_plugin_abi import Caller
from test_quantile import NP, check_kat_result, kat_column, kat_q_method, quantile_kats

pytestmark = pytest.mark.gpu

H = 2048          # groups of more than H rows take the large-group plan (QS_H in quantile.cu)
QS = (0.0, 0.1, 0.25, 0.5, 0.6, 0.9, 1.0)


@pytest.fixture(scope="module", autouse=True)
def device():
    import polars_b200 as plb
    plb.init()
    return plb


def kind_of(q, method):
    return f"quantile:{q!r}:{method}"


def first_occurrence_ids(keys):
    keys = np.asarray(keys)
    _, first, inv = np.unique(keys, return_index=True, return_inverse=True)
    rank = np.empty(first.size, np.int64)
    rank[np.argsort(first, kind="stable")] = np.arange(first.size)
    return rank[inv.reshape(-1)]


def dev_group_quantiles(keys, vals, valid, kinds):
    """group_by_agg_keys over one int64 key column -> [(values, validity)] (validity all-True when None)"""
    import polars_b200 as plb
    col = (vals, valid) if valid is not None else vals
    _, outs = plb.group_by_agg_keys([np.asarray(keys, np.int64)], [(k, col) for k in kinds], maintain_order=True)
    return [(v, np.ones(v.shape, bool) if m is None else m) for v, m in outs]


def assert_same(got, gv, exp, ev, what=""):
    assert got.dtype == exp.dtype, f"{what}: dtype {got.dtype} != {exp.dtype}"
    assert np.array_equal(gv, ev), f"{what}: validity differs at {np.nonzero(gv != ev)[0][:10]}"
    g, e = got[ev], exp[ev]
    bad = ~((g == e) | (np.isnan(g) & np.isnan(e)))          # == : -0.0 equals +0.0; NaN as NaN
    assert not bad.any(), f"{what}: {bad.sum()} differ, first at {np.nonzero(bad)[0][:5]}: got {g[bad][:5]} exp {e[bad][:5]}"


def oracle(keys, vals, valid, q, method):
    return qo.group_quantile(np.asarray(keys).tolist(), vals, valid, q, method)


# ------------------------------------------------------------------------------------------------- known answers
@pytest.mark.parametrize("case", quantile_kats(), ids=lambda c: c["cite"][-70:])
def test_reference_kats(case):
    vals, valid = kat_column(case)
    q, m = kat_q_method(case)
    keys = first_occurrence_ids([str(k) for k in case["keys"]])
    kind = "median" if case["kind"] == "median" else kind_of(q, m)
    (got, ok), = dev_group_quantiles(keys, vals, valid, [kind])
    check_kat_result(case, got, ok)


# ------------------------------------------------------------------------------------------------- dtypes x methods x q
def random_column(rng, dt, n):
    info = np.iinfo(dt) if np.dtype(dt).kind in "iu" else None
    if info is not None:
        if np.dtype(dt).itemsize == 8:      # extremes whose f64 conversion rounds, plus a narrow range with ties
            pool = np.array([info.min, info.max, info.max - 1, 0, 1, 2, 3, (1 << 53) + 1, info.max // 3], dtype=dt)
            return np.where(rng.random(n) < 0.5, rng.choice(pool, n), rng.integers(0, 7, n).astype(dt)).astype(dt)
        return rng.integers(int(info.min), int(info.max) + 1, n).astype(dt)
    x = rng.normal(0, 100, n).astype(dt)
    ties = rng.random(n) < 0.3
    x[ties] = rng.integers(-3, 3, int(ties.sum())).astype(dt)
    return x


@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("dt", ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64"])
def test_every_dtype_method_and_quantile(dt, nulls):
    rng = np.random.default_rng(hash((dt, nulls)) & 0xFFFF)
    n = 1500
    keys = rng.integers(0, 120, n)
    keys[:40] = 1000 + np.arange(40)                          # singletons
    vals = random_column(rng, NP[dt], n)
    valid = (rng.random(n) > 0.25) if nulls else None
    if nulls:
        valid[keys == 7] = False                               # an all-null group
    specs = [(q, m) for m in qo.METHODS for q in QS]
    outs = dev_group_quantiles(keys, vals, valid, [kind_of(q, m) for q, m in specs] + ["median"])
    for (q, m), (got, gv) in zip(specs + [(0.5, "linear")], outs):
        exp, ev = oracle(keys, vals, valid, q, m)
        assert_same(got, gv, exp, ev, f"{dt} nulls={nulls} {m} {q}")


@pytest.mark.parametrize("dt", ["float32", "float64"])
def test_special_floats(dt):
    rng = np.random.default_rng(5)
    pool = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0, -1.0, 2.5], dtype=dt)
    n = 3000
    keys = rng.integers(0, 600, n)                             # groups of ~5: many ties of inf / NaN / zeros
    vals = rng.choice(pool, n)
    valid = rng.random(n) > 0.1
    for m in qo.METHODS:
        outs = dev_group_quantiles(keys, vals, valid, [kind_of(q, m) for q in QS])
        for q, (got, gv) in zip(QS, outs):
            exp, ev = oracle(keys, vals, valid, q, m)
            assert_same(got, gv, exp, ev, f"{dt} {m} {q}")


# ------------------------------------------------------------------------------------------------- group-size mixes, both plans
def sized_groups(rng, sizes):
    """keys whose groups have the given sizes, rows of different groups interleaved"""
    keys = np.repeat(np.arange(len(sizes)), sizes)
    return rng.permutation(keys)


MIXES = {
    "singletons": lambda rng: np.arange(5000)[rng.permutation(5000)],
    "around_half_tile": lambda rng: sized_groups(rng, [H - 1, H, H + 1, 1, 2, 3, 17, H - 1, H + 1] + list(rng.integers(1, 60, 200))),
    "huge_beside_small": lambda rng: sized_groups(rng, [300_000] + list(rng.integers(1, 40, 3000))),
    "several_large": lambda rng: sized_groups(rng, list(rng.integers(H + 1, 3 * H, 40)) + list(rng.integers(1, 9, 500))),
}


@pytest.mark.parametrize("mix", sorted(MIXES))
def test_group_size_mixes_and_both_plans_agree(mix, monkeypatch):
    rng = np.random.default_rng(len(mix))
    keys = MIXES[mix](rng)
    n = keys.size
    vals = rng.normal(size=n)
    vals[rng.random(n) < 0.05] = np.nan
    valid = rng.random(n) > 0.2
    valid[keys == keys[0]] = False                              # the group of the first row is all null
    kinds = ["median", kind_of(0.1, "nearest"), kind_of(0.9, "linear"), kind_of(0.5, "midpoint"), kind_of(0.25, "equiprobable")]
    small = dev_group_quantiles(keys, vals, valid, kinds)
    monkeypatch.setenv("BL_QUANTILE_GLOBAL", "1")
    glob = dev_group_quantiles(keys, vals, valid, kinds)
    for (a, av), (b, bv) in zip(small, glob):
        assert np.array_equal(av, bv) and a.tobytes() == b.tobytes()      # byte for byte
    dense = first_occurrence_ids(keys)
    for kind, (got, gv) in zip(kinds, small):
        q, m = (0.5, "linear") if kind == "median" else (float(kind.split(":")[1]), kind.split(":")[2])
        exp, ev = qo.numpy_group_quantile(dense, vals, valid, q, m, int(dense.max()) + 1)
        assert_same(got, gv, exp, ev, f"{mix} {kind}")


def test_plans_agree_on_integers_with_nulls(monkeypatch):
    rng = np.random.default_rng(9)
    keys = sized_groups(rng, list(rng.integers(1, 3 * H, 300)))
    vals = rng.integers(-(1 << 62), 1 << 62, keys.size)
    valid = rng.random(keys.size) > 0.05
    kinds = [kind_of(q, m) for m in qo.METHODS for q in (0.1, 0.9)]
    a = dev_group_quantiles(keys, vals, valid, kinds)
    monkeypatch.setenv("BL_QUANTILE_GLOBAL", "1")
    b = dev_group_quantiles(keys, vals, valid, kinds)
    for (x, xv), (y, yv) in zip(a, b):
        assert np.array_equal(xv, yv) and x.tobytes() == y.tobytes()


# ------------------------------------------------------------------------------------------------- one sort per column
@pytest.mark.parametrize("force_global", [False, True])
def test_one_sort_per_value_column(force_global, monkeypatch):
    import polars_b200 as plb
    if force_global:
        monkeypatch.setenv("BL_QUANTILE_GLOBAL", "1")
    rng = np.random.default_rng(3)
    keys = rng.integers(0, 500, 50_000)
    x, y = rng.normal(size=50_000), rng.normal(size=50_000)
    plb.profile_enable(True)
    plb.profile_reset()
    try:
        _, outs = plb.group_by_agg_keys([keys], [("median", x), (kind_of(0.25, "linear"), x), ("sum", x), (kind_of(0.75, "nearest"), x), ("median", y)],
                                        maintain_order=True)
        prof = plb.profile()
    finally:
        plb.profile_enable(False)
    sort_kernel = "quantile_encode_large" if force_global else "quantile_small"
    assert prof[sort_kernel]["launches"] == 2, prof                      # x and y: one each
    assert prof["quantile_pick_large" if force_global else "quantile_small"]["launches"] == 2
    for (q, m), col, (got, gv) in zip([(0.5, "linear"), (0.25, "linear"), (0.75, "nearest"), (0.5, "linear")], [x, x, x, y],
                                      [outs[0], outs[1], outs[3], outs[4]]):
        exp, ev = oracle(keys, col, None, q, m)
        assert_same(got, np.ones(got.shape, bool) if gv is None else gv, exp, ev, f"{m} {q}")


# ------------------------------------------------------------------------------------------------- keys
def test_median_with_several_keys_and_string_keys():
    import polars_b200 as plb
    rng = np.random.default_rng(4)
    n = 20_000
    k0, k1 = rng.integers(0, 30, n), rng.integers(0, 7, n).astype(np.int16)
    v = rng.integers(-1000, 1000, n).astype(np.int32)
    vm = rng.random(n) > 0.1
    kouts, outs = plb.group_by_agg_keys([k0, k1], [("median", (v, vm)), (kind_of(0.3, "higher"), (v, vm))], maintain_order=True)
    pair = [(int(a), int(b)) for a, b in zip(k0, k1)]
    for (q, m), (got, gv) in zip([(0.5, "linear"), (0.3, "higher")], outs):
        exp, ev = qo.group_quantile(pair, v, vm, q, m)
        assert_same(got, np.ones(got.shape, bool) if gv is None else gv, exp, ev, f"two keys {m}")
    assert list(zip(kouts[0][0].tolist(), kouts[1][0].tolist())) == list(dict.fromkeys(pair))
    words = [None if i % 97 == 0 else f"w{i % 41}" for i in range(n)]
    f = rng.normal(size=n).astype(np.float32)
    skeys, souts = plb.group_by_agg_strings(plb.StringColumn(words), [("median", f), ("sum", f)], maintain_order=True)
    exp, ev = qo.group_median(words, f, None)
    assert skeys == [None if w is None else w.encode() for w in dict.fromkeys(words)]
    got, gv = souts[0]
    assert_same(got, np.ones(got.shape, bool) if gv is None else gv, exp, ev, "string keys")
    k, (agg,) = plb.group_by_agg(k0, [("median", v)], maintain_order=True)           # single key entry point
    exp, ev = qo.group_median(k0.tolist(), v, None)
    assert_same(agg[0], np.ones(agg[0].shape, bool), exp, ev, "bl_groupby_agg")


# ------------------------------------------------------------------------------------------------- plugin
def test_plugin_median_and_quantile():
    import polars_b200 as plb
    caller = Caller(plb.lib())
    rng = np.random.default_rng(6)
    n = 5000
    k = rng.integers(0, 50, n)
    x = rng.integers(-100, 100, n).astype(np.int8)
    xm = rng.random(n) < 0.1
    X = pa.array(x, mask=xm)
    valid = ~xm
    out = caller.call("group_median", [("k", [pa.array(k)]), ("x", [X.slice(0, 1000), X.slice(1000)])])
    assert out.type.field("agg").type == pa.float64()
    exp, ev = qo.group_median(k.tolist(), x, valid)
    got = out.field("agg")
    assert_same(np.asarray(got.fill_null(0.0)), np.asarray(got.is_valid()), exp, ev, "plugin median")
    assert np.array_equal(np.asarray(out.field("key")), k[np.sort(np.unique(k, return_index=True)[1])])
    f = rng.normal(size=n).astype(np.float32)
    out = caller.call("group_quantile", [("k", [pa.array(k)]), ("f", [pa.array(f)])], kwargs={"quantile": 0.9, "method": "linear"})
    assert out.type.field("agg").type == pa.float32()
    exp, ev = qo.group_quantile(k.tolist(), f, None, 0.9, "linear")
    assert_same(np.asarray(out.field("agg")), np.ones(exp.shape, bool), exp, ev, "plugin quantile")
    out = caller.call("group_quantile", [("k", [pa.array(k)]), ("f", [pa.array(f)])], kwargs={"quantile": 0.25})      # method nearest
    exp, ev = qo.group_quantile(k.tolist(), f, None, 0.25, "nearest")
    assert_same(np.asarray(out.field("agg")), np.ones(exp.shape, bool), exp, ev, "plugin quantile nearest")
    with pytest.raises(RuntimeError, match="`quantile` kwarg is required"):
        caller.call("group_quantile", [("k", [pa.array(k)]), ("f", [pa.array(f)])])
    with pytest.raises(RuntimeError, match="unknown method"):
        caller.call("group_quantile", [("k", [pa.array(k)]), ("f", [pa.array(f)])], kwargs={"quantile": 0.5, "method": "cubic"})


# ------------------------------------------------------------------------------------------------- errors
def raw_params_call(plb, key, vals, kinds, params):
    kc = plb._as_col(key); vc = plb._as_col(vals)
    karr, varr = plb._col_array([kc]), plb._col_array([vc])
    aggs = (plb.BlAgg * len(kinds))(*[plb.BlAgg(k, 1, C.cast(varr, C.POINTER(plb.BlColumn))) for k in kinds])
    parr = None if params is None else (plb.BlAggParam * len(params))(*[plb.BlAggParam(q, m, 0) for q, m in params])
    ok, oa = (plb.BlColumn * 1)(), (plb.BlColumn * len(kinds))()
    return plb.lib().bl_groupby_agg_params(karr, C.c_int32(1), aggs, parr, C.c_int32(len(kinds)), C.c_int32(1), C.c_int32(plb.HOST), ok, oa)


def test_errors():
    import polars_b200 as plb
    key, v = np.array([1, 1, 2]), np.array([1.0, 2.0, 3.0])
    for q in (1.5, -0.1, float("nan")):
        assert raw_params_call(plb, key, v, [plb.QUANTILE], [(q, 0)]) == 4                 # UNSUPPORTED: the caller's CPU path
    assert raw_params_call(plb, key, v, [plb.QUANTILE], [(0.5, 6)]) == 1                  # unknown method
    assert raw_params_call(plb, key, v, [plb.QUANTILE], [(0.5, -1)]) == 1
    assert raw_params_call(plb, key, v, [plb.QUANTILE], None) == 1                        # no params
    assert raw_params_call(plb, key, v, [plb.AGGS["median"]], None) == 0                  # median needs none
    with pytest.raises(plb.B200Error) as e:
        plb.group_by_agg(key, [(kind_of(0.5, "linear"), v)])                               # bl_groupby_agg has no params
    assert e.value.status == 1
    with pytest.raises(plb.B200Error) as e:
        plb.group_by_agg_keys([key], [("median", np.array([True, False, True]))])           # Bool column
    assert e.value.status == 4
    with pytest.raises(plb.B200Error) as e:
        plb.GroupBy(np.int64, [("median", np.float64)])                                     # streaming state
    assert e.value.status == 4
    w = plb.Window(1 << 20)
    try:
        with pytest.raises(plb.B200Error) as e:
            plb.group_by_agg_partitioned(key, [("median", v)], 0, [w.ptr], w.ptr, 16, 1)
        assert e.value.status == 4
    finally:
        w.destroy()


# ------------------------------------------------------------------------------------------------- property, large
def test_property_20m_rows_1m_groups():
    import polars_b200 as plb
    rng = np.random.default_rng(11)
    n, g = 20_000_000, 1_000_000
    gid = rng.integers(0, g, n)
    gid[: 3 * H] = g                                            # one group beyond the small-group plan
    vals = rng.normal(size=n)
    valid = rng.random(n) > 0.05
    dk = plb.to_device(gid.astype(np.int64))
    dv = plb.to_device(vals, valid)
    kinds = ["median", kind_of(0.9, "linear"), kind_of(0.1, "nearest")]
    kout, outs = plb.group_by_agg_keys([dk], [(k, dv) for k in kinds], maintain_order=True)
    dense = first_occurrence_ids(gid)
    assert np.array_equal(kout[0][0], gid[np.sort(np.unique(gid, return_index=True)[1])])
    for kind, (got, gv) in zip(kinds, outs):
        q, m = (0.5, "linear") if kind == "median" else (float(kind.split(":")[1]), kind.split(":")[2])
        exp, ev = qo.numpy_group_quantile(dense, vals, valid, q, m, int(dense.max()) + 1)
        assert_same(got, np.ones(got.shape, bool) if gv is None else gv, exp, ev, f"2e7 {kind}")
