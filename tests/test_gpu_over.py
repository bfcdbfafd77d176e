"""GPU tests of the window functions (bl_over).  Results are compared with tests/window_oracle.py (or, for large inputs, its
numpy restatement below): bit for bit for integer scans, min / max, count, shift and every exact aggregation; float sums and
products under the parallel scan's bound, and bit for bit in deterministic mode.  Sizes derive from sm_count so that the
persistent scan grid takes several tiles per CTA and the look-back crosses many tiles."""
import json
import math
import os
import struct

import numpy as np
import pytest

import window_oracle as wo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TILE = 2048
DTYPES = ["int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64", "float32", "float64", "bool"]
CUMS = ["cum_sum", "cum_prod", "cum_min", "cum_max", "cum_count"]
U = {"float32": 2.0 ** -24, "float64": 2.0 ** -53}


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as plb
    plb.init()
    plb.set_deterministic(False)
    return plb


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


def values(rng, dtype, n, nulls):
    if dtype == "bool":
        x = rng.random(n) < 0.5
    elif dtype.startswith("float"):
        x = rng.integers(-4, 5, n).astype(dtype) * np.asarray(0.5, dtype)
        sp = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0], dtype)
        at = rng.random(n) < 0.05
        x[at] = sp[rng.integers(0, len(sp), at.sum())]
    else:
        info = np.iinfo(dtype)
        x = rng.integers(-3 if info.min < 0 else 0, 4, n).astype(dtype)
        at = rng.random(n) < 0.05
        x[at] = rng.choice(np.array([info.min, info.max, info.max // 2 + 1], dtype), at.sum())
    valid = rng.random(n) >= 0.2 if nulls else None
    return x, valid


def as_list(x, valid):
    out = x.tolist()
    if x.dtype.kind == "f":
        out = [float(v) for v in out]
    if valid is not None:
        out = [v if ok else None for v, ok in zip(out, valid)]
    return out


def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, float) or isinstance(b, float):
        a, b = float(a), float(b)
        return (a != a and b != b) or struct.pack("<d", a) == struct.pack("<d", b)
    return int(a) == int(b)


def check_scan(kind, dtype, got, exp, vals_in_order_groups):
    """got: (values, valid) in row order; exp: oracle list.  Float sums / products under the bound."""
    gv, gm = got
    gl = as_list(gv, gm)
    assert len(gl) == len(exp)
    odt = wo.scan_dtype(kind, dtype)
    assert gv.dtype == np.dtype(odt if odt != "bool" else "bool"), (gv.dtype, odt)
    bad = []
    for r, (a, b) in enumerate(zip(gl, exp)):
        if same(a, b):
            continue
        if kind in ("cum_sum", "cum_prod") and dtype.startswith("float") and a is not None and b is not None:
            k, s = vals_in_order_groups[r]
            u = U["float32" if dtype == "float32" and kind == "cum_prod" else "float64" if kind == "cum_sum" else dtype]
            bound = 2 * max(k - 1, 0) * u * (s if kind == "cum_sum" else abs(b)) + (2.0 ** -24 * abs(b) if dtype == "float32" and kind == "cum_sum" else 0)
            if math.isfinite(b) and abs(a - b) <= bound:
                continue
            if not math.isfinite(b) and (kind == "cum_prod" or not math.isfinite(s)) and (a != a if b != b else a == b):
                continue      # an infinite or NaN result: the bound does not apply, but the class (NaN, +inf, -inf) must agree
        bad.append((r, a, b))
    assert not bad, f"{kind} {dtype}: {len(bad)} rows differ, first {bad[:5]}"


def scan_context(part, vals, reverse):
    """row -> (k, sum |a_i| over the first k valid values of its partition's scan)"""
    ctx = {}
    for rows in part:
        rr = rows[::-1] if reverse else rows
        k, s = 0, 0.0
        for r in rr:
            v = vals[r]
            if v is not None:
                k += 1
                s += abs(float(v)) if not (isinstance(v, float) and v != v) else 0.0
            ctx[r] = (k, s)
    return ctx


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("shape", ["whole", "partitioned", "ordered"])
def test_every_op_vs_oracle(plb, dtype, nulls, shape):
    rng = np.random.default_rng(DTYPES.index(dtype) * 7 + nulls + 3 * len(shape))
    n = 3 * TILE + 77
    x, valid = values(rng, dtype, n, nulls)
    col = (x, valid) if valid is not None else x
    xs = as_list(x, valid)
    keys = [] if shape == "whole" else [rng.integers(0, 5, n)]
    order = rng.integers(0, 50, n) if shape == "ordered" else None
    kinds = CUMS if dtype == "bool" else CUMS + ["shift"]
    kinds = [k for k in kinds if not (dtype == "bool" and k in ("cum_min", "cum_max"))]
    ops, ref_ops = [], []
    for k in kinds:
        for opt in ([{"reverse": False}, {"reverse": True}] if k != "shift" else [{"periods": 1}, {"periods": -2}, {"periods": 0}]):
            ops.append((k, col, opt))
            ref_ops.append((k, xs, dtype, opt))
    got = plb.over(ops, partition_by=keys, order_by=order)
    kl = [k.tolist() for k in keys]
    exp = wo.over(ref_ops, kl, n, order.tolist() if order is not None else None)
    part = wo.partition_order(kl, n, order.tolist() if order is not None else None)
    for (k, _, opt), g, e in zip(ops, got, exp):
        check_scan(k, dtype, g, e, scan_context(part, xs, opt.get("reverse", False)))


@pytest.mark.parametrize("dtype", ["int8", "uint16", "int32", "float32"])
def test_cum_min_max_extremes_and_zeros(plb, dtype):
    """ties between -0.0 and +0.0 and the bounds of the dtype, forward and reverse, over many tiles"""
    rng = np.random.default_rng(11)
    n = 5 * TILE + 3
    if dtype.startswith("float"):
        x = rng.choice(np.array([-0.0, 0.0, np.nan, 1.0, -np.inf, np.inf], dtype), n)
    else:
        info = np.iinfo(dtype)
        x = rng.choice(np.array([info.min, info.max, 0, 1], dtype), n)
    g = rng.integers(0, 3, n)
    ops = [(k, x, {"reverse": r}) for k in ("cum_min", "cum_max") for r in (False, True)]
    got = plb.over(ops, partition_by=[g])
    exp = wo.over([(k, as_list(x, None), dtype, o) for k, _, o in ops], [g.tolist()], n)
    for gg, e in zip(got, exp):
        gl = as_list(*gg)
        assert all(same(a, b) for a, b in zip(gl, e))


def test_kats(plb):
    from test_over import kat_mismatches
    kats = json.load(open(os.path.join(ROOT, "tests", "golden", "window_kats.json")))
    for case in kats:
        cols = case["columns"]

        def c(name):
            v = cols[name]
            dt = case["dtypes"][name]
            if dt == "str":
                return plb.StringColumn(v)
            arr = np.array([0 if a is None else a for a in v], dt)
            ok = np.array([a is not None for a in v])
            return (arr, ok) if not ok.all() else arr
        ops = [(kind, c(col) if col else None, opts) for _, kind, col, opts in case["ops"]]
        got = plb.over(ops, partition_by=[c(k) for k in case["partition_by"]], order_by=c(case["order_by"]) if case["order_by"] else None,
                       descending=case["descending"], nulls_last=case["nulls_last"])
        outs = {name: as_list(*g) for (name, *_), g in zip(case["ops"], got)}
        assert not kat_mismatches(case, outs), (case["src"], kat_mismatches(case, outs))


def np_segments(gid_sorted):
    head = np.ones(len(gid_sorted), bool)
    head[1:] = gid_sorted[1:] != gid_sorted[:-1]
    return head


def np_cumsum_seg(vals_u64, head):
    cs = np.cumsum(vals_u64, dtype=np.uint64)
    start = np.maximum.accumulate(np.where(head, np.arange(len(head)), 0))
    base = np.where(start > 0, cs[start - 1], np.uint64(0))
    return cs - base


@pytest.mark.parametrize("reverse", [False, True])
def test_whole_column_many_tiles_no_sort(plb, sm, reverse):
    """the plain cum_sum over a column that takes several tiles per CTA of the persistent grid: no sort kernel runs"""
    n = sm * 8 * TILE * 3 + 1001
    rng = np.random.default_rng(5)
    x = rng.integers(-(1 << 62), 1 << 62, n, dtype=np.int64)
    x[::977] = np.iinfo(np.int64).min
    plb.profile_reset()
    plb.profile_enable(True)
    got_s = plb.cum_agg("cum_sum", x, reverse=reverse)
    got_mx = plb.cum_agg("cum_max", x, reverse=reverse)
    got_c = plb.cum_agg("cum_count", (x, rng.random(n) < 0.7), reverse=reverse)
    prof = plb.profile()
    plb.profile_enable(False)
    assert not any(k.startswith("sort_") or k.startswith("k5_") for k in prof), prof.keys()
    xr = x[::-1] if reverse else x
    es = np.cumsum(xr.view(np.uint64), dtype=np.uint64).view(np.int64)
    emx = np.maximum.accumulate(xr)
    if reverse:
        es, emx = es[::-1], emx[::-1]
    assert np.array_equal(got_s[0], es) and got_s[1] is None
    assert np.array_equal(got_mx[0], emx)
    assert got_c[0].dtype == np.uint32 and got_c[1] is None


@pytest.mark.parametrize("dtype", ["float32", "float64"])
@pytest.mark.parametrize("reverse", [False, True])
def test_finite_float_cum_prod_many_tiles(plb, sm, dtype, reverse):
    """default-mode float cum_prod across many tiles of the persistent grid, every partial product finite: every row within
    the parallel scan's bound of the sequential det_prod (numpy's multiply.accumulate, left to right in the dtype)"""
    rng = np.random.default_rng(21)
    n = sm * 8 * TILE * 2 + 333
    x = (1.0 + rng.uniform(-1e-3, 1e-3, n)).astype(dtype)
    g = rng.integers(0, 3, n)
    got = plb.over([("cum_prod", x, {"reverse": reverse})], partition_by=[g])[0][0]
    u = U[dtype]
    for key in range(3):
        rows = np.nonzero(g == key)[0]
        if reverse:
            rows = rows[::-1]
        ref = np.multiply.accumulate(x[rows]).astype(np.float64)
        k = np.arange(1, len(rows) + 1)
        err = np.abs(got[rows].astype(np.float64) - ref)
        assert np.all(np.isfinite(ref)) and np.all(err <= 2 * (k - 1) * u * np.abs(ref)), (key, int(np.argmax(err > 2 * (k - 1) * u * np.abs(ref))))


def test_segment_heads_at_tile_boundaries(plb):
    """partition boundaries exactly at a tile boundary and one row either side of it"""
    n = 12 * TILE
    cuts = sorted({TILE, 2 * TILE - 1, 3 * TILE + 1, 5 * TILE, 5 * TILE + 1, 7 * TILE - 1, 9 * TILE})
    g = np.zeros(n, np.int64)
    for c in cuts:
        g[c:] += 1
    x = np.arange(n, dtype=np.int64) % 1000 - 500
    got = plb.over([("cum_sum", x, {}), ("cum_sum", x, {"reverse": True}), ("cum_min", x, {}), ("shift", x, {"periods": 1})], partition_by=[g])
    exp = wo.over([("cum_sum", x.tolist(), "int64", {}), ("cum_sum", x.tolist(), "int64", {"reverse": True}), ("cum_min", x.tolist(), "int64", {}),
                   ("shift", x.tolist(), "int64", {"periods": 1})], [g.tolist()], n)
    for gg, e in zip(got, exp):
        assert all(same(a, b) for a, b in zip(as_list(*gg), e))


def test_million_small_partitions_and_hot_key(plb):
    rng = np.random.default_rng(9)
    sizes = rng.integers(1, 4, 1_000_000)
    g = np.repeat(np.arange(len(sizes)), sizes)
    n = len(g)
    perm = rng.permutation(n)
    g = g[perm]
    hot = rng.random(n) < 0.2
    g[hot] = -1      # one hot key mixed with the singletons
    x = rng.integers(-1000, 1000, n).astype(np.int64)
    got_s, got_c, got_sh = plb.over([("cum_sum", x, {}), ("cum_count", x, {"reverse": True}), ("shift", x, {"periods": -1})], partition_by=[g])
    order = np.lexsort((np.arange(n), g))      # any group order works for per-group values
    gs = g[order]
    head = np_segments(gs)
    es = np.empty(n, np.int64)
    es[order] = np_cumsum_seg(x[order].view(np.uint64), head).view(np.int64)
    assert np.array_equal(got_s[0], es)
    seg_id = np.cumsum(head) - 1
    seg_end = np.r_[np.nonzero(head)[0][1:], n][seg_id]
    ec = np.empty(n, np.uint32)
    ec[order] = seg_end - np.arange(n)
    assert np.array_equal(got_c[0], ec)
    nxt = np.arange(n) + 1
    ok = (nxt < seg_end)
    esh = np.zeros(n, np.int64)
    esh[order[ok]] = x[order[nxt[ok]]]
    ev = np.zeros(n, bool)
    ev[order[ok]] = True
    assert np.array_equal(got_sh[1], ev) and np.array_equal(got_sh[0][ev], esh[ev])


def test_null_key_several_keys_and_string_key(plb):
    rng = np.random.default_rng(2)
    n = 4 * TILE + 5
    k1 = rng.integers(0, 3, n).astype(np.float64)
    k1[rng.random(n) < 0.1] = -0.0
    k1[rng.random(n) < 0.1] = np.nan
    k1v = rng.random(n) >= 0.1
    k2 = rng.integers(0, 2, n).astype(np.int8)
    words = ["a", "bb", None, "", "ccc"]
    s = [words[i] for i in rng.integers(0, len(words), n)]
    x = rng.integers(-50, 50, n).astype(np.int32)
    k1l = [None if not ok else float(v) for v, ok in zip(k1, k1v)]
    for keys, kl in (([(k1, k1v), k2], [k1l, k2.tolist()]), ([plb.StringColumn(s)], [s])):
        got = plb.over([("cum_sum", x, {}), ("sum", x), ("shift", x, {"periods": 2})], partition_by=keys)
        exp = wo.over([("cum_sum", x.tolist(), "int32", {}), ("sum", x.tolist(), "int32", {}), ("shift", x.tolist(), "int32", {"periods": 2})], kl, n)
        for gg, e in zip(got, exp):
            assert all(same(a, b) for a, b in zip(as_list(*gg), e))


@pytest.mark.parametrize("okind", ["int8", "int32", "uint64", "float32", "float64", "bool", "string"])
@pytest.mark.parametrize("descending", [False, True])
@pytest.mark.parametrize("nulls_last", [False, True])
def test_order_by_every_key_form(plb, okind, descending, nulls_last):
    rng = np.random.default_rng(len(okind) * 4 + 2 * descending + nulls_last)
    n = 3 * TILE + 11
    g = rng.integers(0, 6, n)
    if okind == "string":
        words = ["x", "y", "xy", "", "zz"]
        ol = [words[i] if rng.random() > 0.1 else None for i in rng.integers(0, 5, n)]
        okey = plb.StringColumn(ol)
    else:
        if okind == "bool":
            ov = rng.random(n) < 0.5
        elif okind.startswith("float"):
            ov = rng.integers(0, 4, n).astype(okind)      # few values: ties, where row order must win
            ov[rng.random(n) < 0.1] = np.nan
            ov[rng.random(n) < 0.1] = -0.0
        else:
            ov = rng.integers(0, 4, n).astype(okind)
        om = rng.random(n) >= 0.1
        okey = (ov, om)
        ol = as_list(ov, om)
    x = rng.integers(-100, 100, n).astype(np.int64)
    ops = [("shift", x, {"periods": 1}), ("cum_sum", x, {}), ("first", x), ("last", x), ("cum_count", x, {"reverse": True})]
    got = plb.over(ops, partition_by=[g], order_by=okey, descending=descending, nulls_last=nulls_last)
    exp = wo.over([(k, x.tolist(), "int64", o[0] if o else {}) for k, _, *o in ops], [g.tolist()], n, ol, descending, nulls_last)
    for (k, *_), gg, e in zip(ops, got, exp):
        gl = as_list(*gg)
        assert all(same(a, b) for a, b in zip(gl, e)), k


@pytest.mark.parametrize("periods", [0, 1, -1, 3, -3, 40, -40, 10**12, -(10**12)])
def test_shift_periods(plb, periods):
    rng = np.random.default_rng(1)
    n = 2 * TILE + 9
    g = rng.integers(0, 3, n)
    glen = int(np.bincount(g).max())
    x = rng.standard_normal(n)
    for p in (periods, glen, -glen):
        got = plb.over([("shift", x, {"periods": p})], partition_by=[g])[0]
        exp = wo.over([("shift", x.tolist(), "float64", {"periods": p})], [g.tolist()], n)[0]
        assert all(same(a, b) for a, b in zip(as_list(*got), exp))
    got = plb.over([("shift", x, {"periods": periods})])[0]      # no partition: the shifted copy
    exp = wo.over([("shift", x.tolist(), "float64", {"periods": periods})], [], n)[0]
    assert all(same(a, b) for a, b in zip(as_list(*got), exp))


AGGS = ["sum", "mean", "min", "max", "count", "len", "first", "last", "var", "std:0", "n_unique", "median", "quantile:0.3:linear", "quantile:0.7:nearest"]


@pytest.mark.parametrize("dtype", ["int16", "int64", "uint32", "float32", "float64"])
@pytest.mark.parametrize("deterministic", [False, True])
def test_aggregations_equal_group_by(plb, dtype, deterministic):
    """every aggregation broadcast equals bl_groupby_agg_params gathered by group: exact kinds byte for byte; float sums and
    means too in deterministic mode (the same GroupsIdx plan), within the group_by's own bar otherwise"""
    rng = np.random.default_rng(3)
    n = 3 * TILE + 5
    g = rng.integers(0, 40, n)
    x, valid = values(rng, dtype, n, True)
    col = (x, valid)
    plb.set_deterministic(deterministic)
    try:
        got = plb.over([(k, col if k != "len" else None) for k in AGGS], partition_by=[g])
        first_row = {}
        for r, k in enumerate(g.tolist()):
            first_row.setdefault(k, r)
        keys, gb = plb.group_by_agg_keys([g], [(k, col if k != "len" else None) for k in AGGS if k != "n_unique"], maintain_order=True)
        _, nu = plb.group_by_agg(g, [("n_unique", col)], maintain_order=True)
    finally:
        plb.set_deterministic(False)
    ordinal = {int(k): i for i, k in enumerate(keys[0][0])}
    rows_ord = np.array([ordinal[int(k)] for k in g])
    gb = gb[:AGGS.index("n_unique")] + nu + gb[AGGS.index("n_unique"):]
    for kind, gg, (ev, em) in zip(AGGS, got, gb):
        exp_v = ev[rows_ord]
        exp_m = None if em is None else em[rows_ord]
        gv, gm = gg
        assert gv.dtype == ev.dtype, kind
        assert (gm is None) == (exp_m is None) or np.array_equal(gm if gm is not None else np.ones(n, bool), exp_m if exp_m is not None else np.ones(n, bool)), kind
        ok = np.ones(n, bool) if gm is None else gm
        if deterministic or kind not in ("sum", "mean", "var", "std:0") or not dtype.startswith("float") and kind in ("sum",):
            assert np.array_equal(gv[ok].view(np.uint8), exp_v[ok].view(np.uint8)) or np.array_equal(gv[ok], exp_v[ok], equal_nan=True), kind
        else:
            assert np.allclose(gv[ok], exp_v[ok], rtol=1e-9 if dtype == "float64" else 1e-5, equal_nan=True), kind


def test_deterministic_float_scans_bit_identical(plb):
    rng = np.random.default_rng(4)
    n = 5 * TILE + 3
    g = rng.integers(0, 4, n)
    for dtype in ("float32", "float64"):
        x = (rng.standard_normal(n) * 1e3).astype(dtype)
        ops = [("cum_sum", x, {}), ("cum_prod", (rng.random(n) + 0.5).astype(dtype), {"reverse": True})]
        plb.set_deterministic(True)
        try:
            got = plb.over(ops, partition_by=[g])
            whole = plb.cum_agg("cum_sum", x)
        finally:
            plb.set_deterministic(False)
        exp = wo.over([(k, as_list(c, None), dtype, o) for k, c, o in ops], [g.tolist()], n)
        for gg, e in zip(got, exp):
            assert all(same(a, b) for a, b in zip(as_list(*gg), e)), dtype
        assert all(same(a, b) for a, b in zip(as_list(*whole), wo.cum_seq("cum_sum", as_list(x, None), dtype)))


def test_exactly_summable_2e7_rows_in_1e5_partitions(plb):
    rng = np.random.default_rng(6)
    n = 20_000_000
    g = rng.integers(0, 100_000, n)
    x = rng.integers(-1000, 1000, n).astype(np.float64)
    got = plb.over([("cum_sum", x, {}), ("cum_sum", x.astype(np.int64), {"reverse": True}), ("mean", x)], partition_by=[g])
    order = np.lexsort((np.arange(n), g))
    head = np_segments(g[order])
    es = np.empty(n, np.int64)
    es[order] = np_cumsum_seg(x.astype(np.int64)[order].view(np.uint64), head).view(np.int64)
    assert np.array_equal(got[0][0], es.astype(np.float64))
    whole = plb.cum_agg("cum_sum", x)
    assert np.array_equal(whole[0], np.cumsum(x))
    rs = np.empty(n, np.int64)
    rord = order[::-1]
    rs[rord] = np_cumsum_seg(x.astype(np.int64)[rord].view(np.uint64), np_segments(g[rord])).view(np.int64)
    assert np.array_equal(got[1][0], rs)


def test_one_partition_order_per_call(plb):
    rng = np.random.default_rng(8)
    n = 4 * TILE
    g = rng.integers(0, 10, n)
    t = rng.integers(0, 100, n)
    x = rng.integers(0, 9, n)
    for order in (None, t):
        plb.profile_reset()
        plb.profile_enable(True)
        ops = [("cum_sum", x, {}), ("cum_max", x, {"reverse": True}), ("shift", x, {"periods": 2}), ("cum_count", x, {})]
        if order is not None:
            ops.append(("first", x))      # with order_by, aggregations fold over the same order
        plb.over(ops, partition_by=[g], order_by=order)
        prof = plb.profile()
        plb.profile_enable(False)
        assert prof["k5_run_starts"]["launches"] == 1, prof
    plb.profile_reset()
    plb.profile_enable(True)
    plb.over([("sum", x), ("max", x), ("count", x)], partition_by=[g])
    prof = plb.profile()
    plb.profile_enable(False)
    assert not any(k.startswith("sort_") or k.startswith("k5x_") for k in prof), prof.keys()


def test_single_row_and_empty(plb):
    one = plb.over([("cum_sum", np.array([5], np.int8), {}), ("shift", np.array([5.0]), {}), ("sum", np.array([7]))], partition_by=[np.array([1])])
    assert one[0][0].tolist() == [5] and one[0][0].dtype == np.int64
    assert one[1][1].tolist() == [False]
    assert one[2][0].tolist() == [7]
    empty = plb.over([("cum_prod", np.zeros(0, np.int32), {}), ("mean", np.zeros(0, np.int32))], partition_by=[np.zeros(0, np.int64)])
    assert empty[0][0].dtype == np.int64 and len(empty[0][0]) == 0
    assert empty[1][0].dtype == np.float64


def test_device_inputs_and_outputs(plb):
    rng = np.random.default_rng(12)
    n = 3 * TILE
    x = rng.integers(-9, 9, n).astype(np.int32)
    m = rng.random(n) > 0.3
    g = rng.integers(0, 4, n)
    dx, dg = plb.to_device(x, m), plb.to_device(g)
    outs = plb.over([("cum_sum", dx, {}), ("shift", dx, {"periods": 1})], partition_by=[dg], location=plb.DEVICE)
    host = plb.over([("cum_sum", (x, m), {}), ("shift", (x, m), {"periods": 1})], partition_by=[g])
    for d, h in zip(outs, host):
        dv, dm = d.to_numpy()
        assert np.array_equal(dv[h[1]] if h[1] is not None else dv, h[0][h[1]] if h[1] is not None else h[0])
        assert (dm is None) == (h[1] is None) or np.array_equal(dm, h[1])


def test_errors(plb):
    B = plb.B200Error
    with pytest.raises(B, match="UNSUPPORTED"):
        plb.over([("cum_min", np.array([True, False]), {})])
    with pytest.raises(B, match="UNSUPPORTED"):
        plb.over([("shift", np.array([True, False]), {})])
    with pytest.raises(B, match="INVALID"):
        plb.over([("cum_sum", np.arange(3), {}), ("cum_sum", np.arange(4), {})])
    with pytest.raises(B, match="INVALID"):
        plb.over([("cum_sum", np.arange(3), {})], partition_by=[np.arange(4)])
    import ctypes as C
    bad = (plb.BlOverOp * 1)(plb.BlOverOp(99, 0, 0, None, plb.BlAggParam(0.0, 0, 0)))
    x = plb.Column(np.arange(3))
    st = x.struct()
    bad[0].values = C.pointer(st)
    outs = (plb.BlColumn * 1)()
    assert plb.lib().bl_over(None, 0, None, bad, 1, plb.HOST, outs) == 1
    key = plb.BlSortKey(C.pointer(st), None, 0, 1)
    bad[0].kind = 32
    assert plb.lib().bl_over(C.byref(key), 1, None, bad, 1, plb.HOST, outs) == 1      # partition flags must be 0


def test_plugin_entries(plb):
    """_polars_plugin_bl_cum_* / bl_shift through the expression-plugin ABI: input 0 the values, then the partition keys;
    kwargs reverse / periods; one row per input row, nulls included, compared with the oracle"""
    pa = pytest.importorskip("pyarrow")
    from test_gpu_plugin_abi import Caller
    caller = Caller(plb.lib())
    rng = np.random.default_rng(13)
    n = 3 * TILE + 21
    x = rng.integers(-1000, 1000, n).astype(np.int64)
    valid = rng.random(n) >= 0.15
    g1 = rng.integers(0, 7, n)
    g2 = rng.integers(0, 2, n).astype(np.int32)
    xs = as_list(x, valid)
    X = pa.array(x, mask=~valid)
    cases = [
        ("cum_sum", {"reverse": True}, [g1, g2], ("cum_sum", {"reverse": True})),
        ("cum_sum", None, [g1], ("cum_sum", {})),
        ("cum_max", {"reverse": False}, [], ("cum_max", {})),
        ("cum_count", {"reverse": True}, [g1], ("cum_count", {"reverse": True})),
        ("shift", {"periods": -2}, [g1, g2], ("shift", {"periods": -2})),
        ("shift", None, [g1], ("shift", {"periods": 1})),
    ]
    for entry, kwargs, keys, (kind, opts) in cases:
        inputs = [("x", [X.slice(0, 1000), X.slice(1000)])] + [(f"k{i}", [pa.array(k)]) for i, k in enumerate(keys)]
        out = caller.call(entry, inputs, kwargs)
        exp = wo.over([(kind, xs, "int64", opts)], [k.tolist() for k in keys], n)[0]
        assert out.type == (pa.uint32() if kind == "cum_count" else pa.int64()), (entry, out.type)
        got = out.to_pylist()
        assert got == exp, (entry, kwargs, next(i for i, (a, b) in enumerate(zip(got, exp)) if a != b))
