"""CPU tests (-m "not gpu"): pin the oracle against the reference's golden vectors and
cross-check it against independent engines (pyarrow Acero, numpy) on random inputs."""
import zlib

import numpy as np
import pyarrow as pa
import pytest

import join_keys
import oracle
from helpers import IDX_NULL, OracleImpl, assert_close, col, pairs_sorted, run_group_by_kat, run_join_kat, sort_groups


# ---------------------------------------------------------------- golden vectors
def test_hash_partition_kat(kats):
    vecs = kats["hash"][0]["vectors"]
    keys = np.array([int(v["key_u64"]) for v in vecs], dtype=np.uint64)
    h = oracle.dirty_hash(keys)
    assert [int(x) for x in h] == [int(v["dirty_hash"]) for v in vecs]
    for P in (1, 2, 3, 7, 8, 16, 148):
        p = oracle.hash_to_partition(h, P)
        assert [int(x) for x in p] == [v["part"][str(P)] for v in vecs]


@pytest.mark.parametrize("threads", [1, 2, 4, 7])
def test_group_by_kats(kats, threads):
    for case in kats["group_by"]:
        run_group_by_kat(OracleImpl(threads), case)


def test_group_by_ordered_agg_kats(kats):
    """first / last / var / std (GroupsIdx-ordered aggregations) and the shorthand table of the reference's tests."""
    for case in kats["group_by_ordered"]:
        run_group_by_kat(OracleImpl(2), case)


def test_join_kats(kats):
    for case in kats["join"]:
        impl = OracleImpl()
        run_join_kat(impl, case, set_threads=lambda t: setattr(impl, "n_threads", t))


# ---------------------------------------------------------------- cross-checks
def _arrow(values, valid):
    return pa.array(values, mask=None if valid is None else ~valid)


@pytest.mark.parametrize("n,k,nulls", [(0, 5, False), (1, 1, False), (1000, 7, True), (1001, 50, True), (50_000, 1000, True), (200_000, 100_000, False)])
def test_group_by_vs_acero(n, k, nulls):
    rng = np.random.default_rng(n + k)
    key = rng.integers(-k // 2, k // 2 + 1, n).astype(np.int64)
    vi = rng.integers(-1000, 1000, n).astype(np.int64)
    vf = rng.uniform(0, 100, n).round(6)
    kvalid = (rng.random(n) > 0.05) if nulls else None
    ivalid = (rng.random(n) > 0.05) if nulls else None
    fvalid = (rng.random(n) > 0.3) if nulls else None
    aggs = [("sum", vi, ivalid), ("mean", vf, fvalid), ("len", None, None), ("min", vi, ivalid), ("max", vf, fvalid),
            ("count", vf, fvalid), ("sum", vf, fvalid), ("mean", vi, ivalid)]
    for threads, order in [(1, True), (4, True), (8, False)]:
        keys, kv, outs, g = oracle.group_by_agg(key, kvalid, aggs, threads, order)
        if order and n:
            assert np.all(np.diff(g.first.astype(np.int64)) > 0)           # first-occurrence order
            # first really is the first row of that key
            for gi in range(min(len(g), 50)):
                rows = g.idx[g.offsets[gi]:g.offsets[gi + 1]]
                assert rows[0] == g.first[gi] and np.all(np.diff(rows.astype(np.int64)) > 0)
        tbl = pa.table({"k": _arrow(key, kvalid), "vi": _arrow(vi, ivalid), "vf": _arrow(vf, fvalid)})
        ref = tbl.group_by("k", use_threads=False).aggregate(
            [("vi", "sum"), ("vf", "mean"), ([], "count_all"), ("vi", "min"), ("vf", "max"), ("vf", "count"), ("vf", "sum"), ("vi", "mean")])
        rk = ref["k"].to_numpy(zero_copy_only=False)
        rkv = ~np.array(ref["k"].is_null().to_pylist(), dtype=bool) if n else np.zeros(0, bool)
        rk = np.where(rkv, rk, 0).astype(np.int64) if n else np.zeros(0, np.int64)
        names = ["vi_sum", "vf_mean", "count_all", "vi_min", "vf_max", "vf_count", "vf_sum", "vi_mean"]
        routs = []
        for nm, (kind, _, _) in zip(names, aggs):
            c = ref[nm]
            m = ~np.array(c.is_null().to_pylist(), dtype=bool)
            v = np.array([0 if x is None else x for x in c.to_pylist()])
            routs.append((v, None if m.all() else m))
        keys, kv, outs = sort_groups(keys, kv, outs)
        rk, rkv2, routs = sort_groups(rk, None if rkv.all() else rkv, routs)
        assert_close(keys, rk, kv, rkv2, "keys")
        for (kind, _, _), (v, m), (rv, rm) in zip(aggs, outs, routs):
            if kind == "sum":
                # Acero: all-null group sum is null; reference: 0 (aggregations/mod.rs:862-865)
                rv = np.where(np.ones(rv.shape, bool) if rm is None else rm, rv, 0)
                rm = None
            assert_close(v.astype(np.float64) if kind in ("len", "count") else v,
                         rv.astype(np.float64) if kind in ("len", "count") else rv.astype(v.dtype), m, rm, kind)


def test_sum_semantics_edge():
    # wrapping int sum, all-null group sums to 0 / means to null, NaN handling of min/max
    key = np.array([0, 0, 1, 1, 2, 2, 3], np.int64)
    vi = np.array([2**62, 2**62, 1, 2, 5, 6, 7], np.int64)
    valid = np.array([1, 1, 0, 0, 1, 0, 1], bool)
    _, _, outs, _ = oracle.group_by_agg(key, None, [("sum", vi, valid), ("mean", vi, valid), ("min", vi, valid), ("count", vi, valid), ("len", None, None)], 1, True)
    assert outs[0][0].tolist() == [-2**63, 0, 5, 7] and outs[0][1] is None
    assert outs[1][1].tolist() == [True, False, True, True]
    assert outs[2][1].tolist() == [True, False, True, True] and outs[2][0][2] == 5
    assert outs[3][0].tolist() == [2, 0, 1, 1] and outs[4][0].tolist() == [2, 2, 2, 1]
    vf = np.array([np.nan, 1.0, np.nan, np.nan, -0.0, 3.0, np.inf])
    _, _, outs, _ = oracle.group_by_agg(key, None, [("min", vf, None), ("max", vf, None)], 1, True)
    assert outs[0][0][0] == 1.0 and np.isnan(outs[0][0][1]) and outs[1][0][2] == 3.0 and outs[0][0][3] == np.inf


def test_float_keys_canonical():
    key = np.array([0.0, -0.0, np.nan, -np.nan, 1.5, np.float64.fromhex("0x1.8p0")])
    keys, _, outs, g = oracle.group_by_agg(key, None, [("len", None, None)], 1, True)
    assert outs[0][0].tolist() == [2, 2, 2]
    assert np.signbit(keys[0]) == False and g.first.tolist() == [0, 2, 4]  # noqa: E712


@pytest.mark.parametrize("nl,nr,krange,dups", [(0, 0, 10, 1), (5, 0, 10, 1), (300, 100, 150, 1), (2000, 3000, 500, 3), (40_000, 10_000, 20_000, 2)])
def test_join_vs_bruteforce(nl, nr, krange, dups):
    rng = np.random.default_rng(nl * 7 + nr)
    lk = rng.integers(0, krange, nl).astype(np.int64)
    rk = np.repeat(rng.permutation(max(krange, nr))[: max(nr // dups, 0)], dups)[:nr].astype(np.int64)
    rk = np.concatenate([rk, rng.integers(0, krange, nr - rk.size).astype(np.int64)])
    rng.shuffle(rk)
    lv = rng.random(nl) > 0.1
    rv = rng.random(nr) > 0.1
    for nulls_equal in (False, True):
        for threads in (1, 3, 8):
            li, ri = oracle.hash_join(lk, rk, lv, rv, "inner", nulls_equal, "none", threads)
            # brute force with pandas-free numpy: sort-merge on (valid, key)
            exp = []
            from collections import defaultdict
            d = defaultdict(list)
            for j in range(nr):
                if rv[j] or nulls_equal:
                    d[(bool(rv[j]), int(rk[j]) if rv[j] else 0)].append(j)
            for i in range(nl):
                if lv[i] or nulls_equal:
                    for j in d.get((bool(lv[i]), int(lk[i]) if lv[i] else 0), []):
                        exp.append((i, j))
            got = sorted(zip(li.tolist(), ri.tolist()))
            assert got == sorted(exp)
            # ordering rule (hash_join/mod.rs:41-50): probe side ascending, build idx ascending per probe row
            if nl > nr:
                assert np.all(np.diff(li.astype(np.int64)) >= 0)
                same = np.diff(li.astype(np.int64)) == 0
                assert np.all(np.diff(ri.astype(np.int64))[same] > 0)
            elif li.size:
                assert np.all(np.diff(ri.astype(np.int64)) >= 0)
                same = np.diff(ri.astype(np.int64)) == 0
                assert np.all(np.diff(li.astype(np.int64))[same] > 0)
            # left join: every left row appears; misses have null right
            l2, r2 = oracle.hash_join(lk, rk, lv, rv, "left", nulls_equal, "none", threads)
            assert np.all(np.diff(l2.astype(np.int64)) >= 0) and set(l2.tolist()) == set(range(nl))
            hit = r2 != IDX_NULL
            assert np.array_equal(pairs_sorted(l2[hit], r2[hit]), pairs_sorted(li, ri))


def test_join_vs_acero():
    rng = np.random.default_rng(5)
    lk = rng.integers(0, 5000, 30_000).astype(np.int64)
    rk = rng.integers(0, 5000, 8_000).astype(np.int64)
    li, ri = oracle.hash_join(lk, rk, None, None, "inner", False, "none", 4)
    lt = pa.table({"k": lk, "li": np.arange(lk.size, dtype=np.uint32)})
    rt = pa.table({"k": rk, "ri": np.arange(rk.size, dtype=np.uint32)})
    j = lt.join(rt, "k", join_type="inner")
    assert np.array_equal(pairs_sorted(li, ri), pairs_sorted(j["li"].to_numpy(), j["ri"].to_numpy()))


# ---------------------------------------------------------------- elementwise / filter / gather
@pytest.mark.parametrize("dtype", ["int64", "int32", "uint64", "uint32", "float64", "float32"])
def test_arith_vs_numpy(dtype):
    rng = np.random.default_rng(11)
    dt = np.dtype(dtype)
    n = 1000
    if dt.kind == "f":
        a = rng.normal(0, 100, n).astype(dt)
        b = rng.normal(0, 100, n).astype(dt)
        b[::17] = 0
        a[::31] = np.nan
    else:
        lo = 0 if dt.kind == "u" else -1000
        a = rng.integers(lo, 1000, n).astype(dt)
        b = rng.integers(lo, 1000, n).astype(dt)
        b[::17] = 0
        if dt.kind == "i":
            a[0], b[0] = np.iinfo(dt).min, -1          # wrapping_div overflow case
    av = rng.random(n) > 0.1
    with np.errstate(all="ignore"):
        for op, f in [("add", np.add), ("sub", np.subtract), ("mul", np.multiply)]:
            out, v = oracle.arith(op, a, b, av, None)
            assert np.array_equal(out, f(a, b), equal_nan=True) and np.array_equal(v, av)
        out, v = oracle.arith("floordiv", a, b, av, None)
        if dt.kind == "f":
            assert np.array_equal(out, np.floor(a / b), equal_nan=True) and np.array_equal(v, av)
            out, _ = oracle.arith("mod", a, b)
            assert np.array_equal(out, a - b * np.floor(a / b), equal_nan=True)
        else:
            nz = b != 0
            assert np.array_equal(v, av & nz)
            ok = nz.copy()
            ok[0] = False
            assert np.array_equal(out[ok], np.floor_divide(a[ok], b[ok]))
            if dt.kind == "i":
                assert out[0] == np.iinfo(dt).min          # MIN // -1 wraps
            out, v = oracle.arith("mod", a, b, av, None)
            assert np.array_equal(out[ok], np.mod(a[ok], b[ok])) and np.all(out[~nz] == 0)
            out, v = oracle.arith("truediv", a, b)
            assert out.dtype == np.float64 and np.array_equal(out[nz], a[nz].astype(np.float64) / b[nz].astype(np.float64))
        # scalar forms
        out, _ = oracle.arith("add", a, dt.type(3))
        assert np.array_equal(out, a + dt.type(3), equal_nan=True)
        out, _ = oracle.arith("sub", dt.type(3), a)
        assert np.array_equal(out, dt.type(3) - a, equal_nan=True)
        if dt.kind == "f":
            out, _ = oracle.arith("truediv", a, dt.type(3))
            assert np.array_equal(out, a * (dt.type(1) / dt.type(3)), equal_nan=True)   # float.rs:113-115
        else:
            out, v = oracle.arith("floordiv", a, dt.type(0))
            assert v is not None and not v.any()                                      # signed.rs:103-105


@pytest.mark.parametrize("dtype", ["int64", "float64", "float32", "uint32"])
def test_compare_total_order(dtype):
    dt = np.dtype(dtype)
    if dt.kind == "f":
        a = np.array([1.0, np.nan, np.nan, -np.inf, 0.0, -0.0, 5.0], dt)
        b = np.array([2.0, np.nan, 1.0, np.nan, -0.0, 0.0, 5.0], dt)
        exp = {"eq": [0, 1, 0, 0, 1, 1, 1], "ne": [1, 0, 1, 1, 0, 0, 0], "lt": [1, 0, 0, 1, 0, 0, 0], "le": [1, 1, 0, 1, 1, 1, 1],
               "gt": [0, 0, 1, 0, 0, 0, 0], "ge": [0, 1, 1, 0, 1, 1, 1]}
    else:
        a = np.array([1, 5, 3, 0, 7, 7, 2], dt)
        b = np.array([2, 5, 1, 9, 7, 6, 2], dt)
        exp = {op: f(a, b).astype(int).tolist() for op, f in [("eq", np.equal), ("ne", np.not_equal), ("lt", np.less), ("le", np.less_equal), ("gt", np.greater), ("ge", np.greater_equal)]}
    av = np.array([1, 1, 1, 0, 1, 1, 0], bool)
    bv = np.array([1, 1, 1, 1, 1, 1, 0], bool)
    for op, e in exp.items():
        out, v = oracle.compare(op, a, b, av, bv)
        assert out.astype(int).tolist() == e, op
        assert np.array_equal(v, av & bv)
        out, v = oracle.compare(op, a, a[4])
        assert v is None
    out, v = oracle.compare("eq", a, b, av, bv, missing=True)
    assert v is None and out[3] == False and out[6] == True   # noqa: E712
    out, v = oracle.compare("ne", a, b, av, bv, missing=True)
    assert out[3] == True and out[6] == False                 # noqa: E712


def test_filter_gather_kat():
    # filter KAT generator of the reference: py-polars/tests/unit/operations/test_filter.py:271-286
    for size in list(range(0, 64)) + [100, 1000, 10_000]:
        for sel in (0.0, 0.01, 0.1, 0.5, 0.9, 0.99, 1.0):
            rng = np.random.Generator(np.random.PCG64(size * 100 + int(sel * 100)))
            mask = rng.random(size) < sel
            vals = rng.integers(-2**62, 2**62, size).astype(np.int64)
            valid = rng.random(size) > 0.2
            mvalid = rng.random(size) > 0.1
            out, ov = oracle.filter(vals, valid, mask, mvalid)
            keep = mask & mvalid
            assert np.array_equal(out, vals[keep]) and np.array_equal(ov, valid[keep])
    vals = np.arange(10, dtype=np.float64) * 1.5
    valid = np.arange(10) % 3 != 0
    idx = np.array([9, 0, 3, 3, 7], np.uint32)
    iv = np.array([1, 1, 0, 1, 1], bool)
    out, ov = oracle.gather(vals, valid, idx, iv)
    assert out.tolist() == [13.5, 0.0, 0.0, 4.5, 10.5] and ov.tolist() == [False, False, False, False, True]


def test_group_by_multi_kats(kats):
    from helpers import run_group_by_multi_kat
    for case in kats["group_by_multi"]:
        run_group_by_multi_kat(lambda k, v, a, o: oracle.group_by_agg_multi(k, v, a, o)[:2], case)


def test_group_by_multi_matches_single_key_and_pyarrow():
    import pyarrow as pa
    rng = np.random.default_rng(8)
    n = 20_000
    a, b = rng.integers(0, 30, n).astype(np.int32), rng.integers(-5, 5, n).astype(np.int64)
    av = rng.random(n) > 0.1
    v = rng.integers(-100, 100, n).astype(np.int64)
    g1, g2 = oracle.group_by(a, av, 4, True), oracle.group_by_multi([a], [av], True)
    assert np.array_equal(g1.first, g2.first) and np.array_equal(g1.offsets, g2.offsets) and np.array_equal(g1.idx, g2.idx)
    kouts, outs, _ = oracle.group_by_agg_multi([a, b], [av, None], [("sum", v, None), ("len", None, None)], True)
    t = pa.table({"a": pa.array(a, mask=~av), "b": b, "v": v}).group_by(["a", "b"]).aggregate([("v", "sum"), ([], "count_all")]).to_pydict()
    exp = {(x, y): (s, c) for x, y, s, c in zip(t["a"], t["b"], t["v_sum"], t["count_all"])}
    got = {(None if (kouts[0][1] is not None and not kouts[0][1][i]) else int(kouts[0][0][i]), int(kouts[1][0][i])): (int(outs[0][0][i]), int(outs[1][0][i])) for i in range(len(outs[0][0]))}
    assert got == exp


@pytest.mark.parametrize("nulls_equal", [False, True])
def test_semi_anti_vs_bruteforce_and_acero(nulls_equal):
    # single_keys_semi_anti.rs:41-140 restated as set membership; cross-checked against a brute-force loop and Acero
    import pyarrow as pa
    rng = np.random.default_rng(17)
    nl, nr = 600, 90
    lk, rk = rng.integers(0, 120, nl).astype(np.int64), rng.integers(0, 120, nr).astype(np.int64)
    lv, rv = rng.random(nl) > 0.1, rng.random(nr) > 0.1
    right_has_null = bool((~rv).any())
    exp = np.array([(lv[i] and bool(((rk == lk[i]) & rv).any())) or (nulls_equal and not lv[i] and right_has_null) for i in range(nl)])
    semi, _ = oracle.hash_join(lk, rk, lv, rv, "semi", nulls_equal, "none", 4)
    anti, _ = oracle.hash_join(lk, rk, lv, rv, "anti", nulls_equal, "none", 4)
    assert np.array_equal(semi, np.nonzero(exp)[0]) and np.array_equal(anti, np.nonzero(~exp)[0])
    if not nulls_equal:      # Acero's semi/anti joins never match nulls
        lt = pa.table({"k": pa.array(lk, mask=~lv), "i": np.arange(nl)})
        rt = pa.table({"k": pa.array(rk, mask=~rv)})
        for how, got in (("left semi", semi), ("left anti", anti)):
            idx = np.sort(lt.join(rt, keys="k", join_type=how).column("i").to_numpy())
            assert np.array_equal(idx, got), how


@pytest.mark.parametrize("dtype", ["int8", "uint8", "int16", "uint16"])
def test_small_int_aggregation_rules(dtype):
    # series/implementations/mod.rs:145-154: 8/16-bit sums are computed (and returned) as Int64 — no wrap-around
    rng = np.random.default_rng(23)
    info = np.iinfo(dtype)
    n = 50_000
    key = rng.integers(0, 4, n).astype(np.int64)
    val = rng.integers(info.min, int(info.max) + 1, n).astype(dtype)
    valid = rng.random(n) > 0.2
    ek, _, outs, _ = oracle.group_by_agg(key, None, [("sum", val, valid), ("mean", val, valid), ("min", val, valid), ("max", val, valid)], 2, True)
    for g, k in enumerate(ek):
        sel = (key == k) & valid
        wide = val[sel].astype(np.int64)
        assert outs[0][0].dtype == np.int64 and outs[0][0][g] == wide.sum()
        assert outs[1][0].dtype == np.float64 and abs(outs[1][0][g] - wide.mean()) < 1e-9
        assert outs[2][0].dtype == np.dtype(dtype) and outs[2][0][g] == wide.min() and outs[3][0][g] == wide.max()


def test_join_multi_kats(kats):
    # multi-column join keys are not on the GPU path yet (NEXT.md); the oracle restatement is pinned already
    from helpers import col
    for case in kats["join_multi"]:
        lk = [col(k, case["key_dtype"]) for k in case["left_keys"]]
        rk = [col(k, case["key_dtype"]) for k in case["right_keys"]]
        for threads in (1, 4):
            li, ri = oracle.hash_join_multi([k for k, _ in lk], [k for k, _ in rk], [v for _, v in lk], [v for _, v in rk], case["how"], case["nulls_equal"], "none", threads)
            assert li.tolist() == case["expect_left_idx"], case["cite"]
            assert ri.tolist() == [IDX_NULL if x is None else x for x in case["expect_right_idx"]], case["cite"]


def test_join_multi_matches_acero():
    rng = np.random.default_rng(31)
    nl, nr = 3000, 800
    la, lb = rng.integers(0, 40, nl).astype(np.int64), rng.integers(0, 6, nl).astype(np.int32)
    ra, rb = rng.integers(0, 40, nr).astype(np.int64), rng.integers(0, 6, nr).astype(np.int32)
    lbv, rbv = rng.random(nl) > 0.1, rng.random(nr) > 0.1
    li, ri = oracle.hash_join_multi([la, lb], [ra, rb], [None, lbv], [None, rbv], "inner", False, "none", 4)
    lt = pa.table({"a": la, "b": pa.array(lb, mask=~lbv), "i": np.arange(nl)})
    rt = pa.table({"a": ra, "b": pa.array(rb, mask=~rbv), "j": np.arange(nr)})
    j = lt.join(rt, keys=["a", "b"], join_type="inner")
    exp = sorted(zip(j.column("i").to_pylist(), j.column("j").to_pylist()))
    assert sorted(zip(li.tolist(), ri.tolist())) == exp


@pytest.mark.parametrize("nl,nr,krange", [(0, 0, 5), (7, 0, 5), (0, 7, 5), (50, 80, 30), (400, 300, 200), (2000, 2500, 50)])
@pytest.mark.parametrize("nulls_equal", [False, True])
def test_full_join_vs_bruteforce(nl, nr, krange, nulls_equal):
    """hash_join_tuples_outer (single_keys_outer.rs:100-260): the matched pairs are the inner-join pairs, every left and
    every right row appears at least once, unmatched rows carry a null on the other side; the probe-phase tuples come
    first in probe order (longer side probes, tie -> right)."""
    rng = np.random.default_rng(nl * 3 + nr + int(nulls_equal))
    lk = rng.integers(0, krange, nl).astype(np.int64); rk = rng.integers(0, krange, nr).astype(np.int64)
    lv = rng.random(nl) > 0.15; rv = rng.random(nr) > 0.15
    li, ri = oracle.hash_join(lk, rk, lv, rv, "full", nulls_equal, "none", 3)
    NUL = oracle.IDX_NULL
    exp = set()
    lm, rm = np.zeros(nl, bool), np.zeros(nr, bool)
    for i in range(nl):
        for j in range(nr):
            if (lv[i] and rv[j] and lk[i] == rk[j]) or (nulls_equal and not lv[i] and not rv[j]):
                exp.add((i, j)); lm[i] = True; rm[j] = True
    exp |= {(i, int(NUL)) for i in range(nl) if not lm[i]} | {(int(NUL), j) for j in range(nr) if not rm[j]}
    got = list(zip(li.tolist(), ri.tolist()))
    assert len(got) == len(set(got)) == len(exp) and set(got) == exp
    # probe phase first, in probe order; drained build rows last
    probe_side = ri if not (nl > nr) else li
    k = int((probe_side != NUL).sum())
    assert (probe_side[:k] != NUL).all() and np.all(np.diff(probe_side[:k].astype(np.int64)) >= 0) and (probe_side[k:] == NUL).all()


def bruteforce_join(lk, lv, rk, rv, how, nulls_equal, order="none"):
    """The reference's tuple sequence from its rules alone (hash_join/mod.rs:41-50, single_keys_outer.rs:100-260,
    single_keys_semi_anti.rs:8-140, join/mod.rs:577-642, dispatch_left_right.rs:142-170), over join_keys.canon keys.
    Returns (left idx, right idx) as lists; IDX_NULL marks a missing side."""
    NUL = int(IDX_NULL)
    lc, rc = join_keys.canon(lk, lv), join_keys.canon(rk, rv)

    def rows_by_key(c):
        d = {}
        for j, x in enumerate(c):
            if x is not None or nulls_equal:
                d.setdefault(x, []).append(j)
        return d

    def left_join(pc, bc):           # every probe row in order; its matches ascending, or one miss
        d = rows_by_key(bc)
        out = []
        for i, x in enumerate(pc):
            m = d.get(x, []) if (x is not None or nulls_equal) else []
            out += [(i, j) for j in m] or [(i, NUL)]
        return out

    if how in ("semi", "anti"):
        d = rows_by_key(rc)
        hit = [(x is not None or nulls_equal) and x in d for x in lc]
        return [i for i, h in enumerate(hit) if h == (how == "semi")], []
    swapped = not (len(lc) > len(rc)) if how in ("inner", "full") else False
    pc, bc = (rc, lc) if swapped else (lc, rc)
    seq = left_join(pc, bc)
    if how == "inner":
        seq = [t for t in seq if t[1] != NUL]
    if how == "full":
        hit = {j for _, j in seq}
        seq += [(NUL, j) for j in range(len(bc)) if j not in hit]
    if swapped:
        seq = [(b, p) for p, b in seq]
    if order in ("left", "left_right") and how == "inner":
        seq = sorted(seq, key=lambda t: t[0])
    elif order in ("right", "right_left") and how in ("inner", "left"):
        seq = sorted(seq, key=lambda t: t[1])
    return [t[0] for t in seq], [t[1] for t in seq]


def _full_range_cases():
    cases = []
    for dt in join_keys.DTYPES:
        for dups in ("unique", "k", "hot", "dense"):
            if dups == "dense" and dt not in join_keys.INT_DTYPES:
                continue
            for nulls in (0, 0.04):
                cases.append((dt, dups, nulls))
    return cases


@pytest.mark.parametrize("dtype,dups,nulls", _full_range_cases())
def test_join_full_range_vs_bruteforce(dtype, dups, nulls):
    """The oracle's join (every how, both nulls_equal, every maintain_order) against the brute-force restatement above,
    on the key columns of tests/join_keys.py: the dtype's whole range with MIN / MAX / 0 / -1, UInt64 2^63 and 2^64 - 1,
    NaN payloads of both signs, +-0.0, +-inf and subnormals.  These are the inputs the GPU join is compared with the
    oracle on."""
    rng = np.random.default_rng(zlib.crc32(f"{dtype}/{dups}/{nulls}".encode()))
    small = np.dtype(dtype).itemsize == 1
    nr = 200 if small else 700
    if dups == "dense":
        rk, rv = join_keys.keys(rng, dtype, nr, "unique", nulls=nulls, dense=min(3 * nr, 256) if small else 3 * nr)
    else:
        rk, rv = join_keys.keys(rng, dtype, nr, dups, k={"unique": 1, "k": 3, "hot": 40}[dups], nulls=nulls)
    valid_rk = rk if rv is None else rk[rv]
    for nl in (2 * nr + 1, nr // 2, nr):            # left probes / right probes / a tie (right probes)
        lk, lv = join_keys.probe(rng, valid_rk, nl, nulls=nulls, dense_edges=dups == "dense")
        for nulls_equal in (False, True):
            for how, orders in (("inner", ("none", "left", "left_right", "right", "right_left")),
                                ("left", ("none", "left", "right", "right_left")), ("full", ("none",)), ("semi", ("none",)), ("anti", ("none",))):
                for order in orders:
                    eli, eri = bruteforce_join(lk, lv, rk, rv, how, nulls_equal, order)
                    li, ri = oracle.hash_join(lk, rk, lv, rv, how, nulls_equal, order, 3)
                    assert li.tolist() == eli and ri.tolist() == eri, (nl, how, nulls_equal, order)


def test_first_last_var_std_vs_numpy():
    """agg_first / agg_last / agg_var / agg_std restatements against numpy on every group (ddof 0, 1, 2; nulls; count <= ddof -> null)."""
    rng = np.random.default_rng(8)
    n = 30_000
    key = rng.integers(0, 400, n).astype(np.int64)
    x = rng.normal(1e5, 2.0, n); valid = rng.random(n) > 0.2
    key[:3] = 10_000; valid[:3] = [True, False, False]          # a group with one valid value: var(ddof=1) is null, var(ddof=0) is 0
    g = oracle.group_by(key, None, 4, True)
    rows = [np.nonzero(key == k)[0] for k in key[g.first]]
    f, fv = oracle.agg("first", x, valid, g); l, lv = oracle.agg("last", x, valid, g)
    fv = np.ones(len(g), bool) if fv is None else fv; lv = np.ones(len(g), bool) if lv is None else lv
    assert np.array_equal(fv, [valid[r[0]] for r in rows]) and np.array_equal(lv, [valid[r[-1]] for r in rows])
    assert np.array_equal(f[fv], np.array([x[r[0]] for r in rows])[fv]) and np.array_equal(l[lv], np.array([x[r[-1]] for r in rows])[lv])
    for ddof in (0, 1, 2):
        var, vv = oracle.agg(f"var:{ddof}", x, valid, g); std, sv = oracle.agg(f"std:{ddof}", x, valid, g)
        vv = np.ones(len(g), bool) if vv is None else vv
        cnt = np.array([valid[r].sum() for r in rows])
        assert np.array_equal(vv, cnt > ddof)
        exp = np.array([np.var(x[r][valid[r]], ddof=ddof) if c > ddof else 0.0 for r, c in zip(rows, cnt)])
        assert np.allclose(var[vv], exp[vv], rtol=1e-9, atol=0) and np.allclose(std[vv], np.sqrt(exp[vv]), rtol=1e-9, atol=0)


# ---------------------------------------------------------------- string keys (SURVEY.md 8(f1))
def test_string_codes_kats(kats):
    """The oracle's restatement of BinaryChunked::group_tuples against the reference's own string-key tests: the codes, the
    distinct keys in first-occurrence order, and the aggregates the reference asserts (computed over the codes)."""
    for case in kats["group_by_strings"]:
        codes, valid, nd = oracle.string_codes(case["key"])
        assert codes.tolist() == case["expect_codes"] and valid is None, case["cite"]
        assert nd == len(case["expect_key"]), case["cite"]
        run_group_by_kat(OracleImpl(2), dict(case, key=case["expect_codes"], key_dtype="uint32", expect_key=sorted(set(case["expect_codes"]))))
        firsts = list(dict.fromkeys(case["expect_codes"]))
        assert [case["key"][i] for i in firsts] == case["expect_key"], case["cite"]


@pytest.mark.parametrize("n,distinct,nulls", [(0, 1, False), (1, 1, True), (1000, 37, True), (50_000, 20_000, False)])
def test_string_codes_vs_arrow_dictionary(n, distinct, nulls):
    rng = np.random.default_rng(n + distinct)
    pool = [("k%d" % i) * int(rng.integers(0, 6)) + "x" * int(rng.integers(0, 3)) for i in range(distinct)]
    vals = [pool[int(j)] for j in rng.integers(0, distinct, n)]
    if nulls:
        vals = [None if rng.random() < 0.1 else v for v in vals]
    codes, valid, nd = oracle.string_codes(vals)
    d = pa.array(vals, type=pa.large_string()).dictionary_encode()
    idx = d.indices.to_numpy(zero_copy_only=False)
    mask = np.array([v is not None for v in vals], bool)
    assert nd == len(d.dictionary)
    if n:
        # arrow numbers the dictionary in first-occurrence order: value j first appears at the first row with index j
        first_row = np.full(len(d.dictionary), -1, np.int64)
        rows = np.flatnonzero(mask)
        ids = idx[mask].astype(np.int64)
        first_row[ids[::-1]] = rows[::-1]
        assert np.array_equal(codes[mask], first_row[ids].astype(np.uint32))
    assert (valid is None) == bool(mask.all())


def test_n_unique_kat_and_pandas(kats):
    import pandas as pd
    for case in kats["group_by_n_unique"]:
        key, kvalid = col(case["key"], case["key_dtype"])
        for c in case["cols"]:
            v, valid = col(c["col"], c["dtype"])
            _, counts = oracle.group_n_unique(key, kvalid, v, valid)
            assert counts.tolist() == c["expect"], case["cite"]
    rng = np.random.default_rng(3)
    n = 20_000
    key = rng.integers(0, 300, n).astype(np.int64)
    v = rng.integers(0, 40, n).astype(np.float64); v[rng.random(n) < 0.05] = np.nan
    valid = rng.random(n) > 0.1
    firsts, counts = oracle.group_n_unique(key, None, v, valid)
    # pandas: NaN and None are both "NA" there, so map NaN to a sentinel value first and count NA (= null) as one value
    s = pd.Series(np.where(np.isnan(v), -1.0, v)).where(valid)
    exp = s.groupby(key, sort=False).nunique(dropna=False)
    assert np.array_equal(key[firsts], exp.index.to_numpy()) and np.array_equal(counts, exp.to_numpy().astype(np.uint32))
