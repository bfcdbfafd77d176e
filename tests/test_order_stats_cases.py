"""CPU checks of tests/order_stats_cases.py: its references against sort_oracle, rank_oracle and rolling_quantile_oracle
by brute force on small inputs, and its top_k restatement against a brute-force MSD select."""
import math

import numpy as np
import pytest

import order_stats_cases as oc
import rank_oracle
import rolling_quantile_oracle as rqo
import sort_oracle

DTS = ["int8", "int32", "int64", "uint8", "uint64", "float32", "float64", "bool"]


def column(rng, dt, n, distinct=None):
    if dt == "bool":
        return rng.random(n) < 0.5
    if dt.startswith("float"):
        x = rng.integers(-6, 6, n).astype(dt) / 2 if distinct else rng.normal(size=n).astype(dt)
        x[rng.random(n) < 0.05] = np.nan
        x[rng.random(n) < 0.05] = -0.0
        return x
    info = np.iinfo(dt)
    lo, hi = (info.min, int(info.max) + 1) if not distinct else (max(info.min, -distinct), min(int(info.max) + 1, distinct))
    return rng.integers(lo, hi, n, dtype=np.int64 if dt != "uint64" else np.uint64).astype(dt)


def py(x, valid):
    return [None if (valid is not None and not valid[i]) else x[i].item() for i in range(len(x))]


# ------------------------------------------------------------------------------------------------ keys
@pytest.mark.parametrize("dt", DTS)
def test_value_key_orders_as_the_oracle(dt):
    rng = np.random.default_rng(DTS.index(dt))
    x = column(rng, dt, 300)
    key = oc.value_key(x, dt)
    exp = sort_oracle.arg_sort([x])
    got = np.lexsort((np.arange(len(x)), key))
    assert np.array_equal(got, exp)


# ------------------------------------------------------------------------------------------------ top_k
@pytest.mark.parametrize("dt", DTS)
@pytest.mark.parametrize("desc,nl", [(False, False), (True, True), (False, True), (True, False)])
def test_topk_reference_and_restatement(dt, desc, nl):
    rng = np.random.default_rng(100 + DTS.index(dt) * 4 + 2 * desc + nl)
    n = 257
    x = column(rng, dt, n, distinct=4)
    valid = rng.random(n) >= 0.2
    for k in (1, 2, 31, 100, 200, 256):
        exp = np.sort(sort_oracle.arg_sort([x], [valid], desc, nl, limit=k)).astype(np.uint32)
        assert np.array_equal(oc.topk_ref([x], [valid], k, desc, nl), exp), k
        for div in (1, 4, oc.TK_LIST_DIV, n):
            plan = oc.topk_plan([x], [valid], [dt], k, desc, nl, div)
            assert np.array_equal(plan["ids"], exp), (k, div)
            brute = oc.topk_msd_brute([x], [valid], [dt], k, desc, nl)
            for st, (p, sh, b, need, count) in zip(plan["steps"], brute):
                assert (st["part"], st["shift"], st["b"], st["need"], st["count"]) == (p, sh, b, need, count), (k, div)


def test_topk_restatement_two_columns_and_all_null():
    rng = np.random.default_rng(7)
    n = 600
    a = rng.integers(0, 3, n).astype(np.int32)
    b = rng.integers(-5, 5, n).astype(np.int64)
    va = rng.random(n) >= 0.3
    for k in (1, 10, 300, 599):
        for desc in ([False, True], [True, False]):
            exp = np.sort(sort_oracle.arg_sort([a, b], [va, None], desc, [True, False], limit=k)).astype(np.uint32)
            plan = oc.topk_plan([a, b], [va, None], ["int32", "int64"], k, desc, [True, False])
            assert np.array_equal(plan["ids"], exp)
    z = np.zeros(n, np.int32)
    for nl in (False, True):
        plan = oc.topk_plan([z], [np.zeros(n, bool)], ["int32"], 77, False, nl)
        assert np.array_equal(plan["ids"], np.arange(77, dtype=np.uint32))
        assert plan["launches"]["iota"] == 1 and plan["launches"]["topk_pass"] == 0


def test_topk_restatement_counts_row_digits():
    """the row index takes 1..4 digits at n = 2^8, 2^8 + 1, 2^16 + 1 and 2^24 + 1"""
    for n, d in ((2**8, 1), (2**8 + 1, 2), (2**16 + 1, 3), (2**24 + 1, 4)):
        assert (oc.bits_for(n - 1) + 7) // 8 == d


def test_topk_restatement_first_bucket_at_the_list_threshold():
    """a first bucket of n/32 - 1, n/32 and n/32 + 1 rows: a list from the next pass on at n/32, streaming above"""
    n = 32 * 100
    rng = np.random.default_rng(3)
    for size, listed in ((99, True), (100, True), (101, False)):
        x = (np.full(n, 5 << 8) | rng.integers(0, 256, n)).astype(np.uint32)
        x[np.linspace(0, n - 1, size).astype(np.int64)] &= 0xFF
        x[np.linspace(0, n - 1, size).astype(np.int64)] |= 2 << 8
        plan = oc.topk_plan([x], [None], ["uint32"], size - 3, False, False)
        assert plan["steps"][0]["count"] == size
        assert plan["steps"][1]["appends"] == listed and plan["steps"][1]["list"] is False
        exp = np.sort(sort_oracle.numpy_arg_sort([x], None, False, False, limit=size - 3))
        assert np.array_equal(plan["ids"], exp)


# ------------------------------------------------------------------------------------------------ rank
@pytest.mark.parametrize("method", oc.RANK_METHODS)
@pytest.mark.parametrize("parts", [False, True])
@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("desc", [False, True])
def test_rank_reference(method, parts, nulls, desc):
    rng = np.random.default_rng(oc.RANK_METHODS.index(method) * 8 + 4 * parts + 2 * nulls + desc)
    for dt in ("int32", "float64", "uint8"):
        n = 200
        x = column(rng, dt, n, distinct=6)
        valid = rng.random(n) >= 0.25 if nulls else None
        gid = rng.integers(0, 5, n) if parts else None
        if parts:
            valid = None if valid is None else valid & (gid != 4)      # an all-null partition
        got = oc.rank_ref(x, valid, method, desc, gid)
        exp = rank_oracle.rank(py(x, valid), method, desc, None if gid is None else list(gid))
        assert [None if e is None else e for e in exp] == [None if (valid is not None and not valid[i]) else got[i].item() for i in range(n)]


def test_rank_plan_matches_the_allocations():
    for method in oc.RANK_METHODS:
        for parts in (False, True):
            p = oc.rank_plan(5000, method, parts, False, 132)
            assert p["rank_starts"] == (method in ("average", "min", "max") or parts)
            assert p["seg_run"] == (parts and method == "dense")
    p = oc.rank_plan(8 * 132 * oc.RK_TILE + 1, "min", False, False, 132)
    assert p["ntiles"] == 8 * 132 + 1 and p["grid"] == 8 * 132 and p["rounds"] == 2


def test_head_places():
    h = [0, 31, 32, 255, 256, 2047, 2048]
    assert oc.head_places(h) == {"lane0": 4, "lane31": 3, "warp_first": 3, "warp_last": 2, "tile_first": 2, "tile_last": 1}
    lab = oc.labels_from_heads(10, [0, 3, 7])
    assert lab.tolist() == [0, 0, 0, 1, 1, 1, 1, 2, 2, 2]


# ------------------------------------------------------------------------------------------------ rolling quantile
@pytest.mark.parametrize("method", oc.QMETHODS)
def test_rq_reference_against_the_oracle(method):
    rng = np.random.default_rng(oc.QMETHODS.index(method))
    for dt in ("float64", "float32", "int32"):
        n = 150
        x = rng.integers(-20, 20, n).astype(dt)
        valid = rng.random(n) >= 0.3
        for w, center, ms in ((1, False, 1), (5, False, 2), (7, True, 0), (40, False, 40)):
            for q in (0.0, 0.25, 0.5, 0.3, 1.0):
                s, e = oc.fixed_bounds(n, w, center)
                got, ok = oc.rq_ref(x, valid, rqo.out_type(dt), q, method, s, e, ms)
                exp = rqo.rolling_quantile(list(x), list(valid), dt, q, method, w, ms, center)
                assert [v is not None for v in exp] == ok.tolist()
                for i in np.flatnonzero(ok):
                    assert got[i].tobytes() == exp[i].tobytes(), (dt, w, q, i, got[i], exp[i])


def test_q_index_matches_the_oracle():
    for m in range(1, 40):
        for q in (0.0, 0.1, 0.25, 0.5, 0.75, 1.0, 1 / 3):
            for method in oc.QMETHODS:
                lo, hi, _ = oc.q_index(m, q, method)
                elo, ehi = rqo.indices(m, q, method)
                assert lo == elo
                if ehi is not None:
                    assert hi == ehi


@pytest.mark.parametrize("method", oc.QMETHODS)
def test_rq_monotone_closed_form(method):
    n = 3000
    v = (np.arange(n) >> 3).astype(np.float32)
    s, e = oc.fixed_bounds(n, 37)
    full = e - s == 37
    for q in (0.0, 0.5, 0.3, 1.0):
        got = oc.rq_monotone(lambda r: v[r], q, method, s[full], e[full], np.float32)
        exp, ok = oc.rq_ref(v, None, np.float32, q, method, s[full], e[full], 37)
        assert ok.all() and got.tobytes() == exp.tobytes(), (q,)


def test_rq_plan_and_edges():
    assert [oc.rq_levels(n) for n in (1, 2, 3, 4, 5, 2**31, 2**31 + 1, 2**32 - 1)] == [1, 1, 2, 2, 3, 31, 32, 32]
    assert oc.rq_plan(1792, True) == {"L": 11, "wm_count": 12, "tiles": 2}
    s, e = oc.fixed_bounds(1792, 224)
    ed = oc.rq_edges(s, e, 1792)
    assert ed["e_block"] == 7 and ed["e_n_on_tile"] == 1 and ed["s_block"] == 7
    assert math.ceil(math.log2(2**31 + 2**20 + 33)) == oc.rq_levels(2**31 + 2**20 + 33) == 32


def test_rank_heads_follow_the_first_row_partition_order():
    """partitions sort by their first row (partition_ids), not by their values; nulls go last inside each partition"""
    gid = np.array([9, 9, 1, 1, 9, 4])
    assert oc.first_row_ids(gid).tolist() == [0, 0, 2, 2, 0, 5]
    x = np.array([3, 1, 2, 2, 1, 0], np.int64)
    valid = np.array([True, True, True, False, True, True])
    run_h, seg_h = oc.rank_heads(x, valid, gid)
    # order: partition 9 (rows 1, 4 then 0), partition 1 (row 2, then null row 3), partition 4 (row 5)
    assert seg_h.tolist() == [0, 3, 5] and run_h.tolist() == [0, 2, 3, 4, 5]
