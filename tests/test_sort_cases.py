"""CPU cross-checks (-m "not gpu") of the references the sort-family plan tests (tests/test_gpu_sort_plans.py) lean on at
sizes where the plain oracles are too slow: sort_oracle.numpy_arg_sort against the plain sort_oracle.arg_sort on the
same full-range bit-pattern columns, the numpy GroupsIdx against quantile_oracle.group_tuples, the byte-string dense
rank against test_string_sort.dense_rank, quantile_oracle.numpy_group_quantile against group_quantile on the values
whose quantiles are easy to get wrong, and the group layouts of the small-group quantile windows."""
import numpy as np
import pytest

import quantile_oracle as qo
import sort_cases as sc
import sort_oracle
from test_string_sort import dense_rank


def test_full_range_columns_hold_their_bit_patterns():
    rng = np.random.default_rng(0)
    for dt in sc.KEY_DTYPES:
        c = sc.full_range_column(rng, dt, 4000)
        assert c.dtype == sc.NP[dt] and c.size == 4000
        if dt in ("int8", "uint8", "bool"):
            assert np.unique(c).size == (2 if dt == "bool" else 256)
    f = sc.full_range_column(rng, "float64", 100)
    assert set(sc.F64_SPECIAL.view(np.uint64).tolist()) <= set(f.view(np.uint64).tolist())      # payloads and -0.0 survive
    f = sc.full_range_column(rng, "float32", 100)
    assert set(sc.F32_SPECIAL.view(np.uint32).tolist()) <= set(f.view(np.uint32).tolist())


@pytest.mark.parametrize("dt", sc.KEY_DTYPES)
def test_numpy_arg_sort_matches_the_plain_oracle_on_full_range_columns(dt):
    rng = np.random.default_rng(sc.KEY_DTYPES.index(dt))
    n = 700
    c = sc.full_range_column(rng, dt, n)
    valid = rng.random(n) > 0.2
    for v in (None, valid):
        for desc in (False, True):
            for nl in (False, True):
                exp = sort_oracle.arg_sort([c], [v], desc, nl)
                assert np.array_equal(sort_oracle.numpy_arg_sort([c], [v], desc, nl), exp), (dt, v is not None, desc, nl)


def test_numpy_arg_sort_matches_the_plain_oracle_on_several_columns():
    rng = np.random.default_rng(1)
    n = 900
    cols = [rng.choice(np.array([-128, 0, 127], np.int8), n), rng.choice(sc.F64_SPECIAL, n), rng.random(n) < 0.5,
            sc.full_range_column(rng, "uint64", n)]
    valids = [rng.random(n) > 0.1, rng.random(n) > 0.1, rng.random(n) > 0.3, None]
    for trial in range(6):
        desc = [bool(x) for x in rng.random(4) < 0.5]
        nl = [bool(x) for x in rng.random(4) < 0.5]
        limit = [None, 0, 1, 333, n, n + 5][trial]
        exp = sort_oracle.arg_sort(cols, valids, desc, nl, limit)
        assert np.array_equal(sort_oracle.numpy_arg_sort(cols, valids, desc, nl, limit), exp), (desc, nl, limit)


def test_numpy_groups_idx_matches_group_tuples():
    rng = np.random.default_rng(2)
    for n, k in ((1, 1), (2, 2), (255, 3), (256, 200), (5000, 40), (5000, 5000)):
        keys = rng.integers(-(1 << 62), 1 << 62, k)[rng.integers(0, k, n)]
        first, offsets, all_ = sc.groups_idx(keys)
        groups = qo.group_tuples(keys.tolist())
        assert [g[0] for g in groups] == first.tolist()
        assert [all_[offsets[i]:offsets[i + 1]].tolist() for i in range(first.size)] == groups


def test_dense_rank_bytes_matches_dense_rank():
    rng = np.random.default_rng(3)
    pool = [b"", b"a", b"a\0", b"a\0\0", b"\0", b"\xff", b"\xff\xff", b"ab", b"b" * 9, b"b" * 8 + b"\0", None]
    vals = [pool[i] for i in rng.integers(0, len(pool), 400)]
    for desc in (False, True):
        r, v = sc.dense_rank_bytes(vals, desc)
        assert [int(x) if ok else None for x, ok in zip(r, v)] == dense_rank(vals, desc)


def test_refinement_rounds():
    assert sc.refinement_rounds([b"x"] * 5 + [None]) == (0, 0)
    assert sc.refinement_rounds([b"a", b"a\0", b"a\0\0"]) == (1, 0)           # the length byte splits them in round 0
    assert sc.refinement_rounds([b"p" * 8 + b"1", b"p" * 8 + b"2"]) == (2, 1)
    assert sc.refinement_rounds([b"p" * 14, b"p" * 14 + b"\0"]) == (2, 1)       # round 1: length byte 7 against 8


VALUE_CASES = {
    "int64_extremes": lambda rng, n: rng.choice(sc.int_pool(np.int64), n),
    "uint64_extremes": lambda rng, n: rng.choice(sc.int_pool(np.uint64), n),
    "float64_special": lambda rng, n: rng.choice(sc.F64_SPECIAL, n),
    "float32_special": lambda rng, n: rng.choice(sc.F32_SPECIAL, n),
}


@pytest.mark.parametrize("case", sorted(VALUE_CASES))
def test_numpy_group_quantile_matches_group_quantile(case):
    rng = np.random.default_rng(len(case))
    n = 3000
    gid = rng.integers(0, 300, n)
    gid[:300] = np.arange(300)                          # group ids in first-occurrence order
    vals = VALUE_CASES[case](rng, n)
    valid = rng.random(n) > 0.1
    valid[gid == 5] = False
    for m in qo.METHODS:
        for q in (0.0, 0.1, 0.5, 0.75, 1.0):
            exp, ev = qo.group_quantile(gid.tolist(), vals, valid, q, m)
            got, gv = qo.numpy_group_quantile(gid, vals, valid, q, m, 300)
            assert np.array_equal(gv, ev) and got.dtype == exp.dtype, (case, m, q)
            g, e = got[ev], exp[ev]
            assert np.all((g == e) | (np.isnan(g) & np.isnan(e))), (case, m, q)


def test_small_window_layout_of_the_plan_tests():
    sizes, shapes = sc.window_layout(np.random.default_rng(0))
    w = sc.small_windows(sizes)
    for name, (b, want) in shapes.items():
        assert w[b] == want, (name, b, w[b], want)
