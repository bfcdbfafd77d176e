"""CPU checks of tests/window_cases.py: the numpy references against the plain-Python oracles (window_oracle,
rolling_oracle, rolling_by_oracle) on small random inputs with nulls, partitions, `center`, every `closed` and
min_samples, and the branch restatements against a brute-force window reduction."""
import numpy as np
import pytest

import rolling_by_oracle as rbo
import rolling_oracle as ro
import window_cases as wc
import window_oracle as wo


def runs(rng, n, mean_len):
    """contiguous partition ids with random run lengths (the partition order of such ids is the rows)"""
    return wc.gid_from_heads(rng.random(n) < 1.0 / mean_len)


def values(rng, dtype, n):
    if dtype == "bool":
        return rng.random(n) < 0.5, None
    if dtype.startswith("float"):
        return wc.exact_floats(rng, n, dtype)
    if dtype == "int32":
        return rng.integers(-2**31, 2**31, n).astype(np.int32), None
    return rng.integers(0, 2**64, n, dtype=np.uint64), None


def as_list(x, valid):
    return [None if not v else (bool(a) if isinstance(a, np.bool_) else a.item()) for a, v in zip(x, valid)]


CUM = {"int32": ["cum_sum", "cum_prod", "cum_min", "cum_max", "cum_count"], "uint64": ["cum_sum", "cum_prod", "cum_min", "cum_max"],
       "float32": ["cum_sum", "cum_min", "cum_max"], "float64": ["cum_sum", "cum_min", "cum_max"], "bool": ["cum_sum", "cum_count"]}


@pytest.mark.parametrize("dtype", list(CUM))
@pytest.mark.parametrize("reverse", [False, True])
def test_cum_ref_matches_window_oracle(dtype, reverse):
    rng = np.random.default_rng(len(dtype) * 7 + reverse)
    for n, mean_len in ((1, 1), (40, 3), (700, 50), (900, 1e9)):
        x, frac = values(rng, dtype, n)
        valid = rng.random(n) >= 0.2
        gid = runs(rng, n, mean_len)
        for kind in CUM[dtype]:
            got = wc.cum_ref(kind, x, valid, gid, reverse, dtype, frac)
            exp = wo.over([(kind, as_list(x, valid), dtype, {"reverse": reverse})], [gid.tolist()], n)[0]
            mask = np.ones(n, bool) if kind == "cum_count" else valid
            assert as_list(got, mask) == [None if not m else e for e, m in zip(exp, mask)], (kind, n)
            assert all((e is None) == (not m) for e, m in zip(exp, mask)), kind


@pytest.mark.parametrize("center", [False, True])
def test_fixed_window_refs_match_rolling_oracle(center):
    rng = np.random.default_rng(31 + center)
    n = 600
    for w in (1, 2, 3, 7, 64, 700):
        gid = runs(rng, n, 40)
        for dtype in ("int32", "uint64", "bool", "float64", "float32"):
            x, frac = values(rng, dtype, n)
            valid = rng.random(n) >= 0.15
            s, e, lo, hi = wc.fixed_bounds(n, w, center, gid)
            kinds = ["rolling_sum"] + (["rolling_mean", "rolling_min", "rolling_max"] if dtype.startswith("float") else
                                       ["rolling_min", "rolling_max"] if dtype != "bool" else [])
            for kind in kinds:
                for ms in (0, 1, min(w, 3)):
                    v, ok = wc.rolling_ref(kind, x, valid, s, e, ms, frac, dtype)
                    exp = ro.rolling_over(kind, as_list(x, valid), dtype, gid.tolist(), window_size=w, min_samples=ms, center=center)
                    assert as_list(v, ok) == exp, (w, dtype, kind, ms)


@pytest.mark.parametrize("closed", rbo.CLOSED)
def test_by_refs_match_rolling_by_oracle(closed):
    rng = np.random.default_rng(len(closed))
    n = 800
    gid = runs(rng, n, 60)
    t = np.cumsum(rng.integers(0, 4, n)).astype(np.int64)
    for P in (1, 3, 40, 10_000):
        s, e = wc.by_bounds(t, P, closed, gid)
        x, frac = values(rng, "float64", n)
        valid = rng.random(n) >= 0.15
        for kind in ("rolling_sum", "rolling_mean", "rolling_min", "rolling_max"):
            for ms in (0, 2):
                v, ok = wc.rolling_ref(kind, x, valid, s, e, ms, frac, "float64")
                ok &= (e - s) >= ms           # rolling_*_by: min_samples counts the window's rows, nulls included
                wins = rbo.window_values(x.tolist(), list(valid), t.tolist(), [True] * n, P, closed, ms, [gid.tolist()])
                for r in range(n):
                    w = wins[r]
                    if w is None or len(w) < ms or (kind != "rolling_sum" and not w):
                        assert not ok[r], (P, kind, r)
                        continue
                    exp = sum(w) if kind == "rolling_sum" else sum(w) / len(w) if kind == "rolling_mean" else (min(w) if kind == "rolling_min" else max(w))
                    assert ok[r] and v[r] == exp, (P, kind, ms, r, v[r], exp)


def test_sparse_table_matches_brute_force():
    rng = np.random.default_rng(2)
    x = rng.integers(-1000, 1000, 3000)
    s = rng.integers(0, 3000, 5000)
    e = np.minimum(3000, s + 1 + rng.integers(0, 1500, 5000))
    for is_max in (False, True):
        got = wc.SparseTable(x, is_max).query(s, e)
        exp = np.array([(x[a:b].max() if is_max else x[a:b].min()) for a, b in zip(s, e)])
        assert np.array_equal(got, exp)


@pytest.mark.parametrize("B", [1, 2, 3, 31, 127, 128, 129, 1024, 1025])
def test_window_state_branches_cover_their_windows(B):
    rng = np.random.default_rng(B)
    n = 2600
    for center in (False, True):
        for gid in (None, runs(rng, n, 300)):
            s, e, lo, hi = wc.fixed_bounds(n, B, center, gid)
            got = wc.reduce_by_state_branch(s, e, lo, B, n, hi)
            assert all(g == list(range(a, b)) for g, a, b in zip(got, s, e))
            br = wc.window_state_branch(s, e, lo, B)
            if B > 1 and gid is not None:      # the suffix alone only serves a window clipped at its segment's end
                assert ({wc.TWO, wc.PRE, wc.SUF} if center and B > 2 else {wc.TWO, wc.PRE}) <= set(br.tolist()), (B, center)


def test_window_state_branch_equals_rolling_oracle_decomposition():
    rng = np.random.default_rng(8)
    n = 500
    gid = runs(rng, n, 45)
    segs = [(int(a), int(b)) for a, b in zip(np.flatnonzero(wc.scan_heads(gid, False)), np.append(np.flatnonzero(wc.scan_heads(gid, False))[1:], n))]
    for w in (3, 16, 40):
        for center in (False, True):
            dec = ro.decomposed(list(range(n)), w, center, segs, lambda v: (v,), lambda a, b: a + b, ())
            s, e, lo, hi = wc.fixed_bounds(n, w, center, gid)
            assert [list(d) for d in dec] == wc.reduce_by_state_branch(s, e, lo, w, n, hi)


def test_tile_staging_holds_every_window():
    for n in (1, 1023, 1024, 5000, 3 * 1024 + 7):
        for w in (1, 2, 3, 31, 127, 128):
            for center in (False, True):
                s, e, _, _ = wc.fixed_bounds(n, w, center)
                R = (w // 2 + (w & 1)) if center else 1
                L = w - R if center else w - 1
                A, ln, last = wc.tile_staging(n, min(L, n), min(R, n), min(w, n))
                cta = np.arange(n) // wc.RT_TILE
                assert np.all(s >= A[cta]) and np.all(e <= A[cta] + ln[cta])
                assert np.all(ln <= wc.RT_TILE + 3 * wc.RT_MAX_B)


@pytest.mark.parametrize("tile", [True, False])
def test_rollby_branches_cover_their_windows(tile):
    rng = np.random.default_rng(5 + tile)
    n = 3 * wc.RB_B + 300
    for gid in (None, runs(rng, n, 700)):
        t = np.cumsum(rng.integers(0, 3, n)).astype(np.int64)
        t[1500:1700] = t[1500]      # a run of equal times: left / none windows behind it
        t[1700:] += 1
        t = np.maximum.accumulate(t)
        for P, closed in ((5, "right"), (60, "left"), (900, "none"), (4000, "both")):
            s, e = wc.by_bounds(t, P, closed, gid)
            got = wc.reduce_by_rollby_branch(s, e, n, tile, gid)
            for i, (g, a, b) in enumerate(zip(got, s, e)):
                assert g == (None if b <= a else list(range(a, b))), (P, closed, i)
            m = wc.rollby_branch(s, e, n, tile, gid)
            names = [k for k in m if k not in ("level", "stage_l_eq_r", "stage_k")]
            total = sum(m[k].astype(int) for k in names)
            assert np.array_equal(total, (e > s).astype(int)), "every non-empty window takes exactly one branch"


def test_head_shapes():
    n = 5 * wc.OS_TILE
    gid = wc.gid_from_heads(wc.tile_edge_heads(n, 2))
    lanes = wc.head_lanes(gid, False)
    assert lanes["lane0"] == 64 and lanes["lane31"] == 64 and lanes["tile_first"] == 1 and lanes["tile_last"] == 1
    assert list(wc.head_tiles(gid, False)) == [2] and list(wc.head_tiles(gid, True)) == [2, 3]
    g = wc.gid_from_heads(wc.alternating_heads(10 * wc.OS_TILE))
    assert np.all(np.isin(np.arange(1, 10), wc.head_tiles(g, False)))
    assert wc.sparse_levels(1) == 0 and wc.sparse_levels(1024) == 0 and wc.sparse_levels(1025) == 1 and wc.sparse_levels(4097) == 3
