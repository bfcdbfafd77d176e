"""CPU cross-checks (-m "not gpu") of the references and inputs the asof / inequality-join plan tests
(tests/test_gpu_join_asof_ie_plans.py) lean on: the all-groups asof rule against the reference's cursors
(asof_oracle.cursor_asof_by) and the per-group rule, the window restatement against a plain scan, the window case's
windows, the inequality join's y-domain pair counts and numpy brute force against ie_join_oracle's brute force and
serial algorithms, and the string-hash restatement's collisions."""
import numpy as np
import pytest

import asof_ie_cases as cs
import asof_oracle as ao
import ie_join_oracle as io

STRATS = ("backward", "forward", "nearest")


def as_lists(side):
    v, ok = side
    ok = np.ones(len(v), bool) if ok is None else ok
    return [x if o else None for x, o in zip(v, ok)]


def by_lists(g):
    return [(int(x),) if x >= 0 else (None,) for x in g]


def lists_of(res):
    idx, valid = res
    return [int(i) if ok else None for i, ok in zip(idx, valid)]


@pytest.mark.parametrize("dtype", ["int32", "int64", "uint64", "float32", "float64"])
@pytest.mark.parametrize("n_groups", [1, 2, 9, 200])
def test_rule_asof_by_matches_the_cursors(dtype, n_groups):
    rng = np.random.default_rng(n_groups)
    L, R, lg, rg = cs.by_sides(rng, 300, 120, n_groups, dtype, lnull=0.1, bynull=0.1, right_null_groups=1 if n_groups > 1 else 0,
                               one_side=2)
    if dtype.startswith("float"):          # -0.0 on the left against 0.0 on the right
        lv, rv = L[0] - 100, R[0] - 100
        L, R = (np.where(lv == 0, -0.0, lv).astype(dtype), L[1]), (rv, R[1])
    left, right = as_lists(L), as_lists(R)
    for strategy in STRATS:
        for allow_eq in (False, True):
            for tol in (None, np.array([5], dtype)[0]):
                exp = ao.cursor_asof_by(left, right, by_lists(lg), by_lists(rg), strategy, allow_eq, tol)
                assert lists_of(cs.rule_asof_by(L, R, strategy, allow_eq, tol, lg, rg)) == exp, (strategy, allow_eq, tol)
                assert lists_of(ao.rule_asof(L, R, strategy, allow_eq, tol, lg, rg)) == exp


def test_by_sides_keep_every_group_nulls_first_then_sorted():
    rng = np.random.default_rng(4)
    L, R, lg, rg = cs.by_sides(rng, 1000, 800, 30, right_null_groups=3, one_side=2)
    assert np.all(np.diff(L[0]) >= 0)
    for g in np.unique(rg[rg >= 0]):
        vals = [v if ok else None for v, ok in zip(R[0][rg == g], R[1][rg == g])]
        assert ao.precondition_ok([], vals), g
        if g < 3:
            assert all(v is None for v in vals)
    assert set(lg[lg >= 0]) - set(rg[rg >= 0]) and set(rg[rg >= 0]) - set(lg[lg >= 0])        # groups on one side only


def test_kernel_group_order_follows_first_appearance():
    rng = np.random.default_rng(6)
    lg, rg = rng.integers(-1, 9, 300), rng.integers(-1, 12, 200)
    lvalid = rng.random(300) > 0.1
    first = {}
    for i, g in enumerate(list(lg) + list(rg)):
        if g >= 0:
            first.setdefault(int(g), i)

    def plain(groups, keep):
        return sorted(range(len(groups)), key=lambda i: first[int(groups[i])] if groups[i] >= 0 and keep[i] else len(first) + 10**9)
    lo, ro = cs.kernel_group_order(lg, rg, lvalid)
    assert lo.tolist() == plain(lg, lvalid) and ro.tolist() == plain(rg, np.ones(200, bool))


def test_tile_windows_match_a_plain_scan():
    rng = np.random.default_rng(5)
    rv = np.sort(rng.integers(0, 3000, 5000))
    rvalid = np.arange(5000) >= 37
    lv = np.sort(rng.integers(-10, 3100, 3 * cs.AS_TILE + 5))
    lvalid = rng.random(len(lv)) > 0.2
    lvalid[cs.AS_TILE:2 * cs.AS_TILE] = False
    for (wlo, whi), t in zip(cs.tile_windows((lv, lvalid), (rv, rvalid)), range(0, len(lv), cs.AS_TILE)):
        k = lv[t:t + cs.AS_TILE][lvalid[t:t + cs.AS_TILE]]
        if not k.size:
            assert (wlo, whi) == (0, 0)
            continue
        blo = next((j for j in range(37, 5000) if rv[j] >= k.min()), 5000)
        bhi = next((j for j in range(37, 5000) if rv[j] > k.max()), 5000)
        assert (wlo, whi) == (max(37, blo - 1), min(5000, bhi + 1))


@pytest.mark.parametrize("dtype", ["int32", "int64", "uint64", "float32", "float64"])
def test_window_case_builds_the_intended_windows(dtype):
    L, R = cs.window_case(np.random.default_rng(0), dtype)
    lv, lvalid = L
    valid = lv[lvalid]
    assert ao.precondition_ok(list(valid), as_lists(R))
    win = cs.tile_windows(L, R)
    assert [b - a for a, b in win[1:5]] == list(cs.WIN_WIDTHS)
    size = np.dtype(dtype).itemsize
    lim = cs.AS_WIN_BYTES // size
    assert [cs.staged(w, size) for w in win[1:5]] == [w <= lim for w in cs.WIN_WIDTHS]
    assert win[0][0] == 100 and win[5] == (0, 0) and win[-1][1] == len(R[0])
    run = 100 + 2 + cs.RUN_AT
    assert np.all(R[0][run:run + cs.RUN_LEN] == R[0][run]) and win[6][1] == run + 1
    if dtype.startswith("float"):
        assert np.isnan(R[0][-1]) and np.isnan(valid[-1]) and np.signbit(valid[valid == 0]).any() and not np.signbit(valid[valid == 0]).all()
    else:
        assert valid[0] == np.iinfo(dtype).min and valid[-1] == np.iinfo(dtype).max
    # the numpy rule agrees with the cursors on this case (the cursors are slow: every strategy, one option each)
    for strategy, allow_eq in zip(STRATS, (True, False, True)):
        exp = ao.cursor_asof(as_lists(L), as_lists(R), strategy, allow_eq)
        assert lists_of(ao.rule_asof(L, R, strategy, allow_eq)) == exp, strategy


IE_PAIRS = [(a, b) for a in io.OPS for b in io.OPS]


@pytest.mark.parametrize("ops", IE_PAIRS + [(o,) for o in io.OPS], ids=lambda o: "".join(o))
def test_ie_counts_and_brute_rows_match_the_oracle(ops):
    rng = np.random.default_rng(len(ops) * 17 + sum(io.OPS.index(o) for o in ops))
    nl, nr = 60, 90
    pool = np.array([-np.inf, -2.0, -0.0, 0.0, 1.0, 3.5, np.inf, np.nan])
    left = [(rng.integers(-20, 20, nl).astype(np.int64), rng.random(nl) >= 0.1), (pool[rng.integers(0, 8, nl)], rng.random(nl) >= 0.1)][:len(ops)]
    right = [(rng.integers(-20, 20, nr).astype(np.int64), rng.random(nr) >= 0.1), (pool[rng.integers(0, 8, nr)], rng.random(nr) >= 0.1)][:len(ops)]
    ll, rl = ([[(float(x) if c.dtype.kind == "f" else int(x)) if ok else None for x, ok in zip(c, m)] for c, m in side] for side in (left, right))
    pairs = io.brute(ll, rl, list(ops))
    assert io.as_multiset(pairs) == io.as_multiset(io.serial(ll, rl, list(ops)))
    counts = cs.ie_counts(left, right, list(ops))
    assert counts.tolist() == [sum(1 for a, _ in pairs if a == i) for i in range(nl)]
    for i, got in zip(range(nl), cs.ie_brute_rows(left, right, list(ops), range(nl))):
        assert got.tolist() == sorted(b for a, b in pairs if a == i)


@pytest.mark.parametrize("ops", [("<", ">"), (">=", "<="), ("<=", "<"), (">", ">=")], ids=lambda o: "".join(o))
def test_ie_wide_case_shape_and_counts(ops):
    """the large-case builder at a small m: exactly m live right rows, about 5 % nulls per column, and its counts equal
    the brute force"""
    m = 5000
    rng = np.random.default_rng(7)
    left, right = cs.ie_wide_case(rng, m, ops)
    (rx, rxv), (ry, ryv) = right
    assert (rxv & ryv).sum() == m and 0.03 < (~rxv).mean() < 0.07 and 0.03 < (~ryv).mean() < 0.07
    assert len(np.unique(ao.total_keys(ry))) <= 64
    counts = cs.ie_counts(left, right, list(ops))
    rows = range(0, len(left[0][0]), 7)
    assert [len(r) for r in cs.ie_brute_rows(left, right, list(ops), rows)] == counts[list(rows)].tolist()


def test_plan_sizes():
    assert [cs.tree_levels(m) for m in (1 << 20, (1 << 20) + 1, 1 << 24, (1 << 24) + 1)] == [21, 22, 25, 26]
    T, N = cs.AS_TILE, cs.TS_THREADS
    assert [cs.tiles_per_thread(n) for n in (N * T - 1, N * T + 1, int(2.5 * N * T), 3 * N * T + 777)] == [1, 2, 3, 4]
    assert cs.grid_threads(132) == 270_336


def test_string_pairs_collide_under_exactly_their_seed():
    seen = set()
    for k, seed in enumerate(cs.SEEDS):
        a, b = cs.colliding_pair(seed, b"%d" % k)
        assert a != b and len(a) == len(b) == 16 and max(a + b) < 128
        assert [cs.str_hash_bytes(a, s) == cs.str_hash_bytes(b, s) for s in cs.SEEDS] == [s == seed for s in cs.SEEDS]
        seen |= {a, b}
    assert len(seen) == 8
    # the restatement's tail and length handling: values of other lengths keep distinct hashes
    vals = [b"", b"a", b"ab", b"abcdefgh", b"abcdefghi", b"\x00", b"\x00\x00"]
    assert len({cs.str_hash_bytes(v, cs.SEEDS[0]) for v in vals}) == len(vals)
