"""GPU tests of the asof join (asof.cu) and the inequality join (ie_join.cu) on every plan and past their grid caps, and of
the string-code collision retry (strings.cu: op_string_codes), against exact references.

Asof results must equal the per-row rule bit for bit, index and validity (asof_oracle.rule_asof without `by`,
asof_ie_cases.rule_asof_by with `by`; tests/test_asof_ie_cases.py checks both against the reference's cursors on CPU).
Inequality-join results must be the exact multiset of (left row, right row | null) pairs with left rows ascending: the
per-row counts equal a y-domain restatement (asof_ie_cases.ie_counts), every pair satisfies both predicates, no pair
repeats, and sampled rows equal a numpy brute force.  The launch profile shows which kernels ran and how often.
Branches inside one kernel do not show there: which tiles stage their window and how many tiles each thread of
k_asof_tiles_sorted checks are computed from the inputs by CPU restatements (asof_ie_cases.tile_windows / staged,
tiles_per_thread), and so are the segment and left-group positions the `by` kernels walk (kernel_group_order).

Caps.  SM = device_info()["sm_count"] (132 on an H100 SXM); the values in brackets are for SM = 132.
  grid_for(n, 256)        at most 8*SM CTAs x 256 threads = G [270 336] threads; the grid-stride loop wraps at G:
                          asof  k_asof_right_check, k_asof_group_keys, k_asof_segments, k_asof_left_groups;
                          ie    k_ie_keys, k_ie_xpos, k_ie_px, k_ie_level_keys, k_ie_level_rows.
  k_asof_search           2048 left rows per CTA (256 threads x 8 rows); the left check inside a tile runs item ->
                          thread -> warp prefix max.
  k_asof_tiles_sorted     one CTA of 1024 threads, per = ceil(ceil(nl / 2048) / 1024) tiles each: per = 1 up to
                          1024*2048 = 2 097 152 left rows, 2 from 2 097 153, 3 from 4 194 305, 4 from 6 291 457.
  right window            16 384 bytes of shared memory: 2048 keys of 8 bytes, 4096 keys of 4 bytes; one entry more
                          is read from global memory.
  sort_pairs_u32 (`by`)   ceil(bits_for(nl + nr) / 8) passes: 2 at nl + nr = 2^16 - 1, 3 at 2^16 and 2^24 - 1, 4 at 2^24.
  k_ie_count              256 left rows per CTA; the CTA sums are scanned by exclusive_scan_u64.
  k_ie_emit               512 output slots per warp, 8 warps = 4096 slots per CTA; validity words of 32 slots.
  merge-sort tree         L = the smallest L with 2^(L-1) >= m live right rows, at most 32: 21 at m = 2^20, 22 at
                          2^20 + 1, 25 at 2^24, 26 at 2^24 + 1 (the top block of the last level is truncated).
  output slots            u64 throughout; one test goes past 2^31 slots.
"""
import ctypes as C

import numpy as np
import pytest

import asof_ie_cases as cs
import asof_oracle as ao

pytestmark = pytest.mark.gpu
STRATS = ("backward", "forward", "nearest")
NULL = 0xFFFFFFFF
ASOF_DTYPES = ["int32", "int64", "uint64", "float32", "float64"]


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as m
    m.init()
    return m


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


@pytest.fixture(scope="module")
def G(sm):
    return cs.grid_threads(sm)


def profiled(plb, fn):
    """-> (fn(), {kernel name: launches})"""
    plb.profile_reset()
    plb.profile_enable(True)
    try:
        out = fn()
        plb.sync()
        prof = plb.profile()
    finally:
        plb.profile_enable(False)
    return out, {k: int(v.get("launches", 0)) for k, v in prof.items()}


def check_bits(res, exp, what=""):
    vals, valid = res
    exp_idx, exp_valid = exp
    valid = np.ones(len(vals), bool) if valid is None else valid
    assert np.array_equal(valid, exp_valid), f"{what}: validity differs at {np.nonzero(valid != exp_valid)[0][:10]}"
    assert np.array_equal(vals, exp_idx), f"{what}: index differs at {np.nonzero(vals != exp_idx)[0][:10]}"


def unsorted(plb, side, fn):
    """fn must fail with status 4 naming the side whose `on` column is not sorted"""
    with pytest.raises(plb.B200Error, match=f"the {side} `on` column is not sorted") as e:
        fn()
    assert e.value.status == 4


def values_of(dtype, n, start=0, step=3):
    """n strictly increasing keys of the dtype"""
    dt = np.dtype(dtype)
    if dt.kind == "f":
        return (np.arange(n) * step * 0.5 + start - n).astype(dt)
    if dt.kind == "u":
        return (np.arange(n, dtype=np.uint64) * np.uint64(step) + np.uint64(1 << 63) + np.uint64(start)).astype(dt) if dt.itemsize == 8 \
            else (np.arange(n) * step + start).astype(dt)
    return (np.arange(n, dtype=np.int64) * step - n + start).astype(dt)


def swap(v, i, j):
    v = v.copy()
    v[i], v[j] = v[j], v[i]
    return v


# =========================================================================================== asof without `by`
@pytest.mark.parametrize("dtype", ASOF_DTYPES)
def test_left_inversion_at_every_level_of_the_check(plb, dtype):
    """One inversion per case: inside one thread's 8 rows, across two threads of a warp, across warps, across tiles,
    behind a run of nulls, and in a tile whose first thread holds only nulls; the sorted twin must succeed"""
    nl = 4 * cs.AS_TILE + 100
    lv = values_of(dtype, nl)
    rv = values_of(dtype, 3000, start=7, step=5)
    T = cs.AS_TILE
    cases = {"in_thread": (None, 3 * 8 + 3, 3 * 8 + 4),
             "across_threads": (None, 5 * 8 - 1, 5 * 8),
             "across_warps": (None, 256 - 1, 256),
             "across_far_warps": (None, 3 * 256 - 1, 3 * 256),
             "across_tiles": (None, 2 * T - 1, 2 * T),
             "behind_nulls": ("nulls", T + 100, T + 900),
             "first_thread_all_null": ("tile_head", 3 * T - 1, 3 * T + 8)}
    for i, (name, (kind, p, q)) in enumerate(cases.items()):
        lvalid = np.ones(nl, bool)
        if kind == "nulls":
            lvalid[p + 1:q] = False
        elif kind == "tile_head":
            lvalid[3 * T:3 * T + 8] = False
        strategy = STRATS[i % 3]
        exp = ao.rule_asof((lv, lvalid), (rv, None), strategy, bool(i % 2))
        check_bits(plb.join_asof((lv, lvalid), rv, strategy, None, bool(i % 2)), exp, (dtype, name, "sorted twin"))
        unsorted(plb, "left", lambda: plb.join_asof((swap(lv, p, q), lvalid), rv, strategy))


@pytest.mark.parametrize("nl_kind", ["per1", "per2", "per3"])
def test_tiles_sorted_per_thread_chunks(plb, nl_kind):
    """k_asof_tiles_sorted at per = 1, 2, 3: an inversion between the chunks of two threads (and, per >= 2, between two
    tiles of one chunk) must give status 4; the sorted twin must equal the rule"""
    T, N = cs.AS_TILE, cs.TS_THREADS
    nl = {"per1": N * T - 1, "per2": N * T + 1, "per3": int(2.5 * N * T)}[nl_kind]
    per = cs.tiles_per_thread(nl)
    assert per == int(nl_kind[-1])
    rng = np.random.default_rng(per)
    lv = np.arange(nl, dtype=np.int64) * 4
    lvalid = rng.random(nl) >= 0.01
    rv = np.sort(rng.integers(-10, 4 * nl + 10, 300_000)).astype(np.int64)
    exp = ao.rule_asof((lv, lvalid), (rv, None), "nearest", True, 6)
    got, prof = profiled(plb, lambda: plb.join_asof((lv, lvalid), rv, "nearest", 6))
    check_bits(got, exp, nl_kind)
    assert prof.get("asof_tiles_sorted") == 1 and prof.get("asof_search") == 1, prof
    # the first row of tile b below the last row of tile b - 1: b starts thread t's chunk, or is inside it
    for b in sorted({per * 437, per * 437 + per - 1, per * 1000 - (per > 1)}):
        if 0 < b < (nl + T - 1) // T:
            bad = lv.copy()
            bad[b * T] = bad[b * T - 1] - 1
            v = lvalid.copy()
            v[b * T - 1] = v[b * T] = True
            unsorted(plb, "left", lambda: plb.join_asof((bad, v), rv, "backward"))


def test_right_checks_past_the_grid_wrap(plb, G):
    """a descent or a null after a value at k*G and k*G +- 1, and leading null runs longer than the grid (the first
    non-null row comes from atomicMin over every wrap)"""
    nr = 3 * G + 1234
    rv = np.arange(nr, dtype=np.int64) * 2
    lv = np.sort(np.random.default_rng(3).integers(-5, 2 * nr + 5, 50_000)).astype(np.int64)
    for k in (1, 2, 3):
        for p in (k * G - 1, k * G, k * G + 1):
            unsorted(plb, "right", lambda: plb.join_asof(lv, swap(rv, p - 1, p), "forward"))
            valid = np.ones(nr, bool)
            valid[p] = False
            unsorted(plb, "right", lambda: plb.join_asof(lv, (rv, valid), "forward"))
    for z in (G - 1, G, G + 12_345, 2 * G + 1):
        valid = np.arange(nr) >= z
        for strategy in STRATS:
            got, prof = profiled(plb, lambda: plb.join_asof(lv, (rv, valid), strategy, None, strategy != "forward"))
            check_bits(got, ao.rule_asof((lv, None), (rv, valid), strategy, strategy != "forward"), (z, strategy))
            assert prof.get("asof_right_check") == 1


@pytest.mark.parametrize("dtype", ASOF_DTYPES)
def test_window_staging_limits(plb, dtype):
    """tiles whose window holds exactly the staging limit and one more (2048 / 2049 8-byte, 4096 / 4097 4-byte keys),
    windows clipped at z and at e, an all-null tile, nearest ties, a run of equal right values that goes on past the
    window, NaN tails, +-0.0 and integer extremes (asof_ie_cases.window_case)"""
    L, R = cs.window_case(np.random.default_rng(ASOF_DTYPES.index(dtype)), dtype)
    size = np.dtype(dtype).itemsize
    lim = cs.AS_WIN_BYTES // size
    win = cs.tile_windows(L, R)
    widths = [b - a for a, b in win]
    z, e = 100, len(R[0])
    assert lim in widths and lim + 1 in widths, widths
    assert any(cs.staged(w, size) for w in win) and any(w[1] > w[0] and not cs.staged(w, size) for w in win)
    assert win[0][0] == z and win[-1][1] == e and win[5] == (0, 0)
    assert win[6][1] == z + 2 + cs.RUN_AT + 1                # one entry into the run of equal values
    tols = (None, np.array([1.5 if np.dtype(dtype).kind == "f" else 3], dtype))
    for strategy in STRATS:
        for allow_eq in (False, True):
            for tol in tols:
                exp = ao.rule_asof(L, R, strategy, allow_eq, None if tol is None else tol[0])
                got, prof = profiled(plb, lambda: plb.join_asof(L, R, strategy, tol, allow_eq))
                check_bits(got, exp, (dtype, strategy, allow_eq, tol))
                assert prof.get("asof_search") == 1 and prof.get("asof_tiles_sorted") == 1


@pytest.mark.parametrize("nr", [2_000_000, 20_000_000])
def test_scale_every_strategy(plb, nr):
    """3*1024*2048 + 777 left rows (per = 4) with 1 % nulls against 2 M and 20 M right rows"""
    rng = np.random.default_rng(nr % 97)
    nl = 3 * cs.TS_THREADS * cs.AS_TILE + 777
    assert cs.tiles_per_thread(nl) == 4
    lv = np.sort(rng.integers(0, 10**12, nl)).astype(np.int64)
    lvalid = rng.random(nl) >= 0.01
    rv = np.sort(rng.integers(0, 10**12, nr)).astype(np.int64)
    for strategy in STRATS:
        for allow_eq, tol in ((True, None), (False, 10**5)):
            exp = ao.rule_asof((lv, lvalid), (rv, None), strategy, allow_eq, tol)
            check_bits(plb.join_asof((lv, lvalid), rv, strategy, tol, allow_eq), exp, (nr, strategy, tol))


# =========================================================================================== asof with `by`
def run_by(plb, L, R, lg, rg, strategy, allow_eq=True, tol=None):
    return plb.join_asof(L, R, strategy, tol, allow_eq, [cs.groups_as_by(lg)], [cs.groups_as_by(rg)])


@pytest.mark.parametrize("groups", ["one", "two", "sqrt", "per_row"])
def test_by_group_counts(plb, groups):
    """1, 2, about sqrt(n) and one group per left row, with groups on one side only, null `by` keys on both sides and
    groups whose right rows are all null"""
    rng = np.random.default_rng(len(groups))
    nl, nr = 300_000, 120_000
    ng = {"one": 1, "two": 2, "sqrt": int(np.sqrt(nl)), "per_row": nl}[groups]
    L, R, lg, rg = cs.by_sides(rng, nl, nr, ng, right_null_groups=min(ng - 1, 5) if ng > 1 else 0, one_side=3)
    if ng > 1:
        assert not R[1][np.isin(rg, np.arange(min(ng - 1, 5)))].any()
    for strategy in STRATS:
        for allow_eq, tol in ((True, None), (False, 40)):
            exp = cs.rule_asof_by(L, R, strategy, allow_eq, tol, lg, rg)
            got, prof = profiled(plb, lambda: run_by(plb, L, R, lg, rg, strategy, allow_eq, tol))
            check_bits(got, exp, (groups, strategy, allow_eq))
            assert prof.get("asof_segments") == 1 and prof.get("asof_search_by") == 1 and "asof_left_groups" not in prof, prof


@pytest.mark.parametrize("total", [(1 << 16) - 1, 1 << 16, (1 << 24) - 1, 1 << 24])
def test_by_sort_pass_counts(plb, total):
    """nl + nr around 2^16 and 2^24: the stable sort of the right rows by group takes ceil(bits_for(nl + nr) / 8) passes.
    Rows with a null `by` key are sorted too (last), so at 2^24 90 % of them are null-keyed to keep the reference fast."""
    rng = np.random.default_rng(total % 1000)
    nl = total * 2 // 3
    nr = total - nl
    L, R, lg, rg = cs.by_sides(rng, nl, nr, 1000, bynull=0.9 if total > 1 << 20 else 0.02)
    kb = int(total).bit_length()
    exp = cs.rule_asof_by(L, R, "backward", True, None, lg, rg)
    got, prof = profiled(plb, lambda: run_by(plb, L, R, lg, rg, "backward"))
    check_bits(got, exp, total)
    assert prof.get("sort_scatter") == (kb + 7) // 8, (total, prof)


def sorted_groups_right(rng, sizes, null_groups=()):
    """right rows already in group order: group g holds sizes[g] rows, nulls first then ascending"""
    rg = np.repeat(np.arange(len(sizes)), sizes).astype(np.int64)
    rv = np.empty(len(rg), np.int64)
    rvalid = np.ones(len(rg), bool)
    off = np.concatenate([[0], np.cumsum(sizes)])
    for g in range(len(sizes)):
        a, b = off[g], off[g + 1]
        nn = (b - a) if g in null_groups else int(rng.integers(0, 3))
        rvalid[a:a + nn] = False
        rv[a:b] = np.sort(rng.integers(0, 10**7, b - a))
    return (rv, rvalid), rg


def test_by_segments_past_the_grid_wrap(plb, G):
    """group boundaries at segment positions G and 2G and an all-null group starting at G; then a descent or a null after
    a value inside one group at segment positions k*G and k*G +- 1.  The first left rows name the groups in order, so the
    segment order (asof_ie_cases.kernel_group_order) is the right rows' own order."""
    rng = np.random.default_rng(21)
    sizes = [G - 5000, 5000, 3, G - 3 - 7, 7, 777]
    R, rg = sorted_groups_right(rng, sizes, null_groups=(2,))
    nl = 200_000
    L = (np.sort(rng.integers(0, 10**7, nl)).astype(np.int64), rng.random(nl) >= 0.01)
    lg = rng.integers(0, len(sizes), nl).astype(np.int64)
    lg[:len(sizes)] = np.arange(len(sizes))
    seg = cs.kernel_group_order(lg, rg)[1]
    assert np.array_equal(seg, np.arange(len(rg)))
    starts = np.nonzero(np.diff(rg[seg]))[0] + 1
    assert G in starts and 2 * G in starts and rg[G] == 2 and not R[1][G:G + 3].any()
    for strategy in STRATS:
        exp = cs.rule_asof_by(L, R, strategy, True, None, lg, rg)
        check_bits(run_by(plb, L, R, lg, rg, strategy), exp, strategy)
    _, rg2 = sorted_groups_right(rng, [G // 2 + 11, G, G + 5, 999])
    R2 = (np.arange(len(rg2), dtype=np.int64), np.ones(len(rg2), bool))      # distinct values: every swap is a descent
    assert np.array_equal(cs.kernel_group_order(lg, rg2)[1], np.arange(len(rg2)))
    for k in (1, 2):
        for p in (k * G - 1, k * G, k * G + 1):
            assert rg2[p - 1] == rg2[p]
            unsorted(plb, "right", lambda: run_by(plb, L, (swap(R2[0], p - 1, p), R2[1]), lg, rg2, "backward"))
            v = R2[1].copy()
            v[p] = False
            unsorted(plb, "right", lambda: run_by(plb, L, (R2[0], v), lg, rg2, "backward"))


def test_by_left_group_fallback_past_the_grid(plb, G):
    """left rows sorted within every group but not globally, past k_asof_left_groups' grid: the fall-back runs and the
    answer equals the rule; one inversion inside a single group just below G, just past G and past 2G (positions in the
    kernel's group order, asof_ie_cases.kernel_group_order) gives status 4"""
    rng = np.random.default_rng(22)
    nl, nr, ng = 2 * G + 4321, 100_000, 40
    lg = rng.integers(0, ng, nl).astype(np.int64)
    lvals = rng.permutation(10**7)[:nl].astype(np.int64)
    srt = np.argsort(lg, kind="stable")
    lv = np.empty(nl, np.int64)
    lv[srt] = lvals[np.lexsort((lvals, lg))]
    L = (lv, None)
    _, R, _, rg = cs.by_sides(rng, 10, nr, ng)
    assert (np.diff(lv) < 0).any()
    for strategy in STRATS:
        exp = cs.rule_asof_by(L, R, strategy, True, None, lg, rg)
        got, prof = profiled(plb, lambda: run_by(plb, L, R, lg, rg, strategy))
        check_bits(got, exp, strategy)
        assert prof.get("asof_left_groups") == 1, prof
    order = cs.kernel_group_order(lg, rg)[0]
    for p in (G - 1, G + 5, 2 * G + 17):
        while lg[order[p - 1]] != lg[order[p]]:      # a group boundary: the next neighbours of one group
            p += 1
        assert p < G + 100 or p > 2 * G
        a, b = order[p - 1], order[p]
        assert lv[a] < lv[b]
        unsorted(plb, "left", lambda: run_by(plb, (swap(lv, a, b), None), R, lg, rg, "backward"))


# =========================================================================================== inequality join
def check_ie(res, left, right, ops, how, counts, sample_rows=()):
    """exact multiset check of an ie_join result: left rows ascending, per-row counts equal `counts` (left join: one
    null slot for a row without pairs), every pair satisfies every predicate on live rows, no pair repeats, and the
    sampled rows' right sets equal the brute force"""
    (li, lv), (ri, rv) = res
    nl, nr = len(left[0][0]), len(right[0][0])
    assert lv is None and li.dtype == np.uint32
    li64 = li.astype(np.int64)
    assert np.all(np.diff(li64) >= 0), "left rows must come ascending"
    slots = np.maximum(counts, 1) if how == "left" else counts
    assert np.array_equal(np.bincount(li64, minlength=nl), slots), "per-row pair counts differ"
    matched = np.ones(len(li), bool) if rv is None else rv
    if how == "left":
        assert np.array_equal(~matched, counts[li64] == 0), "null slots must be exactly the unmatched rows"
        assert np.all(ri[~matched] == NULL)
    else:
        assert matched.all()
    pl, pr = li64[matched], ri[matched].astype(np.int64)
    for (lc, lm), (rc, rm), op in zip(left, right, ops):
        assert np.all(cs.IE_OP[op](cs.ie_keys(lc)[pl], cs.ie_keys(rc)[pr])), f"a pair fails `{op}`"
        if lm is not None:
            assert lm[pl].all()
        if rm is not None:
            assert rm[pr].all()
    code = np.sort(pl * nr + pr)
    assert not np.any(code[1:] == code[:-1]), "a pair repeats"
    if len(sample_rows):
        starts = np.concatenate([[0], np.cumsum(slots)])
        for i, exp in zip(sample_rows, cs.ie_brute_rows(left, right, ops, sample_rows)):
            got = ri[starts[i]:starts[i + 1]]
            got = np.sort(got[matched[starts[i]:starts[i + 1]]].astype(np.int64))
            assert np.array_equal(got, exp), f"row {i}: {len(got)} pairs, brute force {len(exp)}"


def ie_run(plb, left, right, ops, how, location=None):
    kw = {} if location is None else {"location": location}
    return plb.ie_join([plb.Column(v, m) for v, m in left], [plb.Column(v, m) for v, m in right], list(ops), how, **kw)


IE_OP_PAIRS = [("<", ">"), (">=", "<="), ("<=", "<"), (">", ">=")]      # strict, non-strict, mixed both ways
# every pair at 2^20 and 2^20 + 1 rows; at 2^24 and 2^24 + 1 two each, so that the four pairs are split over the two sizes
IE_SCALE = [(m, ops) for m in (1 << 20, (1 << 20) + 1) for ops in IE_OP_PAIRS] + \
           [(1 << 24, IE_OP_PAIRS[0]), (1 << 24, IE_OP_PAIRS[2]), ((1 << 24) + 1, IE_OP_PAIRS[1]), ((1 << 24) + 1, IE_OP_PAIRS[3])]


@pytest.mark.parametrize("m,ops", IE_SCALE, ids=lambda x: "".join(x) if isinstance(x, tuple) else str(x))
def test_tree_levels_at_scale(plb, m, ops):
    """m live right rows give 21 / 22 / 25 / 26 levels; wide left x-ranges reach the top levels and the truncated last
    block, narrow ones the edge of the x-order; inner and left joins"""
    rng = np.random.default_rng(m % 1009 + 31 * IE_OP_PAIRS.index(ops))
    left, right = cs.ie_wide_case(rng, m, ops)
    counts = cs.ie_counts(left, right, ops)
    assert counts.max() > 0 and (counts == 0).any()
    sample = np.sort(rng.choice(len(left[0][0]), 256 if m < (1 << 24) else 24, replace=False))
    for how in ("inner", "left"):
        res, prof = profiled(plb, lambda: ie_run(plb, left, right, ops, how))
        check_ie(res, left, right, ops, how, counts, sample)
        assert prof.get("ie_level_keys") == cs.tree_levels(m), prof


@pytest.mark.parametrize("total", [512 * k + d for k in (1, 8, 1000) for d in (-1, 0, 1)] + [32 * k + d for k in (1, 5, 63) for d in (-1, 1)])
def test_left_join_validity_words(plb, total):
    """a left join whose unmatched rows alternate with rows that own pairs, to a total of 512k - 1 / 512k / 512k + 1 and
    32k +- 1 slots: every emit warp edge and a last partial validity word"""
    rng = np.random.default_rng(total)
    nr = 64
    rx = np.arange(nr, dtype=np.int64)                   # `l < r`: a row with x = nr - 1 - c owns c pairs
    counts, s = [], 0
    while s < total:
        c = 0 if len(counts) % 2 == 0 else min(int(rng.integers(1, nr)), total - s)
        counts.append(c)
        s += max(c, 1)
    counts = np.array(counts, np.int64)
    assert np.maximum(counts, 1).sum() == total
    lx = nr - 1 - counts
    left, right = [(lx, None)], [(rx, None)]
    res = ie_run(plb, left, right, ["<"], "left")
    check_ie(res, left, right, ["<"], "left", cs.ie_counts(left, right, ["<"]))


@pytest.mark.parametrize("nl", [255, 256, 257, 256 * 37 - 1, 256 * 37 + 1, 256 * 4099 - 1, 256 * 4099 + 1])
def test_count_cta_boundaries(plb, nl):
    """left sides around k_ie_count's 256-row CTA and its offset scan over many CTAs, two predicates, inner and left"""
    rng = np.random.default_rng(nl)
    nr = 40
    right = [(rng.integers(-50, 50, nr).astype(np.int32), rng.random(nr) >= 0.05), (rng.integers(0, 8, nr).astype(np.float64), None)]
    left = [(rng.integers(-60, 60, nl).astype(np.int32), rng.random(nl) >= 0.05), (rng.integers(-1, 9, nl).astype(np.float64), None)]
    for ops in (("<", ">="), (">=", "<")):
        counts = cs.ie_counts(left, right, ops)
        for how in ("inner", "left"):
            res, prof = profiled(plb, lambda: ie_run(plb, left, right, ops, how))
            check_ie(res, left, right, ops, how, counts, np.arange(min(nl, 64)))
            assert prof.get("ie_count") == 1


def test_past_2_31_output_slots(plb):
    """one predicate `<` with every pair accepted: 35 000 x 65 536 = 2 293 760 000 slots (about 18 GB) stay on the
    device and are checked in chunks of 2^28 slots against li = i // nr, ri = i % nr"""
    nl, nr = 35_000, 65_536
    total = nl * nr
    assert total > 1 << 31
    if plb.device_info()["hbm_free"] < 40 * (1 << 30):
        pytest.skip("needs 40 GB of free device memory")
    li, ri = plb.ie_join([np.zeros(nl, np.int64)], [np.ones(nr, np.int64)], ["<"], "inner", location=plb.DEVICE)
    try:
        assert li.length == total and ri.length == total and not ri.validity_ptr
        chunk = 1 << 28
        rows = chunk // nr
        expect_r = np.arange(nr, dtype=np.uint32)[None, :]
        for off in range(0, total, chunk):
            n = min(chunk, total - off)
            got = []
            for out in (li, ri):
                view = plb.Column(out.values_ptr, dtype=np.uint32, length=n, offset=off, location=plb.DEVICE).struct()
                host = plb.BlColumn()
                plb._check(plb.lib().bl_column_to(C.byref(view), C.c_int32(1), C.c_int32(plb.HOST), C.byref(host)))
                got.append(plb.OutColumn(host).to_numpy()[0].reshape(-1, nr))
            r0 = off // nr
            assert np.array_equal(got[0], np.arange(r0, r0 + n // nr, dtype=np.uint32)[:, None] + np.zeros((1, nr), np.uint32)), off
            assert (got[1] == expect_r).all(), off
            del got
    finally:
        li.free()
        ri.free()


# =========================================================================================== string-code collisions
def test_collision_retry_gives_exact_codes(plb):
    """two distinct 16-byte values with one hash under the first seed: the codes must still be exact (two str_hash
    launches), and so must an asof `by` key, a string group_by and a string hash join"""
    a, b = cs.colliding_pair(cs.SEEDS[0])
    vals = [a, b, b"x", a, None, b, b"x", a]
    (codes, valid), nd = plb.string_encode(plb.StringColumn(vals))
    first = {}
    exp = [None if v is None else first.setdefault(v, i) for i, v in enumerate(vals)]
    assert [None if (valid is not None and not valid[i]) else int(c) for i, c in enumerate(codes)] == exp and nd == 3
    _, prof = profiled(plb, lambda: plb.string_encode(plb.StringColumn(vals)))
    assert prof.get("str_hash") == 2, prof

    lvals = np.arange(12, dtype=np.int64) * 2
    rvals = np.arange(9, dtype=np.int64) * 3
    lby = [a, b, a, b, b"x", a, b, None, a, b, a, b]
    rby = [b, a, b, a, b, a, b"x", a, b]
    for strategy in STRATS:
        exp = ao.cursor_asof_by(list(lvals), list(rvals), [(s,) for s in lby], [(s,) for s in rby], strategy)
        vals_, ok = plb.join_asof(lvals, rvals, strategy, left_by=[plb.StringColumn(lby)], right_by=[plb.StringColumn(rby)])
        ok = np.ones(len(vals_), bool) if ok is None else ok
        assert [int(v) if o else None for v, o in zip(vals_, ok)] == exp, strategy

    keys, [(lens, _)] = plb.group_by_agg_strings(plb.StringColumn(vals), [("len", None)], True)
    got = dict(zip(keys, lens.tolist()))
    assert (got[a], got[b], got[b"x"]) == (3, 2, 2)

    (li, _), (ri, _) = plb.hash_join_strings(plb.StringColumn(lby), plb.StringColumn(rby))
    got = sorted(zip(li.tolist(), ri.tolist()))
    assert got == sorted((i, j) for i, x in enumerate(lby) for j, y in enumerate(rby) if x is not None and x == y)


def test_collisions_under_all_four_seeds_are_refused(plb):
    """four pairs, each colliding under a different seed: status 4 from string_encode and from an asof `by` key"""
    pairs = [cs.colliding_pair(s, b"%d" % k) for k, s in enumerate(cs.SEEDS)]
    vals = [v for p in pairs for v in p]
    assert len(set(vals)) == 8
    with pytest.raises(plb.B200Error, match="64-bit hash collisions under four seeds") as e:
        plb.string_encode(plb.StringColumn(vals))
    assert e.value.status == 4
    n = len(vals)
    with pytest.raises(plb.B200Error, match="64-bit hash collisions under four seeds") as e:
        plb.join_asof(np.arange(n, dtype=np.int64), np.arange(n, dtype=np.int64), "backward",
                      left_by=[plb.StringColumn(vals)], right_by=[plb.StringColumn(vals[::-1])])
    assert e.value.status == 4
