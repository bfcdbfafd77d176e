"""GPU tests of the order statistics built on the stable sort -- bl_top_k (top_k.cu), bl_rank (rank.cu) and
bl_rolling_quantile(_by) (rolling_quantile.cu) -- on every plan, past their grid caps and past 2^31 rows, against exact
references (tests/order_stats_cases.py; tests/test_order_stats_cases.py checks those against the plain oracles on CPU).

Row ids and ranks are compared with ==, float results by their bytes.  Which branch a step takes shows in the launch
profile (topk_pass / topk_pass_list / topk_tie / mask_first / topk_mark / topk_mark_list, rank_starts,
rolling_quantile_wm_count), so every test computes the plan of its input with the CPU restatement in order_stats_cases
and asserts the profile equals it.

Caps.  SM = device_info()["sm_count"]; the values in brackets are for SM = 132 (an H100 SXM).
  k_topk_pass / k_topk_andor  grid_for(rows, 256): 8 SM x 256 [270 336] rows per sweep.
  mask_first / mask_rows      grid_for(tiles x 128, 128): 8 SM tiles of 4096 rows [4 325 376 rows] per sweep.
  k_rank_heads / _starts / _out  min(ntiles, 8 SM) [1056] CTAs over tiles of 2048 positions: 8 SM x 2048 [2 162 688]
                              positions per sweep, after which s_w / s_cnt are reused for the next tile.
  k_wm_count / k_wm_split     one CTA per 1792-position tile, n / 1792 + 1 tiles (the last holds position n).
  k_rq_out                    grid_for(n, 256): 8 SM x 256 [270 336] positions per sweep.
No branch named in these kernels' host loops is left unreached; a top_k list that receives no row cannot occur (the
list holds exactly the previous bucket's count, which is at least `need` >= 1).
"""
import zlib

import numpy as np
import pytest

import order_stats_cases as oc
import rolling_quantile_oracle as rqo
import sort_oracle

pytestmark = pytest.mark.gpu

TK_NAMES = ("iota", "topk_andor", "topk_pass", "topk_pass_list", "topk_tie", "mask_first", "topk_mark", "topk_mark_list")
RK_NAMES = ("rank_heads", "rank_starts", "rank_out")


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as m
    m.init()
    return m


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


def profiled(plb, fn):
    plb.profile_reset()
    plb.profile_enable(True)
    try:
        out = fn()
        plb.sync()
        prof = plb.profile()
    finally:
        plb.profile_enable(False)
    return out, {k: int(v.get("launches", 0)) for k, v in prof.items()}


def only(prof, names):
    return {k: v for k, v in prof.items() if k in names and v}


def arg(cols, valids):
    return [(c, v) if v is not None else c for c, v in zip(cols, valids)]


# =========================================================================================== top_k
def run_topk(plb, cols, valids, dtypes, k, desc=False, nl=False, div=oc.TK_LIST_DIV):
    plan = oc.topk_plan(cols, valids, dtypes, k, desc, nl, div)
    got, prof = profiled(plb, lambda: plb.arg_top_k(arg(cols, valids), k, desc, nl))
    exp = oc.topk_ref(cols, valids, k, desc, nl)
    assert np.array_equal(plan["ids"], exp)
    assert got.dtype == np.uint32 and np.array_equal(got, exp), (k, desc, nl, got[:8], exp[:8])
    assert only(prof, TK_NAMES) == only(plan["launches"], TK_NAMES), (prof, plan["launches"])
    return plan


def strided_key(n, stride, at, rest=1):
    """UInt8 0 at rows r % stride == at, `rest` elsewhere: one small bucket spread over every row"""
    x = np.full(n, rest, np.uint8)
    x[at::stride] = 0
    return x


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_topk_first_bucket_at_the_list_threshold(plb, sm, delta):
    """a first bucket of n/32 + delta rows over n = 32 (8 SM 256 + 7) rows: at n/32 or below the next pass appends a
    list and the rest run over it; above, the next pass streams too"""
    n = 32 * (8 * sm * 256 + 7)
    size = n // 32 + delta
    rng = np.random.default_rng(5 + delta)
    x = (np.full(n, 9 << 8) | rng.integers(0, 256, n)).astype(np.uint32)
    pick = np.sort(rng.choice(n, size, replace=False))
    x[pick] = (2 << 8) | rng.integers(0, 4, size)
    for k in (size // 3, size - 1):
        plan = run_topk(plb, [x], [None], ["uint32"], k)
        assert plan["steps"][0]["count"] == size
        assert plan["steps"][1]["appends"] == (delta <= 0) and not plan["steps"][1]["list"]


@pytest.mark.parametrize("n,digits", [(2**8, 1), (2**8 + 1, 2), (2**16 + 1, 3), (2**24 + 1, 4)])
def test_topk_list_into_row_digits(plb, n, digits):
    """one small bucket (rows r % 64 == 5) that reaches the row index: 1-4 row digits, list passes that append shorter
    lists (a pass that keeps its whole list appends none);
    k cuts the bucket in its middle, and k = the bucket's rows below a row-digit boundary takes a last bucket whole
    inside list mode (topk_mark_list)"""
    x = strided_key(n, 64, 5)
    cands = np.flatnonzero(x == 0)
    plan = run_topk(plb, [x], [None], ["uint8"], len(cands) // 2 + 1)
    assert plan["row_digits"] == digits
    sizes = [s["rows"] for s in plan["steps"] if s["list"]]
    assert sizes == sorted(sizes, reverse=True)
    assert plan["launches"]["topk_pass_list"] == digits - 1 and plan["launches"]["topk_mark_list"] == 1
    if digits >= 3:
        assert any(s["list"] and s["appends"] for s in plan["steps"]), plan["steps"]      # a list pass appends a shorter list
        k = int((cands < 256 * 40).sum())
        plan = run_topk(plb, [x], [None], ["uint8"], k)
        assert plan["launches"]["topk_mark_list"] == 1 and plan["launches"]["topk_pass_list"] < digits - 1, plan


def test_topk_bucket_of_exactly_need(plb, sm):
    """the bucket holds exactly `need` rows: one mark pass at or below it, streaming (first bucket, many rows) and in
    list mode (a small bucket taken whole at its first row digit)"""
    n = 3 * 8 * sm * 256 + 11
    x = strided_key(n, 3, 1)
    plan = run_topk(plb, [x], [None], ["uint8"], int((x == 0).sum()))
    assert plan["launches"]["topk_mark"] == 1 and len(plan["steps"]) == 1
    y = strided_key(n, 64, 7)
    c = np.flatnonzero(y == 0)
    top = (oc.bits_for(n - 1) - 1) // 8 * 8
    plan = run_topk(plb, [y], [None], ["uint8"], int((c < (1 << top)).sum()))
    assert plan["launches"]["topk_mark_list"] == 1 and plan["steps"][-1]["count"] == plan["steps"][-1]["need"]


@pytest.mark.parametrize("which", ["1", "F_TILE-1", "F_TILE", "F_TILE+1", "count-1", "second-bucket"])
def test_topk_tie_step(plb, sm, which):
    """candidates that tie on the whole key and hold more than n / 32 rows: one streaming pass (topk_tie) and the first
    `need` of them by 4096-row tile counts (mask_first) over n = 2 x 8 SM x 4096 + 77 rows (two mask sweeps)"""
    n = 2 * 8 * sm * oc.F_TILE + 77
    x = (np.arange(n) % 3 != 0).astype(np.int16) * 5 - 2      # -2 at r % 3 == 0, 3 elsewhere
    c0 = int((x == -2).sum())
    for desc in (False, True):
        c = c0 if not desc else n - c0      # the first bucket's rows
        k = {"1": 1, "F_TILE-1": oc.F_TILE - 1, "F_TILE": oc.F_TILE, "F_TILE+1": oc.F_TILE + 1, "count-1": c - 1,
             "second-bucket": n - 1}[which]
        plan = run_topk(plb, [x], [None], ["int16"], k, desc)
        assert plan["launches"]["topk_tie"] == 1 and plan["launches"]["mask_first"] == 1
        assert plan["tie"] == (k if which != "second-bucket" else n - c - 1)


@pytest.mark.parametrize("desc", [False, True])
@pytest.mark.parametrize("nl", [False, True])
def test_topk_null_parts(plb, sm, desc, nl):
    """a varying null part over a constant value part (only the null digit and the row index decide), and an all-null
    column (no varying digit: rows 0 .. k without a pass)"""
    n = 8 * sm * 256 + 99
    rng = np.random.default_rng(11 + 2 * desc + nl)
    x = np.full(n, 7, np.int32)
    valid = rng.random(n) < 0.5
    for k in (1, int(valid.sum()) - 1, int(valid.sum()) + 5, n - 1):
        plan = run_topk(plb, [x], [valid], ["int32"], k, desc, nl)
        assert plan["steps"][0]["part"] == 0 and all(s["part"] != 1 for s in plan["steps"])
    for k in (1, 4097, n - 1):
        plan = run_topk(plb, [x], [np.zeros(n, bool)], ["int32"], k, desc, nl)
        assert plan["launches"]["iota"] == 1 and plan["launches"]["topk_pass"] == 0


def test_topk_second_column_constant_on_candidates(plb, sm):
    """column b varies over all rows but is constant on the candidates column a leaves: b's digits still get passes,
    each keeping every candidate"""
    n = 8 * sm * 256 + 5
    rng = np.random.default_rng(13)
    a = rng.integers(1, 50, n).astype(np.int64)
    a[::97] = 0
    b = rng.integers(-2**40, 2**40, n)
    b[a == 0] = 12345
    k = int((a == 0).sum()) // 2
    plan = run_topk(plb, [a, b], [None, None], ["int64", "int64"], k)
    bsteps = [s for s in plan["steps"] if s["part"] == 1]
    assert bsteps and all(s["count"] == int((a == 0).sum()) for s in bsteps)
    plan = run_topk(plb, [a, b], [None, None], ["int64", "int64"], k, [False, True])
    assert [s for s in plan["steps"] if s["part"] == 1]


@pytest.mark.parametrize("div", ["1", "n"])
def test_topk_list_div_knob(plb, monkeypatch, div):
    """BL_TOPK_LIST_DIV, read per call: 1 lists every candidate set smaller than the rows, n lists only a single row"""
    n = 300_001
    rng = np.random.default_rng(17)
    x = rng.integers(0, 1000, n).astype(np.int32)
    d = 1 if div == "1" else n
    monkeypatch.setenv("BL_TOPK_LIST_DIV", str(d))
    for k in (1, 150, n // 2):
        plan = run_topk(plb, [x], [None], ["int32"], k, False, False, d)
        if d == 1:
            assert plan["launches"]["topk_pass_list"] > 0 and plan["launches"]["topk_tie"] == 0
        else:
            assert plan["launches"]["topk_pass_list"] == 0


@pytest.mark.parametrize("off", [0, 1])
def test_sort_limit_select_first(plb, sm, off):
    """a sort with limit n/8 selects first (op_top_k), limit n/8 + 1 sorts everything: the same bytes as the full sort"""
    n = 8 * (8 * sm * 256 + 3)
    rng = np.random.default_rng(19 + off)
    x = rng.integers(-2**31, 2**31, n).astype(np.int32)
    x[::5] = 77
    valid = rng.random(n) < 0.95
    limit = n // oc.SELECT_DIV + off
    full = plb.arg_sort([(x, valid)], True, True)
    got, prof = profiled(plb, lambda: plb.arg_sort([(x, valid)], True, True, limit=limit))
    assert got.tobytes() == full[:limit].tobytes()
    assert (prof.get("topk_andor", 0) > 0) == (off == 0), prof


# =========================================================================================== rank
SEG_HEADS = [0, 32, 768, 2047, 2048, 25 * oc.RK_TILE, 40 * oc.RK_TILE + 31, 70 * oc.RK_TILE]


def rank_shape(sm, parts, nulls, rng):
    """sorted positions with run heads on every lane-0 / lane-31 position of the first two tiles' warp words, at warp
    and tile edges, one run over 20 tiles and past the 8 SM tile grid.  parts: partitions starting at SEG_HEADS and
    n - 3 (lane 0 / lane 31, warp and tile edges); row g holds a position of partition g, so the partitions' first rows
    (their ids, partition_ids) sort them in this order.  nulls: every partition's last run is null (a null run after
    valid runs), partition 4 ([2048, 25 x 2048)) wholly so, and without partitions the column's last run.
    Returns (x, valid, gid, designed run heads, designed partition heads)."""
    n = (8 * sm + 3) * oc.RK_TILE + 5
    heads = {p for p in range(2 * oc.RK_TILE) if p % 32 in (0, 31)}
    heads |= {p for t in range(2, 60) for p in (t * oc.RK_TILE - 1, t * oc.RK_TILE, t * oc.RK_TILE + 255, t * oc.RK_TILE + 256)}
    heads |= set(range(80 * oc.RK_TILE, n, 997))      # many short runs past the first wave of tiles
    heads = {h for h in heads if h < n and not (3 * oc.RK_TILE < h < 23 * oc.RK_TILE)}      # one run over 20 tiles
    seg = SEG_HEADS + [n - 3] if parts else [0]
    heads |= set(seg)
    val = oc.labels_from_heads(n, sorted(heads))
    gpos = oc.labels_from_heads(n, seg)
    ok = np.ones(n, bool)
    if nulls:
        ends = seg[1:] + [n]
        hs = np.array(sorted(heads))
        for a, b in zip(seg, ends):
            ok[hs[(hs >= a) & (hs < b)].max():b] = False
        if parts:
            ok[gpos == 4] = False
    perm = rng.permutation(n)      # perm[p]: the row at sorted position p
    for g, p in enumerate(seg):      # row g into partition g's first position
        j = int(np.flatnonzero(perm == g)[0])
        perm[j], perm[p] = perm[p], perm[j]
    x = np.empty(n, np.int64)
    x[perm] = val * 3 - 1_000_000
    gid = np.empty(n, np.int64)
    gid[perm] = gpos * 7919 + 13      # partition values unrelated to the partition order
    valid = np.empty(n, bool)
    valid[perm] = ok
    return x, (valid if nulls else None), (gid if parts else None), sorted(heads), seg


@pytest.mark.parametrize("nulls", [False, True])
@pytest.mark.parametrize("parts", [False, True])
def test_rank_every_method_at_warp_and_tile_edges(plb, sm, parts, nulls):
    """every method over more tiles than the 8 SM grid (each CTA runs two tiles and reuses s_w / s_cnt).  The run and
    partition heads k_rank_heads sees (order_stats_cases.rank_heads: the device's sort by first-row partition id, nulls
    last) are the designed ones, and fall on lane 0 / lane 31 of warp words and on warp and tile edges: a partition head
    at lane 0 decides seg_head from the carried left neighbour.  The launch profile shows rank_starts exactly where
    rank_plan allocates start or seg_pos; the MAX rank of the last run ends at n."""
    rng = np.random.default_rng(23 + 2 * parts + nulls)
    x, valid, gid, heads, seg = rank_shape(sm, parts, nulls, rng)
    n = len(x)
    run_h, seg_h = oc.rank_heads(x, valid, gid)
    assert seg_h.tolist() == seg
    if not nulls:
        assert run_h.tolist() == heads
    places = oc.head_places(run_h)
    assert all(v > 0 for v in places.values()), places
    if parts:
        places = oc.head_places(seg_h)
        assert all(v > 0 for v in places.values()), places
    plans = [oc.rank_plan(n, m, parts, nulls, sm) for m in oc.RANK_METHODS]
    assert all(p["ntiles"] > p["grid"] for p in plans)
    col = (x, valid) if nulls else x
    outs, prof = profiled(plb, lambda: plb.rank([(col, {"method": m}) for m in oc.RANK_METHODS], partition_by=[gid] if parts else []))
    assert only(prof, RK_NAMES) == dict(oc.rank_launches(plans)), prof
    for m, (v, vm) in zip(oc.RANK_METHODS, outs):
        exp = oc.rank_ref(x, valid, m, False, gid)
        assert v.dtype == exp.dtype
        ok = np.ones(n, bool) if valid is None else valid
        assert np.array_equal(np.ones(n, bool) if vm is None else vm, ok), m
        bad = np.flatnonzero((v != exp) & ok)
        assert bad.size == 0, (m, bad[:5], v[bad[:5]], exp[bad[:5]])
    if not parts and not nulls:
        last = x == x.max()
        assert (outs[2][0][last] == n).all()


def test_rank_dense_all_null_partition_and_descending(plb, sm):
    """DENSE and MIN descending over partitions where one is all null and the others end in a null run"""
    rng = np.random.default_rng(29)
    x, valid, gid, _, _ = rank_shape(sm, True, True, rng)
    outs = plb.rank([((x, valid), {"method": "dense", "descending": True}), ((x, valid), {"method": "min", "descending": True})], partition_by=[gid])
    for m, (v, _) in zip(("dense", "min"), outs):
        exp = oc.rank_ref(x, valid, m, True, gid)
        assert np.array_equal(np.where(valid, v, 0), exp), m


# =========================================================================================== rolling quantile
RQ_SIZES = [1, 2, 223, 224, 225, 1791, 1792, 1793, 2**12, 2**12 + 1]


def rq_cases():
    """(q, method) pairs: every method at q = 0 and at q = 0.5 (fi on an integer or exactly at .5 over odd / even
    counts), and the two interpolations at a quarter and at q = 1"""
    return [(q, m) for m in oc.QMETHODS for q in (0.0, 0.5)] + [(q, m) for m in ("midpoint", "linear") for q in (0.25, 1.0)]


@pytest.mark.parametrize("n", RQ_SIZES)
@pytest.mark.parametrize("nulls", [False, True])
def test_rolling_quantile_block_and_tile_edges(plb, n, nulls):
    """windows of 224, 225 and 1792 positions at n around the 224-position block and 1792-position tile: s and e on
    block and tile edges, e == n on a tile edge when n % 1792 == 0.  Nulls: a null run longer than every window (all-null
    windows) and windows below min_samples.  Every method of rq_cases; L levels plus the null bitvector
    in the launch profile."""
    rng = np.random.default_rng(zlib.crc32(f"rq-{n}-{nulls}".encode()))
    x = rng.integers(-50, 50, n).astype(np.float64)
    valid = None
    if nulls:
        valid = rng.random(n) >= 0.2
        valid[n // 3: n // 3 + 2000] = False
    plan = oc.rq_plan(n, nulls and not valid.all())
    edges = {}
    for w in (224, 225, 1792):
        for center in (False, True):
            ms = max(1, w // 2)
            s, e = oc.fixed_bounds(n, w, center)
            for k, v in oc.rq_edges(s, e, n).items():
                edges[k] = edges.get(k, 0) + v
            wins = oc.rq_windows(x, valid, np.float64, s, e)
            cases = rq_cases()
            col = (x, valid) if nulls else x
            outs, prof = profiled(plb, lambda: plb.rolling_quantile([(col, {"quantile": q, "interpolation": m, "window_size": w, "min_samples": ms, "center": center})
                                                                    for q, m in cases]))
            assert prof.get("rolling_quantile_wm_count", 0) == plan["wm_count"], (prof, plan)
            for (q, m), (v, vm) in zip(cases, outs):
                ev, ok = oc.rq_pick(wins, np.float64, q, m, ms)
                gm = np.ones(n, bool) if vm is None else vm
                assert np.array_equal(gm, ok), (w, center, q, m)
                assert v[ok].tobytes() == ev[ok].tobytes(), (w, center, q, m, np.flatnonzero(v[ok] != ev[ok])[:5])
    if n >= 1793:
        assert edges["s_block"] and edges["e_block"] and edges["e_tile"], edges
    if n >= 2**12:
        assert edges["s_tile"], edges
    if n % oc.BV_TILE == 0:
        assert edges["e_n_on_tile"], edges


def test_rolling_quantile_float32_and_equiprobable_at_zero(plb):
    """Float32 arithmetic (midpoint and linear in f32) and EQUIPROBABLE at q = 0 over n = 1793 with nulls"""
    n = 1793
    rng = np.random.default_rng(31)
    x = (rng.integers(-1000, 1000, n) / 8).astype(np.float32)
    valid = rng.random(n) >= 0.1
    s, e = oc.fixed_bounds(n, 225, True)
    wins = oc.rq_windows(x, valid, np.float32, s, e)
    cases = [(0.0, "equiprobable"), (0.5, "midpoint"), (0.5, "linear"), (0.3, "linear"), (0.7, "midpoint")]
    outs = plb.rolling_quantile([((x, valid), {"quantile": q, "interpolation": m, "window_size": 225, "min_samples": 3, "center": True}) for q, m in cases])
    for (q, m), (v, vm) in zip(cases, outs):
        ev, ok = oc.rq_pick(wins, np.float32, q, m, 3)
        assert v.dtype == np.float32 and np.array_equal(np.ones(n, bool) if vm is None else vm, ok)
        assert v[ok].tobytes() == ev[ok].tobytes(), (q, m)


def test_rolling_quantile_over_and_by_past_the_grid(plb, sm):
    """.over() positions (partition order, rows scattered back) and rolling_quantile_by over n > 3 x 8 SM x 256 rows:
    k_rq_out's grid-stride loop runs more than three sweeps.  The references are the wavelet-matrix restatement
    (rolling_quantile_oracle.numpy_rolling_quantile), exact by bytes."""
    n = 3 * 8 * sm * 256 + 101
    rng = np.random.default_rng(37)
    x = rng.integers(-200, 200, n).astype(np.float64)
    valid = rng.random(n) >= 0.1
    gid = rng.integers(0, 500, n)
    order = np.lexsort((np.arange(n), gid))
    gs = gid[order]
    heads = np.flatnonzero(np.r_[True, gs[1:] != gs[:-1]])
    starts = np.repeat(heads, np.diff(np.r_[heads, n]))
    ends = np.repeat(np.r_[heads[1:], n], np.diff(np.r_[heads, n]))
    i = np.arange(n)
    s, e = np.maximum(i - 29, starts), np.minimum(i + 1, ends)
    for q, m in ((0.5, "linear"), (0.25, "nearest"), (1.0, "higher")):
        [(v, vm)] = plb.rolling_quantile([((x, valid), {"quantile": q, "interpolation": m, "window_size": 30, "min_samples": 5})], partition_by=[gid])
        ev, ok = rqo.numpy_rolling_quantile(x[order], valid[order], "float64", q, m, s, e, 5)
        got, gm = np.empty(n), np.empty(n, bool)
        got[order], gm[order] = ev, ok
        assert np.array_equal(np.ones(n, bool) if vm is None else vm, gm), (q, m)
        assert v[gm].tobytes() == got[gm].tobytes(), (q, m)
    t = np.sort(rng.integers(0, n // 3, n)).astype(np.int64)
    s = np.searchsorted(t, t - 40, "right")
    e = np.searchsorted(t, t, "right")
    for q, m in ((0.5, "midpoint"), (0.0, "equiprobable")):
        [(v, vm)] = plb.rolling_quantile_by([((x, valid), {"quantile": q, "interpolation": m, "window_size": 40, "min_samples": 2})], t)
        ev, ok = rqo.numpy_rolling_quantile(x, valid, "float64", q, m, s, e, 2, live=(e - s) >= 2)
        assert np.array_equal(np.ones(n, bool) if vm is None else vm, ok), (q, m)
        assert v[ok].tobytes() == ev[ok].tobytes(), (q, m)


# =========================================================================================== past 2^31 rows
N_BIG = 2**31 + 2**20 + 33
N_MAX = 2**32 - 1
CHUNK = 1 << 27


class _Dev:
    """a device buffer as a torch tensor, without a copy"""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3}


@pytest.fixture(scope="module")
def torch():
    t = pytest.importorskip("torch")
    if not t.cuda.is_available():
        pytest.skip("no CUDA device for torch")
    return t


def need(plb, torch, nbytes):
    """skip unless nbytes of device memory are free once the library's and torch's cached blocks are returned"""
    torch.cuda.empty_cache()
    plb.release_cached()
    free = plb.device_info()["hbm_free"]
    if free < nbytes:
        pytest.skip(f"needs {nbytes / 2**30:.0f} GiB of free device memory, {free / 2**30:.0f} GiB free")


def settle(plb, torch):
    """return torch's temporaries and the library's cached blocks to the driver before a call near the memory limit"""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    plb.release_cached()


def dev_view(torch, out, n, typestr):
    return torch.as_tensor(_Dev(out.values_ptr, n, typestr), device="cuda")


def valid_bits(torch, out, lo, hi):
    """the validity bits of rows [lo, hi) of a device output (lo a multiple of 8)"""
    b = torch.as_tensor(_Dev(out.validity_ptr + lo // 8, (hi - lo + 7) // 8, "|u1"), device="cuda")
    bits = (b.unsqueeze(1) >> torch.arange(8, device="cuda", dtype=torch.uint8)) & 1
    return bits.reshape(-1)[: hi - lo].bool()


def arange_chunks(torch, n):
    for off in range(0, n, CHUNK):
        yield off, torch.arange(off, min(n, off + CHUNK), device="cuda", dtype=torch.int64)


def test_past_2_31_top_k_tie_step(plb, torch):
    """UInt8 v = (r % 4 == 3) over 2^32 - 1 rows, k = 3 x 2^30 - 7: one digit, a first bucket of 3 x 2^30 rows, then the
    tie step with need = k > 2^31 (mask_first's per-tile offsets pass 2^31).  Row i of the answer is the i-th row with
    r % 4 != 3: i + i // 3.  Peak: 4 GiB of keys, 2 x 512 MiB of bitmaps and 12 GiB of ids, about 17 GiB."""
    n, k = N_MAX, 3 * 2**30 - 7
    need(plb, torch, 18 << 30)
    x = torch.empty(n, dtype=torch.uint8, device="cuda")
    for off, r in arange_chunks(torch, n):
        x[off:off + len(r)] = (r % 4 == 3).to(torch.uint8)
    torch.cuda.synchronize()
    xc = plb.Column(x.data_ptr(), dtype=np.uint8, length=n, location=plb.DEVICE)
    out, prof = profiled(plb, lambda: plb.arg_top_k(xc, k, location=plb.DEVICE))
    plb.release_cached()
    assert only(prof, TK_NAMES) == {"topk_andor": 1, "topk_pass": 1, "topk_tie": 1, "mask_first": 1}, prof
    try:
        assert out.length == k
        got = dev_view(torch, out, k, "<u4")
        for off, i in arange_chunks(torch, k):
            assert torch.equal(got[off:off + len(i)].to(torch.int64) & 0xFFFFFFFF, i + i // 3), off
        del got
    finally:
        out.free()
    del x
    torch.cuda.empty_cache()


def test_past_2_31_top_k_list_passes(plb, torch):
    """UInt8 0 at rows r % 64 == 5 and 1 elsewhere over 2^32 - 1 rows, k = 2^25 + 12345: the value digit leaves 2^26
    candidates (< n / 32), the first row digit (shift 24) streams and appends them, the digits at 16, 8 and 0 run over
    lists of 2^26, 2^18 and 1024 32-bit row ids, and the last bucket (one row) is marked from the list.  The answer,
    5 + 64 i for i < k, ends past row 2^31.  Peak: 4 GiB of keys, 256 MiB of lists, 128 MiB of ids."""
    n, k = N_MAX, 2**25 + 12345
    need(plb, torch, 6 << 30)
    x = torch.ones(n, dtype=torch.uint8, device="cuda")
    x[5::64] = 0
    torch.cuda.synchronize()
    xc = plb.Column(x.data_ptr(), dtype=np.uint8, length=n, location=plb.DEVICE)
    out, prof = profiled(plb, lambda: plb.arg_top_k(xc, k, location=plb.DEVICE))
    assert only(prof, TK_NAMES) == {"topk_andor": 1, "topk_pass": 2, "topk_pass_list": 3, "topk_mark_list": 1}, prof
    try:
        got = dev_view(torch, out, k, "<u4").to(torch.int64) & 0xFFFFFFFF
        assert out.length == k and int(got[-1]) > 2**31
        assert torch.equal(got, 5 + 64 * torch.arange(k, device="cuda", dtype=torch.int64))
        del got
    finally:
        out.free()
    del x
    torch.cuda.empty_cache()


def test_past_2_31_rank(plb, torch):
    """MIN and ORDINAL of UInt32 values v_r = (n - 1 - r) >> 1 (descending pairs) over n = 2^31 + 2^20 + 33 rows, and
    MIN of the distinct v_r = n - 1 - r: the sort, start[] and (distinct) the packed run count all pass 2^31.  With
    j = n - 1 - r and P = j >> 1: MIN = 2P + 1; ORDINAL = 2P + 1 + (j even and 2P + 1 < n) (the lower row of a pair
    sorts first).  Distinct: MIN = j + 1.  Peak, one op at a time (the library's blocks are rounded to 1/16 of a power of
    two): 8 GiB of values, 9 GiB of ranks and op_arg_sort's 9 + 9 + 18 + 18 GiB, about 71 GiB."""
    n = N_BIG
    need(plb, torch, 72 << 30)
    x = torch.empty(n, dtype=torch.int32, device="cuda")
    xc = plb.Column(x.data_ptr(), dtype=np.uint32, length=n, location=plb.DEVICE)
    for pairs, method in ((True, "min"), (True, "ordinal"), (False, "min")):
        for off, r in arange_chunks(torch, n):
            j = n - 1 - r
            v = (j >> 1) if pairs else j
            x[off:off + len(r)] = ((v + 2**31) % 2**32 - 2**31).to(torch.int32)      # the UInt32 bits
        settle(plb, torch)
        [out], prof = profiled(plb, lambda: plb.rank([(xc, {"method": method})], location=plb.DEVICE))
        plb.release_cached()      # the sort's blocks go back to the driver for torch's checks
        assert prof.get("rank_starts", 0) == (1 if method == "min" else 0), prof
        try:
            got = dev_view(torch, out, n, "<u4")
            for off, r in arange_chunks(torch, n):
                j = n - 1 - r
                P = j >> 1
                if not pairs:
                    exp = j + 1
                elif method == "min":
                    exp = 2 * P + 1
                else:
                    exp = 2 * P + 1 + ((j % 2 == 0) & (2 * P + 1 < n)).to(torch.int64)
                assert torch.equal(got[off:off + len(r)].to(torch.int64) & 0xFFFFFFFF, exp), (pairs, method, off)
            del got
        finally:
            out.free()
    del x
    torch.cuda.empty_cache()


def test_past_2_31_rolling_quantile(plb, torch):
    """Float32 values r >> 8 (exact) over n = 2^31 + 2^20 + 33 rows, window 1000, two ops sharing one matrix: the
    matrix has 32 levels (rank queries at positions past 2^31, a level bit at 1 << 31) and the closed form of a
    non-decreasing column gives every window's k-th value as v(s + k) with s = max(i - 999, 0), e = i + 1.  LINEAR at
    0.5 keeps the default min_samples = 1000 (the first 999 rows are null); NEAREST at 0.25 takes min_samples = 1, so the
    clipped windows at the start hold 1 .. 999 values.  Validity and values are checked at every row.  Peak: 8 GiB of
    values and op_arg_sort's 54 GiB (the ranks and values are allocated after it), about 63 GiB; then 9 + 9 + 10 + 9 GiB
    of ranks, values, levels and split, and 2 x 9 GiB of outputs."""
    n, w = N_BIG, 1000
    need(plb, torch, 64 << 30)
    x = torch.empty(n, dtype=torch.float32, device="cuda")
    for off, r in arange_chunks(torch, n):
        x[off:off + len(r)] = (r >> 8).to(torch.float32)
    settle(plb, torch)
    xc = plb.Column(x.data_ptr(), dtype=np.float32, length=n, location=plb.DEVICE)
    assert oc.rq_levels(n) == 32
    cases = [(0.5, "linear", w), (0.25, "nearest", 1)]
    outs, prof = profiled(plb, lambda: plb.rolling_quantile([(xc, {"quantile": q, "interpolation": m, "window_size": w, "min_samples": ms})
                                                            for q, m, ms in cases], location=plb.DEVICE))
    plb.release_cached()
    assert prof.get("rolling_quantile_wm_count", 0) == 32, prof
    try:
        for (q, m, ms), out in zip(cases, outs):
            assert out.length == n and out.validity_ptr
            got = dev_view(torch, out, n, "<f4")
            for off, i in arange_chunks(torch, n):
                s = torch.clamp(i - (w - 1), min=0)
                ok = (i + 1 - s) >= ms
                assert torch.equal(valid_bits(torch, out, off, off + len(i)), ok), (q, m, off)
                exp = oc.rq_monotone(lambda r: (r >> 8).to(torch.float32), q, m, s, i + 1, torch.float32, xp=torch)
                g = got[off:off + len(i)]
                assert torch.equal(g[ok], exp[ok]), (q, m, off)
            del got
    finally:
        for out in outs:
            out.free()
    del x
    torch.cuda.empty_cache()


def test_release_cached_returns_the_library_blocks(plb, torch):
    """an arg_sort of 2^26 Int64 rows leaves about 1.5 GiB of sort buffers in the library's cache, which hbm_free does
    not count; release_cached returns them (hbm_free grows by at least 1 GiB) and the next call allocates afresh and
    gives the same order"""
    rng = np.random.default_rng(43)
    x = rng.integers(-2**40, 2**40, 2**26)
    first = plb.arg_sort(x)
    plb.sync()
    torch.cuda.empty_cache()
    before = plb.device_info()["hbm_free"]
    plb.release_cached()
    after = plb.device_info()["hbm_free"]
    assert after - before >= 1 << 30, (before, after)
    assert np.array_equal(plb.arg_sort(x), first)
    assert np.array_equal(first[:1000], np.argsort(x, kind="stable")[:1000].astype(np.uint32))


def test_grouped_past_2_31_and_top_k_past_2_32_refused(plb, torch):
    """headers of 2^31 rows with partitions (rank, rolling_quantile, rolling_quantile_by) and of 2^32 rows (top_k) over
    a small buffer: refused with UNSUPPORTED before any column is read"""
    buf = torch.zeros(64, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    big = plb.Column(buf.data_ptr(), dtype=np.int64, length=2**31, location=plb.DEVICE)
    huge = plb.Column(buf.data_ptr(), dtype=np.int64, length=2**32, location=plb.DEVICE)
    calls = [lambda: plb.rank([(big, {"method": "min"})], partition_by=[big]),
             lambda: plb.rolling_quantile([(big, {"quantile": 0.5, "window_size": 3})], partition_by=[big]),
             lambda: plb.rolling_quantile_by([(big, {"quantile": 0.5, "window_size": 3})], big, partition_by=[big]),
             lambda: plb.arg_top_k(huge, 5)]
    for call, pat in zip(calls, [r"2\^31 - 1 rows", r"2\^31 - 1 rows", r"2\^31 - 1 rows", r"2\^32 - 1 rows"]):
        with pytest.raises(plb.B200Error, match=pat) as e:
            call()
        assert e.value.status == 4
    del buf
