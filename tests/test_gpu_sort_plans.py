"""GPU tests of the sort family on every plan and past its grid caps, against exact references: the stable LSD radix sort
(filter.cu: k_rs_hist / k_rs_scan / k_rs_scatter, radix_sort_pairs_u32 / _u64, sort_pairs_u32), bl_arg_sort / bl_sort
(sort.cu), bl_string_rank / bl_arg_sort_keys (string_rank.cu) and the per-group median / quantile (quantile.cu).

Permutations and ranks must equal the reference element for element (np.argsort(kind="stable"), sort_oracle, a dense
rank from Python's sorted() over bytes, numpy GroupsIdx); quantiles bit for bit up to the sign of a zero and the payload
of a NaN (quantile_oracle; test_gpu_quantile.assert_same).  The launch profile proves which plan ran and how many radix
passes it took.  tests/test_sort_cases.py checks the large-input references against the plain oracles on CPU.

Caps.  SM = device_info()["sm_count"] (132 on an H100 SXM); the values in brackets are for SM = 132.
  k_sort_encode           grid_for(n, 256): at most 8*SM CTAs x 256 threads; its grid-stride loop runs again past
                          8*SM*256 rows [270 336].  N_ENC = 3*8*SM*256 + 77 [811 085] runs it four times, ragged.
  radix_sort_pairs        tiles of 4096 rows; n_ctas0 = min(tiles, SM*per_sm, 1024) with per_sm from an occupancy
                          query (not visible from Python, so every p in 1..8 is tried: SM*p = [132 .. 924], 1024 from p
                          = 8); a CTA owns chunk = ceil(tiles / n_ctas0) tiles, and CTAs = ceil(n / (chunk*4096)):
                          tiles = C0 + 1 (C0 = min(SM*p, 1024)) gives chunks of 2 tiles and drops C0 - ceil((C0 + 1)
                          / 2) trailing CTAs [65 at p = 1], 2*C0 tiles with a ragged last tile gives C0 CTAs of 2
                          tiles [up to 8 387 608 rows].
  k_rs_scatter            16 rounds of 32 lanes per warp, 512 consecutive rows per warp; lanes past the end carry the
                          "no item" digit 256.  4095 / 4096 / 4097 rows and a 37-row last tile.
  sort_pairs_u32          ceil(bits_for(n) / 8) passes for GroupsIdx: 1 up to n = 255, 2 up to 65 535, 3 up to
                          2^24 - 1, 4 from 2^24; an odd count leaves the result in the spare buffer and copies it back.
  k_str_rank_heads/apply  min(ntiles, 8*SM) CTAs of 4096 entries: loop past 8*SM*4096 active entries [4 325 376].
  string bucket stage     digits of the largest bucket id: 3 past 65 536 active buckets.
  k_quantile_small        window b takes the groups starting in [2048 b, 2048 (b+1)), the last dropped if larger than
                          2048; at most 2*2048 - 1 = 4095 keys (a full 4096-key network), 2048 local ids.
  QS_MAX_PICKS            16 quantiles of one column per sort: 17 and 33 take 2 and 3.
  k_quantile_find_large   grid_for(G, 256): past 8*SM*256 groups [270 336].
  k_quantile_pick_large   grid_for(NL*picks, 256): past 8*SM*256 (group, quantile) pairs [270 336].
  segment stage           skipped at NL = 1; ceil(bits_for(NL - 1) / 8) digits: 2 past 256 large groups, 3 past 65 536.
  large-group radix sort  L rows: more than one tile per CTA at any occupancy past 1024*4096 = 4 194 304 rows.
"""
import math

import numpy as np
import pytest

import quantile_oracle as qo
import sort_cases as sc
import sort_oracle
from test_gpu_quantile import assert_same, dev_group_quantiles, kind_of

pytestmark = pytest.mark.gpu

RS_TILE = 4096
RS_MAX_CTAS = 1024
SR_TILE = 4096
H = sc.QS_H
WIDTH = {"u32": np.uint32, "u64": np.uint64}


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as m
    m.init()
    return m


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


def n_enc(sm):
    return 3 * 8 * sm * 256 + 77


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


def bits_for(x):
    b = 1
    while b < 32 and (x >> b):
        b += 1
    return b


# =========================================================================================== 1. the radix sort itself
def set_digit(k, d, byte):
    sh = np.uint64(8 * d)
    return (k & ~(np.uint64(0xFF) << sh)) | (np.asarray(byte, np.uint64) << sh)


def keys_in_digits(rng, n, digits, width, hi=256):
    """keys that vary in exactly the given 8-bit digits (random bytes below `hi`); the others hold 0xA5"""
    k = np.full(n, 0xA5A5A5A5A5A5A5A5 & ((1 << (8 * np.dtype(WIDTH[width]).itemsize)) - 1), np.uint64)
    for d in digits:
        b = rng.integers(0, hi, n, dtype=np.uint64)
        b[:2] = (0, hi - 1)
        k = set_digit(k, d, b)
    return k.astype(WIDTH[width])


def check_arg_sort(plb, keys, what, passes=None):
    """one non-null UInt32 / UInt64 key column: one k_sort_encode, then one radix pass per varying digit"""
    got, prof = profiled(plb, lambda: plb.arg_sort([keys]))
    assert np.array_equal(got, np.argsort(keys, kind="stable")), what
    want = sc.radix_passes(keys)
    assert passes is None or passes == want, (what, passes, want)
    assert prof.get("sort_encode", 0) == 1 and prof.get("sort_scatter", 0) == want and prof.get("sort_hist", 0) == want, (what, prof)


PASS_DIGITS = {"u32": [(0,), (3,), (1, 2), (0, 3), (0, 1, 3), (0, 2, 3), (0, 1, 2, 3)],
               "u64": [(7,), (0,), (0, 7), (2, 5), (0, 3, 7), (1, 4, 6), (1, 2, 5, 6), (0, 2, 4, 6, 7), (0, 1, 2, 3, 4, 5),
                       (1, 2, 3, 4, 5, 6, 7), (0, 1, 2, 3, 4, 5, 7), tuple(range(8))]}


@pytest.mark.parametrize("width", list(WIDTH))
def test_every_pass_count(plb, sm, width):
    """1-4 (u32) and 1-8 (u64) passes, odd and even, with skipped middle digits; few values per digit, so every pass
    moves long runs of equal digits and stability decides the order"""
    rng = np.random.default_rng(1 if width == "u32" else 2)
    n = sm * RS_TILE + 4097
    for digits in PASS_DIGITS[width]:
        check_arg_sort(plb, keys_in_digits(rng, n, digits, width, hi=4 if len(digits) > 2 else 256), (width, digits), passes=len(digits))


@pytest.mark.parametrize("p", range(1, 9))
@pytest.mark.parametrize("width", list(WIDTH))
def test_chunking_for_every_occupancy(plb, sm, width, p):
    """C0 = min(SM*p, 1024) first-guess CTAs: C0 + 1 tiles (the last of one row) make chunks of two tiles and drop the
    empty trailing CTAs; 2*C0 tiles less 1000 rows give C0 CTAs of two tiles, the last ragged"""
    rng = np.random.default_rng(10 * p + len(width))
    c0 = min(sm * p, RS_MAX_CTAS)
    for n in (c0 * RS_TILE + 1, 2 * c0 * RS_TILE - 1000):
        digits = (0, 1, 2) if width == "u32" else (0, 4, 7)         # three passes: the result ends in the spare buffer
        k = keys_in_digits(rng, n, digits, width)
        k[: n // 2] = k[rng.integers(0, 1000, n // 2)]              # duplicates across every chunk
        check_arg_sort(plb, k, (width, p, n), passes=3)


def digit_cases(n, width, rng):
    """key columns over n rows, each built to put one distribution of the low digit in front of k_rs_scatter"""
    i = np.arange(n, dtype=np.uint64)
    top = 3 if width == "u32" else 7
    base = np.full(n, 0x5A5A5A5A5A5A5A5A & ((1 << (8 * (top + 1))) - 1), np.uint64)
    cases = {}
    # a whole 4096-row tile in one digit (every lane of every round in one match class); a second digit breaks no ties
    cases["tile_in_one_digit"] = set_digit(set_digit(base, 0, ((i // RS_TILE) * 37 + 11) % 256), 1, rng.integers(0, 4, n, dtype=np.uint64))
    # every digit twice in every warp's 512 rows, ties in the top digit
    cases["every_digit_in_every_warp"] = set_digit(set_digit(base, 0, (i * 73) % 256), top, rng.integers(0, 2, n, dtype=np.uint64) * 0x80)
    # one digit for all rows but one, the odd row in the middle and at the end
    for at in ("middle", "last"):
        b = np.full(n, 0x11, np.uint64)
        b[n // 2 if at == "middle" else n - 1] = 0x10
        cases[f"one_digit_but_one_{at}"] = set_digit(base, 0, b)
    # descending runs of 5000 rows (across tiles) and of 3 tiles + 17 rows (across CTA chunks)
    cases["runs_across_tiles_and_ctas"] = set_digit(set_digit(base, 0, 255 - (i // 5000) % 256), 1, 255 - (i // (3 * RS_TILE + 17)) % 256)
    # only the top (sign) digit varies
    cases["top_digit_only"] = set_digit(base, top, rng.integers(0, 2, n, dtype=np.uint64) * 0x80)
    return {k: v.astype(WIDTH[width]) for k, v in cases.items()}


@pytest.mark.parametrize("size", ["4095", "4096", "4097", "ragged_multi_cta"])
@pytest.mark.parametrize("width", list(WIDTH))
def test_digit_distributions(plb, sm, width, size):
    n = 3 * sm * RS_TILE + 37 if size == "ragged_multi_cta" else int(size)        # 37 rows: a last tile of two warps' lanes
    rng = np.random.default_rng(n)
    for name, k in digit_cases(n, width, rng).items():
        check_arg_sort(plb, k, (width, n, name), passes=1 if name == "top_digit_only" or name.startswith("one_digit") else None)


@pytest.mark.parametrize("groups", ["few", "many"])
@pytest.mark.parametrize("n", [2, 255, 256, 65_535, 65_536, (1 << 24) - 1, 1 << 24])
def test_group_tuples_pass_counts(plb, n, groups):
    """GroupsIdx sorts the row -> first-row ids with sort_pairs_u32 on bits_for(n) bits: 1, 2, 3 and 4 passes, the odd
    counts copying the result back"""
    rng = np.random.default_rng(n + len(groups))
    k = 3 if groups == "few" else n // 2 + 1
    ids = rng.integers(0, k, n, dtype=np.uint64)
    keys = (ids * np.uint64(0x9E3779B97F4A7C15)).view(np.int64)        # spread over the whole Int64 range
    (first, offsets, all_), prof = profiled(plb, lambda: plb.group_tuples(keys))
    ef, eo, ea = sc.groups_idx(keys)
    assert np.array_equal(first, ef) and np.array_equal(offsets, eo) and np.array_equal(all_, ea), (n, groups)
    assert prof.get("sort_scatter", 0) == (bits_for(n) + 7) // 8, (n, prof)


# =========================================================================================== 2. bl_arg_sort / bl_sort
def one_key(c, v):
    return [(c, v) if v is not None else c]


@pytest.mark.parametrize("dt", sc.KEY_DTYPES)
def test_full_range_bit_patterns(plb, dt):
    """every value of Int8 / UInt8 / Bool, Int64 MIN / MAX, UInt64 >= 2^63, sign-set NaN, quiet and signalling NaN
    payloads, ±0.0, ±inf, subnormals and ±max finite, against the plain oracle"""
    rng = np.random.default_rng(sc.KEY_DTYPES.index(dt) + 100)
    n = 3001
    c = sc.full_range_column(rng, dt, n)
    valid = rng.random(n) > 0.15
    for v in (None, valid):
        for desc in (False, True):
            for nl in (False, True):
                got = plb.arg_sort(one_key(c, v), desc, nl)
                assert np.array_equal(got, sort_oracle.arg_sort([c], [v], desc, nl)), (dt, v is not None, desc, nl)


@pytest.mark.parametrize("dt", sc.KEY_DTYPES)
def test_nullable_full_range_past_the_encode_grid(plb, sm, dt):
    rng = np.random.default_rng(sc.KEY_DTYPES.index(dt) + 200)
    n = n_enc(sm)
    c = sc.full_range_column(rng, dt, n)
    valid = rng.random(n) > 0.15
    for desc in (False, True):
        for nl in (False, True):
            got, prof = profiled(plb, lambda: plb.arg_sort([(c, valid)], desc, nl))
            assert np.array_equal(got, sort_oracle.numpy_arg_sort([c], [valid], desc, nl)), (dt, desc, nl)
            assert prof.get("sort_encode", 0) == 1 and prof.get("sort_encode_nulls", 0) == 1, prof


def test_constant_values_varying_nulls_and_all_null(plb, sm):
    """valid rows all equal (NaNs of every sign and payload are one value): the value stage is skipped and the null
    stage alone sorts; an all-null column takes no pass at all"""
    rng = np.random.default_rng(3)
    n = n_enc(sm)
    valid = rng.random(n) > 0.3
    cols = {"int64": np.full(n, 42, np.int64),
            "nan_payloads": rng.choice(sc.f64_bits(0x7FF8000000000000, 0xFFF8000000000000, 0x7FF8000000000001, 0xFFFFFFFFFFFFFFFF), n),
            "zeros": rng.choice(np.array([0.0, -0.0], np.float32), n)}
    for name, c in cols.items():
        for desc in (False, True):
            for nl in (False, True):
                got, prof = profiled(plb, lambda: plb.arg_sort([(c, valid)], desc, nl))
                assert np.array_equal(got, sort_oracle.numpy_arg_sort([c], [valid], desc, nl)), (name, desc, nl)
                assert prof.get("sort_scatter", 0) == 1, (name, prof)
    for desc in (False, True):
        got, prof = profiled(plb, lambda: plb.arg_sort([(cols["int64"], np.zeros(n, bool))], desc, True))
        assert np.array_equal(got, np.arange(n)) and prof.get("sort_scatter", 0) == 0, prof


def tie_columns(rng, n, k):
    """k key columns where each one leaves ties for the next: Int8 {-128, 0, 127}, special Float64, Bool, all nullable,
    then UInt64 over its full range"""
    cols = [rng.choice(np.array([-128, 0, 127], np.int8), n), rng.choice(sc.F64_SPECIAL, n), rng.random(n) < 0.5,
            sc.full_range_column(rng, "uint64", n)][:k]
    valids = [rng.random(n) > 0.1, rng.random(n) > 0.1, rng.random(n) > 0.3, None][:k]
    return cols, valids


@pytest.mark.parametrize("k", [3, 4])
def test_several_key_columns_past_the_encode_grid(plb, sm, k):
    rng = np.random.default_rng(k)
    n = n_enc(sm)
    cols, valids = tie_columns(rng, n, k)
    by = [(c, v) if v is not None else c for c, v in zip(cols, valids)]
    for trial in range(4):
        desc = [bool(x) for x in rng.random(k) < 0.5]
        nl = [bool(x) for x in rng.random(k) < 0.5]
        got = plb.arg_sort(by, desc, nl)
        assert np.array_equal(got, sort_oracle.numpy_arg_sort(cols, valids, desc, nl)), (k, desc, nl)


def test_limit_and_payloads_past_the_encode_grid(plb, sm):
    rng = np.random.default_rng(4)
    n = n_enc(sm)
    cols, valids = tie_columns(rng, n, 4)
    by = [(c, v) if v is not None else c for c, v in zip(cols, valids)]
    desc, nl = [True, False, False, True], [False, True, True, False]
    full = sort_oracle.numpy_arg_sort(cols, valids, desc, nl)
    p1, p1v = sc.full_range_column(rng, "float64", n), rng.random(n) > 0.2
    p2 = sc.full_range_column(rng, "int32", n)
    p3 = cols[3]
    for limit in (0, 1, n // 3, n - 1, n, n + 7):
        assert np.array_equal(plb.arg_sort(by, desc, nl, limit), full[:limit]), limit
        (g1, m1), (g2, m2), (g3, m3) = plb.sort(by, [(p1, p1v), p2, p3], desc, nl, limit)
        perm = full[:limit]
        assert np.array_equal(m1 if m1 is not None else np.ones(perm.size, bool), p1v[perm]), limit
        assert np.array_equal(g1.view(np.uint64)[p1v[perm]], p1.view(np.uint64)[perm][p1v[perm]]), limit     # bit patterns
        assert np.array_equal(g2, p2[perm]) and m2 is None and np.array_equal(g3, p3[perm]) and m3 is None, limit


# =========================================================================================== 3. string rank / arg_sort_keys
def random_strings(rng, m, lo, hi):
    """m distinct random byte strings of lo..hi (<= 7) bytes, any byte value"""
    cnt = int(m * 1.5) + 1000
    data = rng.integers(0, 256, (cnt, 7), dtype=np.uint8)
    lens = rng.integers(lo, hi + 1, cnt)
    data[np.arange(7)[None, :] >= lens[:, None]] = 0
    key = lens.astype(np.uint64)
    for j in range(7):
        key |= data[:, j].astype(np.uint64) << np.uint64(56 - 8 * j)
    _, first = np.unique(key, return_index=True)
    sel = rng.permutation(first)[:m]
    assert sel.size == m
    return [data[i, :lens[i]].tobytes() for i in sel]


def check_string_rank(plb, vals, both_flags=True):
    """string_rank and arg_sort of one string column against the dense rank from sorted(); -> the profile of the
    ascending string_rank"""
    s = plb.StringColumn(vals)
    r, v = sc.dense_rank_bytes(vals)
    m = int(r.max(initial=0))
    ((gr, gv), nd), prof = profiled(plb, lambda: plb.string_rank(s))
    gv = np.ones(len(vals), bool) if gv is None else gv
    assert nd == m and np.array_equal(gv, v) and np.array_equal(gr[v], r[v])
    (gr, _), _ = plb.string_rank(s, True)
    assert np.array_equal(gr[v], (m + 1 - r)[v])
    for desc, nl in ((False, False), (True, True), (False, True), (True, False))[: 4 if both_flags else 2]:
        assert np.array_equal(plb.arg_sort([s], desc, nl), sort_oracle.numpy_arg_sort([r], [v], desc, nl)), (desc, nl)
    return prof


def test_string_rank_past_the_tile_grid(plb, sm):
    """8*SM*4096 + 4097 distinct strings of 1-7 bytes: one round over every entry, heads / apply loop over their tiles"""
    rng = np.random.default_rng(5)
    m = 8 * sm * SR_TILE + 4097
    distinct = random_strings(rng, m, 1, 7)
    idx = np.concatenate([np.arange(m), rng.integers(0, m, 40_000), np.full(3000, -1)])
    vals = [None if i < 0 else distinct[i] for i in rng.permutation(idx)]
    prof = check_string_rank(plb, vals, both_flags=False)
    assert prof.get("str_rank_key", 0) == 1 and prof.get("str_rank_heads", 0) == 1 and prof.get("str_rank_bucket_keys", 0) == 0, prof


def test_bucket_stage_with_three_digits(plb):
    """70 001 shared 7-byte prefixes with 2-3 suffixes each: round 1 sorts more than 65 536 active buckets by id"""
    rng = np.random.default_rng(6)
    prefixes = random_strings(rng, 70_001, 7, 7)
    vals = []
    for p in prefixes:
        want = int(rng.integers(2, 4))
        tails = set()
        while len(tails) < want:
            tails.add(bytes(rng.integers(0, 256, int(rng.integers(1, 8)), dtype=np.uint8)))
        vals += [p + t for t in tails]
    assert len(prefixes) > 65_536                       # every prefix is an active bucket of round 1
    vals += [None] * 500 + [vals[i] for i in rng.integers(0, len(vals), 5000)]
    vals = [vals[i] for i in rng.permutation(len(vals))]
    assert sc.refinement_rounds(vals) == (2, 0)
    prof = check_string_rank(plb, vals)
    assert prof.get("str_rank_key", 0) == 2 and prof.get("str_rank_bucket_keys", 0) == 1, prof


@pytest.mark.parametrize("plen", [6, 7, 8, 13, 14, 15])
def test_shared_prefix_rounds(plb, plen):
    """every value shares a prefix of 7k - 1, 7k or 7k + 1 bytes: rounds whose chunk every active value shares sort
    nothing (vary == 0), the next one splits"""
    rng = np.random.default_rng(plen)
    p = bytes(rng.integers(0, 256, plen, dtype=np.uint8))
    tails = sorted({bytes(rng.integers(0, 256, int(rng.integers(0, 7)), dtype=np.uint8)) for _ in range(3000)} | {b"", b"\0", b"\0\0", b"\xff"})
    vals = [p + t for t in tails] + [None] * 50
    vals = [vals[i] for i in rng.permutation(len(vals))]
    rounds, skipped = sc.refinement_rounds(vals)
    assert skipped == max(plen // 7 - (plen % 7 == 0), 0), (rounds, skipped)
    prof = check_string_rank(plb, vals)
    assert prof.get("str_rank_key", 0) == rounds and prof.get("str_rank_key", 0) - prof.get("str_rank_heads", 0) == skipped, prof


EDGE = [b"", b"a", b"a\0", b"a\0\0", b"\0", b"\0\0", b"\0" * 7, b"\0" * 8, b"\xff", b"\xff\xff", b"\xff" * 7, b"\xff" * 8,
        b"a\xff", b"a" * 6 + b"\0", b"a" * 7, b"a" * 7 + b"\0", b"a" * 7 + b"\0\0", b"\x7f", b"\x80", b"ab", b"b", None]


def test_byte_edge_cases_past_the_encode_grid(plb, sm):
    rng = np.random.default_rng(7)
    n = n_enc(sm)
    check_string_rank(plb, [EDGE[i] for i in rng.integers(0, len(EDGE), n)])


@pytest.mark.parametrize("pool", [[b"same"], [b"same", None], [b"", None]])
def test_one_distinct_value(plb, sm, pool):
    rng = np.random.default_rng(len(pool))
    vals = [pool[i] for i in rng.integers(0, len(pool), n_enc(sm))]
    prof = check_string_rank(plb, vals)
    assert prof.get("str_rank_key", 0) == 0, prof


# =========================================================================================== 4. median / quantile
def spec(kind):
    return (0.5, "linear") if kind == "median" else (float(kind.split(":")[1]), kind.split(":")[2])


def quantile_run(plb, monkeypatch, keys, vals, valid, kinds, glob):
    if glob:
        monkeypatch.setenv("BL_QUANTILE_GLOBAL", "1")
    else:
        monkeypatch.delenv("BL_QUANTILE_GLOBAL", raising=False)
    return profiled(plb, lambda: dev_group_quantiles(keys, vals, valid, kinds))


def check_quantiles(plb, monkeypatch, keys, vals, valid, kinds, exact_python=False):
    """both plans, byte for byte, and the reference (keys are first-occurrence group ids) -> (small-plan profile,
    large-plan profile)"""
    small, ps = quantile_run(plb, monkeypatch, keys, vals, valid, kinds, False)
    glob, pg = quantile_run(plb, monkeypatch, keys, vals, valid, kinds, True)
    monkeypatch.delenv("BL_QUANTILE_GLOBAL", raising=False)
    for kind, (a, av), (b, bv) in zip(kinds, small, glob):
        assert np.array_equal(av, bv) and a.tobytes() == b.tobytes(), f"plans differ: {kind}"
    G = int(keys.max()) + 1
    for kind, (got, gv) in zip(kinds, small):
        q, m = spec(kind)
        exp, ev = qo.group_quantile(keys.tolist(), vals, valid, q, m) if exact_python else qo.numpy_group_quantile(keys, vals, valid, q, m, G)
        assert_same(got, gv, exp, ev, kind)
    return ps, pg


KINDS = ["median", kind_of(0.0, "nearest"), kind_of(0.1, "lower"), kind_of(0.9, "higher"), kind_of(0.5, "midpoint"),
         kind_of(0.3, "linear"), kind_of(0.25, "equiprobable"), kind_of(1.0, "linear")]


@pytest.mark.parametrize("dt", ["float64", "int64", "float32"])
def test_small_plan_window_shapes(plb, monkeypatch, dt):
    rng = np.random.default_rng(8)
    sizes, shapes = sc.window_layout(rng)
    w = sc.small_windows(sizes)
    for name, (b, want) in shapes.items():
        assert w[b] == want, (name, w[b], want)
    keys = sc.keys_with_group_sizes(rng, sizes)
    n = keys.size
    if dt == "int64":
        vals = np.where(rng.random(n) < 0.3, rng.choice(sc.int_pool(np.int64), n), rng.integers(-50, 50, n))
    else:
        vals = np.where(rng.random(n) < 0.1, rng.choice(sc.F64_SPECIAL, n), rng.normal(size=n)).astype(dt)
    valid = rng.random(n) > 0.1
    ps, _ = check_quantiles(plb, monkeypatch, keys, vals, valid, KINDS, exact_python=True)
    assert ps.get("quantile_small", 0) == 1 and ps.get("quantile_encode_large", 0) == 1, ps


@pytest.mark.parametrize("k", [17, 33])
def test_more_than_16_quantiles_of_one_column(plb, monkeypatch, k):
    rng = np.random.default_rng(k)
    sizes = [int(s) for s in rng.integers(1, 100, 400)] + [3000, 5000, H + 1]
    sizes = [sizes[i] for i in rng.permutation(len(sizes))]
    keys = sc.keys_with_group_sizes(rng, sizes)
    vals = rng.normal(size=keys.size)
    vals[rng.random(keys.size) < 0.05] = np.nan
    valid = rng.random(keys.size) > 0.1
    kinds = [kind_of(i / (k - 1), qo.METHODS[i % len(qo.METHODS)]) for i in range(k)]
    ps, pg = check_quantiles(plb, monkeypatch, keys, vals, valid, kinds)
    sorts = math.ceil(k / 16)
    assert ps.get("quantile_small", 0) == sorts and ps.get("quantile_encode_large", 0) == sorts and ps.get("quantile_pick_large", 0) == sorts, ps
    assert pg.get("quantile_small", 0) == 0 and pg.get("quantile_encode_large", 0) == sorts and pg.get("quantile_pick_large", 0) == sorts, pg


@pytest.mark.parametrize("nl", [1, 2, 257])
def test_large_plan_segment_stage(plb, monkeypatch, nl):
    """NL large groups between small ones: no segment stage at NL = 1, one digit at 2, two at 257 (segment 256 shares
    its low digit with segment 0); the second large group is all null"""
    rng = np.random.default_rng(nl)
    sizes = [int(s) for s in rng.integers(H + 1, H + 60, nl)] + [int(s) for s in rng.integers(1, 40, 300)]
    sizes = [sizes[i] for i in rng.permutation(len(sizes))]
    keys = sc.keys_with_group_sizes(rng, sizes)
    n = keys.size
    vals = np.where(rng.random(n) < 0.05, rng.choice(sc.F64_SPECIAL, n), rng.normal(size=n))
    valid = rng.random(n) > 0.1
    large = [g for g, s in enumerate(sizes) if s > H]
    if nl > 1:
        valid[keys == large[1]] = False
    ps, pg = check_quantiles(plb, monkeypatch, keys, vals, valid, KINDS)
    assert ps.get("quantile_encode_large", 0) == 1 and ps.get("quantile_segment_keys", 0) == (1 if nl > 1 else 0), ps
    assert pg.get("quantile_segment_keys", 0) == 1, pg


@pytest.mark.parametrize("groups", ["65537", "past_find_grid"])
def test_many_large_segments_and_pick_grid(plb, sm, monkeypatch, groups):
    """with BL_QUANTILE_GLOBAL=1 every group is large: 65 537 segments (three digits) and 8*SM*256 + 1001 groups (past
    k_quantile_find_large's grid); 16 quantiles put NL * picks past k_quantile_pick_large's grid"""
    rng = np.random.default_rng(len(groups))
    G = 65_537 if groups == "65537" else 8 * sm * 256 + 1001
    keys = sc.keys_with_group_sizes(rng, rng.integers(1, 5, G))
    vals = rng.integers(-(1 << 40), 1 << 40, keys.size)
    valid = rng.random(keys.size) > 0.1
    kinds = [kind_of(i / 15, qo.METHODS[i % len(qo.METHODS)]) for i in range(16)]
    assert G * len(kinds) > 8 * sm * 256
    _, pg = check_quantiles(plb, monkeypatch, keys, vals, valid, kinds)
    assert pg.get("quantile_segment_keys", 0) == 1 and pg.get("quantile_pick_large", 0) == 1, pg


@pytest.mark.parametrize("case", ["all_equal", "all_null"])
def test_large_group_without_key_pass(plb, monkeypatch, case):
    """the only large group holds one value (or only nulls): its keys do not vary, so the large plan sorts nothing"""
    rng = np.random.default_rng(9)
    sizes = [3 * H + 7] + [int(s) for s in rng.integers(1, 30, 400)]
    keys = sc.keys_with_group_sizes(rng, sizes)
    n = keys.size
    vals = rng.normal(size=n)
    valid = rng.random(n) > 0.1
    if case == "all_equal":
        vals[keys == 0] = 2.5
        valid[keys == 0] = True
    else:
        valid[keys == 0] = False
    _, pt = profiled(plb, lambda: plb.group_tuples(keys))
    small, ps = quantile_run(plb, monkeypatch, keys, vals, valid, KINDS, False)
    assert ps.get("sort_scatter", 0) == pt.get("sort_scatter", 0) and ps.get("quantile_segment_keys", 0) == 0, (ps, pt)
    check_quantiles(plb, monkeypatch, keys, vals, valid, KINDS, exact_python=True)


def test_large_groups_past_the_radix_grid(plb, monkeypatch):
    rng = np.random.default_rng(10)
    sizes = [2_200_003, 7, 2_100_001] + [int(s) for s in rng.integers(1, 50, 500)]
    assert sizes[0] + sizes[2] > RS_MAX_CTAS * RS_TILE
    keys = sc.keys_with_group_sizes(rng, sizes)
    n = keys.size
    vals = np.where(rng.random(n) < 0.02, rng.choice(sc.F64_SPECIAL, n), rng.normal(size=n))
    valid = rng.random(n) > 0.05
    check_quantiles(plb, monkeypatch, keys, vals, valid, ["median", kind_of(0.1, "nearest"), kind_of(0.9, "linear"), kind_of(0.5, "midpoint")])


VALUE_CASES = {
    "int64_extremes": lambda rng, n: rng.choice(sc.int_pool(np.int64), n),
    "uint64_extremes": lambda rng, n: rng.choice(sc.int_pool(np.uint64), n),
    "float64_special": lambda rng, n: rng.choice(sc.F64_SPECIAL, n),
    "float32_special": lambda rng, n: rng.choice(sc.F32_SPECIAL, n),
}


@pytest.mark.parametrize("case", sorted(VALUE_CASES))
def test_quantile_values(plb, monkeypatch, case):
    """values whose f64 conversion rounds, sign-set NaN and NaN payloads, ±0.0, ±inf under linear and midpoint
    interpolation (inf - inf), subnormals; small and large groups, every method, 30 quantiles (two sorts)"""
    rng = np.random.default_rng(len(case) + 11)
    sizes = [2, 2, 3, 2] + [int(s) for s in rng.integers(1, 40, 200)] + [H + 5, 3 * H]
    keys = sc.keys_with_group_sizes(rng, sizes)
    n = keys.size
    vals = VALUE_CASES[case](rng, n)
    valid = rng.random(n) > 0.1
    valid[keys < 4] = True
    if vals.dtype.kind == "f":
        for g, v in enumerate(([-np.inf, np.inf], [np.inf, np.inf], [-0.0, 0.0, -0.0], [sc.F64_SPECIAL[11], -np.inf])):
            vals[keys == g] = np.array(v).astype(vals.dtype)
    kinds = [kind_of(q, m) for m in qo.METHODS for q in (0.0, 0.1, 0.5, 0.75, 1.0)]
    check_quantiles(plb, monkeypatch, keys, vals, valid, kinds, exact_python=True)
