"""GPU tests of the packed records of the partitioned group_by (K5r, groupby_radix.cu), against the exact restatement in
tests/groupby_ref.py.

When the 65,536-row sample (k_gb_estimate: rows (i * n) // m) puts the keys in a range at most 2^31 wide and one value
column in 32 bits (Int32 / UInt32 / Float32 by dtype; Int64 within +-2^30, UInt64 below 2^31 by the sampled range),
the record word 0 carries the key's offset from a base (low half) and that value (high half).  The window holds the
offsets 0 .. 2^32 - 2 centred on the sampled range (offset 2^32 - 1 marks the pad records); a row outside it, or a value
that does not widen back to itself, raises status 4 and the batch is redone once with plain records.  Every attempt
prints a [k5r] line with packed=0/1; the plan on it (buckets, slots, store) is the one of the plain record width.
"""
import numpy as np
import pytest

import groupby_ref as ref
import radix_ref as rr
from test_gpu_groupby_plans import Call, n_loop
from test_gpu_groupby_radix import STORES, check_line, groups_for
from test_gpu_groupby_radix_sizing import SAMPLE_ROWS, attempts

pytestmark = pytest.mark.gpu

FORCE = {"BL_K5_RADIX": "2", "BL_K5_HOTKEYS": "0"}


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as m
    m.init()
    return m


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


@pytest.fixture(scope="module")
def optin(plb):
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def sampled_rows(n):
    return (np.arange(SAMPLE_ROWS, dtype=np.int64) * n) // SAMPLE_ROWS


def unsampled(n):
    return np.setdiff1d(np.arange(n), sampled_rows(n))


def small_ints(rng, n, lo=-1000, hi=1000):
    return rng.integers(lo, hi, n, dtype=np.int64)


def c2_aggs(rng, n, vi=None):
    vi = small_ints(rng, n) if vi is None else vi
    vf = ref.sum_column(rng, "float64", n, exact=True)
    return [("sum", (vi, None)), ("mean", (vf, None)), ("len", None)]


def run(plb, monkeypatch, capfd, keys, aggs, store=None, force=True):
    knobs = dict(FORCE) if force else {}
    if store is not None:
        knobs["BL_K5R_STORE"] = str(STORES[store])
    return attempts(plb, monkeypatch, capfd, keys, aggs, knobs)


def forms(lines):
    return [(int(ln["packed"]), ln["sizing"], int(ln["status"])) for ln in lines]


def one_plain_redo(lines):
    """A packed attempt that met an unfit row (status 4), then one plain attempt with the same sizing."""
    sizing = lines[0]["sizing"]
    assert forms(lines) == [(1, sizing, 4), (0, sizing, 0)], lines


def packed_once(c, lines, aggs, optin, store=None, what=""):
    """One attempt, packed, status 0, the plain-width plan; exact results."""
    assert len(lines) == 1 and int(lines[0]["packed"]) == 1, lines
    check_line(lines[0], aggs, optin, store)
    c.check(None, what)


# ------------------------------------------------------------------ C2 and key bases
def test_c2_packs(plb, monkeypatch, capfd, optin):
    """C2-shaped (1e6 uniform keys in [0, 1e6), sum(Int64 in [-1000, 1000)), mean(Float64), len), no knobs."""
    rng = np.random.default_rng(1)
    n = 6_000_001
    keys = rng.integers(0, 1_000_000, n, dtype=np.int64)
    aggs = c2_aggs(rng, n)
    c, prof, lines = run(plb, monkeypatch, capfd, keys, aggs, force=False)
    assert "k5r_aggregate" in prof and lines and lines[0]["sizing"] == "sample", (sorted(prof), lines)
    packed_once(c, lines, aggs, optin, what="C2 packed")


@pytest.mark.parametrize("where", ["negative", "near_2_40", "uint64_top"])
def test_key_bases(plb, sm, monkeypatch, capfd, optin, where):
    """Keys whose window does not start at 0: all negative, around 2^40, and UInt64 keys just below 2^64."""
    rng = np.random.default_rng(len(where))
    n = n_loop(sm)
    off = rng.integers(0, 1 << 30, 300_000, dtype=np.int64)
    if where == "negative":
        distinct, dt = -(1 << 33) - off, np.int64
    elif where == "near_2_40":
        distinct, dt = (1 << 40) - (1 << 29) + off, np.int64
    else:
        distinct, dt = (np.uint64((1 << 64) - 1) - off.astype(np.uint64)), np.uint64
    keys = distinct[rng.integers(0, distinct.size, n)].astype(dt)
    aggs = c2_aggs(rng, n)
    c, _, lines = run(plb, monkeypatch, capfd, keys, aggs)
    packed_once(c, lines, aggs, optin, what=where)


# ------------------------------------------------------------------ the window's edges
def edge_keys(rng, n, past):
    """The sampled keys span [L, L + 2^31] exactly, so base = L - (2^30 - 1) and the window is [base, base + 2^32 - 2].
    Unsampled rows add the keys at offsets 0 and 2^32 - 2 (past: offsets 2^32 - 1 and -1, outside it); 2000 keys."""
    L = -(1 << 35)
    base = L - ((1 << 30) - 1)
    pool = L + np.concatenate([[0, 1 << 31], rng.integers(1, 1 << 31, 2000)])
    keys = pool[rng.integers(0, pool.size, n)]
    s = sampled_rows(n)
    keys[s[0]], keys[s[1]] = L, L + (1 << 31)
    extra = [base + 0xFFFFFFFF, base - 1] if past else [base, base + 0xFFFFFFFE]
    rest = unsampled(n)
    at = rng.choice(rest, 4000, replace=False)
    keys[at] = np.repeat(extra, 2000)
    return keys


@pytest.mark.parametrize("store", list(STORES))
@pytest.mark.parametrize("past", [False, True])
def test_window_edges(plb, monkeypatch, capfd, optin, store, past):
    """Offsets 0 and 2^32 - 2 pack next to the pad records of every store path (64 buckets); offsets 2^32 - 1 (the pad
    marker) and -1 do not, and the batch is redone once with plain records."""
    rng = np.random.default_rng(11 + past + STORES[store])
    n = rr.MIN_ROWS + 2049
    keys = edge_keys(rng, n, past)
    aggs = c2_aggs(rng, n)
    c, _, lines = run(plb, monkeypatch, capfd, keys, aggs, store)
    if past:
        one_plain_redo(lines)
        check_line(lines[1], aggs, optin, store)
        c.check(None, f"past edge {store}")
    else:
        packed_once(c, lines, aggs, optin, store, f"edges {store}")


# ------------------------------------------------------------------ value widths
@pytest.mark.parametrize("dtype,extremes,packs", [
    ("int64", [(1 << 31) - 1, -(1 << 31)], True),
    ("int64", [1 << 31], False),
    ("int64", [-(1 << 31) - 1], False),
    ("uint64", [(1 << 32) - 1], True),
    ("uint64", [1 << 32], False),
])
def test_int64_boundaries(plb, sm, monkeypatch, capfd, optin, dtype, extremes, packs):
    """The sample sees values within +-1000; unsampled rows carry values at the 32-bit boundaries.  Int64 widens by sign
    extension (2^31 - 1 and -2^31 fit, 2^31 and -2^31 - 1 do not), UInt64 by zero extension (2^32 - 1 fits, 2^32 does
    not)."""
    rng = np.random.default_rng(len(extremes) + 7 * packs)
    n = n_loop(sm)
    keys = rng.integers(0, 400_000, n, dtype=np.int64)
    vals = small_ints(rng, n, 0 if dtype == "uint64" else -1000, 1000)
    at = rng.choice(unsampled(n), 500 * len(extremes), replace=False)
    vals[at] = np.repeat(np.array([e % (1 << 64) for e in extremes], dtype=np.uint64).view(np.int64), 500)
    vals = vals.view(np.uint64) if dtype == "uint64" else vals
    aggs = [("sum", (vals, None)), ("max", (vals, None)), ("min", (vals, None)), ("len", None)]
    c, _, lines = run(plb, monkeypatch, capfd, keys, aggs)
    if packs:
        packed_once(c, lines, aggs, optin, what=f"{dtype} {extremes}")
    else:
        one_plain_redo(lines)
        check_line(lines[1], aggs, optin)
        c.check(None, f"{dtype} {extremes}")


@pytest.mark.parametrize("dtype", ["int32", "uint32", "float32"])
def test_four_byte_columns(plb, sm, monkeypatch, capfd, optin, dtype):
    """4-byte value columns pack by dtype: full-range values (Int32 negatives, UInt32 >= 2^31, Float32 NaN / inf / -0.0
    under min / max) beside a full-range Int64 column that keeps its own word."""
    rng = np.random.default_rng(len(dtype))
    n = n_loop(sm)
    case = ref.Case(rng, "int64", groups=300_000, rest=n - sum(ref.SPECIAL_ROWS.values()))
    keys = np.unique(case.keys, return_inverse=True)[1].astype(np.int64).reshape(-1)      # the case's groups, keys 0 .. G - 1
    s = case.values(rng, dtype, for_sum=True, exact=True)
    mm = case.values(rng, dtype) if dtype == "float32" else s
    wide = case.values(rng, "int64")
    aggs = [("sum", s), ("min", mm), ("max", mm), ("sum", wide), ("len", None)]
    c, _, lines = run(plb, monkeypatch, capfd, keys, aggs)
    packed_once(c, lines, aggs, optin, what=dtype)


# ------------------------------------------------------------------ store paths and bucket counts
@pytest.mark.parametrize("store", list(STORES))
@pytest.mark.parametrize("logB", [6, 10, 12])
def test_store_paths(plb, sm, monkeypatch, capfd, optin, logB, store):
    """Every store path at 64, 1024 and 4096 buckets, n_loop(sm) rows (ragged last tile), keys within 2^30 of 2^36."""
    rng = np.random.default_rng(100 + logB * 3 + STORES[store])
    n = n_loop(sm)
    D = groups_for(logB, 3, 2)
    distinct = (1 << 36) + rng.choice(1 << 30, D, replace=False).astype(np.int64)
    keys = distinct[rng.integers(0, D, n)]
    aggs = c2_aggs(rng, n)
    c, _, lines = run(plb, monkeypatch, capfd, keys, aggs, store)
    packed_once(c, lines, aggs, optin, store, f"{1 << logB} {store}")
    assert int(lines[0]["buckets"]) == 1 << logB, lines


@pytest.mark.parametrize("store", list(STORES))
def test_empty_key_rows(plb, sm, monkeypatch, capfd, optin, store):
    """3000 rows with the GB_EMPTY key (i64::MIN, outside any window) aggregate beside the packed records: no redo."""
    rng = np.random.default_rng(20 + STORES[store])
    n = n_loop(sm)
    keys = rng.integers(-200_000, 200_000, n, dtype=np.int64)
    keys[rng.choice(n, 3000, replace=False)] = np.iinfo(np.int64).min
    aggs = c2_aggs(rng, n)
    c, _, lines = run(plb, monkeypatch, capfd, keys, aggs, store)
    assert int(lines[0]["status"]) == 0, lines
    packed_once(c, lines, aggs, optin, store, f"empty key {store}")


# ------------------------------------------------------------------ bucket streams around one ring stage
def window_keys_in_bucket(rng, logB, bucket, count, avoid):
    """`count` distinct keys in [0, 2^30) whose hash lands in `bucket`, none in `avoid`."""
    out = np.zeros(0, np.int64)
    while out.size < count:
        c = rng.integers(0, 1 << 30, 1 << 22, dtype=np.int64)
        c = c[(rr.bucket_of(rr.table_hash_np(c.view(np.uint64)), logB) == np.uint64(bucket)) & ~np.isin(c, avoid)]
        out = np.unique(np.concatenate([out, c]))
    return rng.permutation(out)[:count]


@pytest.mark.parametrize("store", list(STORES))
def test_stream_edges(plb, monkeypatch, capfd, optin, store):
    """Buckets of 991 / 992 / 993 / 1985 rows (one ring stage of packed records holds 992), 64 buckets, keys in [0, 2^30)."""
    rng = np.random.default_rng(30 + STORES[store])
    n = rr.MIN_ROWS + 2049
    spec = {3: (991, 400), 4: (992, 300), 5: (993, 500), 6: (1985, 700), 7: (1, 1)}
    rest = n - sum(r for r, _ in spec.values())
    spec |= {b: (rest // 56 + (b == 8) * (rest % 56), 1200) for b in range(8, 64)}
    parts, seen = [], np.zeros(0, np.int64)
    for b, (rows, groups) in spec.items():
        k = window_keys_in_bucket(rng, 6, b, groups, seen)
        seen = np.concatenate([seen, k])
        parts.append(np.concatenate([k, k[rng.integers(0, groups, rows - groups)]]))
    keys = np.concatenate(parts)
    keys = keys[rng.permutation(keys.size)]
    assert keys.size == n
    aggs = [("sum", (small_ints(rng, n), None)), ("len", None)]
    c, _, lines = run(plb, monkeypatch, capfd, keys, aggs, store)
    counts = rr.bucket_counts(keys, 6)
    assert [counts[b] for b in (3, 4, 5, 6)] == [991, 992, 993, 1985]
    packed_once(c, lines, aggs, optin, store, f"streams {store}")


# ------------------------------------------------------------------ rows the sample does not see
@pytest.mark.parametrize("store", list(STORES))
@pytest.mark.parametrize("miss", ["key", "value", "key_and_overflow"])
def test_sample_blind(plb, monkeypatch, capfd, optin, miss, store):
    """Only unsampled rows carry a key outside the window or a value outside 32 bits: one redo with plain records,
    exact.  key_and_overflow: the unsampled rows also fill one bucket far past its sampled stream, so the one redo is
    plain and exactly sized."""
    rng = np.random.default_rng(40 + len(miss) + STORES[store])
    n = rr.MIN_ROWS + 4097
    keys = rng.integers(0, 20_000, n, dtype=np.int64)
    rest = unsampled(n)
    if miss == "key_and_overflow":
        heavy = window_keys_in_bucket(rng, 6, 5, 1000, np.zeros(0, np.int64))
        keys[rest] = heavy[rng.integers(0, heavy.size, rest.size)]
    vals = small_ints(rng, n)
    at = rng.choice(rest, 100, replace=False)
    if miss == "value":
        vals[at] = 1 << 40
    else:
        keys[at] = 1 << 45
    aggs = [("sum", (vals, None)), ("len", None)]
    c, prof, lines = run(plb, monkeypatch, capfd, keys, aggs, store)
    if miss == "key_and_overflow":
        assert forms(lines) == [(1, "sample", 6), (0, "exact", 0)], lines
        assert "k5r_histogram" in prof, sorted(prof)
    else:
        one_plain_redo(lines)
    check_line(lines[1], aggs, optin, store, buckets=64)
    c.check(None, f"sample-blind {miss} {store}")
