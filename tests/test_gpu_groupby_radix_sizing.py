"""GPU tests of how the partitioned group_by (K5r, groupby_radix.cu) sizes its bucket streams, against the exact
restatement in tests/groupby_ref.py.

consume_radix sizes every bucket's record stream from the sample (sizing=sample: n / B + 5 sqrt(F2 / B) rows plus the
store path's padding, F2 = the sampled sum over groups of their rows squared) when that margin is at most half the mean,
and otherwise counts the rows of every bucket first (sizing=exact, the k5r_histogram pass).  A bucket that outgrows its
sampled stream raises status 2 and the batch is redone once with exact sizing.  Every attempt prints one BL_K5_DEBUG
[k5r] line; these tests read all of them.
"""
import re

import numpy as np
import pytest

import groupby_ref as ref
import radix_ref as rr
from test_gpu_groupby_plans import BIG, Call, _env, n_loop, profiled, value_cols
from test_gpu_groupby_radix import STORES, check_line

SAMPLE_ROWS = 65536                 # k_gb_estimate: rows (i * n) // m of the batch


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


def attempts(plb, monkeypatch, capfd, keys, aggs, knobs):
    """One device-input group_by_agg; -> (Call, profile, fields of every [k5r] line in order)."""
    for k in ("BL_K5_RADIX", "BL_K5_HOTKEYS", "BL_K5R_STORE"):
        monkeypatch.delenv(k, raising=False)
    _env(monkeypatch, {"BL_K5_DEBUG": "1", **knobs})
    capfd.readouterr()
    c, prof = profiled(plb, lambda: Call(plb, keys, None, aggs, False, device=True))
    lines = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("[k5r]")]
    return c, prof, [dict(re.findall(r"(\w+)=(\S+)", ln)) for ln in lines]


def worst_padding(info, sm, roww, n):
    """Records a bucket stream reserves beyond its rows (k_gbr_offsets): F - 1 per write-combining CTA (two CTAs per SM
    while two chunk buffers per bucket fit the SM's 228 KB), one per 2048-row tile for the runs, none coalesced."""
    B = int(info["buckets"])
    if info["store"] == "wc":
        per_sm = 2 if 2 * (rr.wc_smem(B, roww) + 1024) <= 228 * 1024 else 1
        return (rr.WC_F - 1) * per_sm * sm
    if info["store"] == "runs":
        return -(-n // rr.SCATTER_ROWS)
    return 0


def c2_keys(rng, n):
    distinct = rng.permutation(np.unique(rng.integers(1, 1 << 50, 1_050_000))[:1_000_000])
    return distinct[rng.integers(0, distinct.size, n)]


@pytest.mark.gpu
@pytest.mark.parametrize("order", ["shuffled", "sorted"])
def test_c2_shape_sample_sizing(plb, sm, optin, monkeypatch, capfd, order):
    """C2-shaped call (1e6 uniform Int64 keys, sum(Int64), mean(Float64), len), no knobs: the sample sizes the streams,
    no histogram pass, no redo.  Sorted, the strided sample sees every group at most once (no sampled pairs); the floor
    F2 >= n^2 / est_groups keeps the margin."""
    rng = np.random.default_rng(2)
    n = 6_000_001
    keys = c2_keys(rng, n)
    if order == "sorted":
        keys = np.sort(keys)
    a = ref.sum_column(rng, "int64", n)
    b = ref.sum_column(rng, "float64", n, exact=True)
    aggs = [("sum", (a, None)), ("mean", (b, None)), ("len", None)]
    c, prof, lines = attempts(plb, monkeypatch, capfd, keys, aggs, {})
    assert len(lines) == 1 and lines[0]["sizing"] == "sample", lines
    assert "k5r_histogram" not in prof and "k5r_aggregate" in prof, sorted(prof)
    info = lines[0]
    logB, _ = check_line(info, aggs, optin)
    B, cap = 1 << logB, int(info["cap"])
    pad = worst_padding(info, sm, 3, n)
    real = rr.bucket_counts(keys, logB)
    assert cap >= real.max() + pad, (cap, real.max(), pad)
    assert B * cap <= 1.5 * n + B * (pad + rr.WC_F), (B, cap, n, pad)
    c.check(None, f"C2 {order}")


def sample_blind_keys(rng, n, logB, pool):
    """The strided sample rows carry keys drawn from `pool` keys spread over every bucket; every other row carries one of
    1000 keys of bucket 5, or (3000 rows) the GB_EMPTY key: the sample sees uniform buckets, bucket 5 takes ~all rows."""
    sampled = (np.arange(SAMPLE_ROWS, dtype=np.int64) * n) // SAMPLE_ROWS
    spread = rng.permutation(np.unique(rng.integers(1, 1 << 62, pool + pool // 8, dtype=np.int64))[:pool]).view(np.uint64)
    heavy = rr.keys64_in_bucket(rng, logB, 5, 1000, avoid=spread)
    rest = np.setdiff1d(np.arange(n), sampled)
    fill = heavy[rng.integers(0, heavy.size, rest.size)]
    fill[:3000] = np.uint64(rr.GB_EMPTY)
    bits = np.empty(n, np.uint64)
    bits[rest] = fill[rng.permutation(rest.size)]
    bits[sampled] = spread[rng.integers(0, pool, SAMPLE_ROWS)]
    return rr.as_dtype(bits, "int64")


@pytest.mark.gpu
@pytest.mark.parametrize("store", list(STORES))
@pytest.mark.parametrize("logB", [6, 10])
def test_sample_blind_overflow(plb, optin, monkeypatch, capfd, logB, store):
    """A bucket the sample cannot see overflows its sampled stream: status 2, then one exact attempt with status 0, and
    exact results (the GB_EMPTY-key group, aggregated again by the redo, counted once)."""
    rng = np.random.default_rng(90 + logB + STORES[store])
    n, pool = (rr.MIN_ROWS + 4097, 20_000) if logB == 6 else (4_000_001, 1_300_000)
    keys = sample_blind_keys(rng, n, logB, pool)
    assert rr.bucket_counts(keys, logB)[5] > n // 2
    vals = ref.sum_column(rng, "int64", n)
    aggs = [("sum", (vals, None)), ("len", None)]
    c, prof, lines = attempts(plb, monkeypatch, capfd, keys, aggs, {"BL_K5_RADIX": "2", "BL_K5_HOTKEYS": "0", "BL_K5R_STORE": str(STORES[store])})
    assert [(ln["sizing"], int(ln["status"])) for ln in lines] == [("sample", 2), ("exact", 0)], lines
    assert int(lines[1]["cap"]) == 0 and int(lines[0]["cap"]) > 0, lines
    check_line(lines[1], aggs, optin, store, buckets=1 << logB)
    assert "k5r_histogram" in prof and "k5r_aggregate" in prof, sorted(prof)
    c.check(None, f"sample-blind {1 << logB} {store}")


@pytest.mark.gpu
def test_visible_skew_exact_up_front(plb, sm, optin, monkeypatch, capfd):
    """An ordinary key on 2^20 rows (no heavy-hitter list): the sample sees it, so the streams are sized exactly up
    front, in one attempt."""
    rng = np.random.default_rng(47)
    n = n_loop(sm)
    case = ref.Case(rng, "int64", big=BIG, singletons=10_000, groups=500_000, rest=n - BIG - 10_000 - sum(ref.SPECIAL_ROWS.values()),
                    big_key=np.array(np.iinfo(np.int64).max).astype("int64"))
    cols = value_cols(case, rng, ("int64",), False, exact=True)
    aggs = [("sum", cols[0][1]), ("len", None)]
    c, prof, lines = attempts(plb, monkeypatch, capfd, case.keys, aggs, {"BL_K5_RADIX": "2", "BL_K5_HOTKEYS": "0"})
    assert len(lines) == 1 and lines[0]["sizing"] == "exact" and int(lines[0]["cap"]) == 0, lines
    check_line(lines[0], aggs, optin)
    assert "k5r_histogram" in prof, sorted(prof)
    c.check(None, "visible skew")


def test_key_builders():
    """The CPU side of the cases above: the sample-blind keys put their heavy bucket outside the sampled rows."""
    rng = np.random.default_rng(0)
    n = rr.MIN_ROWS + 4097
    keys = sample_blind_keys(rng, n, 6, 20_000)
    sampled = (np.arange(SAMPLE_ROWS, dtype=np.int64) * n) // SAMPLE_ROWS
    counts = rr.bucket_counts(keys, 6)
    assert counts.sum() == n - 3000 and counts[5] > n - SAMPLE_ROWS - 3000
    assert (rr.bucket_counts(keys[sampled], 6) < 3 * SAMPLE_ROWS / 64).all()
    assert (keys.view(np.uint64) == np.uint64(rr.GB_EMPTY)).sum() == 3000
