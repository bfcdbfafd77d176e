"""GPU tests of the partitioned group_by (K5r, groupby_radix.cu) on every scatter path, bucket count and key form, against
the exact restatement in tests/groupby_ref.py.  Where the keys sit is built and checked with tests/radix_ref.py.

K5r is forced with BL_K5_RADIX=2 and no heavy-hitter list (BL_K5_HOTKEYS=0); BL_K5R_STORE picks the store path of
the scatter (1 coalesced, 2 write-combining, 3 runs) where its shared memory fits.  Every case reads the BL_K5_DEBUG
line back: the bucket count and table size must be what radix_ref.plan() gives for the line's est_groups, the store
what radix_ref.store_path() gives, and the status 0 (or 1 where the case is built to fall back).

Sizes.  Rows are n_loop(sm) = 24576*SM + 4097 (3.25e6 on 132 SMs) unless a case says otherwise: odd, and one row past
a whole number of 2048-row (runs / coalesced) and 1024- or 2048-row (write-combining) tiles.  The bucket count follows
from est_groups (about 1.25x the distinct keys) and the pass-2 table of S slots: with the 5-word records of the
matrix (four value columns, 6 accumulator words: 60-byte entries) S = 512, so 4096 buckets take up to 0.55 * 512 *
4096 = 1.15e6 estimated groups and 8192 buckets the rest up to 0.7 * 512 * 8192 = 2.9e6; each case aims at the
geometric middle of its range.  Integer aggregates, counts and lengths match bit for bit; float sums use exact-summable
values; float min / max are exact.
"""
import re

import numpy as np
import pytest

import groupby_ref as ref
import radix_ref as rr
from test_gpu_groupby_plans import BIG, Call, _env, n_loop, profiled, value_cols

pytestmark = pytest.mark.gpu

STORES = {"coalesced": 1, "wc": 2, "runs": 3}
I64_MIN = np.iinfo(np.int64).min


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


def form(aggs):
    """(record width, accumulator words) of a call: one record word per distinct value column, one accumulator word per
    sum / mean / min / max (the columns carry no validity, so no null counters)."""
    cols = {id(c) for k, c in aggs if c is not None}
    return 1 + len(cols), sum(k in ("sum", "mean", "min", "max") for k, _ in aggs)


def radix_call(plb, monkeypatch, capfd, keys, aggs, store=None, knobs=None, key_valid=None, maintain_order=False):
    """One device-input group_by_agg with K5r forced; -> (Call, profile, fields of the last [k5r] line or None)."""
    kn = {"BL_K5_RADIX": "2", "BL_K5_HOTKEYS": "0", "BL_K5_DEBUG": "1"}
    if store is not None:
        kn["BL_K5R_STORE"] = str(STORES[store])
    kn.update(knobs or {})
    _env(monkeypatch, kn)
    if store is None:
        monkeypatch.delenv("BL_K5R_STORE", raising=False)
    capfd.readouterr()
    c, prof = profiled(plb, lambda: Call(plb, keys, key_valid, aggs, maintain_order, device=True))
    lines = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("[k5r]")]
    return c, prof, (dict(re.findall(r"(\w+)=(\S+)", lines[-1])) if lines else None)


def check_line(info, aggs, optin, store=None, buckets=None, status=0):
    """The [k5r] line: the plan radix_ref restates for its est_groups, the store path, the status."""
    assert info is not None, "K5r did not run"
    roww, nw = form(aggs)
    logB, S = rr.plan(int(info["est_groups"]), roww, nw)
    assert int(info["buckets"]) == 1 << logB and int(info["slots"]) == S, (info, roww, nw)
    if buckets is not None:
        assert int(info["buckets"]) == buckets, info
    want = rr.store_path(logB, roww, optin, STORES.get(store, 0))
    assert info["store"] == want and int(info["status"]) == status, (info, want)
    return logB, S


def groups_for(logB, roww, nw):
    """Distinct keys whose est_groups (~1.25x) sits in the geometric middle of the range that gives 2^logB buckets."""
    _, S = rr.plan(1, roww, nw)
    lo, hi = rr.est_range(logB, S)
    mid = hi / 2 if lo == 0 else (lo * hi) ** 0.5
    return int(mid / 1.25)


def matrix_aggs(case, rng, wide=False):
    """5-word records: Int64, Int32, UInt32 and exact-summable Float64 columns; sum of each, min of Int32 and max of
    Float64 (6 words), or (wide) sum / min / max of each (12 words); + len."""
    cols = [case.values(rng, dt) for dt in ("int64", "int32", "uint32")] + [case.values(rng, "float64", for_sum=True, exact=True)]
    if wide:
        return [(k, c) for c in cols for k in ("sum", "min", "max")] + [("len", None)]
    return [("sum", c) for c in cols] + [("min", cols[1]), ("max", cols[3]), ("len", None)]


# ------------------------------------------------------------------ the recorded wrong results
HEAVY_KEY = {"int32": -1, "uint32": (1 << 31) + 5, "int64": np.iinfo(np.int64).max, "uint64": (1 << 64) - 1}


def test_recorded_i32_1024_three_columns_coalesced(plb, sm, optin, monkeypatch, capfd):
    """Int32 keys, 1024 buckets, three value columns (4-word records), coalesced store."""
    rng = np.random.default_rng(41)
    n = n_loop(sm)
    case = ref.Case(rng, "int32", singletons=10_000, groups=420_000, rest=n - 10_000 - sum(ref.SPECIAL_ROWS.values()))
    cols = value_cols(case, rng, ("int64", "uint32", "int32"), False, exact=True)
    aggs = [("sum", c[1]) for c in cols] + [("len", None)]
    c, prof, info = radix_call(plb, monkeypatch, capfd, case.keys, aggs, "coalesced")
    check_line(info, aggs, optin, "coalesced", buckets=1024)
    c.check(None, "i32 1024 coalesced")


@pytest.mark.parametrize("store", list(STORES))
@pytest.mark.parametrize("key_dt", list(HEAVY_KEY))
def test_recorded_heavy_ordinary_key(plb, sm, optin, monkeypatch, capfd, key_dt, store):
    """One ordinary key (not GB_EMPTY) holds 2^20 of the n_loop(sm) rows; 500k further groups -> 1024 buckets."""
    rng = np.random.default_rng(43 + len(key_dt) + STORES[store])
    n = n_loop(sm)
    case = ref.Case(rng, key_dt, big=BIG, singletons=10_000, groups=500_000, rest=n - BIG - 10_000 - sum(ref.SPECIAL_ROWS.values()),
                    big_key=np.array(HEAVY_KEY[key_dt]).astype(key_dt))
    cols = value_cols(case, rng, ("int64", "float64"), False, exact=True)
    aggs = [("sum", cols[0][1]), ("sum", cols[1][1]), ("min", cols[0][2]), ("max", cols[0][2]), ("len", None)]
    c, prof, info = radix_call(plb, monkeypatch, capfd, case.keys, aggs, store)
    check_line(info, aggs, optin, store, buckets=1024)
    c.check(None, f"heavy {key_dt} {store}")


# ------------------------------------------------------------------ every store path at every bucket count
@pytest.mark.parametrize("store", list(STORES))
@pytest.mark.parametrize("logB", [6, 9, 10, 11, 12, 13])
def test_store_matrix(plb, sm, optin, monkeypatch, capfd, logB, store):
    rng = np.random.default_rng(logB * 10 + STORES[store])
    n = n_loop(sm)
    D = groups_for(logB, 5, 6)
    case = ref.Case(rng, "int64", groups=D, rest=n - sum(ref.SPECIAL_ROWS.values()))
    aggs = matrix_aggs(case, rng)
    c, prof, info = radix_call(plb, monkeypatch, capfd, case.keys, aggs, store)
    check_line(info, aggs, optin, store, buckets=1 << logB)
    c.check(None, f"matrix {1 << logB} {store}")


# ------------------------------------------------------------------ forms
WIDTHS = {          # name: (key dtype, value dtypes; float columns bring a second (min / max) column)
    "w1_u32key": ("uint32", ()),
    "w2_i32": ("int64", ("int32",)),
    "w3_f32": ("int32", ("float32",)),
    "w4_u32_u64_i64": ("uint64", ("uint32", "uint64", "int64")),
    "w5_i32_u32_f64": ("int64", ("int32", "uint32", "float64")),
}


@pytest.mark.parametrize("store", list(STORES))
@pytest.mark.parametrize("name", list(WIDTHS))
def test_widths_and_dtypes(plb, sm, optin, monkeypatch, capfd, name, store):
    """Record widths 1-5, full-range values (Int32 negatives, UInt32 >= 2^31, Int64 MIN / MAX sums that wrap, NaN /
    +-inf / -0.0 under float min / max) under sum, mean, min, max, count and len, 120k groups (512 buckets or fewer:
    1024+ with the forced paths that fit)."""
    key_dt, dts = WIDTHS[name]
    rng = np.random.default_rng(len(name) * 3 + STORES[store])
    n = n_loop(sm)
    case = ref.Case(rng, key_dt, singletons=20_000, groups=100_000, rest=n - 20_000 - sum(ref.SPECIAL_ROWS.values()))
    cols = value_cols(case, rng, dts, False, exact=True)
    aggs = [a for _, s, mm in cols for a in (("sum", s), ("mean", s), ("min", mm), ("max", mm), ("count", mm))] + [("len", None)]
    c, prof, info = radix_call(plb, monkeypatch, capfd, case.keys, aggs, store)
    check_line(info, aggs, optin, store)
    c.check(None, f"{name} {store}")


@pytest.mark.parametrize("store", list(STORES))
@pytest.mark.parametrize("half", [0, 1])
def test_empty_key_group(plb, sm, optin, monkeypatch, capfd, half, store):
    """The GB_EMPTY key (i64::MIN: the pad marker, aggregated beside the record streams by gbr_apply_special and
    appended by k_gbr_append_special) on 3000 rows, with every value dtype (three per call) under sum / min / max."""
    dts = ("int64", "uint64", "int32", "uint32", "float64", "float32")[3 * half: 3 * half + 3]
    rng = np.random.default_rng(70 + half * 5 + STORES[store])
    n = n_loop(sm)
    case = ref.Case(rng, "int64", big=3000, singletons=10_000, groups=300_000, rest=n - 13_000 - sum(ref.SPECIAL_ROWS.values()), big_key=I64_MIN)
    cols = [case.values(rng, dt, for_sum=True, exact=True) for dt in dts]
    aggs = [(k, c) for c in cols for k in ("sum", "min", "max")] + [("len", None)]
    c, prof, info = radix_call(plb, monkeypatch, capfd, case.keys, aggs, store)
    check_line(info, aggs, optin, store)
    c.check(None, f"empty key {dts} {store}")


def test_large_table_branch(plb, sm, optin, monkeypatch, capfd):
    """5-word records with 12 accumulator words (108-byte entries): 512 entries and the 79 KB ring do not fit 110 KB, so
    the table takes 222 KB (S = 1344, one CTA per SM); 1.5e6 groups -> 4096 buckets."""
    rng = np.random.default_rng(77)
    n = n_loop(sm)
    case = ref.Case(rng, "int64", groups=1_500_000, rest=n - sum(ref.SPECIAL_ROWS.values()))
    aggs = matrix_aggs(case, rng, wide=True)
    c, prof, info = radix_call(plb, monkeypatch, capfd, case.keys, aggs)
    _, S = check_line(info, aggs, optin, buckets=4096)
    assert S == 1344, info
    c.check(None, "222 KB table")


# ------------------------------------------------------------------ bucket edges (64 buckets, 2-word records: S = 3968)
def bucket_rows(rng, logB, spec, dtype="int64"):
    """Keys with exactly spec[bucket] = (rows, groups) in the named buckets; -> shuffled key column."""
    parts, seen = [], np.zeros(0, np.uint64)
    for b, (rows, groups) in spec.items():
        k = rr.keys64_in_bucket(rng, logB, b, groups, avoid=seen)
        seen = np.concatenate([seen, k])
        parts.append(np.concatenate([k, k[rng.integers(0, groups, rows - groups)]]))
    bits = np.concatenate(parts)
    return rr.as_dtype(bits[rng.permutation(bits.size)], dtype)


EDGES = {
    # 991 / 992 / 993 / 1985 records: one short of, exactly, one past one 992-record ring stage, and one past two
    "streams": lambda n: {3: (991, 400), 4: (992, 300), 5: (993, 500), 6: (1985, 700), 7: (1, 1)} | {b: ((n - 4962) // 56 + (b == 8) * ((n - 4962) % 56), 1200) for b in range(8, 64)},
    "odd_empty": lambda n: {b: (n // 32 + (b == 0) * (n % 32), 1200) for b in range(0, 64, 2)},
    "one_bucket": lambda n: {17: (n, 1500)},
}


@pytest.mark.parametrize("store", list(STORES))
@pytest.mark.parametrize("edge", list(EDGES))
def test_bucket_edges(plb, sm, optin, monkeypatch, capfd, edge, store):
    """Bucket streams built with radix_ref (64 buckets): 991, 992, 993 and 1985 records (the odd last stage read of the
    coalesced store, whose streams are exactly the rows), every other bucket empty, and all keys in one bucket."""
    rng = np.random.default_rng(len(edge) + STORES[store])
    n = rr.MIN_ROWS + 2049
    keys = bucket_rows(rng, 6, EDGES[edge](n))
    assert keys.size == n
    vals = ref.sum_column(rng, "int64", n)
    aggs = [("sum", (vals, None)), ("len", None)]
    c, prof, info = radix_call(plb, monkeypatch, capfd, keys, aggs, store)
    check_line(info, aggs, optin, store, buckets=64)
    assert (rr.bucket_counts(keys, 6) > 0).sum() == len(EDGES[edge](n))
    c.check(None, f"edge {edge} {store}")


# ------------------------------------------------------------------ fall-backs to the L2 plan
def fallback_case(rng, extra):
    """64 buckets, 2-word records (S = 3968, max_used = 2976): bucket 3 holds `extra` = {"full": k} keys, one per
    start slot spread over the table (no probing), or {"slot": k} keys that share start slot 100; 20k other keys."""
    n = rr.MIN_ROWS + 4097
    S = 3968
    if "full" in extra:
        k = extra["full"]
        slots = (np.arange(k) * S) // k
        special = np.concatenate([rr.keys64_in_bucket(rng, 6, 3, 1, S=S, slot=int(s)) for s in slots])
    else:
        special = rr.keys64_in_bucket(rng, 6, 3, extra["slot"], S=S, slot=100)
    other = np.concatenate([rr.keys64_in_bucket(rng, 6, b, 350, avoid=special) for b in range(64) if b != 3])
    bits = np.concatenate([special, other, other[rng.integers(0, other.size, n - special.size - other.size)]])
    return rr.as_dtype(bits[rng.permutation(n)], "int64")


@pytest.mark.parametrize("shape,status", [("max_used", 0), ("max_used_plus_1", None), ("all_slots", 1), ("probe_128", 0), ("probe_129", 1)])
def test_table_fallbacks(plb, monkeypatch, capfd, optin, shape, status):
    """One bucket at exactly max_used = S - S/4 groups stays on K5r.  Past it a new key gives up once it reads
    s_used >= max_used; up to one key per consumer thread (992) may pass that check together, so one group more may stay
    on K5r (status 0 or 1, exact either way) and S = 3968 groups (all slots) cannot.  128 keys with one start slot fit
    the 128-probe limit, 129 do not.  A raised status makes the L2 plan redo the call, exactly."""
    rng = np.random.default_rng(len(shape))
    extra = {"max_used": {"full": 2976}, "max_used_plus_1": {"full": 2977}, "all_slots": {"full": 3968},
             "probe_128": {"slot": 128}, "probe_129": {"slot": 129}}[shape]
    keys = fallback_case(rng, extra)
    vals = ref.sum_column(rng, "int64", keys.size)
    aggs = [("sum", (vals, None)), ("len", None)]
    c, prof, info = radix_call(plb, monkeypatch, capfd, keys, aggs)
    if status is None:
        status = int(info["status"])
    check_line(info, aggs, optin, buckets=64, status=status)
    assert "k5r_aggregate" in prof and ("k5_extract" in prof) == (status == 1), sorted(prof)
    c.check(None, shape)


def test_dense_bound_fallback(plb, monkeypatch, capfd, optin):
    """More groups than the dense output bound Gb = 3 * est_groups + 65536: every row of the strided 65,536-row sample
    (k_gb_estimate: row i * n / m) carries one key, the other rows 100k further keys -> est_groups = 3, Gb = 65545,
    100,001 groups.  K5r raises the status at the compaction and the L2 plan redoes the call."""
    rng = np.random.default_rng(5)
    n, m = rr.MIN_ROWS + 4097, 65536
    sampled = (np.arange(m, dtype=np.int64) * n) // m
    other = np.unique(rng.integers(1, 1 << 40, 110_000))[:100_000]
    rest = np.setdiff1d(np.arange(n), sampled)
    fill = np.concatenate([other, other[rng.integers(0, other.size, rest.size - other.size)]])
    keys = np.empty(n, np.int64)
    keys[rest] = fill[rng.permutation(rest.size)]
    keys[sampled] = 42
    vals = ref.sum_column(rng, "int64", n)
    aggs = [("sum", (vals, None)), ("len", None)]
    c, prof, info = radix_call(plb, monkeypatch, capfd, keys, aggs)
    assert int(info["est_groups"]) < 100 and np.unique(keys).size > 3 * int(info["est_groups"]) + 65536, info
    check_line(info, aggs, optin, status=1)
    assert "k5r_aggregate" in prof and "k5_extract" in prof, sorted(prof)
    c.check(None, "dense bound")


# ------------------------------------------------------------------ selection and eligibility
@pytest.mark.parametrize("n,taken", [(rr.MIN_ROWS - 1, False), (rr.MIN_ROWS, True)])
def test_min_rows(plb, monkeypatch, capfd, n, taken):
    rng = np.random.default_rng(n)
    case = ref.Case(rng, "int64", groups=50_000, rest=n - sum(ref.SPECIAL_ROWS.values()))
    s = case.values(rng, "int64")
    aggs = [("sum", s), ("len", None)]
    c, prof, info = radix_call(plb, monkeypatch, capfd, case.keys, aggs)
    assert ("k5r_aggregate" in prof) == taken and (info is not None) == taken, (sorted(prof), info)
    c.check(None, f"{n} rows")


@pytest.mark.parametrize("shape", ["float_key", "key_validity", "value_validity", "maintain_order"])
def test_stays_on_l2(plb, sm, monkeypatch, capfd, shape):
    """Float keys (first-row tracking), validity on keys or values and maintain_order keep the L2 plan."""
    rng = np.random.default_rng(len(shape))
    n = n_loop(sm)
    case = ref.Case(rng, "float64" if shape == "float_key" else "int64", groups=300_000, rest=n - 1000 - sum(ref.SPECIAL_ROWS.values()),
                    null_rows=1000 if shape == "key_validity" else 0)
    s = case.values(rng, "int64", nullable=shape == "value_validity")
    aggs = [("sum", s), ("len", None)]
    c, prof, info = radix_call(plb, monkeypatch, capfd, case.keys, aggs, key_valid=case.key_valid, maintain_order=shape == "maintain_order")
    assert info is None and "k5r_aggregate" not in prof and "k5_extract" in prof, (sorted(prof), info)
    c.check(None, shape)


def test_default_rule_c2(plb, monkeypatch, capfd, optin):
    """No knob: a C2-shaped call (1e6 uniform Int64 keys, device input, sum(Int64), mean(Float64), len) takes K5r."""
    rng = np.random.default_rng(2)
    n = 6_000_001
    distinct = rng.permutation(np.unique(rng.integers(1, 1 << 50, 1_050_000))[:1_000_000])
    keys = distinct[rng.integers(0, distinct.size, n)]
    a = ref.sum_column(rng, "int64", n)
    b = ref.sum_column(rng, "float64", n, exact=True)
    aggs = [("sum", (a, None)), ("mean", (b, None)), ("len", None)]
    for k in ("BL_K5_RADIX", "BL_K5_HOTKEYS", "BL_K5R_STORE"):
        monkeypatch.delenv(k, raising=False)
    monkeypatch.setenv("BL_K5_DEBUG", "1")
    capfd.readouterr()
    c, prof = profiled(plb, lambda: Call(plb, keys, None, aggs, False, device=True))
    lines = [ln for ln in capfd.readouterr().err.splitlines() if ln.startswith("[k5r]")]
    assert lines and "k5r_aggregate" in prof, sorted(prof)
    check_line(dict(re.findall(r"(\w+)=(\S+)", lines[-1])), aggs, optin)
    c.check(None, "C2 default")
