"""GPU tests of the hash join (K7 build, K8 probe in join.cu) on every table form and probe path, against the oracle's
join (oracle.hash_join / hash_join_multi), over the full key range of every key dtype and past the grid caps.

Each test selects one plan with the knobs join.cu reads on every call (BL_JOIN_TABLE, BL_JOIN_DENSE, BL_JOIN_FUSED,
BL_JOIN_BUCKET_FILL), proves with the launch profile that the plan ran, and compares (left_idx, right_idx) and their
validity with the oracle exactly, as sequences.  The keys come from tests/join_keys.py; test_oracle.py checks the
oracle by brute force on the same kind of columns.

Plans and their labels:
  DENSE    k7_dense_build (u32 table[key - min]; integer builds of >= 1024 rows whose span is < 8 x rows)
  WIDE     k7_join_build (two-entry buckets; i64::MIN / UInt64 2^63 is the empty marker and lives in a special bucket)
  COMPACT  k7_jc_build (fingerprint:8 | row:24 below 2^24 - 1 build rows, plain row ids from there)
  probe    k8_join_probe_emit (unique build keys, fused), k8_join_probe + k8_join_emit (BL_JOIN_FUSED=0, or duplicate build
           keys: CSR row lists from k7_csr_offsets), k8_join_probe_bits (semi / anti)

Sizes.  The caps come from grid_for (common.cuh) and probe_tuples with SM = device_info()["sm_count"] (132 on an H100
SXM).  N_BUILD = 12288*SM + 777 build rows pass the build loops (8*SM CTAs x 256 threads: twice from 2048*SM rows) and
the CSR scans over the WIDE entries (2*(nb+1) entries in 2048-entry tiles over 8*SM CTAs: from about 8192*SM rows) and
the COMPACT slots (cap + 1 >= 2^22 slots).  N_PROBE = 36864*SM + 1001 probe rows give every fused CTA (6*SM of them)
about three 2048-row tiles, put the look-back more than 32 tiles back, and run the pass-1 (8*SM x 256 x 2 rows), emit
(8*SM tiles) and probe-bits (16*SM x 256) loops several times with a ragged tail.
"""
import numpy as np
import pytest

import join_keys as jk
import oracle
from radix_ref import key_with_hash

pytestmark = pytest.mark.gpu

IDX_NULL = 0xFFFFFFFF
HOWS = ("inner", "left", "semi", "anti", "full")
INNER_ORDERS = ("none", "left", "left_right", "right")
LEFT_ORDERS = ("none", "left", "right", "right_left")
BUILD_LABEL = {"dense": "k7_dense_build", "wide": "k7_join_build", "compact": "k7_jc_build"}


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as m
    m.init()
    return m


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


def n_build(sm):
    return 12288 * sm + 777


def n_probe(sm):
    return 36864 * sm + 1001


def wide_tail_keys(rng, n_rows: int, fill: float, count: int) -> list:
    """`count` keys whose home bucket is one of the last two of a WIDE table built over n_rows rows at `fill` rows per
    bucket (join_build: nb = int(rows / fill) + 1): more than those buckets hold, so the rest wrap to bucket 0."""
    nbk = max(int(n_rows / fill) + 1, 8)
    lo = -(-(nbk - 2) * (1 << 64) // nbk)
    return [key_with_hash(int(x)) for x in rng.integers(lo, 1 << 64, count, dtype=np.uint64, endpoint=False)]


def compact_collision_keys(rng, n_rows: int, groups: int, per_group: int) -> list:
    """Keys for a COMPACT table over n_rows rows: `groups` groups of `per_group` different keys that share their home
    slot AND their 8-bit fingerprint (only the check against the build key column tells them apart); the first group
    sits in the last slot, so its probe sequence wraps to slot 0."""
    cap = 1024
    while cap < n_rows + n_rows // 2:
        cap <<= 1
    top = cap.bit_length() - 1 + 8                  # slot bits + fingerprint bits
    low = 64 - top
    out = []
    for g in range(groups):
        prefix = (1 << top) - 1 if g == 0 else int(rng.integers(0, 1 << top))
        lows = set()
        while len(lows) < per_group:
            lows.add(int(rng.integers(0, 1 << low)))
        out += [key_with_hash((prefix << low) | x) for x in sorted(lows)]
    return out


def as_keys(planted, dtype) -> np.ndarray:
    """Python ints in [0, 2^64) as UInt64 / Int64 keys (the same bit patterns)."""
    return np.array(planted, dtype=np.uint64).view(np.dtype(dtype))


def plant(values, planted):
    """`values` with len(planted) entries replaced by `planted` (the bit patterns of as_keys), spread over the column;
    the specials of join_keys are never the ones replaced."""
    v = values.copy()
    p = as_keys(planted, v.dtype)
    idx = np.flatnonzero(~np.isin(v, p) & ~np.isin(v, jk.specials(v.dtype)))
    v[idx[np.linspace(0, idx.size - 1, p.size).astype(np.int64)]] = p
    return v


def with_probes(rng, lk, planted, copies=3):
    """The probe column `lk` with `copies` rows of every planted key, at random places."""
    p = np.repeat(as_keys(planted, lk.dtype), copies)
    out = lk.copy()
    out[rng.choice(lk.size, p.size, replace=False)] = p
    return out


def set_plan(monkeypatch, table="wide", dense=True, fused=True, fill=None):
    monkeypatch.setenv("BL_JOIN_TABLE", table if table != "dense" else "wide")
    monkeypatch.setenv("BL_JOIN_DENSE", "1" if dense else "0")
    monkeypatch.setenv("BL_JOIN_FUSED", "1" if fused else "0")
    if fill is None:
        monkeypatch.delenv("BL_JOIN_BUCKET_FILL", raising=False)
    else:
        monkeypatch.setenv("BL_JOIN_BUCKET_FILL", str(fill))


def profiled(plb, fn):
    plb.profile_reset()
    plb.profile_enable(True)
    try:
        r = fn()
    finally:
        prof = plb.profile()
        plb.profile_enable(False)
    return r, prof


def assert_seq(got, exp, what):
    got = np.asarray(got)
    exp = np.asarray(exp)
    assert got.size == exp.size, f"{what}: {got.size} tuples, expected {exp.size}"
    bad = np.flatnonzero(got != exp)
    assert bad.size == 0, f"{what}: {bad.size} differ, first at {bad[0]}: got {got[bad[0]:bad[0] + 4]}, expected {exp[bad[0]:bad[0] + 4]}"


def check_join(got, exp, what):
    """got = ((li, valid), (ri, valid)) of the library; exp = the oracle's (li, ri) with IDX_NULL for a missing side."""
    (li, lvd), (ri, rvd) = got
    eli, eri = exp
    assert_seq(li, eli, f"{what} left idx")
    assert_seq(ri, eri, f"{what} right idx")
    for v, e, side in ((lvd, eli, "left"), (rvd, eri, "right")):
        ev = e != IDX_NULL
        assert np.array_equal(np.ones(e.size, bool) if v is None else v, ev), f"{what} {side} validity"


def join(plb, lk, lv, rk, rv, how, nulls_equal=False, order="none", device=False):
    if not device:
        return plb.hash_join(plb.Column(lk, lv), plb.Column(rk, rv), how, nulls_equal, order)
    dl, dr = plb.to_device(lk, lv), plb.to_device(rk, rv)
    ol, orr = plb.hash_join(dl.view(), dr.view(), how, nulls_equal, order, location=plb.DEVICE)
    return ol.to_numpy(), orr.to_numpy()


def run(plb, lk, lv, rk, rv, how, nulls_equal=False, order="none", device=False, what=""):
    """One join checked against the oracle; returns the launch profile of the library call."""
    got, prof = profiled(plb, lambda: join(plb, lk, lv, rk, rv, how, nulls_equal, order, device))
    exp = oracle.hash_join(lk, rk, lv, rv, how, nulls_equal, order, 8)
    check_join(got, exp, f"{what} {how} nulls_equal={nulls_equal} order={order}")
    return prof


def assert_plan(prof, form, probe, csr=False, what=""):
    """form: dense / wide / compact; probe: fused / two_pass / bits."""
    names = sorted(prof)
    for f, label in BUILD_LABEL.items():
        assert (label in prof) == (f == form), (what, form, names)
    if probe == "fused":
        assert "k8_join_probe_emit" in prof and "k8_join_probe" not in prof, (what, names)
    elif probe == "two_pass":
        assert "k8_join_probe" in prof and "k8_join_emit" in prof and "k8_join_probe_emit" not in prof, (what, names)
    else:
        assert "k8_join_probe_bits" in prof and "k8_join_probe" not in prof and "k8_join_probe_emit" not in prof, (what, names)
    assert ("k7_csr_offsets" in prof) == csr, (what, names)


def run_hows(plb, lk, lv, rk, rv, form, fused=True, csr=False, hows=HOWS, nulls_equal=False, what=""):
    """Every join type on one plan.  Inner joins build the shorter side, the others the right side."""
    for how in hows:
        prof = run(plb, lk, lv, rk, rv, how, nulls_equal, what=what)
        probe = "bits" if how in ("semi", "anti") else ("fused" if fused and not csr else "two_pass")
        assert_plan(prof, form, probe, csr and how not in ("semi", "anti"), f"{what} {how}")


# ------------------------------------------------------------------------------------------------ DENSE
def test_dense_large(plb, sm, monkeypatch):
    """Int64 keys crossing zero, every join type and every maintain_order, probe keys on both sides of [kmin, kmax]."""
    set_plan(monkeypatch, "dense")
    rng = np.random.default_rng(1)
    nb, np_ = n_build(sm), n_probe(sm)
    rk, rv = jk.keys(rng, "int64", nb, "unique", nulls=0.01, dense=4 * nb)
    lk, lv = jk.probe(rng, rk, np_, nulls=0.01, dense_edges=True)
    run_hows(plb, lk, lv, rk, rv, "dense", what="dense int64")
    for order in INNER_ORDERS[1:]:
        assert_plan(run(plb, lk, lv, rk, rv, "inner", order=order, what="dense"), "dense", "fused")
        # right probes: the sort by left runs on the build side's indices
        assert_plan(run(plb, rk, rv, lk, lv, "inner", order=order, what="dense swapped"), "dense", "fused")
    for order in LEFT_ORDERS[1:]:
        assert_plan(run(plb, lk, lv, rk, rv, "left", order=order, what="dense"), "dense", "fused")
    set_plan(monkeypatch, "dense", fused=False)
    for how in ("inner", "left"):
        assert_plan(run(plb, lk, lv, rk, rv, how, what="dense two-pass"), "dense", "two_pass")


@pytest.mark.parametrize("dtype", ["int32", "int64", "uint64", "uint32", "uint16"])
def test_dense_dtypes(plb, monkeypatch, dtype):
    """Signed runs cross zero (j_ordered sign-extends and flips the sign bit), unsigned runs end at the dtype's MAX; probe
    keys just outside [kmin, kmax] and at the dtype's extremes, where key - kmin wraps."""
    set_plan(monkeypatch, "dense")
    rng = np.random.default_rng(2)
    nb = 5000
    rk, rv = jk.keys(rng, dtype, nb, "unique", nulls=0.02, dense=3 * nb)
    lk, lv = jk.probe(rng, rk, 3 * nb + 7, nulls=0.02, dense_edges=True)
    run_hows(plb, lk, lv, rk, rv, "dense", what=f"dense {dtype}")


def test_dense_threshold(plb, monkeypatch):
    """max - min = 8*nb - 1 runs DENSE, max - min = 8*nb runs hashed; below 1024 build rows the min / max kernel never
    runs."""
    set_plan(monkeypatch, "dense")
    rng = np.random.default_rng(3)
    for nb, spread, form in ((1024, 8 * 1024 - 1, "dense"), (1024, 8 * 1024, "wide"), (4099, 8 * 4099 - 1, "dense"), (4099, 8 * 4099, "wide"), (1023, 1022, "wide")):
        rk, rv = jk.keys(rng, "int32", nb, "unique", dense=spread + 1)
        assert int(rk.max()) - int(rk.min()) == spread
        lk, lv = jk.probe(rng, rk, 3 * nb, dense_edges=True)
        for how in ("left", "semi"):
            prof = run(plb, lk, lv, rk, rv, how, what=f"nb={nb} max-min={spread}")
            assert_plan(prof, form, "bits" if how == "semi" else "fused", what=(nb, spread, how))
            assert ("k7_join_minmax" in prof) == (nb >= 1024), sorted(prof)


def test_dense_rejected_for_duplicates(plb, monkeypatch):
    """A dense build with duplicates: inner / left build DENSE, see the duplicates and fall back to a hashed table with CSR
    lists; semi / anti only need membership and stay DENSE.  nulls_equal never runs DENSE."""
    set_plan(monkeypatch, "dense")
    rng = np.random.default_rng(4)
    nb = 20_000
    rk, rv = jk.keys(rng, "int64", nb, "k", k=2, nulls=0.01, dense=2 * nb)
    lk, lv = jk.probe(rng, rk, 3 * nb, nulls=0.01, dense_edges=True)
    for how in ("inner", "left", "full"):
        prof = run(plb, lk, lv, rk, rv, how, what="dense dups")
        assert all(x in prof for x in ("k7_dense_build", "k7_join_build", "k7_csr_offsets", "k8_join_probe", "k8_join_emit")), sorted(prof)
    for how in ("semi", "anti"):
        assert_plan(run(plb, lk, lv, rk, rv, how, what="dense dups"), "dense", "bits")
    lk2, lv2 = jk.probe(rng, rk, 3 * nb, nulls=12, dense_edges=True)
    rk2, rv2 = jk.keys(rng, "int64", nb, "unique", nulls=9, dense=2 * nb)
    for how in HOWS:
        prof = run(plb, lk2, lv2, rk2, rv2, how, nulls_equal=True, what="dense nulls_equal")
        assert "k7_join_minmax" not in prof and "k7_dense_build" not in prof, sorted(prof)


# ------------------------------------------------------------------------------------------------ WIDE
@pytest.mark.parametrize("fill", [None, 0.5, 1.9])
def test_wide_large(plb, sm, monkeypatch, fill):
    """UInt64 keys over the full range with 2^63 (the empty marker) on both sides, and keys whose home bucket is one of
    the last two, so their probe sequences wrap to bucket 0.  Unique fused, unique two-pass, and CSR lists."""
    rng = np.random.default_rng(5)
    nb, np_ = n_build(sm), n_probe(sm)
    tail = wide_tail_keys(rng, nb, fill or 1.0, 40)
    rk, _ = jk.keys(rng, "uint64", nb, "unique")
    rk = plant(rk, tail)
    assert (rk == np.uint64(1 << 63)).sum() == 1
    lk, lv = jk.probe(rng, rk, np_, nulls=0.01)
    lk = with_probes(rng, lk, tail + [1 << 63] * 20)
    set_plan(monkeypatch, "wide", dense=False, fill=fill)
    run_hows(plb, lk, lv, rk, None, "wide", hows=("inner", "left", "anti"), what=f"wide fill={fill}")
    set_plan(monkeypatch, "wide", dense=False, fused=False, fill=fill)
    for how in ("inner", "left"):
        assert_plan(run(plb, lk, lv, rk, None, how, what=f"wide two-pass fill={fill}"), "wide", "two_pass")
    # duplicates: runs of 1..8, with 2^63 and the wrapping keys among them (three rows each)
    rd, rdv = jk.keys(rng, "uint64", nb, "runs", k=8, nulls=0.01)
    rd = plant(rd, (tail + [1 << 63]) * 3)
    ld, ldv = jk.probe(rng, rd, np_, nulls=0.01)
    ld = with_probes(rng, ld, tail + [1 << 63] * 20)
    set_plan(monkeypatch, "wide", dense=False, fill=fill)
    run_hows(plb, ld, ldv, rd, rdv, "wide", csr=True, hows=("inner", "left", "semi", "full"), what=f"wide csr fill={fill}")


def test_wide_float64_large(plb, sm, monkeypatch):
    """Float64 keys from random bit patterns: NaN payloads of both signs on the probe side meet the build's one NaN,
    -0.0 meets +0.0, +-inf and subnormals are keys like any other."""
    set_plan(monkeypatch, "wide")
    rng = np.random.default_rng(6)
    nb, np_ = n_build(sm), n_probe(sm)
    rk, rv = jk.keys(rng, "float64", nb, "unique", nulls=0.01)
    lk, lv = jk.probe(rng, rk, np_, nulls=0.01)
    nan = np.array([0x7FF8000000000000, 0xFFF8000000000001, 0x7FF0000000000001, 0xFFFFFFFFFFFFFFFF], np.uint64).view(np.float64)
    lk[rng.integers(0, np_, 40)] = nan[rng.integers(0, nan.size, 40)]
    lk[rng.integers(0, np_, 40)] = -0.0
    run_hows(plb, lk, lv, rk, rv, "wide", hows=("inner", "left", "semi", "full"), what="wide f64")


# ------------------------------------------------------------------------------------------------ COMPACT
def test_compact_large(plb, sm, monkeypatch):
    """fp_mode = 1 (fingerprint | 24-bit row) at N_BUILD, with groups of keys that share both their home slot and their
    fingerprint (one group in the last slot, wrapping to slot 0): unique fused, unique two-pass, CSR lists."""
    rng = np.random.default_rng(7)
    nb, np_ = n_build(sm), n_probe(sm)
    coll = compact_collision_keys(rng, nb, 24, 8)
    rk, rv = jk.keys(rng, "int64", nb, "unique", nulls=0.01)
    rk = plant(rk, coll)
    lk, lv = jk.probe(rng, rk, np_, nulls=0.01)
    lk = with_probes(rng, lk, coll)
    set_plan(monkeypatch, "compact", dense=False)
    run_hows(plb, lk, lv, rk, rv, "compact", what="compact")
    set_plan(monkeypatch, "compact", dense=False, fused=False)
    for how in ("inner", "left"):
        assert_plan(run(plb, lk, lv, rk, rv, how, what="compact two-pass"), "compact", "two_pass")
    for order in INNER_ORDERS[1:]:
        assert_plan(run(plb, rk, rv, lk, lv, "inner", order=order, what="compact swapped"), "compact", "two_pass")
    rd, rdv = jk.keys(rng, "int64", nb, "runs", k=6, nulls=0.01)
    rd = plant(rd, coll * 2)
    ld, ldv = jk.probe(rng, rd, np_, nulls=0.01)
    ld = with_probes(rng, ld, coll)
    set_plan(monkeypatch, "compact", dense=False)
    run_hows(plb, ld, ldv, rd, rdv, "compact", csr=True, hows=("inner", "left", "anti"), what="compact csr")
    for order in LEFT_ORDERS[1:]:
        assert_plan(run(plb, ld, ldv, rd, rdv, "left", order=order, what="compact csr"), "compact", "two_pass", csr=True)


@pytest.mark.parametrize("dups", ["unique", "runs"])
def test_compact_plain_row_ids(plb, monkeypatch, dups):
    """From 2^24 - 1 build rows COMPACT stores plain row ids (fp_mode = 0); matches must reach rows >= 2^24."""
    set_plan(monkeypatch, "compact", dense=False)
    rng = np.random.default_rng(8)
    nb = (1 << 24) + 1000
    rk, _ = jk.keys(rng, "int64", nb, dups, k=3)
    lk, lv = jk.probe(rng, rk, 1_000_003, nulls=0.01)
    lk = np.concatenate([lk, rk[1 << 24:], rk[-5000:]])      # every build row past 2^24 is probed
    lv = np.concatenate([lv, np.ones(lk.size - lv.size, bool)])
    perm = rng.permutation(lk.size)
    lk, lv = lk[perm], lv[perm]
    for how in ("left", "semi"):
        prof = run(plb, lk, lv, rk, None, how, what=f"compact fp_mode=0 {dups}")
        assert_plan(prof, "compact", "bits" if how == "semi" else ("fused" if dups == "unique" else "two_pass"), csr=dups != "unique" and how != "semi")


# ------------------------------------------------------------------------------------------------ probe paths on hashed forms
@pytest.mark.parametrize("form", ["wide", "compact"])
def test_csr_run_lengths(plb, monkeypatch, form):
    """Build keys repeated 1..200 times, so one warp of probe rows emits runs of every length."""
    set_plan(monkeypatch, form, dense=False)
    rng = np.random.default_rng(9)
    rk, rv = jk.keys(rng, "int64", 120_000, "runs", k=200, nulls=0.01)
    lk, lv = jk.probe(rng, rk, 300_001, hit=0.5, nulls=0.01)
    run_hows(plb, lk, lv, rk, rv, form, csr=True, hows=("inner", "left", "full"), what=f"{form} runs")


@pytest.mark.parametrize("form", ["wide", "compact"])
def test_hot_key(plb, monkeypatch, form):
    """One build key with 5000 rows, probed by 2000 rows: 10M tuples, each probe row's run takes many 128-tuple rounds
    of the emit."""
    set_plan(monkeypatch, form, dense=False)
    rng = np.random.default_rng(10)
    rk, rv = jk.keys(rng, "uint64", 60_000, "hot", k=5000, nulls=0.01)
    vals, cnt = np.unique(rk, return_counts=True)
    hot = vals[cnt.argmax()]
    lk, lv = jk.probe(rng, rk, 400_000, hit=0.3, nulls=0.01)
    lk = np.concatenate([lk, np.full(2000, hot)]); lv = np.concatenate([lv, np.ones(2000, bool)])
    perm = rng.permutation(lk.size)
    lk, lv = lk[perm], lv[perm]
    for how in ("inner", "left"):
        assert_plan(run(plb, lk, lv, rk, rv, how, what=f"{form} hot"), form, "two_pass", csr=True)


@pytest.mark.parametrize("form", ["wide", "compact"])
def test_nulls_equal(plb, monkeypatch, form):
    """Null keys join null keys: a single null build row (unique path) and duplicate null rows (CSR), with null rows on
    the probe side; WIDE keeps them in the special bucket's entry 0, COMPACT in tab[cap]."""
    set_plan(monkeypatch, form, dense=False)
    rng = np.random.default_rng(11)
    for dtype in ("int64", "float32"):
        for build_nulls, dups in ((1, "unique"), (30, "unique"), (30, "k")):
            rk, rv = jk.keys(rng, dtype, 20_000, dups, k=2, nulls=build_nulls)
            lk, lv = jk.probe(rng, rk, 50_001, nulls=25)
            csr = build_nulls > 1 or dups != "unique"
            run_hows(plb, lk, lv, rk, rv, form, csr=csr, nulls_equal=True, what=f"{form} {dtype} nulls={build_nulls} {dups}")


def test_empty_key_on_both_sides(plb, monkeypatch):
    """i64::MIN (= UInt64 2^63, the empty marker of WIDE) as a unique and a duplicated key, build and probe side, next to
    null keys in the same special bucket."""
    rng = np.random.default_rng(12)
    for dtype in ("int64", "uint64"):
        for copies in (1, 5):
            # join_keys plants the pattern once among unique keys; five copies among keys that come twice each
            rk, rv = jk.keys(rng, dtype, 30_000, "k", k=2 if copies > 1 else 1, nulls=10)
            if copies > 1:
                rk = plant(rk, [1 << 63] * copies)
            assert (rk == as_keys([1 << 63], dtype)[0]).sum() >= copies
            lk, lv = jk.probe(rng, rk, 70_000, nulls=10)
            lk = with_probes(rng, lk, [1 << 63] * 17, copies=1)
            for form in ("wide", "compact"):
                set_plan(monkeypatch, form, dense=False)
                csr = copies > 1
                for ne in (False, True):
                    run_hows(plb, lk, lv, rk, rv, form, csr=csr or ne, nulls_equal=ne, what=f"{form} {dtype} i64::MIN x{copies}")


# ------------------------------------------------------------------------------------------------ key dtypes, join types
def _shapes(rng, dtype, nb):
    rk, rv = jk.keys(rng, dtype, nb, "k", k=2, nulls=0.05)
    for nl in (2 * nb + 3, nb // 3, nb):                # left longer / right longer / equal (right probes)
        lk, lv = jk.probe(rng, rk, nl, nulls=0.05)
        yield lk, lv, rk, rv


@pytest.mark.parametrize("form", ["wide", "compact"])
@pytest.mark.parametrize("dtype", jk.DTYPES)
def test_key_dtypes(plb, monkeypatch, dtype, form):
    """Every accepted key dtype (8 / 16-bit keys are widened to UInt32 bit patterns first), unique and duplicate builds,
    inner with either side longer and with a tie, left, semi, anti and full, maintain_order."""
    rng = np.random.default_rng(jk.DTYPES.index(dtype) * 2 + (form == "compact"))
    nb = 200 if np.dtype(dtype).itemsize == 1 else 3000
    rk, rv = jk.keys(rng, dtype, nb, "unique", nulls=0.05)
    lk, lv = jk.probe(rng, rk, 2 * nb + 1, nulls=0.05)
    set_plan(monkeypatch, form, dense=False)
    run_hows(plb, lk, lv, rk, rv, form, what=f"{form} {dtype} unique")
    set_plan(monkeypatch, form, dense=False, fused=False)
    run_hows(plb, lk, lv, rk, rv, form, fused=False, hows=("inner", "left"), what=f"{form} {dtype} unique two-pass")
    set_plan(monkeypatch, form, dense=False)
    for lk, lv, rk, rv in _shapes(rng, dtype, nb):
        for how in ("inner", "left", "full"):
            orders = {"inner": INNER_ORDERS, "left": LEFT_ORDERS, "full": ("none",)}[how]
            for order in orders:
                prof = run(plb, lk, lv, rk, rv, how, order=order, what=f"{form} {dtype} nl={lk.size}")
                assert BUILD_LABEL[form] in prof and "k7_dense_build" not in prof, sorted(prof)
        for how in ("semi", "anti"):
            run(plb, lk, lv, rk, rv, how, what=f"{form} {dtype} nl={lk.size}")


@pytest.mark.parametrize("form", ["dense", "wide", "compact"])
def test_maintain_order_sort_width(plb, monkeypatch, form):
    """maintain_order on an inner join sorts the indices of one side on bits_for(len) bits, in 8-bit radix passes, so a
    sort one bit too narrow only shows when len needs 17 bits: 2^16 <= len < 2^17 on the sorted side."""
    set_plan(monkeypatch, form, dense=form == "dense")
    rng = np.random.default_rng(17)
    n_short, n_long = 100_003, 250_001
    rk, rv = jk.keys(rng, "int64", n_short, "unique", nulls=0.01, dense=2 * n_short if form == "dense" else None)
    lk, lv = jk.probe(rng, rk, n_long, hit=0.8, nulls=0.01)
    for order in INNER_ORDERS[1:]:
        assert_plan(run(plb, lk, lv, rk, rv, "inner", order=order, what=f"{form} sort width"), form, "fused")     # sorts right idx
        assert_plan(run(plb, rk, rv, lk, lv, "inner", order=order, what=f"{form} sort width swapped"), form, "fused")   # sorts left idx


# ------------------------------------------------------------------------------------------------ multi-column keys
@pytest.mark.parametrize("how", HOWS)
def test_multi_column_keys(plb, how):
    """bl_hash_join_keys against oracle.hash_join_multi: two Int32 columns (the pair (0, i32::MIN) packs to exactly
    i64::MIN, the WIDE empty marker), one nullable UInt64 key (id compression when nulls are part of the key), and
    (Int64, Float32, UInt8) with validity on some columns."""
    rng = np.random.default_rng(13 + HOWS.index(how))
    nl, nr = 9000, 4000

    def pick(pool, n):
        return pool[rng.integers(0, pool.size, n)]

    i32 = jk.distinct(rng, "int32", 40)
    a = [pick(i32, nl), pick(i32, nr)]
    b = [pick(i32, nl), pick(i32, nr)]
    for x, y in zip(a, b):                   # (0, i32::MIN) on both sides
        idx = rng.choice(x.size, 25, replace=False)
        x[idx], y[idx] = 0, np.iinfo(np.int32).min
    u64 = jk.distinct(rng, "uint64", 300)
    c = [pick(u64, nl), pick(u64, nr)]
    cv = [jk.null_mask(rng, nl, 15), jk.null_mask(rng, nr, 15)]
    i64, f32, u8 = jk.distinct(rng, "int64", 12), jk.distinct(rng, "float32", 8), jk.distinct(rng, "uint8", 5)
    f32 = np.concatenate([f32, np.array([np.nan, -0.0, 0.0], np.float32), np.array([0xFFC00001], np.uint32).view(np.float32)])
    d = [[pick(i64, n), pick(f32, n), pick(u8, n)] for n in (nl, nr)]
    dv = [[jk.null_mask(rng, n, 0.03), None, jk.null_mask(rng, n, 0.03)] for n in (nl, nr)]
    cases = (("i32_i32", [a[0], b[0]], [a[1], b[1]], None, None),
             ("nullable_u64", [c[0]], [c[1]], [cv[0]], [cv[1]]),
             ("i64_f32_u8", d[0], d[1], dv[0], dv[1]))
    for name, L, R, LV, RV in cases:
        for ne in (False, True):
            LV_, RV_ = LV or [None] * len(L), RV or [None] * len(R)
            got, prof = profiled(plb, lambda: plb.hash_join_keys([plb.Column(k, v) for k, v in zip(L, LV_)], [plb.Column(k, v) for k, v in zip(R, RV_)], how, ne, "none"))
            exp = oracle.hash_join_multi(L, R, LV_, RV_, how, ne, "none", 8)
            check_join(got, exp, f"{name} {how} nulls_equal={ne}")
            # two Int32 columns pack side by side; a nullable UInt64 key under nulls_equal, and the nullable Int64
            # column, are replaced by their group ids first
            compressed = name == "i64_f32_u8" or (name == "nullable_u64" and ne)
            assert ("k5_lookup_first" in prof) == compressed, (name, ne, sorted(prof))


# ------------------------------------------------------------------------------------------------ device inputs, payloads
@pytest.mark.parametrize("form", ["dense", "wide", "compact"])
def test_device_resident_keys(plb, monkeypatch, form):
    """Keys already on the device and tuples returned on the device, one case per form."""
    set_plan(monkeypatch, form, dense=form == "dense")
    rng = np.random.default_rng(14)
    nb = 100_003
    rk, rv = jk.keys(rng, "int64", nb, "unique", nulls=0.01, dense=2 * nb if form == "dense" else None)
    lk, lv = jk.probe(rng, rk, 3 * nb, nulls=0.01, dense_edges=form == "dense")
    for how in ("inner", "left", "full"):
        prof = run(plb, lk, lv, rk, rv, how, device=True, what=f"{form} device")
        assert_plan(prof, form, "fused", what=f"{form} device {how}")


def test_join_payloads(plb, monkeypatch):
    """plb.join gathers payloads on both sides at the join tuples; a missing side comes back as null rows."""
    rng = np.random.default_rng(15)
    rk, rv = jk.keys(rng, "uint32", 40_000, "runs", k=4, nulls=0.02)
    lk, lv = jk.probe(rng, rk, 90_001, nulls=0.02)
    lp = (rng.normal(size=lk.size), rng.random(lk.size) > 0.1)
    rp = (rng.integers(-2**63, 2**63 - 1, rk.size, dtype=np.int64, endpoint=True), None)
    for form in ("wide", "compact"):
        set_plan(monkeypatch, form, dense=False)
        for how in ("inner", "left", "full"):
            (lo,), (ro,) = plb.join(plb.Column(lk, lv), plb.Column(rk, rv), [plb.Column(*lp)], [plb.Column(*rp)], how)
            eli, eri = oracle.hash_join(lk, rk, lv, rv, how, False, "none", 8)
            for (vals, valid), e, (pv, pvalid), side in ((lo, eli, lp, "left"), (ro, eri, rp, "right")):
                hit = e != IDX_NULL
                ev = hit & (np.ones(pv.size, bool) if pvalid is None else pvalid)[np.where(hit, e, 0)]
                assert np.array_equal(np.ones(e.size, bool) if valid is None else valid, ev), (form, how, side)
                assert np.array_equal(vals[ev], pv[e[ev]]), (form, how, side)


# ------------------------------------------------------------------------------------------------ result-size guard
def test_result_size_guard(plb, monkeypatch):
    """70 000 x 70 000 rows of one key are 4.9e9 tuples, past the 32-bit index: the count after pass 1 raises before any
    output is allocated, and the next join on the same context is right."""
    set_plan(monkeypatch, "wide", dense=False)
    one = np.full(70_000, -7, np.int64)
    for how in ("inner", "full"):
        with pytest.raises(plb.B200Error) as e:
            plb.hash_join(one, one, how)
        assert e.value.status == 4, str(e.value)
    rng = np.random.default_rng(16)
    rk, rv = jk.keys(rng, "int64", 50_000, "k", k=3, nulls=0.01)
    lk, lv = jk.probe(rng, rk, 120_000, nulls=0.01)
    for how in ("inner", "full"):
        assert_plan(run(plb, lk, lv, rk, rv, how, what="after the guard"), "wide", "two_pass", csr=True)
