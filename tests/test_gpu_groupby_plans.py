"""GPU tests of the fused group_by (K5) on every plan against the exact restatement in tests/groupby_ref.py, over the
full value range of every dtype it accepts and past its grid caps.

Each test selects one plan with the knobs of groupby.cu / groupby_radix.cu (read per call) and, where the plan has a
kernel name of its own, proves it ran with the launch profile.  Integers, counts and validity must match bit for bit;
float sums and means stay within the bound of groupby_ref (0 for exact-summable groups); float min / max are exact.
Every case mixes one group of 2^20 rows (a lost row is visible in its float sum), many singleton groups and the
dedicated groups of groupby_ref.SPECIAL_GROUPS (all NaN, all null, +inf with -inf, subnormals, cancellation, the
dtype's MIN and MAX, a singleton); keys include i64::MIN (the bit pattern of an empty slot), a null key, UInt64 keys
with the top bit set and float keys with NaN payloads and -0.0.

Sizes.  The caps come from grid_for (common.cuh) with SM = device_info()["sm_count"] (132 on an H100 SXM):
  k_gb_consume         24*SM CTAs x 256 threads x 2 rows: the grid-stride loop runs twice from 12288*SM rows
  k_gb_consume_lean    48*SM CTAs: from 24576*SM rows
  k_gb_consume_hot / _smem   up to 4*SM CTAs of 512 threads x 2 rows: from 4096*SM rows
N_LOOP = 24576*SM + 4097 passes every one of them with a ragged tail.  The large float cases use exact-summable values
(integers times 2^-20), so their reference stays vectorised.
"""
import numpy as np
import pytest

import groupby_ref as ref

pytestmark = pytest.mark.gpu

BIG = 1 << 20
NO_PLAN_KNOBS = {"BL_K5_HOTKEYS": "0", "BL_K5_RADIX": "0"}     # no heavy-hitter list, no partitioned plan


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as m
    m.init()
    return m


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


def n_loop(sm):
    return 24576 * sm + 4097


def _env(monkeypatch, knobs):
    for k, v in knobs.items():
        monkeypatch.setenv(k, v)


class Call:
    """One group_by_agg call and its check.  aggs: [(kind, column | None)], column = (values, valid|None); the same
    tuple object is the same value column (one column slot on the device)."""

    def __init__(self, plb, keys, key_valid, aggs, maintain_order=False, device=False):
        self.plb = plb
        objs, keep = {}, []
        for _, c in aggs:
            if c is not None and id(c) not in objs:
                if device:
                    d = plb.to_device(c[0], c[1])
                    keep.append(d)
                    objs[id(c)] = d.view()
                else:
                    objs[id(c)] = plb.Column(c[0], c[1])
        if device:
            dk = plb.to_device(keys, key_valid)
            keep.append(dk)
            kcol = dk.view()
        else:
            kcol = plb.Column(keys, key_valid)
        ok, outs = plb.group_by_agg(kcol, [(k, None if c is None else objs[id(c)]) for k, c in aggs], maintain_order,
                                    location=plb.DEVICE if device else plb.HOST)
        if device:
            ok, outs = ok.to_numpy(), [o.to_numpy() for o in outs]
        self.got = (ok, outs)
        self.args = (keys, key_valid, aggs, maintain_order)

    def check(self, g=None, what="", f32_kahan=False):
        return check_result(self.got, *self.args, g=g, what=what, f32_kahan=f32_kahan)


def check_result(got, keys, key_valid, aggs, maintain_order, g=None, what="", f32_kahan=False):
    """got = ((keys, valid), [(values, valid)]) of a group_by; compared with groupby_ref (unordered: after sorting both
    by key).  f32_kahan: Float32 sums are Kahan sums in f32 (the deterministic path) -> ref.kahan32 bound."""
    (gk, gkv), outs = got
    (ek, ekv), exps, g = ref.expect(keys, key_valid, [(k, *(c if c is not None else (None, None))) for k, c in aggs], maintain_order, g=g)
    if not maintain_order:
        o = ref.canonical_order(gk, gkv)
        gk, gkv = gk[o], (None if gkv is None else gkv[o])
        outs = [(v[o], None if m is None else m[o]) for v, m in outs]
    err = ref.check(gk, gkv, (ek, ekv))
    assert err is None, f"{what} keys: {err}"
    assert len(outs) == len(aggs), (len(outs), len(aggs))
    for (kind, c), exp, (v, m) in zip(aggs, exps, outs):
        if f32_kahan and kind == "sum" and c is not None and c[0].dtype == np.float32:
            exp = ref.kahan32(exp)
        err = ref.check(v, m, exp)
        dt = None if c is None else c[0].dtype
        assert err is None, f"{what} {kind}({dt}): {err}"
    return g


def run(plb, keys, key_valid, aggs, maintain_order=False, device=False, g=None, what=""):
    return Call(plb, keys, key_valid, aggs, maintain_order, device).check(g, what)


def profiled(plb, fn):
    plb.profile_reset()
    plb.profile_enable(True)
    try:
        r = fn()
    finally:
        prof = plb.profile()
        plb.profile_enable(False)
    return r, prof


def value_cols(case, rng, dtypes, nullable, exact):
    """[(dtype, sum/mean column, min/max/count column)]: floats get a magnitude-capped (or exact-summable) column for
    sum / mean and an uncapped one for the rest; integer columns serve every aggregation."""
    out = []
    for dt in dtypes:
        if np.dtype(dt).kind == "f":
            out.append((dt, case.values(rng, dt, for_sum=True, exact=exact, nullable=nullable), case.values(rng, dt, nullable=nullable)))
        else:
            c = case.values(rng, dt, nullable=nullable)
            out.append((dt, c, c))
    return out


def full_aggs(s, mm):
    return [("sum", s), ("mean", s), ("min", mm), ("max", mm), ("count", mm), ("len", None)]


def big_case(rng, n, key_dtype="int64", *, singletons=50_000, groups=200_000, null_rows=1000, big_key=None, **kw):
    rest = n - BIG - singletons - null_rows - sum(ref.SPECIAL_ROWS.values())
    return ref.Case(rng, key_dtype, big=BIG, singletons=singletons, groups=groups, rest=rest, null_rows=null_rows, big_key=big_key, **kw)


# ------------------------------------------------------------------ general k_gb_consume
GENERAL = {"pairs1": {}, "pairs2": {"BL_K5_PAIRS": "2"}, "aos": {"BL_K5_SOA": "0"},
           "hint1": {"BL_K5_HINT": "1"}, "hint2": {"BL_K5_HINT": "2"}, "hint3": {"BL_K5_HINT": "3"}}


@pytest.mark.parametrize("variant", list(GENERAL))
def test_general_plan(plb, sm, monkeypatch, variant):
    """k_gb_consume (PAIRS 1 / 2, word-major / AoS entries, L2 policy / L1 key-load hints): maintain_order needs the
    first-row word, which rules out the lean kernel and the pair layout (groupby.cu note_batch_shape)."""
    _env(monkeypatch, {**NO_PLAN_KNOBS, "BL_K5_SMEM": "0", **GENERAL[variant]})
    rng = np.random.default_rng(len(variant))
    case = big_case(rng, n_loop(sm), big_key=np.iinfo(np.int64).min)
    dtypes = ref.VALUE_DTYPES + (ref.SMALL_DTYPES if variant == "pairs1" else ())
    g = None
    for nullable in (False, True):
        for dt, s, mm in value_cols(case, rng, dtypes, nullable, exact=True):
            c, prof = profiled(plb, lambda: Call(plb, case.keys, case.key_valid, full_aggs(s, mm), True))
            assert "k5_groupby_agg" in prof and "k5_groupby_agg_smem" not in prof and "k5_groupby_agg_hot" not in prof, sorted(prof)
            g = c.check(g, f"{variant} nullable={nullable}")


@pytest.mark.parametrize("key_dtype", ["int64", "uint64", "int32", "uint32", "float64", "float32", "int16", "uint8"])
def test_key_dtypes(plb, monkeypatch, key_dtype):
    """Every key dtype on the default plan, ordered and not: NaN payloads and +-0.0 are one key each, the null key is
    one group, UInt64 keys with the top bit set and i64::MIN stay distinct."""
    rng = np.random.default_rng(7 + len(key_dtype))
    size = np.dtype(key_dtype).itemsize
    singletons, groups = {1: (40, 100), 2: (10_000, 20_000)}.get(size, (20_000, 50_000))
    case = ref.Case(rng, key_dtype, big=BIG, singletons=singletons, groups=groups, rest=300_000, null_rows=500)
    cols = value_cols(case, rng, ("int64", "uint64", "float64", "float32"), True, exact=True)
    for maintain_order in (True, False):
        g = None
        for dt, s, mm in cols:
            g = run(plb, case.keys, case.key_valid, full_aggs(s, mm), maintain_order, g=g, what=f"{key_dtype} order={maintain_order}")


# ------------------------------------------------------------------ lean k_gb_consume_lean
@pytest.mark.parametrize("key_dtype", ["int64", "uint64"])
@pytest.mark.parametrize("nulls", [False, True])
def test_lean_plan(plb, sm, monkeypatch, key_dtype, nulls):
    """k_gb_consume_lean shares the profile name k5_groupby_agg with the general kernel, so the case is pinned by the
    kernel's preconditions (groupby.cu launch_consume and note_batch_shape): an Int64 / UInt64 key, at most three
    8-byte value columns with at most two accumulator words each, an integer sum and len, unordered, no L2 hint, and no
    heavy-hitter list or shared-memory table (hundreds of thousands of groups, BL_K5_HOTKEYS=0).  The same case then
    runs under BL_K5_LEAN=0 (the general bulk kernel on the same pair layout)."""
    _env(monkeypatch, NO_PLAN_KNOBS)
    rng = np.random.default_rng(31 + nulls)
    kmin = np.iinfo(np.int64).min if key_dtype == "int64" else np.uint64(1 << 63)
    case = big_case(rng, n_loop(sm), key_dtype, null_rows=1000 if nulls else 0, big_key=kmin, groups=400_000)
    a = case.values(rng, "int64", nullable=nulls)
    b = case.values(rng, "uint64", nullable=nulls)
    c = case.values(rng, "float64", for_sum=True, exact=True, nullable=nulls)
    if nulls:      # a nullable column's min / max / mean take a null-count word too: two words per column at most
        aggs = [("sum", a), ("count", a), ("len", None), ("mean", b), ("sum", c)]
    else:
        aggs = [("sum", a), ("min", a), ("len", None), ("mean", b), ("max", b), ("sum", c), ("mean", c)]
    g = None
    for lean in ("1", "0"):
        monkeypatch.setenv("BL_K5_LEAN", lean)
        c_, prof = profiled(plb, lambda: Call(plb, case.keys, case.key_valid, aggs, False, device=True))
        assert "k5_groupby_agg" in prof and "k5_groupby_agg_smem" not in prof and "k5_groupby_agg_hot" not in prof, sorted(prof)
        g = c_.check(g, f"lean={lean}")


# ------------------------------------------------------------------ general bulk (pair layout)
@pytest.mark.parametrize("lanes", ["20", "32"])
def test_general_bulk(plb, sm, monkeypatch, lanes):
    """BL_K5_BULK=2: the pair layout and the TMA bulk reduce of {len, sum} cells in the general kernel.  20 lanes: the
    lean kernel needs all 32; 32 lanes with maintain_order (which the lean kernel does not take).  Every call carries an
    Int64 sum (the paired word) and len."""
    _env(monkeypatch, {**NO_PLAN_KNOBS, "BL_K5_BULK": "2", "BL_K5_BULK_LANES": lanes, "BL_K5_SMEM": "0"})
    order = lanes == "32"
    rng = np.random.default_rng(int(lanes))
    case = big_case(rng, n_loop(sm))
    pair = case.values(rng, "int64")
    g = None
    for nullable in (False, True):
        for dt, s, mm in value_cols(case, rng, ref.VALUE_DTYPES, nullable, exact=True):
            aggs = [("sum", pair), ("len", None)] + full_aggs(s, mm)[:-1]
            c, prof = profiled(plb, lambda: Call(plb, case.keys, case.key_valid, aggs, order))
            assert "k5_groupby_agg" in prof, sorted(prof)
            g = c.check(g, f"bulk lanes={lanes} nullable={nullable}")


# ------------------------------------------------------------------ CTA-private shared-memory tables
SMEM = ["few_fast", "few_slow", "k1000_fast", "k1000_slow"]


@pytest.mark.parametrize("shape", SMEM)
def test_smem_plan(plb, sm, monkeypatch, shape):
    """k_gb_consume_smem: a handful of groups (a 16/32-slot table, 32 replicas per CTA) or about 1000 (a 2048-slot table,
    one replica at a 4-word stride: at most two accumulator words per call).  FAST = every value column 8 bytes wide and
    without nulls; the slow shapes use 4-byte, 8/16-bit and nullable columns."""
    _env(monkeypatch, NO_PLAN_KNOBS)
    rng = np.random.default_rng(len(shape) * 3)
    few = shape.startswith("few")
    fast = shape.endswith("fast")
    n = n_loop(sm)
    case = ref.Case(rng, "int64", big=BIG, singletons=20, groups=3 if few else 1000, rest=n - BIG - 100, null_rows=0 if fast else 50,
                    big_key=np.iinfo(np.int64).min)
    dtypes = ("int64", "uint64", "float64") if fast else ("int32", "uint32", "float32") + ref.SMALL_DTYPES
    nulls = (False,) if fast else (False, True)
    g = None
    for nullable in nulls:
        for dt, s, mm in value_cols(case, rng, dtypes, nullable, exact=True):
            if few:
                calls = [full_aggs(s, mm)]
            elif nullable:
                calls = [[("mean", s)], [("min", mm)], [("max", mm)], [("sum", s), ("count", mm), ("len", None)]]
            else:
                calls = [[("sum", s), ("mean", s)], [("min", mm), ("max", mm), ("count", mm), ("len", None)]]
            for aggs in calls:
                c, prof = profiled(plb, lambda: Call(plb, case.keys, case.key_valid, aggs, False))
                assert "k5_groupby_agg_smem" in prof, (shape, dt, sorted(prof))
                g = c.check(g, f"{shape} {dt} nullable={nullable}")


@pytest.mark.parametrize("mode", ["tail", "hot_table"])
def test_smem_overflow(plb, sm, monkeypatch, mode):
    """Keys the CTA-private table cannot take fall through to the global table: 'tail' = a few sampled groups plus
    600 singleton keys, of which the sample sees about a dozen (a table of a few hundred slots); 'hot_table' =
    BL_K5_HOT=64 (the shared-memory kernel with 64 slots on 100 000 groups)."""
    _env(monkeypatch, {**NO_PLAN_KNOBS, **({"BL_K5_HOT": "64"} if mode == "hot_table" else {})})
    rng = np.random.default_rng(77 + len(mode))
    n = n_loop(sm)
    if mode == "tail":
        case = ref.Case(rng, "int64", big=BIG, singletons=600, groups=4, rest=n - BIG - 1000, null_rows=300)
    else:
        case = big_case(rng, n, singletons=20_000, groups=100_000, null_rows=300)
    g = None
    for dt, s, mm in value_cols(case, rng, ("int64", "uint64", "float64", "float32"), True, exact=True):
        c, prof = profiled(plb, lambda: Call(plb, case.keys, case.key_valid, full_aggs(s, mm), False))
        assert "k5_groupby_agg_smem" in prof, sorted(prof)
        g = c.check(g, f"{mode} {dt}")


# ------------------------------------------------------------------ heavy hitters
@pytest.mark.parametrize("hot_key", ["null", "min"])
def test_heavy_hitters(plb, sm, monkeypatch, hot_key):
    """k_gb_consume_hot: Zipf keys with BL_K5_HOT_ROWS=0 (every key seen 12 times in the sample is hot), plus a hot null
    key or a hot i64::MIN key of 2^20 rows.  The warp-private rows combine lanes with hot_combine and merge with
    gb_merge_row: UInt64 values >= 2^63 and negative Int64 values reach both."""
    _env(monkeypatch, {"BL_K5_HOT_ROWS": "0", "BL_K5_RADIX": "0"})
    rng = np.random.default_rng(5 + len(hot_key))
    n = n_loop(sm)
    if hot_key == "null":
        case = ref.Case(rng, "int64", big=0, singletons=10_000, groups=200_000, rest=n - BIG - 10_100, null_rows=BIG, zipf=1.3)
    else:
        case = ref.Case(rng, "int64", big=BIG, singletons=10_000, groups=200_000, rest=n - BIG - 10_100, zipf=1.3,
                        big_key=np.iinfo(np.int64).min)
    g = None
    for nullable in (False, True):
        for dt, s, mm in value_cols(case, rng, ref.VALUE_DTYPES, nullable, exact=True):
            c, prof = profiled(plb, lambda: Call(plb, case.keys, case.key_valid, full_aggs(s, mm), False))
            assert "k5_groupby_agg_hot" in prof, sorted(prof)
            g = c.check(g, f"hot {hot_key} {dt} nullable={nullable}")


# ------------------------------------------------------------------ multipass beyond L2
def test_multipass_beyond_l2(plb, sm, monkeypatch):
    """A table larger than the L2 budget (0.55 x l2_bytes) is filled in slot-range passes, one k_gb_consume launch
    each (groupby.cu launch_batch: pass_bits).  With 32-byte entries (at most two words) the planner keeps the
    smallest power-of-two capacity c* whose table exceeds the budget when the sampled estimate is about 0.6 c*
    groups: two passes."""
    _env(monkeypatch, NO_PLAN_KNOBS)
    info = plb.device_info()
    budget = 0.55 * info["l2_bytes"]
    c_star = 1024
    while c_star * 32 <= budget:
        c_star *= 2
    groups = int(0.6 * c_star)
    rng = np.random.default_rng(99)
    n = max(n_loop(sm), BIG + 4 * groups)
    case = ref.Case(rng, "int64", big=BIG, singletons=0, groups=groups, rest=n - BIG, null_rows=200)
    g = None
    for dt, s, mm in value_cols(case, rng, ref.VALUE_DTYPES, False, exact=True):
        for aggs in ([("sum", s), ("mean", s), ("len", None)], [("min", mm), ("max", mm), ("count", mm)]):
            c, prof = profiled(plb, lambda: Call(plb, case.keys, case.key_valid, aggs, False))
            assert prof.get("k5_groupby_agg", {}).get("launches", 0) >= 2, (c_star, groups, prof)
            g = c.check(g, f"multipass {dt}")


# ------------------------------------------------------------------ partitioned K5r
RADIX = {"bulk_i32": 0, "bulk_4col": 0, "many_buckets": 1, "small_ints": 0}


@pytest.mark.parametrize("shape", list(RADIX))
def test_radix_plan(plb, sm, monkeypatch, capfd, shape):
    """K5r (groupby_radix.cu), forced with BL_K5_RADIX=2 on >= 2^20 rows without nulls: 1 to 4 value columns of 4 and
    8 bytes; at most 512 buckets (the bulk store path) for a few thousand groups, more for about a million.  The
    BL_K5_DEBUG line reports the path taken."""
    _env(monkeypatch, {"BL_K5_RADIX": "2", "BL_K5_HOTKEYS": "0", "BL_K5_DEBUG": "1"})
    rng = np.random.default_rng(len(shape) * 5)
    n = n_loop(sm)
    many = RADIX[shape]
    case = ref.Case(rng, "int64", big=BIG, singletons=100_000 if many else 1000, groups=900_000 if many else 3000,
                    rest=n - BIG - (100_100 if many else 1100), big_key=np.iinfo(np.int64).min)
    if shape == "bulk_i32":
        cols = value_cols(case, rng, ("int32",), False, exact=True)
        calls = [full_aggs(cols[0][1], cols[0][2])]
    elif shape == "small_ints":
        cols = value_cols(case, rng, ref.SMALL_DTYPES, False, exact=True)
        calls = [full_aggs(c[1], c[2]) for c in cols]
    else:
        cols = value_cols(case, rng, ("int64", "uint64", "float64", "float32") if shape == "bulk_4col" else ("int64", "uint64"), False, exact=True)
        calls = [[("sum", c[1]) for c in cols] + [("mean", c[1]) for c in cols] + [("len", None)],
                 [("min", c[2]) for c in cols] + [("max", c[2]) for c in cols] + [("count", cols[0][2])]]
    g = None
    for aggs in calls:
        capfd.readouterr()
        c, prof = profiled(plb, lambda: Call(plb, case.keys, None, aggs, False))
        err = capfd.readouterr().err
        assert "k5r_aggregate" in prof, sorted(prof)
        line = [ln for ln in err.splitlines() if ln.startswith("[k5r]")][-1]
        assert f"bulk={0 if many else 1}" in line and "status=0" in line, line
        g = c.check(g, f"radix {shape}")


# ------------------------------------------------------------------ deterministic
def test_deterministic_plan(plb, monkeypatch):
    """set_deterministic(True): the reference's own order (groupby_exact.cu k5x_fold_groups) over full-range values."""
    rng = np.random.default_rng(123)
    case = ref.Case(rng, "int64", big=BIG, singletons=20_000, groups=20_000, rest=200_000, null_rows=500)
    plb.set_deterministic(True)
    try:
        g = None
        for nullable in (False, True):
            for dt, s, mm in value_cols(case, rng, ref.VALUE_DTYPES, nullable, exact=False):
                c, prof = profiled(plb, lambda: Call(plb, case.keys, case.key_valid, full_aggs(s, mm), True))
                assert "k5x_fold_groups" in prof, sorted(prof)
                g = c.check(g, f"deterministic {dt} nullable={nullable}", f32_kahan=True)
    finally:
        plb.set_deterministic(False)


# ------------------------------------------------------------------ streaming, rehash, export / merge, P2P window
def test_streaming_rehash_merge(plb):
    """GroupBy.consume in three batches whose new keys force the table to grow (k5_rehash), export_partials(2) +
    merge_partials (k5_merge_partials) into a fresh state, the synchronous P2P export (export_partials_p2p) merged back
    with merge_partials, and the P2P window merge into our own window."""
    rng = np.random.default_rng(2024)
    case = ref.Case(rng, "int64", big=BIG, singletons=20_000, groups=100_000, rest=600_000, big_key=np.iinfo(np.int64).min)
    # batches: the first holds a few hundred keys, so the table is sized small; the next two bring ~100 000 new keys
    n = case.n
    cuts = (0, 2000, 400_000, n)
    a = case.values(rng, "int64")
    b = case.values(rng, "uint64")
    f = case.values(rng, "float64", for_sum=True, exact=True)
    spec = [("sum", "int64"), ("min", "int64"), ("max", "int64"), ("min", "uint64"), ("max", "uint64"), ("mean", "uint64"),
            ("sum", "float64"), ("len", None)]
    cols = [a, a, a, b, b, b, f, None]
    aggs = [(k, c) for (k, _), c in zip(spec, cols)]
    nn = [False] * len(spec)

    def check(res, tag):
        check_result(res, case.keys, None, aggs, False, what=tag)

    s = plb.GroupBy(np.int64, spec, nullable=nn)
    def stream():
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            s.consume(case.keys[lo:hi], [None if c is None else c[0][lo:hi] for c in cols], row_base=lo)
        return s.finish()
    res, prof = profiled(plb, stream)
    assert "k5_rehash" in prof, sorted(prof)
    check(res, "stream")
    t = plb.GroupBy(np.int64, spec, nullable=nn)
    t.consume(case.keys, [None if c is None else c[0] for c in cols])
    ptr, rw, offs = t.export_partials(2)
    m = plb.GroupBy(np.int64, spec, nullable=nn)
    def merge():
        for p in range(2):
            m.merge_partials(ptr + int(offs[p]) * rw * 8, int(offs[p + 1] - offs[p]))
        return m.finish()
    res, prof = profiled(plb, merge)
    plb.dev_free(ptr)
    assert "k5_merge_partials" in prof, sorted(prof)
    check(res, "export + merge")
    groups = int(offs[-1])
    rows_per_src = groups + 1024
    # synchronous P2P export as rank 1 of 2: partition p's rows land in region 1 of window p; merge_partials reads both
    wins = [plb.Window(2 * rows_per_src * rw * 8) for _ in range(2)]
    try:
        rw_p2p, sent = t.export_partials_p2p([w.ptr for w in wins], 1, rows_per_src)
        assert rw_p2p == rw and sent.tolist() == np.diff(offs).tolist(), (rw_p2p, rw, sent, offs)
        q = plb.GroupBy(np.int64, spec, nullable=nn)
        for w, c in zip(wins, sent):
            q.merge_partials(w.ptr + rows_per_src * rw * 8, int(c))
        check(q.finish(), "p2p export + merge")
        del q
    finally:
        for w in wins:
            w.destroy()
    win = plb.Window(1024 + rows_per_src * rw * 8)
    try:
        t.export_partials_p2p_async([win.ptr], 0, rows_per_src, 1)
        w = plb.GroupBy(np.int64, spec, expected_groups=groups + 1000, nullable=nn)
        w.merge_window_async(win.ptr, 1, rows_per_src, 1)
        check(w.finish(), "p2p window")
        del w
    finally:
        win.destroy()
    del s, t, m


# ------------------------------------------------------------------ several key columns
@pytest.mark.parametrize("shape", ["packed", "unpacked"])
def test_multi_keys(plb, shape):
    """group_by_agg_keys: narrow keys that pack into one 64-bit key (Int32 + nullable UInt8), and wide ones that are
    replaced by their group ids first (Int64 + nullable Float64 with NaN payloads and -0.0)."""
    rng = np.random.default_rng(len(shape))
    n = 600_000
    if shape == "packed":
        k1 = rng.integers(-3, 3, n).astype(np.int32); k1[:2] = [np.iinfo(np.int32).min, np.iinfo(np.int32).max]
        k2 = rng.integers(0, 256, n).astype(np.uint8)
    else:
        k1 = rng.integers(-5, 5, n).astype(np.int64) * (2 ** 62 // 5); k1[0] = np.iinfo(np.int64).min
        k2 = rng.choice(np.array([0.0, -0.0, np.nan, -np.nan, 1.5, np.inf, 5e-324]), n)
    v2 = ref.validity(rng, n, 0.05)
    case = ref.Case(rng, "int64", big=0, groups=10, rest=n, specials=False)
    cols = value_cols(case, rng, ("int64", "uint64", "float64", "float32"), True, exact=False)
    g = ref.group_multi([k1, k2], [None, v2])
    kout = [(k1[g.first], None), (k2[g.first], v2[g.first])]
    for dt, s, mm in cols:
        aggs = full_aggs(s, mm)
        kouts, outs = plb.group_by_agg_keys([plb.Column(k1), plb.Column(k2, v2)], [(k, None if c is None else plb.Column(*c)) for k, c in aggs], True)
        for (gk, gkv), (ek, ekv) in zip(kouts, kout):
            err = ref.check(gk, gkv, (ek, ekv))
            assert err is None, f"{shape} keys: {err}"
        for (kind, c), (v, m) in zip(aggs, outs):
            exp = ref.aggregate(kind, None if c is None else c[0], None if c is None else c[1], g)
            err = ref.check(v, m, exp)
            assert err is None, f"{shape} {kind}({dt}): {err}"


# ------------------------------------------------------------------ pipelined host path
def test_pipelined_host_path(plb):
    """bl_groupby_agg copies host inputs of >= 2^22 rows without nulls in 8M-row chunks overlapped with K5
    (cabi.cu, GroupByState::consume_pipelined): 2^23 + 2^22 + 4097 rows = two chunks with a ragged tail.  The sample
    comes from the first chunk only; the 200 000 keys that first appear in the second chunk test that estimate."""
    rng = np.random.default_rng(8)
    n = (1 << 23) + (1 << 22) + 4097
    case = ref.Case(rng, "int64", big=BIG, singletons=300_000, groups=500_000, rest=n - BIG - 300_000 - sum(ref.SPECIAL_ROWS.values()),
                    big_key=np.iinfo(np.int64).min)
    late = np.arange(n - 200_000, n)
    case.keys[late] = np.int64(2 ** 62) + late      # keys only the last chunk holds
    g = None
    for dtypes in (("int64", "uint64", "float64"), ("int32", "uint32", "float32")):
        cols = value_cols(case, rng, dtypes, False, exact=True)
        aggs = [a for _, s, mm in cols for a in full_aggs(s, mm)[:-1]] + [("len", None)]
        g = run(plb, case.keys, None, aggs, False, g=g, what=f"pipelined {dtypes}")


# ------------------------------------------------------------------ boundaries
def _status(plb, fn):
    with pytest.raises(plb.B200Error) as e:
        fn()
    return e.value.status


def test_boundaries(plb):
    """8 value columns work and a ninth is BL_ERR_UNSUPPORTED; 14 accumulator words work and a fifteenth is too; the
    library answers the next call correctly after each; 20 aggregations (many counts over non-null columns, which take
    no word) cross the 16-aggregate re-launch of the finalize kernel; empty input, one row and all keys null."""
    rng = np.random.default_rng(4)
    case = ref.Case(rng, "int64", big=5000, singletons=500, groups=2000, rest=40_000, null_rows=20)
    cols = [case.values(rng, ref.VALUE_DTYPES[i % 6], for_sum=True, nullable=False) for i in range(9)]
    eight = [("sum", c) for c in cols[:8]] + [("len", None)]
    run(plb, case.keys, case.key_valid, eight, what="8 columns")
    assert _status(plb, lambda: Call(plb, case.keys, case.key_valid, [("sum", c) for c in cols], False)) == 4
    run(plb, case.keys, case.key_valid, eight, what="after 9 columns")
    c0, c1 = cols[0], cols[1]
    m0 = case.values(rng, "int64")
    f0 = case.values(rng, "float64", for_sum=True)
    fourteen = [("sum", c0), ("min", c0), ("max", c0), ("mean", c0), ("sum", c1), ("min", c1), ("max", c1), ("mean", c1),
                ("min", m0), ("max", m0), ("sum", m0), ("min", f0), ("max", f0), ("mean", f0)]
    run(plb, case.keys, case.key_valid, fourteen, what="14 words")
    assert _status(plb, lambda: Call(plb, case.keys, case.key_valid, fourteen + [("sum", f0)], False)) == 4
    run(plb, case.keys, case.key_valid, fourteen, what="after 15 words")
    # 20 aggregations: the 16th (a sum) triggers the first finalize launch, 17-20 take a second one
    twenty = ([("count", c) for c in cols[:6]] + [("len", None)] * 3 + [("max", c0), ("min", c1), ("count", c0), ("count", c1), ("count", m0),
              ("count", f0), ("sum", m0), ("mean", f0), ("max", m0), ("min", f0), ("count", cols[2])])
    assert len(twenty) == 20 and twenty[15][0] == "sum" and twenty[15][1] is m0
    run(plb, case.keys, case.key_valid, twenty, True, what="20 aggregations")
    nv = case.values(rng, "int64", nullable=True)
    fv = case.values(rng, "float64", for_sum=True, nullable=True)
    small = [("sum", nv), ("mean", fv), ("min", nv), ("max", fv), ("count", nv), ("len", None)]
    for n in (0, 1):
        k = case.keys[:n]
        sl = [(kind, None if c is None else (c[0][:n], c[1][:n])) for kind, c in small]
        run(plb, k, None, sl, True, what=f"{n} rows")
    allnull = np.zeros(case.n, bool)
    run(plb, case.keys, allnull, small, True, what="all keys null")
    run(plb, case.keys, allnull, small, False, device=True, what="all keys null, device")
