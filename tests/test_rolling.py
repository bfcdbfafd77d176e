"""bl_rolling without a GPU: the oracle against the known answers and numpy, the device's decomposition and combine rules
against the reference's sequential machines (exhaustively), the declarations, the plugin field functions and the binding's
argument errors."""
import ctypes as C
import itertools
import json
import math
import os
import random
import struct

import numpy as np
import pytest

import rolling_oracle as ro
from test_cabi_cpu import declared_symbols
from test_over import ArrowSchema

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "rolling_kats.json")))
INF, NAN = math.inf, math.nan
SYMBOLS = [None, -0.0, 0.0, 1.0, INF, -INF, NAN]


def _bits(x):
    return None if x is None else struct.pack("<d", float(x))


@pytest.mark.parametrize("i", range(len(KATS)))
def test_oracle_reproduces_kats(i):
    c = KATS[i]
    got = ro.rolling(c["kind"], c["values"], c["dtype"], c["window_size"], c["min_samples"], c["center"], c["ddof"])
    # the reference's tests compare NaN through its Debug string, so a NaN matches a NaN of either sign
    assert [_bits(x) if x == x else "nan" for x in got] == [_bits(x) if x == x else "nan" for x in c["expected"]], c["src"]


def _np_windows(x, w, center):
    n = len(x)
    offs = ro.det_offsets_center if center else ro.det_offsets
    return [x[slice(*offs(i, w, n))] for i in range(n)]


@pytest.mark.parametrize("dtype", ["int32", "uint32", "int64", "uint64"])
@pytest.mark.parametrize("center", [False, True])
def test_integer_sum_min_max_match_numpy(dtype, center):
    rng = np.random.default_rng(7)
    info = np.iinfo(dtype)
    x = rng.integers(info.min, info.max, size=40, dtype=dtype, endpoint=True)
    for w in (1, 2, 3, 7, 40, 41):
        wins = _np_windows(x, w, center)
        with np.errstate(over="ignore"):
            want_sum = [int(np.sum(v, dtype=dtype)) for v in wins]
        assert ro.rolling("rolling_sum", x.tolist(), dtype, w, 1, center) == want_sum
        assert ro.rolling("rolling_min", x.tolist(), dtype, w, 1, center) == [int(v.min()) for v in wins]
        assert ro.rolling("rolling_max", x.tolist(), dtype, w, 1, center) == [int(v.max()) for v in wins]


def test_sum_non_finite_property_23115():
    # operations/rolling/test_rolling.py:1935-1952: the sum of 4 with min_samples 2 is the naive sum, class by class
    rng = random.Random(23115)
    for with_nulls in (False, True):
        values = [0.0, NAN, INF, -INF, 42.0, -3.0] + ([None] if with_nulls else [])
        data = rng.choices(values, k=1000)
        got = ro.rolling("rolling_sum", data, "float64", 4, 2)
        for i in range(1000):
            win = data[max(0, i - 3): i + 1]
            want = sum(0 if v is None else v for v in win) if sum(v is not None for v in win) >= 2 else None
            same = (got[i] is None and want is None) or (got[i] is not None and want is not None and
                                                       (got[i] == want or (got[i] != got[i] and want != want)))
            assert same, (i, win)      # assert_series_equal: NaN equals NaN whatever its sign


# ---------------------------------------------------------------------------------------------------- the device's rules
def _compositions(n):
    """every split of range(n) into consecutive segments"""
    for cuts in itertools.product((False, True), repeat=max(n - 1, 0)):
        segs, lo = [], 0
        for p, c in enumerate(cuts, start=1):
            if c:
                segs.append((lo, p))
                lo = p
        segs.append((lo, n))
        yield segs


def test_decomposition_covers_exactly_each_window():
    # with tuple concatenation as the operator (associative, order-revealing), the decomposition must give exactly the
    # positions of every clipped window in order: then it is exact for every associative operator, partitions included
    for n in range(1, 10):
        for segs in _compositions(n):
            for w in range(1, n + 2):
                for center in (False, True):
                    got = ro.decomposed(list(range(n)), w, center, segs, lambda p: (p,), lambda a, b: a + b, ())
                    offs = ro.det_offsets_center if center else ro.det_offsets
                    for lo, hi in segs:
                        for i in range(lo, hi):
                            s, e = offs(i - lo, w, hi - lo)
                            assert got[i] == tuple(range(lo + s, lo + e)), (n, segs, w, center, i)


def _mm_combine(is_max):
    # MinMaxSt::combine of rolling.cu: (value, count), the earlier argument first
    def better(b, a):
        if a != a:
            return False
        if b != b:
            return True
        return a < b if is_max else b < a

    def combine(a, b):
        if a[1] == 0:
            return b
        if b[1] == 0:
            return a
        return (b[0] if better(b[0], a[0]) else a[0], a[1] + b[1])
    return combine


@pytest.mark.parametrize("kind", ["rolling_min", "rolling_max"])
def test_min_max_combine_is_associative_and_equals_the_deque(kind):
    combine = _mm_combine(kind == "rolling_max")
    states = [(0.0, 0)] + [(v, 1) for v in SYMBOLS if v is not None]
    for a, b, c in itertools.product(states, repeat=3):
        x, y = combine(combine(a, b), c), combine(a, combine(b, c))
        assert (_bits(x[0]), x[1]) == (_bits(y[0]), y[1]), (a, b, c)
    # with associativity, every window the decomposition forms is the left fold of its values: compare the fold with the
    # reference's deque on every sequence of length <= 6 (the deque's answer for the whole sequence as one window)
    for n in range(1, 7):
        for seq in itertools.product(SYMBOLS, repeat=n):
            fold = (0.0, 0)
            for v in seq:
                fold = combine(fold, (0.0, 0) if v is None else (v, 1))
            want = ro.rolling(kind, list(seq), "float64", n, 0)[-1]
            got = fold[0] if fold[1] else None
            assert _bits(got) == _bits(want), seq


def test_non_finite_counting_gives_the_reference_class():
    # SumFltSt of rolling.cu: the finite sum + the non-null count + counts of +inf / -inf / NaN, decomposed as the device
    # does.  Compared with the reference's SumWindow on every sequence of length <= 6 over {null, finite, +inf, -inf, NaN}
    # (the class depends on nothing else), every w in 1..n + 1 and both center settings: the class of every window and its
    # non-null count, which decides the validity for every min_samples in both (is_valid, rolling/sum.rs:219-221).  Every
    # partition of a split is itself one of these sequences and test_decomposition_covers_exactly_each_window shows that a
    # split changes nothing else; up to length 4 every split is also run explicitly.
    def lift(v):
        f = math.isfinite(v)
        return (v if f else 0.0, 1, int(v == INF), int(v == -INF), int(v != v))

    def combine(a, b):
        return tuple(x + y for x, y in zip(a, b))

    def cls(x):
        return None if x is None else ("nan" if x != x else x if math.isinf(x) else "finite")

    empty = (0.0, 0, 0, 0, 0)
    memo = {}
    for n in range(1, 7):
        for seq in itertools.product([None, 1.0, INF, -INF, NAN], repeat=n):
            for w in range(1, n + 2):
                for center in (False, True):
                    for segs in (_compositions(n) if n <= 4 else [[(0, n)]]):
                        dec = ro.decomposed(list(seq), w, center, segs, lift, combine, empty)
                        for lo, hi in segs:
                            key = (seq[lo:hi], w, center)
                            if key not in memo:
                                memo[key] = ro.rolling("rolling_sum", list(seq[lo:hi]), "float64", w, 0, center, counts=True)
                            ref, cnt = memo[key]
                            for i in range(lo, hi):
                                s, c, p, m, q = dec[i]
                                nf = p + m + q
                                got = s if nf == 0 else INF if nf == p else -INF if nf == m else NAN
                                assert cls(got) == cls(ref[i - lo]), (seq, w, center, segs, i)
                                assert c == cnt[i - lo], (seq, w, center, segs, i)
                                for ms in range(w + 1):
                                    assert (c >= ms) == (cnt[i - lo] >= ms)


# ---------------------------------------------------------------------------------------------------- interface
def test_header_declares_rolling():
    assert "bl_rolling" in declared_symbols()
    hdr = open(os.path.join(ROOT, "include", "polars_b200.h")).read()
    for name in ("BL_ROLLING_SUM = 40", "BL_ROLLING_MEAN = 41", "BL_ROLLING_MIN = 42", "BL_ROLLING_MAX = 43", "BL_ROLLING_VAR = 44",
                 "BL_ROLLING_STD = 45", "bl_rolling_op"):
        assert name in hdr
    rs = open(os.path.join(ROOT, "integration", "polars_b200_sys.rs")).read()
    assert "pub fn bl_rolling(" in rs and "pub struct BlRollingOp" in rs


def test_binding_struct_matches_the_header():
    import polars_b200 as pb
    assert C.sizeof(pb.BlRollingOp) == 40
    assert [f[0] for f in pb.BlRollingOp._fields_] == ["kind", "center", "window_size", "min_samples", "ddof", "reserved", "values"]


def _lib():
    import polars_b200 as pb
    try:
        return pb.lib()
    except ImportError:
        pytest.skip("the library is not built")


@pytest.mark.parametrize("entry,fmt_in,fmt_out", [
    ("rolling_sum", b"c", b"l"), ("rolling_sum", b"b", b"I"), ("rolling_sum", b"i", b"i"), ("rolling_sum", b"f", b"f"), ("rolling_sum", b"L", b"L"),
    ("rolling_mean", b"i", b"g"), ("rolling_mean", b"f", b"f"), ("rolling_mean", b"L", b"g"),
    ("rolling_min", b"s", b"s"), ("rolling_max", b"g", b"g"), ("rolling_max", b"I", b"I"),
    ("rolling_var", b"l", b"g"), ("rolling_var", b"f", b"f"), ("rolling_std", b"C", b"g"), ("rolling_std", b"f", b"f"),
])
def test_plugin_field_functions(entry, fmt_in, fmt_out):
    L = _lib()
    fn = getattr(L, "_polars_plugin_field_bl_" + entry)
    fields = (ArrowSchema * 2)()
    fields[0].format, fields[0].name = fmt_in, b"x"
    fields[1].format, fields[1].name = b"l", b"g"
    out = ArrowSchema()
    fn(fields, C.c_size_t(2), C.byref(out), None, C.c_size_t(0))
    assert out.format == fmt_out
    C.CFUNCTYPE(None, C.POINTER(ArrowSchema))(out.release)(C.byref(out))


@pytest.mark.parametrize("args,msg", [
    (dict(ops=[("rolling_foo", np.arange(3), {"window_size": 2})]), "unknown rolling"),
    (dict(ops=[("rolling_sum", np.arange(3), {})]), "needs a window_size"),
    (dict(ops=[("rolling_sum", np.arange(3), {"window_size": 2, "ddof": 1})]), "no option"),
    (dict(ops=[("rolling_sum", np.arange(3), {"window_size": 2, "reverse": True})]), "no option"),
    (dict(ops=[("rolling_sum", np.arange(3), {"window_size": 2, "min_samples": 3})]), "min_samples"),
    (dict(ops=[("rolling_sum", np.arange(3), {"window_size": 0})]), "at least 1"),
    (dict(ops=[("rolling_sum", np.arange(3), {"window_size": -1})]), "at least 1"),
    (dict(ops=[("rolling_sum", np.arange(3), {"window_size": 2.5})]), "integer"),
    (dict(ops=[("rolling_var", np.arange(3), {"window_size": 2, "ddof": 256})]), "ddof"),
    (dict(ops=[("rolling_sum", None, {"window_size": 2})]), "needs a value column"),
    (dict(ops=[]), "at least one"),
    (dict(ops=[("rolling_sum", np.arange(3))]), "operation is"),
    (dict(ops=[("rolling_sum", np.arange(3), {"window_size": 2})], order_by=[np.arange(3), np.arange(3)]), "one order_by"),
])
def test_binding_argument_errors(args, msg):
    import polars_b200 as pb
    with pytest.raises(ValueError, match=msg):
        pb.rolling(**args)


def test_rolling_agg_rejects_unknown_kind():
    import polars_b200 as pb
    with pytest.raises(ValueError, match="unknown rolling"):
        pb.rolling_agg("sum", np.arange(3), 2)
