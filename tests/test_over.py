"""CPU tests of the window functions (bl_over): the oracle against the reference's known answers and numpy
restatements, the associativity of the parallel min / max tie rules, the C declarations, the plugin field functions and
the binding's argument errors."""
import ctypes as C
import itertools
import json
import math
import os
import struct

import numpy as np
import pytest

import window_oracle as wo
from test_cabi_cpu import declared_symbols

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "window_kats.json")))


def _same(a, b) -> bool:
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, float) or isinstance(b, float):
        a, b = float(a), float(b)
        return (a != a and b != b) or struct.pack("<d", a) == struct.pack("<d", b)
    return a == b


def kat_oracle(case):
    cols = case["columns"]
    n = len(next(iter(cols.values())))
    keys = [cols[k] for k in case["partition_by"]]
    order = cols[case["order_by"]] if case["order_by"] else None
    ops = [(kind, cols[c] if c else None, case["dtypes"][c] if c else "int64", opts) for _, kind, c, opts in case["ops"]]
    return wo.over(ops, keys, n, order, case["descending"], case["nulls_last"])


def kat_mismatches(case, outputs):
    """outputs: output name -> list (None = null).  Returns a description of every difference from the case's answer."""
    bad = []
    rows = case.get("rows")
    rtol = case.get("rtol")
    for name, exp in case["expected"].items():
        got = outputs[name]
        if len(got) != len(exp):
            bad.append((name, "length", len(got), len(exp)))
            continue
        for r in (rows if rows is not None else range(len(exp))):
            a, b = got[r], exp[r]
            if rtol is not None and a is not None and b is not None and abs(float(a) - float(b)) <= 1e-8 + rtol * abs(float(b)):
                continue
            if not _same(a, b):
                bad.append((name, r, a, b))
    for x, y in case.get("equal", []):
        if not all(_same(a, b) for a, b in zip(outputs[x], outputs[y])):
            bad.append((x, y, outputs[x], outputs[y]))
    return bad


@pytest.mark.parametrize("i", range(len(KATS)))
def test_oracle_reproduces_kats(i):
    case = KATS[i]
    got = kat_oracle(case)
    outs = {name: g for (name, *_), g in zip(case["ops"], got)}
    assert not kat_mismatches(case, outs), (case["src"], kat_mismatches(case, outs))


def _np_cum(kind, x, dtype):
    if kind == "cum_sum":
        return np.cumsum(x.astype(np.int64 if dtype.startswith("int") or dtype.startswith("uint") else x.dtype), dtype=x.dtype if dtype in ("int64", "uint64", "float64") else None)
    if kind == "cum_min":
        return np.minimum.accumulate(x)
    return np.maximum.accumulate(x)


@pytest.mark.parametrize("dtype", ["int64", "uint64", "int32", "float64"])
@pytest.mark.parametrize("kind", ["cum_sum", "cum_min", "cum_max"])
@pytest.mark.parametrize("reverse", [False, True])
def test_oracle_matches_numpy(dtype, kind, reverse):
    rng = np.random.default_rng(7)
    n = 400
    if dtype.startswith("float"):
        x = rng.integers(-1000, 1000, n).astype(np.float64)      # exactly summable: numpy's order gives the same sums
    else:
        info = np.iinfo(dtype)
        x = rng.integers(info.min, info.max, n, dtype=dtype, endpoint=True)
    g = rng.integers(0, 7, n)
    got = wo.over([(kind, x.tolist(), dtype, {"reverse": reverse})], [g.tolist()], n)[0]
    exp = np.empty(n, dtype=np.float64 if dtype.startswith("float") else object)
    for key in np.unique(g):
        rows = np.nonzero(g == key)[0]
        if reverse:
            rows = rows[::-1]
        with np.errstate(over="ignore"):
            vals = x[rows]
            if kind == "cum_sum" and not dtype.startswith("float"):
                acc = np.cumsum(vals.astype(np.uint64) if dtype in ("uint64", "int64") else vals.astype(np.int64)).astype(np.uint64)
                r = [wo.wrap(int(v), dtype) for v in acc]
            else:
                r = _np_cum(kind, vals, dtype).tolist()
        for row, v in zip(rows, r):
            exp[row] = v
    assert all(_same(a, b) for a, b in zip(got, exp.tolist()))


def test_oracle_cum_count_and_shift():
    v = [1, None, 3, 4, None, 6]
    g = [0, 0, 1, 0, 1, 1]
    out = wo.over([("cum_count", v, "int64", {}), ("cum_count", v, "int64", {"reverse": True}), ("shift", v, "int64", {"periods": 1}),
                   ("shift", v, "int64", {"periods": -1}), ("shift", v, "int64", {"periods": 3})], [g], 6)
    assert out[0] == [1, 1, 1, 2, 1, 2]
    assert out[1] == [2, 1, 2, 1, 1, 1]
    assert out[2] == [None, 1, None, None, 3, None]
    assert out[3] == [None, 4, None, None, 6, None]
    assert out[4] == [None] * 6


def test_oracle_float32_sum_accumulates_in_f64():
    x = [16777216.0, 1.0, 1.0]       # 2^24 + 1 + 1: f32 steps would stall at 2^24
    assert wo.cum_seq("cum_sum", x, "float32") == [16777216.0, 16777216.0, 16777218.0]


SPECIALS = [None, -0.0, 0.0, 1.0, -math.inf, math.inf, math.nan]


def _bits(x):
    return None if x is None else ("nan" if x != x else struct.pack("<d", x))


def _bracketings(xs, combine):
    if len(xs) == 1:
        yield xs[0]
        return
    for k in range(1, len(xs)):
        for a in _bracketings(xs[:k], combine):
            for b in _bracketings(xs[k:], combine):
                yield combine(a, b)


@pytest.mark.parametrize("kind", ["cum_min", "cum_max"])
def test_min_max_tie_rules_are_associative(kind):
    """The device combines scan pieces in any bracketing, a null being the identity (NaN).  Every bracketing of every
    sequence of length <= 5 over {null, -0, +0, 1, -inf, +inf, NaN}, forward and reverse, equals the sequential det_min /
    det_max (the last output of the scan), bit for bit."""
    fn = wo.min_ignore_nan if kind == "cum_min" else wo.max_ignore_nan
    nan = math.nan
    for length in range(1, 6):
        for seq in itertools.product(SPECIALS, repeat=length):
            for order in (seq, seq[::-1]):
                outs = [x for x in wo.cum_seq(kind, list(order), "float64") if x is not None]
                want = outs[-1] if outs else nan      # the state after the last row (a null leaves it unchanged)
                lifted = [nan if v is None else v for v in order]
                for got in _bracketings(lifted, fn):
                    assert _bits(got) == _bits(want), (order, got, want)


def test_header_declares_over():
    assert "bl_over" in declared_symbols()
    hdr = open(os.path.join(ROOT, "include", "polars_b200.h")).read()
    for name in ("BL_CUM_SUM = 32", "BL_CUM_PROD = 33", "BL_CUM_MIN = 34", "BL_CUM_MAX = 35", "BL_CUM_COUNT = 36", "BL_SHIFT = 37", "bl_over_op"):
        assert name in hdr


def _lib():
    import polars_b200 as pb
    try:
        return pb.lib()
    except ImportError:
        pytest.skip("the library is not built")


class ArrowSchema(C.Structure):
    pass


ArrowSchema._fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64), ("n_children", C.c_int64),
                        ("children", C.c_void_p), ("dictionary", C.c_void_p), ("release", C.c_void_p), ("private_data", C.c_void_p)]


@pytest.mark.parametrize("entry,fmt_in,fmt_out", [
    ("cum_sum", b"c", b"l"), ("cum_sum", b"b", b"I"), ("cum_sum", b"i", b"i"), ("cum_sum", b"f", b"f"), ("cum_sum", b"L", b"L"),
    ("cum_prod", b"i", b"l"), ("cum_prod", b"I", b"l"), ("cum_prod", b"b", b"l"), ("cum_prod", b"L", b"L"), ("cum_prod", b"f", b"f"),
    ("cum_min", b"s", b"s"), ("cum_max", b"g", b"g"), ("cum_count", b"g", b"I"), ("cum_count", b"b", b"I"), ("shift", b"C", b"C"),
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
    (dict(ops=[("cum_foo", np.arange(3), {})]), "unknown over"),
    (dict(ops=[("cum_sum", np.arange(3), {"periods": 2})]), "no option"),
    (dict(ops=[("shift", np.arange(3), {"reverse": True})]), "no option"),
    (dict(ops=[("sum", None)]), "needs a value column"),
    (dict(ops=[]), "at least one"),
    (dict(ops=[("sum", np.arange(3))], order_by=[np.arange(3), np.arange(3)]), "one order_by"),
    (dict(ops=["sum"]), "operation is"),
])
def test_binding_argument_errors(args, msg):
    import polars_b200 as pb
    with pytest.raises(ValueError, match=msg):
        pb.over(**args)


def test_cum_agg_rejects_unknown_kind():
    import polars_b200 as pb
    with pytest.raises(ValueError, match="unknown cumulative"):
        pb.cum_agg("sum", np.arange(3))
