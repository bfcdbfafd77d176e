"""CPU checks of the time-based rolling windows (bl_rolling_by): the kernel's binary-search bounds against the reference's
iterator, the block decomposition against tuple concatenation, known answers of the reference's tests, and the Python
binding's duration parsing and argument errors.  No GPU needed."""
import datetime
import itertools

import numpy as np
import pytest

from rolling_by_oracle import CLOSED, I64_MAX, I64_MIN, bs_windows, decompose, ref_windows, window_values

ALPHABET = [I64_MIN, I64_MIN + 2, -3, -1, 0, 2, I64_MAX]


@pytest.mark.parametrize("closed", CLOSED)
def test_bounds_equal_reference_iterator(closed):
    # every non-decreasing sequence of length <= 7 over the alphabet (negative times, i64::MIN and i64::MAX included: t - P
    # wraps below i64::MIN + P), every P in 1..5
    for n in range(1, 8):
        for times in itertools.combinations_with_replacement(ALPHABET, n):
            for P in range(1, 6):
                assert bs_windows(list(times), P, closed) == ref_windows(list(times), P, closed), (times, P)


def test_wrapped_lower_bound_pins_the_start():
    # i64::MIN + 1 - 3 wraps to i64::MAX - 1: the first run's window is itself, and the later rows never start before it
    times = [I64_MIN, I64_MIN + 1, I64_MIN + 1, I64_MIN + 5]
    assert ref_windows(times, 3, "right") == [(0, 1), (1, 3), (1, 3), (3, 4)]
    assert ref_windows(times, 3, "left") == [(0, 0), (1, 1), (1, 1), (3, 3)]
    assert bs_windows(times, 3, "right") == ref_windows(times, 3, "right")


def test_decomposition_gives_each_window_exactly():
    # tuple concatenation as the combine: every window of every split into partitions comes out as its positions in order
    for n in range(1, 13):
        for B, SUB in ((4, 2), (8, 2), (4, 1), (2, 1)):
            for cuts in itertools.product((0, 1), repeat=n - 1):
                seg = [0]
                for c in cuts:
                    seg.append(seg[-1] + c)
                lo = 0
                while lo < n:
                    hi = lo
                    while hi < n and seg[hi] == seg[lo]:
                        hi += 1
                    for s in range(lo, hi):
                        for e in range(s + 1, hi + 1):
                            got = decompose(s, e, seg, n, B, SUB, lambda q: (q,), lambda a, b: a + b)
                            assert got == tuple(range(s, e)), (n, B, SUB, seg, s, e)
                    lo = hi
            if n > 8:
                break


def test_kat_rolling_by_integer():
    # py-polars/tests/unit/operations/rolling/test_rolling.py:1033 (test_rolling_by_integer), :1045 (test_rolling_sum_by_integer)
    w = window_values([1, 2, 3], [True] * 3, [0, 1, 2], [True] * 3, 2, "right", 0)
    assert [sum(x) for x in w] == [1, 3, 5]


def test_kat_rolling_by_date():
    # test_rolling.py:1019 (test_rolling_by_date): "2d" over Date -> Datetime(us)
    import polars_b200 as pb
    days = np.array(["2020-01-01", "2020-01-02", "2020-01-03"], dtype="datetime64[D]")
    col, unit = pb._by_column(days)
    P = pb.window_size_in("2d", unit)
    w = window_values([1, 2, 3], [True] * 3, list(col), [True] * 3, P, "right", 0)
    assert [sum(x) for x in w] == [1, 3, 5]


def test_kat_min_samples_and_nulls():
    # a window below min_samples is null whatever its values (shared.rs:109-204); a null `by` row is null (dispatch.rs:101-129)
    w = window_values([1, None, 3, 4], [True, False, True, True], [0, 1, 2, 5], [True, True, True, False], 2, "right", 2)
    assert w == [None, [1], [3], None]


def test_durations():
    import polars_b200 as pb
    assert pb.window_size_in("30s", "us") == 30_000_000
    assert pb.window_size_in("1d12h", "ms") == 129_600_000
    assert pb.window_size_in("1w", "ns") == 7 * 86_400 * 10**9
    assert pb.window_size_in("1500ns", "us") == 1      # truncated as add_us does
    assert pb.window_size_in("3i", None) == 3
    assert pb.window_size_in(datetime.timedelta(minutes=5), "us") == 300_000_000
    assert pb.window_size_in(7, None) == 7


@pytest.mark.parametrize("ws,unit", [("1mo", "us"), ("2q", "ns"), ("1y", "ms"), ("3i", "us"), ("1d", None), ("500ns", "us"),
                                     ("5x", "us"), ("-5s", "us"), (0, None), (-1, "us"), (1.5, "us"), ("3i2s", "us")])
def test_duration_errors(ws, unit):
    # test_rolling.py:304 / :324 (test_rolling_by_invalid / test_rolling_by_non_temporal_window_size) as ValueErrors
    import polars_b200 as pb
    with pytest.raises(ValueError):
        pb.window_size_in(ws, unit)


def test_rolling_by_argument_errors():
    import polars_b200 as pb
    v, t = np.arange(4.0), np.arange(4)
    for ops in ([], [("rolling_median", v, {"window_size": "2i"})], [("rolling_sum", v, {})],
                [("rolling_sum", v, {"window_size": "2i", "closed": "middle"})], [("rolling_sum", v, {"window_size": "2i", "min_samples": -1})],
                [("rolling_var", v, {"window_size": "2i", "ddof": 256})], [("rolling_sum", v, {"window_size": "2i", "center": True})]):
        with pytest.raises(ValueError):
            pb.rolling_by(ops, t)
    with pytest.raises(ValueError):
        pb.rolling_by([("rolling_sum", v, {"window_size": "2i"})], np.array(["2020-01-01"] * 4, dtype="datetime64[s]"))


def _kats():
    import json
    import os
    with open(os.path.join(os.path.dirname(__file__), "golden", "rolling_by_kats.json")) as f:
        return json.load(f)


def test_kats_through_the_oracle():
    # tests/golden/rolling_by_kats.json (transcribe_rolling_by.py): every case's windows and values through the oracle
    from rolling_by_oracle import windows_of
    cases = _kats()
    assert len(cases) >= 30
    for c in cases:
        if c.get("error"):
            assert c["by_dtype"] not in ("int32", "int64", "uint32", "uint64")
            continue
        n = len(c["values"])
        bv = [v is not None for v in c["by"]]
        by = [0 if v is None else v for v in c["by"]]
        wins = window_values(c["values"], [v is not None for v in c["values"]], by, bv, c["window_size"], c["closed"], c["min_samples"], c["parts"])
        got = []
        for w in wins:
            if w is None or len(w) < c["min_samples"]:
                got.append(None)
            elif c["kind"] == "rolling_sum":
                got.append(sum(w))
            elif c["kind"] == "rolling_mean":
                got.append(sum(w) / len(w) if w else None)
            else:
                got.append(min(w) if w else None)
        assert got == c["expected"], c["src"]
        if "windows" in c:
            win, _ = windows_of(by, bv, c["parts"], c["window_size"], c["closed"])
            assert [[s, e - s] for s, e in win] == c["windows"], c["src"]
        assert n == len(c["expected"])


def test_plugin_field_functions():
    # the output schema of _polars_plugin_field_bl_rolling_*_by follows rolling_dtype from the values' format
    import ctypes as C
    import polars_b200 as pb
    try:
        L = pb.lib()
    except ImportError:
        pytest.skip("the library is not built")

    class ArrowSchema(C.Structure):
        _fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64), ("n_children", C.c_int64),
                    ("children", C.c_void_p), ("dictionary", C.c_void_p), ("release", C.c_void_p), ("private_data", C.c_void_p)]
    for entry, fmt_in, fmt_out in [("sum", b"c", b"l"), ("sum", b"b", b"I"), ("sum", b"i", b"i"), ("sum", b"f", b"f"), ("mean", b"i", b"g"),
                                   ("mean", b"f", b"f"), ("min", b"s", b"s"), ("max", b"L", b"L"), ("var", b"l", b"g"), ("std", b"f", b"f")]:
        fn = getattr(L, f"_polars_plugin_field_bl_rolling_{entry}_by")
        fields = (ArrowSchema * 2)()
        fields[0].format, fields[0].name = fmt_in, b"x"
        fields[1].format, fields[1].name = b"l", b"t"
        out = ArrowSchema()
        fn(fields, C.c_size_t(2), C.byref(out), None, C.c_size_t(0))
        assert out.format == fmt_out, (entry, fmt_in, out.format)
        C.CFUNCTYPE(None, C.POINTER(ArrowSchema))(out.release)(C.byref(out))
