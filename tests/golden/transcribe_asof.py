"""Asof join: known-answer vectors transcribed BY HAND from the reference's own tests (pola-rs/polars @ 4db92c1).

Each case is one asof join: the `on` columns `left` / `right` (dtype `dtype`, `null` = a null slot), `strategy`,
`allow_eq`, `tol` (null = none) and optional `by` columns (`left_by` / `right_by`: one list of values per column).  `by_dtype`
(default Int64, or Float64 / String as the values say) is the dtype of every `by` column.  `expect` holds, per left row,
`payload[j]` of the matched right row j (`null` = no match); `payload` defaults to the right row index.  Datetimes are
written as integer microseconds since the epoch and dates as days (their physical Int64 / Int32), tolerances in the same
unit.  Frames the reference sorts before joining are written sorted.

Run `python tests/golden/transcribe_asof.py` to regenerate tests/golden/asof_kats.json.
"""
import itertools
import json
import math
import os
import random
from datetime import date, datetime, timezone

N = None
NAN = math.nan
RS = "crates/polars-ops/src/frame/join/asof/default.rs"
PY = "py-polars/tests/unit/operations/test_join_asof.py"
S = 1_000_000      # one second in microseconds


def case(cite, dtype, left, right, strategy, expect, allow_eq=True, tol=None, left_by=None, right_by=None, payload=None, by_dtype=None):
    return {"cite": cite, "dtype": dtype, "left": left, "right": right, "strategy": strategy, "allow_eq": allow_eq, "tol": tol,
            "left_by": left_by, "right_by": right_by, "by_dtype": by_dtype, "payload": payload, "expect": expect}


def us(*dt):
    """a naive datetime as microseconds since the epoch (Datetime("us") physical)"""
    return int(datetime(*dt, tzinfo=timezone.utc).timestamp()) * 1_000_000


KATS = [
    case(f"{RS}:186-195 (test_asof_backward 1)", "int32", [-1, 2, 3, 3, 3, 4], [1, 2, 3, 3], "backward", [N, 1, 3, 3, 3, 3]),
    case(f"{RS}:197-202 (test_asof_backward 2)", "int32", [-1, 2, 3, 3, 3, 4], [1, 2, 4, 5], "backward", [N, 1, 1, 1, 1, 2]),
    case(f"{RS}:204-207 (test_asof_backward 3)", "int32", [2, 4, 4, 4], [1, 2, 3, 3], "backward", [1, 3, 3, 3]),
    case(f"{RS}:211-219 (test_asof_backward_tolerance)", "int32", [-1, 20, 25, 30, 30, 40], [10, 20, 30, 30], "backward", [N, 1, N, 3, 3, N], tol=4),
    case(f"{RS}:222-230 (test_asof_forward_tolerance)", "int32", [-1, 20, 25, 30, 30, 40, 52], [10, 20, 33, 55], "forward", [N, 1, N, 2, 2, N, 3], tol=4),
    case(f"{RS}:233-240 (test_asof_forward)", "int32", [-1, 1, 2, 4, 6], [1, 2, 4, 5], "forward", [0, 0, 1, 2, N]),
    case(f"{PY}:186-197 (test_join_asof_floats)", "float64", [1.0, 2.0, 3.0], [0.59, 1.49, 2.89], "backward", ["rrow1", "rrow2", "rrow3"],
         payload=["rrow1", "rrow2", "rrow3"]),
    case(f"{PY}:199-224 (test_join_asof_floats, by c, 5740)", "float64",
         [0.0, 0.8333333333333334, 1.6666666666666667, 2.5, 3.3333333333333335, 4.166666666666667, 5.0],
         [0.0, 2.5, 2.6, 2.7, 3.4, 4.0, 5.0], "backward", [0.0, 0.0, 0.0, 2.5, 2.7, 4.0, 5.0],
         left_by=[["x", "x", "x", "x", "y", "y", "y"]], right_by=[["x", "x", "x", "y", "y", "y", "y"]], payload=[0.0, 2.5, 2.6, 2.7, 3.4, 4.0, 5.0]),
]
TRADES = dict(left=[1 * S, 1 * S, 3 * S, 6 * S], left_by=[["A", "B", "B", "C"]])
QUOTES = dict(right=[0, 2 * S, 4 * S, 6 * S], right_by=[["A", "B", "C", "A"]], payload=[100, 300, 501, 102])
KATS.append(case(f"{PY}:227-275 (test_join_asof_tolerance, 2s)", "int64", strategy="backward", tol=2 * S, expect=[100, N, 300, 501], **TRADES, **QUOTES))
KATS.append(case(f"{PY}:277-289 (test_join_asof_tolerance, 1s)", "int64", strategy="backward", tol=1 * S, expect=[100, N, 300, N], **TRADES, **QUOTES))
MS = 1000
KATS.append(case(f"{PY}:1317-1370 (test_join_asof_no_exact_matches)", "int64",
                 [23 * MS, 38 * MS, 48 * MS, 48 * MS, 48 * MS], [23 * MS, 23 * MS, 30 * MS, 41 * MS, 48 * MS, 49 * MS, 72 * MS, 75 * MS], "backward",
                 [N, 51.97, N, N, N], allow_eq=False, tol=10 * MS,
                 left_by=[["MSFT", "MSFT", "GOOG", "GOOG", "AAPL"]], right_by=[["GOOG", "MSFT", "MSFT", "MSFT", "GOOG", "AAPL", "GOOG", "MSFT"]],
                 payload=[720.50, 51.95, 51.97, 51.99, 720.50, 97.99, 720.50, 52.01]))
BIG = 1608129000134000123
for strat in ("backward", "forward", "nearest"):
    KATS.append(case(f"{PY}:1495-1518 (test_join_asof_large_int_21276, {strat})", "int64", [BIG + 2], [BIG + 1, BIG + 3], strat,
                     [111 if strat == "backward" else 333], payload=[111, 333]))
for left, right, exp in [([], [], []), ([1], [2], [2]), ([], [1, 2], []), ([1, 2], [], [N, N]), ([1, 2], [1, 2], [2, 1]), ([1, 1], [1, 1], [N, N]),
                         ([1, 2, 2, 2, 3], [1, 2, 2, 2, 3], [2, 3, 3, 3, 2])]:
    KATS.append(case(f"{PY}:1680-1708 (test_join_asof_nearest_no_exact_matches_25468, {left} {right})", "int32", left, right, "nearest", exp,
                     allow_eq=False, payload=right))
for strat in ("backward", "nearest"):
    KATS.append(case(f"{PY}:1710-1733 (test_join_asof_nans, {strat})", "float64", [0.0, 6.0, NAN, NAN], [0.0, 5.0, 10.0, 42.0], strat,
                     [100, 200, 400, 400], payload=[100, 200, 300, 400]))
KATS.append(case(f"{PY}:1793-1808 (test_join_asof_by_nulls_27165)", "float64", [1.0], [0.0], "nearest", [N], left_by=[[0]], right_by=[[N]]))
KATS.append(case(f"{PY}:1811-1848 (test_join_asof_by_nulls_27165_2)", "float64", [N, 0.0], [N, N, N, 1.0], "nearest", [N, 3], allow_eq=False,
                 left_by=[[N, 0]], right_by=[[N, N, N, 0]]))

# test_join_asof_tolerance_forward: quotes (left) joined forward to trades (right) by stock; the trades are sorted by time
# only within each stock
QUOTES_F = dict(left=[0, 2 * S, 4 * S, 6 * S, 7 * S], left_by=[["A", "B", "C", "A", "D"]])
TRADES_F = dict(right=[2 * S, 1 * S, 3 * S, 6 * S, 7 * S], right_by=[["A", "B", "B", "C", "D"]], payload=[101, 299, 301, 500, 10])
for t, exp, lines in [(2, [101, 301, 500, N, 10], "295-336"), (1, [N, 301, N, N, 10], "339-352"), (0, [N, N, N, N, 10], "354-368")]:
    KATS.append(case(f"{PY}:{lines} (test_join_asof_tolerance_forward, {t}s)", "int64", strategy="forward", tol=t * S, expect=exp, **QUOTES_F, **TRADES_F))

# test_asof_join_nearest
KATS.append(case(f"{PY}:482-503 (test_asof_join_nearest)", "int64", [-1, 1, 2, 4, 6], [-1, 2, 4, 5], "nearest", [1, 2, 2, 3, 4], payload=[1, 2, 3, 4]))
KATS.append(case(f"{PY}:505-527 (test_asof_join_nearest, last right item matches several left rows)", "int64", [9, 9, 10, 10, 10], [1, 2, 3, 10],
                 "nearest", [4, 4, 4, 4, 4], payload=[1, 2, 3, 4]))

# test_asof_join_nearest_with_tolerance, cases 1-7 and 9 (case 8 is case 7 with the tolerance spelled as a timedelta)
B5 = [1, 2, 3, 4, 5]
for no, dt, left, right, tol, exp, lines in [
        (1, "int64", [1, 2, 3, 4, 5], [7, 8, 9, 10, 11], 1, [N] * 5, "602-612"),
        (2, "int64", [7, 8, 9, 10, 11], [1, 2, 3, 4, 5], 1, [N] * 5, "614-624"),
        (3, "int64", [1, 2, 3, 4, 5], [6, 7, 8, 9, 10], 1, [N, N, N, N, 1], "626-636"),
        (4, "int64", [1, 2, 3, 4, 5], [-4, -3, -2, -1, 0], 1, [5, N, N, N, N], "638-648"),
        (5, "float64", [1.0, 2.0, 3.0, 4.0, 5.0], [0.0, 2.0, 2.4, 3.4, 10.0], 1.0, [2, 2, 4, 4, N], "650-662"),
        (6, "float64", [1.0, 2.0, 3.0, 4.0, 5.0], [0.0, 2.0, 2.4, 3.4, 10.0], 0.0, [N, 2, N, N, N], "664-676")]:
    KATS.append(case(f"{PY}:{lines} (test_asof_join_nearest_with_tolerance, case {no})", dt, left, right, "nearest", exp, tol=tol, payload=B5))
KATS.append(case(f"{PY}:678-711 (test_asof_join_nearest_with_tolerance, case 7, tolerance 1d4h)", "int64",
                 [us(2023, 1, 1), us(2023, 1, 2), us(2023, 1, 3), us(2023, 1, 4), us(2023, 1, 6)],
                 [us(2022, 1, 1), us(2022, 1, 2), us(2022, 1, 3), us(2023, 1, 2, 21, 30, 0), us(2023, 1, 7)], "nearest", [N, 4, 4, 4, 5],
                 tol=(24 + 4) * 3600 * S, payload=B5))
KATS.append(case(f"{PY}:719-743 (test_asof_join_nearest_with_tolerance, case 9)", "float64", [10.00001, 20.0, 30.0], [10.00001, 20.0001, 29.0], "nearest",
                 [10.00001, 20.0001, N], tol=0.5, payload=[10.00001, 20.0001, 29.0]))

# test_asof_join_nearest_by (its first frame is overwritten before any join and asserts nothing)
KATS.append(case(f"{PY}:773-800 (test_asof_join_nearest_by, last right item matches several left rows)", "int64", [9, 9, 10, 10, 10], [-1, 1, 1, 10],
                 "nearest", [2, 2, 2, 4, 4], left_by=[[1, 1, 1, 2, 2]], right_by=[[1, 1, 2, 2]], payload=[1, 2, 3, 4]))
KATS.append(case(f"{PY}:802-825 (test_asof_join_nearest_by, code / time)", "int64", [364360, 364370, 364380, 365400, 367440],
                 [364000, 365000, 365000, 366000, 367000], "nearest", [1.0, 50.0, 1.0, 2.0, N],
                 left_by=[[676, 35, 676, 676, 676]], right_by=[[676, 676, 35, 676, 676]], payload=[1.0, 2.0, 50.0, 3.0, N]))
KATS.append(case(f"{PY}:827-855 (test_asof_join_nearest_by, last item is closest match)", "float64", [10.00001, 20.0, 30.0], [10.00001, 20.0001, 29.0],
                 "nearest", [10.00001, 20.0001, 29.0], left_by=[[1, 1, 1]], right_by=[[1, 1, 1]], payload=[10.00001, 20.0001, 29.0]))

# test_asof_join_nearest_by_with_tolerance: both frames sorted by (group, asof_key), so the left side is sorted only within
# each group; `b` of the right frame moves with its sort
G6 = [g for g in range(1, 7) for _ in range(5)]
L6 = [1, 2, 3, 4, 5, 7, 8, 9, 10, 11] + [1, 2, 3, 4, 5] * 4
R6 = [(g, k, b) for g, ks in zip(range(1, 7), [[7, 8, 9, 10, 11], [1, 2, 3, 4, 5], [6, 7, 8, 9, 10], [5, -3, -2, -1, 0], [0, 2, 2.4, 3.4, 10], [-3, 3, 8, 9, 10]])
      for k, b in zip(ks, B5)]
R6.sort(key=lambda t: (t[0], t[1]))
KATS.append(case(f"{PY}:857-1108 (test_asof_join_nearest_by_with_tolerance)", "float32", [float(x) for x in L6], [float(k) for _, k, _ in R6], "nearest",
                 [N] * 14 + [1, 5, N, N, 1, 1, 2, 2, 4, 4, N, N, 2, 2, 2, N], tol=1.0,
                 left_by=[G6], right_by=[[g for g, _, _ in R6]], payload=[b for _, _, b in R6]))
KATS.append(case(f"{PY}:1111-1139 (test_asof_join_nearest_by_with_tolerance, last item is closest match)", "float64", [10.00001, 20.0, 30.0],
                 [10.00001, 20.0001, 29.0], "nearest", [10.00001, 20.0001, N], tol=0.5, left_by=[[1, 1, 1]], right_by=[[1, 1, 1]],
                 payload=[10.00001, 20.0001, 29.0]))

# test_join_asof_int_dtypes_24383: a `by` column of every integer dtype, on a Date
D = (date(2025, 12, 31) - date(1970, 1, 1)).days
for dt in ("uint8", "uint16", "uint32", "uint64", "int8", "int16", "int32", "int64"):
    KATS.append(case(f"{PY}:1620-1657 (test_join_asof_int_dtypes_24383, {dt})", "int32", [D], [D], "backward", [2.5],
                     left_by=[[1]], right_by=[[1]], by_dtype=dt, payload=[2.5]))


def nearest_reference(left, right, right_values, allow_eq):
    """asof_join_nearest_reference (test_join_asof.py:536-570): the smallest |key - key_right|, ties to the largest right
    index; without allow_exact_matches the equal keys are dropped first"""
    out = []
    for k in left:
        cand = [(abs(k - kr), -j) for j, kr in enumerate(right) if allow_eq or kr != k]
        out.append(right_values[-min(cand)[1]] if cand else None)
    return out


# test_asof_join_nearest_reference: its 81 frames (the same generator, random.Random(0)), a fixed sample of 40 pairs per
# allow_exact_matches, answered by the test's own brute-force reference
_rng = random.Random(0)
FRAMES = []
for n_a, n_b, n_c, n_d in itertools.product([0, 1, 2], repeat=4):
    a, b, c, d = (_rng.randint(0, 10) for _ in range(4))
    keys = [a] * n_a + [b] * n_b + [c] * n_c + [d] * n_d
    values = [_rng.randint(0, 100000) for _ in keys]
    order = sorted(range(len(keys)), key=lambda i: keys[i])
    FRAMES.append(([keys[i] for i in order], [values[i] for i in order]))
_pick = random.Random(1)
for allow_eq in (True, False):
    for _ in range(40):
        (lk, _lv), (rk, rv) = FRAMES[_pick.randrange(len(FRAMES))], FRAMES[_pick.randrange(len(FRAMES))]
        KATS.append(case(f"{PY}:530-594 (test_asof_join_nearest_reference, allow_exact_matches={allow_eq}, {lk} {rk})", "int32", lk, rk, "nearest",
                         nearest_reference(lk, rk, rv, allow_eq), allow_eq=allow_eq, payload=rv))


if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "asof_kats.json")
    with open(path, "w") as f:
        json.dump({"asof": KATS}, f, indent=1)
        f.write("\n")
    print(f"wrote {len(KATS)} cases to {path}")
