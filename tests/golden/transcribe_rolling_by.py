"""Known answers of the reference's time-based rolling aggregations (rolling_*_by), transcribed by hand from its own tests,
each with its file:line (py-polars paths under py-polars/tests/unit, Rust paths under crates/polars-time/src).
`python tests/golden/transcribe_rolling_by.py` writes rolling_by_kats.json next to this file.

A case: values (None = null) and their dtype, kind (one of polars_b200.ROLLINGS), `by` (physical Int64: a Date as days x
86 400 000 000 us, as the reference casts it to Datetime(us); None = null), its dtype, window_size in that unit, closed,
min_samples, ddof, partition keys (`parts`, may be empty) and the expected output (None = null).  A case with "windows"
pins the (start, len) pairs of the window iterator instead of an aggregate; one with "error" expects the call to fail.

Reference tests that cannot be expressed as a case, or only in part:
- operations/rolling/test_rolling.py:304-321 test_rolling_by_invalid / :324-331 test_rolling_by_non_temporal_window_size:
  the Int16 `by` is an error case below; the "2i" window over a Date column is a ValueError of the Python binding
  (window_size_in), which has no C ABI form (the C ABI takes window_size in the physical unit), so it is checked in
  tests/test_rolling_by.py.
- windows/test.rs:742-764, the "partial lookbehind" half of test_rolling_lookback: an offset other than -period is
  `DataFrame.rolling(offset=...)`, not rolling_*_by.
- windows/test.rs:864-930 (test_group_by_windows_membership_2791, _duplicates_2931, _offsets_3776) and
  group_by/dynamic.rs:497-620 (test_rolling_group_by_tu, test_rolling_group_by_aggs): group_by_dynamic / DataFrame.rolling
  with offsets, every / period pairs or list aggregations, outside rolling_*_by.
- operations/rolling/test_rolling.py test_rolling_by_1mo_saturating_12216 and the other calendar (mo / q / y) and
  time-zone-aware cases: calendar durations are not expressible on the device.
"""
import json
import os

DAY_US = 86_400_000_000
CASES = []


def days(*ds):
    """dates as day numbers from 2020-01-01 (the tests' dates differ only by days) -> Datetime(us)"""
    return [None if d is None else d * DAY_US for d in ds]


def case(src, kind, values, vdtype, by, bdtype, window_size, closed, min_samples, expected, parts=(), ddof=1, **extra):
    CASES.append(dict(src=src, kind=kind, values=values, dtype=vdtype, by=by, by_dtype=bdtype, window_size=window_size, closed=closed,
                      min_samples=min_samples, ddof=ddof, parts=[list(p) for p in parts], expected=expected, **extra))


T = "py-polars/tests/unit/operations/rolling/test_rolling.py"
# test_rolling_by_date: "2d" over Date, min_samples default 0 for rolling_sum_by
case(f"{T}:1019-1029", "rolling_sum", [1, 2, 3], "int64", days(0, 1, 2), "int64", 2 * DAY_US, "right", 0, [1, 3, 5])
# test_rolling_by_integer: "2i" over Int64 / Int32 / UInt64 / UInt32 row indices
for bd in ("int64", "int32", "uint64", "uint32"):
    case(f"{T}:1032-1041", "rolling_sum", [1, 2, 3], "int64", [0, 1, 2], bd, 2, "right", 0, [1, 3, 5])
# test_rolling_sum_by_integer: every integer value dtype; Int8 / Int16 / UInt8 / UInt16 sum as Int64
for vd in ("int8", "int16", "int32", "int64", "uint8", "uint16", "uint32", "uint64"):
    case(f"{T}:1044-1057", "rolling_sum", [1, 2, 3], vd, [0, 1, 2], "uint32", 2, "right", 0, [1, 3, 5])
# test_rolling_aggregations_with_over_11225: rolling_mean_by("date", "2d", closed="left").over("group") of the row index
case(f"{T}:867-897", "rolling_mean", [0, 1, 2, 3, 4], "uint32", days(0, 1, 2, 3, 4), "int64", 2 * DAY_US, "left", 1,
     [None, 0.0, None, 2.0, 2.5], parts=[["A", "A", "B", "B", "B"]])
# test_rolling_min_samples: rolling_sum_by("date", "2d", min_samples=2, closed=...) of [1, 2, 3]; each case twice, as the
# test does: sorted, and from the rows in descending date order (an unsorted `by`)
MS = [((0, 1, 2), "right", [None, 3, 5]), ((0, 1, 2), "left", [None, None, 3]), ((0, 1, 2), "both", [None, 3, 6]),
      ((0, 1, 2), "none", [None, None, None]), ((0, 1, 3), "right", [None, 3, None]), ((0, 2, 3), "right", [None, None, 5]),
      ((0, 2, 4), "right", [None, None, None])]
for k, (ds, closed, exp) in enumerate(MS):
    line = 1170 + 5 * k
    case(f"{T}:{line}-{line + 4},1207-1218", "rolling_sum", [1, 2, 3], "int64", days(*ds), "int64", 2 * DAY_US, closed, 2, exp)
    case(f"{T}:{line}-{line + 4},1219-1229", "rolling_sum", [3, 2, 1], "int64", days(*ds[::-1]), "int64", 2 * DAY_US, closed, 2, exp[::-1])
# test_rolling_by_invalid: an Int16 `by` is InvalidOperation
case(f"{T}:304-313", "rolling_min", [4, 5, 6], "int64", [1, 2, 3], "int16", 2, "right", 1, None, error=True)
# windows/test.rs test_rolling_lookback, full lookbehind: "2h" right-closed over 30-minute steps in ms, (start, len) pairs
case("crates/polars-time/src/windows/test.rs:699-740", "rolling_sum", [1] * 9, "int64", [k * 1_800_000 for k in range(9)], "int64",
     7_200_000, "right", 0, [1, 2, 3, 4, 4, 4, 4, 4, 4],
     windows=[[0, 1], [0, 2], [0, 3], [0, 4], [1, 4], [2, 4], [3, 4], [4, 4], [5, 4]])

if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "rolling_by_kats.json")
    with open(path, "w") as f:
        json.dump(CASES, f, indent=1)
        f.write("\n")
    print(f"wrote {len(CASES)} cases to {path}")
