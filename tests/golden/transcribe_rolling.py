"""Known answers of the reference's fixed-window rolling aggregations, transcribed by hand from its own tests, each with
its file:line (py-polars paths under py-polars/tests/unit, Rust paths under crates/polars-compute/src/rolling).
`python tests/golden/transcribe_rolling.py` writes rolling_kats.json next to this file.

A case: values (None = null), dtype, kind (one of polars_b200.ROLLINGS), window_size, min_samples, center, ddof and the
expected output (None = null).

Reference tests named for this transcription that cannot be expressed as a case, or only in part:
- operations/rolling/test_rolling.py:867-900 test_rolling_aggregations_with_over_11225: a temporal `rolling_mean_by` with
  `closed="left"`, a duration window; `_by` windows are outside bl_rolling.
- operations/rolling/test_rolling.py:1195-1215 test_rolling_min_samples: `rolling_sum_by` over dates with a duration
  window and `closed`; `_by` windows are outside bl_rolling.
- operations/rolling/test_rolling.py:1935-1952 test_rolling_sum_non_finite_23115: random data checked against a naive sum;
  tests/test_rolling.py restates it as a property over seeded data (non-finite class of every window).
- operations/rolling/test_rolling.py:396-416, the shuffled half of test_rolling_extrema: its rows come from
  `shuffle(seed=0)`, whose permutation the test does not state.  The sorted half is transcribed below for the numeric
  dtypes of its parametrization (the temporal ones roll their physical Int64 / Int32).
- The reference has no unweighted centered rolling var / std / min / max test (every centered case at
  test_rolling.py:1853-1914 has weights); centered windows are pinned by the centered sums of nulls/mod.rs and
  no_nulls/sum.rs below.
- weights, rolling_*_by, rolling_quantile / median / rank / skew / kurtosis and temporal dtypes: outside bl_rolling."""
import json
import os

NAN = float("nan")
NULL_ARR = [1.0, None, -1.0, 4.0]       # nulls/mod.rs:107-115 get_null_arr
CASES = []


def case(src, values, dtype, kind, w, ms, expected, center=False, ddof=1):
    CASES.append(dict(src=src, values=values, dtype=dtype, kind=kind, window_size=w, min_samples=ms, center=center, ddof=ddof,
                      expected=expected))


S = "nulls/mod.rs:121-154 test_rolling_sum_nulls"
arr = [1.0, None, 3.0, 4.0]
case(S, arr, "float64", "rolling_sum", 2, 2, [None, None, None, 7.0])
case(S, arr, "float64", "rolling_sum", 2, 1, [1.0, 1.0, 3.0, 7.0])
case(S, arr, "float64", "rolling_sum", 4, 1, [1.0, 1.0, 4.0, 8.0])
case(S, arr, "float64", "rolling_sum", 4, 1, [1.0, 4.0, 8.0, 7.0], center=True)
case(S, arr, "float64", "rolling_sum", 4, 4, [None, None, None, None], center=True)
S = "nulls/mod.rs:156-175 test_rolling_mean_nulls"
case(S, NULL_ARR, "float64", "rolling_mean", 2, 2, [None, None, None, 1.5])
case(S, NULL_ARR, "float64", "rolling_mean", 2, 1, [1.0, 1.0, -1.0, 1.5])
case(S, NULL_ARR, "float64", "rolling_mean", 4, 1, [1.0, 1.0, 0.0, 4.0 / 3.0])
S = "nulls/mod.rs:177-207 test_rolling_var_nulls"
case(S, NULL_ARR, "float64", "rolling_var", 3, 1, [None, None, 2.0, 12.5])
case(S, NULL_ARR, "float64", "rolling_var", 3, 1, [0.0, 0.0, 1.0, 6.25], ddof=0)
case(S, NULL_ARR, "float64", "rolling_var", 4, 1, [None, None, 2.0, 6.333333333333334])
case(S, NULL_ARR, "float64", "rolling_var", 4, 1, [0.0, 0.0, 1.0, 4.222222222222222], ddof=0)
S = "nulls/mod.rs:209-247 test_rolling_max_no_nulls"
case(S, [1.0, 2.0, 3.0, 4.0], "float64", "rolling_max", 4, 1, [1.0, 2.0, 3.0, 4.0])
case(S, [1.0, 2.0, 3.0, 4.0], "float64", "rolling_max", 2, 2, [None, 2.0, 3.0, 4.0])
case(S, [1.0, 2.0, 3.0, 4.0], "float64", "rolling_max", 4, 4, [None, None, None, 4.0])
case(S, [4.0, 3.0, 2.0, 1.0], "float64", "rolling_max", 2, 1, [4.0, 4.0, 3.0, 2.0])
S = "nulls/mod.rs:249-272 test_rolling_extrema_nulls"
case(S, [3, 3, 3, 10, 10, 10, 9, 8, 7, 6, 5, 4, 3, 2, 1], "int32", "rolling_max", 3, 3,
     [None, None, 3, 10, 10, 10, 10, 10, 9, 8, 7, 6, 5, 4, 3])
S = "operations/rolling/test_rolling.py:984-989 test_rolling_std_nulls_min_samples_1_20076"
case(S, [1, 2, None, 4], "int64", "rolling_std", 3, 1, [None, 0.7071067811865476, 0.7071067811865476, 1.4142135623730951])

S = "no_nulls/sum.rs:69-118 test_rolling_sum"
vals = [1.0, 2.0, 3.0, 4.0]
case(S, vals, "float64", "rolling_sum", 2, 2, [None, 3.0, 5.0, 7.0])
case(S, vals, "float64", "rolling_sum", 2, 1, [1.0, 3.0, 5.0, 7.0])
case(S, vals, "float64", "rolling_sum", 4, 1, [1.0, 3.0, 6.0, 10.0])
case(S, vals, "float64", "rolling_sum", 4, 1, [3.0, 6.0, 10.0, 9.0], center=True)
case(S, vals, "float64", "rolling_sum", 4, 4, [None, None, 10.0, None], center=True)
NANS = [1.0, 2.0, 3.0, NAN, 5.0, 6.0, 7.0]
case(S, NANS, "float64", "rolling_sum", 3, 3, [None, None, 6.0, NAN, NAN, NAN, 18.0])
S = "no_nulls/min_max.rs:78-145 test_rolling_min_max"
vals = [1.0, 5.0, 3.0, 4.0]
case(S, vals, "float64", "rolling_min", 2, 2, [None, 1.0, 3.0, 3.0])
case(S, vals, "float64", "rolling_max", 2, 2, [None, 5.0, 5.0, 4.0])
case(S, vals, "float64", "rolling_min", 2, 1, [1.0, 1.0, 3.0, 3.0])
case(S, vals, "float64", "rolling_max", 2, 1, [1.0, 5.0, 5.0, 4.0])
case(S, vals, "float64", "rolling_max", 3, 1, [1.0, 5.0, 5.0, 5.0])
case(S, NANS, "float64", "rolling_min", 3, 3, [None, None, 1.0, NAN, NAN, NAN, 5.0])
case(S, NANS, "float64", "rolling_max", 3, 3, [None, None, 3.0, NAN, NAN, NAN, 7.0])
S = "no_nulls/moment.rs:104-148 test_rolling_var"
case(S, vals, "float64", "rolling_var", 2, 2, [None, 8.0, 2.0, 0.5])
case(S, vals, "float64", "rolling_var", 2, 2, [None, 4.0, 1.0, 0.25], ddof=0)
case(S, vals, "float64", "rolling_var", 2, 1, [None, 8.0, 2.0, 0.5])
case(S, [-10.0, 2.0, 3.0, NAN, 5.0, 6.0, 7.0], "float64", "rolling_var", 3, 3, [None, None, 52.33333333333333, NAN, NAN, NAN, 1.0])
S = "operations/rolling/test_rolling.py:351-395 test_rolling_extrema (sorted frame)"
up, down = list(range(7)), list(range(6, -1, -1))
for dt in ("uint8", "int64", "float32", "float64"):
    conv = float if dt.startswith("float") else int
    u, d = [conv(v) for v in up], [conv(v) for v in down]
    un, dn = [None, None] + u[2:], [None, None] + d[2:]
    E = lambda xs: [None if v is None else conv(v) for v in xs]      # noqa: E731
    case(S, u, dt, "rolling_min", 3, 3, E([None, None, 0, 1, 2, 3, 4]))
    case(S, d, dt, "rolling_min", 3, 3, E([None, None, 4, 3, 2, 1, 0]))
    case(S, un, dt, "rolling_min", 3, 3, E([None, None, None, None, 2, 3, 4]))
    case(S, dn, dt, "rolling_min", 3, 3, E([None, None, None, None, 2, 1, 0]))
    case(S, u, dt, "rolling_max", 3, 3, E([None, None, 2, 3, 4, 5, 6]))
    case(S, d, dt, "rolling_max", 3, 3, E([None, None, 6, 5, 4, 3, 2]))
    case(S, un, dt, "rolling_max", 3, 3, E([None, None, None, None, 4, 5, 6]))
    case(S, dn, dt, "rolling_max", 3, 3, E([None, None, None, None, 4, 3, 2]))

if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "rolling_kats.json")
    with open(path, "w") as f:
        json.dump(CASES, f, indent=1)
        f.write("\n")
    print(f"wrote {len(CASES)} cases to {path}")
