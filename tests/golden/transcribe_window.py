"""Known answers of the reference's window / cumulative functions, transcribed by hand from its own tests, each with its
file:line (paths under py-polars/tests/unit of the reference).  `python tests/golden/transcribe_window.py` writes
window_kats.json next to this file.

A case: columns (name -> list, None = null) with their dtypes ("str" = a string column), ops [[output name, kind, value
column, options]], partition_by (column names), order_by (a column name or null), descending, nulls_last, expected (output
name -> list).  Kinds are those of polars_b200.over().  Optional: rows (only these rows are pinned by the reference test),
rtol (the reference compares with np.isclose: |got - expected| <= 1e-8 + rtol * |expected|), equal (pairs of outputs the
reference test asserts to be equal, without stating their value).

Reference tests named for this transcription that cannot be expressed as a case:
- operations/test_window.py:433-446 test_sorted_window_expression: the windowed expression is elementwise (`a + b`), not an
  aggregation, scan or shift, and its data are random; the test asserts that sorting the frame first does not change it.
- operations/test_over.py:146-148, :156-158 (test_first_last_over with ignore_nulls=True): first / last skipping nulls is
  not a kind of bl_over (BL_AGG_FIRST / LAST take the value at the group's first / last row, nulls included).  The other
  two halves of that test are transcribed below.
- operations/test_shift.py: every case with a fill_value (:17, :24, :52-63, :74-76, :84-85, :91-93, :104-112,
  :127-129, :138-145, :161-187) — BL_SHIFT gives null outside the partition and has no fill value; shift(None) (:132-145),
  whose periods is null; Object / Categorical / List columns (:20-25, :88-93, :190-194); a frame-level shift of string
  columns (:33-49).  The integer-column cases without a fill value are transcribed below."""
import json
import os

INF = float("inf")
NAN = float("nan")
CASES = [
    # series/test_series.py:45-51 test_cum_agg
    dict(src="series/test_series.py:45-51 test_cum_agg", columns={"a": [1, 2, 3, 2]}, dtypes={"a": "int64"},
         ops=[["s", "cum_sum", "a", {}], ["mn", "cum_min", "a", {}], ["mx", "cum_max", "a", {}], ["p", "cum_prod", "a", {}]],
         expected={"s": [1, 3, 6, 8], "mn": [1, 1, 1, 1], "mx": [1, 2, 3, 3], "p": [1, 2, 6, 12]}),
    # series/test_series.py:54-60 test_cum_agg_with_nulls
    dict(src="series/test_series.py:54-60 test_cum_agg_with_nulls", columns={"a": [None, 2, None, 7, 8, None]}, dtypes={"a": "int64"},
         ops=[["s", "cum_sum", "a", {}], ["mn", "cum_min", "a", {}], ["mx", "cum_max", "a", {}], ["p", "cum_prod", "a", {}]],
         expected={"s": [None, 2, None, 9, 17, None], "mn": [None, 2, None, 2, 2, None], "mx": [None, 2, None, 7, 8, None],
                   "p": [None, 2, None, 14, 112, None]}),
    # series/test_series.py:63-69 test_cum_agg_with_infs
    dict(src="series/test_series.py:63-66 test_cum_agg_with_infs", columns={"a": [INF, 0.0, 1.0]}, dtypes={"a": "float64"},
         ops=[["mn", "cum_min", "a", {}]], expected={"mn": [INF, 0.0, 0.0]}),
    dict(src="series/test_series.py:68-69 test_cum_agg_with_infs", columns={"a": [-INF, 0.0, 1.0]}, dtypes={"a": "float64"},
         ops=[["mx", "cum_max", "a", {}]], expected={"mx": [-INF, 0.0, 1.0]}),
    # operations/test_window.py:669-689 test_window_order_by_8662
    dict(src="operations/test_window.py:669-689 test_window_order_by_8662",
         columns={"g": [1, 1, 1, 1, 2, 2, 2, 2], "t": [1, 2, 3, 4, 4, 1, 2, 3], "x": [10, 20, 30, 40, 10, 20, 30, 40]},
         dtypes={"g": "int64", "t": "int64", "x": "int64"},
         ops=[["x_lag0", "shift", "x", {"periods": 1}]], partition_by=["g"],
         expected={"x_lag0": [None, 10, 20, 30, None, 10, 20, 30]}),
    dict(src="operations/test_window.py:669-689 test_window_order_by_8662",
         columns={"g": [1, 1, 1, 1, 2, 2, 2, 2], "t": [1, 2, 3, 4, 4, 1, 2, 3], "x": [10, 20, 30, 40, 10, 20, 30, 40]},
         dtypes={"g": "int64", "t": "int64", "x": "int64"},
         ops=[["x_lag1", "shift", "x", {"periods": 1}]], partition_by=["g"], order_by="t",
         expected={"x_lag1": [None, 10, 20, 30, 40, None, 20, 30]}),
    dict(src="operations/test_window.py:669-689 test_window_order_by_8662",
         columns={"g": [1, 1, 1, 1, 2, 2, 2, 2], "t": [1, 2, 3, 4, 4, 1, 2, 3], "x": [10, 20, 30, 40, 10, 20, 30, 40]},
         dtypes={"g": "int64", "t": "int64", "x": "int64"},
         ops=[["x_lag2", "shift", "x", {"periods": 1}]], partition_by=["g"], order_by="t", descending=True,
         expected={"x_lag2": [20, 30, 40, None, None, 30, 40, 10]}),
    # operations/test_over.py:36-40 test_over_no_partition_by
    dict(src="operations/test_over.py:36-40 test_over_no_partition_by", columns={"a": [1, 1, 2], "i": [2, 1, 3]}, dtypes={"a": "int64", "i": "int64"},
         ops=[["b", "cum_sum", "a", {}]], order_by="i", expected={"b": [2, 1, 4]}),
    # operations/test_window.py:18-40 test_over_args
    dict(src="operations/test_window.py:18-31 test_over_args (single input)", columns={"a": ["a", "a", "b"], "b": [1, 2, 3], "c": [3, 2, 1]},
         dtypes={"a": "str", "b": "int64", "c": "int64"}, ops=[["c", "max", "c", {}]], partition_by=["a"], expected={"c": [3, 3, 1]}),
    dict(src="operations/test_window.py:33-40 test_over_args (several inputs)", columns={"a": ["a", "a", "b"], "b": [1, 2, 3], "c": [3, 2, 1]},
         dtypes={"a": "str", "b": "int64", "c": "int64"}, ops=[["c", "max", "c", {}]], partition_by=["a", "b"], expected={"c": [3, 2, 1]}),
    # operations/test_window.py:42-65 test_std, parametrized over Float32, Float64, Int32; only row 0 is checked, with np.isclose
    *[dict(src=f"operations/test_window.py:42-65 test_std[{dt}]", columns={"groups": ["a", "a", "b", "b"], "values": [1, 2, 3, 4] if dt == "int32" else [1.0, 2.0, 3.0, 4.0]},
           dtypes={"groups": "str", "values": dt}, partition_by=["groups"], rows=[0], rtol=1e-5,
           ops=[["std", "std", "values", {}], ["var", "var", "values", {}], ["mean", "mean", "values", {}]],
           expected={"std": [0.7071067690849304, None, None, None], "var": [0.5, None, None, None], "mean": [1.5, None, None, None]})
      for dt in ("float32", "float64", "int32")],
    # operations/test_window.py:68-85 test_issue_2529: mean / std over `cat` of two equal columns must agree (no value stated)
    dict(src="operations/test_window.py:68-85 test_issue_2529", columns={"cat": [0, 0, 1, 1], "val1": [0, 1, 1, 2], "val2": [0, 1, 1, 2]},
         dtypes={"cat": "int64", "val1": "int64", "val2": "int64"}, partition_by=["cat"],
         ops=[["m1", "mean", "val1", {}], ["m2", "mean", "val2", {}], ["s1", "std", "val1", {}], ["s2", "std", "val2", {}]],
         equal=[["m1", "m2"], ["s1", "s2"]], expected={}),
    # operations/test_window.py:138-150 test_no_panic_on_nan_3067
    dict(src="operations/test_window.py:138-150 test_no_panic_on_nan_3067", columns={"group": ["a", "a", "a", "b", "b", "b"], "total": [1.0, 2.0, 3.0, 4.0, 5.0, NAN]},
         dtypes={"group": "str", "total": "float64"}, partition_by=["group"], ops=[["total", "shift", "total", {"periods": 1}]],
         expected={"total": [None, 1.0, 2.0, None, 4.0, 5.0]}),
    # operations/test_window.py:153-165 test_quantile_as_window (pl.quantile's default method: nearest)
    dict(src="operations/test_window.py:153-165 test_quantile_as_window", columns={"group": [0, 0, 1, 1], "value": [0, 1, 0, 2]},
         dtypes={"group": "int64", "value": "int64"}, partition_by=["group"], ops=[["value", "quantile:0.9:nearest", "value", {}]],
         expected={"value": [1.0, 1.0, 2.0, 2.0]}),
    # operations/test_window.py:383-392 test_len_window
    dict(src="operations/test_window.py:383-392 test_len_window", columns={"a": [1, 1, 2]}, dtypes={"a": "int64"}, partition_by=["a"],
         ops=[["len", "len", None, {}]], expected={"len": [2, 2, 1]}),
    # operations/test_over.py:138-164 test_first_last_over (ignore_nulls=False halves)
    dict(src="operations/test_over.py:138-152 test_first_last_over (first)", columns={"a": [1, 1, 1, 1, 2, 2, 2, 2], "b": [1, 2, 3, None, None, 4, 5, 6]},
         dtypes={"a": "int64", "b": "int32"}, partition_by=["a"], ops=[["b", "first", "b", {}]], expected={"b": [1, 1, 1, 1, None, None, None, None]}),
    dict(src="operations/test_over.py:138-143,150-154 test_first_last_over (last)", columns={"a": [1, 1, 1, 1, 2, 2, 2, 2], "b": [1, 2, 3, None, None, 4, 5, 6]},
         dtypes={"a": "int64", "b": "int32"}, partition_by=["a"], ops=[["b", "last", "b", {}]], expected={"b": [None, None, None, None, 6, 6, 6, 6]}),
    # operations/test_over.py:167-190 test_nulls_last_over_24989: the expected frame is sorted by `i` (rows 1, 0, 2); here in row order
    dict(src="operations/test_over.py:167-190 test_nulls_last_over_24989", columns={"a": [1, 1, 2], "b": [4, 5, 6], "c": [None, 7, 8], "i": [1, None, 2]},
         dtypes={"a": "int64", "b": "int64", "c": "int64", "i": "int64"}, partition_by=["a"], order_by="i", nulls_last=True,
         ops=[["b_first", "first", "b", {}], ["c_first", "first", "c", {}]], expected={"b_first": [4, 4, 6], "c_first": [None, None, 8]}),
    # operations/test_shift.py
    *[dict(src=f"operations/test_shift.py:12-16 test_shift (periods {k})", columns={"a": [1, 2, 3]}, dtypes={"a": "int64"},
           ops=[["a", "shift", "a", {"periods": k}]], expected={"a": e})
      for k, e in ((1, [None, 1, 2]), (-1, [2, 3, None]), (-2, [3, None, None]))],
    dict(src="operations/test_shift.py:28-31 test_shift_frame", columns={"a": [1, 2, 3, 4, 5]}, dtypes={"a": "int64"},
         ops=[["a", "shift", "a", {"periods": 1}]], expected={"a": [None, 1, 2, 3, 4]}),
    dict(src="operations/test_shift.py:66-82 test_shift_expr (n = min(b) = 1; n = 3)", columns={"a": [1, 2, 3, 4, 5], "b": [1, 2, 3, 4, 5]},
         dtypes={"a": "int64", "b": "int64"}, ops=[["a1", "shift", "a", {"periods": 1}], ["a3", "shift", "a", {"periods": 3}], ["b3", "shift", "b", {"periods": 3}]],
         expected={"a1": [None, 1, 2, 3, 4], "a3": [None, None, None, 1, 2], "b3": [None, None, None, 1, 2]}),
    dict(src="operations/test_shift.py:197-210 test_streaming_shift_25226", columns={"a": [1, 2, 3, 4]}, dtypes={"a": "int64"},
         ops=[["b", "shift", "a", {"periods": 1}], ["b_neg", "shift", "a", {"periods": -1}], ["c", "min", "a", {}]],
         expected={"b": [None, 1, 2, 3], "b_neg": [2, 3, 4, None], "c": [1, 1, 1, 1]}),
]

def main():
    out = []
    for c in CASES:
        c = dict(c)
        c.setdefault("partition_by", [])
        c.setdefault("order_by", None)
        c.setdefault("descending", False)
        c.setdefault("nulls_last", False)
        out.append(c)
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "window_kats.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, allow_nan=True)
        f.write("\n")
    print("wrote", path, len(out), "cases")


if __name__ == "__main__":
    main()
