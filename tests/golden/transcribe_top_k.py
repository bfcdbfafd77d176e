"""Writes tests/golden/top_k_kats.json: known answers of the reference's top_k / bottom_k / top_k_by / bottom_k_by tests and
of a sort with a limit, transcribed by hand with the file:line of each case (paths relative to the reference's repository
root).

Every case: frame (column name -> values, None = null; a column of str values is a string column), dtypes (column name ->
"int64", "float64", "bool" or "str"), op ("top_k" / "bottom_k" of one column, "top_k_by" / "bottom_k_by" of payload
columns by `by` with `reverse`, or "sort" = sort(by, descending, nulls_last).head(k)), k, expected (column name -> values)
and order: "pinned" when the reference test compares the row order, "multiset" when it compares with check_order=False /
check_row_order=False or sorts the result first.

Not transcribed: the `pl.lit(None)` / length-2 `k` errors (test_top_k.py:86-92: `k` is a Python int here), the
group_by().agg(top_k_by) cases (:198-225, list output is out of scope), the hypothesis tests (:404-436: their null-count
rules are checked on random inputs by tests/test_gpu_top_k.py) and the struct / categorical cases."""
import json
import os

PY = "py-polars/tests/unit/operations/test_top_k.py"
SORT = "py-polars/tests/unit/operations/test_sort.py"
D1 = {"test": [2, 4, 1, 3], "val": [2, 4, 9, 3], "bool_val": [False, True, True, False], "str_value": ["d", "b", "a", "c"]}
D1T = {"test": "int64", "val": "int64", "bool_val": "bool", "str_value": "str"}
AB = {"a": [1, 2, 3, 4, 2, 2, None], "b": [None, 2, 1, 4, 3, 2, None]}
ABT = {"a": "int64", "b": "int64"}
D2 = {"a": [1, 2, 3, 4, 5, 6], "b": [12, 11, 10, 9, 8, 7], "c": ["Apple", "Orange", "Apple", "Apple", "Banana", "Banana"]}
D2T = {"a": "int64", "b": "int64", "c": "str"}
TD = [3, 4, 1, 2, 5]
TD2 = [1, None, None, 4, 5]

CASES = [
    dict(src=f"{PY}:39", frame={"a": [3, 8, 1, 5, 2]}, dtypes={"a": "int64"}, op="top_k", col="a", k=3, expected={"a": [8, 5, 3]}, order="multiset"),
    dict(src=f"{PY}:40", frame={"a": [3, 8, 1, 5, 2]}, dtypes={"a": "int64"}, op="bottom_k", col="a", k=4, expected={"a": [3, 2, 1, 5]}, order="multiset"),
    dict(src=f"{PY}:51-55", frame=D1, dtypes=D1T, op="top_k", col="test", k=10, expected={"test": [4, 3, 2, 1]}, order="multiset"),
    dict(src=f"{PY}:57-63", frame=D1, dtypes=D1T, op="top_k", col="test", k=2, expected={"test": [3, 4]}, order="multiset"),
    dict(src=f"{PY}:57-63", frame=D1, dtypes=D1T, op="bottom_k", col="test", k=2, expected={"test": [1, 2]}, order="multiset"),
    dict(src=f"{PY}:65-72", frame=D1, dtypes=D1T, op="top_k", col="bool_val", k=2, expected={"bool_val": [True, True]}, order="multiset"),
    dict(src=f"{PY}:65-72", frame=D1, dtypes=D1T, op="bottom_k", col="bool_val", k=2, expected={"bool_val": [False, False]}, order="multiset"),
    dict(src=f"{PY}:74-78", frame=D1, dtypes=D1T, op="top_k", col="str_value", k=2, expected={"str_value": ["d", "c"]}, order="multiset"),
    dict(src=f"{PY}:80-84", frame=D1, dtypes=D1T, op="bottom_k", col="str_value", k=2, expected={"str_value": ["a", "b"]}, order="multiset"),
    dict(src=f"{PY}:102-106", frame=AB, dtypes=ABT, op="top_k_by", cols=["a", "b"], by=["a", "b"], k=3, reverse=False,
         expected={"a": [4, 3, 2], "b": [4, 1, 3]}, order="multiset"),
    dict(src=f"{PY}:108-112", frame=AB, dtypes=ABT, op="top_k_by", cols=["a", "b"], by=["a", "b"], k=3, reverse=True,
         expected={"a": [1, 2, 2], "b": [None, 2, 2]}, order="multiset"),
    dict(src=f"{PY}:113-117", frame=AB, dtypes=ABT, op="bottom_k_by", cols=["a", "b"], by=["a", "b"], k=4, reverse=True,
         expected={"a": [4, 3, 2, 2], "b": [4, 1, 3, 2]}, order="multiset"),
    dict(src=f"{PY}:124-140", frame=D2, dtypes=D2T, op="top_k_by", cols=["a", "b"], by=["a"], k=2, reverse=False, expected={"a": [5, 6], "b": [7, 8]}, order="multiset"),
    dict(src=f"{PY}:124-140", frame=D2, dtypes=D2T, op="top_k_by", cols=["a", "b"], by=["b"], k=2, reverse=False, expected={"a": [1, 2], "b": [11, 12]}, order="multiset"),
    dict(src=f"{PY}:142-161", frame=D2, dtypes=D2T, op="top_k_by", cols=["a", "b"], by=["a"], k=2, reverse=True, expected={"a": [1, 2], "b": [11, 12]}, order="multiset"),
    dict(src=f"{PY}:142-161", frame=D2, dtypes=D2T, op="top_k_by", cols=["a", "b"], by=["b"], k=2, reverse=True, expected={"a": [5, 6], "b": [7, 8]}, order="multiset"),
    dict(src=f"{PY}:163-176", frame=D2, dtypes=D2T, op="bottom_k_by", cols=["a", "b"], by=["a"], k=2, reverse=False, expected={"a": [1, 2], "b": [11, 12]}, order="multiset"),
    dict(src=f"{PY}:163-176", frame=D2, dtypes=D2T, op="bottom_k_by", cols=["a", "b"], by=["b"], k=2, reverse=False, expected={"a": [5, 6], "b": [7, 8]}, order="multiset"),
    dict(src=f"{PY}:178-193", frame=D2, dtypes=D2T, op="bottom_k_by", cols=["a", "b"], by=["a"], k=2, reverse=True, expected={"a": [5, 6], "b": [7, 8]}, order="multiset"),
    dict(src=f"{PY}:178-193", frame=D2, dtypes=D2T, op="bottom_k_by", cols=["a", "b"], by=["b"], k=2, reverse=True, expected={"a": [1, 2], "b": [11, 12]}, order="multiset"),
    dict(src=f"{PY}:227-246", frame=D2, dtypes=D2T, op="top_k_by", cols=["a", "b", "c"], by=["c", "a"], k=2, reverse=False,
         expected={"a": [2, 6], "b": [11, 7], "c": ["Orange", "Banana"]}, order="multiset"),
    dict(src=f"{PY}:227-246", frame=D2, dtypes=D2T, op="top_k_by", cols=["a", "b", "c"], by=["c", "b"], k=2, reverse=False,
         expected={"a": [2, 5], "b": [11, 8], "c": ["Orange", "Banana"]}, order="multiset"),
    dict(src=f"{PY}:379-383", frame={"a": [1, 2, 3], "b": [4, 5, 6]}, dtypes=ABT, op="top_k_by", cols=["a", "b"], by=["a", "b"], k=1, reverse=True,
         expected={"a": [1], "b": [4]}, order="multiset"),
    dict(src=f"{PY}:384-385", frame={"a": [1, 2, 3], "b": [4, 5, 6]}, dtypes=ABT, op="top_k_by", cols=["a", "b"], by=["a", "b"], k=1, reverse=[True, True],
         expected={"a": [1], "b": [4]}, order="multiset"),
    dict(src=f"{PY}:393-396", frame={"b": [True, False]}, dtypes={"b": "bool"}, op="sort", by=["b"], descending=False, nulls_last=False, k=1,
         expected={"b": [False]}, order="pinned"),
    dict(src=f"{PY}:399-402", frame={"test": []}, dtypes={"test": "int64"}, op="top_k", col="test", k=2, expected={"test": []}, order="pinned"),
    # test_top_k_df: the same answers for the frame as given and sorted either way (:444-462)
    dict(src=f"{PY}:471-472", frame={"a": TD}, dtypes={"a": "int64"}, op="top_k_by", cols=["a"], by=["a"], k=3, reverse=False, expected={"a": [5, 4, 3]}, order="pinned"),
    dict(src=f"{PY}:474-475", frame={"a": TD}, dtypes={"a": "int64"}, op="bottom_k_by", cols=["a"], by=["a"], k=3, reverse=False, expected={"a": [1, 2, 3]}, order="pinned"),
    dict(src=f"{PY}:479-483", frame={"a": TD2}, dtypes={"a": "int64"}, op="top_k_by", cols=["a"], by=["a"], k=4, reverse=False, expected={"a": [5, 4, 1, None]}, order="pinned"),
    dict(src=f"{PY}:484-492", frame={"a": TD2}, dtypes={"a": "int64"}, op="bottom_k_by", cols=["a"], by=["a"], k=4, reverse=False, expected={"a": [1, 4, 5, None]}, order="pinned"),
    dict(src=f"{PY}:494-496", frame={"a": TD2}, dtypes={"a": "int64"}, op="sort", by=["a"], descending=False, nulls_last=False, k=4, expected={"a": [None, None, 1, 4]}, order="pinned"),
    dict(src=f"{PY}:497-499", frame={"a": TD2}, dtypes={"a": "int64"}, op="sort", by=["a"], descending=True, nulls_last=False, k=4, expected={"a": [None, None, 5, 4]}, order="pinned"),
    dict(src=f"{PY}:479-481", frame={"a": TD2}, dtypes={"a": "int64"}, op="sort", by=["a"], descending=True, nulls_last=True, k=4, expected={"a": [5, 4, 1, None]}, order="pinned"),
    # test_sort_top_k_fast_path: head(3) of sort("b") over three rows
    dict(src=f"{SORT}:858-871", frame={"a": [1, 2, None], "b": [6.0, 5.0, 4.0], "c": ["a", "c", "b"]}, dtypes={"a": "int64", "b": "float64", "c": "str"},
         op="sort", by=["b"], descending=False, nulls_last=False, k=3, expected={"a": [None, 2, 1], "b": [4.0, 5.0, 6.0], "c": ["b", "c", "a"]}, order="pinned"),
]

if __name__ == "__main__":
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "top_k_kats.json")
    with open(out, "w") as f:
        json.dump(CASES, f, indent=1)
    print(f"wrote {len(CASES)} cases to {out}")
