"""Writes tests/golden/unique_kats.json: known answers of the reference's unique / is_unique / is_duplicated /
is_first_distinct / is_last_distinct tests, transcribed by hand with the file:line of each case (paths relative to the
reference's repository root).

Every case has a frame (column name -> values, None = null; `int_range` n stands for the frame {"x": 0 .. n - 1} and the
same expected column) and dtypes (column name -> "int64", "float64", "bool" or
"str"; a column of the reference's Null dtype is an all-null "int64" column here).  A column named in `prefix` is built
from prefix + values and then sliced past the prefix, as the reference's `.slice(k)` / `.head(k)` does, so that its
Boolean bits start at a bit offset.  Then either
  op "unique": DataFrame.unique(subset, keep, maintain_order).slice(*slice) -> expected (column name -> values) with
               order "pinned" when the reference compares the row order and "multiset" when it does not
               (maintain_order=False, check_order=False or a height check);
  op "mask":   kind ("unique", "duplicated", "first", "last") over the key columns `keys` -> expected (one bool per row).

Not transcribed: the list / array / struct / Int128 / categorical / enum cases, the bad-subset errors
(test_unique.py:197-222: column names are not part of the device call), the predicate-pushdown and agg-context cases
(test_unique.py:18-62, :281-291, :388-401: they test the query optimiser) and Series.unique on an empty series of each
dtype (test_unique.py:108-111: covered by the n = 0 cases of tests/test_gpu_unique.py)."""
import json
import os

U = "py-polars/tests/unit/operations/unique/test_unique.py"
IU = "py-polars/tests/unit/operations/unique/test_is_unique.py"
FL = "py-polars/tests/unit/operations/test_is_first_last_distinct.py"

NUM = [1, 1, None, 2, None, 3, 3]
STR = ["x", "x", None, "y", None, "z", "z"]
BOOL = [True, True, None, False, None, False, False]
FIRST = [True, False, True, True, False, True, False]

CASES = [
    # ---- DataFrame / Series.unique
    dict(src=f"{U}:114-119", frame={"a": [1, 2, 2], "b": [3, 3, 3]}, dtypes={"a": "int64", "b": "int64"}, op="unique", subset=None, keep="any",
         maintain_order=True, expected={"a": [1, 2], "b": [3, 3]}, order="pinned"),
    dict(src=f"{U}:121-123", frame={"a": [1, 2, 2], "b": [3, 3, 3]}, dtypes={"a": "int64", "b": "int64"}, op="unique", subset=["b"], keep="any",
         maintain_order=True, expected={"a": [1], "b": [3]}, order="pinned"),
    dict(src=f"{U}:125-127", frame={"a": [1, 2, None, 2]}, dtypes={"a": "int64"}, op="unique", subset=None, keep="any", maintain_order=True,
         expected={"a": [1, 2, None]}, order="pinned"),
    dict(src=f"{U}:128", frame={"a": [1, 2, None, 2]}, dtypes={"a": "int64"}, op="unique", subset=None, keep="any", maintain_order=False,
         expected={"a": [1, 2, None]}, order="multiset"),
    dict(src=f"{U}:152-155", frame={"s": []}, dtypes={"s": "int64"}, op="unique", subset=None, keep="any", maintain_order=True, expected={"s": []}, order="pinned"),
    dict(src=f"{U}:157-158", frame={"s": [None]}, dtypes={"s": "int64"}, op="unique", subset=None, keep="any", maintain_order=True,
         expected={"s": [None]}, order="pinned"),
    dict(src=f"{U}:160-161", frame={"s": [None, None]}, dtypes={"s": "int64"}, op="unique", subset=None, keep="any", maintain_order=True,
         expected={"s": [None]}, order="pinned"),
    dict(src=f"{U}:160-161", frame={"s": [None, None]}, dtypes={"s": "int64"}, op="unique", subset=None, keep="any", maintain_order=False,
         expected={"s": [None]}, order="multiset"),
    dict(src=f"{U}:183-194", frame={"a": [1, 1, 2, 2, 3, 4], "b": ["a", "a", "b", "b", "c", "c"], "c": [None] * 6},
         dtypes={"a": "int64", "b": "str", "c": "int64"}, op="unique", subset=None, keep="any", maintain_order=True,
         expected={"a": [1, 2, 3, 4], "b": ["a", "b", "c", "c"], "c": [None] * 4}, order="pinned"),
    dict(src=f"{U}:306-309", frame={"x": [float("nan")]}, dtypes={"x": "float64"}, op="unique", subset=None, keep="any", maintain_order=False,
         expected={"x": [float("nan")]}, order="multiset"),
    dict(src=f"{U}:318-322", frame={"x": [0, 1, 2, 3, 4, 5, 6, 7, 3, 4, 5, 6, 7, 8, 9, 10]}, dtypes={"x": "int64"}, op="unique", subset=None,
         keep="last", maintain_order=True, slice=[3, 4], expected={"x": [3, 4, 5, 6]}, order="pinned"),
    dict(src=f"{U}:325-329", frame={"b": [None] * 128}, prefix={"b": [None, None, True]}, dtypes={"b": "bool"}, op="unique", subset=None,
         keep="any", maintain_order=False, expected={"b": [None]}, order="multiset"),
    dict(src=f"{U}:331-334", frame={"b": [None, None]}, dtypes={"b": "bool"}, op="unique", subset=None, keep="any", maintain_order=False,
         expected={"b": [None]}, order="multiset"),
    dict(src=f"{U}:344-347", frame={"a": [1, 3, 2], "b": [4, 4, 6]}, dtypes={"a": "int64", "b": "int64"}, op="unique", subset=["b"], keep="none",
         maintain_order=False, expected={"a": [2], "b": [6]}, order="pinned"),
    dict(src=f"{IU}:24-28", frame={"foo": [1, 2, 2], "bar": [6, 7, 7]}, dtypes={"foo": "int64", "bar": "int64"}, op="unique", subset=None,
         keep="any", maintain_order=True, expected={"foo": [1, 2], "bar": [6, 7]}, order="pinned"),
]
# DataFrame.unique() of int_range(n) keeps every row (test_unique.py:312-315); `int_range`: the frame and the expected
# column are both {"x": 0 .. n - 1}, expanded by the reader
for n in range(0, 1000, 37):
    CASES.append(dict(src=f"{U}:312-315", int_range=n, dtypes={"x": "int64"}, op="unique", subset=None, keep="any", maintain_order=False,
                      order="multiset"))

CASES += [
    # ---- is_unique / is_duplicated
    dict(src=f"{IU}:5-7", frame={"a": [1, 2, 2, 3]}, dtypes={"a": "int64"}, op="mask", kind="unique", keys=["a"], expected=[True, False, False, True]),
    dict(src=f"{IU}:9-15", frame={"s": ["a", "b", "c", "a"]}, dtypes={"s": "str"}, op="mask", kind="duplicated", keys=["s"], expected=[True, False, False, True]),
    dict(src=f"{IU}:16-21", frame={"s": ["a", "b", "c", "a"]}, dtypes={"s": "str"}, op="mask", kind="unique", keys=["s"], expected=[False, True, True, False]),
    dict(src=f"{IU}:24-27", frame={"foo": [1, 2, 2], "bar": [6, 7, 7]}, dtypes={"foo": "int64", "bar": "int64"}, op="mask", kind="unique", keys=["foo", "bar"],
         expected=[True, False, False]),
    dict(src=f"{IU}:32-35", frame={"a": [4, 1, 4]}, dtypes={"a": "int64"}, op="mask", kind="unique", keys=["a"], expected=[False, True, False]),
    dict(src=f"{IU}:38-41", frame={"s": []}, dtypes={"s": "int64"}, op="mask", kind="unique", keys=["s"], expected=[]),
    dict(src=f"{IU}:43-45", frame={"s": [None]}, dtypes={"s": "int64"}, op="mask", kind="unique", keys=["s"], expected=[True]),
    dict(src=f"{IU}:47-49", frame={"s": [None, None, None]}, dtypes={"s": "int64"}, op="mask", kind="unique", keys=["s"], expected=[False, False, False]),
    dict(src=f"{IU}:108-110", frame={"a": [1, 2, 2, 3]}, dtypes={"a": "int64"}, op="mask", kind="duplicated", keys=["a"], expected=[False, True, True, False]),
    dict(src=f"{IU}:113-115", frame={"foo": [1, 2, 2], "bar": [6, 7, 7]}, dtypes={"foo": "int64", "bar": "int64"}, op="mask", kind="duplicated",
         keys=["foo", "bar"], expected=[False, True, True]),
    dict(src=f"{IU}:118-120", frame={"a": [4, 1, 4]}, dtypes={"a": "int64"}, op="mask", kind="duplicated", keys=["a"], expected=[True, False, True]),
    dict(src=f"{IU}:123-126", frame={"s": []}, dtypes={"s": "int64"}, op="mask", kind="duplicated", keys=["s"], expected=[]),
    dict(src=f"{IU}:128-130", frame={"s": [None]}, dtypes={"s": "int64"}, op="mask", kind="duplicated", keys=["s"], expected=[False]),
    dict(src=f"{IU}:132-134", frame={"s": [None, None, None]}, dtypes={"s": "int64"}, op="mask", kind="duplicated", keys=["s"], expected=[True, True, True]),
    # ---- is_first_distinct / is_last_distinct
    dict(src=f"{FL}:16-20", frame={"a": [4, 1, 4]}, dtypes={"a": "int64"}, op="mask", kind="first", keys=["a"], expected=[True, True, False]),
    dict(src=f"{FL}:27-29", frame={"b": [True] + 63 * [False]}, dtypes={"b": "bool"}, op="mask", kind="first", keys=["b"], expected=[True, True] + 62 * [False]),
    dict(src=f"{FL}:31-33", frame={"b": [False] + 63 * [True]}, dtypes={"b": "bool"}, op="mask", kind="first", keys=["b"], expected=[True, True] + 62 * [False]),
    dict(src=f"{FL}:35-37", frame={"b": 2 * [True] + 2 * [False] + 60 * [None]}, dtypes={"b": "bool"}, op="mask", kind="first", keys=["b"],
         expected=[True, False, True, False, True] + 59 * [False]),
    dict(src=f"{FL}:39-41", frame={"b": 2 * [False] + 2 * [None] + 60 * [True]}, dtypes={"b": "bool"}, op="mask", kind="first", keys=["b"],
         expected=[True, False, True, False, True] + 59 * [False]),
    dict(src=f"{FL}:95-97", frame={"s": NUM}, dtypes={"s": "int64"}, op="mask", kind="first", keys=["s"], expected=FIRST),
    dict(src=f"{FL}:99-101", frame={"s": STR}, dtypes={"s": "str"}, op="mask", kind="first", keys=["s"], expected=FIRST),
    dict(src=f"{FL}:103-105", frame={"s": BOOL}, dtypes={"s": "bool"}, op="mask", kind="first", keys=["s"], expected=[True, False, True, True, False, False, False]),
    dict(src=f"{FL}:128-130", frame={"s": NUM}, dtypes={"s": "int64"}, op="mask", kind="last", keys=["s"], expected=[False, True, False, True, True, False, True]),
    dict(src=f"{FL}:132-134", frame={"s": STR}, dtypes={"s": "str"}, op="mask", kind="last", keys=["s"], expected=[False, True, False, True, True, False, True]),
    dict(src=f"{FL}:136-138", frame={"s": BOOL}, dtypes={"s": "bool"}, op="mask", kind="last", keys=["s"], expected=[False, True, False, False, True, False, True]),
]
for dt in ("int64", "str", "bool"):      # test_is_first_last_distinct_all_null (:156-159), List(Int32) skipped
    CASES.append(dict(src=f"{FL}:156-158", frame={"s": [None] * 3}, dtypes={"s": dt}, op="mask", kind="first", keys=["s"], expected=[True, False, False]))
    CASES.append(dict(src=f"{FL}:156-159", frame={"s": [None] * 3}, dtypes={"s": dt}, op="mask", kind="last", keys=["s"], expected=[False, False, True]))


if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "unique_kats.json")
    with open(path, "w") as f:
        f.write("[\n" + ",\n".join(json.dumps(c) for c in CASES) + "\n]\n")
    print(f"wrote {len(CASES)} cases to {path}")
