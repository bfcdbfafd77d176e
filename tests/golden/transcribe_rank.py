"""Writes tests/golden/rank_kats.json: known answers of the reference's rank tests, transcribed by hand with the file:line of
each case (paths relative to the reference's repository root).

Every case: values (None = null), dtype ("int64", "uint32", "float64", "str"), method, descending, parts (a partition label
per row, or None for a plain rank), expected (None = null).  The reference's RANDOM answer cannot be reproduced (the header
of bl_rank says why): its case records only what holds for any seed, the run sums, as `random_runs` = [[rows], sum].

Not expressible here: test_rank_random_expr (test_rank.py:13-24) only compares two runs with the same seed, which
tests/test_gpu_rank.py checks for this library's seed; test_rank_series' dtype asserts (:117-118) are the method dtypes every
case checks."""
import json
import os

RS = "crates/polars-ops/src/series/ops/rank.rs"
PY = "py-polars/tests/unit/operations/test_rank.py"
S7 = [1, 2, 3, 2, 2, 3, 0]

CASES = [
    # rank.rs test_rank
    dict(src=f"{RS}:204-211", values=S7, dtype="int32", method="ordinal", expected=[2, 3, 6, 4, 5, 7, 1]),
    dict(src=f"{RS}:214-224", values=S7, dtype="int32", method="random", expected=None,
         random_runs=[[[0], 2], [[6], 1], [[1, 3, 4], 12], [[2, 5], 13]]),
    dict(src=f"{RS}:227-231", values=S7, dtype="int32", method="dense", expected=[2, 3, 4, 3, 3, 4, 1]),
    dict(src=f"{RS}:233-237", values=S7, dtype="int32", method="max", expected=[2, 5, 7, 5, 5, 7, 1]),
    dict(src=f"{RS}:239-243", values=S7, dtype="int32", method="min", expected=[2, 3, 6, 3, 3, 6, 1]),
    dict(src=f"{RS}:245-249", values=S7, dtype="int32", method="average", expected=[2.0, 4.0, 6.5, 4.0, 4.0, 6.5, 1.0]),
    dict(src=f"{RS}:251-271", values=[1, 2, 3, 2, None, None, 0], dtype="int32", method="average",
         expected=[2.0, 3.5, 5.0, 3.5, None, None, 1.0]),
    dict(src=f"{RS}:273-303", values=[5, 6, 4, None, 78, 4, 2, 8], dtype="int32", method="max",
         expected=[4, 5, 3, None, 7, 3, 1, 6]),
    # test_rank_all_null
    dict(src=f"{RS}:309-314", values=[None, None, None], dtype="uint32", method="average", expected=[None, None, None]),
    dict(src=f"{RS}:315-319", values=[None, None, None], dtype="uint32", method="dense", expected=[None, None, None]),
    # test_rank_empty (the dtypes: Float64 for average, IdxSize otherwise)
    dict(src=f"{RS}:325-327", values=[], dtype="uint32", method="average", expected=[]),
    dict(src=f"{RS}:328-329", values=[], dtype="uint32", method="max", expected=[]),
    # test_rank_reverse
    dict(src=f"{RS}:334-339", values=[None, 1, 1, 5, None], dtype="int32", method="dense", descending=True,
         expected=[None, 2, 2, 1, None]),
    # test_rank.py
    dict(src=f"{PY}:8", values=[], dtype="float64", method="average", expected=[]),
    dict(src=f"{PY}:9", values=[None], dtype="float64", method="average", expected=[None]),
    dict(src=f"{PY}:10", values=[None, None], dtype="float64", method="average", expected=[None, None]),
    dict(src=f"{PY}:28-32 (seed 1; the reference's bytes are [2, 5, 7, 3, 4, 6, 1], not reproduced)", values=S7, dtype="int64",
         method="random", expected=None, random_runs=[[[0], 2], [[6], 1], [[1, 3, 4], 12], [[2, 5], 13]]),
    dict(src=f"{PY}:36-44", values=[1, 1, 2, 2, 3], dtype="int64", method="average", expected=[1.5, 1.5, 3.5, 3.5, 5.0]),
    dict(src=f"{PY}:46-48", values=[1, 1, 2, 2, 3], dtype="int64", method="max", expected=[2, 2, 4, 4, 5]),
    dict(src=f"{PY}:97-98", values=[None, "", "z", None, "a"], dtype="str", method="average", expected=[None, 1.0, 3.0, None, 2.0]),
    dict(src=f"{PY}:104-107", values=S7, dtype="int64", method="dense", expected=[2, 3, 4, 3, 3, 4, 1]),
    dict(src=f"{PY}:110", values=S7, dtype="int64", method="dense", expected=[2, 3, 4, 3, 3, 4, 1]),
    dict(src=f"{PY}:112-115", values=S7, dtype="int64", method="dense", descending=True, expected=[3, 2, 1, 2, 2, 1, 4]),
    # test_window.py:395-411: rank(method="ordinal").over("customer_ID") after sorting by (customer_ID, date)
    dict(src="py-polars/tests/unit/operations/test_window.py:404", values=[1, 2, 3], dtype="int64", method="ordinal",
         parts=["0", "0", "1"], expected=[1, 2, 1]),
    # test_sort.py:519-536: NaN is the greatest value
    dict(src="py-polars/tests/unit/operations/test_sort.py:524-535", values=[1.0, float("nan")], dtype="float64", method="average",
         expected=[1.0, 2.0]),
]

# test_rank.py:52-93 (so_4109): rank inside group_by().agg() gives list outputs; per group it is the rank of the group's
# values, so each group is one partition of a rank().over("id") here, on the frame sorted by (id, rank) as the test does.
_ID = [1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4]
_ORIG = [None, 2, 3, 4, 1, 2, 3, 4, None, 1, 3, 4, None, 1, 3, 4]
CASES += [
    dict(src=f"{PY}:52-93 (dense)", values=_ORIG, dtype="int64", method="dense", parts=_ID,
         expected=[None, 1, 2, 3, 1, 2, 3, 4, None, 1, 2, 3, None, 1, 2, 3]),
    dict(src=f"{PY}:52-93 (average)", values=_ORIG, dtype="int64", method="average", parts=_ID,
         expected=[None, 1.0, 2.0, 3.0, 1.0, 2.0, 3.0, 4.0, None, 1.0, 2.0, 3.0, None, 1.0, 2.0, 3.0]),
]

if __name__ == "__main__":
    for c in CASES:
        c.setdefault("descending", False)
        c.setdefault("parts", None)
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "rank_kats.json")
    with open(out, "w") as f:
        json.dump(CASES, f, indent=1, allow_nan=True)
        f.write("\n")
    print(f"wrote {len(CASES)} cases to {out}")
