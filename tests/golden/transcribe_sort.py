"""Sort known-answer vectors transcribed BY HAND from the reference's own tests (pola-rs/polars @ 4db92c1).

Each case: key columns `by` (with `dtypes`), `descending` / `nulls_last` (a bool or one bool per column), an optional
`limit`, and the expected permutation `expect_idx` (or, where the test compares frames, `payload` / `expect_payload`:
the payload columns after the sort).  `null` in a list = a null slot.  Where the reference does not pin the order of
tied rows the test data has no observable tie, so the stable permutation is the expected one.

Run `python tests/golden/transcribe_sort.py` to regenerate tests/golden/sort_kats.json.
"""
import json
import os

N = None
NAN, INF = float("nan"), float("inf")


def _descending_nulls_last_cases():
    """py-polars/tests/unit/operations/test_sort.py:1005-1026 (test_sort_descending_nulls_last): the expected frame is
    built with Python's stable list.sort and a null sentinel of +-100"""
    out = []
    for descending in (False, True):
        for nulls_last in (False, True):
            sentinel = 100 if descending ^ nulls_last else -100
            ref_x = [1, 3, N, 2, N]
            ref_x.sort(key=lambda k: sentinel if k is None else k, reverse=descending)
            ref_y = [1, 3, 0, 2, 0]
            ref_y.sort(key=lambda k: sentinel if k == 0 else k, reverse=descending)
            for by in (["x"], ["x", "y"]):
                cols = {"x": [1, 3, N, 2, N], "y": [1, 3, 0, 2, 0]}
                out.append({"cite": f"py-polars/tests/unit/operations/test_sort.py:1005-1026 (test_sort_descending_nulls_last, by={by}, "
                                    f"descending={descending}, nulls_last={nulls_last})",
                            "by": [cols[b] for b in by], "dtypes": ["int64"] * len(by), "descending": descending, "nulls_last": nulls_last,
                            "payload": [cols["x"], cols["y"]], "payload_dtypes": ["int64", "int64"], "expect_payload": [ref_x, ref_y]})
    return out


KATS = [
    {"cite": "py-polars/tests/unit/operations/test_sort.py:200-230 (test_arg_sort_nulls, identity)",
     "by": [[1.0, 2.0, 3.0, N, N]], "dtypes": ["float64"], "descending": False, "nulls_last": True, "expect_idx": [0, 1, 2, 3, 4]},
    {"cite": "py-polars/tests/unit/operations/test_sort.py:200-230 (test_arg_sort_nulls, identity)",
     "by": [[1.0, 2.0, 3.0, N, N]], "dtypes": ["float64"], "descending": False, "nulls_last": False, "expect_idx": [3, 4, 0, 1, 2]},
    {"cite": "py-polars/tests/unit/operations/test_sort.py:200-230 (test_arg_sort_nulls, after sort(nulls_last=False))",
     "by": [[N, N, 1.0, 2.0, 3.0]], "dtypes": ["float64"], "descending": False, "nulls_last": True, "expect_idx": [2, 3, 4, 0, 1]},
    {"cite": "py-polars/tests/unit/operations/test_sort.py:200-230 (test_arg_sort_nulls, after sort(nulls_last=False))",
     "by": [[N, N, 1.0, 2.0, 3.0]], "dtypes": ["float64"], "descending": False, "nulls_last": False, "expect_idx": [0, 1, 2, 3, 4]},
    {"cite": "py-polars/tests/unit/operations/test_sort.py:233-239 (test_arg_sort_by_nulls): all-null x, y; z breaks the tie",
     "by": [[N] * 5, [N] * 5, [0, 2, 1, 3, 4]], "dtypes": ["float64", "int32", "int64"], "descending": False, "nulls_last": False,
     "expect_idx": [0, 2, 1, 3, 4]},
] + [
    {"cite": f"py-polars/tests/unit/operations/test_sort.py:242-267 (test_expr_arg_sort_nulls_last, nulls_last={nl})",
     "by": [[1, 2, N, N, 5], [1, 2, N, 1, N]], "dtypes": ["int64", "int64"], "descending": False, "nulls_last": nl, "expect_idx": exp}
    for nl, exp in ((True, [0, 1, 4, 3, 2]), (False, [2, 3, 0, 1, 4]), ([True, False], [0, 1, 4, 2, 3]), ([False, True], [3, 2, 0, 1, 4]))
] + [
    {"cite": "py-polars/tests/unit/operations/test_sort.py:301-309 (test_sort_nans_3740): key after sort == [2, 4, 1, 5, 3]",
     "by": [[0.0, N, NAN, -INF, INF]], "dtypes": ["float64"], "descending": False, "nulls_last": False, "expect_idx": [1, 3, 0, 4, 2]},
    {"cite": "py-polars/tests/unit/operations/test_sort.py:803-814 (test_sort_descending)",
     "by": [[1, 2, 3], [4, 5, 6]], "dtypes": ["int64", "int64"], "descending": True, "nulls_last": False, "expect_idx": [2, 1, 0]},
    {"cite": "py-polars/tests/unit/operations/test_sort.py:803-814 (test_sort_descending, descending=[True, True])",
     "by": [[1, 2, 3], [4, 5, 6]], "dtypes": ["int64", "int64"], "descending": [True, True], "nulls_last": False, "expect_idx": [2, 1, 0]},
    {"cite": "py-polars/tests/unit/operations/test_sort.py:831-844 (test_arg_sort_by_descending)",
     "by": [[1, 2, 3], [4, 5, 6]], "dtypes": ["int64", "int64"], "descending": True, "nulls_last": False, "expect_idx": [2, 1, 0]},
    {"cite": "py-polars/tests/unit/operations/test_sort.py:803-844: descending=[True] for two columns raises "
             "'the length of `descending` (1) does not match the length of `by` (2)'",
     "by": [[1, 2, 3], [4, 5, 6]], "dtypes": ["int64", "int64"], "descending": [True], "nulls_last": False, "expect_error": "descending"},
    {"cite": "py-polars/tests/unit/operations/test_sort.py:847-855 (test_arg_sort_struct): a struct sorts by its fields in order",
     "by": [[100, 300, 100, 200, 200, 100, 300, 200, 400, 400], [5, 5, 6, 7, 8, 1, 1, 2, 2, 3]], "dtypes": ["int64", "int64"],
     "descending": False, "nulls_last": False, "expect_idx": [5, 0, 2, 7, 3, 4, 6, 1, 8, 9]},
] + [
    {"cite": f"py-polars/tests/unit/operations/test_sort.py:925-961 (test_sort_with_null_12139, descending={d}, nulls_last={nl}, maintain_order)",
     "by": [[True, False, N, True, False]], "dtypes": ["bool"], "descending": d, "nulls_last": nl,
     "payload": [[1.0, 2.0, 3.0, 4.0, 5.0]], "payload_dtypes": ["float64"], "expect_payload": [exp]}
    for d, nl, exp in ((False, False, [3.0, 2.0, 5.0, 1.0, 4.0]), (False, True, [2.0, 5.0, 1.0, 4.0, 3.0]),
                       (True, True, [1.0, 4.0, 2.0, 5.0, 3.0]), (True, False, [3.0, 1.0, 4.0, 2.0, 5.0]))
] + _descending_nulls_last_cases() + [
    {"cite": "py-polars/tests/unit/operations/test_sort.py:1166-1168 (test_sort_multicolum_null): shape (1, 2)",
     "by": [[1], [N]], "dtypes": ["int64", "int64"], "descending": False, "nulls_last": False, "expect_idx": [0]},
] + [
    {"cite": f"py-polars/tests/unit/operations/test_sort.py:1177-1194 (test_sort_bool_nulls_last, nulls_last={nl}, descending={d})",
     "by": [col], "dtypes": ["bool"], "descending": d, "nulls_last": nl, "expect_idx": exp}
    for col, nl, d, exp in (([False], True, False, [0]), ([N, True, False], True, False, [2, 1, 0]), ([N, True, False], False, False, [0, 2, 1]),
                            ([N, True, False], True, True, [1, 2, 0]), ([N, True, False], False, True, [0, 1, 2]))
] + [
    {"cite": "crates/polars-core/src/chunked_array/ops/sort/arg_sort.rs:339-352 (test_arg_sort_descending_with_limit)",
     "by": [[4, 2, 5, 1, 3]], "dtypes": ["int32"], "descending": True, "nulls_last": False, "limit": 3, "expect_idx": [2, 0, 4]},
    {"cite": "crates/polars-core/src/chunked_array/ops/sort/arg_sort.rs:354-367 (test_arg_sort_asc_with_limit)",
     "by": [[4, 2, 5, 1, 3]], "dtypes": ["int32"], "descending": False, "nulls_last": False, "limit": 3, "expect_idx": [3, 1, 4]},
    {"cite": "crates/polars-core/src/chunked_array/ops/sort/arg_sort.rs:369-384 (test_arg_sort_desc_limit_nulls)",
     "by": [[4, N, 5, 1, N, 3]], "dtypes": ["int32"], "descending": True, "nulls_last": True, "limit": 3, "expect_idx": [2, 0, 5]},
    {"cite": "crates/polars-core/src/chunked_array/ops/sort/options.rs:58-79 (SortMultipleOptions doc example, maintain_order)",
     "by": [[1, 2, N, 4, N], [5, N, 3, 2, 1]], "dtypes": ["int64", "int64"], "descending": [False, True], "nulls_last": True,
     "payload": [[1, 2, N, 4, N], [5, N, 3, 2, 1]], "payload_dtypes": ["int64", "int64"],
     "expect_payload": [[1, 2, 4, N, N], [5, N, 2, 3, 1]], "expect_idx": [0, 1, 3, 2, 4]},
]


def main():
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "sort_kats.json")
    with open(out, "w") as f:
        json.dump({"sort": KATS}, f, indent=1)      # NaN / Infinity are written as JSON's NaN / Infinity extensions
    print("wrote", out)


if __name__ == "__main__":
    main()
