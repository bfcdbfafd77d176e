"""Sorting by string keys: known-answer vectors transcribed BY HAND from the reference's own tests (pola-rs/polars @ 4db92c1).

Each case is one sort of a frame: `columns` maps a name to its `dtype` ("str" or a numpy dtype name) and `values`
(`null` = a null slot); the frame is sorted by the columns named in `by` with `descending` / `nulls_last` (a bool for every
column or one per column), and `expect` holds the sorted values of the columns the reference checks.

Run `python tests/golden/transcribe_string_sort.py` to regenerate tests/golden/string_sort_kats.json.
"""
import json
import os

N = None
SORT = "crates/polars-core/src/chunked_array/ops/sort/mod.rs"
PY = "py-polars/tests/unit/operations/test_sort.py"


def case(cite, columns, by, descending, nulls_last, expect):
    return {"cite": cite, "columns": {k: {"dtype": dt, "values": v} for k, (dt, v) in columns.items()}, "by": by,
            "descending": descending, "nulls_last": nulls_last, "expect": expect}


KATS = [
    # test_arg_sort_multiple: three keys, the last one a string
    case(f"{SORT}:1023-1048 (test_arg_sort_multiple, a, b, c)",
         {"a": ("int32", [1, 2, 1, 1, 3, 4, 3, 3]), "b": ("int64", [0, 1, 2, 3, 4, 5, 6, 1]), "c": ("str", ["a", "b", "c", "d", "e", "f", "g", "h"])},
         ["a", "b", "c"], False, False, {"b": [0, 2, 3, 1, 1, 4, 6, 5]}),
    # the first key a string
    case(f"{SORT}:1050-1064 (test_arg_sort_multiple, string first)",
         {"a": ("str", ["a", "b", "c", "a", "b", "c"]), "b": ("int32", [5, 4, 2, 3, 4, 5])},
         ["a", "b"], False, False, {"a": ["a", "a", "b", "b", "c", "c"], "b": [3, 5, 4, 4, 2, 5]}),
    case(f"{SORT}:1066-1079 (test_arg_sort_multiple, descending [true, false])",
         {"groups": ("int32", [1, 2, 3]), "values": ("str", ["a", "a", "b"])},
         ["groups", "values"], [True, False], False, {"groups": [3, 2, 1], "values": ["b", "a", "a"]}),
    case(f"{SORT}:1081-1089 (test_arg_sort_multiple, descending [false, true])",
         {"groups": ("int32", [1, 2, 3]), "values": ("str", ["a", "a", "b"])},
         ["values", "groups"], [False, True], False, {"groups": [2, 1, 3], "values": ["a", "a", "b"]}),
]

S = ["a", N, "c", N, "b"]
for desc, nl, exp, lines in [(False, False, [N, N, "a", "b", "c"], "1100-1108"), (True, False, [N, N, "c", "b", "a"], "1110-1119"),
                             (False, True, ["a", "b", "c", N, N], "1121-1129"), (True, True, ["c", "b", "a", N, N], "1131-1139")]:
    KATS.append(case(f"{SORT}:{lines} (test_sort_string, descending={desc}, nulls_last={nl})", {"a": ("str", S)}, ["a"], desc, nl, {"a": exp}))
KATS.append(case(f"{SORT}:1141-1148 (test_sort_string, no nulls, ascending)", {"a": ("str", ["a", "c", "b"])}, ["a"], False, False, {"a": ["a", "b", "c"]}))
KATS.append(case(f"{SORT}:1150-1152 (test_sort_string, no nulls, descending)", {"a": ("str", ["a", "c", "b"])}, ["a"], True, False, {"a": ["c", "b", "a"]}))

B = ["a", N, "c", N, "x", "z", "y", N]
for desc, nl, exp, lines in [(False, False, [N, N, N, "a", "c", "x", "y", "z"], "1063-1072"), (True, False, [N, N, N, "z", "y", "x", "c", "a"], "1073-1082"),
                             (True, True, ["z", "y", "x", "c", "a", N, N, N], "1083-1092"), (False, True, ["a", "c", "x", "y", "z", N, N, N], "1093-1102")]:
    KATS.append(case(f"{PY}:{lines} (test_sort_string_nulls, descending={desc}, nulls_last={nl})", {"b": ("str", B)}, ["b"], desc, nl, {"b": exp}))


if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "string_sort_kats.json")
    with open(path, "w") as f:
        json.dump({"sort": KATS}, f, indent=1)
        f.write("\n")
    print(f"wrote {len(KATS)} cases to {path}")
