"""Inequality join: known-answer vectors transcribed BY HAND from the reference's own examples (pola-rs/polars).

Each case is one join_where with one or two inequality predicates, written as the planner lowers them: `left` / `right` hold
one column per predicate (`null` = a null slot), `ops[k]` compares left[k] (on the left of the operator) with right[k], and
`dtypes[k]` is the physical dtype of predicate k.  A predicate written with the right frame's column first is normalised
(`b < a` becomes `a > b`).  `how` is inner, left or right.  `expect` is the result as a set of [left row, right row] pairs,
`null` for the null side of an unmatched row.  Datetimes are written as their physical Int64 microseconds since the epoch.

Run `python tests/golden/transcribe_ie_join.py` to regenerate tests/golden/ie_join_kats.json.
"""
import json
import os
from datetime import datetime, timezone

N = None
PY = "py-polars/tests/unit/operations/test_inequality_join.py"
DOC = "py-polars/src/polars/dataframe/frame.py"


def case(cite, dtypes, left, right, ops, expect, how="inner"):
    return {"cite": cite, "dtypes": dtypes, "left": left, "right": right, "ops": ops, "how": how,
            "expect": sorted(expect, key=lambda p: (p[0] is None, p[0] or 0, p[1] is None, p[1] or 0))}


def us(*dt):
    """a naive datetime as microseconds since the epoch (Datetime("us") physical)"""
    return int(datetime(*dt, tzinfo=timezone.utc).timestamp()) * 1_000_000


# west of test_self_join / test_basic_ie_join: time, cost
WEST_TIME, WEST_COST = [100, 140, 80, 90], [6, 11, 10, 5]
# test_join_where_predicates
JW_TIME = [us(2024, 8, 26, 15, 34, 30), us(2024, 8, 26, 15, 35, 30), us(2024, 8, 26, 15, 36, 30), us(2024, 8, 26, 15, 37, 30),
           us(2024, 8, 26, 15, 38, 0), us(2024, 8, 26, 15, 39, 0)]
JW_START = [us(2024, 8, 26, 15, 34, 0), us(2024, 8, 26, 15, 35, 0), us(2024, 8, 26, 15, 38, 0)]
JW_END = [us(2024, 8, 26, 15, 36, 0), us(2024, 8, 26, 15, 37, 0), us(2024, 8, 26, 15, 39, 0)]

KATS = [
    # east: dur, rev; west: time, cost; dur < time, rev < cost -> ids 100/498, 100/676, 100/742, 101/676, 101/742
    case(f"{DOC}:8575-8607 (join_where docstring)", ["int64", "int64"], [[120, 140, 160], [12, 14, 16]],
         [[90, 130, 150, 170], [9, 13, 15, 16]], ["<", "<"], [[0, 1], [0, 2], [0, 3], [1, 2], [1, 3]]),
    # time > time_right, cost < cost_right -> t_id 742/676 and 404/676
    case(f"{PY}:23-54 (test_self_join, parametrisation 1)", ["int64", "int64"], [WEST_TIME, WEST_COST], [WEST_TIME, WEST_COST],
         [">", "<"], [[3, 2], [0, 2]]),
    # time_right < time, cost_right > cost: normalised to the same predicates and the same answer
    case(f"{PY}:23-54 (test_self_join, parametrisation 2)", ["int64", "int64"], [WEST_TIME, WEST_COST], [WEST_TIME, WEST_COST],
         [">", "<"], [[3, 2], [0, 2]]),
    # east: dur [140, 100, 90], rev [12, 12, 5]; dur < time, rev > cost -> id 101 / t_id 498
    case(f"{PY}:57-97 (test_basic_ie_join)", ["int64", "int64"], [[140, 100, 90], [12, 12, 5]], [WEST_TIME, WEST_COST],
         ["<", ">"], [[1, 1]]),
    # time >= start_time, time < end_time -> (id, id_right) 0/0, 1/0, 1/1, 2/1, 4/2
    case(f"{PY}:188-241 (test_join_where_predicates, the IEJoin assertion)", ["int64", "int64"], [JW_TIME, JW_TIME], [JW_START, JW_END],
         [">=", "<"], [[0, 0], [1, 0], [1, 1], [2, 1], [4, 2]]),
    # a > b, how="left" -> a 1, 2, 3 with b null, null, 2
    case(f"{PY}:472-479 (test_join_where_how_left)", ["int64"], [[1, 2, 3]], [[2]], [">"], [[0, N], [1, N], [2, 0]], how="left"),
    # a > b, how="right" -> a 3 with b 2
    case(f"{PY}:482-488 (test_join_where_how_right)", ["int64"], [[1, 2, 3]], [[2]], [">"], [[2, 0]], how="right"),
    case(f"{PY}:507-513 (test_join_where_how_left_dataframe)", ["int64"], [[1, 2, 3]], [[2]], [">"], [[0, N], [1, N], [2, 0]], how="left"),
    # a >= b, a <= b -> a 2 with x_right 1, 3, 7 (right rows 1, 2, 0)
    case(f"{PY}:562-577 (test_ie_join_use_keys_multiple)", ["int64", "int64"], [[1, 2, 3], [1, 2, 3]], [[2, 2, 2], [2, 2, 2]],
         [">=", "<="], [[1, 0], [1, 1], [1, 2]]),
]

if __name__ == "__main__":
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ie_join_kats.json")
    with open(out, "w") as f:
        json.dump({"ie_join": KATS}, f, indent=1)
        f.write("\n")
    print(f"{len(KATS)} cases -> {out}")
