"""Median / quantile known-answer vectors transcribed BY HAND from the reference's own tests (pola-rs/polars @ 4db92c1).

Each case is one group_by: per-row group `keys`, a value column `values` of `dtype` (`null` = a null slot), the aggregation
(`kind` "median", or "quantile" with `q` and `method`) and the expected per-group result `expect` in first-occurrence
group order (`null` = a null group).  `approx` marks a result the reference only checks within 1e-7.  Results are Float64,
Float32 for a Float32 column.  The ChunkedArray tests of aggregate/mod.rs run on one array: here that is one group.

Run `python tests/golden/transcribe_quantile.py` to regenerate tests/golden/quantile_kats.json.
"""
import json
import os

N = None
METHODS = ["nearest", "lower", "higher", "midpoint", "linear", "equiprobable"]
AGG = "crates/polars-core/src/chunked_array/ops/aggregate/mod.rs"
GB = "py-polars/tests/unit/operations/test_group_by.py"


def one_group(cite, values, dtype, q, method, expect, approx=False):
    c = {"cite": cite, "keys": [0] * len(values), "values": values, "dtype": dtype, "kind": "quantile", "q": q, "method": method, "expect": [expect]}
    if approx:
        c["approx"] = True
    return c


KATS = []
for dt in ("float32", "int32", "float64", "int64"):
    for m in METHODS:
        KATS.append(one_group(f"{AGG}:828-851 (test_quantile_all_null, {dt}, {m})", [N, N, N], dt, 0.9, m, N))
        KATS.append(one_group(f"{AGG}:853-875 (test_quantile_single_value, {dt}, {m})", [1], dt, 0.5, m, 1.0))
        vals = [N, 1, 5, 1]
        KATS.append(one_group(f"{AGG}:877-930 (test_quantile_min_max, {dt}, {m}, q=0 == min)", vals, dt, 0.0, m, 1.0))
        KATS.append(one_group(f"{AGG}:877-930 (test_quantile_min_max, {dt}, {m}, q=1 == max)", vals, dt, 1.0, m, 5.0))
        if dt == "float64":
            KATS.append(one_group(f"{AGG}:877-930 (test_quantile_min_max, {dt}, {m}, q=0.5 == median)", vals, dt, 0.5, m, 1.0))

# test_quantile: two UInt32 columns with nulls, every method
_A = [2, 1, N, 3, 5, N, 4]
for q, m, e in ((0.1, "nearest", 1.0), (0.9, "nearest", 5.0), (0.6, "nearest", 3.0), (0.1, "lower", 1.0), (0.9, "lower", 4.0), (0.6, "lower", 3.0),
                (0.1, "higher", 2.0), (0.9, "higher", 5.0), (0.6, "higher", 4.0), (0.1, "midpoint", 1.5), (0.9, "midpoint", 4.5), (0.6, "midpoint", 3.5),
                (0.1, "linear", 1.4), (0.9, "linear", 4.6), (0.15, "equiprobable", 1.0), (0.25, "equiprobable", 2.0), (0.6, "equiprobable", 3.0)):
    KATS.append(one_group(f"{AGG}:932-990 (test_quantile, first column, {m} {q})", _A, "uint32", q, m, e))
KATS.append(one_group(f"{AGG}:975-977 (test_quantile, first column, linear 0.6 within 1e-7)", _A, "uint32", 0.6, "linear", 3.4, approx=True))
_B = [N, 7, 6, 2, 1, N, 3, 5, N, 4]
for q, m, e in ((0.1, "nearest", 2.0), (0.9, "nearest", 6.0), (0.6, "nearest", 5.0), (0.1, "lower", 1.0), (0.9, "lower", 6.0), (0.6, "lower", 4.0),
                (0.1, "higher", 2.0), (0.9, "higher", 7.0), (0.6, "higher", 5.0), (0.1, "midpoint", 1.5), (0.9, "midpoint", 6.5), (0.6, "midpoint", 4.5),
                (0.1, "linear", 1.6), (0.9, "linear", 6.4), (0.6, "linear", 4.6), (0.14, "equiprobable", 1.0), (0.15, "equiprobable", 2.0),
                (0.6, "equiprobable", 5.0)):
    KATS.append(one_group(f"{AGG}:992-1058 (test_quantile, second column, {m} {q})", _B, "uint32", q, m, e))

# group_by shorthands over the fixture df (:279-287): a = [1..5], b = ["a", "a", "b", "b", "b"], c = [None, 1, None, 1, None]
_KEYS = ["a", "a", "b", "b", "b"]
for col, vals, med, qn in (("a", [1, 2, 3, 4, 5], [1.5, 4.0], [2.0, 4.0]), ("c", [N, 1, N, 1, N], [1.0, 1.0], [1.0, 1.0])):
    KATS.append({"cite": f"{GB}:290-313 (test_group_by_shorthands, median, column {col})", "keys": _KEYS, "values": vals, "dtype": "int64",
                 "kind": "median", "expect": med})
    KATS.append({"cite": f"{GB}:316-322 (test_group_by_shorthand_quantile, quantile(0.5), column {col})", "keys": _KEYS, "values": vals,
                 "dtype": "int64", "kind": "quantile", "q": 0.5, "method": "nearest", "expect": qn})

# Duration quantiles: the physical Int64 values (the reference casts the Float64 result back to Int64 and then Duration)
for tu, per_hour in (("ms", 3_600_000), ("us", 3_600_000_000), ("ns", 3_600_000_000_000)):
    vals = [x * per_hour for x in range(1, 9)]
    for m, e in (("nearest", [3, 7]), ("higher", [3, 7]), ("lower", [2, 6]), ("linear", [2.5, 6.5])):
        KATS.append({"cite": f"{GB}:428-468 (test_group_by_quantile_duration, tu={tu}, {m})", "keys": [1, 1, 1, 1, 2, 2, 2, 2], "values": vals,
                     "dtype": "int64", "kind": "quantile", "q": 0.5, "method": m, "expect": [h * per_hour for h in e]})


def main():
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "quantile_kats.json")
    with open(out, "w") as f:
        json.dump({"quantile": KATS}, f, indent=1)
    print("wrote", out, len(KATS), "cases")


if __name__ == "__main__":
    main()
