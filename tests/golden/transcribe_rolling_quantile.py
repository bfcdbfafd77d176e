"""Writes rolling_quantile_kats.json: known answers of the reference's rolling quantile / median tests, each with the
file:line it comes from (paths relative to the reference's crates/ and py-polars/).  Run from anywhere:
    python tests/golden/transcribe_rolling_quantile.py

A case is {"src", "values" (None = null), "quantile", "method", and either "window_size", "min_samples", "center"
(fixed windows) or "by", "window_size" (P), "closed", "min_samples" (time windows), "expected" (None = null)}.

Not transcribed, with the reason:
- the weighted tests (test_rolling_weighted_quantile*, test_rolling.py): `weights` are not in the ABI;
- rolling_quantile_by over Date / Datetime expecting a temporal output dtype (series/test_rolling.py): the cast back to the
  temporal dtype is the caller's, so those outputs are not this call's values;
- test_rolling_median / test_rolling_median_2 (test_rolling.py:1143-1170): random inputs compared with pandas or a sum of
  approximate floats, with no fixed answer to transcribe.
"""
import json
import os

HERE = os.path.dirname(os.path.abspath(__file__))
METHODS = ["nearest", "lower", "higher", "midpoint", "linear", "equiprobable"]


def fixed(src, values, q, method, w, ms, center, expected):
    return {"src": src, "values": values, "quantile": q, "method": method, "window_size": w, "min_samples": ms, "center": center,
            "expected": expected}


def by_case(src, values, by, P, closed, ms, q, method, expected):
    return {"src": src, "values": values, "by": by, "window_size": P, "closed": closed, "min_samples": ms, "quantile": q,
            "method": method, "expected": expected}


def cases():
    out = []
    nn = "polars-compute/src/rolling/no_nulls/quantile.rs"
    v = [1.0, 2.0, 3.0, 4.0]
    out.append(fixed(f"{nn}:284-315 (test_rolling_median)", v, 0.5, "linear", 2, 2, False, [None, 1.5, 2.5, 3.5]))
    out.append(fixed(f"{nn}:284-315 (test_rolling_median)", v, 0.5, "linear", 2, 1, False, [1.0, 1.5, 2.5, 3.5]))
    out.append(fixed(f"{nn}:284-315 (test_rolling_median)", v, 0.5, "linear", 4, 1, False, [1.0, 1.5, 2.0, 2.5]))
    out.append(fixed(f"{nn}:284-315 (test_rolling_median)", v, 0.5, "linear", 4, 1, True, [1.5, 2.0, 2.5, 3.0]))
    out.append(fixed(f"{nn}:284-315 (test_rolling_median)", v, 0.5, "linear", 4, 4, True, [None, None, 2.5, None]))
    for m in METHODS:      # q = 0 is rolling_min, q = 1 rolling_max (window 2, min_samples 2)
        out.append(fixed(f"{nn}:317-356 (test_rolling_quantile_limits)", v, 0.0, m, 2, 2, False, [None, 1.0, 2.0, 3.0]))
        out.append(fixed(f"{nn}:317-356 (test_rolling_quantile_limits)", v, 1.0, m, 2, 2, False, [None, 2.0, 3.0, 4.0]))

    nl = "polars-compute/src/rolling/nulls/quantile.rs"
    v = [1.0, None, 3.0, 4.0]
    out.append(fixed(f"{nl}:184-219 (test_rolling_median_nulls)", v, 0.5, "linear", 2, 2, False, [None, None, None, 3.5]))
    out.append(fixed(f"{nl}:184-219 (test_rolling_median_nulls)", v, 0.5, "linear", 2, 1, False, [1.0, 1.0, 3.0, 3.5]))
    out.append(fixed(f"{nl}:184-219 (test_rolling_median_nulls)", v, 0.5, "linear", 4, 1, False, [1.0, 1.0, 2.0, 3.0]))
    out.append(fixed(f"{nl}:184-219 (test_rolling_median_nulls)", v, 0.5, "linear", 4, 1, True, [1.0, 2.0, 3.0, 3.5]))
    out.append(fixed(f"{nl}:184-219 (test_rolling_median_nulls)", v, 0.5, "linear", 4, 4, True, [None, None, None, None]))
    v = [1.0, None, None, 4.0, 5.0]
    for m in METHODS:      # q = 0 / 1 against rolling_min / rolling_max (window 2, min_samples 1)
        out.append(fixed(f"{nl}:221-267 (test_rolling_quantile_nulls_limits)", v, 0.0, m, 2, 1, False, [1.0, 1.0, None, 4.0, 4.0]))
        out.append(fixed(f"{nl}:221-267 (test_rolling_quantile_nulls_limits)", v, 1.0, m, 2, 1, False, [1.0, 1.0, None, 4.0, 5.0]))

    py = "py-polars/tests/unit/operations/rolling/test_rolling.py"
    # rolling("index", period="2i").agg(quantile(0.5, m)): rolling_quantile_by with by = index, closed "right", min 1
    for m in METHODS:
        out.append(by_case(f"{py}:1571-1585", [None, None, 1.0, None, None, 1.0, 1.0, None, None], list(range(9)), 2, "right", 1, 0.5, m,
                           [None, None, 1.0, 1.0, None, 1.0, 1.0, 1.0, None]))
    # nearest over range(11), window 11: [None] * 10 + [round(q * 10)] for q in arange(0, 1, 0.02)
    for k in range(50):
        q = k * 0.02
        out.append(fixed(f"{py}:1587-1609", [float(i) for i in range(11)], q, "nearest", 11, 11, False, [None] * 10 + [float(round(q * 10.0))]))
    return out


if __name__ == "__main__":
    path = os.path.join(HERE, "rolling_quantile_kats.json")
    with open(path, "w") as f:
        json.dump(cases(), f, indent=1)
    print("wrote", path, len(cases()), "cases")
