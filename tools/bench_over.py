"""Window function benchmark (bl_over), device-resident inputs and outputs.  Prints one JSON line.

  W1  whole-column cum_sum of Int64 (plan 1: one decoupled look-back scan; HBM bound 16 B/row)
  W2  sum().over(g) of Float64 with 1e6 groups (plan 2: the fused group_by on the group ids + one K4 broadcast)
  W3  cum_sum().over(g) of Int64 with 1e6 groups (plan 3: the group-id sort, then the segmented scan)
  W4  shift(1).over(g, order_by=t) with 1e4 groups and Int64 timestamps (plan 3 with the (group, t) arg_sort)

Every result is checked against numpy outside the timed region.  Per workload: ms/step (CUDA-synchronised wall time of
`--steps` steps after `--warmup`), the per-kernel ms of one profiled step, and for every kernel of the window path its share
of the HBM roofline: its algorithmic bytes per row (ROW_BYTES) x rows / 3.35 TB/s over its kernel time.  The group-id,
group_by and sort kernels are the library's own (DESIGN.md §4 gives their bytes).
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_sort import card  # noqa: E402

HBM_TBPS = 3.35      # H100 SXM data sheet
# algorithmic bytes per row of the window kernels (8-byte values, 4-byte ids / permutation entries)
ROW_BYTES = {
    "over_scan": 16,            # value read + result written (the validity is the input's: not touched)
    "over_scan_seg": 24,        # permutation 4 + segment id 4 + gathered value 8 + scattered result 8
    "over_shift": 32 + 1 / 8,   # inverse 4 + seg[p] 4 + seg[q] 4 + perm[q] 4 + value 8 + result 8 + validity bit
    "over_inverse": 8,          # permutation read 4 + scattered write 4
    "over_seg_ids": 12,         # permutation 4 + gathered group id 4 + write 4
    "over_row_ordinal": 12,     # group id 4 + gathered ordinal 4 + write 4
    "k4_gather": 20,            # ordinal 4 + gathered aggregate 8 + result 8 (one aggregate column)
}


def seg_cumsum(x, g):
    """per-group running sum in row order (Int64, wrapping), groups of any order"""
    n = len(x)
    order = np.lexsort((np.arange(n), g))
    gs = g[order]
    head = np.ones(n, bool)
    head[1:] = gs[1:] != gs[:-1]
    cs = np.cumsum(x[order].view(np.uint64), dtype=np.uint64)
    start = np.maximum.accumulate(np.where(head, np.arange(n), 0))
    base = np.where(start > 0, cs[start - 1], np.uint64(0))
    out = np.empty(n, np.int64)
    out[order] = (cs - base).view(np.int64)
    return out


def run(a):
    import polars_b200 as plb
    plb.init(0)
    rng = np.random.default_rng(0)
    n = a.rows
    x = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    xf = rng.standard_normal(n)
    g6 = rng.integers(0, 1_000_000, n)
    g4 = rng.integers(0, 10_000, n)
    t = rng.integers(0, 10**12, n, dtype=np.int64)
    dx, dxf, dg6, dg4, dt = plb.to_device(x), plb.to_device(xf), plb.to_device(g6), plb.to_device(g4), plb.to_device(t)

    def check_w1(o):
        return np.array_equal(o[0].to_numpy()[0], np.cumsum(x.view(np.uint64), dtype=np.uint64).view(np.int64))

    def check_w2(o):
        sums = np.bincount(g6, weights=xf, minlength=1_000_000)
        got = o[0].to_numpy()[0]
        return bool(np.allclose(got, sums[g6], rtol=1e-9, atol=1e-9))

    def check_w3(o):
        return np.array_equal(o[0].to_numpy()[0], seg_cumsum(x, g6))

    def check_w4(o):
        order = np.lexsort((np.arange(n), t, g4))
        prev = np.empty(n, np.int64)
        prev[order[1:]] = order[:-1]
        ok = np.zeros(n, bool)
        ok[order[1:]] = g4[order[1:]] == g4[order[:-1]]
        v, m = o[0].to_numpy()
        return bool(np.array_equal(m, ok) and np.array_equal(v[ok], x[prev[ok]]))

    work = {
        "W1": (lambda: plb.over([("cum_sum", dx, {})], location=plb.DEVICE), check_w1),
        "W2": (lambda: plb.over([("sum", dxf)], partition_by=[dg6], location=plb.DEVICE), check_w2),
        "W3": (lambda: plb.over([("cum_sum", dx, {})], partition_by=[dg6], location=plb.DEVICE), check_w3),
        "W4": (lambda: plb.over([("shift", dx, {"periods": 1})], partition_by=[dg4], order_by=dt, location=plb.DEVICE), check_w4),
    }
    res = {"bench": "over", **card(), "rows": n, "steps": a.steps, "warmup": a.warmup, "workloads": {}}
    for name, (step, check) in work.items():
        if a.only and name not in a.only.split(","):
            continue
        ok = bool(check(step()))
        for _ in range(a.warmup):
            step()
        plb.sync()
        plb.profile_reset(); plb.profile_enable(True)
        step()
        plb.sync()
        prof = plb.profile()
        plb.profile_enable(False)
        t0 = time.perf_counter()
        for _ in range(a.steps):
            step()
        plb.sync()
        ms = (time.perf_counter() - t0) / a.steps * 1e3
        w = {"ok": ok, "ms_per_step": round(ms, 3), "rows_per_s": round(n / ms * 1e3),
             "kernels_ms": {k: round(v["ms"], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])}}
        w["roofline"] = {}
        for k, b in ROW_BYTES.items():
            if k in prof:
                roof = n * b / (HBM_TBPS * 1e12) * 1e3
                w["roofline"][k] = {"ms": round(prof[k]["ms"], 3), "roofline_ms": round(roof, 3), "share": round(roof / prof[k]["ms"], 3)}
        res["workloads"][name] = w
    print(json.dumps(res))
    return 0 if all(w["ok"] for w in res["workloads"].values()) else 1


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--only", default="", help="comma-separated workload names")
    sys.exit(run(ap.parse_args()))


if __name__ == "__main__":
    main()
