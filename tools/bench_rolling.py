"""Rolling window benchmark (bl_rolling), device-resident inputs and outputs.  Prints one JSON line.

  R1  whole-column rolling_mean(20) of Float64 (small-window plan: k_roll_tile, one pass)
  R2  whole-column rolling_sum(100_000) of Int64 (large-window plan: the prefix / suffix scans through HBM, then the output)
  R3  rolling_std(50, min_samples=25) of Float32 with 10 % nulls (small-window plan)
  R4  rolling_mean(10).over(g, order_by=t) of Float64 with 1e4 groups and Int64 timestamps (the (group, t) arg_sort, then
      the small-window plan over the partition order)

Every result is checked against numpy outside the timed region.  Per workload: ms/step (CUDA-synchronised wall time of
`--steps` steps after `--warmup`), the per-kernel ms of one profiled step, and for each rolling kernel its share of the HBM
roofline: its algorithmic bytes per row (ROW_BYTES, which depend on the state size of the workload's operator) x rows /
3.35 TB/s over its kernel time.
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
# bytes per row: the prefix / suffix scans read the value and write one state (integer SUM: 16 B); the output kernel reads
# two states and writes the result and its validity bit.
# The tile kernel reads the value (and its validity bit; in R4 the permutation and segment id too) and writes the result and
# its validity bit; the halo it re-reads is not counted.
ROW_BYTES = {
    "R1": {"rolling_tile": 8 + 8 + 1 / 8},
    "R2": {"rolling_prefix": 8 + 16, "rolling_suffix": 8 + 16, "rolling_out": 32 + 8 + 1 / 8},
    "R3": {"rolling_tile": 4 + 1 / 8 + 4 + 1 / 8},
    "R4": {"rolling_tile": 4 + 4 + 8 + 8 + 4},
}


def trailing(c, w, start=None):
    """window sums from an exclusive prefix array c (len n + 1): c[i + 1] - c[max(i - w + 1, start_i)]"""
    n = len(c) - 1
    i = np.arange(n)
    lo = np.maximum(i - (w - 1), 0 if start is None else start)
    return c[i + 1] - c[lo], i + 1 - lo


def run(a):
    import polars_b200 as plb
    plb.init(0)
    rng = np.random.default_rng(0)
    n = a.rows
    xf = rng.standard_normal(n)
    xi = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    x32 = rng.standard_normal(n).astype(np.float32)
    m32 = rng.random(n) >= 0.1
    g4 = rng.integers(0, 10_000, n)
    t = rng.integers(0, 10**12, n, dtype=np.int64)
    dxf, dxi, dx32, dg4, dt = plb.to_device(xf), plb.to_device(xi), plb.to_device(x32, m32), plb.to_device(g4), plb.to_device(t)

    def check_r1(o):
        v, m = o[0].to_numpy()
        s, k = trailing(np.concatenate([[0.0], np.cumsum(xf)]), 20)
        ok = k == 20
        return bool(np.array_equal(m, ok) and np.allclose(v[ok], s[ok] / 20, rtol=0, atol=1e-9))

    def check_r2(o):
        v, m = o[0].to_numpy()
        c = np.concatenate([np.zeros(1, np.uint64), np.cumsum(xi.view(np.uint64), dtype=np.uint64)])
        s, k = trailing(c, 100_000)
        ok = k == 100_000
        return bool(np.array_equal(m, ok) and np.array_equal(v[ok], s[ok].view(np.int64)))

    def check_r3(o):
        v, m = o[0].to_numpy()
        xv = np.where(m32, x32.astype(np.float64), 0.0)
        s1, _ = trailing(np.concatenate([[0.0], np.cumsum(xv)]), 50)
        s2, _ = trailing(np.concatenate([[0.0], np.cumsum(xv * xv)]), 50)
        k, _ = trailing(np.concatenate([[0], np.cumsum(m32)]), 50)
        ok = k >= 25
        var = (s2[ok] - s1[ok] ** 2 / k[ok]) / (k[ok] - 1)
        return bool(np.array_equal(m, ok) and np.allclose(v[ok], np.sqrt(np.maximum(var, 0)), rtol=1e-4, atol=1e-5))

    def check_r4(o):
        v, m = o[0].to_numpy()
        order = np.lexsort((np.arange(n), t, g4))
        gs = g4[order]
        head = np.ones(n, bool)
        head[1:] = gs[1:] != gs[:-1]
        start = np.maximum.accumulate(np.where(head, np.arange(n), 0))
        s, k = trailing(np.concatenate([[0.0], np.cumsum(xf[order])]), 10, start)
        want_ok = np.empty(n, bool)
        want_ok[order] = k == 10
        want = np.empty(n)
        want[order] = s / 10
        return bool(np.array_equal(m, want_ok) and np.allclose(v[want_ok], want[want_ok], rtol=0, atol=1e-6))

    work = {
        "R1": (lambda: plb.rolling([("rolling_mean", dxf, {"window_size": 20})], location=plb.DEVICE), check_r1),
        "R2": (lambda: plb.rolling([("rolling_sum", dxi, {"window_size": 100_000})], location=plb.DEVICE), check_r2),
        "R3": (lambda: plb.rolling([("rolling_std", dx32, {"window_size": 50, "min_samples": 25})], location=plb.DEVICE), check_r3),
        "R4": (lambda: plb.rolling([("rolling_mean", dxf, {"window_size": 10})], partition_by=[dg4], order_by=dt, location=plb.DEVICE), check_r4),
    }
    res = {"bench": "rolling", **card(), "rows": n, "steps": a.steps, "warmup": a.warmup, "workloads": {}}
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
             "kernels_ms": {k: round(v["ms"], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])}, "roofline": {}}
        for k, b in ROW_BYTES[name].items():
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
