"""Per-group median / quantile benchmark (BL_AGG_MEDIAN / BL_AGG_QUANTILE through bl_groupby_agg_params), device-resident
inputs, 1e8 rows by default.  Prints one JSON line.

  Q1  Float64 median, 1e6 groups (~100 rows each)             small-group plan
  Q2  Float64 median, 100 groups (~1e6 rows each)             large-group plan (radix sort)
  Q3  Q1 with quantiles 0.25, 0.5, 0.75 (linear) of the same column: one sort, three picks
  Q4  Int64 values with 5 % nulls, quantile 0.9 linear, 1e6 groups

Every workload is checked once against the vectorised numpy restatement (tests/quantile_oracle.py: one lexsort), outside
the timed region; that host computation is timed on the way and reported as numpy_ms (numpy, not Polars).  Q1 and Q2 are
also timed with every group forced through the large-group plan (BL_QUANTILE_GLOBAL=1), and the two plans' outputs are
compared byte for byte.  A step is the whole call: GroupsIdx (bl_group_tuples' kernels) + the quantile kernels.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, watts = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"card": name, "power_limit_w": float(watts)}
    except Exception as e:      # noqa: BLE001
        return {"card": None, "power_limit_w": None, "card_error": str(e)}


def timed(plb, fn, steps, warmup):
    for _ in range(warmup):
        fn()
    plb.sync()
    plb.profile_reset()
    plb.profile_enable(True)
    fn()                      # one profiled step: per-kernel times without the event overhead in the wall clock
    plb.sync()
    prof = plb.profile()
    plb.profile_enable(False)
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    plb.sync()
    return (time.perf_counter() - t0) / steps * 1e3, prof


def same(got, exp):
    (g, gv), (e, ev) = got, exp
    gv = np.ones(g.shape, bool) if gv is None else gv
    if g.dtype != e.dtype or not np.array_equal(gv, ev):
        return False
    g, e = g[ev], e[ev]
    return bool(((g == e) | (np.isnan(g) & np.isnan(e))).all())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default="")
    a = ap.parse_args()
    import polars_b200 as plb
    import quantile_oracle as qo
    plb.init(0)
    n = a.rows
    rng = np.random.default_rng(0)
    g_small = rng.integers(0, max(n // 100, 1), n)
    g_large = rng.integers(0, 100, n)
    x = rng.normal(size=n)
    iv, ivm = rng.integers(-(1 << 40), 1 << 40, n), rng.random(n) >= 0.05
    dev = {"gs": plb.to_device(g_small), "gl": plb.to_device(g_large), "x": plb.to_device(x), "iv": plb.to_device(iv, ivm)}
    D = plb.DEVICE
    work = {
        "Q1": dict(key="gs", gid=g_small, col="x", host=(x, None), kinds=["median"], qm=[(0.5, "linear")], both=True),
        "Q2": dict(key="gl", gid=g_large, col="x", host=(x, None), kinds=["median"], qm=[(0.5, "linear")], both=True),
        "Q3": dict(key="gs", gid=g_small, col="x", host=(x, None), kinds=["quantile:0.25:linear", "quantile:0.5:linear", "quantile:0.75:linear"],
                   qm=[(0.25, "linear"), (0.5, "linear"), (0.75, "linear")]),
        "Q4": dict(key="gs", gid=g_small, col="iv", host=(iv, ivm), kinds=["quantile:0.9:linear"], qm=[(0.9, "linear")]),
    }
    res = {"rows": n, "steps": a.steps, "warmup": a.warmup, **card(), "workloads": {}}
    for name, w in work.items():
        if a.only and name not in a.only.split(","):
            continue
        key, col = dev[w["key"]], dev[w["col"]]
        fn = lambda: plb.group_by_agg_keys([key], [(k, col) for k in w["kinds"]], maintain_order=True, location=D)       # noqa: E731

        def host_outs():
            _, outs = plb.group_by_agg_keys([key], [(k, col) for k in w["kinds"]], maintain_order=True)
            return outs
        outs = host_outs()
        # numpy restatement: group ids in first-occurrence order, one lexsort for all quantiles of the workload
        t0 = time.perf_counter()
        _, first, inv = np.unique(w["gid"], return_index=True, return_inverse=True)
        rank = np.empty(first.size, np.int64)
        rank[np.argsort(first, kind="stable")] = np.arange(first.size)
        dense = rank[inv.reshape(-1)]
        exps = qo.numpy_group_quantile(dense, w["host"][0], w["host"][1], [q for q, _ in w["qm"]], w["qm"][0][1], first.size)
        np_ms = (time.perf_counter() - t0) * 1e3
        verified = all(same(o, e) for o, e in zip(outs, exps))
        ms, prof = timed(plb, fn, a.steps, a.warmup)
        r = {"verified": verified, "groups": int(first.size), "ms": round(ms, 3), "rows_per_s": n / (ms / 1e3), "numpy_ms": round(np_ms, 1),
             "kernels_ms": {k: round(v["ms"], 3) for k, v in prof.items()}, "launches": {k: v["launches"] for k, v in prof.items()}}
        if w.get("both"):
            os.environ["BL_QUANTILE_GLOBAL"] = "1"
            try:
                gouts = host_outs()
                r["plans_identical"] = all(np.array_equal(a_[0].view(np.uint8), b_[0].view(np.uint8)) and
                                           np.array_equal(np.ones(a_[0].shape, bool) if a_[1] is None else a_[1], np.ones(b_[0].shape, bool) if b_[1] is None else b_[1])
                                           for a_, b_ in zip(outs, gouts))
                gms, gprof = timed(plb, fn, a.steps, a.warmup)
            finally:
                del os.environ["BL_QUANTILE_GLOBAL"]
            r["ms_global_plan"] = round(gms, 3)
            r["kernels_ms_global_plan"] = {k: round(v["ms"], 3) for k, v in gprof.items()}
        res["workloads"][name] = r
    res["verified"] = all(w["verified"] for w in res["workloads"].values())
    print(json.dumps(res))


if __name__ == "__main__":
    main()
