"""Device sort benchmark (bl_arg_sort / bl_sort), device-resident inputs, 1e8 rows by default.  Prints one JSON line.

  S1  Int64 keys over the full 64-bit range                      (8 radix passes)
  S2  Int64 keys in [0, 1e6)                                     (3 passes: the constant digits are skipped)
  S3  Float64 keys, 5 % nulls, descending, nulls_last            (8 value passes + 1 null-rank pass)
  S4  (Int32 in [0, 1000) descending, Float64)                   (8 passes on the Float64, 2 on the Int32)
  S5  bl_sort of S2 with an Int64 and a Float64 payload column
  S6  S5 with limit = 1000

Every workload is checked once against numpy (stable argsort / lexsort), outside the timed region.  Per workload:
ms/step (CUDA-synchronised wall time of `--steps` steps after `--warmup`), rows/s, per-kernel ms from bl_profile_*,
the radix passes actually run (launches of sort_scatter), the achieved bytes/s of the scatter passes
(2 * (key bytes + 4) per row and pass), and the host numpy.argsort(kind="stable") time of the same keys.

--compare LIB_A LIB_B: instead, time the existing callers of the radix sort (sort_pairs_u32) with two builds of the
library, alternating A B A B ... in fresh processes, and print both series plus the sort_scatter launches of one step:
  join_left_right  inner join, left = the 1e7-row build side, right = the 1e8-row probe side, maintain_order="left_right":
                   the right side probes (the longer relation), so the 1e8 tuples are re-sorted by left row (3 passes)
  group_tuples     bl_group_tuples over 1e8 rows / 1e6 keys: GroupsIdx row lists (the row sort, 4 passes, + the group sort)
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


def run_sort(a):
    import polars_b200 as plb
    import sort_oracle
    plb.init(0)
    n = a.rows
    rng = np.random.default_rng(0)
    s1 = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, dtype=np.int64)
    s2 = rng.integers(0, 1_000_000, n, dtype=np.int64)
    s3, s3v = rng.normal(size=n), rng.random(n) >= 0.05
    s4a = rng.integers(0, 1000, n).astype(np.int32)
    pf = rng.normal(size=n)
    dev = {k: plb.to_device(*v) for k, v in {"s1": (s1,), "s2": (s2,), "s3": (s3, s3v), "s4a": (s4a,), "s4b": (s3,), "pf": (pf,)}.items()}
    D = plb.DEVICE
    work = {
        "S1": dict(by=[dev["s1"]], desc=False, nl=False, keys=[(s1, None)], pass_keys=[8] * 8),
        "S2": dict(by=[dev["s2"]], desc=False, nl=False, keys=[(s2, None)], pass_keys=[8] * 3),
        "S3": dict(by=[dev["s3"]], desc=True, nl=True, keys=[(s3, s3v)], pass_keys=[8] * 8 + [4]),
        "S4": dict(by=[dev["s4a"], dev["s4b"]], desc=[True, False], nl=False, keys=[(s4a, None), (s3, None)], pass_keys=[8] * 8 + [4] * 2),
        "S5": dict(by=[dev["s2"]], desc=False, nl=False, keys=[(s2, None)], pass_keys=[8] * 3, payload=[dev["s1"], dev["pf"]]),
        "S6": dict(by=[dev["s2"]], desc=False, nl=False, keys=[(s2, None)], pass_keys=[8] * 3, payload=[dev["s1"], dev["pf"]], limit=1000),
    }
    res = {"rows": n, "steps": a.steps, "warmup": a.warmup, **card(), "workloads": {}}
    for name, w in work.items():
        if a.only and name not in a.only.split(","):
            continue
        by, limit = [d.view() for d in w["by"]], w.get("limit")
        if "payload" in w:
            pay = [d.view() for d in w["payload"]]
            fn = lambda: plb.sort(by, pay, w["desc"], w["nl"], limit=limit, location=D)       # noqa: E731
        else:
            fn = lambda: plb.arg_sort(by, w["desc"], w["nl"], limit=limit, location=D)        # noqa: E731
        # verification (once, untimed); the host reference is timed on the way (numpy, not Polars)
        out = fn()
        cols, valids = [k for k, _ in w["keys"]], [v for _, v in w["keys"]]
        simple = len(cols) == 1 and valids[0] is None and not w["desc"]
        t0 = time.perf_counter()
        exp = np.argsort(cols[0], kind="stable") if simple else sort_oracle.numpy_arg_sort(cols, valids, w["desc"], w["nl"])
        np_ms = (time.perf_counter() - t0) * 1e3
        exp = exp[:limit] if limit is not None else exp
        if "payload" in w:
            got0 = out[0].to_numpy()[0]
            ok = np.array_equal(got0, s1[exp]) and np.array_equal(out[1].to_numpy()[0], pf[exp])
        else:
            ok = np.array_equal(out.to_numpy()[0], exp)
        del out
        ms, prof = timed(plb, fn, a.steps, a.warmup)
        passes = int(prof.get("sort_scatter", {}).get("launches", 0))
        scatter_ms = prof.get("sort_scatter", {}).get("ms", 0.0)
        # bytes of the scatter passes, from the key width of every pass the workload is expected to run
        pass_bytes = sum(2 * (kb + 4) * n for kb in w["pass_keys"]) if passes == len(w["pass_keys"]) else None
        res["workloads"][name] = {"ok": bool(ok), "ms_per_step": round(ms, 3), "rows_per_s": n / ms * 1e3, "radix_passes": passes,
                                  "scatter_ms": round(scatter_ms, 3), "scatter_gbytes_per_s": round(pass_bytes / (scatter_ms * 1e-3) / 1e9, 1) if scatter_ms and pass_bytes else None,
                                  "kernels_ms": {k: round(v["ms"], 3) for k, v in prof.items() if v["ms"] > 0.01},
                                  "kernel_launches": {k: int(v["launches"]) for k, v in prof.items()},
                                  "numpy_ms": round(np_ms, 1), "numpy_method": "argsort(kind='stable')" if simple else "lexsort on transformed keys"}
        print(name, json.dumps(res["workloads"][name]), file=sys.stderr, flush=True)
    print(json.dumps(res), flush=True)
    return 0 if all(w["ok"] for w in res["workloads"].values()) else 1


def compare_child(a):
    import bench
    import polars_b200 as plb
    plb.init(0)
    probe, build = bench.gen_join(a.rows, a.build_rows, 2)
    dp, db = plb.to_device(probe), plb.to_device(build)
    key = plb.to_device(bench.gen_groupby(a.rows, 1_000_000, 1)[0])
    shapes = {"join_left_right": lambda: plb.hash_join(db.view(), dp.view(), "inner", False, "left_right", location=plb.DEVICE),
              "group_tuples": lambda: plb.group_tuples(key.view(), location=plb.DEVICE)}
    out = {"lib": plb.loaded_library()}
    for name, fn in shapes.items():
        ms, prof = timed(plb, fn, a.steps, a.warmup)
        out[name] = {"ms": ms, "sort_scatter_launches": int(prof.get("sort_scatter", {}).get("launches", 0)),
                     "sort_scatter_ms": prof.get("sort_scatter", {}).get("ms", 0.0)}
    print(json.dumps(out), flush=True)
    return 0


def compare(a):
    libs = [os.path.abspath(x) for x in a.compare]
    series = {lib: [] for lib in libs}
    for _ in range(a.rounds):
        for lib in libs:
            env = dict(os.environ, POLARS_B200_LIB=lib)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--compare-child", "--rows", str(a.rows), "--build-rows", str(a.build_rows),
                                "--steps", str(a.steps), "--warmup", str(a.warmup)], env=env, capture_output=True, text=True)
            if r.returncode != 0:
                print(r.stderr[-2000:], file=sys.stderr)
                return 1
            series[lib].append(json.loads(r.stdout.strip().splitlines()[-1]))
            print(json.dumps(series[lib][-1]), file=sys.stderr, flush=True)
    summary = {lib: {shape: {"ms": [round(x[shape]["ms"], 3) for x in runs], "median_ms": round(float(np.median([x[shape]["ms"] for x in runs])), 3),
                             "sort_scatter_launches": runs[0][shape]["sort_scatter_launches"]}
                     for shape in ("join_left_right", "group_tuples")} for lib, runs in series.items()}
    print(json.dumps({"rows": a.rows, "build_rows": a.build_rows, **card(), "libraries": a.compare, "results": summary}), flush=True)
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--build-rows", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default="", help="comma-separated workload names (S1..S6)")
    ap.add_argument("--compare", nargs=2, metavar="LIB", help="two builds of libpolars_b200.so to compare on the existing radix-sort callers")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--compare-child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.compare_child:
        return compare_child(a)
    if a.compare:
        return compare(a)
    return run_sort(a)


if __name__ == "__main__":
    sys.exit(main())
