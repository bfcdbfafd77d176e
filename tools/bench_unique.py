"""Device unique benchmark (bl_unique, bl_unique_mask), device-resident inputs, 1e8 rows by default.  Prints one JSON line.

  U1  Int64, 1e6 distinct keys, uniform
  U2  Int64, 1e3 distinct keys                    (the shared-memory K5 plan)
  U3  Int64, Zipf(1.1)                            (heavy hitters)
  U4  Int64, all distinct, shuffled               (the table leaves L2)
  U5  (Int32, Int64) pairs, 1e6 distinct pairs    (op_pack_keys)
  U6  1e7 rows holding 1e6 distinct 10-byte strings (the string codes first); --rows / 10 rows

Per workload: keep = first / last / none (bl_unique) and the four masks (bl_unique_mask), each as ms/step
(CUDA-synchronised wall time of `--steps` steps after `--warmup`) with per-kernel ms from bl_profile_*; the baselines
bl_group_tuples(key).out_first (U1-U4: the only device answer before bl_unique, which must give the same bytes as
keep="first") and a host np.unique(return_index=True) of the same key.  Every result is checked once against numpy,
outside the timed region.  The card name and power limit are read in the same run.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_sort import card, timed      # noqa: E402

KEEPS = {"first": "first", "last": "last", "none": "unique"}
MASKS = ("first", "last", "unique", "duplicated")


def masks_of(g):
    """the four masks from an int64 group id per row (the oracle's (first, last, count) table, in numpy)"""
    n = g.size
    _, first, inv, count = np.unique(g, return_index=True, return_inverse=True, return_counts=True)
    inv = inv.reshape(-1)
    last = n - 1 - np.unique(g[::-1], return_index=True)[1]
    rows = np.arange(n)
    return {"first": first[inv] == rows, "last": last[inv] == rows, "unique": count[inv] == 1, "duplicated": count[inv] > 1}


def fixed_strings(ids, width=10):
    """LargeUtf8 buffers of 'k' + the id in width - 1 decimal digits, built without Python strings"""
    n = ids.size
    digits = np.zeros((n, width), np.uint8)
    digits[:, 0] = ord("k")
    v = ids.astype(np.int64).copy()
    for j in range(width - 1, 0, -1):
        digits[:, j] = ord("0") + v % 10
        v //= 10
    return np.arange(n + 1, dtype=np.int64) * width, digits.reshape(-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--only", default="", help="comma-separated workload names (U1..U6)")
    a = ap.parse_args()
    import polars_b200 as plb
    plb.init(0)
    n = a.rows
    rng = np.random.default_rng(0)
    want = set(a.only.split(",")) if a.only else None
    res = {"rows": n, "steps": a.steps, "warmup": a.warmup, **card(), "workloads": {}}
    D = plb.DEVICE

    def run(name, keys, group_ids, baseline_key=None):
        """keys: the device key arguments; group_ids: int64 group id per row (numpy) for the check"""
        t0 = time.perf_counter()
        m = masks_of(group_ids)
        check_s = time.perf_counter() - t0
        r = {"distinct": int(m["first"].sum()), "ok": True, "ops": {}}
        for keep, kind in KEEPS.items():
            got = plb.arg_unique(keys, keep)
            ok = bool(np.array_equal(got, np.flatnonzero(m[kind])))
            ms, prof = timed(plb, lambda: plb.arg_unique(keys, keep, location=D), a.steps, a.warmup)
            r["ops"]["keep_" + keep] = {"ok": ok, "ms_per_step": round(ms, 3), "kernels_ms": {k: round(v["ms"], 3) for k, v in prof.items() if v["ms"] > 0.005}}
            r["ok"] &= ok
        fns = {"first": plb.is_first_distinct, "last": plb.is_last_distinct, "unique": plb.is_unique, "duplicated": plb.is_duplicated}
        for kind in MASKS:
            ok = bool(np.array_equal(fns[kind](keys), m[kind]))
            ms, prof = timed(plb, lambda: fns[kind](keys, location=D), a.steps, a.warmup)
            r["ops"]["is_" + kind] = {"ok": ok, "ms_per_step": round(ms, 3), "kernels_ms": {k: round(v["ms"], 3) for k, v in prof.items() if v["ms"] > 0.005}}
            r["ok"] &= ok
        if baseline_key is not None:
            dev, host = baseline_key
            first, _, _ = plb.group_tuples(dev, location=D)
            same = bool(np.array_equal(first.to_numpy()[0], plb.arg_unique(keys, "first")))
            del first
            ms, prof = timed(plb, lambda: plb.group_tuples(dev, location=D), a.steps, a.warmup)
            r["baseline_group_tuples"] = {"same_bytes_as_keep_first": same, "ms_per_step": round(ms, 3),
                                          "kernels_ms": {k: round(v["ms"], 3) for k, v in prof.items() if v["ms"] > 0.005}}
            r["ok"] &= same
            t0 = time.perf_counter()
            _, idx = np.unique(host, return_index=True)
            r["baseline_host_np_unique_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
            r["ok"] &= bool(np.array_equal(np.sort(idx), np.flatnonzero(m["first"])))
        r["check_s"] = round(check_s, 1)
        res["workloads"][name] = r
        print(name, json.dumps(r), file=sys.stderr, flush=True)

    def single(name, x):
        d = plb.to_device(x)
        run(name, d.view(), x, (d.view(), x))
        del d

    if want is None or "U1" in want:
        single("U1", rng.integers(0, 1_000_000, n, dtype=np.int64) * 7919 - 10**12)
    if want is None or "U2" in want:
        single("U2", rng.integers(0, 1000, n, dtype=np.int64))
    if want is None or "U3" in want:
        single("U3", rng.zipf(1.1, n).astype(np.int64))
    if want is None or "U4" in want:
        single("U4", rng.permutation(n).astype(np.int64))
    if want is None or "U5" in want:
        p, q = rng.integers(0, 1000, n).astype(np.int32), rng.integers(0, 1000, n, dtype=np.int64) << 40
        dp, dq = plb.to_device(p), plb.to_device(q)
        run("U5", [dp.view(), dq.view()], p.astype(np.int64) * 1000 + (q >> 40))
        del dp, dq
    if want is None or "U6" in want:
        ns = n // 10
        ids = rng.integers(0, 1_000_000, ns) * 997 % 1_000_000_007
        offs, data = fixed_strings(ids)
        ds = plb.DeviceStringColumn(plb.StringColumn(offsets=offs, data=data))
        run("U6", [ds], ids)
        del ds
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
