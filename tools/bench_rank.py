"""Rank benchmark (bl_rank), device-resident inputs and outputs.  Prints one JSON line.

  R1  rank("average") of 1e8 Int64 (about 10 rows per tie run), next to bl_arg_sort of the same column in the same call
  R2  rank("dense", descending=True) of 1e8 Float64 with 10 % nulls
  R3  rank("ordinal").over(g) of 1e8 Int32 with 1e6 groups
  R4  rank("min") of 1e7 strings (1 to 8 lower-case letters)
  R5  rank("random") of R1's column

Every result is checked against numpy outside the timed region.  Per workload: ms/step (CUDA-synchronised wall time of
`--steps` steps after `--warmup`), the per-kernel ms of one profiled step, and for each rank kernel its share of the HBM
roofline: its algorithmic bytes (row_bytes below: what the kernel must read and write once, with runs / groups counted
from the data) over 3.35 TB/s, divided by its kernel time.  The random gather of the value in rank_heads and the random
scatter of the rank in rank_out move whole 32-byte sectors; the algorithmic bytes count only the element, so a share well
below 1 is expected there.
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


def row_bytes(name, runs, groups):
    """algorithmic bytes per row of each rank kernel; runs / groups: tie runs and partitions per row"""
    bm = 1 / 8      # one position bitmap
    if name in ("R1", "R4"):
        e = 8 if name == "R1" else 4      # R4 ranks the strings' UInt32 dense rank
        out = 8 if name == "R1" else 4
        return {"rank_heads": 4 + e + bm, "rank_starts": bm + 4 * runs, "rank_out": bm + 4 + 4 * runs + out}
    if name == "R2":
        return {"rank_heads": 4 + 8 + bm + 2 * bm, "rank_out": 2 * bm + 4 + 4}
    if name == "R3":
        return {"rank_heads": 4 + 4 + 2 * bm, "rank_starts": 2 * bm + 4 * groups, "rank_out": 2 * bm + 4 + 4 * groups + 4}
    return {"rank_random_key": 4, "rank_heads": 4 + bm, "rank_out": bm + 4 + 4}      # R5


def run(a):
    import polars_b200 as plb
    plb.init(0)
    rng = np.random.default_rng(0)
    n = a.rows
    x1 = rng.integers(0, max(n // 10, 1), n, dtype=np.int64)
    x2 = rng.integers(-10**6, 10**6, n).astype(np.float64) / 8
    m2 = rng.random(n) >= 0.1
    x3 = rng.integers(-10**5, 10**5, n).astype(np.int32)
    g3 = rng.integers(0, 1_000_000, n)
    ns = max(n // 10, 1)
    lens = rng.integers(1, 9, ns)
    offs = np.zeros(ns + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    data = rng.integers(ord("a"), ord("z") + 1, int(offs[-1])).astype(np.uint8)
    s4 = plb.DeviceStringColumn(plb.StringColumn(offsets=offs, data=data))
    d1, d2, d3, dg3 = plb.to_device(x1), plb.to_device(x2, m2), plb.to_device(x3), plb.to_device(g3)
    u1, inv1, c1 = np.unique(x1, return_inverse=True, return_counts=True)
    hi1 = np.cumsum(c1)
    lo1 = hi1 - c1 + 1

    def check_r1(o):
        v, m = o[0].to_numpy()
        return m is None and bool(np.array_equal(v, (0.5 * (lo1 + hi1.astype(np.float64)))[inv1]))

    def check_r2(o):
        v, m = o[0].to_numpy()
        u, inv = np.unique(x2[m2], return_inverse=True)
        want = np.zeros(n, np.uint32)
        want[m2] = len(u) - inv
        return bool(np.array_equal(m, m2) and np.array_equal(v, want))

    def check_r3(o):
        v, m = o[0].to_numpy()
        key = g3.astype(np.int64) * (1 << 32) + (x3.astype(np.int64) + (1 << 31))
        order = np.argsort(key, kind="stable")
        gs = g3[order]
        head = np.ones(n, bool)
        head[1:] = gs[1:] != gs[:-1]
        pos = np.arange(n)
        start = np.maximum.accumulate(np.where(head, pos, 0))
        want = np.empty(n, np.uint32)
        want[order] = pos - start + 1
        return m is None and bool(np.array_equal(v, want))

    def check_r4(o):
        v, m = o[0].to_numpy()
        fixed = np.zeros((ns, 8), np.uint8)
        idx = np.arange(int(offs[-1])) - np.repeat(offs[:-1], lens)
        fixed[np.repeat(np.arange(ns), lens), idx] = data
        s = fixed.view("S8").ravel()      # NUL padding sorts first: a proper prefix first, as bytes compare (no NULs in the data)
        _, inv, c = np.unique(s, return_inverse=True, return_counts=True)
        lo = np.cumsum(c) - c + 1
        return m is None and bool(np.array_equal(v, lo[inv.ravel()].astype(np.uint32)))

    def check_r5(o):
        v, m = o[0].to_numpy()
        v = v.astype(np.int64)
        perm_ok = bool(np.all(np.bincount(v, minlength=n + 1)[1:] == 1))
        return m is None and perm_ok and bool(np.all((v >= lo1[inv1]) & (v <= hi1[inv1])))

    work = {
        "R1": (lambda: plb.rank([(d1, {"method": "average"})], location=plb.DEVICE), check_r1),
        "R2": (lambda: plb.rank([(d2, {"method": "dense", "descending": True})], location=plb.DEVICE), check_r2),
        "R3": (lambda: plb.rank([(d3, {"method": "ordinal"})], partition_by=[dg3], location=plb.DEVICE), check_r3),
        "R4": (lambda: plb.rank([(s4, {"method": "min"})], location=plb.DEVICE), check_r4),
        "R5": (lambda: plb.rank([(d1, {"method": "random", "seed": 7})], location=plb.DEVICE), check_r5),
    }
    runs = {"R1": len(u1) / n, "R4": None, "R5": len(u1) / n}
    res = {"bench": "rank", **card(), "rows": n, "string_rows": ns, "steps": a.steps, "warmup": a.warmup, "workloads": {}}

    def timed(step):
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
        return (time.perf_counter() - t0) / a.steps * 1e3, prof

    for name, (step, check) in work.items():
        if a.only and name not in a.only.split(","):
            continue
        ok = bool(check(step()))
        ms, prof = timed(step)
        rows = ns if name == "R4" else n
        rho = runs.get(name)
        if name == "R4":
            rho = len(np.unique(plb.rank([(s4, {"method": "dense"})])[0][0])) / ns
        w = {"ok": ok, "ms_per_step": round(ms, 3), "rows_per_s": round(rows / ms * 1e3),
             "kernels_ms": {k: round(v["ms"], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])}, "roofline": {}}
        rank_ms = 0.0
        for k, b in row_bytes(name, rho or 0.0, 1_000_000 / n).items():
            if k in prof:
                rank_ms += prof[k]["ms"]
                roof = rows * b / (HBM_TBPS * 1e12) * 1e3
                w["roofline"][k] = {"ms": round(prof[k]["ms"], 3), "bytes_per_row": round(b, 3), "roofline_ms": round(roof, 3),
                                    "share": round(roof / prof[k]["ms"], 3)}
        w["rank_kernels_ms"] = round(rank_ms, 3)
        if name == "R1":
            sort_ms, _ = timed(lambda: plb.arg_sort(d1, location=plb.DEVICE))
            w["arg_sort_ms_per_step"] = round(sort_ms, 3)
            w["rank_kernels_over_arg_sort"] = round(rank_ms / sort_ms, 3)
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
