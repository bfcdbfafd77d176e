"""Time-based rolling window benchmark (bl_rolling_by), device-resident inputs and outputs.  Prints one JSON line.

  RB1  Float64 rolling_mean_by("t", "30s") over sorted irregular Datetime(us) times (exponential gaps, mean 1 s): ~30 rows
       per window, no sort, the small-window plan (W <= 128)
  RB2  Int64 rolling_sum_by("t", "1d") on the same times: ~86 400 rows per window (windows across many blocks)
  RB3  Float32 rolling_std_by, 10 % nulls, closed="both", "30s", over the shuffled times: the sort, then the same plan
  RB4  rolling_mean_by("t", "5m").over("sym") with 1e4 symbols
  RB0  by = arange, "20i", next to bl_rolling(20) on the same Float64 values in the same call

Results are checked outside the timed region against numpy: on 4096 sampled rows (searchsorted bounds, exact slice sums),
and RB0 on every row (prefix sums) and against bl_rolling.
Per workload: ms/step (CUDA-synchronised wall time of `--steps` steps after `--warmup`), the per-kernel ms of one profiled
step, and for each rolling_by kernel its share of the HBM roofline: its algorithmic bytes per row (ROW_BYTES) x rows /
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
# bytes per row each kernel must move: values / times read, states written and read, bounds, results (24 B float SUM state,
# 16 B integer SUM state, 32 B VAR state)
ROW_BYTES = {
    "RB1": {"rolling_by_bounds": 8 + 8, "rolling_by_tile": 8 + 8 + 8 + 1 / 8, "rolling_by_prefix": 8 + 24, "rolling_by_suffix": 8 + 24, "rolling_by_out": 8 + 8 + 8 + 1 / 8},
    "RB2": {"rolling_by_bounds": 8 + 8, "rolling_by_prefix": 8 + 16, "rolling_by_suffix": 8 + 16, "rolling_by_out": 8 + 8 + 8 + 1 / 8},
    "RB3": {"rolling_by_bounds": 4 + 8 + 8, "rolling_by_tile": 4 + 4 + 1 / 8 + 4 + 4 + 4 + 4, "rolling_by_prefix": 4 + 4 + 4 + 32, "rolling_by_suffix": 4 + 4 + 4 + 32, "rolling_by_out": 8 + 4 + 4 + 4 + 4},
    "RB4": {"rolling_by_bounds": 4 + 8 + 8, "rolling_by_tile": 4 + 4 + 8 + 8 + 4 + 4 + 8, "rolling_by_prefix": 4 + 4 + 8 + 24, "rolling_by_suffix": 4 + 4 + 8 + 24, "rolling_by_out": 8 + 4 + 4 + 8 + 8},
    "RB0": {"rolling_by_bounds": 8 + 8, "rolling_by_tile": 8 + 8 + 8 + 1 / 8, "rolling_tile": 8 + 8},
}


def sample_check(got, valid_out, x, xvalid, t, tvalid, groups, P, closed, kind, ms, rows):
    """the exact value of `rows` from their windows: partition + time order, searchsorted bounds"""
    n = len(t)
    g = np.zeros(n, np.int64) if groups is None else groups.astype(np.int64)
    order = np.lexsort((np.arange(n), np.where(tvalid, t, 0), ~tvalid, g))
    gs, ts, tv = g[order], t[order], tvalid[order]
    pos = np.empty(n, np.int64)
    pos[order] = np.arange(n)
    for r in rows:
        p = pos[r]
        if not tv[p]:
            if valid_out[r]:
                return False
            continue
        lo = np.searchsorted(gs, gs[p], "left")
        hi = lo + np.count_nonzero(tv[lo:np.searchsorted(gs, gs[p], "right")])
        seg = ts[lo:hi]
        s = lo + np.searchsorted(seg, ts[p] - P, "left" if closed in ("left", "both") else "right")
        e = lo + np.searchsorted(seg, ts[p], "right" if closed in ("right", "both") else "left")
        rr = order[s:e]
        vals = x[rr][xvalid[rr]].astype(np.float64)
        k = len(vals)
        if e - s < ms or (kind != "rolling_sum" and k == 0) or (kind == "rolling_std" and k <= 1):
            if valid_out[r]:
                return False
            continue
        if not valid_out[r]:
            return False
        if kind == "rolling_sum":
            want = int(x[rr][xvalid[rr]].sum(dtype=np.int64)) if x.dtype.kind == "i" else vals.sum()
            if want != got[r] and not np.isclose(got[r], want, rtol=1e-9, atol=1e-6):
                return False
        elif kind == "rolling_mean":
            if not np.isclose(got[r], vals.mean(), rtol=1e-9, atol=1e-9):
                return False
        elif not np.isclose(got[r], vals.std(ddof=1), rtol=1e-4, atol=1e-4):
            return False
    return True


def run(a):
    import polars_b200 as plb
    plb.init(0)
    rng = np.random.default_rng(0)
    n = a.rows
    t = (np.cumsum(rng.exponential(1e6, n)) + 1.6e15).astype(np.int64)      # Datetime(us), mean gap 1 s
    ts = rng.permutation(t)
    xf = rng.standard_normal(n)
    xi = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    x32 = rng.standard_normal(n).astype(np.float32)
    m32 = rng.random(n) >= 0.1
    sym = rng.integers(0, 10_000, n).astype(np.int64)
    one = np.ones(n, bool)
    d = {k: plb.to_device(v) for k, v in (("t", t), ("ts", ts), ("xf", xf), ("xi", xi), ("sym", sym), ("ar", np.arange(n, dtype=np.int64)))}
    d["x32"] = plb.to_device(x32, m32)
    rows = rng.integers(0, n, 4096)
    S30, D1, M5 = 30_000_000, 86_400_000_000, 300_000_000

    def chk(o, x, xv, tt, gg, P, closed, kind, ms):
        v, m = o[0].to_numpy()
        m = one if m is None else m
        return sample_check(v, m, x, xv, tt, one, gg, P, closed, kind, ms, rows)

    def check_rb0(o):
        (a1, m1), (a2, m2) = o[0].to_numpy(), o[1].to_numpy()
        m1, m2 = (one if m is None else m for m in (m1, m2))
        c = np.concatenate([[0.0], np.cumsum(xf)])
        i = np.arange(n)
        lo = np.maximum(i - 19, 0)
        want = (c[i + 1] - c[lo]) / (i + 1 - lo)
        if not (m1.all() and np.allclose(a1, want, rtol=0, atol=1e-9)):
            return False
        return bool(np.array_equal(m1, m2) and np.allclose(a1[m1], a2[m2], rtol=1e-12, atol=1e-12))

    work = {
        "RB1": (lambda: plb.rolling_by([("rolling_mean", d["xf"], {"window_size": S30})], d["t"], location=plb.DEVICE),
                lambda o: chk(o, xf, one, t, None, S30, "right", "rolling_mean", 1)),
        "RB2": (lambda: plb.rolling_by([("rolling_sum", d["xi"], {"window_size": D1})], d["t"], location=plb.DEVICE),
                lambda o: chk(o, xi, one, t, None, D1, "right", "rolling_sum", 0)),
        "RB3": (lambda: plb.rolling_by([("rolling_std", d["x32"], {"window_size": S30, "closed": "both"})], d["ts"], location=plb.DEVICE),
                lambda o: chk(o, x32, m32, ts, None, S30, "both", "rolling_std", 1)),
        "RB4": (lambda: plb.rolling_by([("rolling_mean", d["xf"], {"window_size": M5})], d["t"], partition_by=[d["sym"]], location=plb.DEVICE),
                lambda o: chk(o, xf, one, t, sym, M5, "right", "rolling_mean", 1)),
        "RB0": (lambda: [plb.rolling_by([("rolling_mean", d["xf"], {"window_size": 20})], d["ar"], location=plb.DEVICE)[0],
                         plb.rolling([("rolling_mean", d["xf"], {"window_size": 20, "min_samples": 1})], location=plb.DEVICE)[0]], check_rb0),
    }
    res = {"bench": "rolling_by", **card(), "rows": n, "steps": a.steps, "warmup": a.warmup, "workloads": {}}
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
