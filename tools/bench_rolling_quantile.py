"""Rolling quantile benchmark (bl_rolling_quantile / bl_rolling_quantile_by), device-resident inputs and outputs.  Prints one
JSON line.

  RQ1  rolling_median(20), Float64
  RQ2  the same with window_size = 100 000: the wavelet matrix's cost does not depend on the window width
  RQ3  rolling_quantile(0.95, "linear", 1000, min_samples=1, center=True), Int64 with 10 % nulls (with the default
       min_samples = window_size every window, ~900 valid values, would be null)
  RQ4  rolling_median(10).over(g, order_by=t), Float32, 1e6 groups
  RQ5  rolling_median_by("t", "1h") over sorted irregular Datetime(us) times (exponential gaps, mean 1 s): ~3600 rows
  RQ6  RQ5 over the same times shuffled (the sort of the positions, then the same query)

Results are checked outside the timed region: 1024 sampled rows against a brute force (the window's values sorted by numpy,
the reference's index and arithmetic from tests/rolling_quantile_oracle.py), and, when rows <= --full-max, every row of
RQ1 / RQ3 against the oracle's numpy wavelet matrix.
Per workload: ms/step (CUDA-synchronised wall time of `--steps` steps after `--warmup`), the per-kernel ms of one profiled
step, and the build's share of the HBM roofline: per level k_wm_count reads 4 bytes per row and k_wm_split reads 4 and
writes 4 + 1/7, so L x rows x (12 + 1/7) bytes / 3.35 TB/s over the two kernels' time.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_sort import card  # noqa: E402
import rolling_quantile_oracle as rq  # noqa: E402

HBM_TBPS = 3.35      # H100 SXM data sheet
BUILD_ROW_BYTES = 4 + 4 + 4 + 1 / 7


def brute(x, xv, rows_of_window, q, method, T):
    """the quantile of one window (row indices) from numpy's sort (NaN-free data), or None"""
    v = x[rows_of_window][xv[rows_of_window]].astype(T)
    if len(v) == 0:
        return None
    return rq.window_quantile(np.sort(v).tolist(), q, method, T)


def sample_fixed(got, gm, x, xv, order, seg_start, seg_end, pos, w, center, ms, q, method, T, rows):
    for r in rows:
        p = pos[r] if pos is not None else r
        lo, hi = (seg_start[p], seg_end[p]) if seg_start is not None else (0, len(x))
        if center:
            rr = w // 2 + (w & 1)
            s, e = max(p - (w - rr), lo), min(p + rr, hi)
        else:
            s, e = max(p - w + 1, lo), p + 1
        win = order[s:e] if order is not None else np.arange(s, e)
        k = int(xv[win].sum())
        want = brute(x, xv, win, q, method, T) if k >= max(ms, 1) else None
        if (want is None) != (not gm[r]):
            return False
        if want is not None and T(got[r]) != T(want):
            return False
    return True


def run(a):
    import polars_b200 as plb
    plb.init(0)
    rng = np.random.default_rng(0)
    n = a.rows
    one = np.ones(n, bool)
    xf = rng.standard_normal(n)
    xi = rng.integers(-(1 << 40), 1 << 40, n, dtype=np.int64)
    mi = rng.random(n) >= 0.1
    x32 = rng.standard_normal(n).astype(np.float32)
    g = rng.integers(0, 1_000_000, n).astype(np.int64)
    tg = rng.permutation(n).astype(np.int64)
    t = (np.cumsum(rng.exponential(1e6, n)) + 1.6e15).astype(np.int64)      # Datetime(us), mean gap 1 s
    ts = rng.permutation(t)
    d = {k: plb.to_device(v) for k, v in (("xf", xf), ("x32", x32), ("g", g), ("tg", tg), ("t", t), ("ts", ts))}
    d["xi"] = plb.to_device(xi, mi)
    rows = rng.integers(0, n, 1024)
    H1 = 3_600_000_000

    def host(o):
        v, m = o[0].to_numpy()
        return v, (one if m is None else m)

    def check_plain(w, center, ms, q, method, x, xv, T, full):
        def chk(o):
            v, m = host(o)
            if not sample_fixed(v, m, x, xv, None, None, None, None, w, center, ms, q, method, T, rows):
                return False
            if full and n <= a.full_max:
                i = np.arange(n)
                if center:
                    rr = w // 2 + (w & 1)
                    s, e = np.maximum(i - (w - rr), 0), np.minimum(i + rr, n)
                else:
                    s, e = np.maximum(i - w + 1, 0), i + 1
                ev, ok = rq.numpy_rolling_quantile(x, xv, "float32" if T is np.float32 else "float64", q, method, s, e, ms)
                return bool(np.array_equal(ok, m) and np.array_equal(np.where(ok, v, 0), np.where(ok, ev, 0)))
            return True
        return chk

    def check_over(o):
        v, m = host(o)
        order = np.lexsort((tg, g))
        pos = np.empty(n, np.int64)
        pos[order] = np.arange(n)
        gs = g[order]
        heads = np.concatenate([[0], np.nonzero(gs[1:] != gs[:-1])[0] + 1, [n]])
        idx = np.searchsorted(heads, np.arange(n), "right") - 1
        return sample_fixed(v, m, x32, one, order, heads[idx], heads[idx + 1], pos, 10, False, 10, 0.5, "linear", np.float32, rows)

    def check_by(tt):
        def chk(o):
            v, m = host(o)
            order = np.argsort(tt, kind="stable")
            st = tt[order]
            pos = np.empty(n, np.int64)
            pos[order] = np.arange(n)
            for r in rows:
                p = pos[r]
                s = np.searchsorted(st, st[p] - H1, "right")
                e = np.searchsorted(st, st[p], "right")
                want = brute(xf, one, order[s:e], 0.5, "linear", np.float64)
                if not m[r] or v[r] != want:
                    return False
            return True
        return chk

    med = {"quantile": 0.5, "interpolation": "linear"}
    work = {
        "RQ1": (lambda: plb.rolling_quantile([(d["xf"], dict(med, window_size=20))], location=plb.DEVICE),
                check_plain(20, False, 20, 0.5, "linear", xf, one, np.float64, True)),
        "RQ2": (lambda: plb.rolling_quantile([(d["xf"], dict(med, window_size=100_000))], location=plb.DEVICE),
                check_plain(100_000, False, 100_000, 0.5, "linear", xf, one, np.float64, False)),
        "RQ3": (lambda: plb.rolling_quantile([(d["xi"], {"quantile": 0.95, "interpolation": "linear", "window_size": 1000, "min_samples": 1,
                                              "center": True})],
                                             location=plb.DEVICE),
                check_plain(1000, True, 1, 0.95, "linear", xi, mi, np.float64, True)),
        "RQ4": (lambda: plb.rolling_quantile([(d["x32"], dict(med, window_size=10))], partition_by=[d["g"]], order_by=d["tg"], location=plb.DEVICE),
                check_over),
        "RQ5": (lambda: plb.rolling_quantile_by([(d["xf"], dict(med, window_size=H1))], d["t"], location=plb.DEVICE), check_by(t)),
        "RQ6": (lambda: plb.rolling_quantile_by([(d["xf"], dict(med, window_size=H1))], d["ts"], location=plb.DEVICE), check_by(ts)),
    }
    L = max(1, int(n - 1).bit_length())
    res = {"bench": "rolling_quantile", **card(), "rows": n, "levels": L, "steps": a.steps, "warmup": a.warmup, "workloads": {}}
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
        build_ms = sum(prof.get(k, {"ms": 0.0})["ms"] for k in ("rolling_quantile_wm_count", "rolling_quantile_wm_split"))
        roof = n * L * BUILD_ROW_BYTES / (HBM_TBPS * 1e12) * 1e3
        res["workloads"][name] = {
            "ok": ok, "ms_per_step": round(ms, 3), "rows_per_s": round(n / ms * 1e3),
            "kernels_ms": {k: round(v["ms"], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])},
            "build": {"ms": round(build_ms, 3), "roofline_ms": round(roof, 3), "share": round(roof / build_ms, 3) if build_ms else None}}
    print(json.dumps(res))
    return 0 if all(w["ok"] for w in res["workloads"].values()) else 1


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--full-max", type=int, default=20_000_000, help="check every row against the numpy wavelet matrix up to this many rows")
    ap.add_argument("--only", default="", help="comma-separated workload names")
    sys.exit(run(ap.parse_args()))


if __name__ == "__main__":
    main()
