"""Device top-k benchmark (bl_top_k, and bl_arg_sort / bl_sort with a limit), device-resident inputs, 1e8 rows by default.
Prints one JSON line.

  T1  Int64 over the full 64-bit range, k = 1000                  (bl_top_k)
  T2  the S6 shape of tools/bench_sort.py: bl_sort of Int64 keys in [0, 1e6) with an Int64 and a Float64 payload,
      limit = 1000                                                (the selection plan inside bl_sort)
  T3  Float64, 5 % nulls, descending, nulls last, k = 1e6          (bl_top_k)
  T4  (Int32 in [0, 1000) descending, Float64), k = 1e5            (bl_top_k)
  T5  all keys equal, k = 1000                                     (bl_top_k: only the row-index digits decide)
  T7  T5's keys through bl_arg_sort(limit = 1000) (the selection plan) and the full bl_arg_sort (the sort plan: no radix
      pass runs on equal keys), the case least favourable to the selection
  T6  the k sweep over the T1 keys, k = 1, 10, ..., n / 2: bl_top_k, bl_arg_sort(limit = k) and the full bl_arg_sort.
  T8  the limit rule: bl_arg_sort(limit = k) under both plans (BL_SORT_SELECT_DIV=1: always select, =0: always sort) for
      the T1 keys and the S2 keys (Int64 in [0, 1e6)), k = 1000 ... n / 2.  Both plans must give the same bytes.
  T9  low-cardinality keys: Int64 with 1, 2, 16 and 256 distinct values, limit = 1000, n / 64 and n / 8, both plans.
  T10 the list threshold: UInt32 keys whose top byte takes 4, 8, 16 or 32 values (the first bucket holds n / 4 ... n / 32
      rows) over random low bytes, bl_top_k(k = 1000) under BL_TOPK_LIST_DIV = 4, 8, 16, 32 and 64.

Every result is checked once against numpy (argpartition / lexsort), outside the timed region.  Per workload: ms/step
(CUDA-synchronised wall time of `--steps` steps after `--warmup`), per-kernel ms and launches from bl_profile_*, and the
streaming passes' bytes per second (the key bytes of every row, per pass).  The card name and power limit are read in
the same run.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_sort import card, timed      # noqa: E402


def first_k(order_keys, k):
    """ascending row ids of the first k rows of the stable order given by np.lexsort keys (least significant first)"""
    n = order_keys[0].size
    if len(order_keys) == 1 and k < n:
        key = order_keys[0]
        part = np.argpartition(key, k - 1)[:k] if k else np.zeros(0, np.int64)
        kth = key[part].max() if k else None
        if k:      # rows strictly below the k-th key, then the first rows of its tie run
            below = np.flatnonzero(key < kth)
            ties = np.flatnonzero(key == kth)[: k - below.size]
            return np.sort(np.concatenate([below, ties])).astype(np.uint32)
        return np.zeros(0, np.uint32)
    return np.sort(np.lexsort(order_keys)[:k]).astype(np.uint32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--only", default="", help="comma-separated workload names (T1..T10)")
    a = ap.parse_args()
    import polars_b200 as plb
    import sort_oracle
    plb.init(0)
    n = a.rows
    rng = np.random.default_rng(0)
    t1 = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, n, dtype=np.int64)
    s2 = rng.integers(0, 1_000_000, n, dtype=np.int64)
    t3, t3v = rng.normal(size=n), rng.random(n) >= 0.05
    t4a = rng.integers(0, 1000, n).astype(np.int32)
    pf = rng.normal(size=n)
    eq = np.full(n, 42, np.int64)
    dev = {k: plb.to_device(*v) for k, v in {"t1": (t1,), "s2": (s2,), "t3": (t3, t3v), "t4a": (t4a,), "t4b": (t3,), "pf": (pf,), "eq": (eq,)}.items()}
    D = plb.DEVICE
    res = {"rows": n, "steps": a.steps, "warmup": a.warmup, **card(), "workloads": {}}
    want = set(a.only.split(",")) if a.only else None

    def record(name, fn, expect, key_bytes, extra=None):
        out = fn()
        got = out.to_numpy()[0] if hasattr(out, "to_numpy") else out
        ok = bool(np.array_equal(got, expect()))
        del out
        ms, prof = timed(plb, fn, a.steps, a.warmup)
        stream = prof.get("topk_pass", {})
        r = {"ok": ok, "ms_per_step": round(ms, 3), "rows_per_s": n / ms * 1e3,
             "streaming_passes": int(stream.get("launches", 0)), "streaming_ms": round(stream.get("ms", 0.0), 3),
             "streaming_gbytes_per_s": round(key_bytes * n * stream["launches"] / (stream["ms"] * 1e-3) / 1e9, 1) if stream.get("ms") else None,
             "kernels_ms": {k: round(v["ms"], 3) for k, v in prof.items() if v["ms"] > 0.005},
             "kernel_launches": {k: int(v["launches"]) for k, v in prof.items()}, **(extra or {})}
        res["workloads"][name] = r
        print(name, json.dumps(r), file=sys.stderr, flush=True)
        return r

    v = lambda k: dev[k].view()      # noqa: E731
    if want is None or "T1" in want:
        record("T1", lambda: plb.arg_top_k(v("t1"), 1000, location=D), lambda: first_k([t1], 1000), 8)
    if want is None or "T2" in want:
        def t2():
            return plb.sort(v("s2"), [v("t1"), v("pf")], limit=1000, location=D)
        exp = np.argsort(s2, kind="stable")[:1000]
        out = t2()
        ok = np.array_equal(out[0].to_numpy()[0], t1[exp]) and np.array_equal(out[1].to_numpy()[0], pf[exp])
        del out
        r = record("T2", lambda: t2()[0], lambda: t1[exp], 8)
        r["ok"] = bool(ok)
    if want is None or "T3" in want:
        k3 = 1_000_000
        record("T3", lambda: plb.arg_top_k(v("t3"), k3, True, True, location=D),
               lambda: np.sort(sort_oracle.numpy_arg_sort([t3], [t3v], True, True, limit=k3)).astype(np.uint32), 8)
    if want is None or "T4" in want:
        k4 = 100_000
        record("T4", lambda: plb.arg_top_k([v("t4a"), v("t4b")], k4, [True, False], False, location=D),
               lambda: np.sort(np.lexsort([t3, -t4a.astype(np.int64)])[:k4]).astype(np.uint32), 12)
    if want is None or "T5" in want:
        record("T5", lambda: plb.arg_top_k(v("eq"), 1000, location=D), lambda: np.arange(1000, dtype=np.uint32), 8)
    if want is None or "T7" in want:
        sel_ms, sel_prof = timed(plb, lambda: plb.arg_sort(v("eq"), limit=1000, location=D), a.steps, a.warmup)
        srt_ms, _ = timed(plb, lambda: plb.arg_sort(v("eq"), location=D), a.steps, a.warmup)
        got = plb.arg_sort(v("eq"), limit=1000)
        res["workloads"]["T7"] = r = {"ok": bool(np.array_equal(got, np.arange(1000))), "select_ms": round(sel_ms, 3), "full_sort_ms": round(srt_ms, 3),
                                      "limit_plan": "select" if "topk_pass" in sel_prof else "sort"}
        print("T7", json.dumps(r), file=sys.stderr, flush=True)
    def both_plans(key_dev, k):
        """-> (select ms, sort ms, same bytes) of bl_arg_sort(limit = k) under the two plans"""
        fn = lambda: plb.arg_sort(key_dev.view(), limit=k, location=D)      # noqa: E731
        out = {}
        for plan, div in (("select", "1"), ("sort", "0")):
            os.environ["BL_SORT_SELECT_DIV"] = div
            got = plb.arg_sort(key_dev.view(), limit=k)
            ms, prof = timed(plb, fn, a.steps, a.warmup)
            assert ("topk_andor" in prof) == (plan == "select"), (plan, prof.keys())
            out[plan] = (ms, got)
        del os.environ["BL_SORT_SELECT_DIV"]
        return round(out["select"][0], 3), round(out["sort"][0], 3), bool(np.array_equal(out["select"][1], out["sort"][1]))

    if want is None or "T8" in want:
        rows, ok = [], True
        for name in ("t1", "s2"):
            for k in (1000, n // 64, n // 16, n // 8, n // 4, n // 2):
                sel_ms, srt_ms, same = both_plans(dev[name], k)
                ok = ok and same
                rows.append({"keys": name, "k": k, "select_ms": sel_ms, "sort_ms": srt_ms, "same_bytes": same})
                print("T8", json.dumps(rows[-1]), file=sys.stderr, flush=True)
        res["workloads"]["T8"] = {"ok": ok, "sweep": rows}
    if want is None or "T9" in want:
        rows, ok = [], True
        for distinct in (1, 2, 16, 256):
            lc = plb.to_device(rng.integers(0, distinct, n).astype(np.int64) * 7919 - 3)
            for k in (1000, n // 64, n // 8):
                sel_ms, srt_ms, same = both_plans(lc, k)
                ok = ok and same
                rows.append({"distinct": distinct, "k": k, "select_ms": sel_ms, "sort_ms": srt_ms, "same_bytes": same})
                print("T9", json.dumps(rows[-1]), file=sys.stderr, flush=True)
            del lc
        res["workloads"]["T9"] = {"ok": ok, "sweep": rows}
    if want is None or "T10" in want:
        rows, ok = [], True
        low = rng.integers(0, 1 << 24, n).astype(np.uint32)
        for tops in (4, 8, 16, 32):
            keys = (rng.integers(0, tops, n).astype(np.uint32) << np.uint32(24)) | low
            kd = plb.to_device(keys)
            exp = first_k([keys], 1000)
            for div in (4, 8, 16, 32, 64):
                os.environ["BL_TOPK_LIST_DIV"] = str(div)
                got = plb.arg_top_k(kd.view(), 1000)
                ms, prof = timed(plb, lambda: plb.arg_top_k(kd.view(), 1000, location=D), a.steps, a.warmup)
                same = bool(np.array_equal(got, exp))
                ok = ok and same
                rows.append({"first_bucket": f"n/{tops}", "list_div": div, "ms": round(ms, 3), "ok": same,
                             "passes_ms": {k: [int(v["launches"]), round(v["ms"], 3)] for k, v in prof.items() if k.startswith("topk")}})
                print("T10", json.dumps(rows[-1]), file=sys.stderr, flush=True)
            del os.environ["BL_TOPK_LIST_DIV"]
            del kd
        res["workloads"]["T10"] = {"ok": ok, "sweep": rows}
    if want is None or "T6" in want:
        full_ms, _ = timed(plb, lambda: plb.arg_sort(v("t1"), location=D), a.steps, a.warmup)
        sweep = []
        k = 1
        ks = []
        while k < n // 2:
            ks.append(k)
            k *= 10
        ks += [n // 256, n // 128, n // 64, n // 64 + 1, n // 32, n // 16, n // 8, n // 4, n // 2]
        order = None
        for k in sorted(set(ks)):
            ids = plb.arg_top_k(v("t1"), k, location=D)
            exp = first_k([t1], k)
            ok = np.array_equal(ids.to_numpy()[0], exp)
            del ids
            lim = plb.arg_sort(v("t1"), limit=k, location=D)
            if order is None:
                order = np.argsort(t1, kind="stable")
            ok = ok and np.array_equal(lim.to_numpy()[0], order[:k])
            del lim
            tk_ms, tk_prof = timed(plb, lambda: plb.arg_top_k(v("t1"), k, location=D), a.steps, a.warmup)
            lim_ms, lim_prof = timed(plb, lambda: plb.arg_sort(v("t1"), limit=k, location=D), a.steps, a.warmup)
            row = {"k": k, "ok": bool(ok), "top_k_ms": round(tk_ms, 3), "arg_sort_limit_ms": round(lim_ms, 3), "full_sort_ms": round(full_ms, 3),
                   "limit_plan": "select" if "topk_pass" in lim_prof else "sort",
                   "top_k_streaming_passes": int(tk_prof.get("topk_pass", {}).get("launches", 0)),
                   "top_k_list_passes": int(tk_prof.get("topk_pass_list", {}).get("launches", 0))}
            sweep.append(row)
            print("T6", json.dumps(row), file=sys.stderr, flush=True)
        res["workloads"]["T6"] = {"ok": all(r["ok"] for r in sweep), "full_sort_ms": round(full_ms, 3), "sweep": sweep}
    print(json.dumps(res), flush=True)
    return 0 if all(w["ok"] for w in res["workloads"].values()) else 1


if __name__ == "__main__":
    sys.exit(main())
