"""Asof join benchmark (bl_join_asof), device-resident inputs.  Prints one JSON line.

  A1  1e8 left x 1e7 right sorted Int64 timestamps, backward
  A2  A1 with nearest and a tolerance
  A3  A1 with an Int64 `by` of 1e4 symbols; both sides sorted by time globally, so the fused left check suffices
  A4  A3 with a string `by` ("SYM%05d"); the left side sorted by (symbol, time) only, so the left rows are sorted by group
      and checked per group (the second check path)

A1 / A2 / A3 / A4 cover both sides of the one input-dependent choice (the fused global left check, or the per-group
sort-and-check when it fails).  Every result is checked against the vectorised per-row rule of tests/asof_oracle.py (numpy
searchsorted) outside the timed region.  Per workload: ms/step (CUDA-synchronised wall time of `--steps` steps after
`--warmup`), the per-kernel ms of one profiled step, and the algorithmic bytes of the plan without `by` (left keys read,
index and validity written, the right keys read by the check and by the searches) over the step time.
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

from bench_sort import card  # noqa: E402

HBM_TBPS = 3.35      # H100 SXM data sheet


def symbol_column(plb, n_sym, idx):
    words = [b"SYM%05d" % i for i in range(n_sym)]
    offs = np.arange(n_sym + 1, dtype=np.int64) * 8
    vocab = plb.StringColumn(offsets=offs, data=np.frombuffer(b"".join(words), np.uint8))
    return plb.string_gather(vocab, idx.astype(np.uint32), location=plb.DEVICE)


def run(a):
    import asof_oracle as ao
    import polars_b200 as plb
    plb.init(0)
    rng = np.random.default_rng(0)
    nl, nr, n_sym = a.rows, a.rows // 10, 10_000
    span = 10**12
    lv = np.sort(rng.integers(0, span, nl)).astype(np.int64)
    rv = np.sort(rng.integers(0, span, nr)).astype(np.int64)
    lsym, rsym = rng.integers(0, n_sym, nl), rng.integers(0, n_sym, nr)
    dl, dr = plb.to_device(lv), plb.to_device(rv)
    dls, drs = plb.to_device(lsym.astype(np.int64)), plb.to_device(rsym.astype(np.int64))
    # A4: left rows ordered by (symbol, time)
    order = np.lexsort((lv, lsym))
    lv4, lsym4 = lv[order], lsym[order]
    dl4 = plb.to_device(lv4)
    sl4, sr = symbol_column(plb, n_sym, lsym4), symbol_column(plb, n_sym, rsym)
    tol = span // nr
    work = {
        "A1": dict(args=(dl, dr, "backward", None), by=None, check=lambda: ao.rule_asof((lv, None), (rv, None), "backward")),
        "A2": dict(args=(dl, dr, "nearest", tol), by=None, check=lambda: ao.rule_asof((lv, None), (rv, None), "nearest", True, tol)),
        "A3": dict(args=(dl, dr, "backward", None), by=([dls], [drs]), check=lambda: ao.rule_asof((lv, None), (rv, None), "backward", True, None, lsym, rsym)),
        "A4": dict(args=(dl4, dr, "backward", None), by=([sl4], [sr]), check=lambda: ao.rule_asof((lv4, None), (rv, None), "backward", True, None, lsym4, rsym)),
    }
    res = {"bench": "join_asof", **card(), "left_rows": nl, "right_rows": nr, "steps": a.steps, "warmup": a.warmup, "workloads": {}}
    for name, w in work.items():
        if a.only and name not in a.only.split(","):
            continue
        l, r, strategy, t = w["args"]
        lb, rb = w["by"] if w["by"] else (None, None)

        def step():
            return plb.join_asof(l, r, strategy, t, True, lb, rb, location=plb.DEVICE)
        idx, valid = step().to_numpy()
        valid = np.ones(nl, bool) if valid is None else valid
        eidx, evalid = w["check"]()
        ok = bool(np.array_equal(valid, evalid) and np.array_equal(idx, eidx))
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
        bytes_moved = nl * 8 + nl * 4 + nl / 8 + 2 * nr * 8
        res["workloads"][name] = {"ok": ok, "ms_per_step": round(ms, 3), "left_rows_per_s": round(nl / ms * 1e3),
                                  "matched": int(evalid.sum()),
                                  "kernels_ms": {k: round(v["ms"], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])},
                                  "plan_bytes_without_by": int(bytes_moved), "roofline_ms": round(bytes_moved / (HBM_TBPS * 1e12) * 1e3, 3)}
    print(json.dumps(res))
    return 0 if all(w["ok"] for w in res["workloads"].values()) else 1


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=int, default=100_000_000, help="left rows; the right side has a tenth")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--only", default="", help="comma-separated workload names")
    sys.exit(run(ap.parse_args()))


if __name__ == "__main__":
    main()
