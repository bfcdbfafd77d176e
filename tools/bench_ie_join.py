"""Inequality join benchmark (bl_ie_join), device-resident inputs and outputs.  Prints one JSON line.

  I1  a single `<` on Int64, 1e5 left x 2e4 right random values: about 1e9 pairs (bound by the emit's stores)
  I2  point-in-interval: 1e7 Int64 points x 1e6 disjoint intervals in shuffled order, l.t >= r.start, l.t < r.end
  I3  interval overlap on Float64: 1e6 x 1e6 short intervals, l.start < r.end, l.end > r.start
  I4  I2 as a left join with 5 % nulls in every predicate column

Every output is checked against numpy outside the timed region: I2-I4 exactly (searchsorted over the sorted right side);
I1 by the per-left-row pair count and the per-left-row sum of right rows (both against searchsorted and a suffix sum) plus
the predicate on every emitted pair.  Per workload: ms/step (CUDA-synchronised wall time of `--steps` steps after `--warmup`),
the per-kernel ms of one profiled step, the pair count, and the emit's algorithmic bytes (8 B written and 4 B read per
pair) over the step time.
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
CHUNK = 100_000_000


def host_pairs(res):
    (li, _), (ri, rv) = res[0].to_numpy(), res[1].to_numpy()
    return np.array(li), np.array(ri), (None if rv is None else np.array(rv))


def check_i1(l, r, li, ri):
    """counts and sums of right rows per left row against the sorted right side; the predicate on every pair"""
    if li.size and np.any(np.diff(li.astype(np.int64)) < 0):
        return False
    order = np.argsort(r, kind="stable")
    rs = r[order]
    start = np.searchsorted(rs, l, "right")              # l < r: the suffix of the sorted right side from `start`
    exp_cnt = len(r) - start
    suffix = np.concatenate([np.cumsum(order[::-1].astype(np.int64))[::-1], [0]])
    exp_sum = suffix[start]
    cnt = np.bincount(li, minlength=len(l))
    got_sum = np.zeros(len(l), np.int64)
    for a in range(0, li.size, CHUNK):
        lc, rc = li[a:a + CHUNK], ri[a:a + CHUNK]
        if not np.all(l[lc] < r[rc]):
            return False
        got_sum += np.bincount(lc, weights=rc.astype(np.float64), minlength=len(l)).astype(np.int64)      # exact: sums < 2^53
    return bool(np.array_equal(cnt, exp_cnt) and np.array_equal(got_sum, exp_sum))


def interval_expect(t, tvalid, start, end, rvalid, how):
    """points t against disjoint intervals [start, end): at most one right row per point"""
    live = np.nonzero(rvalid)[0]
    order = live[np.argsort(start[live], kind="stable")]
    s, e = start[order], end[order]
    k = np.searchsorted(s, t, "right") - 1
    hit = tvalid & (k >= 0) & (t < e[np.maximum(k, 0)])
    rows = np.nonzero(hit if how == "inner" else np.ones(len(t), bool))[0]
    rr = np.where(hit, order[np.maximum(k, 0)], 0xFFFFFFFF).astype(np.uint32)[rows]
    return rows.astype(np.uint32), rr, hit[rows]


def overlap_expect(ls, le, rs, re_, maxlen):
    """l.start < r.end and l.end > r.start for right intervals no longer than maxlen: candidates from a searchsorted window"""
    order = np.argsort(rs, kind="stable")
    s, e = rs[order], re_[order]
    lo = np.searchsorted(s, ls - maxlen, "left")
    hi = np.searchsorted(s, le, "left")
    li, ri = [], []
    for k in range(int((hi - lo).max()) if len(ls) else 0):
        j = lo + k
        ok = j < hi
        jj = np.minimum(j, len(s) - 1)
        ok &= e[jj] > ls
        li.append(np.nonzero(ok)[0])
        ri.append(order[jj[ok]])
    li = np.concatenate(li) if li else np.zeros(0, np.int64)
    ri = np.concatenate(ri) if ri else np.zeros(0, np.int64)
    key = li.astype(np.int64) * len(rs) + ri
    return np.sort(key)


def run(a):
    import polars_b200 as plb
    plb.init(0)
    rng = np.random.default_rng(0)
    D = plb.DEVICE
    # I1
    l1, r1 = rng.integers(0, 10**9, 100_000).astype(np.int64), rng.integers(0, 10**9, 20_000).astype(np.int64)
    # I2 / I4: 1e6 disjoint intervals of random lengths with gaps, shuffled; 1e7 points over the whole span
    n_int, n_pt = 1_000_000, 10_000_000
    gaps = rng.integers(1, 1000, n_int).astype(np.int64)
    lens = rng.integers(1, 1000, n_int).astype(np.int64)
    starts = np.cumsum(gaps + lens) - lens
    ends = starts + lens
    perm = rng.permutation(n_int)
    st2, en2 = starts[perm], ends[perm]
    pts = rng.integers(0, int(ends[-1]) + 1000, n_pt).astype(np.int64)
    ptv = rng.random(n_pt) >= 0.05
    stv, env = rng.random(n_int) >= 0.05, rng.random(n_int) >= 0.05
    # I3: 1e6 x 1e6 intervals of length < 2 over [0, 1e6)
    n3 = 1_000_000
    ls3 = rng.random(n3) * 1e6
    le3 = ls3 + rng.random(n3) * 2.0
    rs3 = rng.random(n3) * 1e6
    re3 = rs3 + rng.random(n3) * 2.0
    dev = plb.to_device
    work = {
        "I1": dict(args=([dev(l1)], [dev(r1)], ["<"], "inner")),
        "I2": dict(args=([dev(pts), dev(pts)], [dev(st2), dev(en2)], [">=", "<"], "inner")),
        "I3": dict(args=([dev(ls3), dev(le3)], [dev(re3), dev(rs3)], ["<", ">"], "inner")),
        "I4": dict(args=([dev(pts, ptv), dev(pts, ptv)], [dev(st2, stv), dev(en2, env)], [">=", "<"], "left")),
    }
    res = {"bench": "ie_join", **card(), "steps": a.steps, "warmup": a.warmup, "workloads": {}}
    for name, w in work.items():
        if a.only and name not in a.only.split(","):
            continue
        lon, ron, ops, how = w["args"]

        def step():
            return plb.ie_join(lon, ron, ops, how, location=D)
        li, ri, rv = host_pairs(step())
        if name == "I1":
            ok = check_i1(l1, r1, li, ri)
        elif name in ("I2", "I4"):
            if name == "I2":
                erows, err, ehit = interval_expect(pts, np.ones(n_pt, bool), st2, en2, np.ones(n_int, bool), "inner")
            else:
                erows, err, ehit = interval_expect(pts, ptv, st2, en2, stv & env, "left")
            valid = np.ones(len(ri), bool) if rv is None else rv
            ok = bool(np.array_equal(li, erows) and np.array_equal(valid, ehit) and np.array_equal(ri, err))
        else:
            ok = bool(np.array_equal(np.sort(li.astype(np.int64) * n3 + ri), overlap_expect(ls3, le3, rs3, re3, 2.0))
                      and not np.any(np.diff(li.astype(np.int64)) < 0))
        pairs = int(li.size)
        del li, ri, rv
        for _ in range(a.warmup):
            step()
        plb.sync()
        plb.profile_reset()
        plb.profile_enable(True)
        step()
        plb.sync()
        prof = plb.profile()
        plb.profile_enable(False)
        t0 = time.perf_counter()
        for _ in range(a.steps):
            step()
        plb.sync()
        ms = (time.perf_counter() - t0) / a.steps * 1e3
        emit_bytes = pairs * 12
        res["workloads"][name] = {"verified": ok, "ms_per_step": round(ms, 3), "pairs": pairs,
                                  "kernels_ms": {k: round(v["ms"], 3) for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])},
                                  "emit_bytes": emit_bytes, "emit_roofline_ms": round(emit_bytes / (HBM_TBPS * 1e12) * 1e3, 3)}
    res["verified"] = all(w["verified"] for w in res["workloads"].values())
    print(json.dumps(res))
    return 0 if res["verified"] else 1


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--only", default="", help="comma-separated workload names")
    sys.exit(run(ap.parse_args()))


if __name__ == "__main__":
    main()
