"""Device string predicate benchmark (bl_string_compare, bl_string_match, bl_string_filter), device-resident inputs
generated from a seed, 1e8 rows unless noted.  Prints one JSON line.

  SM1  == "Brand#23" over 8-byte brands (25 values)
  SM2  starts_with("PROMO") over p_type-like rows (150 values, about 21 B)
  SM3  contains("green") over p_name-like rows (five of 92 colour words, about 33 B), both contains plans
  SM4  NOT LIKE '%special%requests%' with NO_NEWLINE over o_comment-like rows of 19-78 B
  SM5  contains("requests") over 1e6 rows of about 1 KB, both contains plans
  SM6  column < column over two p_name-like columns
  SM7  bl_string_filter at 10 % selectivity over the p_name-like rows
  SM8  contains("requests") over the o_comment-like rows (about 48 B), both contains plans

Rows are drawn from a pool of distinct values built on the host; the device columns are assembled on the GPU with torch.
Each result is checked once against pyarrow.compute run on the pool (result[pick]), outside the timed region.  Per
workload: ms/step (wall time of --steps steps ending in a device synchronise, after --warmup), per-kernel ms from one
profiled step, the algorithmic bytes (offsets + string bytes + the output bitmap, computed from the shapes) and their
share of the 3.35 TB/s HBM3 roofline, and a host pyarrow.compute time over the same rows (one run).  Both contains plans
run where both can (BL_STR_SCAN_MIN_ROW moves the plan rule).  The card name and power limit are read in the same run.
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

from bench_sort import card, timed      # noqa: E402

HBM = 3.35e12
COLOURS = ("almond antique aquamarine azure beige bisque black blanched blue blush brown burlywood burnished chartreuse chiffon chocolate "
           "coral cornflower cornsilk cream cyan dark deep dim dodger drab firebrick floral forest frosted gainsboro ghost goldenrod green "
           "grey honeydew hot indian ivory khaki lace lavender lawn lemon light lime linen magenta maroon medium metallic midnight mint "
           "misty moccasin navajo navy olive orange orchid pale papaya peach peru pink plum powder puff purple red rose rosy royal saddle "
           "salmon sandy seashell sienna sky slate smoke snow spring steel tan thistle tomato turquoise violet wheat white yellow").split()
WORDS = ("furiously quickly carefully blithely slyly ironic final regular express pending special bold even unusual silent idle "
         "deposits requests packages accounts theodolites instructions dependencies foxes pinto beans asymptotes platelets sleep "
         "wake haggle nag boost cajole detect integrate use among about above against along").split()


def pool_brands():
    return [f"Brand#{a}{b}".encode() for a in range(1, 6) for b in range(1, 6)]


def pool_types():
    return [f"{a} {b} {c}".encode() for a in ("STANDARD", "SMALL", "MEDIUM", "LARGE", "ECONOMY", "PROMO")
            for b in ("ANODIZED", "BURNISHED", "PLATED", "POLISHED", "BRUSHED") for c in ("TIN", "NICKEL", "BRASS", "STEEL", "COPPER")]


def pool_names(rng, k=65536):
    return [" ".join(rng.choice(COLOURS, 5, replace=False)).encode() for _ in range(k)]


def pool_comments(rng, k=65536, lo=19, hi=78):
    out = []
    while len(out) < k:
        target = int(rng.integers(lo, hi + 1))
        s = ""
        while len(s) < target:
            s += ("" if not s else " ") + str(rng.choice(WORDS))
        out.append(s[:target].encode())
    return out


def pool_long(rng, k=2048, width=1024):
    return [pool_comments(rng, 1, width, width)[0] for _ in range(k)]


class DevRows:
    """n rows drawn from `pool` by a seeded pick, assembled on the device (LargeUtf8 buffers)"""

    def __init__(self, torch, plb, pool, n, seed):
        g = torch.Generator(device="cuda").manual_seed(seed)
        lens_h = np.array([len(p) for p in pool], np.int64)
        w = int(lens_h.max())
        mat = np.zeros((len(pool), w), np.uint8)
        for i, p in enumerate(pool):
            mat[i, :len(p)] = np.frombuffer(p, np.uint8)
        self.pool, self.n = pool, n
        pmat = torch.from_numpy(mat).cuda()
        plens = torch.from_numpy(lens_h).cuda()
        self.pick = torch.randint(0, len(pool), (n,), generator=g, device="cuda")
        lens = plens[self.pick]
        self.offsets = torch.zeros(n + 1, dtype=torch.int64, device="cuda")
        self.offsets[1:] = torch.cumsum(lens, 0)
        total = int(self.offsets[-1])
        self.data = torch.empty(max(total, 1), dtype=torch.uint8, device="cuda")
        step = 5_000_000
        for r0 in range(0, n, step):
            r1 = min(n, r0 + step)
            ln = lens[r0:r1]
            rep = torch.repeat_interleave(torch.arange(r0, r1, device="cuda"), ln)
            j = torch.arange(rep.numel(), device="cuda", dtype=torch.int64) - (self.offsets[rep] - self.offsets[r0])
            self.data[int(self.offsets[r0]):int(self.offsets[r1])] = pmat[self.pick[rep], j]
            del rep, j
        torch.cuda.synchronize()
        self.bytes = total
        self.col = plb.DeviceStringColumn(st=plb.BlStringColumn(plb.DEVICE, 0, n, 0, 0, self.offsets.data_ptr(), self.data.data_ptr(), None, None))

    def arrow(self, pa):
        """the same rows on the host as a pyarrow LargeStringArray"""
        return pa.LargeStringArray.from_buffers(self.n, pa.py_buffer(self.offsets.cpu().numpy()), pa.py_buffer(self.data.cpu().numpy()))


def check(torch, got, pool_res, pick):
    vals, valid = got
    want = torch.from_numpy(np.asarray(pool_res, bool)).cuda()[pick].cpu().numpy()
    assert valid is None and np.array_equal(vals, want), "device result differs from pyarrow"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=100_000_000)
    ap.add_argument("--long-rows", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import pyarrow as pa
    import pyarrow.compute as pc
    import torch
    import polars_b200 as plb
    plb.init()
    rng = np.random.default_rng(a.seed)
    n = a.rows
    res = {"bench": "string_match", "rows": n, **card()}

    def run(name, fn, algo_bytes, host_fn, plan=None):
        if plan is not None:
            os.environ["BL_STR_SCAN_MIN_ROW"] = {"rows": "1e18", "scan": "0"}[plan]
        ms, prof = timed(plb, fn, a.steps, a.warmup)
        os.environ.pop("BL_STR_SCAN_MIN_ROW", None)
        t0 = time.perf_counter()
        host_fn()
        host_ms = (time.perf_counter() - t0) * 1e3
        res[name] = {"ms": round(ms, 3), "kernels_ms": {k: round(v["ms"], 3) for k, v in prof.items()}, "algo_bytes": int(algo_bytes),
                     "hbm_share": round(algo_bytes / HBM / (ms * 1e-3), 3), "host_pyarrow_ms": round(host_ms, 1)}

    out_bits = n / 8

    # SM1
    pool = pool_brands()
    r = DevRows(torch, plb, pool, n, a.seed + 1)
    pw = pa.array(pool, pa.large_binary())
    check(torch, plb.str_compare("eq", r.col, b"Brand#23"), pc.equal(pw, pa.scalar(b"Brand#23", pa.large_binary())).to_numpy(zero_copy_only=False), r.pick)
    ha = r.arrow(pa)
    run("SM1_eq", lambda: plb.str_compare("eq", r.col, b"Brand#23", location=plb.DEVICE), 8 * (n + 1) + r.bytes + out_bits,
        lambda: pc.equal(ha, "Brand#23"))
    del r, ha
    # SM2
    pool = pool_types()
    r = DevRows(torch, plb, pool, n, a.seed + 2)
    check(torch, plb.str_starts_with(r.col, b"PROMO"), pc.starts_with(pa.array(pool, pa.large_binary()), pattern="PROMO").to_numpy(zero_copy_only=False), r.pick)
    ha = r.arrow(pa)
    run("SM2_starts_with", lambda: plb.str_starts_with(r.col, b"PROMO", location=plb.DEVICE), 8 * (n + 1) + r.bytes + out_bits,
        lambda: pc.starts_with(ha, pattern="PROMO"))
    del ha
    # SM3, SM6, SM7 over p_name-like rows
    names = pool_names(rng)
    r = DevRows(torch, plb, names, n, a.seed + 3)
    pn = pa.array(names, pa.large_binary())
    check(torch, plb.str_contains(r.col, b"green", literal=True), pc.match_substring(pn, pattern="green").to_numpy(zero_copy_only=False), r.pick)
    os.environ["BL_STR_SCAN_MIN_ROW"] = "0"
    check(torch, plb.str_contains(r.col, b"green", literal=True), pc.match_substring(pn, pattern="green").to_numpy(zero_copy_only=False), r.pick)
    os.environ.pop("BL_STR_SCAN_MIN_ROW")
    ha = r.arrow(pa)
    for plan in ("rows", "scan"):
        run(f"SM3_contains_{plan}", lambda: plb.str_contains(r.col, b"green", literal=True, location=plb.DEVICE), 8 * (n + 1) + r.bytes + out_bits,
            lambda: pc.match_substring(ha, pattern="green"), plan)
    r2 = DevRows(torch, plb, names, n, a.seed + 4)
    ha2 = r2.arrow(pa)
    lt_ref = pc.less(ha, ha2).to_numpy(zero_copy_only=False)
    vals, valid = plb.str_compare("lt", r.col, r2.col)
    assert valid is None and np.array_equal(vals, lt_ref)
    run("SM6_lt_columns", lambda: plb.str_compare("lt", r.col, r2.col, location=plb.DEVICE), 16 * (n + 1) + r.bytes + r2.bytes + out_bits,
        lambda: pc.less(ha, ha2))
    del r2, ha2, lt_ref
    mask = np.random.default_rng(a.seed + 5).random(n) < 0.1
    mdev = plb.to_device(mask)
    kept = np.flatnonzero(mask)
    got = plb.str_filter(r.col, mdev, location=plb.DEVICE)
    lens = (r.offsets[1:] - r.offsets[:-1]).cpu().numpy()
    kept_bytes = int(lens[kept].sum())
    assert got.length == kept.size and int(got.st.length) == kept.size
    sample = kept[:: max(1, kept.size // 1000)]
    idx_in_out = np.searchsorted(kept, sample).astype(np.uint32)
    assert plb.string_gather(got, idx_in_out) == [names[i] for i in r.pick[torch.from_numpy(sample).cuda()].cpu().numpy()]
    del got
    hmask = pa.array(mask)
    run("SM7_filter", lambda: plb.str_filter(r.col, mdev, location=plb.DEVICE), 8 * (n + 1) + n / 8 + 8 * kept.size * 2 + 2 * kept_bytes,
        lambda: pc.filter(ha, hmask))
    del r, ha, mdev
    # SM4, SM8 over o_comment-like rows
    comments = pool_comments(rng)
    r = DevRows(torch, plb, comments, n, a.seed + 6)
    pcm = pa.array(comments, pa.large_binary())
    like_ref = ~pc.match_like(pa.array([c.decode() for c in comments], pa.large_string()), pattern="%special%requests%").to_numpy(zero_copy_only=False)
    check(torch, plb.str_like(r.col, "%special%requests%", negate=True, no_newline=True), like_ref, r.pick)
    ha = r.arrow(pa)
    hs = ha.cast(pa.large_string())
    run("SM4_not_like", lambda: plb.str_like(r.col, "%special%requests%", negate=True, no_newline=True, location=plb.DEVICE),
        8 * (n + 1) + r.bytes + out_bits, lambda: pc.invert(pc.match_like(hs, pattern="%special%requests%")))
    check(torch, plb.str_contains(r.col, b"requests", literal=True), pc.match_substring(pcm, pattern="requests").to_numpy(zero_copy_only=False), r.pick)
    for plan in ("rows", "scan"):
        run(f"SM8_contains_{plan}", lambda: plb.str_contains(r.col, b"requests", literal=True, location=plb.DEVICE), 8 * (n + 1) + r.bytes + out_bits,
            lambda: pc.match_substring(ha, pattern="requests"), plan)
    del r, ha, hs
    # SM5
    nl = a.long_rows
    longs = pool_long(rng)
    r = DevRows(torch, plb, longs, nl, a.seed + 7)
    ref = pc.match_substring(pa.array(longs, pa.large_binary()), pattern="requests").to_numpy(zero_copy_only=False)
    for plan in ("rows", "scan"):
        os.environ["BL_STR_SCAN_MIN_ROW"] = {"rows": "1e18", "scan": "0"}[plan]
        check(torch, plb.str_contains(r.col, b"requests", literal=True), ref, r.pick)
        os.environ.pop("BL_STR_SCAN_MIN_ROW")
    ha = r.arrow(pa)
    for plan in ("rows", "scan"):
        run(f"SM5_contains_1kb_{plan}", lambda: plb.str_contains(r.col, b"requests", literal=True, location=plb.DEVICE),
            8 * (nl + 1) + r.bytes + nl / 8, lambda: pc.match_substring(ha, pattern="requests"), plan)
    res["SM5_rows"] = nl
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
