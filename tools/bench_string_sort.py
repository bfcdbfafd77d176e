"""Sort-by-string-key benchmark (bl_arg_sort_keys, bl_string_rank), device-resident inputs.  Prints one JSON line.

  T1  1e8 rows, 25 distinct short names (n_name-like), ascending
  T2  1e7 unique "Customer#%09d", shuffled: the constant 7-byte chunks ("Custome", ...) cost no sort
  T3  1e7 rows drawn from 1e6 random strings of length 0-40 over a 4-letter alphabet (deep refinement), 10 % nulls,
      descending, nulls_last
  T4  (T1's key, Int64 in [0, 1e6) descending) over 1e8 rows

Every workload is built as indices into a vocabulary whose order is known (the string column is gathered on the device
from the vocabulary), so its one correctness check, outside the timed region, is a numpy lexsort over integers.  Per
workload: ms/step (CUDA-synchronised wall time of `--steps` steps after `--warmup`), per-kernel ms of one profiled
bl_string_rank step split into encode (dedup: hash, group, verify) and rank (refinement rounds + rows), the row-sort ms
(one profiled arg_sort step minus its rank), the number of refinement rounds run (launches of str_rank_key), and the host
numpy stable argsort / lexsort time of the integer ranks (a lower bound for any host sort of the strings themselves).
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

NAMES = [b"ALGERIA", b"ARGENTINA", b"BRAZIL", b"CANADA", b"EGYPT", b"ETHIOPIA", b"FRANCE", b"GERMANY", b"INDIA", b"INDONESIA", b"IRAN", b"IRAQ",
         b"JAPAN", b"JORDAN", b"KENYA", b"MOROCCO", b"MOZAMBIQUE", b"PERU", b"CHINA", b"ROMANIA", b"SAUDI ARABIA", b"VIETNAM", b"RUSSIA",
         b"UNITED KINGDOM", b"UNITED STATES"]


def vocab_column(plb, words):
    lens = np.array([len(w) for w in words], np.int64)
    offs = np.zeros(len(words) + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    return plb.StringColumn(offsets=offs, data=np.frombuffer(b"".join(words), np.uint8))


def dense_ranks(words):
    _, inv = np.unique(np.array(list(words) + [b""], dtype=object)[:-1], return_inverse=True)
    return inv.astype(np.int64)


def kernel_split(prof):
    enc = {k: v for k, v in prof.items() if not (k.startswith("str_rank_") or k.startswith("sort_") or k.startswith("k3_") or k.startswith("scan_"))}
    rank = {k: v for k, v in prof.items() if k not in enc}
    return enc, rank


def run(a):
    import polars_b200 as plb
    import sort_oracle
    plb.init(0)
    rng = np.random.default_rng(0)
    N1, N2, N3 = a.rows, a.rows // 10, a.rows // 10
    # T1 / T4
    name_col, name_rank = vocab_column(plb, NAMES), dense_ranks(NAMES)
    i1 = rng.integers(0, len(NAMES), N1).astype(np.uint32)
    t1 = plb.string_gather(name_col, i1, location=plb.DEVICE)
    k1 = name_rank[i1]
    x4 = rng.integers(0, 1_000_000, N1, dtype=np.int64)
    d4 = plb.to_device(x4)
    # T2: "Customer#%09d" of a permutation, built directly (its rank is the number + 1)
    p2 = rng.permutation(N2).astype(np.int64)
    digits = ((p2[:, None] // 10 ** np.arange(8, -1, -1)) % 10 + 48).astype(np.uint8)
    mat = np.concatenate([np.tile(np.frombuffer(b"Customer#", np.uint8), (N2, 1)), digits], axis=1)
    t2 = plb.DeviceStringColumn(plb.StringColumn(offsets=np.arange(N2 + 1, dtype=np.int64) * 18, data=mat.ravel()))
    del mat, digits
    # T3: 1e6 random strings over "ACGT", lengths 0-40
    V3 = max(N3 // 10, 1)
    lens = rng.integers(0, 41, V3)
    alphabet = np.frombuffer(b"ACGT", np.uint8)
    data3 = alphabet[rng.integers(0, 4, int(lens.sum()))]
    offs3 = np.zeros(V3 + 1, np.int64)
    np.cumsum(lens, out=offs3[1:])
    words3 = [data3[offs3[i]:offs3[i + 1]].tobytes() for i in range(V3)]
    v3_rank = dense_ranks(words3)
    i3, valid3 = rng.integers(0, V3, N3).astype(np.uint32), rng.random(N3) >= 0.10
    t3 = plb.string_gather(plb.StringColumn(offsets=offs3, data=data3), (i3, valid3), location=plb.DEVICE)
    work = {
        "T1": dict(by=[t1], desc=False, nl=False, keys=[(k1, None)], n=N1),
        "T2": dict(by=[t2], desc=False, nl=False, keys=[(p2, None)], n=N2),
        "T3": dict(by=[t3], desc=True, nl=True, keys=[(v3_rank[i3], valid3)], n=N3),
        "T4": dict(by=[t1, d4], desc=[False, True], nl=False, keys=[(k1, None), (x4, None)], n=N1),
    }
    res = {"bench": "string_sort", **card(), "steps": a.steps, "warmup": a.warmup, "workloads": {}}
    for name, w in work.items():
        if a.only and name not in a.only.split(","):
            continue

        def step():
            return plb.arg_sort(w["by"], w["desc"], w["nl"], location=plb.DEVICE)
        got = step().to_numpy()[0]
        exp = sort_oracle.numpy_arg_sort([k for k, _ in w["keys"]], [v for _, v in w["keys"]], w["desc"], w["nl"])
        ok = bool(np.array_equal(got, exp))
        for _ in range(a.warmup):
            step()
        plb.sync()
        plb.profile_reset(); plb.profile_enable(True)
        for s in w["by"]:
            if isinstance(s, plb.DeviceStringColumn):
                plb.string_rank(s, location=plb.DEVICE)
        plb.sync()
        rank_prof = plb.profile()
        plb.profile_reset()
        step()
        plb.sync()
        full_prof = plb.profile()
        plb.profile_enable(False)
        t0 = time.perf_counter()
        for _ in range(a.steps):
            step()
        plb.sync()
        ms = (time.perf_counter() - t0) / a.steps * 1e3
        enc, rank = kernel_split(rank_prof)
        enc_ms, rank_ms = sum(v["ms"] for v in enc.values()), sum(v["ms"] for v in rank.values())
        full_ms = sum(v["ms"] for v in full_prof.values())
        t0 = time.perf_counter()
        cols = [k if v is None else np.where(v, -k if d else k, 0) for (k, v), d in zip(w["keys"], w["desc"] if isinstance(w["desc"], list) else [w["desc"]] * len(w["keys"]))]
        np.lexsort(cols[::-1]) if len(cols) > 1 else np.argsort(cols[0], kind="stable")
        host_ms = (time.perf_counter() - t0) * 1e3
        res["workloads"][name] = {"rows": w["n"], "ok": ok, "ms_per_step": round(ms, 3), "rows_per_s": round(w["n"] / ms * 1e3),
                                  "encode_ms": round(enc_ms, 3), "rank_ms": round(rank_ms, 3), "row_sort_ms": round(full_ms - enc_ms - rank_ms, 3),
                                  "rank_rounds": rank.get("str_rank_key", {}).get("launches", 0),
                                  "kernels_ms": {k: round(v["ms"], 3) for k, v in sorted(rank_prof.items(), key=lambda kv: -kv[1]["ms"])},
                                  "host_numpy_ms": round(host_ms, 1)}
    print(json.dumps(res))
    return 0 if all(w["ok"] for w in res["workloads"].values()) else 1


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=int, default=100_000_000, help="rows of T1 / T4; T2 and T3 use a tenth")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--only", default="", help="comma-separated workload names")
    sys.exit(run(ap.parse_args()))


if __name__ == "__main__":
    main()
