"""CPU restatement of where the group_by plans put a key: table_hash (dev_utils.cuh), the bucket and pass-2 start slot of
the partitioned group_by (K5r, groupby_radix.cu), the bucket count / table size that consume_radix picks, the shared
memory of its scatter paths, and key builders that land keys in a chosen bucket (and start slot).

  h      = table_hash(key)                  key = the 64-bit pattern the kernels load (4-byte keys zero-extended)
  bucket = h >> (64 - logB)
  slot   = umulhi((u32)((h << logB) >> 32), S)     (the 32 hash bits below the bucket bits, scaled to S slots)
"""
import numpy as np

M64 = (1 << 64) - 1
HASH_MUL = 0x9E3779B97F4A7C15                       # table_hash: (k ^ (k >> 31)) * HASH_MUL
HASH_INV = pow(HASH_MUL, -1, 1 << 64)
GB_EMPTY = 1 << 63                                  # i64::MIN: the empty-slot / pad marker
MAX_LOGB = 13                                       # GBR_MAX_LOGB
NCT = 31 * 32                                       # GBR_NCT: records per pass-2 ring stage (one per consumer thread)
NST = 2                                             # GBR_NST: ring stages
SCATTER_ROWS = 512 * 4                              # k_gbr_scatter tile (GBR_THREADS x GBR_RPT)
WC_F = 4                                            # GBR_WC_F: records per write-combining chunk
MIN_ROWS = 1 << 20                                  # consume_radix takes no smaller batch


def wc_tile(roww: int) -> int:
    """Rows of one k_gbr_scatter_wc tile: 256 threads x 8 rows (records of <= 3 words) or x 4."""
    return 256 * (8 if roww <= 3 else 4)


def table_hash(k: int) -> int:
    return ((k ^ (k >> 31)) * HASH_MUL) & M64


def key_with_hash(h: int) -> int:
    """The 64-bit key whose table_hash is h (both steps of the hash are invertible)."""
    x = (h * HASH_INV) & M64
    k = x ^ (x >> 31) ^ (x >> 62)
    assert table_hash(k) == h
    return k


def table_hash_np(bits) -> np.ndarray:
    """table_hash of an array of 64-bit patterns (uint64 arithmetic wraps mod 2^64)."""
    k = np.asarray(bits).astype(np.uint64)
    with np.errstate(over="ignore"):
        return (k ^ (k >> np.uint64(31))) * np.uint64(HASH_MUL)


def keys_with_hash_np(h) -> np.ndarray:
    h = np.asarray(h, np.uint64)
    with np.errstate(over="ignore"):
        x = h * np.uint64(HASH_INV)
    return x ^ (x >> np.uint64(31)) ^ (x >> np.uint64(62))


def key_bits(keys) -> np.ndarray:
    """The 64-bit pattern the K5r kernels load: 8-byte keys as is, 4-byte keys zero-extended."""
    keys = np.asarray(keys)
    if keys.dtype.itemsize == 8:
        return keys.view(np.uint64)
    return keys.view(np.uint32).astype(np.uint64)


def bucket_of(h, logB: int):
    return np.asarray(h, np.uint64) >> np.uint64(64 - logB)


def start_slot(h, logB: int, S: int):
    t = (np.asarray(h, np.uint64) << np.uint64(logB)) >> np.uint64(32)
    return (t * np.uint64(S)) >> np.uint64(32)


def bucket_counts(keys, logB: int) -> np.ndarray:
    """Rows per bucket (k_gbr_hist): GB_EMPTY-key rows are not in any bucket."""
    b = key_bits(keys)
    b = b[b != np.uint64(GB_EMPTY)]
    return np.bincount(bucket_of(table_hash_np(b), logB).astype(np.int64), minlength=1 << logB)


def plan(est_groups: int, roww: int, n_words: int):
    """(logB, S) of consume_radix: the shared-memory table of pass 2 is what is left of 110 KB (2 CTAs / SM) after the
    2-stage ring, or of 222 KB (1 CTA / SM) when 8192 buckets of the smaller table cannot take the estimate; the fewest
    buckets with at most 0.55 * S estimated groups each.  None: the plan does not apply."""
    entry = 12 + 8 * n_words
    ring = NST * NCT * roww * 8
    for total_kb in (110, 222):
        if total_kb * 1024 < ring + 1024 + 512 * entry:
            continue
        S = ((total_kb * 1024 - ring - 1024) // entry) & ~31
        logB = 6
        while logB < MAX_LOGB and est_groups / (1 << logB) > 0.55 * S:
            logB += 1
        if est_groups / (1 << logB) <= 0.7 * S:
            return logB, S
    return None


def max_used(S: int) -> int:
    """Groups one bucket's table takes before pass 2 gives up (status -> the L2 plan)."""
    return S - S // 4


def est_range(logB: int, S: int):
    """(lo, hi]: the est_groups for which plan() picks 2^logB buckets (of the same S)."""
    lo = 0.0 if logB == 6 else 0.55 * S * (1 << (logB - 1))
    hi = 0.55 * S * (1 << logB) if logB < MAX_LOGB else 0.7 * S * (1 << logB)
    return lo, hi


def scatter_smem(B: int, roww: int, runs: bool) -> int:
    """Dynamic shared memory of k_gbr_scatter: the staged tile (+ a pad record per bucket for the runs), three
    per-bucket counters, and (coalesced store) the bucket of every staged record."""
    return (SCATTER_ROWS + (B if runs else 0)) * roww * 8 + 3 * B * 4 + (0 if runs else SCATTER_ROWS * 2)


def wc_smem(B: int, roww: int) -> int:
    """Dynamic shared memory of k_gbr_scatter_wc: a chunk of WC_F records and a fill counter per bucket."""
    return B * (WC_F * roww * 8 + 4)


def store_path(logB: int, roww: int, optin: int, knob: int = 0) -> str:
    """The scatter's store path: runs up to 512 buckets, then write-combining where its buffers fit, else coalesced;
    BL_K5R_STORE = knob (1 coalesced, 2 write-combining, 3 runs) wherever that path's shared memory fits."""
    B = 1 << logB
    if knob == 1 and scatter_smem(B, roww, False) <= optin:
        return "coalesced"
    if knob == 2 and wc_smem(B, roww) <= optin:
        return "wc"
    if knob == 3 and scatter_smem(B, roww, True) <= optin:
        return "runs"
    if logB <= 9:
        return "runs"
    return "wc" if wc_smem(B, roww) <= optin else "coalesced"


def keys64_in_bucket(rng, logB: int, bucket: int, count: int, S: int | None = None, slot: int | None = None,
                     avoid=()) -> np.ndarray:
    """`count` distinct 64-bit key patterns (uint64) in `bucket`, by exact inversion of the hash: the top logB hash bits
    are the bucket; with `slot`, the next 32 bits are drawn from the range that umulhi maps to that start slot of an
    S-slot table.  Never GB_EMPTY; never a pattern in `avoid`."""
    lo_bits = 32 - logB                              # hash bits below the 32 start-slot bits
    if slot is not None:
        t_lo = -(-slot * (1 << 32) // S)             # smallest t with umulhi(t, S) == slot
        t_hi = -(-(slot + 1) * (1 << 32) // S)
    else:
        t_lo, t_hi = 0, 1 << 32
    avoid = np.asarray(avoid, np.uint64)
    out = np.zeros(0, np.uint64)
    while out.size < count:
        t = rng.integers(t_lo, t_hi, 2 * count + 16, dtype=np.uint64)
        low = rng.integers(0, 1 << lo_bits, 2 * count + 16, dtype=np.uint64)
        h = (np.uint64(bucket) << np.uint64(64 - logB)) | (t << np.uint64(lo_bits)) | low
        k = keys_with_hash_np(h)
        k = k[(k != np.uint64(GB_EMPTY)) & ~np.isin(k, avoid)]
        out = np.concatenate([out, k])
        _, first = np.unique(out, return_index=True)
        out = out[np.sort(first)]
    return out[:count]


def keys32_in_bucket(rng, logB: int, bucket: int, count: int, avoid=()) -> np.ndarray:
    """`count` distinct 32-bit key patterns (as uint64, zero-extended) whose hash lands in `bucket`: random 32-bit
    candidates, filtered."""
    avoid = np.asarray(avoid, np.uint64)
    out = np.zeros(0, np.uint64)
    while out.size < count:
        c = rng.integers(0, 1 << 32, 1 << 22, dtype=np.uint64)
        c = c[(bucket_of(table_hash_np(c), logB) == np.uint64(bucket)) & ~np.isin(c, avoid)]
        out = np.concatenate([out, c])
        _, first = np.unique(out, return_index=True)
        out = out[np.sort(first)]
    return out[:count]


def as_dtype(bits: np.ndarray, dtype) -> np.ndarray:
    """Key patterns from the builders as a key column of `dtype` (4-byte dtypes take the low 32 bits)."""
    dt = np.dtype(dtype)
    if dt.itemsize == 8:
        return np.asarray(bits, np.uint64).view(dt)
    return np.asarray(bits, np.uint64).astype(np.uint32).view(dt)
