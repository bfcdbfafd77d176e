"""CPU checks of tests/radix_ref.py (the placement rules of the partitioned group_by) against brute force: Python integers
for the hash, its inverse, the bucket and the start slot; an exhaustive search for the plan's bucket count."""
import numpy as np
import pytest

import radix_ref as rr

EDGE = [0, 1, 2, (1 << 31) - 1, 1 << 31, (1 << 32) - 1, 1 << 32, rr.GB_EMPTY, rr.GB_EMPTY - 1, rr.M64, rr.M64 - 1]


def test_table_hash_vectorised():
    rng = np.random.default_rng(1)
    ks = EDGE + [int(x) for x in rng.integers(0, 1 << 64, 2000, dtype=np.uint64)]
    got = rr.table_hash_np(np.array(ks, np.uint64))
    assert [int(x) for x in got] == [rr.table_hash(k) for k in ks]


def test_inverse():
    rng = np.random.default_rng(2)
    hs = EDGE + [int(x) for x in rng.integers(0, 1 << 64, 2000, dtype=np.uint64)]
    ks = rr.keys_with_hash_np(np.array(hs, np.uint64))
    assert [int(k) for k in ks] == [rr.key_with_hash(h) for h in hs]
    assert [rr.table_hash(int(k)) for k in ks] == hs


@pytest.mark.parametrize("logB", [6, 9, 10, 13])
def test_bucket_and_slot(logB):
    rng = np.random.default_rng(logB)
    S = 1312
    hs = EDGE + [int(x) for x in rng.integers(0, 1 << 64, 500, dtype=np.uint64)]
    b = rr.bucket_of(np.array(hs, np.uint64), logB)
    s = rr.start_slot(np.array(hs, np.uint64), logB, S)
    for h, bb, ss in zip(hs, b, s):
        assert int(bb) == h >> (64 - logB)
        t = ((h << logB) & rr.M64) >> 32
        assert int(ss) == (t * S) >> 32 and 0 <= int(ss) < S


@pytest.mark.parametrize("logB,S", [(6, 3968), (10, 1312), (13, 288)])
def test_keys64_in_bucket(logB, S):
    rng = np.random.default_rng(logB + S)
    B = 1 << logB
    for bucket in (0, 1, B // 2, B - 1):
        k = rr.keys64_in_bucket(rng, logB, bucket, 300, avoid=[rr.GB_EMPTY])
        assert k.size == 300 and np.unique(k).size == 300
        assert all(rr.table_hash(int(x)) >> (64 - logB) == bucket for x in k)
        for slot in (0, 1, S - 1):
            k = rr.keys64_in_bucket(rng, logB, bucket, 129, S=S, slot=slot)
            assert np.unique(k).size == 129
            for x in k:
                h = rr.table_hash(int(x))
                assert h >> (64 - logB) == bucket and ((((h << logB) & rr.M64) >> 32) * S) >> 32 == slot
    k = rr.keys64_in_bucket(rng, logB, 3, 50)
    k2 = rr.keys64_in_bucket(rng, logB, 3, 50, avoid=k)
    assert not np.isin(k2, k).any()


@pytest.mark.parametrize("logB", [6, 10, 13])
@pytest.mark.parametrize("dtype", ["int32", "uint32"])
def test_keys32_in_bucket(logB, dtype):
    rng = np.random.default_rng(logB)
    B = 1 << logB
    for bucket in (0, B - 1):
        bits = rr.keys32_in_bucket(rng, logB, bucket, 200)
        col = rr.as_dtype(bits, dtype)
        assert col.dtype == np.dtype(dtype) and np.unique(col).size == 200
        # the kernels load the 32-bit pattern zero-extended: Int32 negatives hash as 2^32 + k
        for v in col:
            pat = int(v) & 0xFFFFFFFF
            assert rr.table_hash(pat) >> (64 - logB) == bucket
        assert (rr.bucket_counts(col, logB) == np.bincount([bucket], minlength=B) * 200).all()


def test_bucket_counts_skip_empty_key():
    k = np.array([np.iinfo(np.int64).min, 5, 5, 7], np.int64)
    c = rr.bucket_counts(k, 6)
    assert c.sum() == 3 and c[rr.table_hash(5) >> 58] >= 2


@pytest.mark.parametrize("roww,n_words", [(1, 0), (2, 1), (3, 2), (4, 3), (5, 4), (5, 12)])
def test_plan_brute_force(roww, n_words):
    entry = 12 + 8 * n_words
    ring = 2 * 992 * roww * 8
    for est in [1, 1000, 10_000, 100_000, 400_000, 700_000, 1_000_000, 1_500_000, 3_000_000, 10_000_000, 40_000_000]:
        want = None
        for kb in (110, 222):
            if kb * 1024 < ring + 1024 + 512 * entry:
                continue
            S = ((kb * 1024 - ring - 1024) // entry) // 32 * 32
            ok = [lb for lb in range(6, 14) if est / 2 ** lb <= 0.55 * S]
            lb = ok[0] if ok else 13
            if est / 2 ** lb <= 0.7 * S:
                want = (lb, S)
                break
        assert rr.plan(est, roww, n_words) == want, (est, roww, n_words)
        # the table and the ring fit the block's budget
        if want:
            assert want[1] * entry + ring + 16 <= 222 * 1024
    lb, S = rr.plan(700_000, 3, 2)
    assert (lb, S) == (10, 2272)
    lo, hi = rr.est_range(lb, S)
    assert lo < 700_000 <= hi


def test_store_path():
    optin = 227 * 1024
    assert rr.store_path(6, 2, optin) == "runs" and rr.store_path(9, 5, optin) == "runs"
    assert rr.store_path(10, 3, optin) == "wc" and rr.store_path(11, 5, optin) == "coalesced"
    assert rr.store_path(10, 4, optin, knob=1) == "coalesced"
    assert rr.store_path(6, 2, optin, knob=2) == "wc"
    assert rr.store_path(13, 5, optin, knob=3) == "coalesced"     # runs do not fit: the automatic choice stays
    assert rr.store_path(13, 5, optin, knob=1) == "coalesced"
