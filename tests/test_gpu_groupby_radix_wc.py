"""GPU tests of the partitioned group_by's many-bucket scatter (groupby_radix.cu k_gbr_scatter_wc: per-bucket chunk
buffers in shared memory, written out as whole-sector cp.async.bulk copies) against tests/groupby_ref.py.

K5r is forced with BL_K5_RADIX=2.  The bucket count follows from the sampled group estimate (about 1.25x the distinct
keys) and the shared-memory table of pass 2 (S slots for entries of 12 + 8 * words bytes): the plan takes the fewest
buckets with at most 0.55 * S estimated groups each.  Each case picks its group count in the middle of the range that
gives the bucket count it names, and the BL_K5_DEBUG line proves the bucket count and the store path.  Past what one
CTA's shared memory holds (B * 4 records of ROWW words) the plan keeps the coalesced-store scatter ("far" case).

Record widths 1 to 5 words (key + up to 4 value columns) with 4- and 8-byte value columns, 4- and 8-byte keys, and the
GB_EMPTY key (i64::MIN / u64 2^63: the pad marker of the record streams) on a group of 2^20 rows.  4-byte keys cannot
carry that bit pattern; their group of 2^20 rows is on an ordinary key.  Row counts are multiples of n_loop(sm_count) from
test_gpu_groupby_plans.py with a ragged tail, so every CTA of the persistent grid ends with partial chunks.  Float keys are not covered here: group_by_agg tracks first rows for them, which keeps them on the
L2 plan.  Integer aggregates and counts match bit for bit; float sums use exact-summable values.
"""
import re

import numpy as np
import pytest

import groupby_ref as ref
from test_gpu_groupby_plans import BIG, Call, _env, n_loop, profiled, value_cols

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as m
    m.init()
    return m


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


# name: (key dtype, value column dtypes (record width = 1 + len), extra min/max, distinct groups, rows / N_LOOP, buckets, store)
CASES = {
    "w1_i32key_1024": ("int32", (), False, 2_600_000, 3, 1024, "wc"),
    "w2_u64key_1024": ("uint64", ("uint32",), True, 700_000, 1, 1024, "wc"),
    "w3_c2_1024": ("int64", ("int64", "float64"), False, 700_000, 1, 1024, "wc"),
    "w3_c2_2048": ("int64", ("int64", "float64"), False, 1_400_000, 2, 2048, "wc"),
    "w4_i32key_1024": ("int32", ("int64", "uint32", "float32"), False, 420_000, 1, 1024, "wc"),
    "w5_1024": ("int64", ("int32", "uint64", "float64", "int64"), False, 225_000, 1, 1024, "wc"),
    "w5_2048_far": ("int64", ("int32", "uint64", "float64", "int64"), False, 450_000, 1, 2048, "coalesced"),
}
EMPTY_KEY = {"int64": np.iinfo(np.int64).min, "uint64": np.uint64(1 << 63), "int32": None}


@pytest.mark.parametrize("name", list(CASES))
def test_radix_many_buckets(plb, sm, monkeypatch, capfd, name):
    key_dt, dts, minmax, groups, mult, buckets, store = CASES[name]
    _env(monkeypatch, {"BL_K5_RADIX": "2", "BL_K5_HOTKEYS": "0", "BL_K5_DEBUG": "1"})
    rng = np.random.default_rng(len(name) * 7 + buckets)
    n = mult * n_loop(sm)
    singletons = 10_000
    case = ref.Case(rng, key_dt, big=BIG, singletons=singletons, groups=groups,
                    rest=n - BIG - singletons - sum(ref.SPECIAL_ROWS.values()), big_key=EMPTY_KEY[key_dt])
    cols = value_cols(case, rng, dts, False, exact=True)
    aggs = [("sum", c[1]) for c in cols]
    if minmax:
        aggs += [("min", c[2]) for c in cols] + [("max", c[2]) for c in cols]
    aggs.append(("len", None))
    capfd.readouterr()
    c, prof = profiled(plb, lambda: Call(plb, case.keys, None, aggs, False, device=True))      # host inputs this large take the pipelined L2 plan
    err = capfd.readouterr().err
    assert "k5r_scatter" in prof and "k5r_aggregate" in prof, sorted(prof)
    line = [ln for ln in err.splitlines() if ln.startswith("[k5r]")][-1]
    assert re.search(rf"\bbuckets={buckets}\b", line) and "bulk=0" in line and f"store={store}" in line and "status=0" in line, line
    c.check(None, f"radix {name}")
