"""CPU tests (-m "not gpu") of the asof join: the cursor oracle against the reference's known answers
(tests/golden/asof_kats.json), an exhaustive proof over small alphabets that the per-row rule the device computes gives the
cursors' answer under the precondition, the vectorised rule against the scalar one, and the binding's argument handling."""
import ctypes as C
import itertools
import json
import os
import re

import numpy as np
import pytest

import asof_oracle as ao
from test_cabi_cpu import declared_symbols

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRATS = (ao.BACKWARD, ao.FORWARD, ao.NEAREST)


def asof_kats():
    with open(os.path.join(ROOT, "tests", "golden", "asof_kats.json")) as f:
        return json.load(f)["asof"]


def typed(values, dtype):
    """None-list -> numpy scalars of the dtype (None kept)"""
    return [None if v is None else np.dtype(dtype).type(v) for v in values]


def by_rows(cols, n):
    return [tuple(c[i] for c in cols) for i in range(n)] if cols else None


def oracle_kat(case):
    left, right = typed(case["left"], case["dtype"]), typed(case["right"], case["dtype"])
    tol = None if case["tol"] is None else np.dtype(case["dtype"]).type(case["tol"])
    if case["left_by"]:
        return ao.cursor_asof_by(left, right, by_rows(case["left_by"], len(left)), by_rows(case["right_by"], len(right)), case["strategy"], case["allow_eq"], tol)
    return ao.cursor_asof(left, right, case["strategy"], case["allow_eq"], tol)


def kat_payload(case, idx):
    pay = case["payload"] if case["payload"] is not None else list(range(len(case["right"])))
    return [None if j is None else pay[j] for j in idx]


def same(got, exp):
    return len(got) == len(exp) and all((g is None and e is None) or (g is not None and e is not None and (g == e or (g != g and e != e))) for g, e in zip(got, exp))


@pytest.mark.parametrize("case", asof_kats(), ids=lambda c: c["cite"][-70:])
def test_oracle_matches_reference_kats(case):
    assert same(kat_payload(case, oracle_kat(case)), case["expect"])


KAT_SOURCES = {"test_asof_backward", "test_asof_backward_tolerance", "test_asof_forward_tolerance", "test_asof_forward",
               "test_join_asof_floats", "test_join_asof_tolerance", "test_join_asof_tolerance_forward", "test_asof_join_nearest",
               "test_asof_join_nearest_reference", "test_asof_join_nearest_with_tolerance", "test_asof_join_nearest_by",
               "test_asof_join_nearest_by_with_tolerance", "test_join_asof_no_exact_matches", "test_join_asof_large_int_21276",
               "test_join_asof_int_dtypes_24383", "test_join_asof_nans", "test_join_asof_by_nulls_27165", "test_join_asof_by_nulls_27165_2"}


def test_kats_cover_every_source_strategy_and_option():
    ks = asof_kats()
    assert KAT_SOURCES <= {re.search(r"\((test_[a-z0-9_]+)", k["cite"]).group(1) for k in ks}
    assert {k["strategy"] for k in ks} == set(STRATS)
    assert any(k["tol"] is not None for k in ks) and any(not k["allow_eq"] for k in ks) and any(k["left_by"] for k in ks)


def test_nan_quirks_of_the_nearest_cursor():
    """inside the precondition the nearest cursor picks the NaN row for a larger left value, and not the exact match when a
    NaN follows it"""
    r = typed([0.0, 5.0, np.nan], "float64")
    assert ao.cursor_asof(typed([6.0], "float64"), r, ao.NEAREST, True) == [2]
    assert ao.cursor_asof(typed([5.0], "float64"), r, ao.NEAREST, True) == [0]
    assert ao.rule_lists([6.0], [0.0, 5.0, np.nan], ao.NEAREST, True, dtype="float64") == [2]
    assert ao.rule_lists([5.0], [0.0, 5.0, np.nan], ao.NEAREST, True, dtype="float64") == [0]


def test_interspersed_right_nulls_break_the_rule():
    """why the precondition rejects right nulls after the first non-null: the nearest cursor then skips the exact match"""
    r = typed([3, None, 5], "int32")
    assert not ao.precondition_ok(typed([3], "int32"), r)
    assert ao.cursor_asof(typed([3], "int32"), r, ao.NEAREST, True) == [2]


# ------------------------------------------------------------------------------------------------ exhaustive proof
ALPHABETS = {
    "int32": [-1, 0, 1, 2],
    "float32": [-1.0, -0.0, 0.0, 1.0, 2.0, np.nan],
    "float64": [-1.0, -0.0, 0.0, 1.0, 2.0, np.nan],
}
MAXLEN = 4


def sorted_sequences(alpha, dtype, right):
    """every sequence of length <= MAXLEN over alpha + null satisfying the precondition of its side"""
    syms = typed([None] + alpha, dtype)
    out = []
    for n in range(MAXLEN + 1):
        for seq in itertools.product(syms, repeat=n):
            seq = list(seq)
            if right:
                ok = ao.precondition_ok([], seq)
            else:
                ok = ao.precondition_ok(seq, [])
            if ok:
                out.append(seq)
    return out


def scalar_rule(l, right, strategy, allow_eq):
    """the per-row rule of the header, literally, on a None-list whose nulls come first"""
    n = len(right)
    z = 0
    while z < n and right[z] is None:
        z += 1
    V = range(z, n)
    k = ao.tot_key(l)
    if strategy == ao.BACKWARD:
        c = [j for j in V if ao.tot_key(right[j]) < k or (allow_eq and ao.tot_key(right[j]) == k)]
        return c[-1] if c else None
    if strategy == ao.FORWARD:
        c = [j for j in V if ao.tot_key(right[j]) > k or (allow_eq and ao.tot_key(right[j]) == k)]
        return c[0] if c else None
    U = next((j for j in V if right[j] > l), n)
    if allow_eq and U > z and right[U - 1] == l:
        return U - 1
    if U < n:
        while U + 1 < n and right[U + 1] == right[U]:
            U += 1
    L = next((j for j in range(z, U) if right[j] >= l), None)
    L = U - 1 if L is None else L - 1
    hasL, hasU = L >= z, U < n
    if hasL and hasU:
        return U if ao.abs_diff(l, right[U]) <= ao.abs_diff(l, right[L]) else L
    return U if hasU else (L if hasL else None)


@pytest.mark.parametrize("dtype", sorted(ALPHABETS))
@pytest.mark.parametrize("strategy", STRATS)
def test_per_row_rule_equals_the_cursors_exhaustively(dtype, strategy):
    """all left sequences x all right sequences (length <= 4, precondition holds) x allow_eq x tolerance {none, 0, 1}.
    The left sequences are walked as a prefix tree, so each cursor step is taken once per right sequence.  The cursor side
    is the reference restated (the cursor step, then join_asof_impl's tolerance filter, default.rs:43,60,127-135); the rule
    side is the header's rule twice over: scalar_rule without a tolerance, and the vectorised rule_asof, with its own
    tolerance arithmetic, for every tolerance."""
    alpha = ALPHABETS[dtype]
    rights = sorted_sequences(alpha, dtype, right=True)
    lsyms = typed([None] + alpha, dtype)
    avals = np.array(alpha, dtype)
    tols = [None, np.dtype(dtype).type(0), np.dtype(dtype).type(1)]
    filters = [ao._filter(t) for t in tols]
    checked = 0
    for allow_eq in (False, True):
        for right in rights:
            table = {i: scalar_rule(v, right, strategy, allow_eq) for i, v in enumerate(lsyms) if v is not None}
            rv = np.array([0 if v is None else v for v in right], dtype)
            rvalid = np.array([v is not None for v in right], bool)
            vec = []      # per tolerance: symbol index -> the vectorised rule's answer
            for t in tols:
                idx, ok = ao.rule_asof((avals, None), (rv, rvalid), strategy, allow_eq, t)
                vec.append({i + 1: (int(j) if o else None) for i, (j, o) in enumerate(zip(idx, ok))})
            all_null_right = all(v is None for v in right)
            stack = [([], ao.STATES[strategy](allow_eq))]
            while stack:
                seq, st = stack.pop()
                if len(seq) == MAXLEN:
                    continue
                for si, v in enumerate(lsyms):
                    nseq = seq + [v]
                    if not ao.precondition_ok(nseq, []):
                        continue
                    nst = ao.STATES[strategy](allow_eq)
                    nst.__dict__.update(st.__dict__)
                    got = None if v is None or all_null_right else nst.next(v, right)
                    exp = None if v is None else table[si]
                    assert got == exp, (dtype, strategy, allow_eq, right, nseq)
                    for t, keep, vt in zip(tols, filters, vec):
                        g = got if got is not None and keep(v, right[got]) else None
                        assert g == (None if v is None else vt[si]), (dtype, strategy, allow_eq, t, right, nseq)
                    checked += 1
                    stack.append((nseq, nst))
    assert checked > 10_000


def test_sweep_covers_every_sorted_sequence():
    """every sequence of length <= 4 over {null, -1.0, -0.0, 0.0, 1.0, 2.0, NaN}: 768 left and 386 right sequences"""
    assert len(sorted_sequences(ALPHABETS["float64"], "float64", right=False)) == 768
    assert len(sorted_sequences(ALPHABETS["float64"], "float64", right=True)) == 386


def sorted_side(rng, n, dtype, nulls, right, pool):
    vals = rng.choice(pool, n).astype(dtype)
    vals = vals[np.argsort(ao.total_keys(vals), kind="stable")]
    valid = rng.random(n) >= nulls
    if right:
        k = int((~valid).sum())
        valid = np.arange(n) >= k
    return vals, valid


@pytest.mark.parametrize("dtype", ["int8", "int32", "int64", "uint16", "uint64", "float32", "float64"])
def test_vectorised_rule_equals_the_cursors(dtype):
    rng = np.random.default_rng(7)
    if np.dtype(dtype).kind == "f":
        pool = np.array([-3.5, -1.0, -0.0, 0.0, 0.25, 1.0, 2.0, 7.0, np.inf, -np.inf, np.nan], dtype)
    elif np.dtype(dtype).kind == "u":
        pool = np.array([0, 1, 2, 5, 9, np.iinfo(dtype).max - 1, np.iinfo(dtype).max], dtype)
    else:
        info = np.iinfo(dtype)
        pool = np.array([info.min, info.min + 1, -2, 0, 1, 3, 4, info.max - 1, info.max], dtype)
    for trial in range(60):
        nl, nr = int(rng.integers(0, 40)), int(rng.integers(0, 25))
        lv, lvalid = sorted_side(rng, nl, dtype, 0.2, False, pool)
        rv, rvalid = sorted_side(rng, nr, dtype, 0.2, True, pool)
        left = [v if ok else None for v, ok in zip(lv, lvalid)]
        right = [v if ok else None for v, ok in zip(rv, rvalid)]
        for strategy in STRATS:
            for allow_eq in (False, True):
                for tol in (None, pool[int(rng.integers(0, len(pool)))]):
                    exp = ao.cursor_asof(left, right, strategy, allow_eq, tol)
                    idx, valid = ao.rule_asof((lv, lvalid), (rv, rvalid), strategy, allow_eq, tol)
                    got = [int(i) if ok else None for i, ok in zip(idx, valid)]
                    assert got == exp, (trial, strategy, allow_eq, tol)


def test_by_groups_equal_the_per_group_cursors():
    """two groups and a null group per side, groups sorted only within themselves, against cursor_asof_by"""
    rng = np.random.default_rng(11)
    for trial in range(300):
        dtype = ["int64", "float64"][trial % 2]
        nl, nr = int(rng.integers(0, 14)), int(rng.integers(0, 10))
        lg = rng.choice([0, 1, -1], nl)
        rg = rng.choice([0, 1, -1], nr)
        lv, rv = np.zeros(nl, dtype), np.zeros(nr, dtype)
        lvalid, rvalid = rng.random(nl) > 0.15, np.ones(nr, bool)
        for g in (0, 1, -1):
            li, ri = np.nonzero(lg == g)[0], np.nonzero(rg == g)[0]
            pool = np.array([-1.0, 0.0, 1.0, 2.0, 3.0] + ([np.nan] if dtype == "float64" else [])).astype(dtype)
            lv[li] = np.sort(rng.choice(pool, len(li)))
            rv[ri] = np.sort(rng.choice(pool, len(ri)))
            rvalid[ri[:int(rng.integers(0, len(ri) + 1))]] = False      # the right nulls of a group come first
        left = [v if ok else None for v, ok in zip(lv, lvalid)]
        right = [v if ok else None for v, ok in zip(rv, rvalid)]
        lb = [(None,) if g < 0 else (int(g),) for g in lg]
        rb = [(None,) if g < 0 else (int(g),) for g in rg]
        for strategy in STRATS:
            for allow_eq in (False, True):
                exp = ao.cursor_asof_by(left, right, lb, rb, strategy, allow_eq)
                idx, valid = ao.rule_asof((lv, lvalid), (rv, rvalid), strategy, allow_eq, None, lg, rg)
                got = [int(i) if ok else None for i, ok in zip(idx, valid)]
                assert got == exp, (trial, strategy, allow_eq)


# ------------------------------------------------------------------------------------------------ binding
def test_header_and_library_declare_the_entry_point():
    assert "bl_join_asof" in declared_symbols()
    import polars_b200 as plb
    assert hasattr(plb.lib(), "bl_join_asof")


class FakeLib:
    """stands in for the library: records bl_join_asof calls and returns BL_OK with an empty output"""

    def __init__(self):
        self.calls = []

    def bl_join_asof(self, lo, ro, lb, rb, n_by, strategy, allow_eq, tol, loc, out):
        self.calls.append({"n_by": n_by.value, "strategy": strategy.value, "allow_eq": allow_eq.value, "tol": tol is not None, "loc": loc.value,
                           "tol_dtype": tol._obj.dtype if tol is not None else None})
        return 0


@pytest.fixture
def fake(monkeypatch):
    import polars_b200 as plb
    f = FakeLib()
    monkeypatch.setattr(plb, "_lib", f)
    return plb, f


def test_binding_rejects_bad_arguments_before_any_call(fake):
    plb, f = fake
    l, r = np.array([1, 2], np.int64), np.array([1], np.int64)
    with pytest.raises(ValueError, match="unknown asof strategy"):
        plb.join_asof(l, r, strategy="closest")
    with pytest.raises(ValueError, match="together"):
        plb.join_asof(l, r, left_by=[l])
    with pytest.raises(ValueError, match="columns"):
        plb.join_asof(l, r, left_by=[l, l], right_by=[r])
    with pytest.raises(ValueError, match="not representable"):
        plb.join_asof(l, r, tolerance=1.5)
    with pytest.raises(ValueError, match="not representable"):
        plb.join_asof(l.astype(np.int8), r.astype(np.int8), tolerance=2**40)
    assert f.calls == []


def test_binding_widens_a_small_int_tolerance_to_int32(fake):
    """the reference extracts the tolerance of an 8/16-bit key as Int32 (asof/mod.rs:333-338, default.rs:128): 200 is a
    valid tolerance for an Int8 key"""
    plb, f = fake
    for dt in (np.int8, np.uint8, np.int16, np.uint16):
        plb.join_asof(np.array([1, 2], dt), np.array([1], dt), tolerance=200)
        assert f.calls[-1]["tol_dtype"] == 2
    plb.join_asof(np.array([1, 2], np.uint32), np.array([1], np.uint32), tolerance=200)
    assert f.calls[-1]["tol_dtype"] == 6


def test_binding_passes_the_options(fake):
    plb, f = fake
    l, r = np.array([1, 2], np.int64), np.array([1], np.int64)
    plb.join_asof(l, r, "nearest", tolerance=3, allow_exact_matches=False, left_by=[plb.StringColumn(["a", "b"])], right_by=[plb.StringColumn(["a"])],
                  location=plb.DEVICE)
    assert f.calls == [{"n_by": 1, "strategy": 2, "allow_eq": 0, "tol": True, "loc": plb.DEVICE, "tol_dtype": 3}]
    assert C.sizeof(plb.BlSortKey) == 24
