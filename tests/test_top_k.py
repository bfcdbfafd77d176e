"""CPU tests of top-k selection: the checker (the first k rows of sort_oracle's stable order) against the reference's known
answers (tests/golden/top_k_kats.json) and against brute force, the Python binding's argument errors, and the declared
bl_top_k symbol, the plugin entries and their schemas.  tests/test_gpu_top_k.py holds the device against this checker."""
import ctypes as C
import itertools
import json
import os

import numpy as np
import pytest

import sort_oracle

KATS = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "top_k_kats.json")))


def checker_ids(cols, valids, k, descending=False, nulls_last=False) -> np.ndarray:
    """bl_top_k's answer: the first k rows of the stable order, in ascending row order"""
    return np.sort(sort_oracle.arg_sort(cols, valids, descending, nulls_last, limit=k)).astype(np.uint32)


def kat_plan(case):
    """-> (key names, descending, nulls_last, payload names) of a known-answer case, as the bindings run it"""
    op = case["op"]
    if op in ("top_k", "bottom_k"):
        return [case["col"]], op == "top_k", True, [case["col"]]
    if op == "sort":
        return case["by"], case["descending"], case["nulls_last"], list(case["frame"])
    rev = case["reverse"]
    rev = [rev] * len(case["by"]) if isinstance(rev, bool) else rev
    return case["by"], [(not r) if op == "top_k_by" else r for r in rev], True, case["cols"]


def kat_columns(case, name):
    vals = case["frame"][name]
    return vals, [v is not None for v in vals]


def kat_matches(case, got: dict) -> bool:
    """got: payload name -> values (None = null) in output order"""
    for name, exp in case["expected"].items():
        g = list(got[name])
        if case["order"] == "pinned":
            if g != exp:
                return False
        elif sorted(g, key=lambda v: (v is None, v if v is not None else 0)) != sorted(exp, key=lambda v: (v is None, v if v is not None else 0)):
            return False
    return True


@pytest.mark.parametrize("case", KATS, ids=[f"{i}-{c['op']}" for i, c in enumerate(KATS)])
def test_checker_known_answers(case):
    keys, desc, nl, payload = kat_plan(case)
    cols = [kat_columns(case, k)[0] for k in keys]
    valids = [kat_columns(case, k)[1] for k in keys]
    k = case["k"]
    ids = checker_ids(cols, valids, k, desc, nl)
    assert len(ids) == min(k, len(cols[0]))
    order = sort_oracle.arg_sort(cols, valids, desc, nl, limit=k)      # the sorted form: arg_sort with the limit
    assert np.array_equal(np.sort(order), ids)
    got = {p: [case["frame"][p][i] for i in order] for p in payload}
    assert kat_matches(case, got), (case["src"], got)


def brute_force_ids(cols, valids, k, desc, nl):
    """every row's full key as a tuple, sorted with the row index last: the first k rows"""
    n = len(cols[0])

    def key(r):
        t = []
        for c, v, d, l in zip(cols, valids, desc, nl):
            null = not v[r]
            x = c[r]
            if not null and isinstance(x, float) and np.isnan(x):
                x = float("inf")
                nan = 1
            else:
                nan = 0
            x = 0 if null else (x + 0.0 if isinstance(x, float) else x)
            t += [null if l else not null, 0 if null else (-nan if d else nan), 0 if null else (-x if d else x)]
        return tuple(t) + (r,)
    return np.sort(np.array(sorted(range(n), key=key)[:k], dtype=np.int64)).astype(np.uint32)


def test_checker_equals_brute_force_exhaustively():
    rng = np.random.default_rng(7)
    vals = [0.0, -0.0, 1.5, np.nan, -np.inf]
    for n in range(0, 6):
        for _ in range(20):
            c0 = [vals[i] for i in rng.integers(0, len(vals), n)]
            c1 = [int(x) for x in rng.integers(-2, 3, n)]
            v0, v1 = list(rng.random(n) < 0.7), list(rng.random(n) < 0.8)
            for desc, nl in itertools.product([(False, True), (True, False)], [(True, False), (False, True)]):
                for k in range(0, n + 2):
                    assert np.array_equal(checker_ids([c0, c1], [v0, v1], k, list(desc), list(nl)),
                                          brute_force_ids([c0, c1], [v0, v1], k, desc, nl))


def test_checker_equals_brute_force_random():
    rng = np.random.default_rng(11)
    for trial in range(30):
        n = int(rng.integers(1, 200))
        cols = [[int(x) for x in rng.integers(-5, 5, n)], [float(x) for x in rng.normal(size=n).round(1)]]
        valids = [list(rng.random(n) < 0.9), list(rng.random(n) < 0.9)]
        desc, nl = [bool(x) for x in rng.random(2) < 0.5], [bool(x) for x in rng.random(2) < 0.5]
        k = int(rng.integers(0, n + 3))
        assert np.array_equal(checker_ids(cols, valids, k, desc, nl), brute_force_ids(cols, valids, k, desc, nl))
        # the numpy restatement used at large sizes agrees
        assert np.array_equal(np.sort(sort_oracle.numpy_arg_sort([np.array(c) for c in cols], [np.array(v) for v in valids], desc, nl, limit=k)),
                              checker_ids(cols, valids, k, desc, nl))


def test_binding_argument_errors():
    import polars_b200 as plb
    a = np.arange(3)
    with pytest.raises(ValueError, match=r"the length of `reverse` \(2\) does not match the length of `by` \(1\)"):
        plb.top_k_by([a], a, 2, reverse=[True, False])
    with pytest.raises(ValueError, match=r"the length of `reverse` \(2\) does not match the length of `by` \(1\)"):
        plb.bottom_k_by([a], [a], 2, reverse=[True, False])
    with pytest.raises(ValueError, match=r"the length of `reverse` \(1\) does not match the length of `by` \(2\)"):
        plb.top_k_by([a], [a, a], 1, reverse=[True])
    for fn in (lambda: plb.top_k(a, -1), lambda: plb.bottom_k(a, -1), lambda: plb.top_k_by([a], a, -1), lambda: plb.arg_top_k(a, -1)):
        with pytest.raises(ValueError, match="non-negative"):
            fn()


class ArrowSchema(C.Structure):
    _fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64), ("n_children", C.c_int64),
                ("children", C.c_void_p), ("dictionary", C.c_void_p), ("release", C.c_void_p), ("private_data", C.c_void_p)]


def test_declared_symbol():
    import polars_b200 as plb
    assert hasattr(plb.lib(), "bl_top_k")
    header = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "include", "polars_b200.h")).read()
    assert "bl_status bl_top_k(const bl_sort_key* by, int32_t n_by, int64_t k, int32_t out_location, bl_column* out_idx);" in header
    rs = open(os.path.join(os.path.dirname(os.path.dirname(__file__)), "integration", "polars_b200_sys.rs")).read()
    assert "pub fn bl_top_k(" in rs


@pytest.mark.parametrize("name", ["top_k_idx", "bottom_k_idx"])
def test_plugin_entries_and_schemas(name):
    import polars_b200 as plb
    L = plb.lib()
    assert hasattr(L, f"_polars_plugin_bl_{name}")
    fn = getattr(L, f"_polars_plugin_field_bl_{name}")
    for fmt_in in (b"c", b"l", b"g", b"b", b"u"):
        fields = (ArrowSchema * 2)()
        fields[0].format, fields[0].name = fmt_in, b"x"
        fields[1].format, fields[1].name = b"l", b"y"
        out = ArrowSchema()
        fn(fields, C.c_size_t(2), C.byref(out), None, C.c_size_t(0))
        assert out.format == b"I", (name, fmt_in, out.format)      # UInt32 row ids
        assert out.name == b"x"
        C.CFUNCTYPE(None, C.POINTER(ArrowSchema))(out.release)(C.byref(out))
