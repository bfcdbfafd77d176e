"""CPU checks of rank (bl_rank): the oracle against the reference's known answers and against the definitions by brute
force, the numpy restatement against the oracle, the Python binding's argument errors and the plugin entries' symbols and
schemas.  No GPU needed."""
import itertools
import json
import os

import numpy as np
import pytest

import rank_oracle as ro

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KATS = json.load(open(os.path.join(ROOT, "tests", "golden", "rank_kats.json")))


def same(a, b):
    return all((x is None and y is None) or (x is not None and y is not None and x == y) for x, y in zip(a, b)) and len(a) == len(b)


@pytest.mark.parametrize("case", KATS, ids=[c["src"].split("/")[-1] for c in KATS])
def test_oracle_known_answers(case):
    vals = [v.encode() if isinstance(v, str) else v for v in case["values"]]
    got = ro.rank(vals, case["method"], case["descending"], case["parts"], seed=1)
    if case["expected"] is not None:
        assert same(got, case["expected"]), (got, case["expected"])
        return
    for rows, total in case["random_runs"]:
        assert sum(got[r] for r in rows) == total
        assert len({got[r] for r in rows}) == len(rows)


ALPHABET = [None, -1.5, -0.0, 0.0, 2.0, float("nan"), float("inf")]


@pytest.mark.parametrize("descending", [False, True])
def test_oracle_equals_brute_force_exhaustively(descending):
    # every sequence of length <= 4 over an alphabet with a null, both zeros, NaN and inf
    for n in range(0, 5):
        for vals in itertools.product(ALPHABET, repeat=n):
            vals = list(vals)
            for m in ("average", "min", "max", "dense"):
                assert same(ro.rank(vals, m, descending), ro.brute(vals, m, descending)), (vals, m, descending)


def test_oracle_equals_brute_force_random():
    rng = np.random.default_rng(5)
    for _ in range(300):
        n = int(rng.integers(0, 40))
        kind = rng.integers(0, 3)
        if kind == 0:
            vals = [int(v) for v in rng.integers(-3, 4, n)]
        elif kind == 1:
            vals = [float(v) for v in rng.choice([-1.0, -0.0, 0.0, 1.0, np.nan, np.inf, -np.inf], n)]
        else:
            vals = [bytes(rng.integers(0, 3, rng.integers(0, 3)).astype(np.uint8)) for _ in range(n)]
        vals = [None if rng.random() < 0.2 else v for v in vals]
        desc = bool(rng.integers(0, 2))
        for m in ("average", "min", "max", "dense"):
            assert same(ro.rank(vals, m, desc), ro.brute(vals, m, desc))
        # ordinal / random: a permutation of each run's [s + 1, e]
        mn, mx = ro.rank(vals, "min", desc), ro.rank(vals, "max", desc)
        for m in ("ordinal", "random"):
            got = ro.rank(vals, m, desc, seed=int(rng.integers(0, 2**63)))
            runs = {}
            for i, v in enumerate(vals):
                if v is not None:
                    runs.setdefault((mn[i], mx[i]), []).append(got[i])
            for (s1, e), rk in runs.items():
                assert sorted(rk) == list(range(s1, e + 1))


def test_partitions_and_order_by():
    vals = [3, 1, 3, None, 1, 3, 2, 3]
    parts = ["a", "b", "a", "a", "b", None, None, "a"]
    order = [5, 0, 2, 9, 1, 4, 3, 1]
    assert ro.rank(vals, "dense", parts=parts) == [1, 1, 1, None, 1, 2, 1, 1]
    # ordinal ties of partition "a" (rows 0, 2, 7 hold 3) by the order_by positions 5, 2, 1
    pos = ro.order_ranks(order)
    assert ro.rank(vals, "ordinal", parts=parts, order=pos) == [3, 1, 2, None, 2, 2, 1, 1]
    assert ro.rank(vals, "ordinal", parts=parts) == [1, 1, 2, None, 2, 2, 1, 3]
    assert ro.order_ranks([2, None, 1], descending=True, nulls_last=True) == [0, 2, 1]
    assert ro.order_ranks([2, None, 1]) == [2, 0, 1]


@pytest.mark.parametrize("method", ro.METHODS)
def test_numpy_restatement_equals_oracle(method):
    rng = np.random.default_rng(7)
    for dt in ("int64", "uint64", "float64", "int8", "bool"):
        for _ in range(20):
            n = int(rng.integers(0, 60))
            if dt == "float64":
                x = rng.choice(np.array([-2.0, -0.0, 0.0, 1.0, np.nan, -np.nan, np.inf]), n)
            elif dt == "bool":
                x = rng.random(n) < 0.5
            else:
                info = np.iinfo(dt)
                x = rng.choice(np.array([info.min, info.min + 1, 0, 1, info.max], dtype=dt), n)
            valid = rng.random(n) >= 0.25
            g = rng.integers(0, 3, n)
            desc = bool(rng.integers(0, 2))
            seed = int(rng.integers(0, 2**64, dtype=np.uint64))
            tie = np.array([ro.random_key(r, seed) for r in range(n)], np.int64) if method == "random" else None
            got, _ = ro.rank_np(x, valid, method, desc, g, tie)
            vals = [None if not ok else (float(v) if dt == "float64" else (bool(v) if dt == "bool" else int(v))) for v, ok in zip(x, valid)]
            exp = ro.rank(vals, method, desc, [int(k) for k in g], seed=seed)
            assert [0 if e is None else e for e in exp] == got.tolist(), (dt, method, desc)


def test_random_key_is_a_bijection_sample():
    keys = {ro.random_key(r, 0x1234_5678_9ABC_DEF0) for r in range(1 << 16)}
    assert len(keys) == 1 << 16


def test_binding_argument_errors():
    import polars_b200 as pb
    x = np.array([1, 2, 3])
    with pytest.raises(ValueError, match="unknown rank method"):
        pb.rank([(x, {"method": "first"})])
    with pytest.raises(ValueError, match="takes no option"):
        pb.rank([(x, {"window_size": 3})])
    with pytest.raises(ValueError, match="seed"):
        pb.rank([(x, {"method": "random", "seed": -1})])
    with pytest.raises(ValueError, match="seed"):
        pb.rank([(x, {"method": "random", "seed": 1.5})])
    with pytest.raises(ValueError, match="seed"):
        pb.rank_column(x, "random", seed=2**64)
    with pytest.raises(ValueError, match="needs a value column"):
        pb.rank([(None, {})])
    with pytest.raises(ValueError, match="at least one operation"):
        pb.rank([])
    with pytest.raises(ValueError, match=r"\(column, options\)"):
        pb.rank([("average", x, {})])
    with pytest.raises(ValueError, match="one order_by column"):
        pb.rank([(x, {"method": "ordinal"})], order_by=[x, x])


def test_plugin_entries_are_exported():
    import ctypes as C
    import polars_b200 as pb
    try:
        L = pb.lib()
    except ImportError:
        pytest.skip("the library is not built")

    class ArrowSchema(C.Structure):
        _fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64), ("n_children", C.c_int64),
                    ("children", C.c_void_p), ("dictionary", C.c_void_p), ("release", C.c_void_p), ("private_data", C.c_void_p)]
    for m in ro.METHODS:
        assert hasattr(L, f"_polars_plugin_bl_rank_{m}")
        fn = getattr(L, f"_polars_plugin_field_bl_rank_{m}")
        for fmt_in in (b"c", b"l", b"g", b"b"):
            fields = (ArrowSchema * 2)()
            fields[0].format, fields[0].name = fmt_in, b"x"
            fields[1].format, fields[1].name = b"l", b"g"
            out = ArrowSchema()
            fn(fields, C.c_size_t(2), C.byref(out), None, C.c_size_t(0))
            assert out.format == (b"g" if m == "average" else b"I"), (m, fmt_in, out.format)
            C.CFUNCTYPE(None, C.POINTER(ArrowSchema))(out.release)(C.byref(out))
