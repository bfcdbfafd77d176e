"""CPU tests of unique: the oracle (tests/unique_oracle.py) against the reference's known answers
(tests/golden/unique_kats.json) and against brute-force definitions, its numpy form against the dict form, the Python
binding's argument errors, the declared bl_unique / bl_unique_mask symbols, the plugin schemas and the B2 matcher of
Distinct nodes.  tests/test_gpu_unique.py holds the device against this oracle."""
import ctypes as C
import itertools
import json
import math
import os

import numpy as np
import pytest

import unique_oracle as uo
from polars_b200 import engine

KATS = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "unique_kats.json")))
for _c in KATS:      # int_range cases: frame and expected are 0 .. n - 1
    if "int_range" in _c:
        _c["frame"] = {"x": list(range(_c["int_range"]))}
        _c["expected"] = {"x": list(range(_c["int_range"]))}
ROOT = os.path.dirname(os.path.dirname(__file__))


def kat_result(case):
    """the oracle's answer to a known-answer case: (column name -> values) for "unique", the bool list for "mask"."""
    frame = case["frame"]
    if case["op"] == "mask":
        return uo.masks([frame[c] for c in case["keys"]])[case["kind"]]
    subset = list(frame) if case["subset"] is None else case["subset"]
    ids = uo.arg_unique([frame[c] for c in subset], case["keep"])
    if case.get("slice"):
        off, ln = case["slice"]
        ids = ids[off:off + ln]
    return {c: [v[i] for i in ids] for c, v in frame.items()}


def same(a, b):
    return a is b or (a is None) == (b is None) and (a == b or (isinstance(a, float) and isinstance(b, float) and math.isnan(a) and math.isnan(b)))


def rows_of(cols: dict):
    names = list(cols)
    return [tuple(cols[c][i] for c in names) for i in range(len(cols[names[0]]))]


@pytest.mark.parametrize("case", KATS, ids=[f"{i}:{c['src'].rsplit('/', 1)[-1]}" for i, c in enumerate(KATS)])
def test_oracle_known_answers(case):
    got = kat_result(case)
    if case["op"] == "mask":
        assert got == case["expected"], case["src"]
        return
    exp = case["expected"]
    assert list(got) == list(exp)
    g, e = rows_of(got), rows_of(exp)
    if case["order"] == "multiset":
        key = lambda r: tuple(uo.canon(v) for v in r)
        g, e = sorted(g, key=key), sorted(e, key=key)
    assert len(g) == len(e) and all(all(same(x, y) for x, y in zip(rg, re)) for rg, re in zip(g, e)), case["src"]


def brute(cols):
    n = len(cols[0])
    k = [tuple(uo.canon(c[i]) for c in cols) for i in range(n)]
    return {"first": [all(k[j] != k[i] for j in range(i)) for i in range(n)],
            "last": [all(k[j] != k[i] for j in range(i + 1, n)) for i in range(n)],
            "unique": [sum(k[j] == k[i] for j in range(n)) == 1 for i in range(n)],
            "duplicated": [sum(k[j] == k[i] for j in range(n)) > 1 for i in range(n)]}


POOLS = {"int": [0, 1, -1, 2**63 - 1, None], "float": [0.0, -0.0, float("nan"), 1.5, None], "bool": [True, False, None], "str": ["", "a", "a\x00", None]}


def test_oracle_equals_brute_force_exhaustively():
    for pool in POOLS.values():
        for n in range(5):
            for vals in itertools.product(pool, repeat=n):
                assert uo.masks([list(vals)]) == brute([list(vals)])


def test_oracle_equals_brute_force_random():
    rng = np.random.default_rng(7)
    for _ in range(300):
        n = int(rng.integers(0, 40))
        kinds = rng.choice(list(POOLS), size=int(rng.integers(1, 4)))
        cols = [[POOLS[k][i] for i in rng.integers(0, len(POOLS[k]), n)] for k in kinds]
        m, b = uo.masks(cols), brute(cols)
        assert m == b
        for keep, kind in (("first", "first"), ("any", "first"), ("last", "last"), ("none", "unique")):
            assert uo.arg_unique(cols, keep) == [i for i in range(n) if b[kind][i]]


def test_numpy_oracle_equals_dict_oracle():
    rng = np.random.default_rng(11)
    for _ in range(100):
        n = int(rng.integers(0, 200))
        cols, np_cols = [], []
        for kind in rng.choice(["i64", "f32", "f64", "bool", "str", "u8"], size=int(rng.integers(1, 4))):
            valid = rng.random(n) > 0.2 if rng.random() < 0.5 else None
            if kind == "str":
                vals = [["", "x", "x\x00", "y"][i] for i in rng.integers(0, 4, n)]
            elif kind == "bool":
                vals = rng.random(n) < 0.5
            elif kind in ("f32", "f64"):
                vals = rng.choice(np.array([0.0, -0.0, np.nan, 1.0, -np.nan], dtype=np.float32 if kind == "f32" else np.float64), n)
            elif kind == "u8":
                vals = rng.integers(0, 3, n).astype(np.uint8)
            else:
                vals = rng.integers(-2, 2, n).astype(np.int64)
            np_cols.append((vals, valid))
            cols.append([None if valid is not None and not valid[i] else (vals[i] if kind == "str" else vals[i].item()) for i in range(n)])
        m, nm = uo.masks(cols), uo.np_masks(np_cols)
        for kind in uo.KINDS:
            assert list(nm[kind]) == m[kind], kind
        for keep in uo.KEEP:
            assert list(uo.np_arg_unique(np_cols, keep)) == uo.arg_unique(cols, keep)


def test_binding_argument_errors():
    import polars_b200 as plb
    a = np.arange(3)
    for fn in (lambda: plb.arg_unique(a, keep="fist"), lambda: plb.unique([a], keep="fist")):
        with pytest.raises(ValueError, match=r"`keep` must be one of \{'first', 'last', 'any', 'none'\}, got fist"):
            fn()


def test_declared_symbols():
    import polars_b200 as plb
    assert hasattr(plb.lib(), "bl_unique") and hasattr(plb.lib(), "bl_unique_mask")
    header = open(os.path.join(ROOT, "include", "polars_b200.h")).read()
    assert "bl_status bl_unique(const bl_sort_key* subset, int32_t n_subset, int32_t keep, int32_t out_location, bl_column* out_idx);" in header
    assert "bl_status bl_unique_mask(const bl_sort_key* keys, int32_t n_keys, int32_t kind, int32_t out_location, bl_column* out_mask);" in header
    assert "enum { BL_UNIQUE_FIRST = 0, BL_UNIQUE_LAST = 1, BL_UNIQUE_ANY = 2, BL_UNIQUE_NONE = 3 };" in header
    assert "enum { BL_DISTINCT_FIRST = 0, BL_DISTINCT_LAST = 1, BL_DISTINCT_UNIQUE = 2, BL_DISTINCT_DUPLICATED = 3 };" in header
    rs = open(os.path.join(ROOT, "integration", "polars_b200_sys.rs")).read()
    assert "pub fn bl_unique(" in rs and "pub fn bl_unique_mask(" in rs and "pub const BL_DISTINCT_DUPLICATED: i32 = 3;" in rs
    assert plb.UNIQUE_KEEP == {"first": 0, "last": 1, "any": 2, "none": 3}


class ArrowSchema(C.Structure):
    _fields_ = [("format", C.c_char_p), ("name", C.c_char_p), ("metadata", C.c_char_p), ("flags", C.c_int64), ("n_children", C.c_int64),
                ("children", C.c_void_p), ("dictionary", C.c_void_p), ("release", C.c_void_p), ("private_data", C.c_void_p)]


@pytest.mark.parametrize("name,fmt", [("arg_unique", b"I"), ("is_unique", b"b"), ("is_duplicated", b"b"), ("is_first_distinct", b"b"),
                                      ("is_last_distinct", b"b")])
def test_plugin_entries_and_schemas(name, fmt):
    import polars_b200 as plb
    L = plb.lib()
    assert hasattr(L, f"_polars_plugin_bl_{name}")
    fn = getattr(L, f"_polars_plugin_field_bl_{name}")
    for fmt_in in (b"c", b"l", b"g", b"b", b"I"):
        for n in (1, 2):
            fields = (ArrowSchema * 2)()
            fields[0].format, fields[0].name = fmt_in, b"x"
            fields[1].format, fields[1].name = b"l", b"y"
            out = ArrowSchema()
            fn(fields, C.c_size_t(n), C.byref(out), None, C.c_size_t(0))
            assert out.format == fmt, (name, fmt_in, out.format)
            assert out.name == b"x"
            C.CFUNCTYPE(None, C.POINTER(ArrowSchema))(out.release)(C.byref(out))


# ---- B2: Distinct(input=DataFrameScan, options=(keep, subset, maintain_order, slice)) (visitor/nodes.rs:678-695)
def make(_kind, **fields):
    obj = type(_kind, (), {})()
    for k, v in fields.items():
        setattr(obj, k, v)
    return obj


class FakeTraverser:
    def __init__(self, nodes, root, schema):
        self.nodes, self.cur, self.udf, self.schema = nodes, root, None, schema

    def view_current_node(self):
        return self.nodes[self.cur]

    def set_node(self, n):
        self.cur = n

    def get_node(self):
        return self.cur

    def get_schema(self):
        return self.schema

    def set_udf(self, fn):
        self.udf = fn


SCHEMA = {"a": "Int64", "f": "Float64", "b": "Boolean", "s": "String", "t": "Int8"}


def distinct_plan(options, schema=SCHEMA, input_kind="DataFrameScan"):
    scan = make(input_kind, df=object(), projection=None, selection=None, input=0)
    return FakeTraverser({10: scan, 11: make("Distinct", input=10, options=options)}, 11, schema)


@pytest.mark.parametrize("options", [
    ("first", ["a"], True, None), ("last", ["a", "b"], True, None), ("any", ["f", "t"], False, None), ("none", ["b"], False, None),
    ("first", None, True, None), ("last", ["a"], True, (3, 4)), ("any", ["a"], True, (-2, 10)),
])
def test_distinct_is_taken(options):
    schema = SCHEMA if options[1] is not None else {k: v for k, v in SCHEMA.items() if k != "s"}
    nt = distinct_plan(options, schema)
    engine.execute_with_b200(nt, raise_on_fail=True)
    assert callable(nt.udf)
    assert nt.cur == 11          # the traverser is back on the Distinct node


@pytest.mark.parametrize("options,schema,input_kind", [
    (("first", ["s"], True, None), SCHEMA, "DataFrameScan"),              # String subset
    (("first", ["a", "s"], True, None), SCHEMA, "DataFrameScan"),
    (("first", None, True, None), SCHEMA, "DataFrameScan"),               # every column, one of them String
    (("first", ["missing"], True, None), SCHEMA, "DataFrameScan"),
    (("First", ["a"], True, None), SCHEMA, "DataFrameScan"),              # not a keep name the visitor produces
    (("first", ["a"], True, None, None), SCHEMA, "DataFrameScan"),        # unknown option shape
    (("first", "a", True, None), SCHEMA, "DataFrameScan"),
    (("first", ["a"], "yes", None), SCHEMA, "DataFrameScan"),
    (("first", ["a"], True, (0, -1)), SCHEMA, "DataFrameScan"),
    (("first", ["a"], True, (0, 1, 2)), SCHEMA, "DataFrameScan"),
    (("first", ["a"], True, None), {"a": "Datetime(time_unit='us', time_zone=None)"}, "DataFrameScan"),
    (("first", ["a"], True, None), SCHEMA, "Filter"),                     # not over a DataFrameScan
])
def test_distinct_left_to_polars(options, schema, input_kind):
    nt = distinct_plan(options, schema, input_kind)
    engine.execute_with_b200(nt)
    assert nt.udf is None
    with pytest.raises(Exception):
        engine.execute_with_b200(nt, raise_on_fail=True)


@pytest.mark.parametrize("slc", [None, (0, 0), (1, 2), (3, 10), (-2, 1), (-10, 3), (7, 1)])
def test_distinct_slice_matches_the_reference(slc):
    ids = np.arange(5)
    got = list(engine._slice_ids(ids, slc))
    if slc is None:
        assert got == list(ids)
        return
    off, ln = slc
    start = min(max(off + 5 if off < 0 else off, 0), 5)              # slice_offsets, polars-core/src/utils/mod.rs:340-357
    stop = min(max((off + 5 if off < 0 else off) + ln, 0), 5)
    assert got == list(ids[start:stop])
