"""CPU tests (-m "not gpu") of multi-column sort: the plain-Python oracle against the reference's known answers
(tests/golden/sort_kats.json) and against numpy, the C ABI / plugin symbols, and the B2 matcher for Sort nodes."""
import json
import os
import types

import numpy as np
import pytest

import sort_oracle
from polars_b200 import engine
from test_cabi_cpu import declared_symbols
from test_engine_matcher import FakeTraverser, make

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NP = {"int8": np.int8, "int16": np.int16, "int32": np.int32, "int64": np.int64, "uint8": np.uint8, "uint16": np.uint16, "uint32": np.uint32,
      "uint64": np.uint64, "float32": np.float32, "float64": np.float64, "bool": np.bool_}


def sort_kats():
    with open(os.path.join(ROOT, "tests", "golden", "sort_kats.json")) as f:
        return json.load(f)["sort"]


def kat_columns(values_list, dtypes):
    """JSON lists with nulls -> (numpy columns with null slots zero-filled, validity arrays or None)"""
    cols, valids = [], []
    for vals, dt in zip(values_list, dtypes):
        valid = np.array([v is not None for v in vals], bool)
        fill = False if dt == "bool" else 0
        cols.append(np.array([fill if v is None else v for v in vals], dtype=NP[dt]))
        valids.append(None if valid.all() else valid)
    return cols, valids


def expected_payload_ok(got_vals, got_valid, expect):
    for i, e in enumerate(expect):
        null = got_valid is not None and not got_valid[i]
        if (e is None) != null or (e is not None and got_vals[i] != e):
            return False
    return True


@pytest.mark.parametrize("case", sort_kats(), ids=lambda c: c["cite"][-60:])
def test_oracle_matches_reference_kats(case):
    cols, valids = kat_columns(case["by"], case["dtypes"])
    if "expect_error" in case:
        with pytest.raises(ValueError, match=case["expect_error"]):
            sort_oracle.arg_sort(cols, valids, case["descending"], case["nulls_last"], case.get("limit"))
        return
    idx = sort_oracle.arg_sort(cols, valids, case["descending"], case["nulls_last"], case.get("limit"))
    if "expect_idx" in case:
        assert idx.tolist() == case["expect_idx"]
    for vals, dt, exp in zip(case.get("payload", []), case.get("payload_dtypes", []), case.get("expect_payload", [])):
        (pc,), (pv,) = kat_columns([vals], [dt])
        assert expected_payload_ok(pc[idx], None if pv is None else pv[idx], exp)


def random_columns(rng, n):
    f = rng.choice(np.array([0.0, -0.0, 1.5, -1.5, np.nan, np.inf, -np.inf, 2.0]), n)
    some = rng.random(n) < 0.2
    f[some] = rng.normal(size=int(some.sum()))
    cols = [rng.integers(-3, 3, n).astype(np.int8), f, rng.integers(0, 4, n).astype(np.uint64), rng.random(n) < 0.5,
            rng.choice(np.array([np.nan, -0.0, 0.0, 3.25], np.float32), n)]
    valids = [rng.random(n) > 0.2 if i % 2 == 0 else (rng.random(n) > 0.1) for i in range(len(cols))]
    return cols, valids


@pytest.mark.parametrize("seed", range(6))
def test_oracle_agrees_with_numpy(seed):
    rng = np.random.default_rng(seed)
    n = 300
    cols, valids = random_columns(rng, n)
    k = 1 + seed % len(cols)
    order = rng.permutation(len(cols))[:k]
    cs, vs = [cols[i] for i in order], [valids[i] if seed % 3 else None for i in order]
    desc = [bool(x) for x in rng.random(k) < 0.5]
    nl = [bool(x) for x in rng.random(k) < 0.5]
    limit = [None, 0, 1, 17, n, n + 5][seed % 6]
    a = sort_oracle.arg_sort(cs, vs, desc, nl, limit)
    b = sort_oracle.numpy_arg_sort(cs, vs, desc, nl, limit)
    assert np.array_equal(a, b)


def test_oracle_float_total_order():
    x = np.array([np.nan, 1.0, -0.0, 0.0, -np.inf, np.inf, np.nan, -1.0])
    assert sort_oracle.arg_sort([x]).tolist() == [4, 7, 2, 3, 1, 5, 0, 6]              # -0.0 == +0.0 keep row order, NaN last
    assert sort_oracle.arg_sort([x], descending=True).tolist() == [0, 6, 5, 1, 2, 3, 7, 4]
    assert np.array_equal(sort_oracle.numpy_arg_sort([x], descending=True), sort_oracle.arg_sort([x], descending=True))


def test_header_and_library_export_sort():
    import ctypes as C

    import polars_b200 as plb
    syms = declared_symbols()
    assert "bl_arg_sort" in syms and "bl_sort" in syms
    lib = plb.lib()
    for s in ("bl_arg_sort", "bl_sort", "_polars_plugin_bl_arg_sort", "_polars_plugin_field_bl_arg_sort"):
        assert hasattr(lib, s), s
    hdr = open(os.path.join(ROOT, "include", "polars_b200.h")).read()
    assert "BL_SORT_DESCENDING = 1" in hdr and "BL_SORT_NULLS_LAST = 2" in hdr
    assert plb.SORT_DESCENDING == 1 and plb.SORT_NULLS_LAST == 2
    # the field function needs no device: the output is the UInt32 permutation
    lib._polars_plugin_field_bl_arg_sort.restype = None
    from test_gpu_plugin_abi import ArrowSchema
    import pyarrow as pa
    fields = (ArrowSchema * 2)()
    pa.field("a", pa.int64())._export_to_c(C.addressof(fields[0]))
    pa.field("b", pa.float64())._export_to_c(C.addressof(fields[1]))
    out = ArrowSchema()
    lib._polars_plugin_field_bl_arg_sort(fields, C.c_size_t(2), C.byref(out), None, C.c_size_t(0))
    assert out.format == b"I" and out.name == b"a"


def test_python_flags_length_mismatch_raises():
    import polars_b200 as plb
    with pytest.raises(ValueError, match=r"the length of `descending` \(1\) does not match the length of `by` \(2\)"):
        plb._sort_flags(2, [True], False)
    assert list(plb._sort_flags(2, True, [False, True])) == [1, 3]


# ---------------------------------------------------------------------------- B2 matcher
def expr_ir(node, name):
    return types.SimpleNamespace(node=node, output_name=name)


class SchemaTraverser(FakeTraverser):
    """FakeTraverser + get_schema (visit.rs:127-131: the schema of the current root node, here the Sort)"""

    def __init__(self, nodes, exprs, root, schema):
        super().__init__(nodes, exprs, root)
        self.schema = schema

    def get_schema(self):
        assert type(self.nodes[self.cur]).__name__ == "Sort", "the schema is read on the Sort node"
        return dict(self.schema)


SCHEMA = {"a": "Int64", "b": "Float64", "c": "Int64", "s": "String"}


def sort_plan(by=("a",), nulls_last=(False,), descending=(False,), slc=None, input_kind="DataFrameScan", key_kind="Column", options=None,
              schema=None, with_schema=True):
    exprs = {0: make("Column", name="a"), 1: make("Column", name="b"), 2: make(key_kind, name="c"), 3: make("Column", name="s")}
    ids = {"a": 0, "b": 1, "c": 2, "s": 3}
    nodes = {30: make(input_kind, df=object(), projection=None, selection=None)}
    nodes[31] = make("Sort", input=30, by_column=[expr_ir(ids[b], b) for b in by],
                     sort_options=options if options is not None else (False, list(nulls_last), list(descending)), slice=slc)
    if not with_schema:
        return FakeTraverser(nodes, exprs, 31)
    return SchemaTraverser(nodes, exprs, 31, SCHEMA if schema is None else schema)


@pytest.mark.parametrize("kwargs", [dict(), dict(by=("a", "b"), nulls_last=(True,), descending=(False, True)), dict(slc=(0, 10, None)), dict(slc=(0, 0)),
                                    dict(by=("b", "a"), nulls_last=(True, False), descending=(True,)),
                                    # columns the device gather cannot take (String, Date, Boolean, Int8) are no reason to leave the node:
                                    # they are taken by Polars with the device permutation
                                    dict(schema={"a": "Int64", "s": "String", "d": "Date", "f": "Boolean", "g": "Int8"}),
                                    dict(by=("a", "b"), schema={"a": "Boolean", "b": "Int16", "s": "String"}),
                                    dict(by=("a",), schema={"a": "UInt8"})])
def test_sort_shapes_taken(kwargs):
    nt = sort_plan(**kwargs)
    engine.execute_with_b200(nt)
    assert callable(nt.udf) and nt.cur == 31


@pytest.mark.parametrize("kwargs", [dict(slc=(5, 10, None)), dict(slc=(-3, 3, None)), dict(slc=(0, 10, 12345)), dict(input_kind="Filter"),
                                    dict(by=("c",), key_kind="BinaryExpr"), dict(by=("a", "b"), descending=(True, False, True)),
                                    dict(options=(False, [False])), dict(by=()),
                                    # keys the device cannot order stay with Polars; so does a plan without a schema to check them
                                    dict(by=("s",)), dict(by=("a", "s")), dict(by=("a",), schema={"a": "Date"}),
                                    dict(by=("a",), schema={"a": "Datetime(time_unit='us', time_zone=None)"}), dict(by=("b",), schema={"a": "Int64"}),
                                    dict(with_schema=False)])
def test_sort_shapes_left_to_polars(kwargs):
    nt = sort_plan(**kwargs)
    engine.execute_with_b200(nt)
    assert nt.udf is None
    with pytest.raises(Exception):
        engine.execute_with_b200(sort_plan(**kwargs), raise_on_fail=True)


def test_sort_slice_limit():
    assert engine._sort_slice_limit(None) is None
    assert engine._sort_slice_limit((0, 7, None)) == 7
    assert engine._sort_slice_limit((0, 7)) == 7
