"""CPU tests (-m "not gpu") of sorting by string keys: the oracle against the reference's known answers
(tests/golden/string_sort_kats.json), a plain-Python dense rank against numpy, the binding's argument handling for
string keys, and the new C ABI symbols."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import sort_oracle
from test_cabi_cpu import declared_symbols

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def string_sort_kats():
    with open(os.path.join(ROOT, "tests", "golden", "string_sort_kats.json")) as f:
        return json.load(f)["sort"]


def as_bytes(values):
    return [None if v is None else (v.encode() if isinstance(v, str) else bytes(v)) for v in values]


def kat_frame(case):
    """-> {name: (column, valid | None, dtype)}: string columns as lists of bytes / None, others as numpy arrays"""
    out = {}
    for name, c in case["columns"].items():
        vals = c["values"]
        valid = np.array([v is not None for v in vals], bool)
        if c["dtype"] == "str":
            out[name] = (as_bytes(vals), None if valid.all() else valid, "str")
        else:
            out[name] = (np.array([0 if v is None else v for v in vals], dtype=c["dtype"]), None if valid.all() else valid, c["dtype"])
    return out


def oracle_key(col):
    """a bytes / None list -> what sort_oracle takes: the values (nulls as None) and no separate validity"""
    return list(col)


def check_sorted_frame(frame, idx, expect):
    for name, exp in expect.items():
        col, valid, dt = frame[name]
        got = [None if (valid is not None and not valid[i]) else col[i] for i in idx]
        if dt == "str":
            assert got == as_bytes(exp), (name, got, exp)
        else:
            assert [None if g is None else g.item() for g in got] == exp, (name, got, exp)


def dense_rank(values, descending=False):
    """RankMethod::Dense (polars-ops/src/series/ops/rank.rs:61-188) restated: walk the stable order of the non-null values
    and start a new rank wherever the value changes; 1-based, nulls stay null, descending ranks the largest value 1."""
    valid = [i for i, v in enumerate(values) if v is not None]
    order = sorted(valid, key=lambda i: values[i], reverse=descending)
    out = [None] * len(values)
    rank, prev = 0, object()
    for i in order:
        if values[i] != prev:
            rank, prev = rank + 1, values[i]
        out[i] = rank
    return out


def edge_strings():
    base = [b"", b"a", b"a\x00", b"a\x00\x00", b"ab", b"b", b"\x00", b"\x7f", b"\x80", b"\xff", b"\xff\xff", "é".encode(), "日本".encode(), "😀".encode()]
    base += [b"x" * k for k in range(0, 65)] + [b"x" * k + b"\x00" for k in (6, 7, 8, 13, 14, 15)] + [b"x" * k + b"\xff" for k in (6, 7, 8, 13, 14, 15)]
    return base


@pytest.mark.parametrize("case", string_sort_kats(), ids=lambda c: c["cite"][-60:])
def test_oracle_matches_reference_kats(case):
    frame = kat_frame(case)
    cols = [oracle_key(frame[b][0]) if frame[b][2] == "str" else frame[b][0] for b in case["by"]]
    valids = [None if frame[b][2] == "str" else frame[b][1] for b in case["by"]]
    idx = sort_oracle.arg_sort(cols, valids, case["descending"], case["nulls_last"])
    check_sorted_frame(frame, idx, case["expect"])


def test_oracle_byte_order():
    """unsigned lexicographic order, a proper prefix first (tot_cmp on &[u8], sort/mod.rs:405-499)"""
    vals = [b"ab", b"a\x00", b"", b"\xff", b"a", b"\x80", b"\x7f", b"a\x00\x00"]
    idx = sort_oracle.arg_sort([vals])
    assert [vals[i] for i in idx] == [b"", b"a", b"a\x00", b"a\x00\x00", b"ab", b"\x7f", b"\x80", b"\xff"]


def test_numpy_oracle_matches_plain_oracle_on_strings():
    rng = np.random.default_rng(3)
    pool = edge_strings()
    for n in (0, 1, 50, 300):
        vals = [pool[i] for i in rng.integers(0, len(pool), n)]
        valid = rng.random(n) > 0.2
        with_nulls = [v if ok else None for v, ok in zip(vals, valid)]
        obj = np.array(vals + [b""], dtype=object)[:n]
        for desc in (False, True):
            for nl in (False, True):
                exp = sort_oracle.arg_sort([with_nulls], None, desc, nl)
                assert np.array_equal(sort_oracle.numpy_arg_sort([obj], [valid], desc, nl), exp), (n, desc, nl)


def test_dense_rank_oracle_against_numpy():
    rng = np.random.default_rng(5)
    pool = edge_strings()
    for n in (0, 1, 10, 500):
        vals = [pool[i] for i in rng.integers(0, len(pool), n)]
        valid = rng.random(n) > 0.1
        with_nulls = [v if ok else None for v, ok in zip(vals, valid)]
        kept = np.array([v for v in with_nulls if v is not None] + [b""], dtype=object)[:-1]
        uniq, inv = np.unique(kept, return_inverse=True) if len(kept) else (kept, np.zeros(0, np.int64))
        exp = [None] * n
        for i, r in zip([i for i in range(n) if valid[i]], inv):
            exp[i] = int(r) + 1
        assert dense_rank(with_nulls) == exp
        exp_desc = [None if r is None else len(uniq) + 1 - r for r in exp]
        assert dense_rank(with_nulls, descending=True) == exp_desc
    assert dense_rank([None, None]) == [None, None]
    assert dense_rank([b"b", b"a", b"b", b""]) == [3, 2, 3, 1]


def test_header_and_library_declare_the_new_entry_points():
    syms = declared_symbols()
    assert "bl_string_rank" in syms and "bl_arg_sort_keys" in syms
    import polars_b200 as plb
    assert hasattr(plb.lib(), "bl_string_rank") and hasattr(plb.lib(), "bl_arg_sort_keys")
    # the binding's descriptor matches the header's struct: two pointers and two int32
    assert C.sizeof(plb.BlSortKey) == 24


class FakeLib:
    """stands in for the library: records the sort calls and returns BL_OK with an empty device output"""

    def __init__(self):
        self.calls = []

    def bl_arg_sort_keys(self, descs, n, limit, loc, out):
        keys = []
        for i in range(n.value):
            d = descs[i]
            keys.append({"column": bool(d.column), "strings": bool(d.strings), "n_chunks": d.n_chunks, "flags": d.flags,
                         "len": d.column[0].length if d.column else sum(d.strings[j].length for j in range(d.n_chunks))})
        self.calls.append(("bl_arg_sort_keys", keys, limit.value, loc.value))
        return 0

    def bl_arg_sort(self, arr, n, flags, limit, loc, out):
        self.calls.append(("bl_arg_sort", n.value))
        return 0


@pytest.fixture
def fake(monkeypatch):
    import polars_b200 as plb
    f = FakeLib()
    monkeypatch.setattr(plb, "_lib", f)
    return plb, f


def test_binding_routes_string_keys_to_arg_sort_keys(fake):
    plb, f = fake
    s = plb.StringColumn(["b", None, "a"])
    plb.arg_sort([np.array([3, 1, 2]), s], [True, False], True, limit=2, location=plb.DEVICE)
    (name, keys, limit, loc), = f.calls
    assert name == "bl_arg_sort_keys" and limit == 2 and loc == plb.DEVICE
    assert keys == [{"column": True, "strings": False, "n_chunks": 0, "flags": 3, "len": 3},
                    {"column": False, "strings": True, "n_chunks": 1, "flags": 2, "len": 3}]
    f.calls.clear()
    plb.arg_sort([[plb.StringColumn(["x"]), plb.StringColumn(["y", "z"])]], location=plb.DEVICE)      # one key in two chunks
    (_, keys, limit, _), = f.calls
    assert keys == [{"column": False, "strings": True, "n_chunks": 2, "flags": 0, "len": 3}] and limit == -1
    f.calls.clear()
    plb.arg_sort(s, descending=True, location=plb.DEVICE)                     # a single string key
    assert f.calls[0][1][0]["flags"] == 1
    f.calls.clear()
    plb.arg_sort([np.array([3, 1, 2])], location=plb.DEVICE)                  # numeric keys keep going through bl_arg_sort
    assert f.calls == [("bl_arg_sort", 1)]


def test_binding_rejects_flag_lengths_with_string_keys(fake):
    plb, f = fake
    s = plb.StringColumn(["b", "a"])
    with pytest.raises(ValueError, match="length of `descending`"):
        plb.arg_sort([s, np.array([1, 2])], descending=[True])
    with pytest.raises(ValueError, match="length of `nulls_last`"):
        plb.sort([s], [np.array([1, 2])], nulls_last=[True, False])
    assert f.calls == []
