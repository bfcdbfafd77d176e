"""polars_b200 — host-side Python binding of libpolars_b200.so (the C ABI in include/polars_b200.h).

This module is plumbing: ctypes structs, numpy <-> bl_column marshalling and error translation.
All compute happens in the CUDA library; if the library (or a GPU) is missing every call raises —
there is no CPU fallback and this package never imports oracle/.
"""
from __future__ import annotations

import ctypes as C
import datetime as _dt
import json
import os
import re
from typing import Sequence

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_lib", "libpolars_b200.so")

HOST, DEVICE = 0, 1
IDX_NULL = 0xFFFFFFFF

DTYPES = {np.dtype("int8"): 0, np.dtype("int16"): 1, np.dtype("int32"): 2, np.dtype("int64"): 3,
          np.dtype("uint8"): 4, np.dtype("uint16"): 5, np.dtype("uint32"): 6, np.dtype("uint64"): 7,
          np.dtype("float32"): 8, np.dtype("float64"): 9, np.dtype("bool"): 10}
NP_OF = {v: k for k, v in DTYPES.items()}
BOOL = 10
OPS = {"add": 0, "sub": 1, "mul": 2, "floordiv": 3, "mod": 4, "truediv": 5}
CMPS = {"eq": 0, "ne": 1, "lt": 2, "le": 3, "gt": 4, "ge": 5}
AGGS = {"sum": 0, "mean": 1, "min": 2, "max": 3, "count": 4, "len": 5, "first": 6, "last": 7, "var": 8 | (1 << 16), "std": 9 | (1 << 16), "n_unique": 10,
        "median": 11}
QUANTILE = 12
QUANTILE_METHODS = {"nearest": 0, "lower": 1, "higher": 2, "midpoint": 3, "linear": 4, "equiprobable": 5}


def _agg_kind(kind: str) -> int:
    """"var" / "std" default to ddof = 1 (Polars); "var:0", "std:2" ... carry an explicit ddof (BL_AGG_WITH_DDOF).
    "quantile:<q>[:<method>]" is BL_AGG_QUANTILE; its parameters come from _agg_param."""
    name, _, dd = kind.partition(":")
    if name == "quantile":
        return QUANTILE
    return (AGGS[name] & 0xFFFF) | (int(dd) << 16) if dd else AGGS[name]


def _agg_param(kind: str) -> tuple[float, int] | None:
    """"quantile:<q>" (method nearest, Polars' default) or "quantile:<q>:<method>" -> (q, BL_QUANTILE_*); None for other kinds."""
    name, _, rest = kind.partition(":")
    if name != "quantile":
        return None
    q, _, method = rest.partition(":")
    if not q:
        raise ValueError(f"{kind!r}: a quantile is written 'quantile:<q>' or 'quantile:<q>:<method>'")
    method = method or "nearest"
    if method not in QUANTILE_METHODS:
        raise ValueError(f"{kind!r}: unknown quantile method {method!r} (one of {', '.join(QUANTILE_METHODS)})")
    return float(q), QUANTILE_METHODS[method]
JOINS = {"inner": 0, "left": 1, "semi": 2, "anti": 3, "full": 4}
ORDERS = {"none": 0, "left": 1, "left_right": 2, "right": 3, "right_left": 4}
STATUS = {1: "INVALID", 2: "CUDA", 3: "OOM", 4: "UNSUPPORTED", 5: "DTYPE", 6: "BOUNDS"}


class BlColumn(C.Structure):
    _fields_ = [("dtype", C.c_int32), ("location", C.c_int32), ("length", C.c_int64), ("offset", C.c_int64),
                ("null_count", C.c_int64), ("values", C.c_void_p), ("validity", C.c_void_p), ("owner", C.c_void_p)]


class BlStringColumn(C.Structure):
    _fields_ = [("location", C.c_int32), ("reserved", C.c_int32), ("length", C.c_int64), ("offset", C.c_int64), ("null_count", C.c_int64),
                ("offsets", C.c_void_p), ("data", C.c_void_p), ("validity", C.c_void_p), ("owner", C.c_void_p)]


class BlAgg(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n_chunks", C.c_int32), ("values", C.POINTER(BlColumn))]


class BlAggParam(C.Structure):
    _fields_ = [("quantile", C.c_double), ("method", C.c_int32), ("reserved", C.c_int32)]


class BlSortKey(C.Structure):
    _fields_ = [("column", C.POINTER(BlColumn)), ("strings", C.POINTER(BlStringColumn)), ("n_chunks", C.c_int32), ("flags", C.c_int32)]


class B200Error(RuntimeError):
    def __init__(self, status: int, msg: str):
        super().__init__(f"[{STATUS.get(status, status)}] {msg}")
        self.status = status


class ComputeError(B200Error):
    """dtype mismatches etc. — the reference raises ComputeError (join/mod.rs:231-241)."""


class OutOfBoundsError(B200Error):
    pass


_lib = None


def lib() -> C.CDLL:
    """Loads libpolars_b200.so.  Fails loudly when it has not been built (python -m polars_b200.build)."""
    global _lib, _SO
    if _lib is None:
        _SO = os.environ.get("POLARS_B200_LIB", _SO)      # another build of the library
        if not os.path.exists(_SO):
            raise ImportError(f"{_SO} is missing: build it with `python -m polars_b200.build` (nvcc, sm_90a). "
                              "polars_b200 has no CPU fallback.")
        L = C.CDLL(_SO)
        L.bl_last_error.restype = C.c_char_p
        L.bl_profile_json.restype = C.c_int64
        L.bl_launch_count.restype = C.c_int64
        L.bl_stream.restype = C.c_void_p
        for name in ("bl_column_free", "bl_free_pinned", "bl_dev_free", "bl_profile_enable", "bl_profile_reset", "bl_shutdown",
                     "bl_groupby_reset", "bl_groupby_destroy"):
            getattr(L, name).restype = None
        _lib = L
    return _lib


def _check(st: int):
    if st != 0:
        msg = lib().bl_last_error().decode("utf-8", "replace")
        if st == 5:
            raise ComputeError(st, msg)
        if st == 6:
            raise OutOfBoundsError(st, msg)
        raise B200Error(st, msg)


def init(device: int = -1):
    _check(lib().bl_init(C.c_int32(device)))


def device_info() -> dict:
    sm, l2, tot, free = C.c_int32(), C.c_int64(), C.c_int64(), C.c_int64()
    _check(lib().bl_device_info(C.byref(sm), C.byref(l2), C.byref(tot), C.byref(free)))
    return {"sm_count": sm.value, "l2_bytes": l2.value, "hbm_total": tot.value, "hbm_free": free.value}


def set_deterministic(on: bool = True):
    """Bit-stable group_by aggregation in the reference's own order (bl_set_deterministic)."""
    lib().bl_set_deterministic.restype = None
    lib().bl_set_deterministic(C.c_int32(int(on)))


def loaded_library() -> str:
    """Path of the shared library this process has loaded (after the first call into it)."""
    lib()
    return _SO


def sync():
    _check(lib().bl_sync())


def stream() -> int:
    return int(lib().bl_stream() or 0)


def profile_enable(on: bool):
    lib().bl_profile_enable(C.c_int32(int(on)))


def profile_reset():
    lib().bl_profile_reset()


def profile() -> dict:
    n = lib().bl_profile_json(None, C.c_int64(0))
    buf = C.create_string_buffer(int(n) + 16)
    lib().bl_profile_json(buf, C.c_int64(len(buf)))
    return json.loads(buf.value.decode() or "{}")


def launch_count() -> int:
    return int(lib().bl_launch_count())


# ---------------------------------------------------------------------------------- pinned memory
def pinned_empty(n: int, dtype) -> np.ndarray:
    """numpy array backed by library pinned host memory (DMA-able without staging).
    The buffer is returned to the library's pinned cache when the array is garbage collected."""
    dt = np.dtype(dtype)
    nbytes = max(int(n) * dt.itemsize, 1)
    p = C.c_void_p()
    _check(lib().bl_alloc_pinned(C.c_size_t(nbytes), C.byref(p)))
    buf = (C.c_char * nbytes).from_address(p.value)
    arr = np.frombuffer(buf, dtype=dt, count=int(n))
    import weakref
    weakref.finalize(buf, lib().bl_free_pinned, C.c_void_p(p.value))
    return arr


def to_pinned(a: np.ndarray) -> np.ndarray:
    out = pinned_empty(a.size, a.dtype)
    out[:] = a
    return out


# ---------------------------------------------------------------------------------- columns
def pack_bits(valid: np.ndarray) -> np.ndarray:
    return np.packbits(np.asarray(valid, dtype=np.bool_), bitorder="little")


def unpack_bits(buf: np.ndarray, n: int) -> np.ndarray:
    return np.unpackbits(buf, count=n, bitorder="little").astype(np.bool_)


class Column:
    """A caller-owned host (numpy) or device column view passed INTO the library.

    values: numpy array (host) or an int device pointer; valid: bool array / packed bitmap (host) or
    device pointer to a bitmap.  `offset` exercises Arrow slicing semantics."""

    def __init__(self, values, valid=None, *, dtype=None, length=None, offset: int = 0, location: int = HOST, null_count: int = -1):
        self.location = location
        self.offset = int(offset)
        self._keep = []
        if location == HOST:
            values = np.asarray(values)
            if values.dtype == np.bool_:
                self.length = int(values.size - offset) if length is None else int(length)
                bits = pack_bits(values)
                self._keep.append(bits)
                self.dtype = BOOL
                self._vptr = bits.ctypes.data
            else:
                values = np.ascontiguousarray(values)
                self._keep.append(values)
                self.dtype = DTYPES[values.dtype]
                self.length = int(values.size - offset) if length is None else int(length)
                self._vptr = values.ctypes.data
            if valid is None:
                self._mptr, self.null_count = None, 0
            else:
                valid = np.asarray(valid)
                bits = pack_bits(valid) if valid.dtype == np.bool_ else np.ascontiguousarray(valid, dtype=np.uint8)
                self._keep.append(bits)
                self._mptr, self.null_count = bits.ctypes.data, null_count
        else:
            self.dtype = DTYPES[np.dtype(dtype)] if not isinstance(dtype, int) else dtype
            self.length = int(length)
            self._vptr = int(values)
            self._mptr = None if valid is None else int(valid)
            self.null_count = 0 if valid is None else null_count

    def struct(self) -> BlColumn:
        return BlColumn(self.dtype, self.location, self.length, self.offset, self.null_count, self._vptr, self._mptr, None)


class OutColumn:
    """A library-owned output column.  `.to_numpy()` copies host outputs out; device outputs expose
    raw pointers (`.values_ptr`, `.validity_ptr`).  Freed on `.free()` / garbage collection."""

    def __init__(self, st: BlColumn):
        self.st = st

    @property
    def length(self):
        return int(self.st.length)

    @property
    def location(self):
        return int(self.st.location)

    @property
    def values_ptr(self):
        return int(self.st.values or 0)

    @property
    def validity_ptr(self):
        return int(self.st.validity or 0)

    def view(self) -> Column:
        """Re-use a device output as an input column (no copy)."""
        assert self.location == DEVICE
        return Column(self.values_ptr, self.validity_ptr or None, dtype=int(self.st.dtype), length=self.length, location=DEVICE, null_count=int(self.st.null_count))

    def to_numpy(self):
        """-> (values, valid|None).  BOOL columns come back as numpy bool arrays."""
        st, n = self.st, int(self.st.length)
        if st.location == DEVICE:
            host = BlColumn()
            _check(lib().bl_column_to(C.byref(st), C.c_int32(1), C.c_int32(HOST), C.byref(host)))
            return OutColumn(host).to_numpy()      # the returned view keeps the host copy alive
        if st.dtype == BOOL:
            raw = np.ctypeslib.as_array(C.cast(st.values, C.POINTER(C.c_uint8)), shape=((n + 7) // 8 or 1,)) if n else np.zeros(0, np.uint8)
            vals = unpack_bits(raw, n)
        else:
            dt = NP_OF[int(st.dtype)]
            if n:
                # zero-copy: the array views the library-owned pinned buffer and keeps this OutColumn alive
                buf = (C.c_char * (n * dt.itemsize)).from_address(st.values)
                buf._owner = self
                vals = np.frombuffer(buf, dtype=dt, count=n)
                self._exported = True
            else:
                vals = np.zeros(0, dt)
        valid = None
        if st.validity:
            raw = np.ctypeslib.as_array(C.cast(st.validity, C.POINTER(C.c_uint8)), shape=((n + 7) // 8 or 1,)) if n else np.zeros(0, np.uint8)
            valid = unpack_bits(raw, n)
            if valid.all():
                valid = None
        return vals, valid

    def free(self):
        if self.st.owner:
            lib().bl_column_free(C.byref(self.st))

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _as_col(x) -> Column:
    if isinstance(x, Column):
        return x
    if isinstance(x, OutColumn):
        return x.view()
    if isinstance(x, tuple):
        return Column(x[0], x[1])
    if np.isscalar(x):
        raise TypeError("scalars must be passed as length-1 arrays with the column's dtype")
    return Column(x)


def _scalar_col(x, like: Column) -> Column:
    if isinstance(x, (Column, OutColumn, tuple, np.ndarray)):
        return _as_col(x)
    return Column(np.array([x], dtype=NP_OF[like.dtype]))


def _finish(outs, location):
    res = [OutColumn(o) for o in outs]
    if location == HOST:
        np_res = [r.to_numpy() for r in res]
        for r in res:
            if not getattr(r, "_exported", False):
                r.free()       # value arrays that view the buffer keep their OutColumn alive instead
        return np_res
    return res


# ---------------------------------------------------------------------------------- string keys
class StringColumn:
    """A caller-owned host string / binary column in Arrow LargeUtf8 layout, built from a sequence of str / bytes / None
    (or from ready-made `offsets` (int64, n + 1), `data` (uint8) and an optional bool `valid`).  `offset` / `length`
    exercise Arrow slicing."""

    def __init__(self, values=None, *, offsets=None, data=None, valid=None, offset: int = 0, length: int | None = None):
        if values is not None:
            enc = [None if v is None else (v.encode() if isinstance(v, str) else bytes(v)) for v in values]
            lens = np.fromiter((0 if b is None else len(b) for b in enc), dtype=np.int64, count=len(enc))
            offsets = np.zeros(len(enc) + 1, np.int64)
            np.cumsum(lens, out=offsets[1:])
            data = np.frombuffer(b"".join(b for b in enc if b is not None), dtype=np.uint8)
            valid = None if all(b is not None for b in enc) else np.array([b is not None for b in enc], bool)
        self.offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        self.data = np.ascontiguousarray(data, dtype=np.uint8) if data is not None and len(data) else np.zeros(1, np.uint8)
        self.bits = None if valid is None else pack_bits(np.asarray(valid, bool))
        self.offset = int(offset)
        self.length = int(self.offsets.size - 1 - offset) if length is None else int(length)

    def struct(self) -> BlStringColumn:
        return BlStringColumn(HOST, 0, self.length, self.offset, 0 if self.bits is None else -1, self.offsets.ctypes.data, self.data.ctypes.data,
                              None if self.bits is None else self.bits.ctypes.data, None)


class DeviceStringColumn:
    """A library-owned device copy of a string column (bl_string_column_to with BL_DEVICE; chunks are concatenated).
    Every string entry point takes it wherever it takes a StringColumn.  Freed on `.free()` / garbage collection."""

    def __init__(self, col=None, *, st: BlStringColumn | None = None):
        """col: a StringColumn or a list of chunks, copied to the device; st: a library-owned device output to wrap"""
        if st is None:
            chunks = col if isinstance(col, list) else [col]
            st = BlStringColumn()
            _check(lib().bl_string_column_to(_str_array(chunks), C.c_int32(len(chunks)), C.c_int32(DEVICE), C.byref(st)))
        self.st = st
        self.length = int(self.st.length)

    def struct(self) -> BlStringColumn:
        return self.st

    def free(self):
        if self.st.owner:
            lib().bl_string_column_free.restype = None
            lib().bl_string_column_free(C.byref(self.st))

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def _str_array(cols: Sequence):
    return (BlStringColumn * len(cols))(*[c.struct() for c in cols])


def _is_string_key(x) -> bool:
    """a string column, or a list of string chunks"""
    if isinstance(x, list):
        return bool(x) and all(isinstance(c, (StringColumn, DeviceStringColumn)) for c in x)
    return isinstance(x, (StringColumn, DeviceStringColumn))


def string_rank(col, descending: bool = False, location: int = HOST):
    """bl_string_rank: -> ((ranks, valid) | OutColumn, n_distinct).  Dense 1-based UInt32 rank in unsigned byte order
    (a proper prefix first); descending ranks the largest value 1; null rows are null."""
    chunks = col if isinstance(col, list) else [col]
    arr = _str_array(chunks)
    out, nd = BlColumn(), C.c_int64()
    _check(lib().bl_string_rank(arr, C.c_int32(len(chunks)), C.c_int32(int(descending)), C.c_int32(location), C.byref(out), C.byref(nd)))
    return _finish([out], location)[0], int(nd.value)


def string_encode(col, location: int = HOST):
    """bl_string_encode: -> ((codes, valid) | OutColumn, n_distinct).  codes[i] = first row holding the same bytes as row i."""
    chunks = col if isinstance(col, list) else [col]
    arr = _str_array(chunks)
    out, nd = BlColumn(), C.c_int64()
    _check(lib().bl_string_encode(arr, C.c_int32(len(chunks)), C.c_int32(location), C.byref(out), C.byref(nd)))
    return _finish([out], location)[0], int(nd.value)


def _string_out_to_list(out: BlStringColumn) -> list:
    """host BlStringColumn (library-owned) -> list of bytes / None; frees it."""
    try:
        n = int(out.length)
        offs = np.ctypeslib.as_array(C.cast(out.offsets, C.POINTER(C.c_int64)), shape=(n + 1,)).copy()
        total = int(offs[-1])
        data = bytes(np.ctypeslib.as_array(C.cast(out.data, C.POINTER(C.c_uint8)), shape=(max(total, 1),))[:total])
        valid = None
        if out.validity:
            valid = unpack_bits(np.ctypeslib.as_array(C.cast(out.validity, C.POINTER(C.c_uint8)), shape=((n + 7) // 8 or 1,)), n)
        return [None if (valid is not None and not valid[i]) else data[offs[i]:offs[i + 1]] for i in range(n)]
    finally:
        lib().bl_string_column_free.restype = None
        lib().bl_string_column_free(C.byref(out))


def string_gather(col, idx, location: int = HOST):
    """bl_string_gather: -> list of bytes / None (host output) or a DeviceStringColumn (device output)."""
    chunks = col if isinstance(col, list) else [col]
    arr = _str_array(chunks)
    ic = _as_col(idx)
    ist = ic.struct()
    out = BlStringColumn()
    _check(lib().bl_string_gather(arr, C.c_int32(len(chunks)), C.byref(ist), C.c_int32(location), C.byref(out)))
    return _string_out_to_list(out) if location == HOST else DeviceStringColumn(st=out)


def group_by_agg_strings(key, aggs: Sequence, maintain_order: bool = False):
    """bl_groupby_agg_strings (host outputs): key = StringColumn or list of chunks; aggs as in group_by_agg.
    -> (group keys as a list of bytes / None, [agg outputs])."""
    chunks = key if isinstance(key, list) else [key]
    karr = _str_array(chunks)
    keep, agg_structs, cache = [], [], {}
    for kind, vals in aggs:
        if kind == "len" or vals is None:
            agg_structs.append(BlAgg(_agg_kind(kind), 0, None))
            continue
        ident = id(vals)
        if ident not in cache:
            cs = [_as_col(c) for c in (vals if isinstance(vals, list) else [vals])]
            cache[ident] = (cs, _col_array(cs))
        cs, arr = cache[ident]
        keep.append((cs, arr))
        agg_structs.append(BlAgg(_agg_kind(kind), len(cs), C.cast(arr, C.POINTER(BlColumn))))
    aarr = (BlAgg * max(len(agg_structs), 1))(*agg_structs)
    out_key, out_aggs = BlStringColumn(), (BlColumn * max(len(agg_structs), 1))()
    _check(lib().bl_groupby_agg_strings(karr, C.c_int32(len(chunks)), aarr, C.c_int32(len(agg_structs)), C.c_int32(int(maintain_order)), C.c_int32(HOST),
                                        C.byref(out_key), out_aggs))
    return _string_out_to_list(out_key), _finish(list(out_aggs)[: len(agg_structs)], HOST)


def hash_join_strings(left, right, how: str = "inner", nulls_equal: bool = False, maintain_order: str = "none", location: int = HOST):
    """bl_hash_join_strings: row-index tuples of a join on a string key (both sides encoded together on the device)."""
    lc = left if isinstance(left, list) else [left]
    rc = right if isinstance(right, list) else [right]
    la, ra = _str_array(lc), _str_array(rc)
    ol, orr = BlColumn(), BlColumn()
    _check(lib().bl_hash_join_strings(la, C.c_int32(len(lc)), ra, C.c_int32(len(rc)), C.c_int32(JOINS[how]), C.c_int32(int(nulls_equal)), C.c_int32(ORDERS[maintain_order]),
                                      C.c_int32(location), C.byref(ol), C.byref(orr)))
    return tuple(_finish([ol, orr], location))


# ---------------------------------------------------------------------------------- operators
def elementwise(op: str, lhs, rhs, location: int = HOST):
    l = _as_col(lhs) if not np.isscalar(lhs) else None
    r = _as_col(rhs) if not np.isscalar(rhs) else None
    if l is None:
        l = _scalar_col(lhs, r)
    if r is None:
        r = _scalar_col(rhs, l)
    out = BlColumn()
    ls, rs = l.struct(), r.struct()
    _check(lib().bl_elementwise(C.c_int32(OPS[op]), C.byref(ls), C.byref(rs), C.c_int32(location), C.byref(out)))
    return _finish([out], location)[0]


def compare(op: str, lhs, rhs, missing: bool = False, location: int = HOST):
    l = _as_col(lhs)
    r = _scalar_col(rhs, l)
    out = BlColumn()
    ls, rs = l.struct(), r.struct()
    _check(lib().bl_compare(C.c_int32(CMPS[op]), C.byref(ls), C.byref(rs), C.c_int32(int(missing)), C.c_int32(location), C.byref(out)))
    return _finish([out], location)[0]


def _col_array(cols: Sequence[Column]):
    arr = (BlColumn * len(cols))(*[c.struct() for c in cols])
    return arr


def filter(cols: Sequence, mask, location: int = HOST):
    cs = [_as_col(c) for c in cols]
    m = _as_col(mask)
    arr, outs = _col_array(cs), (BlColumn * len(cs))()
    ms = m.struct()
    _check(lib().bl_filter(arr, C.c_int32(len(cs)), C.byref(ms), C.c_int32(location), outs))
    return _finish(list(outs), location)


def filter_cmp(cols: Sequence, pred_col: int, op: str, scalar, location: int = HOST):
    cs = [_as_col(c) for c in cols]
    s = _scalar_col(scalar, cs[pred_col])
    arr, outs = _col_array(cs), (BlColumn * len(cs))()
    ss = s.struct()
    _check(lib().bl_filter_cmp(arr, C.c_int32(len(cs)), C.c_int32(pred_col), C.c_int32(CMPS[op]), C.byref(ss), C.c_int32(location), outs))
    return _finish(list(outs), location)


def gather(cols: Sequence, idx, check_bounds: bool = True, location: int = HOST):
    cs = [_as_col(c) for c in cols]
    ix = _as_col(idx)
    arr, outs = _col_array(cs), (BlColumn * len(cs))()
    ixs = ix.struct()
    _check(lib().bl_gather(arr, C.c_int32(len(cs)), C.byref(ixs), C.c_int32(int(check_bounds)), C.c_int32(location), outs))
    return _finish(list(outs), location)


def group_by_agg(key, aggs: Sequence, maintain_order: bool = False, location: int = HOST):
    """key: column or list of chunks; aggs: [(kind, column | [chunks] | None)].
    Returns (key_out, [agg_outs])."""
    kchunks = [_as_col(c) for c in (key if isinstance(key, list) else [key])]
    karr = _col_array(kchunks)
    keep, agg_structs = [], []
    cache = {}
    for kind, vals in aggs:
        if kind == "len" or vals is None:
            agg_structs.append(BlAgg(_agg_kind(kind), 0, None))
            continue
        ident = id(vals)
        if ident not in cache:
            chunks = [_as_col(c) for c in (vals if isinstance(vals, list) else [vals])]
            cache[ident] = (chunks, _col_array(chunks))
        chunks, arr = cache[ident]
        keep.append((chunks, arr))
        agg_structs.append(BlAgg(_agg_kind(kind), len(chunks), C.cast(arr, C.POINTER(BlColumn))))
    aarr = (BlAgg * max(len(agg_structs), 1))(*agg_structs)
    out_key, out_aggs = BlColumn(), (BlColumn * max(len(agg_structs), 1))()
    _check(lib().bl_groupby_agg(karr, C.c_int32(len(kchunks)), aarr, C.c_int32(len(agg_structs)), C.c_int32(int(maintain_order)), C.c_int32(location),
                                C.byref(out_key), out_aggs))
    res = _finish([out_key] + list(out_aggs)[: len(agg_structs)], location)
    return res[0], res[1:]


def group_by_agg_partitioned(key, aggs: Sequence, my_rank: int, peer_halves: Sequence[int], own_half: int, rows_per_src: int, epoch: int,
                             expected_groups: int = 0, location: int = HOST):
    """One rank's step of the multi-GPU group_by in one C call (bl_groupby_agg_partitioned): local pre-aggregation, fused
    partition + P2P exchange, merge of the rows this rank owns, finish.  aggs as in group_by_agg (one chunk per column)."""
    k = _as_col(key)
    ks = k.struct()
    keep, agg_structs, cache = [], [], {}
    for kind, vals in aggs:
        if kind == "len" or vals is None:
            agg_structs.append(BlAgg(_agg_kind(kind), 0, None))
            continue
        ident = id(vals)
        if ident not in cache:
            chunks = [_as_col(vals)]
            cache[ident] = (chunks, _col_array(chunks))
        chunks, arr = cache[ident]
        keep.append((chunks, arr))
        agg_structs.append(BlAgg(_agg_kind(kind), 1, C.cast(arr, C.POINTER(BlColumn))))
    aarr = (BlAgg * max(len(agg_structs), 1))(*agg_structs)
    n = len(peer_halves)
    parr = (C.c_void_p * n)(*[C.c_void_p(w) for w in peer_halves])
    out_key, out_aggs = BlColumn(), (BlColumn * max(len(agg_structs), 1))()
    _check(lib().bl_groupby_agg_partitioned(C.byref(ks), aarr, C.c_int32(len(agg_structs)), C.c_int32(n), C.c_int32(my_rank), parr, C.c_void_p(own_half),
                                            C.c_int64(rows_per_src), C.c_uint64(epoch), C.c_int64(expected_groups), C.c_int32(location), C.byref(out_key), out_aggs))
    res = _finish([out_key] + list(out_aggs)[: len(agg_structs)], location)
    return res[0], res[1:]


def group_by_agg_keys(keys: Sequence, aggs: Sequence, maintain_order: bool = False, location: int = HOST):
    """Several key columns (one chunk each); aggs as in group_by_agg, plus "quantile:<q>[:<method>]" (bl_groupby_agg_params).
    Returns ([key_outs], [agg_outs])."""
    kcols = [_as_col(c) for c in keys]
    karr = _col_array(kcols)
    keep, agg_structs = [], []
    cache = {}
    for kind, vals in aggs:
        if kind == "len" or vals is None:
            agg_structs.append(BlAgg(_agg_kind(kind), 0, None))
            continue
        ident = id(vals)
        if ident not in cache:
            chunks = [_as_col(c) for c in (vals if isinstance(vals, list) else [vals])]
            cache[ident] = (chunks, _col_array(chunks))
        chunks, arr = cache[ident]
        keep.append((chunks, arr))
        agg_structs.append(BlAgg(_agg_kind(kind), len(chunks), C.cast(arr, C.POINTER(BlColumn))))
    aarr = (BlAgg * max(len(agg_structs), 1))(*agg_structs)
    out_keys, out_aggs = (BlColumn * len(kcols))(), (BlColumn * max(len(agg_structs), 1))()
    params = [_agg_param(kind) for kind, _ in aggs]
    if any(p is not None for p in params):
        parr = (BlAggParam * len(params))(*[BlAggParam(*(p or (0.0, 0)), 0) for p in params])
        _check(lib().bl_groupby_agg_params(karr, C.c_int32(len(kcols)), aarr, parr, C.c_int32(len(agg_structs)), C.c_int32(int(maintain_order)),
                                           C.c_int32(location), out_keys, out_aggs))
    else:
        _check(lib().bl_groupby_agg_keys(karr, C.c_int32(len(kcols)), aarr, C.c_int32(len(agg_structs)), C.c_int32(int(maintain_order)), C.c_int32(location),
                                         out_keys, out_aggs))
    res = _finish(list(out_keys) + list(out_aggs)[: len(agg_structs)], location)
    return res[: len(kcols)], res[len(kcols):]


def group_tuples(key, location: int = HOST):
    """GroupsIdx of the reference (first, offsets, all): groups in first-occurrence order, rows ascending."""
    kch = [_as_col(c) for c in (key if isinstance(key, list) else [key])]
    ka = _col_array(kch)
    of, oo, oa = BlColumn(), BlColumn(), BlColumn()
    _check(lib().bl_group_tuples(ka, C.c_int32(len(kch)), C.c_int32(location), C.byref(of), C.byref(oo), C.byref(oa)))
    res = _finish([of, oo, oa], location)
    if location == HOST:
        return res[0][0], res[1][0], res[2][0]
    return res[0], res[1], res[2]


def hash_join(left_key, right_key, how: str = "inner", nulls_equal: bool = False, maintain_order: str = "none", location: int = HOST):
    lch = [_as_col(c) for c in (left_key if isinstance(left_key, list) else [left_key])]
    rch = [_as_col(c) for c in (right_key if isinstance(right_key, list) else [right_key])]
    la, ra = _col_array(lch), _col_array(rch)
    ol, orr = BlColumn(), BlColumn()
    _check(lib().bl_hash_join(la, C.c_int32(len(lch)), ra, C.c_int32(len(rch)), C.c_int32(JOINS[how]), C.c_int32(int(nulls_equal)),
                              C.c_int32(ORDERS[maintain_order]), C.c_int32(location), C.byref(ol), C.byref(orr)))
    res = _finish([ol, orr], location)
    return res[0], res[1]


def hash_join_keys(left_keys: Sequence, right_keys: Sequence, how: str = "inner", nulls_equal: bool = False, maintain_order: str = "none", location: int = HOST):
    """Join on several key columns per side (bl_hash_join_keys)."""
    lc, rc = [_as_col(c) for c in left_keys], [_as_col(c) for c in right_keys]
    assert len(lc) == len(rc) and lc
    la, ra = _col_array(lc), _col_array(rc)
    ol, orr = BlColumn(), BlColumn()
    _check(lib().bl_hash_join_keys(la, ra, C.c_int32(len(lc)), C.c_int32(JOINS[how]), C.c_int32(int(nulls_equal)), C.c_int32(ORDERS[maintain_order]), C.c_int32(location),
                                   C.byref(ol), C.byref(orr)))
    res = _finish([ol, orr], location)
    return res[0], res[1]


def join(left_key, right_key, left_cols: Sequence, right_cols: Sequence, how: str = "inner", nulls_equal: bool = False,
         maintain_order: str = "none", location: int = HOST):
    """hash_join + gather of both sides on the device (the reference's _finish_join).  Returns
    (left outputs, right outputs), each a list like `gather` returns."""
    lk, rk = _as_col(left_key), _as_col(right_key)
    lc, rc = [_as_col(c) for c in left_cols], [_as_col(c) for c in right_cols]
    lks, rks = lk.struct(), rk.struct()
    la, ra = (_col_array(lc) if lc else None), (_col_array(rc) if rc else None)
    lo, ro = (BlColumn * max(len(lc), 1))(), (BlColumn * max(len(rc), 1))()
    _check(lib().bl_join(C.byref(lks), C.byref(rks), la, C.c_int32(len(lc)), ra, C.c_int32(len(rc)), C.c_int32(JOINS[how]), C.c_int32(int(nulls_equal)),
                         C.c_int32(ORDERS[maintain_order]), C.c_int32(location), lo, ro))
    return _finish(list(lo)[:len(lc)], location), _finish(list(ro)[:len(rc)], location)


SORT_DESCENDING, SORT_NULLS_LAST = 1, 2


def _sort_flags(n_by: int, descending, nulls_last):
    """bool (every column) or one bool per column -> BL_SORT_* words; a length mismatch raises as Polars does."""
    def per_col(v, what):
        if isinstance(v, (bool, np.bool_)):
            return [bool(v)] * n_by
        v = [bool(x) for x in v]
        if len(v) != n_by:
            raise ValueError(f"the length of `{what}` ({len(v)}) does not match the length of `by` ({n_by})")
        return v
    d, nl = per_col(descending, "descending"), per_col(nulls_last, "nulls_last")
    return (C.c_int32 * n_by)(*[(SORT_DESCENDING if a else 0) | (SORT_NULLS_LAST if b else 0) for a, b in zip(d, nl)])


def _sort_keys(by):
    """one key column (array / Column / OutColumn / (values, valid)) or a list of them"""
    return [_as_col(c) for c in by] if isinstance(by, list) else [_as_col(by)]


def _has_string_key(by) -> bool:
    return any(_is_string_key(k) for k in by) if isinstance(by, list) else _is_string_key(by)


def _arg_sort_keys(by, descending, nulls_last, limit, location):
    """bl_arg_sort_keys: `by` holds numeric keys and string keys (a StringColumn / DeviceStringColumn, or a list of chunks)"""
    keys = by if isinstance(by, list) else [by]
    flags = _sort_flags(len(keys), descending, nulls_last)
    descs, keep = (BlSortKey * len(keys))(), []
    for i, k in enumerate(keys):
        if _is_string_key(k):
            chunks = k if isinstance(k, list) else [k]
            arr = _str_array(chunks)
            keep.append(arr)
            descs[i] = BlSortKey(None, C.cast(arr, C.POINTER(BlStringColumn)), len(chunks), flags[i])
        else:
            c = _as_col(k)
            st = c.struct()
            keep.append((c, st))
            descs[i] = BlSortKey(C.pointer(st), None, 0, flags[i])
    out = BlColumn()
    _check(lib().bl_arg_sort_keys(descs, C.c_int32(len(keys)), C.c_int64(-1 if limit is None else int(limit)), C.c_int32(location), C.byref(out)))
    return _finish([out], location)[0]


def arg_sort(by, descending=False, nulls_last=False, limit: int | None = None, location: int = HOST):
    """bl_arg_sort: the UInt32 permutation that sorts the rows by the key column(s) `by` (stable; see the header).
    descending / nulls_last: a bool for every column or one bool per column.  limit: keep the first `limit` rows.
    A key may be a string column (StringColumn / DeviceStringColumn, or a list of its chunks): then bl_arg_sort_keys.
    Host output: a numpy uint32 array; device output: an OutColumn."""
    if _has_string_key(by):
        res = _arg_sort_keys(by, descending, nulls_last, limit, location)
        return res[0] if location == HOST else res
    ks = _sort_keys(by)
    arr, out = _col_array(ks), BlColumn()
    _check(lib().bl_arg_sort(arr, C.c_int32(len(ks)), _sort_flags(len(ks), descending, nulls_last), C.c_int64(-1 if limit is None else int(limit)),
                             C.c_int32(location), C.byref(out)))
    res = _finish([out], location)[0]
    return res[0] if location == HOST else res


def sort(by, cols: Sequence, descending=False, nulls_last=False, limit: int | None = None, location: int = HOST):
    """bl_sort: the payload columns `cols` (4- and 8-byte dtypes) in the order arg_sort(by, ...) gives, on the device.
    With a string key: bl_arg_sort_keys on the device, then bl_gather of the payload (string payloads: string_gather of
    the permutation).  Returns a list like `gather` returns."""
    if _has_string_key(by):
        perm = _arg_sort_keys(by, descending, nulls_last, limit, DEVICE)
        return gather(cols, perm, check_bounds=False, location=location) if len(cols) else []
    ks = _sort_keys(by)
    cs = [_as_col(c) for c in cols]
    karr = _col_array(ks)
    carr, outs = (_col_array(cs) if cs else None), (BlColumn * max(len(cs), 1))()
    _check(lib().bl_sort(karr, C.c_int32(len(ks)), _sort_flags(len(ks), descending, nulls_last), carr, C.c_int32(len(cs)),
                         C.c_int64(-1 if limit is None else int(limit)), C.c_int32(location), outs))
    return _finish(list(outs)[:len(cs)], location)


ASOF_STRATEGIES = {"backward": 0, "forward": 1, "nearest": 2}


def _by_key(k, keep) -> BlSortKey:
    """one `by` column -> a bl_sort_key with flags 0: a string column (StringColumn / DeviceStringColumn / list of chunks)
    or a numeric one"""
    if _is_string_key(k):
        chunks = k if isinstance(k, list) else [k]
        arr = _str_array(chunks)
        keep.append(arr)
        return BlSortKey(None, C.cast(arr, C.POINTER(BlStringColumn)), len(chunks), 0)
    c = _as_col(k)
    st = c.struct()
    keep.append((c, st))
    return BlSortKey(C.pointer(st), None, 0, 0)


def join_asof(left_on, right_on, strategy: str = "backward", tolerance=None, allow_exact_matches: bool = True,
              left_by=None, right_by=None, right_cols: Sequence = (), location: int = HOST):
    """bl_join_asof: for each left row, the right row an asof search picks (see the header for the rule and the
    precondition: sorted `on` columns, per group with `by`; otherwise B200Error with status UNSUPPORTED).
    Returns the UInt32 index column as hash_join does: (values, valid) on the host, an OutColumn on the device.
    left_by / right_by: a list of `by` columns per side (numeric columns, StringColumn or DeviceStringColumn).
    tolerance: a scalar (converted exactly to the key dtype, or to Int32 for an 8/16-bit key as the reference does) or a
    length-1 column of that dtype.
    right_cols: payload columns of the right frame, gathered on the device at the index (bl_gather, or string_gather for
    string columns); then the result is (index, [payloads])."""
    if strategy not in ASOF_STRATEGIES:
        raise ValueError(f"unknown asof strategy {strategy!r} (one of {', '.join(ASOF_STRATEGIES)})")
    if (left_by is None) != (right_by is None):
        raise ValueError("left_by and right_by must be given together")
    left_by, right_by = list(left_by or []), list(right_by or [])
    if len(left_by) != len(right_by):
        raise ValueError(f"left_by has {len(left_by)} columns and right_by {len(right_by)}")
    lc, rc = _as_col(left_on), _as_col(right_on)
    tc = None
    if tolerance is not None:
        if isinstance(tolerance, (Column, OutColumn, tuple, np.ndarray)):
            tc = _as_col(tolerance)
        else:
            if lc.dtype == BOOL:
                raise ValueError("a tolerance needs a numeric key")
            tdt = np.dtype(np.int32) if lc.dtype in (0, 1, 4, 5) else NP_OF[lc.dtype]      # Int8/16, UInt8/16: extracted as Int32
            try:
                t = np.array([tolerance], dtype=tdt)
            except (OverflowError, ValueError, TypeError):
                t = None
            if t is None or not (t[0] == tolerance or (t[0] != t[0] and tolerance != tolerance)):
                raise ValueError(f"tolerance {tolerance!r} is not representable as {tdt}")
            tc = Column(t)
    keep = []
    n_by = len(left_by)
    lb = (BlSortKey * max(n_by, 1))(*[_by_key(k, keep) for k in left_by])
    rb = (BlSortKey * max(n_by, 1))(*[_by_key(k, keep) for k in right_by])
    ls, rs = lc.struct(), rc.struct()
    ts = tc.struct() if tc is not None else None
    out = BlColumn()
    out_loc = DEVICE if right_cols else location
    _check(lib().bl_join_asof(C.byref(ls), C.byref(rs), lb if n_by else None, rb if n_by else None, C.c_int32(n_by),
                              C.c_int32(ASOF_STRATEGIES[strategy]), C.c_int32(int(allow_exact_matches)), C.byref(ts) if ts is not None else None,
                              C.c_int32(out_loc), C.byref(out)))
    idx = _finish([out], out_loc)[0]
    if not right_cols:
        return idx
    payloads = [string_gather(c, idx, location) if _is_string_key(c) else gather([c], idx, check_bounds=False, location=location)[0]
                for c in right_cols]
    return (idx.to_numpy() if location == HOST else idx), payloads


IE_OPS = {"<": 0, "<=": 1, ">": 2, ">=": 3}
IE_FLIP = {"<": ">", "<=": ">=", ">": "<", ">=": "<="}


def ie_join(left_on, right_on, ops, how: str = "inner", left_cols: Sequence = (), right_cols: Sequence = (), location: int = HOST):
    """bl_ie_join: every (left row, right row) pair with left_on[k] ops[k] right_on[k] for each of one or two predicates,
    compared in the total order, every predicate value non-null (see the header for the rule and the order).
    left_on / right_on: a column or a list of one or two columns; ops: one of "<" "<=" ">" ">=" or a list of them.
    how: "inner", "left" (plus (i, null) for every unmatched left row) or "right" (the left join with the sides swapped and
    every operator flipped; then every unmatched right row appears once with a null left index).
    Returns (left_idx, right_idx) as hash_join does.  With left_cols / right_cols, both sides are gathered on the device
    (bl_gather, or string_gather for string columns) and the result is (left outputs, right outputs) as `join` returns."""
    lon = list(left_on) if isinstance(left_on, list) else [left_on]
    ron = list(right_on) if isinstance(right_on, list) else [right_on]
    opl = list(ops) if isinstance(ops, (list, tuple)) else [ops]
    if not 1 <= len(lon) <= 2 or len(ron) != len(lon) or len(opl) != len(lon):
        raise ValueError(f"ie_join needs one or two predicates with one column per side and one operator each, got {len(lon)} left, "
                         f"{len(ron)} right columns and {len(opl)} operators")
    for op in opl:
        if op not in IE_OPS:
            raise ValueError(f"unknown inequality operator {op!r} (one of {', '.join(IE_OPS)})")
    if how not in ("inner", "left", "right"):
        raise ValueError(f"ie_join supports how = 'inner', 'left' or 'right', got {how!r}")
    flip = how == "right"
    if flip:
        lon, ron, opl = ron, lon, [IE_FLIP[op] for op in opl]
    lc, rc = [_as_col(c) for c in lon], [_as_col(c) for c in ron]
    la, ra = _col_array(lc), _col_array(rc)
    opa = (C.c_int32 * len(opl))(*[IE_OPS[op] for op in opl])
    gather_after = bool(left_cols) or bool(right_cols)
    out_loc = DEVICE if gather_after else location
    ol, orr = BlColumn(), BlColumn()
    _check(lib().bl_ie_join(la, ra, opa, C.c_int32(len(opl)), C.c_int32(JOINS["inner" if how == "inner" else "left"]), C.c_int32(out_loc),
                            C.byref(ol), C.byref(orr)))
    li, ri = _finish([ol, orr], out_loc)
    if flip:
        li, ri = ri, li
    if not gather_after:
        return li, ri

    def take(cols, idx):
        return [string_gather(c, idx, location) if _is_string_key(c) else gather([c], idx, check_bounds=False, location=location)[0] for c in cols]
    return take(left_cols, li), take(right_cols, ri)


CUMS = {"cum_sum": 32, "cum_prod": 33, "cum_min": 34, "cum_max": 35, "cum_count": 36}
SHIFT = 37


class BlOverOp(C.Structure):
    _fields_ = [("kind", C.c_int32), ("reverse", C.c_int32), ("periods", C.c_int64), ("values", C.POINTER(BlColumn)), ("param", BlAggParam)]


def _over_op(kind: str, column, options: dict, keep: list) -> BlOverOp:
    """one (kind, column, options) tuple of over() -> a bl_over_op"""
    if not isinstance(kind, str):
        raise ValueError(f"an over() kind is a string, not {kind!r}")
    options = dict(options or {})
    name = kind.partition(":")[0]
    allowed = {"reverse"} if name in CUMS else {"periods"} if name == "shift" else set()
    unknown = set(options) - allowed
    if unknown:
        raise ValueError(f"{kind!r} takes no option(s) {', '.join(sorted(unknown))}")
    if name in CUMS:
        code = CUMS[name]
    elif name == "shift":
        code = SHIFT
    elif name in AGGS or name == "quantile":
        code = _agg_kind(kind)
    else:
        raise ValueError(f"unknown over() kind {kind!r}")
    param = _agg_param(kind) if name == "quantile" else None
    if column is None and name != "len":
        raise ValueError(f"{kind!r} needs a value column")
    ptr = None
    if column is not None:
        c = _as_col(column)
        st = c.struct()
        keep.append((c, st))
        ptr = C.pointer(st)
    return BlOverOp(code, int(bool(options.get("reverse", False))), int(options.get("periods", 1)), ptr, BlAggParam(*(param or (0.0, 0)), 0))


def over(ops: Sequence, partition_by=(), order_by=None, descending: bool = False, nulls_last: bool = False, location: int = HOST):
    """bl_over: window functions with one output row per input row (`expr.over(partition_by, order_by=...)`).
    ops: (kind, column, options) tuples; kind is an aggregation of AGGS ("sum" ... "quantile:<q>:<method>", broadcast to the
    rows of each partition) or "cum_sum" / "cum_prod" / "cum_min" / "cum_max" / "cum_count" (option `reverse`) or "shift"
    (option `periods`, default 1).  partition_by: key columns (numeric, StringColumn / DeviceStringColumn); none = one
    partition.  order_by: one key column (numeric, Bool or string) with `descending` / `nulls_last`.
    Returns one output per op, as gather returns them."""
    if isinstance(partition_by, (np.ndarray, Column, OutColumn, StringColumn, DeviceStringColumn)):
        partition_by = [partition_by]
    partition_by = list(partition_by or [])
    if isinstance(order_by, list):
        if len(order_by) != 1:
            raise ValueError(f"over() takes one order_by column, not {len(order_by)}")
        order_by = order_by[0]
    if not ops:
        raise ValueError("over() needs at least one operation")
    keep = []
    descs = []
    for op in ops:
        if not isinstance(op, tuple) or len(op) not in (2, 3):
            raise ValueError(f"an over() operation is (kind, column[, options]), not {op!r}")
        descs.append(_over_op(op[0], op[1], op[2] if len(op) == 3 else {}, keep))
    parr = (BlSortKey * max(len(partition_by), 1))(*[_by_key(k, keep) for k in partition_by])
    okey = None
    if order_by is not None:
        okey = _by_key(order_by, keep)
        okey.flags = (SORT_DESCENDING if descending else 0) | (SORT_NULLS_LAST if nulls_last else 0)
    oarr = (BlOverOp * len(descs))(*descs)
    outs = (BlColumn * len(descs))()
    _check(lib().bl_over(parr if partition_by else None, C.c_int32(len(partition_by)), C.byref(okey) if okey is not None else None, oarr,
                         C.c_int32(len(descs)), C.c_int32(location), outs))
    return _finish(list(outs), location)


def cum_agg(kind: str, column, reverse: bool = False, location: int = HOST):
    """The plain cum_sum() / cum_prod() / cum_min() / cum_max() / cum_count() of a column: over() with no partition."""
    if kind not in CUMS:
        raise ValueError(f"unknown cumulative kind {kind!r} (one of {', '.join(CUMS)})")
    return over([(kind, column, {"reverse": reverse})], location=location)[0]


ROLLINGS = {"rolling_sum": 40, "rolling_mean": 41, "rolling_min": 42, "rolling_max": 43, "rolling_var": 44, "rolling_std": 45}


class BlRollingOp(C.Structure):
    _fields_ = [("kind", C.c_int32), ("center", C.c_int32), ("window_size", C.c_int64), ("min_samples", C.c_int64), ("ddof", C.c_int32),
                ("reserved", C.c_int32), ("values", C.POINTER(BlColumn))]


def _rolling_op(kind: str, column, options: dict, keep: list) -> BlRollingOp:
    """one (kind, column, options) tuple of rolling() -> a bl_rolling_op"""
    if kind not in ROLLINGS:
        raise ValueError(f"unknown rolling kind {kind!r} (one of {', '.join(ROLLINGS)})")
    options = dict(options or {})
    allowed = {"window_size", "min_samples", "center"} | ({"ddof"} if kind in ("rolling_var", "rolling_std") else set())
    unknown = set(options) - allowed
    if unknown:
        raise ValueError(f"{kind!r} takes no option(s) {', '.join(sorted(unknown))}")
    if "window_size" not in options:
        raise ValueError(f"{kind!r} needs a window_size")
    ws = options["window_size"]
    ms = options.get("min_samples")
    ms = ws if ms is None else ms
    ddof = options.get("ddof", 1)
    for name, v in (("window_size", ws), ("min_samples", ms), ("ddof", ddof)):
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
            raise ValueError(f"{kind!r}: {name} must be an integer, not {v!r}")
    if ws < 1:
        raise ValueError(f"{kind!r}: window_size must be at least 1, not {ws}")
    if not 0 <= ms <= ws:
        raise ValueError(f"{kind!r}: min_samples ({ms}) must be in 0..window_size ({ws})")
    if not 0 <= ddof <= 255:
        raise ValueError(f"{kind!r}: ddof must be in 0..255, not {ddof}")
    if column is None:
        raise ValueError(f"{kind!r} needs a value column")
    c = _as_col(column)
    st = c.struct()
    keep.append((c, st))
    return BlRollingOp(ROLLINGS[kind], int(bool(options.get("center", False))), int(ws), int(ms), int(ddof), 0, C.pointer(st))


def rolling(ops: Sequence, partition_by=(), order_by=None, descending: bool = False, nulls_last: bool = False, location: int = HOST):
    """bl_rolling: fixed-window rolling aggregations, one output row per input row (`expr.rolling_*(...)`, and with
    partition_by / order_by `expr.rolling_*(...).over(partition_by, order_by=...)`).
    ops: (kind, column, options) tuples; kind is one of ROLLINGS; options: window_size (required), min_samples (default
    window_size), center (default False) and, for rolling_var / rolling_std, ddof (default 1).  partition_by / order_by /
    descending / nulls_last as over() takes them.  Returns one output per op, as gather returns them."""
    if isinstance(partition_by, (np.ndarray, Column, OutColumn, StringColumn, DeviceStringColumn)):
        partition_by = [partition_by]
    partition_by = list(partition_by or [])
    if isinstance(order_by, list):
        if len(order_by) != 1:
            raise ValueError(f"rolling() takes one order_by column, not {len(order_by)}")
        order_by = order_by[0]
    if not ops:
        raise ValueError("rolling() needs at least one operation")
    keep = []
    descs = []
    for op in ops:
        if not isinstance(op, tuple) or len(op) != 3:
            raise ValueError(f"a rolling() operation is (kind, column, options), not {op!r}")
        descs.append(_rolling_op(op[0], op[1], op[2], keep))
    parr = (BlSortKey * max(len(partition_by), 1))(*[_by_key(k, keep) for k in partition_by])
    okey = None
    if order_by is not None:
        okey = _by_key(order_by, keep)
        okey.flags = (SORT_DESCENDING if descending else 0) | (SORT_NULLS_LAST if nulls_last else 0)
    oarr = (BlRollingOp * len(descs))(*descs)
    outs = (BlColumn * len(descs))()
    _check(lib().bl_rolling(parr if partition_by else None, C.c_int32(len(partition_by)), C.byref(okey) if okey is not None else None, oarr,
                            C.c_int32(len(descs)), C.c_int32(location), outs))
    return _finish(list(outs), location)


def rolling_agg(kind: str, column, window_size: int, min_samples=None, center: bool = False, ddof: int = 1, location: int = HOST):
    """The plain rolling_sum() ... rolling_std() of a column: rolling() with no partition."""
    opts = {"window_size": window_size, "min_samples": min_samples, "center": center}
    if kind in ("rolling_var", "rolling_std"):
        opts["ddof"] = ddof
    return rolling([(kind, column, opts)], location=location)[0]


RANK_METHODS = {"average": 0, "min": 1, "max": 2, "dense": 3, "ordinal": 4, "random": 5}


class BlRankOp(C.Structure):
    _fields_ = [("method", C.c_int32), ("descending", C.c_int32), ("seed", C.c_uint64), ("values", C.POINTER(BlSortKey))]


def _rank_op(column, options: dict, keep: list) -> BlRankOp:
    """one (column, options) tuple of rank() -> a bl_rank_op"""
    options = dict(options or {})
    unknown = set(options) - {"method", "descending", "seed"}
    if unknown:
        raise ValueError(f"rank takes no option(s) {', '.join(sorted(unknown))}")
    method = options.get("method", "average")
    if method not in RANK_METHODS:
        raise ValueError(f"unknown rank method {method!r} (one of {', '.join(RANK_METHODS)})")
    seed = options.get("seed")
    if seed is None:
        seed = int.from_bytes(os.urandom(8), "little")
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= int(seed) < 2**64:
        raise ValueError(f"rank: seed must be an integer in 0..2^64 - 1 or None, not {seed!r}")
    if column is None:
        raise ValueError("rank needs a value column")
    key = C.pointer(_by_key(column, keep))
    keep.append(key)
    return BlRankOp(RANK_METHODS[method], int(bool(options.get("descending", False))), int(seed), key)


def rank(ops: Sequence, partition_by=(), order_by=None, descending: bool = False, nulls_last: bool = False, location: int = HOST):
    """bl_rank: `expr.rank(method, descending, seed)`, and with partition_by / order_by `expr.rank(...).over(partition_by,
    order_by=...)`, one output row per input row.
    ops: (column, options) tuples; the column is numeric, Bool or a string column (StringColumn / DeviceStringColumn / list
    of chunks); options: method (one of RANK_METHODS, default "average" as in Polars), descending (default False), seed
    (for "random"; None draws one).  partition_by / order_by / descending / nulls_last as over() takes them; order_by
    changes only "ordinal".  Returns one output per op (Float64 for "average", UInt32 otherwise), as gather returns them."""
    if isinstance(partition_by, (np.ndarray, Column, OutColumn, StringColumn, DeviceStringColumn)):
        partition_by = [partition_by]
    partition_by = list(partition_by or [])
    if isinstance(order_by, list):
        if len(order_by) != 1:
            raise ValueError(f"rank() takes one order_by column, not {len(order_by)}")
        order_by = order_by[0]
    if not ops:
        raise ValueError("rank() needs at least one operation")
    keep = []
    descs = []
    for op in ops:
        if not isinstance(op, tuple) or len(op) != 2:
            raise ValueError(f"a rank() operation is (column, options), not {op!r}")
        descs.append(_rank_op(op[0], op[1], keep))
    parr = (BlSortKey * max(len(partition_by), 1))(*[_by_key(k, keep) for k in partition_by])
    okey = None
    if order_by is not None:
        okey = _by_key(order_by, keep)
        okey.flags = (SORT_DESCENDING if descending else 0) | (SORT_NULLS_LAST if nulls_last else 0)
    oarr = (BlRankOp * len(descs))(*descs)
    outs = (BlColumn * len(descs))()
    _check(lib().bl_rank(parr if partition_by else None, C.c_int32(len(partition_by)), C.byref(okey) if okey is not None else None, oarr,
                         C.c_int32(len(descs)), C.c_int32(location), outs))
    return _finish(list(outs), location)


def rank_column(column, method: str = "average", descending: bool = False, seed=None, location: int = HOST):
    """The plain rank() of a column: rank() with no partition."""
    return rank([(column, {"method": method, "descending": descending, "seed": seed})], location=location)[0]


CLOSED = {"right": 0, "left": 1, "both": 2, "none": 3}
_NS_OF = {"ns": 1, "us": 1_000, "ms": 1_000_000, "s": 1_000_000_000, "m": 60_000_000_000, "h": 3_600_000_000_000}
_NS_DAY = 86_400_000_000_000
_DIV_OF = {"ns": 1, "us": 1_000, "ms": 1_000_000}


def window_size_in(window_size, unit) -> int:
    """The window size P of rolling_*_by in the physical unit of `by`: an int is taken as it is; a duration string
    ("30s", "1d12h", "3i") or a timedelta is converted as the reference's Duration::add_ns / add_us / add_ms do
    (polars-time/src/windows/duration.rs:929-1045: weeks and days in whole units, the rest truncated to the unit).
    unit: "ns" / "us" / "ms" for a temporal `by`, None for an integer one (which takes only "Ni" durations)."""
    if isinstance(window_size, (int, np.integer)) and not isinstance(window_size, bool):
        p = int(window_size)
    else:
        weeks = days = nsecs = index = 0
        if isinstance(window_size, _dt.timedelta):
            days, nsecs = window_size.days, (window_size.seconds * 1_000_000 + window_size.microseconds) * 1_000
        elif isinstance(window_size, str):
            parts = re.findall(r"(\d+)([a-z]+)", window_size)
            if not parts or "".join(a + b for a, b in parts) != window_size:
                raise ValueError(f"window_size {window_size!r} is not a duration such as '30s', '1d12h' or '3i'")
            for num, u in parts:
                k = int(num)
                if u in ("mo", "q", "y"):
                    raise ValueError(f"window_size {window_size!r}: calendar durations ({u}) are not supported on the device")
                if u == "w":
                    weeks += k
                elif u == "d":
                    days += k
                elif u == "i":
                    index += k
                elif u in _NS_OF:
                    nsecs += k * _NS_OF[u]
                else:
                    raise ValueError(f"window_size {window_size!r}: unknown unit {u!r}")
            if index and (weeks or days or nsecs):
                raise ValueError(f"window_size {window_size!r} mixes 'i' with temporal units")
        else:
            raise ValueError(f"window_size must be an int, a duration string or a timedelta, not {window_size!r}")
        if unit is None:
            if weeks or days or nsecs:
                raise ValueError(f"an integer `by` column takes a window_size in 'i' units (such as '3i'), not {window_size!r}")
            p = index
        else:
            if index:
                raise ValueError(f"a temporal `by` column takes a temporal window_size, not {window_size!r}")
            div = _DIV_OF[unit]
            p = (weeks * 7 + days) * (_NS_DAY // div) + nsecs // div
    if p <= 0:
        raise ValueError(f"window_size must be strictly positive in the unit of `by` ({unit or 'i'}), got {p} from {window_size!r}")
    if p >= 2 ** 63:
        raise ValueError(f"window_size {window_size!r} does not fit in Int64 in the unit of `by`")
    return p


def _by_column(by):
    """A `by` column -> (column for _as_col, unit).  numpy datetime64[ns|us|ms] keep their unit; datetime64[D] (Date)
    becomes microseconds, as the reference casts Date to Datetime(us); NaT is null."""
    if isinstance(by, np.ndarray) and by.dtype.kind == "M":
        unit = np.datetime_data(by.dtype)[0]
        if unit not in ("ns", "us", "ms", "D"):
            raise ValueError(f"a datetime64[{unit}] `by` column is not supported (ns, us, ms or D)")
        valid = ~np.isnat(by)
        v = by.view(np.int64)
        if unit == "D":
            v, unit = np.where(valid, v, 0) * 86_400_000_000, "us"
        return ((np.ascontiguousarray(v), valid) if not valid.all() else np.ascontiguousarray(v)), unit
    return by, None


class BlRollingByOp(C.Structure):
    _fields_ = [("kind", C.c_int32), ("closed", C.c_int32), ("window_size", C.c_int64), ("min_samples", C.c_int64), ("ddof", C.c_int32),
                ("reserved", C.c_int32), ("values", C.POINTER(BlColumn))]


def rolling_by(ops: Sequence, by, partition_by=(), location: int = HOST):
    """bl_rolling_by: time-based rolling aggregations, one output row per input row (`expr.rolling_*_by(by, ...)`, and with
    partition_by `expr.rolling_*_by(...).over(partition_by)`).
    ops: (kind, column, options) tuples; kind is one of ROLLINGS; options: window_size (required: see window_size_in),
    min_samples (default 0 for rolling_sum, 1 otherwise), closed ("right", "left", "both" or "none"; default "right") and,
    for rolling_var / rolling_std, ddof (default 1).  by: an Int32 / Int64 / UInt32 / UInt64 column or a numpy datetime64
    array.  Returns one output per op, as gather returns them."""
    if isinstance(partition_by, (np.ndarray, Column, OutColumn, StringColumn, DeviceStringColumn)):
        partition_by = [partition_by]
    partition_by = list(partition_by or [])
    if not ops:
        raise ValueError("rolling_by() needs at least one operation")
    byc, unit = _by_column(by)
    keep = []
    descs = []
    for op in ops:
        if not isinstance(op, tuple) or len(op) != 3:
            raise ValueError(f"a rolling_by() operation is (kind, column, options), not {op!r}")
        kind, column, options = op[0], op[1], dict(op[2] or {})
        if kind not in ROLLINGS:
            raise ValueError(f"unknown rolling kind {kind!r} (one of {', '.join(ROLLINGS)})")
        allowed = {"window_size", "min_samples", "closed"} | ({"ddof"} if kind in ("rolling_var", "rolling_std") else set())
        unknown = set(options) - allowed
        if unknown:
            raise ValueError(f"{kind!r} takes no option(s) {', '.join(sorted(unknown))}")
        if "window_size" not in options:
            raise ValueError(f"{kind!r} needs a window_size")
        ws = window_size_in(options["window_size"], unit)
        ms = options.get("min_samples")
        ms = (0 if kind == "rolling_sum" else 1) if ms is None else ms
        ddof = options.get("ddof", 1)
        for name, v in (("min_samples", ms), ("ddof", ddof)):
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
                raise ValueError(f"{kind!r}: {name} must be an integer, not {v!r}")
        if ms < 0:
            raise ValueError(f"{kind!r}: min_samples must not be negative, not {ms}")
        if not 0 <= ddof <= 255:
            raise ValueError(f"{kind!r}: ddof must be in 0..255, not {ddof}")
        closed = options.get("closed", "right")
        if closed not in CLOSED:
            raise ValueError(f"{kind!r}: closed must be one of {', '.join(CLOSED)}, not {closed!r}")
        if column is None:
            raise ValueError(f"{kind!r} needs a value column")
        c = _as_col(column)
        st = c.struct()
        keep.append((c, st))
        descs.append(BlRollingByOp(ROLLINGS[kind], CLOSED[closed], ws, int(ms), int(ddof), 0, C.pointer(st)))
    bc = _as_col(byc)
    bst = bc.struct()
    parr = (BlSortKey * max(len(partition_by), 1))(*[_by_key(k, keep) for k in partition_by])
    oarr = (BlRollingByOp * len(descs))(*descs)
    outs = (BlColumn * len(descs))()
    _check(lib().bl_rolling_by(parr if partition_by else None, C.c_int32(len(partition_by)), C.byref(bst), oarr, C.c_int32(len(descs)),
                               C.c_int32(location), outs))
    return _finish(list(outs), location)


def rolling_agg_by(kind: str, column, by, window_size, min_samples=None, closed: str = "right", ddof: int = 1, location: int = HOST):
    """The plain rolling_sum_by() ... rolling_std_by() of a column: rolling_by() with no partition."""
    opts = {"window_size": window_size, "min_samples": min_samples, "closed": closed}
    if kind in ("rolling_var", "rolling_std"):
        opts["ddof"] = ddof
    return rolling_by([(kind, column, opts)], by, location=location)[0]


class BlRollingQuantileOp(C.Structure):
    _fields_ = [("quantile", C.c_double), ("method", C.c_int32), ("center", C.c_int32), ("window_size", C.c_int64), ("min_samples", C.c_int64),
                ("values", C.POINTER(BlColumn))]


class BlRollingQuantileByOp(C.Structure):
    _fields_ = [("quantile", C.c_double), ("method", C.c_int32), ("closed", C.c_int32), ("window_size", C.c_int64), ("min_samples", C.c_int64),
                ("values", C.POINTER(BlColumn))]


def _rolling_quantile_ops(ops: Sequence, who: str, place: str, keep: list) -> list:
    """(column, options) tuples -> (quantile, method, place option, window_size option, min_samples option, column struct
    pointer); ops that pass the same column object share one struct, so the library builds that column's matrix once.
    place: "center" (fixed windows) or "closed" (time windows)."""
    if not ops:
        raise ValueError(f"{who}() needs at least one operation")
    structs = {}
    out = []
    for op in ops:
        if not isinstance(op, tuple) or len(op) != 2:
            raise ValueError(f"a {who}() operation is (column, options), not {op!r}")
        column, options = op[0], dict(op[1] or {})
        unknown = set(options) - {"quantile", "interpolation", "window_size", "min_samples", place}
        if unknown:
            raise ValueError(f"{who} takes no option(s) {', '.join(sorted(unknown))}")
        for name in ("quantile", "window_size"):
            if name not in options:
                raise ValueError(f"{who} needs a {name}")
        q = options["quantile"]
        if isinstance(q, bool) or not isinstance(q, (int, float, np.integer, np.floating)) or not 0.0 <= float(q) <= 1.0:
            raise ValueError(f"{who}: quantile must be a number in [0, 1], not {q!r}")
        method = options.get("interpolation", "nearest")
        if method not in QUANTILE_METHODS:
            raise ValueError(f"{who}: unknown interpolation {method!r} (one of {', '.join(QUANTILE_METHODS)})")
        if column is None:
            raise ValueError(f"{who} needs a value column")
        if id(column) not in structs:
            c = _as_col(column)
            st = c.struct()
            keep.append((c, st))
            structs[id(column)] = C.pointer(st)
        out.append((float(q), QUANTILE_METHODS[method], options.get(place), options["window_size"], options.get("min_samples"), structs[id(column)]))
    return out


def rolling_quantile(ops: Sequence, partition_by=(), order_by=None, descending: bool = False, nulls_last: bool = False, location: int = HOST):
    """bl_rolling_quantile: fixed-window rolling quantiles, one output row per input row (`expr.rolling_quantile(...)` /
    `rolling_median(...)`, and with partition_by / order_by `.over(partition_by, order_by=...)`).
    ops: (column, options) tuples; options: quantile (required, in [0, 1]), interpolation (one of QUANTILE_METHODS, default
    "nearest"), window_size (required), min_samples (default window_size), center (default False).  Ops given the same
    column object share one device structure.  partition_by / order_by / descending / nulls_last as over() takes them.
    Returns one Float32 (for a Float32 column) or Float64 output per op, as gather returns them."""
    if isinstance(partition_by, (np.ndarray, Column, OutColumn, StringColumn, DeviceStringColumn)):
        partition_by = [partition_by]
    partition_by = list(partition_by or [])
    if isinstance(order_by, list):
        if len(order_by) != 1:
            raise ValueError(f"rolling_quantile() takes one order_by column, not {len(order_by)}")
        order_by = order_by[0]
    keep = []
    descs = []
    for q, method, center, ws, ms, ptr in _rolling_quantile_ops(ops, "rolling_quantile", "center", keep):
        ms = ws if ms is None else ms
        for name, v in (("window_size", ws), ("min_samples", ms)):
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
                raise ValueError(f"rolling_quantile: {name} must be an integer, not {v!r}")
        if ws < 1:
            raise ValueError(f"rolling_quantile: window_size must be at least 1, not {ws}")
        if not 0 <= ms <= ws:
            raise ValueError(f"rolling_quantile: min_samples ({ms}) must be in 0..window_size ({ws})")
        descs.append(BlRollingQuantileOp(q, method, int(bool(center)), int(ws), int(ms), ptr))
    parr = (BlSortKey * max(len(partition_by), 1))(*[_by_key(k, keep) for k in partition_by])
    okey = None
    if order_by is not None:
        okey = _by_key(order_by, keep)
        okey.flags = (SORT_DESCENDING if descending else 0) | (SORT_NULLS_LAST if nulls_last else 0)
    oarr = (BlRollingQuantileOp * len(descs))(*descs)
    outs = (BlColumn * len(descs))()
    _check(lib().bl_rolling_quantile(parr if partition_by else None, C.c_int32(len(partition_by)), C.byref(okey) if okey is not None else None, oarr,
                                     C.c_int32(len(descs)), C.c_int32(location), outs))
    return _finish(list(outs), location)


def rolling_quantile_by(ops: Sequence, by, partition_by=(), location: int = HOST):
    """bl_rolling_quantile_by: time-based rolling quantiles, one output row per input row (`expr.rolling_quantile_by(by,
    ...)` / `rolling_median_by(...)`, and with partition_by `.over(partition_by)`).
    ops: (column, options) tuples; options: quantile (required), interpolation (default "nearest"), window_size (required:
    see window_size_in), min_samples (default 1), closed (default "right").  by: as rolling_by() takes it."""
    if isinstance(partition_by, (np.ndarray, Column, OutColumn, StringColumn, DeviceStringColumn)):
        partition_by = [partition_by]
    partition_by = list(partition_by or [])
    byc, unit = _by_column(by)
    keep = []
    descs = []
    for q, method, closed, ws, ms, ptr in _rolling_quantile_ops(ops, "rolling_quantile_by", "closed", keep):
        ws = window_size_in(ws, unit)
        ms = 1 if ms is None else ms
        if isinstance(ms, bool) or not isinstance(ms, (int, np.integer)) or ms < 0:
            raise ValueError(f"rolling_quantile_by: min_samples must be a non-negative integer, not {ms!r}")
        closed = "right" if closed is None else closed
        if closed not in CLOSED:
            raise ValueError(f"rolling_quantile_by: closed must be one of {', '.join(CLOSED)}, not {closed!r}")
        descs.append(BlRollingQuantileByOp(q, method, CLOSED[closed], ws, int(ms), ptr))
    bc = _as_col(byc)
    bst = bc.struct()
    parr = (BlSortKey * max(len(partition_by), 1))(*[_by_key(k, keep) for k in partition_by])
    oarr = (BlRollingQuantileByOp * len(descs))(*descs)
    outs = (BlColumn * len(descs))()
    _check(lib().bl_rolling_quantile_by(parr if partition_by else None, C.c_int32(len(partition_by)), C.byref(bst), oarr, C.c_int32(len(descs)),
                                        C.c_int32(location), outs))
    return _finish(list(outs), location)


def rolling_quantile_agg(column, quantile: float, interpolation: str = "nearest", window_size: int = 2, min_samples=None, center: bool = False,
                         location: int = HOST):
    """The plain rolling_quantile() of a column: rolling_quantile() with no partition."""
    return rolling_quantile([(column, {"quantile": quantile, "interpolation": interpolation, "window_size": window_size, "min_samples": min_samples,
                                       "center": center})], location=location)[0]


def rolling_median_agg(column, window_size: int, min_samples=None, center: bool = False, location: int = HOST):
    """The plain rolling_median() of a column: quantile 0.5, "linear" (the reference's definition)."""
    return rolling_quantile_agg(column, 0.5, "linear", window_size, min_samples, center, location)


def rolling_quantile_agg_by(column, by, quantile: float, window_size, interpolation: str = "nearest", min_samples=None, closed: str = "right",
                            location: int = HOST):
    """The plain rolling_quantile_by() of a column: rolling_quantile_by() with no partition."""
    return rolling_quantile_by([(column, {"quantile": quantile, "interpolation": interpolation, "window_size": window_size, "min_samples": min_samples,
                                          "closed": closed})], by, location=location)[0]


def rolling_median_agg_by(column, by, window_size, min_samples=None, closed: str = "right", location: int = HOST):
    """The plain rolling_median_by() of a column: quantile 0.5, "linear"."""
    return rolling_quantile_agg_by(column, by, 0.5, window_size, "linear", min_samples, closed, location)


def hash_partition(key, payload: Sequence, n_partitions: int, location: int = HOST):
    k = _as_col(key)
    ps = [_as_col(p) for p in payload]
    parr = _col_array(ps) if ps else None
    ok, op = BlColumn(), (BlColumn * max(len(ps), 1))()
    offs = (C.c_int64 * (n_partitions + 1))()
    ks = k.struct()
    _check(lib().bl_hash_partition(C.byref(ks), parr, C.c_int32(len(ps)), C.c_int32(n_partitions), C.c_int32(location), C.byref(ok), op, offs))
    res = _finish([ok] + list(op)[: len(ps)], location)
    return res[0], res[1:], np.array(list(offs), dtype=np.int64)


class GroupBy:
    """Streaming group_by state (bl_groupby_*): consume batches, exchange partial aggregates, finish."""

    def __init__(self, key_dtype, aggs: Sequence, expected_groups: int = 0, track_first: bool = False, nullable: Sequence | None = None):
        """aggs: [(kind, value_dtype | None)]; nullable[i] = False promises a null-free column (smaller entries)"""
        self.kinds = [AGGS[k] for k, _ in aggs]
        dts = [DTYPES[np.dtype(d)] if d is not None else 3 for _, d in aggs]
        n = len(aggs)
        self.n = n
        self.h = C.c_void_p()
        nl = None if nullable is None else (C.c_int32 * max(n, 1))(*[int(bool(x)) for x in nullable])
        _check(lib().bl_groupby_create(C.c_int32(DTYPES[np.dtype(key_dtype)]), (C.c_int32 * max(n, 1))(*self.kinds), (C.c_int32 * max(n, 1))(*dts), nl,
                                       C.c_int32(n), C.c_int64(expected_groups), C.c_int32(int(track_first)), C.byref(self.h)))

    def consume(self, key, values: Sequence, row_base: int = 0):
        k = _as_col(key)
        cols = [(_as_col(v) if v is not None else Column(np.zeros(0, np.int64))) for v in values]
        arr = _col_array(cols) if cols else None
        ks = k.struct()
        _check(lib().bl_groupby_consume(self.h, C.byref(ks), arr, C.c_int64(row_base)))

    def export_partials(self, n_partitions: int):
        """-> (device pointer, row_words, offsets[n_partitions+1]); free the pointer with dev_free()."""
        p, rw = C.c_void_p(), C.c_int32()
        offs = (C.c_int64 * (n_partitions + 1))()
        _check(lib().bl_groupby_export_partials(self.h, C.c_int32(n_partitions), C.byref(p), C.byref(rw), offs))
        return int(p.value or 0), int(rw.value), np.array(list(offs), dtype=np.int64)

    def export_partials_p2p(self, windows: Sequence[int], my_rank: int, rows_per_src: int):
        """Fused partition + exchange: stores this rank's partial rows into the peers' windows.
        -> (row_words, sent_rows[n_ranks])"""
        n = len(windows)
        arr = (C.c_void_p * n)(*[C.c_void_p(w) for w in windows])
        rw = C.c_int32()
        sent = (C.c_int64 * n)()
        _check(lib().bl_groupby_export_partials_p2p(self.h, C.c_int32(n), C.c_int32(my_rank), arr, C.c_int64(rows_per_src), C.byref(rw), sent))
        return int(rw.value), np.array(list(sent), dtype=np.int64)

    def export_partials_p2p_async(self, window_halves: Sequence[int], my_rank: int, rows_per_src: int, epoch: int) -> int:
        """Fused partition + exchange + count publication (no host round trip).  -> row_words"""
        n = len(window_halves)
        arr = (C.c_void_p * n)(*[C.c_void_p(w) for w in window_halves])
        rw = C.c_int32()
        _check(lib().bl_groupby_export_partials_p2p_async(self.h, C.c_int32(n), C.c_int32(my_rank), arr, C.c_int64(rows_per_src), C.c_uint64(epoch), C.byref(rw)))
        return int(rw.value)

    def merge_window_async(self, own_half: int, n_ranks: int, rows_per_src: int, epoch: int):
        _check(lib().bl_groupby_merge_window_async(self.h, C.c_void_p(own_half), C.c_int32(n_ranks), C.c_int64(rows_per_src), C.c_uint64(epoch)))

    def defer_status(self, on: bool = True):
        lib().bl_groupby_defer_status.restype = None
        lib().bl_groupby_defer_status(self.h, C.c_int32(int(on)))

    def status(self) -> int:
        st = C.c_int32()
        _check(lib().bl_groupby_status(self.h, C.byref(st)))
        return int(st.value)

    def estimated_groups(self) -> int:
        lib().bl_groupby_estimated_groups.restype = C.c_int64
        return int(lib().bl_groupby_estimated_groups(self.h))

    def merge_partials(self, rows_dev_ptr: int, n_rows: int):
        _check(lib().bl_groupby_merge_partials(self.h, C.c_void_p(rows_dev_ptr), C.c_int64(n_rows)))

    def merge_partial_regions(self, ptrs: Sequence[int], counts: Sequence[int]):
        n = len(ptrs)
        pa = (C.c_void_p * n)(*[C.c_void_p(int(p)) for p in ptrs])
        ca = (C.c_int64 * n)(*[int(c) for c in counts])
        _check(lib().bl_groupby_merge_partial_regions(self.h, pa, ca, C.c_int32(n)))

    def finish(self, maintain_order: bool = False, location: int = HOST):
        ok, oa = BlColumn(), (BlColumn * max(self.n, 1))()
        _check(lib().bl_groupby_finish(self.h, C.c_int32(int(maintain_order)), C.c_int32(location), C.byref(ok), oa))
        res = _finish([ok] + list(oa)[: self.n], location)
        return res[0], res[1:]

    def reset(self):
        lib().bl_groupby_reset(self.h)

    def __del__(self):
        try:
            if self.h:
                lib().bl_groupby_destroy(self.h)
                self.h = None
        except Exception:
            pass


class Window:
    """Device memory exported over CUDA IPC so peer ranks can store into it (bl_window_*)."""

    def __init__(self, nbytes: int):
        self.h = C.c_void_p()
        buf = C.create_string_buffer(64)
        _check(lib().bl_window_create(C.c_size_t(nbytes), C.byref(self.h), buf))
        self.ipc_handle = bytes(buf.raw)
        lib().bl_window_ptr.restype = C.c_void_p
        self.ptr = int(lib().bl_window_ptr(self.h))
        self.nbytes = nbytes

    @staticmethod
    def open(ipc_handle: bytes) -> int:
        p = C.c_void_p()
        _check(lib().bl_window_open(C.create_string_buffer(ipc_handle, 64), C.byref(p)))
        return int(p.value)

    @staticmethod
    def close(ptr: int):
        lib().bl_window_close.restype = None
        lib().bl_window_close(C.c_void_p(ptr))

    def destroy(self):
        if self.h:
            lib().bl_window_destroy.restype = None
            lib().bl_window_destroy(self.h)
            self.h = None


def dev_free(ptr: int):
    lib().bl_dev_free(C.c_void_p(ptr))


def dev_alloc(nbytes: int) -> int:
    p = C.c_void_p()
    _check(lib().bl_dev_alloc(C.c_size_t(nbytes), C.byref(p)))
    return int(p.value)


def to_device(values: np.ndarray, valid=None) -> OutColumn:
    """Uploads a numpy column; returns a library-owned device column."""
    c = Column(values, valid)
    out = BlColumn()
    cs = c.struct()
    _check(lib().bl_column_to(C.byref(cs), C.c_int32(1), C.c_int32(DEVICE), C.byref(out)))
    return OutColumn(out)
