"""Boundary B2 — post-optimisation IR callback (SURVEY.md §8(b)): run Filter→GroupBy and single-key Join
subtrees of an optimised Polars plan on the GPU library, everything else on Polars' own engine.

    import polars as pl
    from polars_b200.engine import execute_with_b200
    out = lf.collect(post_opt_callback=execute_with_b200)        # py-polars/src/polars/lazyframe/frame.py:2191-2192

The reference hands the optimised IR to a Python callable `(NodeTraverser, duration) -> None`
(crates/polars-python/src/lazyframe/general.rs:57-85).  The callable may inspect nodes
(`view_current_node`, `get_inputs`, `view_expression`, crates/polars-python/src/lazyframe/visit.rs:110-190)
and replace the current subtree by a Python UDF with `set_udf` (visit.rs:156-175), which the in-memory
engine then calls instead of executing the subtree.  This is the seam the reference's own GPU engine uses
(py-polars/src/polars/lazyframe/engine.py:946-970).

There is no Polars wheel in the authoring image or on the GPU box (no Rust toolchain to build one), so the
UDF bodies are written against the reference source only; the plan matcher (which shapes are taken, which are
left to Polars) is tested with a mock NodeTraverser in tests/test_engine_matcher.py.  It is deliberately
conservative: any node shape it does not recognise is left untouched (Polars executes it).
Recognised:
  * GroupBy(keys=[col, ...], aggs ⊆ {col.sum/mean/min/max/count/first/last/var/std/n_unique, len}) over a DataFrameScan, optionally through
    one Filter(col <cmp> literal)                      -> bl_filter_cmp + bl_groupby_agg / bl_groupby_agg_keys
  * Join(inner|left|semi|anti, one key column per side) of two DataFrameScans -> bl_hash_join + bl_gather
  * Sort(by=[col, ...] of numeric / Boolean columns, slice None or (0, k)) of a DataFrameScan -> bl_arg_sort (limit = k)
    + bl_gather of the numeric columns (other columns: Polars' take of the same permutation)
  * Distinct(keep, subset of numeric / Boolean columns or None, maintain_order, slice) of a DataFrameScan -> bl_unique
    + bl_gather of the numeric columns (other columns: Polars' take of the same row ids)
"""
from __future__ import annotations

from typing import Any

import numpy as np

_NUMERIC = {"Int32": np.int32, "Int64": np.int64, "UInt32": np.uint32, "UInt64": np.uint64, "Float32": np.float32, "Float64": np.float64}
_CMP = {"Eq": "eq", "NotEq": "ne", "Lt": "lt", "LtEq": "le", "Gt": "gt", "GtEq": "ge"}
_AGG = {"sum": "sum", "mean": "mean", "min": "min", "max": "max", "count": "count", "first": "first", "last": "last", "var": "var", "std": "std",
        "n_unique": "n_unique"}


class _Unsupported(Exception):
    pass


def _series_to_column(plb, s):
    """pl.Series (numeric, any chunking, nulls) -> list of plb.Column chunks over the Arrow buffers (zero copy)."""
    import pyarrow as pa
    if str(s.dtype) not in _NUMERIC:
        raise _Unsupported(f"dtype {s.dtype}")
    chunks = []
    arr = s.to_arrow()
    for ch in (arr.chunks if isinstance(arr, pa.ChunkedArray) else [arr]):
        bufs = ch.buffers()
        values = np.frombuffer(bufs[1], dtype=_NUMERIC[str(s.dtype)])
        valid = None if bufs[0] is None or ch.null_count == 0 else np.frombuffer(bufs[0], dtype=np.uint8)
        chunks.append(plb.Column(values, valid, offset=ch.offset, length=len(ch), null_count=ch.null_count))
    return chunks


def _column_name(nt, node: int) -> str:
    e = nt.view_expression(node)
    if type(e).__name__ != "Column":
        raise _Unsupported(type(e).__name__)
    return str(e.name)


def _parse_agg(nt, expr_ir):
    """Agg / Len expression view -> (library aggregation, column | None, output name).
    Agg.options carries the per-aggregation switch (visitor/expr_nodes.rs:953-1032): min/max -> propagate_nans
    (the library ignores NaNs like the default `min()`/`max()`, so True is left to Polars), count -> include_nulls
    (`pl.col(x).len()` lowers to count(include_nulls=True) = the group length, dsl/mod.rs:923-929)."""
    e = nt.view_expression(expr_ir.node)
    name = type(e).__name__
    if name == "Len":
        return "len", None, expr_ir.output_name
    if name == "Agg" and str(e.name) in _AGG and len(e.arguments) == 1:
        kind, opt = _AGG[str(e.name)], getattr(e, "options", None)
        col = _column_name(nt, e.arguments[0])
        if kind in ("min", "max") and opt not in (None, False):
            raise _Unsupported(f"{kind}(propagate_nans=True)")
        if kind == "count":
            if opt is True:
                return "len", None, expr_ir.output_name          # include_nulls: every row of the group counts
            if opt not in (None, False):
                raise _Unsupported("count options")
        elif kind in ("var", "std"):
            # options = ddof (visitor/expr_nodes.rs:1027-1040); the library carries it in the aggregation kind ("var:0", BL_AGG_WITH_DDOF)
            if not isinstance(opt, int) or isinstance(opt, bool) or not 0 <= opt <= 255:
                raise _Unsupported(f"{kind} ddof {opt!r}")
            return f"{kind}:{opt}", col, expr_ir.output_name
        elif kind in ("sum", "mean", "first", "last", "n_unique") and opt is not None:      # these carry no option
            raise _Unsupported(f"{kind} options")
        return kind, col, expr_ir.output_name
    raise _Unsupported(f"aggregation {name}")


def _parse_filter(nt, node):
    """Filter(input, BinaryExpr(Column, cmp, Literal)) -> (input node id, column, op, python scalar)."""
    pred = nt.view_expression(node.predicate.node)
    if type(pred).__name__ != "BinaryExpr":
        raise _Unsupported("filter predicate")
    op = str(pred.op).split(".")[-1]
    if op not in _CMP:
        raise _Unsupported(f"operator {op}")
    col = _column_name(nt, pred.left)
    lit = nt.view_expression(pred.right)
    if type(lit).__name__ != "Literal":
        raise _Unsupported("filter rhs")
    return node.input, col, _CMP[op], lit.value


def _scan_frame(nt, node_id):
    """DataFrameScan node -> a thunk producing the pl.DataFrame (polars is imported only when the UDF runs)."""
    nt.set_node(node_id)
    n = nt.view_current_node()
    if type(n).__name__ != "DataFrameScan" or n.selection is not None:
        raise _Unsupported(type(n).__name__)
    pydf, projection = n.df, n.projection

    def frame():
        import polars as pl
        df = pl.DataFrame._from_pydf(pydf) if hasattr(pl.DataFrame, "_from_pydf") else pydf
        return df.select(list(projection)) if projection is not None else df

    return frame


def _plan_group_by(plb, nt, root_id, node):
    if len(node.keys) < 1:
        raise _Unsupported("group_by without keys")
    # GroupbyOptions (visitor/expr_nodes.rs:757-790): a pushed-down slice, dynamic or rolling windows change the result
    opts = getattr(node, "options", None)
    if opts is not None and any(getattr(opts, f, None) is not None for f in ("slice", "dynamic", "rolling")):
        raise _Unsupported("group_by options (slice / dynamic / rolling)")
    key_names = [_column_name(nt, k.node) for k in node.keys]       # several plain columns -> bl_groupby_agg_keys
    key_name = key_names[0]
    aggs = [_parse_agg(nt, a) for a in node.aggs]
    if len(key_names) > 1 and any(kind == "n_unique" for kind, _, _ in aggs):
        raise _Unsupported("n_unique with several key columns")       # BL_AGG_N_UNIQUE is a bl_groupby_agg (single key) aggregation
    nt.set_node(node.input)
    child = nt.view_current_node()
    flt = None
    if type(child).__name__ == "Filter":
        inp, fcol, fop, fval = _parse_filter(nt, child)
        flt = (fcol, fop, fval)
        frame = _scan_frame(nt, inp)
    else:
        frame = _scan_frame(nt, node.input)
    nt.set_node(root_id)
    maintain_order = bool(node.maintain_order)

    def run(*_args: Any, **_kwargs: Any):
        import polars as pl
        df = frame()
        needed = key_names + [c for _, c, _ in aggs if c is not None]
        cols = {c: _series_to_column(plb, df.get_column(c)) for c in dict.fromkeys(needed)}
        if flt is not None:
            fcol, fop, fval = flt
            names = list(dict.fromkeys(needed + [fcol]))
            dev = [plb.to_device(*_concat(df.get_column(c))) for c in names]
            outs = plb.filter_cmp([d.view() for d in dev], names.index(fcol), fop, fval, location=plb.DEVICE)
            view = {c: outs[i].view() for i, c in enumerate(names)}
            vals = {c: view[c] for c in needed}
        else:
            vals = cols
        agg_args = [(kind, None if c is None else vals[c]) for kind, c, _ in aggs]
        if len(key_names) == 1:
            kout, outs = plb.group_by_agg(vals[key_name], agg_args, maintain_order)
            kouts = [kout]
        else:
            if flt is None and any(len(vals[c]) != 1 for c in key_names):
                raise plb.B200Error(4, "multi-column keys need single-chunk columns")      # the caller rechunks and retries on CPU
            kouts, outs = plb.group_by_agg_keys([vals[c][0] if isinstance(vals[c], list) else vals[c] for c in key_names], agg_args, maintain_order)
        res = {}
        for name, (k, kv) in zip(key_names, kouts):
            res[name] = pl.Series(name, k).set(pl.Series(~kv), None) if kv is not None else pl.Series(name, k)
        for (kind, c, out_name), (v, m) in zip(aggs, outs):
            s = pl.Series(out_name, v)
            res[out_name] = s.set(pl.Series(~m), None) if m is not None else s
        return pl.DataFrame(res)

    return run


def _concat(series):
    a = series.to_numpy()
    return (a, None) if series.null_count() == 0 else (np.where(series.is_null().to_numpy(), 0, a), ~series.is_null().to_numpy())


_JOIN_HOW = {"Inner": "inner", "Left": "left", "Semi": "semi", "Anti": "anti"}
_JOIN_ORDER = {"none": "none", "left": "left", "right": "right", "left_right": "left_right", "right_left": "right_left"}


def _join_options(options):
    """Join.options = (how, nulls_equal, slice, suffix, coalesce, maintain_order) (visitor/nodes.rs:590-651).
    `how` is a plain str for the equi-joins (a tuple for asof / iejoin: never taken).  Returns
    (how, nulls_equal, suffix, maintain_order) or raises when an option asks for something the UDF does not do."""
    if not isinstance(options, (tuple, list)) or len(options) != 6:
        raise _Unsupported("join options")
    how, nulls_equal, slc, suffix, coalesce, order = options
    if not isinstance(how, str) or how not in _JOIN_HOW:
        raise _Unsupported(f"join type {how!r}")
    if slc is not None:
        raise _Unsupported("join with a pushed-down slice")
    if not isinstance(nulls_equal, bool) or not isinstance(suffix, str) or str(order) not in _JOIN_ORDER:
        raise _Unsupported("join options")
    how = _JOIN_HOW[how]
    if how in ("inner", "left") and coalesce is not True:
        raise _Unsupported("coalesce=False keeps both key columns")          # the UDF drops the right key (general.rs:17-49)
    if how in ("semi", "anti") and str(order) != "none":
        raise _Unsupported("maintain_order on a semi/anti join")
    return how, nulls_equal, suffix, _JOIN_ORDER[str(order)]


def _plan_join(plb, nt, root_id, node):
    how, nulls_equal, suffix, order = _join_options(node.options)
    if len(node.left_on) != 1 or len(node.right_on) != 1:
        raise _Unsupported("multi-key join")
    lkey, rkey = _column_name(nt, node.left_on[0].node), _column_name(nt, node.right_on[0].node)
    left_frame, right_frame = _scan_frame(nt, node.input_left), _scan_frame(nt, node.input_right)
    nt.set_node(root_id)

    def run(*_args: Any, **_kwargs: Any):
        import polars as pl
        left, right = left_frame(), right_frame()
        (li, _), (ri, rv) = plb.hash_join(_series_to_column(plb, left.get_column(lkey)), _series_to_column(plb, right.get_column(rkey)), how,
                                          nulls_equal, order)
        if how in ("semi", "anti"):          # only left rows survive (single_keys_semi_anti.rs:41-140)
            return left[pl.Series(li)]
        ridx = pl.Series(ri) if rv is None else pl.Series(ri).set(pl.Series(~rv), None)
        out_l = left[pl.Series(li)]
        out_r = right.drop(rkey)[ridx] if how == "inner" else right.drop(rkey).select(pl.all().gather(ridx))
        clash = [c for c in out_r.columns if c in out_l.columns]
        return out_l.hstack(out_r.rename({c: c + suffix for c in clash}))      # general.rs:17-49

    return run


def _host_column(series):
    """pl.Series -> (values, valid | None) numpy arrays with null slots filled (Boolean included)."""
    if series.null_count() == 0:
        return series.to_numpy(), None
    fill = False if str(series.dtype) == "Boolean" else 0
    return series.fill_null(fill).to_numpy(), ~series.is_null().to_numpy()


_SORTABLE = set(_NUMERIC) | {"Int8", "Int16", "UInt8", "UInt16", "Boolean"}


def _sort_slice_limit(slc):
    """Sort.slice = None | (offset, len, id) (visitor/nodes.rs:246-257, 533-549): offset 0 becomes the limit."""
    if slc is None:
        return None
    if not isinstance(slc, (tuple, list)) or len(slc) not in (2, 3) or (len(slc) == 3 and slc[2] is not None):
        raise _Unsupported("sort slice")
    offset, length = slc[0], slc[1]
    if not isinstance(offset, int) or not isinstance(length, int) or offset != 0 or length < 0:
        raise _Unsupported("sort slice with a nonzero offset")
    return length


def _plan_sort(plb, nt, root_id, node):
    """Sort(input=DataFrameScan, by_column=[Column, ...], sort_options=(maintain_order, nulls_last, descending), slice).
    The library's sort is always stable, which is what maintain_order asks for and a valid order when it is not set.
    Key dtypes are checked here, on the Sort node's schema (NodeTraverser.get_schema, visit.rs:127-131): a key the device
    cannot order (String, temporal, nested ...) leaves the node to Polars.  Every column of the frame is materialised:
    the 4- and 8-byte numeric ones with K4 on the device, any other column with Polars' own take of the same permutation."""
    opts, by_column = getattr(node, "sort_options", None), getattr(node, "by_column", None)
    if not isinstance(opts, (tuple, list)) or len(opts) != 3 or not isinstance(by_column, (tuple, list)):
        raise _Unsupported("sort options")
    _maintain_order, nulls_last, descending = opts
    by = [_column_name(nt, e.node) for e in by_column]
    if not by:
        raise _Unsupported("sort without keys")
    nulls_last, descending = list(nulls_last), list(descending)
    # Polars broadcasts a single flag to every key (SortMultipleOptions)
    if len(nulls_last) == 1:
        nulls_last *= len(by)
    if len(descending) == 1:
        descending *= len(by)
    if len(nulls_last) != len(by) or len(descending) != len(by):
        raise _Unsupported("sort flags")
    limit = _sort_slice_limit(getattr(node, "slice", None))
    if not hasattr(nt, "get_schema"):
        raise _Unsupported("no schema to check the sort keys against")
    schema = {str(k): str(v) for k, v in dict(nt.get_schema()).items()}
    for c in by:
        if schema.get(c) not in _SORTABLE:
            raise _Unsupported(f"sort key {c}: dtype {schema.get(c)}")
    frame = _scan_frame(nt, node.input)
    nt.set_node(root_id)

    def run(*_args: Any, **_kwargs: Any):
        import polars as pl
        df = frame().rechunk()
        dev_cols = [c for c in df.columns if str(df.schema[c]) in _NUMERIC]          # K4 takes 4- and 8-byte elements
        idx = plb.arg_sort([_host_column(df.get_column(c)) for c in by], descending=descending, nulls_last=nulls_last, limit=limit,
                           location=plb.DEVICE)
        res = {}
        if dev_cols:
            outs = plb.gather([_host_column(df.get_column(c)) for c in dev_cols], idx.view(), check_bounds=False)
            for c, (v, m) in zip(dev_cols, outs):
                s = pl.Series(c, v)
                res[c] = s.set(pl.Series(~m), None) if m is not None else s
        rest = [c for c in df.columns if c not in res]
        if rest:
            taken = df.select(rest)[pl.Series(idx.to_numpy()[0])]
            for c in rest:
                res[c] = taken.get_column(c)
        return pl.DataFrame([res[c] for c in df.columns])

    return run


_KEEP = {"first", "last", "any", "none"}


def _distinct_options(options):
    """Distinct.options = (keep, subset | None, maintain_order, slice | None) (visitor/nodes.rs:678-695); keep is the
    strategy's snake_case name.  Returns (keep, subset, slice) or raises for a shape the UDF does not take."""
    if not isinstance(options, (tuple, list)) or len(options) != 4:
        raise _Unsupported("distinct options")
    keep, subset, maintain_order, slc = options
    if not isinstance(keep, str) or keep not in _KEEP or not isinstance(maintain_order, bool):
        raise _Unsupported(f"distinct keep {keep!r}")
    if subset is not None and (not isinstance(subset, (tuple, list)) or not subset or not all(isinstance(c, str) for c in subset)):
        raise _Unsupported("distinct subset")
    if slc is not None and (not isinstance(slc, (tuple, list)) or len(slc) != 2 or not all(isinstance(v, int) and not isinstance(v, bool) for v in slc)
                            or slc[1] < 0):
        raise _Unsupported("distinct slice")
    return keep, None if subset is None else list(subset), None if slc is None else tuple(slc)


def _slice_ids(ids, slc):
    """the (offset, len) slice of the kept row ids, as the reference's slice_offsets clamps it (a negative offset counts
    from the end)"""
    if slc is None:
        return ids
    offset, length = slc
    n = len(ids)
    start = offset + n if offset < 0 else offset
    stop = min(max(start + length, 0), n)
    start = min(max(start, 0), n)
    return ids[start:stop]


def _plan_distinct(plb, nt, root_id, node):
    """Distinct(input=DataFrameScan, options=(keep, subset, maintain_order, slice)): DataFrame.unique, SELECT DISTINCT,
    UNION.  The kept rows come from bl_unique in ascending row order, which is what maintain_order asks for and a valid
    order when it is not set; the slice applies to them.  The subset (every column when None) must be numeric or Boolean,
    checked on the node's schema: anything else (String, temporal, nested ...) leaves the node to Polars.  The 4- and 8-byte
    numeric columns are gathered with K4, the others with Polars' own take of the same ids."""
    keep, subset, slc = _distinct_options(getattr(node, "options", None))
    if not hasattr(nt, "get_schema"):
        raise _Unsupported("no schema to check the subset against")
    schema = {str(k): str(v) for k, v in dict(nt.get_schema()).items()}
    names = list(schema) if subset is None else subset
    if not names:
        raise _Unsupported("distinct over no columns")
    for c in names:
        if schema.get(c) not in _SORTABLE:
            raise _Unsupported(f"distinct key {c}: dtype {schema.get(c)}")
    frame = _scan_frame(nt, node.input)
    nt.set_node(root_id)

    def run(*_args: Any, **_kwargs: Any):
        import polars as pl
        df = frame().rechunk()
        ids = _slice_ids(plb.arg_unique([_host_column(df.get_column(c)) for c in (df.columns if subset is None else subset)], keep), slc)
        dev_cols = [c for c in df.columns if str(df.schema[c]) in _NUMERIC]          # K4 takes 4- and 8-byte elements
        res = {}
        if dev_cols:
            outs = plb.gather([_host_column(df.get_column(c)) for c in dev_cols], np.ascontiguousarray(ids, dtype=np.uint32), check_bounds=False)
            for c, (v, m) in zip(dev_cols, outs):
                s = pl.Series(c, v)
                res[c] = s.set(pl.Series(~m), None) if m is not None else s
        rest = [c for c in df.columns if c not in res]
        if rest:
            taken = df.select(rest)[pl.Series(ids)]
            for c in rest:
                res[c] = taken.get_column(c)
        return pl.DataFrame([res[c] for c in df.columns])

    return run


def execute_with_b200(nt: Any, duration_since_start: int | None = None, *, raise_on_fail: bool = False) -> None:
    """The post-optimisation callback.  Leaves the plan untouched when the root is not a supported shape."""
    import polars_b200 as plb
    try:
        root = nt.view_current_node()
        kind = type(root).__name__
        root_id = nt.get_node() if hasattr(nt, "get_node") else None
        if kind == "GroupBy":
            fn = _plan_group_by(plb, nt, root_id, root)
        elif kind == "Join":
            fn = _plan_join(plb, nt, root_id, root)
        elif kind == "Sort":
            fn = _plan_sort(plb, nt, root_id, root)
        elif kind == "Distinct":
            fn = _plan_distinct(plb, nt, root_id, root)
        else:
            raise _Unsupported(kind)
        nt.set_udf(fn)
    except _Unsupported:
        if raise_on_fail:
            raise
    except plb.B200Error:
        if raise_on_fail:
            raise
