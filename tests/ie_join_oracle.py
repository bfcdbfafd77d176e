"""Plain-Python oracle of the inequality join (bl_ie_join).  Values are Python numbers or None (null); floats are compared
in the total order (tot_lt / tot_le ..., polars-utils/src/total_ord.rs: NaN greatest and equal to NaN, -0.0 == +0.0).

(a) `brute`: the rule itself, the reference's own test oracle `east.join(west, how="cross").filter(expr)`
    (py-polars/tests/unit/operations/test_inequality_join.py:417-460, 591-610): every pair whose predicate values are all
    non-null and satisfy every predicate; a left join adds (i, None) for every left row without a pair.
(b) `serial`: a literal restatement of the reference's two serial algorithms (paths relative to crates/polars-ops/src/frame/
    join/iejoin/): one predicate, piecewise_merge_join_tuples + piecewise_merge_join_impl_t (mod.rs:155-226, 667-799); two
    predicates, iejoin_tuples + ie_join_impl_t (mod.rs:75-154, 572-665) with the L1 / L2 arrays and the bit array of
    l1_l2.rs and filtered_bit_array.rs; then append_unmatched_left (mod.rs:232-265) for a left join.
Both return a list of (left row, right row | None) pairs; compare them as multisets."""
import math

LT, LE, GT, GE = "<", "<=", ">", ">="
OPS = (LT, LE, GT, GE)


def tot_key(v):
    """sort / comparison key of the total order"""
    if isinstance(v, float) and math.isnan(v):
        return (1, 0.0)
    return (0, v + 0.0 if isinstance(v, float) else v)


def holds(a, op, b) -> bool:
    ka, kb = tot_key(a), tot_key(b)
    return {LT: ka < kb, LE: ka <= kb, GT: ka > kb, GE: ka >= kb}[op]


def flip(op):
    return {LT: GT, LE: GE, GT: LT, GE: LE}[op]


def brute(left, right, ops, how="inner"):
    """left / right: one value list per predicate; ops: one operator per predicate; how: inner / left / right"""
    if how == "right":
        return [(l, r) for r, l in brute(right, left, [flip(o) for o in ops], "left")]
    nl, nr = len(left[0]), len(right[0])
    out = []
    for i in range(nl):
        hit = False
        for j in range(nr):
            ok = True
            for k, op in enumerate(ops):
                a, b = left[k][i], right[k][j]
                if a is None or b is None or not holds(a, op, b):
                    ok = False
                    break
            if ok:
                out.append((i, j))
                hit = True
        if how == "left" and not hit:
            out.append((i, None))
    return out


def arg_sort_non_null(values, descending):
    """arg_sort(SortOptions{nulls_last: false, maintain_order: true, descending}) with the leading nulls sliced off: the
    non-null positions, stably ordered (ties keep their original order, also when descending)"""
    idx = [i for i, v in enumerate(values) if v is not None]
    return sorted(idx, key=lambda i: tot_key(values[i]), reverse=descending)


def partition_point(seq, pred):
    """the first position whose element fails `pred` (pred holds on a prefix of seq)"""
    p = 0
    while p < len(seq) and pred(seq[p]):
        p += 1
    return p


def piecewise_merge_join(left, right, op):
    """piecewise_merge_join_tuples / piecewise_merge_join_impl_t for the single predicate `left op right`"""
    descending = op in (GT, GE)
    left_order = arg_sort_non_null(left, descending)
    right_order = arg_sort_non_null(right, descending)
    left_ordered = [left[i] for i in left_order]
    right_ordered = [right[i] for i in right_order]
    pairs = []
    left_idx = right_idx = 0
    while left_idx < len(left_ordered):
        left_val = left_ordered[left_idx]
        while right_idx < len(right_ordered):
            if holds(left_val, op, right_ordered[right_idx]):
                # the predicate then holds for every remaining right row
                for included in range(right_idx, len(right_ordered)):
                    pairs.append((left_order[left_idx], right_order[included]))
                break
            right_idx += 1
        if right_idx == len(right_ordered):
            break
        left_idx += 1
    return pairs


def find_search_start_index(l1, index, op1):
    """l1_l2.rs find_search_start_index: partition_point over l1[index..] from the entry's own value"""
    value = l1[index][1]
    sub = l1[index:]
    pred = {GT: lambda a: holds(a[1], GE, value),
            LT: lambda a: holds(a[1], LE, value),
            GE: lambda a: holds(value, LT, a[1]),
            LE: lambda a: holds(value, GT, a[1])}[op1]
    return partition_point(sub, pred) + index


def find_matches_in_l1(l1, l1_index, row_index, bits, op1, pairs):
    start = find_search_start_index(l1, l1_index, op1)
    for set_bit in range(start, len(l1)):
        if bits[set_bit]:
            right_row_index = l1[set_bit][0]
            assert right_row_index < 0
            pairs.append((row_index - 1, -right_row_index - 1))


def iejoin(left, right, op1, op2):
    """iejoin_tuples / ie_join_impl_t for `left[0] op1 right[0] and left[1] op2 right[1]`"""
    l1_descending = op1 in (GT, GE)
    l2_descending = op2 in (LT, LE)
    left_height = len(left[0])
    x = list(left[0]) + list(right[0])
    y = list(left[1]) + list(right[1])
    l1_order = arg_sort_non_null(x, l1_descending)
    y_ordered_by_x = [y[i] for i in l1_order]
    l2_order = arg_sort_non_null(y_ordered_by_x, l2_descending)
    # L1: (row_index, x value); row_index > 0 for a left row (row + 1), < 0 for a right row (-(row + 1))
    l1 = [((i + 1) if i < left_height else -(i - left_height) - 1, x[i]) for i in l1_order]
    bits = [False] * len(l1)
    pairs = []
    if op2 in (LT, GT):
        # strict: the stable l2 sort makes p increase along a run of equal y values
        for p in l2_order:
            row_index = l1[p][0]
            if row_index > 0:
                find_matches_in_l1(l1, p, row_index, bits, op1, pairs)
            else:
                bits[p] = True
    else:
        # non-strict: mark a whole run of equal y values visited before any of its left entries looks for matches
        l2 = []
        for i, p in enumerate(l2_order):
            run_end = i + 1 == len(l2_order) or tot_key(y_ordered_by_x[l2_order[i + 1]]) != tot_key(y_ordered_by_x[p])
            l2.append((p, run_end))
        run_start = 0
        for i, (p, run_end) in enumerate(l2):
            if l1[p][0] < 0:
                bits[p] = True
            if run_end:
                for q, _ in l2[run_start:i + 1]:
                    row_index = l1[q][0]
                    if row_index > 0:
                        find_matches_in_l1(l1, q, row_index, bits, op1, pairs)
                run_start = i + 1
    return pairs


def append_unmatched_left(pairs, left_height):
    matched = {l for l, _ in pairs}
    return list(pairs) + [(i, None) for i in range(left_height) if i not in matched]


def serial(left, right, ops, how="inner"):
    """the reference's serial dispatch: one predicate -> piecewise merge join, two -> IEJoin; left -> unmatched appended;
    right -> the flipped left join (emit_unmatched_right_via_flip, mod.rs:279-296)"""
    if how == "right":
        return [(l, r) for r, l in serial(right, left, [flip(o) for o in ops], "left")]
    pairs = piecewise_merge_join(left[0], right[0], ops[0]) if len(ops) == 1 else iejoin(left, right, ops[0], ops[1])
    return append_unmatched_left(pairs, len(left[0])) if how == "left" else pairs


def as_multiset(pairs):
    return sorted(pairs, key=lambda p: (p[0] is None, p[0] or 0, p[1] is None, p[1] or 0))
