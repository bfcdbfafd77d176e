"""CPU tests (-m "not gpu") of the inequality join: the oracle against the reference's known answers
(tests/golden/ie_join_kats.json), an exhaustive proof over small alphabets that the reference's serial algorithms (b) compute
the brute-force rule (a) as a multiset, a seeded random sweep with heavy ties, and the binding's argument checks."""
import itertools
import json
import math
import os
import random

import pytest

import ie_join_oracle as io
from test_cabi_cpu import declared_symbols

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N, NAN, INF = None, math.nan, math.inf
FLOATS = [N, -1.0, -0.0, 0.0, 1.0, 2.0, INF, -INF, NAN]
INTS = [N, -1, 0, 1, 2]
HOWS = ("inner", "left")


def ie_kats():
    with open(os.path.join(ROOT, "tests", "golden", "ie_join_kats.json")) as f:
        return json.load(f)["ie_join"]


def same(a, b):
    return io.as_multiset(a) == io.as_multiset(b)


@pytest.mark.parametrize("k", ie_kats(), ids=lambda k: k["cite"].split("(")[-1].rstrip(")"))
def test_oracle_reproduces_known_answers(k):
    exp = [tuple(p) for p in k["expect"]]
    assert same(io.brute(k["left"], k["right"], k["ops"], k["how"]), exp)
    assert same(io.serial(k["left"], k["right"], k["ops"], k["how"]), exp)


def sides(alphabet, max_len):
    for n in range(max_len + 1):
        yield from (list(t) for t in itertools.product(alphabet, repeat=n))


@pytest.mark.parametrize("alphabet,max_len", [(FLOATS, 2), (INTS, 3)], ids=["float", "int32"])
def test_serial_equals_rule_one_predicate(alphabet, max_len):
    for L in sides(alphabet, max_len):
        for R in sides(alphabet, max_len):
            for op in io.OPS:
                for how in HOWS:
                    assert same(io.serial([L], [R], [op], how), io.brute([L], [R], [op], how)), (L, R, op, how)


# two predicates: every row is an (x, y) pair; x over a float alphabet with NaN and +-0, y over a smaller one, all pairs of
# sides with at most three rows in total
ROWS_F = list(itertools.product([N, -0.0, 0.0, 1.0, NAN], [N, 0.0, 1.0, NAN]))
ROWS_I = list(itertools.product([N, 0, 1, 2], [N, 0, 1]))


@pytest.mark.parametrize("rows", [ROWS_F, ROWS_I], ids=["float", "int32"])
@pytest.mark.parametrize("op1", io.OPS)
def test_serial_equals_rule_two_predicates(rows, op1):
    for nl, nr in ((0, 1), (1, 0), (1, 1), (1, 2), (2, 1)):
        for Ls in itertools.product(rows, repeat=nl):
            for Rs in itertools.product(rows, repeat=nr):
                left = [[r[0] for r in Ls], [r[1] for r in Ls]]
                right = [[r[0] for r in Rs], [r[1] for r in Rs]]
                for op2 in io.OPS:
                    for how in HOWS:
                        assert same(io.serial(left, right, [op1, op2], how), io.brute(left, right, [op1, op2], how)), (left, right, op1, op2, how)


def test_random_sweep_heavy_ties():
    rnd = random.Random(20261015)
    for _ in range(300):
        alpha = rnd.choice([[N, 0, 1, 2], [N, -0.0, 0.0, 1.0, NAN, INF], [0, 1]])
        nl, nr = rnd.randint(0, 12), rnd.randint(0, 12)
        k = rnd.choice([1, 2])
        left = [[rnd.choice(alpha) for _ in range(nl)] for _ in range(k)]
        right = [[rnd.choice(alpha) for _ in range(nr)] for _ in range(k)]
        ops = [rnd.choice(io.OPS) for _ in range(k)]
        for how in ("inner", "left", "right"):
            assert same(io.serial(left, right, ops, how), io.brute(left, right, ops, how)), (left, right, ops, how)


def test_symbol_declared():
    assert "bl_ie_join" in declared_symbols()


def test_binding_rejects_bad_arguments():
    import numpy as np
    import polars_b200 as plb
    a = np.arange(3, dtype=np.int64)
    bad = [
        dict(ops="=="),
        dict(ops=["<", "<"]),                              # two operators for one predicate
        dict(left_on=[a, a, a], right_on=[a, a, a], ops=["<", "<", "<"]),
        dict(left_on=[a, a], right_on=[a], ops=["<", "<"]),
        dict(how="full"),
        dict(how="semi"),
        dict(how="cross"),
    ]
    for kw in bad:
        args = dict(left_on=a, right_on=a, ops="<", how="inner")
        args.update(kw)
        with pytest.raises(ValueError):
            plb.ie_join(args["left_on"], args["right_on"], args["ops"], args["how"])
