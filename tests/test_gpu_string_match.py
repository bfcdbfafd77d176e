"""GPU tests of the string predicates (string_match.cu: k_str_rows, the byte-parallel contains plan k_str_tile_rows /
k_str_scan / k_str_scan_finish) and of bl_string_filter (op_mask_rows + op_string_gather).

Every result must equal the oracle (tests/string_match_oracle.py, which tests/test_string_match.py checks) exactly,
values and validity.  Each input is run in three forms: one host chunk, three host chunks, and one caller-owned device
chunk that is a slice of a longer column (Arrow offset 5, so its first offset is not 0 and its validity starts at bit 5),
which the library reads in place.

Caps.  SM = device_info()["sm_count"].  k_str_rows runs grid_for(.., 16 per SM) CTAs of 256 threads, one row per thread:
N_BIG = 3 * 16 * SM * 256 + 77 rows pass its grid-stride loop three times with a ragged tail.  k_str_scan runs 8 CTAs
per SM over 8 KB tiles; the N_BIG rows of about 100 bytes span several grid strides of tiles.  The contains plan rule is
the average row length (64 bytes); BL_STR_SCAN_MIN_ROW moves it so that both plans run on the same inputs."""
import ctypes as C
import random

import numpy as np
import pytest

import string_match_oracle as so
from test_string_match import KATS, mapped_oracle

pytestmark = pytest.mark.gpu

INVALID, UNSUPPORTED, DTYPE = 1, 4, 5
PREFIX = [b"p0", None, b"", b"prefix-3", b"p4"]      # the rows a sliced device chunk hides before its own


@pytest.fixture(scope="module")
def plb():
    import polars_b200 as m
    m.init()
    return m


@pytest.fixture(scope="module")
def sm(plb):
    return plb.device_info()["sm_count"]


class DevChunk:
    """a caller-owned device string chunk: rows `vals` as the slice [len(prefix), ...) of prefix + vals"""

    def __init__(self, plb, vals, prefix=PREFIX):
        allv = list(prefix) + list(vals)
        sc = plb.StringColumn(allv)
        self.plb, self.ptrs = plb, []

        def up(a: np.ndarray) -> int:
            p = plb.dev_alloc(max(a.nbytes, 1))
            self.ptrs.append(p)
            if a.nbytes:
                plb._check(plb.lib().bl_memcpy_h2d(C.c_void_p(p), a.ctypes.data_as(C.c_void_p), C.c_size_t(a.nbytes)))
            return p
        data = sc.data[: int(sc.offsets[-1])]
        # exactly the bytes the offsets name: a kernel that reads past them reads past the allocation
        po, pd = up(sc.offsets), up(np.ascontiguousarray(data))
        pv = up(sc.bits) if sc.bits is not None else None
        self.st = plb.BlStringColumn(plb.DEVICE, 0, len(vals), len(prefix), -1 if pv else 0, po, pd, pv, None)
        self.length = len(vals)

    def struct(self):
        return self.st

    def free(self):
        for p in self.ptrs:
            self.plb.dev_free(p)
        self.ptrs = []

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def forms(plb, vals):
    """(name, column) for one host chunk, three host chunks and a sliced device chunk"""
    out = [("host", plb.StringColumn(vals))]
    if len(vals) >= 3:
        k = len(vals) // 3
        out.append(("chunks", [plb.StringColumn(vals[:k]), plb.StringColumn(vals[k:2 * k]), plb.StringColumn(vals[2 * k:])]))
    out.append(("device", DevChunk(plb, vals)))
    return out


def as_list(res):
    vals, valid = res
    return [None if valid is not None and not valid[i] else bool(vals[i]) for i in range(len(vals))]


def profiled(plb, fn):
    plb.profile_reset()
    plb.profile_enable(True)
    try:
        out = fn()
        plb.sync()
        prof = plb.profile()
    finally:
        plb.profile_enable(False)
    return out, {k: int(v.get("launches", 0)) for k, v in prof.items()}


def check_all(plb, vals, pattern, monkeypatch, kinds=("contains", "starts_with", "ends_with")):
    """each kind over every input form, the contains plans both ways, against the oracle"""
    for name, col in forms(plb, vals):
        for kind in kinds:
            want = getattr(so, kind)(vals, pattern)
            fn = {"contains": lambda: plb.str_contains(col, pattern, literal=True), "starts_with": lambda: plb.str_starts_with(col, pattern),
                  "ends_with": lambda: plb.str_ends_with(col, pattern)}[kind]
            for rule in (("0", "1e18") if kind == "contains" else (None,)):
                if rule is not None:
                    monkeypatch.setenv("BL_STR_SCAN_MIN_ROW", rule)
                assert as_list(fn()) == want, (name, kind, pattern, rule)
        monkeypatch.delenv("BL_STR_SCAN_MIN_ROW", raising=False)


EDGE = [b"", b"green", b"gree", b"xgreen", b"greenx", b"xxgre", b"enxx", b"greengreen", None, b"\x00green\xff", b"\xff\xff",
        b"\x00", b"g", b"n", b"reen", b"a" * 40 + b"green", b"green" + b"b" * 40, None, b"grEen"]


@pytest.mark.parametrize("pattern", [b"", b"g", b"green", b"greengreen", b"greengreenx", b"\x00", b"\xff\xff", b"en", b"a" * 41])
def test_edges_every_form(plb, monkeypatch, pattern):
    """empty rows and pattern, needles longer than / equal to the row, at its start and end, and straddling two rows
    (b"xxgre" + b"enxx" hold "green" only across their boundary), NUL and 0xFF bytes"""
    check_all(plb, EDGE, pattern, monkeypatch)


def test_known_answers(plb):
    for case in KATS:
        for name, col in forms(plb, case["col"]):
            op, pat = case["op"], case["pattern"]
            per_row = isinstance(pat, list)
            p = (plb.StringColumn(pat) if name != "device" else DevChunk(plb, pat)) if per_row else pat
            if op == "like":
                got = plb.str_like(col, pat, negate=case["negate"])
            elif op == "contains":
                got = plb.str_contains(col, p, literal=True)
            elif op == "starts_with":
                got = plb.str_starts_with(col, p)
            elif op == "ends_with":
                got = plb.str_ends_with(col, p)
            else:
                if case["expected"] is None:
                    with pytest.raises(plb.B200Error) as e:
                        plb.str_contains(col, pat)
                    assert e.value.status == UNSUPPORTED
                    continue
                got = plb.str_contains(col, pat)
            assert as_list(got) == case["expected"], (case["src"], name)


LIKE_ROWS = ["", "a", "é", "😀", "€", "ab", "a\nb", "a\n", "\n", "a%b", "a_b", "a\\b", "aé€😀b", "abcabc", "x" * 70 + "y", None, "%", "_",
             "special requests", "special\nrequests", "xx special yy requests zz", "Customer Complaints", "\x00", "a\x00b"]
LIKE_PATTERNS = [("", None), ("%", None), ("_", None), ("__", None), ("a%", None), ("%b", None), ("a_b", None), ("a%b", None), ("%a%", None),
                 ("_é_", None), ("a___b", None), ("%😀%", None), ("a\\%b", "\\"), ("a\\_b", "\\"), ("a\\\\b", "\\"), ("a!%b", "!"),
                 ("%special%requests%", None), ("x%y", None), ("%_%_%", None), ("a_\x00%", None), ("a" + "_" * 62, None),
                 ("%" + "x" * 63, None)]


@pytest.mark.parametrize("pattern,escape", LIKE_PATTERNS)
def test_like_every_form(plb, pattern, escape):
    """'_' over 2-, 3- and 4-byte UTF-8, '\\n' with and without NO_NEWLINE, NOT, escapes, the 63-state limit"""
    for name, col in forms(plb, LIKE_ROWS):
        for nn in (False, True):
            for neg in (False, True):
                want = so.like(LIKE_ROWS, pattern, negate=neg, no_newline=nn, escape=escape)
                got = plb.str_like(col, pattern, negate=neg, no_newline=nn, escape=escape)
                assert as_list(got) == want, (name, pattern, nn, neg)


@pytest.mark.parametrize("regex", ["special.*requests", ".*Customer.*Complaints.*", "^a.b$", "(?s)^a.b$", "a$", "^$", "é.", r"a\\b", "(?s)a.*b",
                                   "^x", "b$", "%", "_.%", "_"])
def test_regex_subset_on_device(plb, regex):
    kind, p, flags, esc = plb.regex_to_device(regex)
    want = mapped_oracle(LIKE_ROWS, kind, p, flags, esc)
    assert want == so.regex_search(LIKE_ROWS, regex)
    for name, col in forms(plb, LIKE_ROWS):
        assert as_list(plb.str_contains(col, regex)) == want, (name, regex)


CMP_ROWS = [b"", b"a", b"a\x00", b"b", b"abcdefgh", b"abcdefgh\x00", b"abcdefghi", b"abcdefghij", b"abcdefgh" * 3, b"abcdefgh" * 3 + b"\xff",
            b"\xff", b"\xff" * 9, None, b"abcdefgi", b"abcdefg", None]


@pytest.mark.parametrize("scalar", [b"", b"a", b"a\x00", b"abcdefgh", b"abcdefghi", b"abcdefgh" * 3, b"\xff" * 9, None])
def test_compare_scalar(plb, scalar):
    """prefix ties beyond 8 bytes, a proper prefix first, NUL and 0xFF, missing, a null scalar"""
    for name, col in forms(plb, CMP_ROWS):
        for op in so.CMPS:
            assert as_list(plb.str_compare(op, col, scalar)) == so.compare(op, CMP_ROWS, scalar), (name, op, scalar)
        for op in ("eq", "ne"):
            assert as_list(plb.str_compare(op, col, scalar, missing=True)) == so.compare(op, CMP_ROWS, scalar, missing=True), (name, op)


def test_compare_columns_and_per_row_patterns(plb):
    rng = random.Random(1)
    other = [None if rng.random() < 0.2 else rng.choice([v for v in CMP_ROWS if v is not None]) for _ in CMP_ROWS]
    pats = [None if rng.random() < 0.2 else rng.choice([b"", b"a", b"ab", b"abcdefgh", b"\xff"]) for _ in CMP_ROWS]
    for (name, col), (_, oc), (_, pc) in zip(forms(plb, CMP_ROWS), forms(plb, other), forms(plb, pats)):
        for op in so.CMPS:
            assert as_list(plb.str_compare(op, col, oc)) == so.compare(op, CMP_ROWS, other), (name, op)
        for op in ("eq", "ne"):
            assert as_list(plb.str_compare(op, col, oc, missing=True)) == so.compare(op, CMP_ROWS, other, missing=True)
        assert as_list(plb.str_contains(col, pc, literal=True)) == so.contains(CMP_ROWS, pats), name
        assert as_list(plb.str_starts_with(col, pc)) == so.starts_with(CMP_ROWS, pats), name
        assert as_list(plb.str_ends_with(col, pc)) == so.ends_with(CMP_ROWS, pats), name


def rand_rows(rng, n, mean_len, alphabet=b"abgrenx\x00\xff", null_p=0.05):
    lens = rng.integers(0, 2 * mean_len + 1, size=n)
    data = rng.choice(np.frombuffer(alphabet, np.uint8), size=int(lens.sum()))
    offs = np.zeros(n + 1, np.int64)
    np.cumsum(lens, out=offs[1:])
    valid = rng.random(n) >= null_p
    rows = [bytes(data[offs[i]:offs[i + 1]]) if valid[i] else None for i in range(n)]
    return rows


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33])
def test_small_sizes(plb, monkeypatch, n):
    rows = rand_rows(np.random.default_rng(n), n, 5)
    check_all(plb, rows, b"gr", monkeypatch)
    text = rand_rows(np.random.default_rng(n + 100), n, 5, alphabet=b"abgren\n")      # LIKE reads UTF-8
    for (name, col), (_, tcol) in zip(forms(plb, rows), forms(plb, text)):
        assert as_list(plb.str_like(tcol, "%g_e%")) == so.like(text, "%g_e%"), name
        assert as_list(plb.str_compare("lt", col, b"gr")) == so.compare("lt", rows, b"gr"), name


def test_past_the_grids(plb, sm, monkeypatch):
    """N_BIG rows of about 100 bytes (k_str_rows' grid three times over, many tile strides of k_str_scan), ragged tail"""
    n = 3 * 16 * sm * 256 + 77
    rng = np.random.default_rng(9)
    rows = rand_rows(rng, n, 50, alphabet=b"abgren")
    col = DevChunk(plb, rows)
    for needle in (b"green", b"ab", b"r"):
        want = so.contains(rows, needle)
        for rule, kernel in (("0", "str_scan"), ("1e18", "str_contains_rows")):
            monkeypatch.setenv("BL_STR_SCAN_MIN_ROW", rule)
            got, prof = profiled(plb, lambda: plb.str_contains(col, needle, literal=True))
            assert kernel in prof and "str_rebase" not in prof, prof
            assert as_list(got) == want, (needle, rule)
        monkeypatch.delenv("BL_STR_SCAN_MIN_ROW")
        assert as_list(plb.str_starts_with(col, needle)) == so.starts_with(rows, needle)
        assert as_list(plb.str_ends_with(col, needle)) == so.ends_with(rows, needle)
        assert as_list(plb.str_compare("ge", col, needle)) == so.compare("ge", rows, needle)
    col.free()
    # LIKE over rows drawn from a few distinct values, so that the recursive oracle runs once per value
    distinct = [None] + [bytes(rng.choice(np.frombuffer(b"abgren\n", np.uint8), size=rng.integers(0, 30))) for _ in range(300)]
    pick = rng.integers(0, len(distinct), size=n)
    rows = [distinct[i] for i in pick]
    col = DevChunk(plb, rows)
    for pat in ("%gr_en%", "a%b", "%e\n%"):
        for nn in (False, True):
            per = so.like(distinct, pat, no_newline=nn)
            assert as_list(plb.str_like(col, pat, no_newline=nn)) == [per[i] for i in pick], (pat, nn)


def test_tile_edges_and_long_rows(plb, monkeypatch):
    """rows across 8 KB tile edges and longer than a tile, needles across a tile edge, at row starts and ends"""
    rng = np.random.default_rng(4)
    rows = []
    for ln in (8190, 8191, 8192, 8193, 3, 20000, 16384, 5, 40000):
        r = bytearray(rng.choice(np.frombuffer(b"abc", np.uint8), size=ln).tobytes())
        rows.append(bytes(r))
    base = list(rows)
    for at in (0, 8188, 8190, 8191, 16380, 19995):      # plant the needle at these positions of the 20000-byte row
        r = bytearray(base[5])
        r[at:at + 5] = b"green"
        rows.append(bytes(r))
    rows += [b"gre", b"en" + b"x" * 9000, b"green"]
    for needle in (b"green", b"c", b"abcab", bytes(rows[5][100:400])):
        check_all(plb, rows, needle, monkeypatch, kinds=("contains",))


def test_long_needles(plb, monkeypatch):
    """needles past the scan halo (512) and past the shared-memory staging (16 KB), up to 64 KB"""
    rng = np.random.default_rng(2)
    big = rng.choice(np.frombuffer(b"ab", np.uint8), size=70000).tobytes()
    rows = [big, big[:65536], big[1:65537], big[:600], None, b"", big[-65536:]]
    for m in (511, 512, 513, 16384, 16385, 65536):
        for needle in (big[:m], big[1:m + 1], big[-m:]):
            check_all(plb, rows, needle, monkeypatch)


def test_nulls_scalars_and_profile(plb):
    rows = [b"a", None, b"b", b"ab", None] * 7
    for name, col in forms(plb, rows):
        for fn in (plb.str_starts_with, plb.str_ends_with, lambda c, p: plb.str_contains(c, p, literal=True)):
            assert as_list(fn(col, None)) == [None] * len(rows), name
        assert as_list(plb.str_like(col, None)) == [None] * len(rows)
        assert as_list(plb.str_compare("lt", col, None)) == [None] * len(rows)
    col = DevChunk(plb, rows)
    for fn in (lambda: plb.str_contains(col, b"a", literal=True), lambda: plb.str_like(col, "a%"), lambda: plb.str_compare("eq", col, b"a"),
               lambda: plb.str_starts_with(col, b"a")):
        _, prof = profiled(plb, fn)
        assert "str_rebase" not in prof, prof      # the single device chunk is read in place
    host = plb.StringColumn(rows)
    _, prof = profiled(plb, lambda: plb.str_starts_with(host, b"a"))
    assert prof.get("str_rebase", 0) >= 1 and prof.get("str_starts", 0) == 1, prof


def test_plan_rule(plb):
    """average row length below 64 bytes: the per-row plan; from 64: the byte-parallel plan; a needle past the halo: per-row"""
    short = [b"x" * 30 + b"green"] * 1000
    long_ = [b"x" * 80 + b"green"] * 1000
    for rows, kernel in ((short, "str_contains_rows"), (long_, "str_scan")):
        col = DevChunk(plb, rows)
        got, prof = profiled(plb, lambda: plb.str_contains(col, b"green", literal=True))
        assert prof.get(kernel, 0) == 1 and as_list(got) == [True] * 1000, prof
    col = DevChunk(plb, long_)
    _, prof = profiled(plb, lambda: plb.str_contains(col, b"x" * 513, literal=True))
    assert "str_scan" not in prof and prof.get("str_contains_rows", 0) == 1, prof


@pytest.mark.parametrize("kind", ["random", "none", "all", "nulls"])
def test_filter(plb, kind):
    rng = np.random.default_rng(8)
    rows = rand_rows(rng, 5000, 12)
    mask = {"random": rng.random(5000) < 0.1, "none": np.zeros(5000, bool), "all": np.ones(5000, bool), "nulls": rng.random(5000) < 0.5}[kind]
    mvalid = rng.random(5000) < 0.7 if kind == "nulls" else None
    eff = mask & (mvalid if mvalid is not None else True)
    want = so.filter_rows(rows, eff)
    for name, col in forms(plb, rows):
        m = (mask, mvalid) if mvalid is not None else mask
        assert plb.str_filter(col, m) == want, name
        dev = plb.str_filter(col, m, location=plb.DEVICE)
        assert dev.length == len(want)
        assert plb.string_gather(dev, np.arange(len(want), dtype=np.uint32)) == want, name
    # a mask produced on the device, without leaving it
    col = DevChunk(plb, rows)
    pm = plb.str_contains(col, b"gr", literal=True, location=plb.DEVICE)
    assert plb.str_filter(col, pm) == so.filter_rows(rows, [bool(x) for x in so.contains(rows, b"gr")])


def test_errors(plb):
    col = plb.StringColumn([b"a", b"b", b"c"])
    two = plb.StringColumn([b"a", b"b"])
    cases = [
        (lambda: plb.str_compare("eq", col, two), INVALID),
        (lambda: plb.str_contains(col, two, literal=True), INVALID),
        (lambda: plb.str_like(col, "a\\b", escape="\\"), INVALID),
        (lambda: plb.str_like(col, "a\\", escape="\\"), INVALID),
        (lambda: plb.str_like(col, "x" * 64), UNSUPPORTED),
        (lambda: plb.str_like(col, "_" * 64), UNSUPPORTED),
        (lambda: plb.str_filter(col, np.array([True, False])), INVALID),
        (lambda: plb.str_filter(col, np.array([1, 0, 1], np.int32)), DTYPE),
        (lambda: plb._str_match("like", col, plb.StringColumn([b"a", b"b", b"c"])), INVALID),
        (lambda: plb._str_match("contains", col, b"a", flags=plb.LIKE_NO_NEWLINE), INVALID),
        (lambda: plb._str_match("contains", col, b"a", escape="\\"), INVALID),
        (lambda: plb._str_match("contains", col, b"a", flags=64), INVALID),
        (lambda: plb.str_compare("lt", col, b"a", missing=True), INVALID),
    ]
    for fn, st in cases:
        with pytest.raises(plb.B200Error) as e:
            fn()
        assert e.value.status == st, e.value
    out = plb.BlColumn()
    arr = (plb.BlStringColumn * 1)(col.struct())
    assert plb.lib().bl_string_match(C.c_int32(9), 0, 0, arr, 1, arr, 1, plb.HOST, C.byref(out)) == INVALID
    assert plb.lib().bl_string_compare(C.c_int32(7), arr, 1, arr, 1, 0, plb.HOST, C.byref(out)) == INVALID
    assert as_list(plb.str_like(col, "x" * 63)) == [False] * 3 and as_list(plb.str_like(col, "%" * 200 + "a")) == [True, False, False]


def test_data_past_4_gib(plb, monkeypatch):
    """one device data buffer of more than 2^32 bytes: 32-bit positions would alias"""
    torch = pytest.importorskip("torch")
    W = 1024
    n = (1 << 32) // W + 4096                       # 4.3 GB
    data = torch.full((n * W,), ord("a"), dtype=torch.uint8, device="cuda")
    offs = torch.arange(n + 1, dtype=torch.int64, device="cuda") * W
    hits = {n - 1: 1000, n - 3: 0, n - 10: 500}      # row -> needle position inside the row
    for r, at in hits.items():
        data[r * W + at: r * W + at + 5] = torch.tensor(list(b"green"), dtype=torch.uint8, device="cuda")
    s = n - 20                                       # "green" across the boundary of rows s and s + 1: no row holds it
    data[s * W + W - 2: s * W + W + 3] = torch.tensor(list(b"green"), dtype=torch.uint8, device="cuda")
    assert (n - 20) * W > (1 << 32)
    torch.cuda.synchronize()
    st = plb.BlStringColumn(plb.DEVICE, 0, n, 0, 0, offs.data_ptr(), data.data_ptr(), None, None)
    col = plb.DeviceStringColumn(st=st)
    want = np.zeros(n, bool)
    want[list(hits)] = True
    for rule, kernel in (("0", "str_scan"), ("1e18", "str_contains_rows")):
        monkeypatch.setenv("BL_STR_SCAN_MIN_ROW", rule)
        (vals, valid), prof = profiled(plb, lambda: plb.str_contains(col, b"green", literal=True))
        assert kernel in prof and valid is None and np.array_equal(vals, want), rule
    monkeypatch.delenv("BL_STR_SCAN_MIN_ROW")
    vals, _ = plb.str_like(col, "%green%")
    assert np.array_equal(vals, want)
    vals, _ = plb.str_ends_with(col, b"green" + b"a" * 19)
    assert np.array_equal(np.flatnonzero(vals), [n - 1])
    vals, _ = plb.str_compare("gt", col, b"a" * W)
    assert np.array_equal(np.flatnonzero(vals), sorted([n - 20, n - 19, n - 10, n - 3, n - 1]))
    mask = np.zeros(n, bool)
    mask[[0, n - 1]] = True
    assert plb.str_filter(col, mask) == [b"a" * W, bytes(data[(n - 1) * W:n * W].cpu().numpy())]
    del col, data, offs
    torch.cuda.empty_cache()
