"""Writes tests/golden/string_match_kats.json: known answers of the reference's string predicate tests, transcribed by
hand with the file:line of each case (paths relative to the reference's repository root).

Every case has a column `col` (str / None), an `op` and the expected Booleans (None = null):
  "like"         SQL `col LIKE pattern` (negate: NOT LIKE); the reference's polars-sql builds ^(?s)...$ (sql_expr.rs:435-479)
  "contains"     str.contains(pattern, literal=True) on the bytes; `pattern` is a str / None scalar or a per-row list
  "regex"        str.contains(pattern, literal=False): a regex of the device subset; expected None for the whole case
                 means the device must refuse it (status 4) and the caller falls back
  "starts_with" / "ends_with"   with a scalar (str / None) or a per-row list

Not transcribed: the ILIKE / `~~*` rows of test_string_like (:214, :216, :218, :223, :226, :227; case folding is out of
scope), the ILIKE half of test_string_like_multiline (:261, :268), the regex column of test_contains_expr (:1120-1124: a
per-row regex is refused as a whole, checked by tests/test_string_match.py), the ShapeError of test_str_contains_wrong_length
(:257-260: a length check, covered by the argument-error tests) and the non-strict null output for an invalid regex
(:1061-1064: the device refuses every regex outside its subset, invalid or not)."""
import json
import os

SQL = "py-polars/tests/unit/sql/test_strings.py"
STR = "py-polars/tests/unit/operations/namespaces/string/test_string.py"

TXT = ["ABC", "abc", "000", "A[0]*C", "a0c?"]
LIKE_TABLE = [      # (line, pattern, operator, matching idx) of test_string_like (:210-231)
    (213, "a%", "LIKE", [1, 4]), (215, "ab%", "LIKE", [1]), (217, "ab_", "LIKE", [1]), (219, "_0%_", "LIKE", [2, 4]),
    (220, "%0", "LIKE", [2]), (221, "0%", "LIKE", [2]), (222, "__0%", "~~", [2, 3]),
    (224, "____", "~~", [4]), (225, "a%C", "~~", []), (228, "a0c?", "~~", [4]), (229, "000", "~~", [2]), (230, "00", "~~", []),
]

CASES = []
for line, pat, op, idx in LIKE_TABLE:
    hit = [i in idx for i in range(len(TXT))]
    CASES.append(dict(src=f"{SQL}:{line}", op="like", col=TXT, pattern=pat, negate=False, expected=hit))
    CASES.append(dict(src=f"{SQL}:{line},241-249", op="like", col=TXT, pattern=pat, negate=True, expected=[not h for h in hit]))

S1, S2, S3 = "Hello World", "Hello\nWorld", "hello\nWORLD"
ML = [S1, S2, S3]
CASES += [
    dict(src=f"{SQL}:260,263", op="like", col=ML, pattern="Hello%", negate=False, expected=[True, True, False]),
    dict(src=f"{SQL}:267,270", op="like", col=ML, pattern="%WORLD", negate=False, expected=[False, False, True]),
]
for s in ML:      # test_string_like_multiline exact matches (:274-275)
    CASES.append(dict(src=f"{SQL}:274-275", op="like", col=ML, pattern=s, negate=False, expected=[t == s for t in ML]))

CASES.append(dict(src=f"{STR}:251-254", op="regex", col=["messi", "ronaldo", "ibrahimovic"], pattern="mes", expected=[True, False, False]))
T123 = ["123", "456", "789"]
CASES += [
    dict(src=f"{STR}:1065-1066", op="regex", col=T123, pattern="(not_valid_regex", expected=None),
    dict(src=f"{STR}:1067-1070", op="regex", col=T123, pattern="1", expected=[True, False, False]),
]
TEXT = ["some * * text", "(with) special\n * chars", "**etc...?$"]
for line, pat, literal, exp in [
    (1078, r"\* \*", False, [True, False, False]), (1079, r"* *", True, [True, False, False]),
    (1080, r"^\(", False, [False, True, False]), (1081, r"^\(", True, [False, False, False]),
    (1082, r"(", True, [False, True, False]), (1083, r"e", False, [True, True, True]),
    (1084, r"e", True, [True, True, True]), (1085, r"^\S+$", False, None),
    (1086, r"\?\$", False, [False, False, True]), (1087, r"?$", True, [False, False, True]),
]:
    CASES.append(dict(src=f"{STR}:{line}", op="contains" if literal else "regex", col=TEXT, pattern=pat, expected=exp))
CASES.append(dict(src=f"{STR}:1107-1131", op="contains", col=["some text", "(with) special\n .* chars", "**etc...?$", None, "b", "invalid_regex"],
                  pattern=[r"[me]", r".*", r"^\(", "a", None, "*"], expected=[False, True, False, None, None, False]))

A = ["hamburger_with_tomatoes", "nuts", "lollypop", None]
SUB = ["ham", "ts", None, "anything"]
CASES += [
    dict(src=f"{STR}:1665,1672", op="ends_with", col=A, pattern="pop", expected=[False, False, True, None]),
    dict(src=f"{STR}:1666,1673", op="ends_with", col=A, pattern=None, expected=[None, None, None, None]),
    dict(src=f"{STR}:1667,1674", op="ends_with", col=A, pattern=SUB, expected=[False, True, None, None]),
    dict(src=f"{STR}:1668,1675", op="starts_with", col=A, pattern="ham", expected=[True, False, False, None]),
    dict(src=f"{STR}:1669,1676", op="starts_with", col=A, pattern=None, expected=[None, None, None, None]),
    dict(src=f"{STR}:1670,1677", op="starts_with", col=A, pattern=SUB, expected=[True, False, None, None]),
]


if __name__ == "__main__":
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "string_match_kats.json")
    with open(path, "w") as f:
        f.write("[\n" + ",\n".join(json.dumps(c) for c in CASES) + "\n]\n")
    print(f"wrote {len(CASES)} cases to {path}")
