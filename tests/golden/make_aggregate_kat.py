#!/usr/bin/env python3
"""Transcribe the reference's known answers for avg / sum of vector and halfvec into tests/golden/aggregate_kat.json.

    python tests/golden/make_aggregate_kat.py

Every case below is one statement of test/expected/vector_type.out:629-750 or halfvec.out:593-682 with its result,
written as data: a table of rows (a NULL row is group -1, unnest(ARRAY[]...) the empty table) or a call of a transition,
combine or final function on state-array literals (nested lists, None = NULL, [] = '{}', {"series": [a, b]} = the
float8 array a, a + 1, .., b).  Results are a list (the
vector), None (SQL NULL) or {"error": text}.  Where the reference tree is present (PGV_REFERENCE, default
/root/reference) the script checks that each statement is followed by that result in the .out file before writing.
The dimension-mismatch statements are recorded as not applicable: a table has one dimension.  The last entry is
test/t/018_aggregates.pl's sum(v::halfvec) over a three-participant Partial Aggregate.
"""
import json
import os

REF = os.environ.get("PGV_REFERENCE", "/root/reference")
OUT = os.path.dirname(os.path.abspath(__file__))

OVERFLOW = {"error": "value out of range: overflow"}
BIG = list(range(1, 16003))      # array_agg(n) FROM generate_series(1, 16002) n


def err(text):
    return {"error": text}


def cases_for(t):
    v = "vector" if t == "vector" else "halfvec"
    big = 3e38 if t == "vector" else 65504
    big_lit = "3e38" if t == "vector" else "65504"
    big_out = "[3e+38]" if t == "vector" else "[65504]"

    def st(f):
        return err(f"{f}: expected state array")
    table = [
        (f"SELECT avg(v) FROM unnest(ARRAY['[1,2,3]'::{v}, '[3,5,7]']) v;", "avg", [[1, 2, 3], [3, 5, 7]], [2, 3.5, 5], "[2,3.5,5]"),
        (f"SELECT avg(v) FROM unnest(ARRAY['[1,2,3]'::{v}, '[3,5,7]', NULL]) v;", "avg", [[1, 2, 3], [3, 5, 7], None], [2, 3.5, 5],
         "[2,3.5,5]"),
        (f"SELECT avg(v) FROM unnest(ARRAY[]::{v}[]) v;", "avg", [], None, ""),
        (f"SELECT avg(v) FROM unnest(ARRAY['[{big_lit}]'::{v}, '[{big_lit}]']) v;", "avg", [[big], [big]], [big], big_out),
        (f"SELECT sum(v) FROM unnest(ARRAY['[1,2,3]'::{v}, '[3,5,7]']) v;", "sum", [[1, 2, 3], [3, 5, 7]], [4, 7, 10], "[4,7,10]"),
        (f"SELECT sum(v) FROM unnest(ARRAY['[1,2,3]'::{v}, '[3,5,7]', NULL]) v;", "sum", [[1, 2, 3], [3, 5, 7], None], [4, 7, 10],
         "[4,7,10]"),
        (f"SELECT sum(v) FROM unnest(ARRAY[]::{v}[]) v;", "sum", [], None, ""),
        (f"SELECT sum(v) FROM unnest(ARRAY['[{big_lit}]'::{v}, '[{big_lit}]']) v;", "sum", [[big], [big]], OVERFLOW,
         "ERROR:  value out of range: overflow"),
    ]
    fa, fc = f"{v}_avg", f"{v}_accum"
    calls = [
        (f"SELECT {fa}('{{2,2,4,6}}');", fa, [[2, 2, 4, 6]], [1, 2, 3], "[1,2,3]"),
        (f"SELECT {fa}('{{0}}');", fa, [[0]], None, ""),
        (f"SELECT {fa}('{{1}}');", fa, [[1]], err(f"{v} must have at least 1 dimension"), None),
        (f"SELECT {fa}('{{{{2,2,4,6}}}}');", fa, [[[2, 2, 4, 6]]], st(fa), None),
        (f"SELECT {fa}('{{NULL,2,4,6}}');", fa, [[None, 2, 4, 6]], st(fa), None),
        (f"SELECT {fa}('{{}}');", fa, [[]], st(fa), None),
        (f"SELECT {fa}(array_agg(n)) FROM generate_series(1, 16002) n;", fa, [BIG], err(f"{v} cannot have more than 16000 dimensions"),
         None),
        (f"SELECT {fc}('{{0}}', '[1,2,3]');", fc, [[0], [1, 2, 3]], [1, 1, 2, 3], "{1,1,2,3}"),
        (f"SELECT {fc}('{{0,0,0,0}}', '[1,2,3]');", fc, [[0, 0, 0, 0], [1, 2, 3]], [1, 1, 2, 3], "{1,1,2,3}"),
        (f"SELECT {fc}('{{{{0}}}}', '[1,2,3]');", fc, [[[0]], [1, 2, 3]], st(fc), None),
        (f"SELECT {fc}('{{NULL}}', '[1,2,3]');", fc, [[None], [1, 2, 3]], st(fc), None),
        (f"SELECT {fc}('{{}}', '[1,2,3]');", fc, [[], [1, 2, 3]], st(fc), None),
        (f"SELECT {fc}('{{0,0}}', '[1,2,3]');", fc, [[0, 0], [1, 2, 3]], err("expected 1 dimensions, not 3"), None),
    ]
    if t == "vector":
        fm = "vector_combine"
        calls += [
            ("SELECT vector_combine('{1,2}', '{3,4}');", fm, [[1, 2], [3, 4]], [4, 6], "{4,6}"),
            ("SELECT vector_combine('{1,2}', '{3,4,5}');", fm, [[1, 2], [3, 4, 5]], err("expected 1 dimensions, not 2"), None),
            ("SELECT vector_combine('{{1,2}}', '{3,4}');", fm, [[[1, 2]], [3, 4]], st(fm), None),
            ("SELECT vector_combine('{1,2}', '{{3,4}}');", fm, [[1, 2], [[3, 4]]], st(fm), None),
            ("SELECT vector_combine('{NULL,2}', '{3,4}');", fm, [[None, 2], [3, 4]], st(fm), None),
            ("SELECT vector_combine('{1,2}', '{3,NULL}');", fm, [[1, 2], [3, None]], st(fm), None),
            ("SELECT vector_combine('{}', '{0}');", fm, [[], [0]], st(fm), None),
            ("SELECT vector_combine('{0}', '{}');", fm, [[0], []], st(fm), None),
            ("SELECT vector_combine('{0}', '{0}');", fm, [[0], [0]], [0], "{0}"),
            ("SELECT vector_combine('{0}', (SELECT array_agg(n) FROM generate_series(1, 16002) n));", fm, [[0], BIG],
             err("vector cannot have more than 16000 dimensions"), None),
            ("SELECT vector_combine((SELECT array_agg(n) FROM generate_series(1, 16002) n), '{0}');", fm, [BIG, [0]],
             err("vector cannot have more than 16000 dimensions"), None),
            ("SELECT vector_combine((SELECT array_agg(n) FROM generate_series(1, 16002) n), (SELECT array_agg(n) FROM "
             "generate_series(1, 16002) n));", fm, [BIG, BIG], err("vector cannot have more than 16000 dimensions"), None),
        ]
    na = [
        (f"SELECT avg(v) FROM unnest(ARRAY['[1,2]'::{v}, '[3]']) v;", "ERROR:  expected 2 dimensions, not 1"),
        (f"SELECT sum(v) FROM unnest(ARRAY['[1,2]'::{v}, '[3]']) v;", f"ERROR:  different {v} dimensions 2 and 1"),
    ]
    return table, calls, na


def check_in_out(out_text, stmt, shown):
    i = out_text.find(stmt + "\n")
    assert i >= 0, stmt
    tail = out_text[i + len(stmt) + 1:].split("\n")
    if shown is None:            # an error: the next line
        return tail[0]
    if shown.startswith("ERROR"):
        assert tail[0] == shown, (stmt, tail[0])
        return
    assert tail[2].strip() == shown, (stmt, tail[:3])


def main():
    kat = {"source": "test/expected/vector_type.out:629-750, test/expected/halfvec.out:593-682, test/t/018_aggregates.pl",
           "table": [], "calls": [], "not_applicable": []}
    for t, fname in (("vector", "vector_type.out"), ("halfvec", "halfvec.out")):
        path = os.path.join(REF, "test", "expected", fname)
        text = open(path).read() if os.path.exists(path) else None
        table, calls, na = cases_for(t)
        for stmt, agg, rows, want, shown in table:
            if text is not None:
                check_in_out(text, stmt, shown)
            groups = [-1 if r is None else 0 for r in rows]
            dim = 3 if not rows else len(next(r for r in rows if r is not None))
            kat["table"].append({"type": t, "statement": stmt, "agg": agg, "dim": dim,
                                 "rows": [r if r is not None else [0] * dim for r in rows], "groups": groups, "expect": want})
        for stmt, fn, args, want, shown in calls:
            if text is not None:
                line = check_in_out(text, stmt, shown)
                if isinstance(want, dict):
                    assert line == "ERROR:  " + want["error"], (stmt, line)
            args = [{"series": [1, 16002]} if a is BIG else a for a in args]   # array_agg(n) of generate_series, kept short
            kat["calls"].append({"type": t, "statement": stmt, "function": fn, "args": args, "expect": want})
        for stmt, shown in na:
            if text is not None:
                check_in_out(text, stmt, shown)
            kat["not_applicable"].append({"type": t, "statement": stmt, "reference": shown[len("ERROR:  "):],
                                          "why": "a table has one dimension"})
    kat["partial_aggregate_018"] = {
        "statement": "SELECT sum(v::halfvec) FROM tst;  -- 1M rows [random() + 1.01, random() + 2.01, random() + 3.01], "
                     "Partial Aggregate over 3 participants",
        "rows": 1000000, "participants": 3, "expect": [24576, 24576, 49152]}
    with open(os.path.join(OUT, "aggregate_kat.json"), "w") as f:
        json.dump(kat, f, indent=1)
        f.write("\n")


if __name__ == "__main__":
    main()
