#!/usr/bin/env python3
"""Transcribe the reference's known answers of the type I/O into tests/golden/text_io_kat.json.

    python tests/golden/make_text_io_kat.py

Every statement `SELECT '<literal>'::vector[(n)];` (halfvec, sparsevec) of test/expected/vector_type.out, halfvec.out
and sparsevec.out, with what the server printed: the output text, or the ERROR and DETAIL lines.  Errors of the typmod
input function (a modifier out of range) are marked "typmod_in": the batch calls refuse such a typmod as an argument.  Reads the reference
tree at PGV_REFERENCE (default /root/reference).
"""
import json
import os
import re

REF = os.environ.get("PGV_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "text_io_kat.json")
STMT = re.compile(r"^SELECT '((?:[^']|'')*)'::(vector|halfvec|sparsevec)(?:\((\d+)\))?;$")


def cases(path):
    lines = open(path).read().split("\n")
    out = []
    for i, line in enumerate(lines):
        m = STMT.match(line)
        if not m:
            continue
        lit, typ, tm = m.group(1).replace("''", "'"), m.group(2), m.group(3)
        case = {"type": typ, "literal": lit, "typmod": int(tm) if tm else -1, "source": f"{os.path.basename(path)}:{i + 1}"}
        nxt = lines[i + 1]
        if nxt.startswith("ERROR:  "):
            case["error"] = nxt[len("ERROR:  "):]
            case["detail"] = ""
            for follow in lines[i + 2:]:     # LINE 1: / caret lines may come before the DETAIL
                if not follow or follow.startswith("SELECT"):
                    break
                if follow.startswith("DETAIL:  "):
                    case["detail"] = follow[len("DETAIL:  "):]
            # a type modifier out of range fails in the typmod input function, before the input function runs
            case["typmod_in"] = case["error"].startswith("dimensions for type ")
        else:
            assert lines[i + 2].startswith("-") and lines[i + 4] == "(1 row)", (path, i)
            case["output"] = lines[i + 3].strip()
        out.append(case)
    return out


def main():
    allc = []
    for f in ("vector_type.out", "halfvec.out", "sparsevec.out"):
        allc += cases(os.path.join(REF, "test", "expected", f))
    with open(OUT, "w") as fh:
        json.dump({"cases": allc}, fh, indent=1)
        fh.write("\n")
    print(f"{len(allc)} cases -> {OUT}")


if __name__ == "__main__":
    main()
