#!/usr/bin/env python3
"""Write the known answers of array_to_sparsevec to tests/golden/array_cast_kat.json.

    python tests/golden/make_array_cast_kat.py

Every array -> sparsevec case of test/expected/cast.out, and its numeric[] -> vector and -> halfvec cases, with the
answer the reference prints there: the vector / halfvec / sparsevec text or the errmsg.  The cases are found by their
SQL line in the reference tree at PGV_REFERENCE (default /root/reference).  numeric[] elements are written as their
decimal literals (ARRAY[1.0, ...] is numeric[] with dscale 1).  Left out: {NULL} and {{1}}, whose checks stay with the
caller that unpacks the ArrayType.
"""
import json
import os

REF = os.environ.get("PGV_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "array_cast_kat.json")
EXPECTED = "test/expected/cast.out"

# SQL -> (target type, source type, the array's elements as JSON values, typmod); for real[] and double precision[]
# "inf", "-inf", "nan" stand for the specials; numeric[] elements are decimal literals
NUMERIC = [
    ("SELECT ARRAY[1.0,2.0,3.0]::vector;", "vector", "numeric", ["1.0", "2.0", "3.0"], -1),
    ("SELECT ARRAY[1,2,3]::numeric[]::vector;", "vector", "numeric", ["1", "2", "3"], -1),
    ("SELECT ARRAY[1.0,2.0,3.0]::halfvec;", "halfvec", "numeric", ["1.0", "2.0", "3.0"], -1),
    ("SELECT ARRAY[1,2,3]::numeric[]::halfvec;", "halfvec", "numeric", ["1", "2", "3"], -1),
    ("SELECT ARRAY[1.0,0.0,2.0,0.0,3.0,0.0]::sparsevec;", "sparsevec", "numeric", ["1.0", "0.0", "2.0", "0.0", "3.0", "0.0"], -1),
    ("SELECT ARRAY[1,0,2,0,3,0]::numeric[]::sparsevec;", "sparsevec", "numeric", ["1", "0", "2", "0", "3", "0"], -1),
]
CASES = [
    ("SELECT ARRAY[1,0,2,0,3,0]::sparsevec;", "int4", [1, 0, 2, 0, 3, 0], -1),
    ("SELECT ARRAY[1,0,2,0,3,0]::real[]::sparsevec;", "float4", [1, 0, 2, 0, 3, 0], -1),
    ("SELECT ARRAY[1,0,2,0,3,0]::double precision[]::sparsevec;", "float8", [1, 0, 2, 0, 3, 0], -1),
    ("SELECT '{1,0,2,0,3,0}'::real[]::sparsevec;", "float4", [1, 0, 2, 0, 3, 0], -1),
    ("SELECT '{1,0,2,0,3,0}'::real[]::sparsevec(6);", "float4", [1, 0, 2, 0, 3, 0], 6),
    ("SELECT '{1,0,2,0,3,0}'::real[]::sparsevec(5);", "float4", [1, 0, 2, 0, 3, 0], 5),
    ("SELECT '{NaN}'::real[]::sparsevec;", "float4", ["nan"], -1),
    ("SELECT '{Infinity}'::real[]::sparsevec;", "float4", ["inf"], -1),
    ("SELECT '{-Infinity}'::real[]::sparsevec;", "float4", ["-inf"], -1),
    ("SELECT '{}'::real[]::sparsevec;", "float4", [], -1),
    ("SELECT '{1,0,2,0,3,0}'::double precision[]::sparsevec;", "float8", [1, 0, 2, 0, 3, 0], -1),
    ("SELECT '{1,0,2,0,3,0}'::double precision[]::sparsevec(6);", "float8", [1, 0, 2, 0, 3, 0], 6),
    ("SELECT '{1,0,2,0,3,0}'::double precision[]::sparsevec(5);", "float8", [1, 0, 2, 0, 3, 0], 5),
    ("SELECT '{4e38,-4e38}'::double precision[]::sparsevec;", "float8", [4e38, -4e38], -1),
    ("SELECT '{1e-46,-1e-46}'::double precision[]::sparsevec;", "float8", [1e-46, -1e-46], -1),
    ("SELECT array_agg(n)::sparsevec FROM generate_series(1, 16001) n;", "int4", {"range": [1, 16002]}, -1),
]


def answer(lines, i):
    """the reference's answer to the statement on line i: ("error", errmsg) or ("expected", the one result value)"""
    nxt = lines[i + 1]
    if nxt.startswith("ERROR:  "):
        return "error", nxt[len("ERROR:  "):].rstrip("\n")
    assert lines[i + 2].startswith("---"), lines[i + 2]
    assert lines[i + 4].startswith("(1 row)"), lines[i + 4]
    return "expected", lines[i + 3].strip()


def main():
    with open(os.path.join(REF, EXPECTED)) as f:
        lines = f.readlines()
    cases = []
    for sql, typ, src, elems, typmod in [(c[0], "sparsevec") + c[1:] for c in CASES] + NUMERIC:
        at = [i for i, line in enumerate(lines) if line.rstrip("\n") == sql]
        assert len(at) == 1, sql
        key, value = answer(lines, at[0])
        cases.append({"sql": sql, "source": f"{EXPECTED}:{at[0] + 1}", "type": typ, "src": src, "elems": elems, "typmod": typmod,
                      key: value})
    doc = {"source": "pgvector " + EXPECTED + ": the array to sparsevec section, the 16001-element case of the max "
                     "dimensions section, and the numeric[] -> vector / halfvec cases.  {NULL} and {{1}} are left out: "
                     "the caller that unpacks the ArrayType keeps those checks.",
           "cases": cases}
    with open(OUT, "w") as f:
        f.write("{\n")
        f.write(f'  "source": {json.dumps(doc["source"])},\n  "cases": [\n')
        f.write(",\n".join("    " + json.dumps(c) for c in cases))
        f.write("\n  ]\n}\n")
    print(f"wrote {len(cases)} cases to {OUT}")


if __name__ == "__main__":
    main()
