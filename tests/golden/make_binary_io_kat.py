#!/usr/bin/env python3
"""Write the known answers of the binary type I/O to tests/golden/binary_io_kat.json.

    python tests/golden/make_binary_io_kat.py

The payloads are written out by hand from the reference's recv / send functions (src/vector.c:376-422,
src/halfvec.c:43-72, 373-419, src/sparsevec.c:514-585), not computed by the code under test:
  - "copy": the rows of test/sql/copy.sql as the exact bytes vector_send / halfvec_send / sparsevec_send write, with
    the text the table prints after the COPY round trip (test/expected/copy.out);
  - "error": one payload per error a receive function can raise, with its errmsg and where it comes from.  Two texts
    are PostgreSQL's, not pgvector's: "insufficient data left in message" (pq_copymsgbytes, raised by pq_getmsgint /
    pq_getmsgfloat4 reading past the end) and "incorrect binary data format" (CopyReadBinaryAttribute, bytes left over
    after the receive function returned);
  - "order": payloads with two defects, whose expected error is the one the reference's read / check order meets first.
Source lines are found by searching the reference tree at PGV_REFERENCE (default /root/reference) for each errmsg.
"""
import json
import os
import re
import struct

REF = os.environ.get("PGV_REFERENCE", "/root/reference")
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "binary_io_kat.json")
SHORT = "insufficient data left in message"
TRAILING = "incorrect binary data format"
PG = {SHORT: "PostgreSQL pq_copymsgbytes (src/backend/libpq/pqformat.c)",
      TRAILING: "PostgreSQL CopyReadBinaryAttribute (src/backend/commands/copyfromparse.c)"}
F = {"nan": 0x7fc00000, "inf": 0x7f800000, "-inf": 0xff800000, "0": 0, "-0": 0x80000000, "1": 0x3f800000,
     "2": 0x40000000, "3": 0x40400000}
H = {"nan": 0x7e00, "inf": 0x7c00, "-inf": 0xfc00, "0": 0, "1": 0x3c00, "2": 0x4000, "3": 0x4200}


def dense(dim, unused, elems, half=False):
    bits = [(H if half else F)[e] if isinstance(e, str) else e for e in elems]
    return struct.pack(">HH", dim, unused) + b"".join(struct.pack(">H" if half else ">I", b) for b in bits)


def sparse(dim, nnz, unused, idx, vals):
    return (struct.pack(">iii", dim, nnz, unused) + b"".join(struct.pack(">i", i) for i in idx)
            + b"".join(struct.pack(">I", F[v] if isinstance(v, str) else v) for v in vals))


def source_of(msg, typ):
    """the reference line that raises msg (numbers stand for its %d), or PostgreSQL's function for its two texts"""
    if msg in PG:
        return PG[msg]
    fmt = re.sub(r"(?<=not )-?\d+|(?<=than )\d+|(?<=expected )\d+", "%d", msg)
    path = f"src/{typ}.c"
    for i, line in enumerate(open(os.path.join(REF, path)).read().split("\n")):
        if f'"{fmt}"' in line:
            return f"{path}:{i + 1}"
    raise SystemExit(f"no source line for {msg!r} in {path}")


def main():
    cases = []

    def add(group, typ, payload, typmod=-1, error=None, **kw):
        c = {"group": group, "type": typ, "typmod": typmod, "payload": payload.hex()}
        if error is not None:
            c["error"] = error
            c["source"] = source_of(error, typ)
        c.update(kw)
        cases.append(c)

    # test/sql/copy.sql: vector(3) / halfvec(3) rows '[0,0,0]', '[1,2,3]', '[1,1,1]' and NULL; sparsevec(3) rows
    # '{}/3', '{1:1,2:2,3:3}/3', '{1:1,2:1,3:1}/3' and NULL
    for typ, half in (("vector", False), ("halfvec", True)):
        for elems, text in ((["0", "0", "0"], "[0,0,0]"), (["1", "2", "3"], "[1,2,3]"), (["1", "1", "1"], "[1,1,1]")):
            tab = H if half else F
            add("copy", typ, dense(3, 0, elems, half), 3, text=text, bits=[tab[e] for e in elems])
    for idx, vals, text in (([], [], "{}/3"), ([0, 1, 2], ["1", "2", "3"], "{1:1,2:2,3:3}/3"),
                            ([0, 1, 2], ["1", "1", "1"], "{1:1,2:1,3:1}/3")):
        add("copy", "sparsevec", sparse(3, len(idx), 0, idx, vals), 3, text=text, dim=3, indices=idx,
            bits=[F[v] for v in vals])

    for typ, half in (("vector", False), ("halfvec", True)):
        d = lambda *a, **k: dense(*a, half=half, **k)  # noqa: E731
        add("error", typ, b"", error=SHORT)
        add("error", typ, b"\x00", error=SHORT)
        add("error", typ, b"\x00\x03\x00", error=SHORT)
        add("error", typ, d(0, 0, []), error=f"{typ} must have at least 1 dimension")
        add("error", typ, d(16001, 0, []), error=f"{typ} cannot have more than 16000 dimensions")
        add("error", typ, d(65535, 0, []), error=f"{typ} cannot have more than 16000 dimensions")
        add("error", typ, d(4, 0, ["1"] * 4), 3, error="expected 3 dimensions, not 4")
        add("error", typ, d(3, 7, ["1"] * 3), error="expected unused to be 0, not 7")
        add("error", typ, d(3, 65535, ["1"] * 3), error="expected unused to be 0, not 65535")
        add("error", typ, d(3, 0, ["1", "nan", "1"]), error=f"NaN not allowed in {typ}")
        add("error", typ, d(3, 0, ["1", "1", "inf"]), error=f"infinite value not allowed in {typ}")
        add("error", typ, d(3, 0, ["-inf", "1", "1"]), error=f"infinite value not allowed in {typ}")
        add("error", typ, d(3, 0, ["1", "2"]), error=SHORT)
        add("error", typ, d(3, 0, ["1", "2", "3"]) + b"\x00", error=TRAILING)
        add("error", typ, d(3, 0, ["1", "2", "3"])[:-1], error=SHORT)
        # order: the read / check sequence decides
        add("order", typ, d(11, 0, ["1", "1", "1", "nan", "1"]), error=f"NaN not allowed in {typ}")
        add("order", typ, d(6, 0, ["1", "1"]), error=SHORT)
        add("order", typ, d(0, 0, []) + b"\x00" * 8, 3, error=f"{typ} must have at least 1 dimension")
        add("order", typ, d(16001, 5, []), 3, error=f"{typ} cannot have more than 16000 dimensions")
        add("order", typ, d(4, 1, []), 3, error="expected 3 dimensions, not 4")
        add("order", typ, d(3, 1, []), error="expected unused to be 0, not 1")
        add("order", typ, d(3, 0, ["inf", "nan", "1"]) + b"\x00", error=f"infinite value not allowed in {typ}")
        add("order", typ, d(2, 0, ["1", "2", "3"]), error=TRAILING)

    s = sparse
    add("error", "sparsevec", b"\x00\x00\x00", error=SHORT)
    add("error", "sparsevec", struct.pack(">i", 3) + b"\x00\x00", error=SHORT)
    add("error", "sparsevec", struct.pack(">ii", 3, 0) + b"\x00", error=SHORT)
    add("error", "sparsevec", s(0, 0, 0, [], []), error="sparsevec must have at least 1 dimension")
    add("error", "sparsevec", s(-5, 0, 0, [], []), error="sparsevec must have at least 1 dimension")
    add("error", "sparsevec", s(1000000001, 0, 0, [], []), error="sparsevec cannot have more than 1000000000 dimensions")
    add("error", "sparsevec", s(3, -1, 0, [], []), error="sparsevec cannot have negative number of elements")
    add("error", "sparsevec", s(100000, 16001, 0, [], []), error="sparsevec cannot have more than 16000 non-zero elements")
    add("error", "sparsevec", s(3, 4, 0, [], []), error="sparsevec cannot have more elements than dimensions")
    add("error", "sparsevec", s(4, 1, 0, [0], ["1"]), 3, error="expected 3 dimensions, not 4")
    add("error", "sparsevec", s(3, 1, 7, [0], ["1"]), error="expected unused to be 0, not 7")
    add("error", "sparsevec", s(3, 1, -2, [0], ["1"]), error="expected unused to be 0, not -2")
    add("error", "sparsevec", s(3, 1, 0, [3], ["1"]), error="sparsevec index out of bounds")
    add("error", "sparsevec", s(3, 1, 0, [-1], ["1"]), error="sparsevec index out of bounds")
    add("error", "sparsevec", s(3, 2, 0, [2, 1], ["1", "1"]), error="sparsevec indices must be in ascending order")
    add("error", "sparsevec", s(3, 2, 0, [1, 1], ["1", "1"]), error="sparsevec indices must not contain duplicates")
    add("error", "sparsevec", s(3, 2, 0, [0, 1], ["1", "nan"]), error="NaN not allowed in sparsevec")
    add("error", "sparsevec", s(3, 2, 0, [0, 1], ["inf", "1"]), error="infinite value not allowed in sparsevec")
    add("error", "sparsevec", s(3, 1, 0, [0], ["0"]),
        error="binary representation of sparsevec cannot contain zero values")
    add("error", "sparsevec", s(3, 1, 0, [0], ["-0"]),
        error="binary representation of sparsevec cannot contain zero values")
    add("error", "sparsevec", s(3, 2, 0, [0], []), error=SHORT)
    add("error", "sparsevec", s(3, 2, 0, [0, 1], ["1"]), error=SHORT)
    add("error", "sparsevec", s(3, 1, 0, [0], ["1"]) + b"\x00", error=TRAILING)
    add("order", "sparsevec", s(3, 2, 0, [0, 1], ["0", "nan"]),
        error="binary representation of sparsevec cannot contain zero values")
    add("order", "sparsevec", s(3, 2, 0, [0, 1], ["nan", "0"]), error="NaN not allowed in sparsevec")
    add("order", "sparsevec", s(4, 5, 0, [], []), 3, error="sparsevec cannot have more elements than dimensions")
    add("order", "sparsevec", s(0, -1, 0, [], []), error="sparsevec must have at least 1 dimension")
    add("order", "sparsevec", s(4, 1, 9, [0], ["1"]), 3, error="expected 3 dimensions, not 4")
    add("order", "sparsevec", s(3, 2, 0, [1, 1], ["nan", "1"]), error="sparsevec indices must not contain duplicates")
    add("order", "sparsevec", s(3, 3, 0, [0, 1, 2], ["nan"]), error="NaN not allowed in sparsevec")
    add("order", "sparsevec", s(3, 3, 0, [0, 5], []), error="sparsevec index out of bounds")
    add("order", "sparsevec", s(3, 3, 0, [0, 1], []), error=SHORT)
    add("order", "sparsevec", s(3, 1, 0, [0], ["nan"]) + b"\x00\x00", error="NaN not allowed in sparsevec")
    add("order", "sparsevec", s(3, 0, 0, [], []) + b"\x00", error=TRAILING)

    with open(OUT, "w") as fh:
        json.dump({"cases": cases}, fh, indent=1)
        fh.write("\n")
    print(f"{len(cases)} cases -> {OUT}")


if __name__ == "__main__":
    main()
