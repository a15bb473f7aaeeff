"""The binary type I/O restatement against the known answers, without a device."""
import json
import os
import struct

import numpy as np
import pytest

from tests import binary_io_oracle as O

KAT = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "binary_io_kat.json")))["cases"]


def _recv(c):
    p = bytes.fromhex(c["payload"])
    if c["type"] == "sparsevec":
        return O.recv_sparse(p, c["typmod"])
    return O.recv_dense(p, c["typmod"], c["type"] == "halfvec")


@pytest.mark.parametrize("i", range(len(KAT)))
def test_known_answer(i):
    c = KAT[i]
    if "error" in c:
        with pytest.raises(O.RecvError) as e:
            _recv(c)
        assert str(e.value) == c["error"]
        return
    got = _recv(c)
    if c["type"] == "sparsevec":
        dim, idx, val = got
        assert dim == c["dim"] and idx.tolist() == c["indices"] and val.tolist() == c["bits"]
        assert O.send_sparse(dim, idx, val).hex() == c["payload"]
    else:
        assert got.tolist() == c["bits"]
        assert O.send_dense(got, c["type"] == "halfvec").hex() == c["payload"]


def test_every_error_has_a_case():
    errors = {c["error"] for c in KAT if "error" in c}
    for typ in ("vector", "halfvec"):
        for msg in (f"{typ} must have at least 1 dimension", f"{typ} cannot have more than 16000 dimensions",
                    f"NaN not allowed in {typ}", f"infinite value not allowed in {typ}"):
            assert msg in errors
    for msg in ("sparsevec cannot have negative number of elements", "sparsevec indices must be in ascending order",
                "sparsevec indices must not contain duplicates", "sparsevec index out of bounds",
                "binary representation of sparsevec cannot contain zero values", O.SHORT, O.TRAILING):
        assert msg in errors


def test_client_encodings_round_trip():
    """payloads packed as the client libraries pack them ('>HH' then '>f4' / '>e' values; '>iii' then indices and
    '>f4' values) decode to their values and send back byte for byte"""
    rng = np.random.default_rng(7)
    for dim in (1, 3, 17, 1536):
        v = rng.standard_normal(dim).astype(np.float32)
        p = struct.pack(">HH", dim, 0) + v.astype(">f4").tobytes()
        got = O.recv_dense(p)
        assert np.array_equal(got.view(np.float32), v) and O.send_dense(got) == p
        h = v.astype(np.float16)
        p = struct.pack(">HH", dim, 0) + h.astype(">f2").tobytes()
        got = O.recv_dense(p, half=True)
        assert np.array_equal(got, h.view(np.uint16)) and O.send_dense(got, half=True) == p
    idx = np.sort(rng.choice(30000, 120, replace=False)).astype(np.int32)
    val = rng.standard_normal(120).astype(np.float32)
    p = struct.pack(">iii", 30000, 120, 0) + idx.astype(">i4").tobytes() + val.astype(">f4").tobytes()
    dim, gi, gv = O.recv_sparse(p)
    assert dim == 30000 and np.array_equal(gi, idx) and np.array_equal(gv.view(np.float32), val)
    assert O.send_sparse(dim, gi, gv) == p


def test_batch_first_offender_and_copy_stream():
    good = O.send_dense(np.array([1, 2, 3], dtype=np.float32).view(np.uint32))
    nan = O.send_dense(np.array([1, np.nan, 3], dtype=np.float32).view(np.uint32))
    short = good[:-2]
    assert O.recv_batch([good, short, nan])[1] == (1, O.SHORT)
    assert O.recv_batch([good, nan, short])[1] == (1, "NaN not allowed in vector")
    stream, spans = O.copy_stream([good, None, nan])
    assert stream.startswith(b"PGCOPY\n\xff\r\n\0") and spans[0][0] == 25
    assert [stream[a:b] for a, b in spans] == [good, nan]
