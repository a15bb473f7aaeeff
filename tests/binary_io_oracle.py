"""A step-by-step restatement of the binary type I/O (src/vector.c:376-422, src/halfvec.c:43-72, 373-419,
src/sparsevec.c:514-585) with struct and numpy, as the server runs it for one field of COPY ... (FORMAT binary).

Receive reads the field front to back as pq_getmsgint / pq_getmsgfloat4 do; a read past the end raises PostgreSQL's
"insufficient data left in message" (pq_copymsgbytes) where it happens, and bytes left after a good decode raise COPY's
"incorrect binary data format" (CopyReadBinaryAttribute).  Results are bit patterns: float rows as uint32, halfvec rows
as uint16.
"""
import struct

import numpy as np

SHORT = "insufficient data left in message"
TRAILING = "incorrect binary data format"
MAX_DIM = 16000
SPARSE_MAX_DIM = 1000000000


class RecvError(ValueError):
    pass


class _Buf:
    def __init__(self, data):
        self.data, self.pos = bytes(data), 0

    def get(self, fmt):
        size = struct.calcsize(fmt)
        if self.pos + size > len(self.data):
            raise RecvError(SHORT)
        v = struct.unpack_from(fmt, self.data, self.pos)[0]
        self.pos += size
        return v


def _check_element(bits, half, name):
    exp, man = (0x7c00, 0x3ff) if half else (0x7f800000, 0x7fffff)
    if bits & exp == exp:
        raise RecvError(f"NaN not allowed in {name}" if bits & man else f"infinite value not allowed in {name}")


def recv_dense(payload, typmod=-1, half=False):
    """vector_recv / halfvec_recv of one field: the element bits (uint32 / uint16), or RecvError"""
    name = "halfvec" if half else "vector"
    b = _Buf(payload)
    dim = b.get(">H")
    unused = b.get(">H")
    if dim < 1:
        raise RecvError(f"{name} must have at least 1 dimension")
    if dim > MAX_DIM:
        raise RecvError(f"{name} cannot have more than {MAX_DIM} dimensions")
    if typmod != -1 and typmod != dim:
        raise RecvError(f"expected {typmod} dimensions, not {dim}")
    if unused != 0:
        raise RecvError(f"expected unused to be 0, not {unused}")
    out = np.empty(dim, dtype=np.uint16 if half else np.uint32)
    for i in range(dim):
        out[i] = b.get(">H" if half else ">I")
        _check_element(int(out[i]), half, name)
    if b.pos != len(b.data):
        raise RecvError(TRAILING)
    return out


def recv_sparse(payload, typmod=-1):
    """sparsevec_recv of one field: (dim, int32 indices, uint32 value bits), or RecvError"""
    b = _Buf(payload)
    dim = b.get(">i")
    nnz = b.get(">i")
    unused = b.get(">i")
    if dim < 1:
        raise RecvError("sparsevec must have at least 1 dimension")
    if dim > SPARSE_MAX_DIM:
        raise RecvError(f"sparsevec cannot have more than {SPARSE_MAX_DIM} dimensions")
    if nnz < 0:
        raise RecvError("sparsevec cannot have negative number of elements")
    if nnz > MAX_DIM:
        raise RecvError(f"sparsevec cannot have more than {MAX_DIM} non-zero elements")
    if nnz > dim:
        raise RecvError("sparsevec cannot have more elements than dimensions")
    if typmod != -1 and typmod != dim:
        raise RecvError(f"expected {typmod} dimensions, not {dim}")
    if unused != 0:
        raise RecvError(f"expected unused to be 0, not {unused}")
    idx = np.empty(nnz, dtype=np.int32)
    for i in range(nnz):
        idx[i] = b.get(">i")
        if idx[i] < 0 or idx[i] >= dim:
            raise RecvError("sparsevec index out of bounds")
        if i > 0 and idx[i] < idx[i - 1]:
            raise RecvError("sparsevec indices must be in ascending order")
        if i > 0 and idx[i] == idx[i - 1]:
            raise RecvError("sparsevec indices must not contain duplicates")
    val = np.empty(nnz, dtype=np.uint32)
    for i in range(nnz):
        val[i] = b.get(">I")
        _check_element(int(val[i]), False, "sparsevec")
        if int(val[i]) & 0x7fffffff == 0:
            raise RecvError("binary representation of sparsevec cannot contain zero values")
    if b.pos != len(b.data):
        raise RecvError(TRAILING)
    return dim, idx, val


def send_dense(bits, half=False):
    """vector_send / halfvec_send of one row given as its element bits"""
    bits = np.asarray(bits, dtype=np.uint16 if half else np.uint32)
    return struct.pack(">HH", len(bits), 0) + bits.astype(">u2" if half else ">u4").tobytes()


def send_sparse(dim, idx, val_bits):
    """sparsevec_send of one row: 0-based indices and value bits"""
    idx = np.asarray(idx, dtype=np.int32)
    return (struct.pack(">iii", dim, len(idx), 0) + idx.astype(">i4").tobytes()
            + np.asarray(val_bits, dtype=np.uint32).astype(">u4").tobytes())


def recv_batch(payloads, typmod=-1, kind="vector"):
    """the receive of a batch field by field: (results, None) or (None, (first failing field, message))"""
    out = []
    for i, p in enumerate(payloads):
        try:
            out.append(recv_sparse(p, typmod) if kind == "sparsevec" else recv_dense(p, typmod, kind == "halfvec"))
        except RecvError as e:
            return None, (i, str(e))
    return out, None


def copy_stream(fields):
    """a PGCOPY binary stream of one-column tuples (None: a NULL field) and the byte offset of every non-NULL payload;
    the first payload starts at byte 25"""
    head = b"PGCOPY\n\xff\r\n\0" + struct.pack(">ii", 0, 0)
    parts, starts, pos = [head], [], len(head)
    for f in fields:
        if f is None:
            parts.append(struct.pack(">hi", 1, -1))
            pos += 6
            continue
        parts.append(struct.pack(">hi", 1, len(f)))
        starts.append((pos + 6, pos + 6 + len(f)))
        parts.append(f)
        pos += 6 + len(f)
    parts.append(struct.pack(">h", -1))
    return b"".join(parts), starts
