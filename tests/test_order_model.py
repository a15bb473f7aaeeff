"""CPU checks of the btree order (vb_order): the oracle comparators against the reference's known answers (btree.out and
the comparison cases of vector_type.out / halfvec.out / sparsevec.out, different dimensions included), a numpy
restatement of the key encodings the GPU sorts by against the oracle comparators on random rows of one dimension (-0,
stored zeros and +-inf included), and the loud no-device error of every new Python entry point."""
import json
import os
import types

import numpy as np
import pytest

from tests import order_oracle as OO

HERE = os.path.dirname(os.path.abspath(__file__))
KAT = json.load(open(os.path.join(HERE, "golden", "btree_kat.json")))
SPECIAL = np.array([-2.0, -1.0, -0.0, 0.0, 1.0, 2.0, np.inf, -np.inf], np.float32)


def parse(typ, text):
    from pgvector_b200.sparsevec import SparseVector
    if typ == "sparsevec":
        return SparseVector.from_text(text)
    return np.array(json.loads(text), np.float32)


def cmp(typ, a, b):
    if typ == "vector":
        return OO.vector_cmp(a, b)
    if typ == "halfvec":
        return OO.halfvec_cmp(a, b)
    return OO.sparsevec_cmp(a, b)


OPS = {"<": lambda c: c < 0, "<=": lambda c: c <= 0, "=": lambda c: c == 0, "!=": lambda c: c != 0, ">=": lambda c: c >= 0,
       ">": lambda c: c > 0, "cmp": lambda c: c}


@pytest.mark.parametrize("case", KAT["compare"], ids=lambda c: f"{c['type']} {c['a']} {c['op']} {c['b']}")
def test_oracle_comparators_reproduce_the_reference(case):
    c = cmp(case["type"], parse(case["type"], case["a"]), parse(case["type"], case["b"]))
    assert OPS[case["op"]](c) == case["expect"]


@pytest.mark.parametrize("case", KAT["btree"], ids=lambda c: c["type"])
def test_oracle_order_reproduces_btree_out(case):
    from pgvector_b200.sparsevec import SparseRows
    typ = case["type"]
    texts = [t for t in case["rows"] if t is not None]   # NULLs sort last (btree's default NULLS LAST); tables hold none
    kind = {"vector": OO.VECTOR, "halfvec": OO.HALFVEC, "sparsevec": OO.SPARSE}[typ]
    vals = [parse(typ, t) for t in texts]
    rows = SparseRows.from_vectors(vals, case["dim"]) if kind == OO.SPARSE else np.stack(vals)
    perm, gor, gst = OO.order(kind, rows)
    want = [t for t in case["order"] if t is not None]
    assert [texts[i] for i in perm] == want
    assert case["order"][-1] is None
    q = parse(typ, case["eq"]["query"])
    qrows = SparseRows.from_vectors([q], case["dim"]) if kind == OO.SPARSE else q.reshape(1, -1)
    lo, hi = OO.bounds(kind, rows, qrows)
    assert [texts[i] for i in perm[lo[0]:hi[0]]] == case["eq"]["rows"]
    assert len(gst) == len(texts) + 1 and gst[-1] == len(texts)


# ------------------------------------------------------------------ the key encodings of vb_order.cu, restated

def f32_keys(x):
    b = np.ascontiguousarray(x, np.float32).view(np.uint32).copy()
    b[b == 0x80000000] = 0
    return np.where(b >> 31 != 0, b ^ np.uint32(0xFFFFFFFF), b ^ np.uint32(0x80000000)).astype(np.uint64)


def f16_keys(h):
    b = OO.half_bits(h).astype(np.uint32)
    b[b == 0x8000] = 0
    return np.where(b >> 15 != 0, b ^ 0xFFFF, b ^ 0x8000).astype(np.uint64)


def half_words(h):
    """two halves per 32-bit key word, element 2w in the high half; the missing half of an odd dimension is 0"""
    k = f16_keys(h)
    if k.shape[1] % 2:
        k = np.concatenate([k, np.zeros((k.shape[0], 1), np.uint64)], axis=1)
    return (k[:, 0::2] << np.uint64(16)) | k[:, 1::2]


def sparse_keys(idx, val):
    """one 64-bit key per stored entry, then the terminator 1 << 62"""
    f = f32_keys(np.asarray(val, np.float32).reshape(1, -1))[0] if len(val) else np.zeros(0, np.uint64)
    out = []
    for i, v, fv in zip(idx, val, f):
        if v < 0:
            out.append((int(i) << 32) | int(fv))
        else:
            out.append((2 << 62) | (((1 << 30) - 1 - int(i)) << 32) | int(fv))
    return out + [1 << 62]


def lex_sign(ka, kb):
    """sign of the lexicographic comparison of equal-length key rows [npairs, L]"""
    d = ka != kb
    first = np.argmax(d, axis=1)
    r = np.arange(ka.shape[0])
    return np.where(d.any(axis=1), np.where(ka[r, first] < kb[r, first], -1, 1), 0)


@pytest.mark.parametrize("dim", [1, 2, 3, 5, 8])
def test_fp32_keys_order_like_vector_cmp(dim):
    rng = np.random.default_rng(dim)
    a = rng.choice(SPECIAL, size=(40000, dim))
    b = np.where(rng.random((40000, dim)) < 0.7, a, rng.choice(SPECIAL, size=(40000, dim))).astype(np.float32)
    np.testing.assert_array_equal(lex_sign(f32_keys(a), f32_keys(b)), OO.dense_cmp_pairs(False, a, b))


@pytest.mark.parametrize("dim", [1, 2, 3, 5, 8])
def test_half_keys_order_like_halfvec_cmp(dim):
    rng = np.random.default_rng(100 + dim)
    vals = np.concatenate([SPECIAL, np.array([6e-8, -6e-8, 1e-5, -1e-5, 65504, -65504], np.float32)])   # with subnormals
    a = rng.choice(vals, size=(40000, dim)).astype(np.float16)
    b = np.where(rng.random((40000, dim)) < 0.7, a, rng.choice(vals, size=(40000, dim)).astype(np.float16))
    np.testing.assert_array_equal(lex_sign(half_words(a), half_words(b)), OO.dense_cmp_pairs(True, a, b))


def random_sparse(rng, n, dim, p=0.5):
    from pgvector_b200.sparsevec import SparseRows
    mask = rng.random((n, dim)) < p
    vals = rng.choice(SPECIAL, size=(n, dim))
    off = np.zeros(n + 1, np.int64)
    off[1:] = np.cumsum(mask.sum(axis=1))
    r, c = np.nonzero(mask)
    return SparseRows(dim, off, c.astype(np.int32), vals[r, c].astype(np.float32))   # stored zeros of both signs included


@pytest.mark.parametrize("dim", [1, 3, 6])
def test_sparse_keys_order_like_sparsevec_cmp(dim):
    rng = np.random.default_rng(200 + dim)
    n = 30000
    a = random_sparse(rng, n, dim)
    b = random_sparse(rng, n, dim)
    want = OO.sparse_cmp_pairs(a, b)
    got = np.empty(n, np.int32)
    for k in range(n):
        ka = sparse_keys(a.idx[a.row_off[k]:a.row_off[k + 1]], a.val[a.row_off[k]:a.row_off[k + 1]])
        kb = sparse_keys(b.idx[b.row_off[k]:b.row_off[k + 1]], b.val[b.row_off[k]:b.row_off[k + 1]])
        got[k] = (ka > kb) - (ka < kb)
    np.testing.assert_array_equal(got, want)
    assert (want == 0).sum() > 0 and (want < 0).sum() > 0 and (want > 0).sum() > 0


def test_sparse_key_cases_named_by_the_encoding():
    """a negative entry at a smaller index than a positive one, a stored zero against no entry, -0 against +0"""
    def SV(dim, idx, val):   # SparseVector's input refuses inf, as sparsevec_in does; device rows can hold it
        return types.SimpleNamespace(dim=dim, indices=np.array(idx, np.int32), values=np.array(val, np.float32))
    for a, b in [(SV(4, [0], [-1.0]), SV(4, [1], [1.0])), (SV(4, [1], [0.0]), SV(4, [], [])),
                 (SV(4, [2], [-0.0]), SV(4, [2], [0.0])), (SV(4, [0, 3], [1.0, -np.inf]), SV(4, [0], [1.0])),
                 (SV(4, [3], [np.inf]), SV(4, [0], [-np.inf]))]:
        ka, kb = sparse_keys(a.indices, a.values), sparse_keys(b.indices, b.values)
        assert (ka > kb) - (ka < kb) == OO.sparsevec_cmp(a, b)


# ------------------------------------------------------------------ no device: a loud error from every entry point

def test_every_order_entry_point_fails_loudly_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a device is visible")
    from pgvector_b200 import _lib
    if not os.path.exists(_lib.LIB_PATH):
        import __graft_entry__
        __graft_entry__.build()
    import pgvector_b200 as pv
    from pgvector_b200.sparsevec import SparseRows
    dense = types.SimpleNamespace(h=None, elem=pv.VECTOR, dim=3)
    sparse = types.SimpleNamespace(h=None, dim=3)
    o_dense = pv.Order(dense, None, False)
    o_sparse = pv.Order(sparse, None, True)
    calls = [lambda: pv.Table.order(dense), lambda: pv.SparseTable.order(sparse), lambda: o_dense.read(),
             lambda: o_dense.perm, lambda: o_dense.group_of_row, lambda: o_dense.group_start,
             lambda: o_dense.bounds(np.zeros((2, 3), np.float32)),
             lambda: o_sparse.bounds(SparseRows(3, [0, 1], [0], [1.0]))]
    for call in calls:
        with pytest.raises(pv.VecB200Error) as e:
            call()
        assert e.value.code == _lib.ENODEVICE
