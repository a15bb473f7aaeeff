"""FindInsertPage (src/ivfinsert.c:19-67), the list an IVFFlat insert goes to, restated in tests/ivf_insert_oracle.c:
it agrees with the build's choice (the oracle's pgv_ivf_assign, AddTupleToSort) on finite data, and keeps list 0 where
the distance to centre 0 is NaN, where the build's choice does not."""
import numpy as np
import pytest

import oracle as O
from tests.ivf_insert_oracle import insert_lists
from tests.util import f32_to_half_bits, mixture


@pytest.mark.parametrize("elem,metric", [(O.VECTOR, O.L2_SQUARED), (O.VECTOR, O.NEG_IP), (O.HALFVEC, O.L2_SQUARED),
                                         (O.HALFVEC, O.NEG_IP), (O.BIT, O.HAMMING)])
def test_insert_lists_equal_build_assignment_on_finite_data(elem, metric):
    x, c = mixture(500, 32, 24, seed=11)
    if elem == O.HALFVEC:
        x, c = f32_to_half_bits(x), f32_to_half_bits(c)
    elif elem == O.BIT:
        x, c = np.packbits(x > 0, axis=1), np.packbits(c > 0, axis=1)
    want = O.ivf_assign(elem, metric, x, c, dim=32)
    got = insert_lists(elem, metric, x, c, dim=32)
    assert np.array_equal(got, want)


def test_nan_distance_to_centre_zero_keeps_list_zero():
    # vector_ip_ops: the products +3e38 * 3e38 and -3e38 * 3e38 overflow to +Inf and -Inf, whose sum is NaN -- for
    # centre 0 only; the other centres give finite distances
    c = np.zeros((3, 2), np.float32)
    c[0] = [3e38, 3e38]
    c[1] = [1.0, 0.0]
    c[2] = [0.0, 1.0]
    x = np.array([[3e38, -3e38], [2.0, 0.5]], np.float32)
    assert np.isnan(O.distance(O.VECTOR, O.NEG_IP, x[0], c[0]))
    got = insert_lists(O.VECTOR, O.NEG_IP, x, c)
    want = O.ivf_assign(O.VECTOR, O.NEG_IP, x, c)
    assert got[0] == 0 and want[0] != 0
    assert got[1] == want[1]
