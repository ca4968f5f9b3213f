"""-m gpu: fe_mul_tw (fp128.cuh), the NTT pass kernels' product with a fixed twiddle and its companion w * 2^64 mod M, against fe_mul and
Python integers on the device, through dg.field_op("mul_tw") (companion computed on the device as the twiddle tables compute it)."""
import os
import random
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

M = 2**128 - 45 * 2**40 + 1
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    assert backend.device_info()["sm_count"] > 0
    return distaff_b200


def _check(dg, xs, ys):
    from distaff_b200 import felt
    a, b = felt.from_ints(xs), felt.from_ints(ys)
    want = [x * y % M for x, y in zip(xs, ys)]
    got = dg.field_op("mul_tw", a, b)
    assert np.array_equal(got, dg.field_op("mul", a, b))
    assert np.array_equal(got, dg.field_op("mul_tw", a, b, impl=1))     # the portable twin
    assert felt.to_ints(got) == want


def test_edge_operands(dg):
    edge = [0, 1, 2, M - 1, M - 2, 2**64 - 1, 2**64, 2**64 + 1, M - 2**64, 2**127, 2**128 - 2**96 - 1, 45 * 2**40 - 1, 45 * 2**40,
            (2**32 - 1) * (2**96 + 2**64 + 2**32 + 1) % M, (2**32 - 1) * (2**96 + 2**32) % M, (2**32 - 1) * (2**64 + 1)]
    _check(dg, [x for x in edge for _ in edge], [y for _ in edge for y in edge])


def test_slow_paths(dg):
    """operands whose folded value overflows 2^128 or ends with an all-ones top limb (tools/model_mul_tw.py), and the crafted pairs of
    fe_mul's own rare paths (tools/gen_mul_vectors.py)"""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import gen_mul_vectors
    import model_mul_tw
    pairs = model_mul_tw.slow_pairs(random.Random(11), 2000) + gen_mul_vectors.pairs()
    _check(dg, [p[0] for p in pairs], [p[1] for p in pairs])


def test_random_pairs(dg):
    rnd = random.Random(12)
    n = 10**6
    _check(dg, [rnd.randrange(M) for _ in range(n)], [rnd.randrange(M) for _ in range(n)])


def test_root_table_products(dg):
    """every power of the 2^10-th root of unity as the twiddle, the stage roots of a 1024-point pass"""
    from distaff_b200 import felt
    g = felt.root_of_unity(2**10)
    ws = [pow(g, j, M) for j in range(2**10)]
    rnd = random.Random(13)
    _check(dg, [rnd.randrange(M) for _ in range(4 * len(ws))], ws * 4)
