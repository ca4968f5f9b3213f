"""CPU checks of fe_mul_tw (fp128.cuh), the NTT pass kernels' product with a fixed twiddle w and its companion w * 2^64 mod M, through
its limb-level model tools/model_mul_tw.py: every carry chain and bound of the PTX restated in Python integers."""
import os
import random
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
import model_mul_tw as mt  # noqa: E402

M = mt.M


def test_edge_operands():
    ops = [0, 1, M - 1, 2**64 - 1, 2**64, M - 2**64] + mt.EDGE
    for a in ops:
        for w in ops:
            a, w = a % M, w % M
            assert mt.mul_tw(a, w, mt.companion(w))[0] == a * w % M, (a, w)


def test_all_ones_limbs():
    """every limb of a, w and the companion slot 0 or 2^32 - 1; any canonical companion gives a0 w + a1 w_c mod M"""
    masks = [x for x in (sum((2**32 - 1) << (32 * i) for i in range(4) if (m >> i) & 1) for m in range(16)) if x < M]
    for a in masks:
        for w in masks:
            for wc in masks:
                assert mt.mul_tw(a, w, wc)[0] == ((a % 2**64) * w + (a >> 64) * wc) % M


def test_slow_paths():
    """operands whose folded value overflows 2^128 or has an all-ones top limb, both kinds present"""
    pairs = mt.slow_pairs(random.Random(5), 400)
    over = 0
    for a, w in pairs:
        r, slow = mt.mul_tw(a, w, mt.companion(w))
        assert slow and r == a * w % M
        p = (a % 2**64) * w + (a >> 64) * mt.companion(w)
        over += (p % 2**128) + (p >> 128) * mt.C >= 2**128
    assert 0 < over < len(pairs)


def test_random_pairs():
    """10^6 seeded random pairs: the first 10^5 through the limb model, all of them through the identity a w == a0 w + a1 w_c (mod M)
    and the bound a0 w + a1 w_c < 2^193 the fold relies on"""
    rnd = random.Random(1)
    for i in range(10**6):
        a, w = rnd.randrange(M), rnd.randrange(M)
        wc = mt.companion(w)
        p = (a % 2**64) * w + (a >> 64) * wc
        assert p < 2**193 and p % M == a * w % M
        if i < 10**5:
            assert mt.mul_tw(a, w, wc)[0] == a * w % M


def test_companions_of_a_root_table():
    """the companion of every power of the 2^10-th root of unity is w * 2^64 mod M, and the model multiplies by the power with it"""
    from distaff_b200 import felt
    g = felt.root_of_unity(2**10)
    rnd = random.Random(3)
    w = 1
    for _ in range(2**10):
        wc = mt.companion(w)
        assert wc == w * 2**64 % M and wc < M
        a = rnd.randrange(M)
        assert mt.mul_tw(a, w, wc)[0] == a * w % M
        w = w * g % M
    assert w == 1
