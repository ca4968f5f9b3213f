#!/usr/bin/env python3
"""Limb-level model of fe_mul_tw (fp128.cuh): the product a*w modulo M = 2^128 - C, C = K*2^32 - 1, K = 11520, of a canonical a
with a fixed twiddle w whose companion w_c = w*2^64 mod M is precomputed.  For a = a1*2^64 + a0,

    a*w == a0*w + a1*w_c  (mod M),   a0*w + a1*w_c < 2^193,

so the 256-bit product and the first fold of fe_reduce_v4 are replaced by two 64x128-bit products summed into the same seven
32-bit columns, and only the cheap second fold remains.  Every carry chain below is the PTX one instruction for instruction: a carry
flag that would be lost, a multiply-add leaving 64 bits or a borrow out of the top limb fails an assertion; every result is compared
with Python integers.  python tools/model_mul_tw.py"""
import random

M = 2**128 - 45 * 2**40 + 1
C = 2**128 - M
K = 11520
MASK32 = 2**32 - 1


def companion(w):
    return (w << 64) % M


def limbs(x, n=4):
    return [(x >> (32 * i)) & MASK32 for i in range(n)]


def wmad(a, b, c):
    assert 0 <= a < 2**32 and 0 <= b < 2**32 and 0 <= c < 2**64
    d = a * b + c
    assert d < 2**64, "mad.wide overflow"
    return d


class Chain:
    """one PTX carry chain: mad{c}.{lo,hi}{.cc} and addc on 32-bit registers sharing one carry flag"""

    def __init__(self):
        self.cf = 0

    def mad(self, part, a, b, c, cin, cout):
        p = a * b
        p = p & MASK32 if part == "lo" else p >> 32
        s = p + c + (self.cf if cin else 0)
        if cout:
            self.cf = s >> 32
        else:
            assert s >> 32 == 0, "carry lost at the end of a chain"
        return s & MASK32

    def addc(self, x, y, cout=False):
        s = x + y + self.cf
        if cout:
            self.cf = s >> 32
        else:
            assert s >> 32 == 0, "carry lost at the end of a chain"
        return s & MASK32


def row(acc_lo_idx, acc, a, b0, b1, cin_first, carry_to, fresh_top):
    """acc[i..i+3] += a*b0 + (a*b1 << 64) on one chain; the carry out goes to acc[carry_to] (fresh: set, else added)"""
    ch = Chain()
    i = acc_lo_idx
    acc[i] = ch.mad("lo", a, b0, acc[i], cin_first, True)
    acc[i + 1] = ch.mad("hi", a, b0, acc[i + 1], True, True)
    acc[i + 2] = ch.mad("lo", a, b1, acc[i + 2], True, True)
    if fresh_top:
        acc[i + 3] = ch.mad("hi", a, b1, acc[i + 3], True, carry_to is not None)
    else:
        acc[i + 3] = ch.mad("hi", a, b1, acc[i + 3], True, True)
    if carry_to is not None:
        acc[carry_to] = ch.addc(acc.get(carry_to, 0), 0)


def mul_tw(a, w, wc):
    """returns (value, slow) where slow says whether the out-of-line canonicalisation ran"""
    x = limbs(a)
    y = limbs(w)
    z = limbs(wc)
    # E holds the even columns (E[c]:E[c+1] a 64-bit accumulator at column c, c = 0, 2, 4), O the odd ones (c = 1, 3, 5)
    E = {}
    O = {}
    # row A: x0 * w at column 0 (plain products, no carries)
    E[0], E[1] = (x[0] * y[0]) & MASK32, (x[0] * y[0]) >> 32
    E[2], E[3] = (x[0] * y[2]) & MASK32, (x[0] * y[2]) >> 32
    O[1], O[2] = (x[0] * y[1]) & MASK32, (x[0] * y[1]) >> 32
    O[3], O[4] = (x[0] * y[3]) & MASK32, (x[0] * y[3]) >> 32
    # row B: x2 * w_c at column 0: E0..E3 += x2 (z0 + z2 2^64), carry -> E4 (fresh);  O1..O4 += x2 (z1 + z3 2^64), carry -> O5 (fresh)
    row(0, E, x[2], z[0], z[2], False, 4, False)
    row(1, O, x[2], z[1], z[3], False, 5, False)
    # row C: x1 * w at column 1: O1..O4 += x1 (y0 + y2 2^64), carry added to O5;  E2..E5 += x1 (y1 + y3 2^64), E5 fresh (hi + carry)
    row(1, O, x[1], y[0], y[2], False, 5, False)
    E[5] = 0
    row(2, E, x[1], y[1], y[3], False, None, True)
    # row D: x3 * w_c at column 1: O1..O4 += x3 (z0 + z2 2^64), carry added to O5;  E2..E5 += x3 (z1 + z3 2^64), carry -> E6 (fresh)
    row(1, O, x[3], z[0], z[2], False, 5, False)
    row(2, E, x[3], z[1], z[3], False, 6, False)
    assert all(0 <= v <= MASK32 for v in list(E.values()) + list(O.values()))
    P = sum(E[c] << (32 * c) for c in E) + sum(O[c] << (32 * c) for c in O)
    x0_64, x1_64 = a & (2**64 - 1), a >> 64
    assert P == x0_64 * w + x1_64 * wc, "partial products"
    assert P < 2**193
    # r = E + (O << 32): one chain over columns 1..6
    ch = Chain()
    r = [E[0], ch.addc(E[1], O[1], True)]
    r.append(ch.addc(E[2], O[2], True))
    r.append(ch.addc(E[3], O[3], True))
    r.append(ch.addc(E[4], O[4], True))
    r.append(ch.addc(E[5], O[5], True))
    r.append(ch.addc(E[6], 0, False))
    assert sum(v << (32 * i) for i, v in enumerate(r)) == P
    assert r[6] <= 1
    # fold the 65-bit top T = r6:r5:r4:  + (T*K) << 32 on a multiply-add chain (T*K < 2^79), then - T
    u1 = wmad(r[4], K, r[1])
    u2 = wmad(r[2], 1, wmad(r[5], K, u1 >> 32))
    u3 = wmad(r[3], 1, wmad(r[6], K, u2 >> 32))
    v = [r[0], u1 & MASK32, u2 & MASK32, u3 & MASK32]
    cy = u3 >> 32
    # 5-limb borrow chain: v0 - r4, v1 - r5, v2 - r6, v3, cy
    Vv = sum(t << (32 * i) for i, t in enumerate(v)) + (cy << 128)
    T = r[4] + (r[5] << 32) + (r[6] << 64)
    W = Vv - T
    assert 0 <= W < 2**128 + 2**111, "fold bound"
    assert W == (P & (2**128 - 1)) + (P >> 128) * C
    cy = W >> 128
    assert cy in (0, 1)
    lo = W & (2**128 - 1)
    slow = bool(cy or (lo >> 96) == MASK32)
    if slow:
        q = lo + C
        g = q >> 128
        if cy or g:
            lo = q & (2**128 - 1)
    assert lo < M
    return lo, slow


EDGE = [0, 1, M - 1, 2**64 - 1, 2**64, M - 2**64, 2**128 - 2**96 - 1, M - 2, C, C + 1, 2**64 + 1, MASK32 * (2**96 + 2**64 + 2**32 + 1) % M]


def slow_pairs(rnd, count):
    """canonical (a, w) whose folded value overflows 2^128 or lies in [2^128 - 2^96, 2^128): a1 small, w near (k+1) 2^128 / a0"""
    out = []
    while len(out) < count:
        a1 = rnd.randrange(0, 2**rnd.randrange(1, 40))
        k = rnd.randrange(1, 2**rnd.randrange(1, 60))
        a0 = rnd.randrange(2**63, 2**64)
        w = rnd.randrange(1, M)
        wc = companion(w)
        # pick w so that a0*w + a1*wc lands just below (k+1) 2^128 (the rare paths sit there); w = wc*2^-64 so solve for wc via w
        target = (k + 1) * 2**128 - rnd.randrange(0, k * C + 2**97)
        w = (target - a1 * wc) // a0
        if not 0 < w < M:
            continue
        wc = companion(w)
        a = a0 + (a1 << 64)
        if a >= M:
            continue
        if mul_tw(a, w, wc)[1]:
            out.append((a, w))
    return out


def main():
    n = slow = 0
    for a in EDGE:
        for w in EDGE:
            a, w = a % M, w % M
            r, s = mul_tw(a, w, companion(w))
            assert r == a * w % M, (a, w)
            n += 1
            slow += s
    # all-ones limbs: every limb of a, w and w_c either 0 or 2^32 - 1 (the canonical ones), w_c taken as given
    masks = [sum(MASK32 << (32 * i) for i in range(4) if (m >> i) & 1) for m in range(16)]
    masks = [x for x in masks if x < M]
    for a in masks:
        for w in masks:
            for wc in masks:
                # fe_mul_tw(a, w, wc) = a0*w + a1*wc mod M for any canonical w, wc; the companion only makes it a*w
                r, s = mul_tw(a, w, wc)
                assert r == ((a & (2**64 - 1)) * w + (a >> 64) * wc) % M
                n += 1
                slow += s
    rnd = random.Random(20)
    sp = slow_pairs(rnd, 2000)
    for a, w in sp:
        r, s = mul_tw(a, w, companion(w))
        assert s and r == a * w % M
        n += 1
        slow += 1
    ov = sum(1 for a, w in sp if (((a & (2**64 - 1)) * w + (a >> 64) * companion(w)) & (2**128 - 1)) +
             (((a & (2**64 - 1)) * w + (a >> 64) * companion(w)) >> 128) * C >= 2**128)
    for _ in range(200000):
        a, w = rnd.randrange(M), rnd.randrange(M)
        r, s = mul_tw(a, w, companion(w))
        assert r == a * w % M
        n += 1
        slow += s
    print(n, "products correct,", slow, "through the slow path,", ov, "of them overflowing 2^128")


if __name__ == "__main__":
    main()
