#!/usr/bin/env python3
"""Model of the fold-1 coset first pass (ct_coset_regs in ntt_pass.cuh, coset_roots_fill_kernel in ntt.cu) over a small NTT prime.

An L-point pass on coset c evaluates X[k] = sum_j x_j (t w_L^k)^j.  Instead of scaling x_j by t^j first, Cooley-Tukey butterflies
(a + rho b, a - rho b) run on the natural-order input; stage st, block r of L >> st points multiplies by

    rho_{st,r} = (t w_L^rev_st(r))^(L >> (st+1)),

and position q ends up holding X[bitrev(q)], the order the decimation-in-frequency rounds of the other kinds leave.  With t = w_(L b)^c
and w_L = w_(L b)^b, rho_{st,r} is w_(L b) to the power (c + b rev_st(r)) << (log L - st - 1): the exponent the table fill uses.  The
table is laid out as on the device: heap index 2^st - 1 + r.  Every coset of several (L, b) shapes is compared with the direct sum.
python tools/model_coset_ct.py"""
import random

P = 998244353          # 119 * 2^23 + 1, generator 3
G = 3


def root(order):
    return pow(G, (P - 1) // order, P)


def rev(x, bits):
    return int(format(x, "0%db" % bits)[::-1], 2) if bits else 0


def table(log_l, log_b, c):
    """the heap of one coset as coset_roots_fill_kernel writes it (entry L - 1 unused)"""
    L = 1 << log_l
    w = root(L << log_b)
    out = [0] * L
    for st in range(log_l):
        for r in range(1 << st):
            e = (c + (rev(r, st) << log_b)) << (log_l - st - 1)
            out[(1 << st) - 1 + r] = pow(w, e % (L << log_b), P)
    return out


def check(log_l, log_b, rng):
    L = 1 << log_l
    wL, wLb = root(L), root(L << log_b)
    x = [rng.randrange(P) for _ in range(L)]
    for c in range(1 << log_b):
        t = pow(wLb, c, P)
        rho = table(log_l, log_b, c)
        for st in range(log_l):           # the table is the definition of rho
            for r in range(1 << st):
                assert rho[(1 << st) - 1 + r] == pow(t * pow(wL, rev(r, st), P) % P, L >> (st + 1), P)
        y = x[:]
        for st in range(log_l):
            h = L >> (st + 1)
            for q in range(L):
                if q & h:
                    continue
                f = rho[(1 << st) - 1 + (q >> (log_l - st))]     # block index of position q at stage st
                a, b = y[q], y[q + h] * f % P
                y[q], y[q + h] = (a + b) % P, (a - b) % P
        want = [sum(x[j] * pow(t * pow(wL, k, P), j, P) for j in range(L)) % P for k in range(L)]
        assert [y[rev(k, log_l)] for k in range(L)] == want, (log_l, log_b, c)


if __name__ == "__main__":
    rng = random.Random(7)
    for log_l, log_b in [(1, 1), (2, 3), (4, 2), (6, 3), (5, 5)]:
        check(log_l, log_b, rng)
    print("ok: coset butterflies equal the direct sums on every coset")
