"""References of the prover's coefficient-domain stage kernels (poly.cu, ntt.cu fold-8, fri.cu), composed from the oracle's restatement
of the reference (oracle/pyoracle.py) so that they run in C++ at 2^25 points.  test_gpu_poly_stages.py compares the kernels with them;
test_poly_stage_hooks_cpu.py checks them against plain Python integers at small sizes.

Vectors are (n, 2) uint64 arrays (distaff_b200.felt)."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from distaff_b200 import felt
from oracle import pyoracle as po

M = felt.M
M_LO, M_HI = np.uint64(M & (2**64 - 1)), np.uint64(M >> 64)
# the oracle's calls release the GIL: independent references run side by side
POOL = ThreadPoolExecutor(max_workers=os.cpu_count() or 1)


def fe(v):
    return po._f(v % M)


def vec(a):
    return np.ascontiguousarray(a, dtype=np.uint64).reshape(-1, 2)


def add(a, b):
    """element-wise a + b mod M of two canonical vectors"""
    a, b = vec(a), vec(b)
    lo = a[:, 0] + b[:, 0]
    top = a[:, 1] + b[:, 1]
    hi = top + (lo < a[:, 0]).astype(np.uint64)
    over = (top < a[:, 1]) | (hi < top)                      # the sum passed 2^128
    ge = over | (hi > M_HI) | ((hi == M_HI) & (lo >= M_LO))
    out = np.stack([lo, hi], axis=1)
    out[ge, 1] = hi[ge] - M_HI - (lo[ge] < M_LO).astype(np.uint64)
    out[ge, 0] = lo[ge] - M_LO
    return out


def syn_div(a, b):
    """polynom::syn_div_in_place: the quotient of a / (x - b), the remainder dropped"""
    out, b = vec(a).copy(), fe(b)                           # arrays held for the call, not temporaries
    po.lib().or_syn_div(out.ctypes.data, len(out), b.ctypes.data)
    return out


def syn_div_expanded(a, n, e):
    """polynom::syn_div_expanded_in_place(a, 8n, n, [e]): a / ((x^n - 1) / (x - e))"""
    out, e = vec(a).copy(), fe(e)
    assert len(out) == 8 * n
    po.lib().or_syn_div_expanded(out.ctypes.data, len(out), n, e.ctypes.data, 1)
    return out


def poly_eval(p, x):
    p, x, out = vec(p), fe(x), np.zeros(2, dtype=np.uint64)
    po.lib().or_poly_eval(p.ctypes.data, len(p), x.ctypes.data, out.ctypes.data)
    return int(out[0]) | (int(out[1]) << 64)


def poly_evals(jobs):
    """[(polynomial, x)] -> [P(x)], in parallel"""
    return list(POOL.map(lambda j: poly_eval(*j), jobs))


def power_series(b, n):
    b, out = fe(b), np.zeros((n, 2), dtype=np.uint64)
    po.lib().or_power_series(b.ctypes.data, n, out.ctypes.data)
    return out


def fold8_extension(coeffs, log_b):
    """the 8n coefficients evaluated on the whole domain of N = n 2^log_b points (or_fft of the zero-padded vector), as cosets [c][k] =
    P(w_N^(k b + c))"""
    coeffs = vec(coeffs)
    n, b = len(coeffs) // 8, 1 << log_b
    padded = np.zeros((n * b, 2), dtype=np.uint64)
    padded[:8 * n] = coeffs
    return po.fft(padded).reshape(n, b, 2).transpose(1, 0, 2).copy()


def coset_evaluations(coeffs):
    """the 8n coefficients evaluated on the 8n-point domain, by coset: [c][k] = P(w_8n^(8k + c))"""
    coeffs = vec(coeffs)
    n = len(coeffs) // 8
    return po.fft(coeffs).reshape(n, 8, 2).transpose(1, 0, 2).copy()


# ---- one FRI layer (fri/prover.rs: reduce) --------------------------------------------------------------------------------------------
def phys(i, log_d, log_b):
    """storage index of logical index i in a layer of 2^log_d values (poly.h Layout)"""
    i = np.asarray(i, dtype=np.int64)
    if log_b < 0:
        return i
    return ((i & ((1 << log_b) - 1)) << (log_d - log_b)) + (i >> log_b)


def rows_layout(log_d, log_b):
    """the layout the prover gives a layer's rows (and so the next layer): coset-major while a row block still holds every coset"""
    log_r = log_d - 2
    return log_r, (log_b if log_b >= 0 and log_r >= log_b else -1)


def quartic_rows(values, rows):
    """quartic::transpose(values, 1) restricted to the given rows: row r = (v[r], v[r + R], v[r + 2R], v[r + 3R])"""
    values = vec(values)
    D = len(values)
    t = np.zeros((D // 4, 4, 2), dtype=np.uint64)
    po.lib().or_quartic_transpose(values.ctypes.data, D, 1, t.ctypes.data)
    return np.ascontiguousarray(t[rows])


def blake3_rows(msgs):
    """blake3 of every 64-byte row (k, 4, 2): the first tree level of or_merkle_nodes over the rows' 32-byte halves"""
    k = len(msgs)
    m = 1
    while m < k:
        m *= 2
    pad = np.zeros((max(m, 2), 4, 2), dtype=np.uint64)
    pad[:k] = msgs
    nodes = np.frombuffer(po.merkle_nodes("blake3", pad.tobytes()), dtype=np.uint8).reshape(-1, 32)
    return nodes[len(pad):len(pad) + k].copy()


def fri_fold_rows(values, rows, log_N, alpha):
    """the folded values of the given rows of a layer (logical order) on the domain x = w_N^(i << shift): each row's cubic through
    (x_r t^j, v[r + jR]) (quartic::interpolate_batch) evaluated at alpha (quartic::evaluate_batch)"""
    values = vec(values)
    D = len(values)
    w_d = pow(felt.root_of_unity(2**log_N), 2**log_N // D, M)            # w_N^(2^shift)
    xs = quartic_rows(power_series(w_d, D), rows)
    ys = quartic_rows(values, rows)
    k = len(rows)
    polys = np.zeros((k, 4, 2), dtype=np.uint64)
    po.lib().or_quartic_interpolate_batch(xs.ctypes.data, ys.ctypes.data, k, polys.ctypes.data)
    alpha, out = fe(alpha), np.zeros((k, 2), dtype=np.uint64)
    po.lib().or_quartic_evaluate_batch(polys.ctypes.data, k, alpha.ctypes.data, out.ctypes.data)
    return out
