"""References of the prover's evaluation-domain stage kernels (ntt.cu fold-1 coset extension, hash.cu row hashing and Merkle trees,
shard.cu constraint items), composed from the oracle's restatement of the reference (oracle/pyoracle.py) so that they run in C++ at
2^27 points.  test_gpu_trace_stages.py compares the kernels with them; test_trace_stage_hooks_cpu.py checks them against plain Python
integers at small sizes.

Vectors are (n, 2) uint64 arrays (distaff_b200.felt); digests are (count, 32) uint8 arrays."""
import contextlib
import os

import numpy as np

from distaff_b200 import felt
from oracle import pyoracle as po
from tests.poly_stage_refs import POOL, power_series, vec

M = felt.M
M_LO, M_HI = np.uint64(M & (2**64 - 1)), np.uint64(M >> 64)
_W32 = np.uint64(0xFFFFFFFF)
_S32 = np.uint64(32)
_C = (0xFFFFFFFF, 11519)                      # 2^128 mod M = 45 2^40 - 1, as 32-bit limbs


# ---- element-wise products mod M (32-bit limbs in uint64 lanes) -------------------------------------------------------------------------
def _carry(cols):
    out, carry = [], np.zeros_like(cols[0])
    for col in cols:
        v = col + carry
        out.append(v & _W32)
        carry = v >> _S32
    return out


def _product(x, y):
    """limbs of x * y: every 32 x 32-bit product is split into halves, so a column sum stays below 2^36"""
    shape = np.broadcast(x[0], y[0]).shape
    cols = [np.zeros(shape, dtype=np.uint64) for _ in range(len(x) + len(y))]
    for i, xi in enumerate(x):
        for j, yj in enumerate(y):
            t = xi * yj
            cols[i + j] += t & _W32
            cols[i + j + 1] += t >> _S32
    return _carry(cols)


def _sum(x, y):
    n = max(len(x), len(y))
    zero = np.zeros(np.broadcast(x[0], y[0]).shape, dtype=np.uint64)
    return _carry([(x[i] if i < len(x) else zero) + (y[i] if i < len(y) else zero) for i in range(n)] + [zero])


def mul(a, b):
    """element-wise a b mod M of canonical vectors; b may be one element (a (1, 2) array), applied to every element of a"""
    a, b = vec(a), vec(b)
    if len(a) <= _BLOCK:
        return _mul_block(a, b)
    out = np.empty((len(a), 2), dtype=np.uint64)
    for i in range(0, len(a), _BLOCK):                             # blocks whose temporaries stay in cache
        out[i:i + _BLOCK] = _mul_block(a[i:i + _BLOCK], b if len(b) == 1 else b[i:i + _BLOCK])
    return out


_BLOCK = 1 << 14


def _mul_block(a, b):
    limbs = lambda v: [v[:, 0] & _W32, v[:, 0] >> _S32, v[:, 1] & _W32, v[:, 1] >> _S32]
    x = _product(limbs(a), limbs(b))                              # < 2^256
    c = [np.uint64(v) for v in _C]
    # x = lo + hi 2^128 = lo + hi (45 2^40 - 1) (mod M): below 2^174, then 2^128 + 2^92, then 2^128
    for _ in range(3):
        x = _sum(x[:4], _product(x[4:], c))
    lo, hi = x[0] | (x[1] << _S32), x[2] | (x[3] << _S32)
    ge = (hi > M_HI) | ((hi == M_HI) & (lo >= M_LO))
    out = np.stack([lo, hi], axis=1)
    out[ge, 1] = hi[ge] - M_HI - (lo[ge] < M_LO).astype(np.uint64)
    out[ge, 0] = lo[ge] - M_LO
    return out


# ---- the trace extension --------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def oracle_threads(jobs):
    """the oracle's host threads for `jobs` transforms side by side in POOL: the machine's cores (at most 32, as the whole-proof
    comparisons use) shared among them"""
    cpus = os.cpu_count() or 1
    po.set_threads(max(1, min(32, cpus) // max(1, min(jobs, cpus))))
    try:
        yield
    finally:
        po.set_threads(1)


def coset_extension(poly, log_b, cosets):
    """P(w_N^(k b + c)) of the n coefficients `poly` on each coset c of `cosets`, N = n 2^log_b: [len(cosets)][n], coset c =
    or_fft(poly (.) the powers of w_N^c)"""
    poly = vec(poly)
    n = len(poly)
    w = felt.root_of_unity(n << log_b)
    cosets = list(cosets)
    with oracle_threads(len(cosets)):
        out = list(POOL.map(lambda c: po.fft(mul(poly, power_series(pow(w, c, M), n))), cosets))
    return np.stack(out)


def monomial_extension(j, log_n, log_b, cosets):
    """the same for P = x^j, in closed form: [c][k] = (w_n^j)^k w_N^(j c), the scaling as the cubics 0 + row[k] x at x = w_N^(j c)
    (or_quartic_evaluate_batch)"""
    n, N = 1 << log_n, 1 << (log_n + log_b)
    w = felt.root_of_unity(N)
    rows = np.zeros((n, 4, 2), dtype=np.uint64)
    rows[:, 1] = power_series(pow(w, j << log_b, M), n)
    out = np.zeros((len(cosets), n, 2), dtype=np.uint64)
    with oracle_threads(1):
        for i, c in enumerate(cosets):
            x = felt.from_ints([pow(w, j * c, M)])
            po.lib().or_quartic_evaluate_batch(rows.ctypes.data, n, x.ctypes.data, out[i].ctypes.data)
    return out


# ---- commitments ----------------------------------------------------------------------------------------------------------------------
def hash_rows(cols):
    """or_hash_rows: blake3 of every row of a column-major (w, rows, 2) matrix"""
    cols = np.ascontiguousarray(cols, dtype=np.uint64)
    w, rows = cols.shape[0], cols.shape[1]
    out = np.zeros((rows, 32), dtype=np.uint8)
    with oracle_threads(1):
        po.lib().or_hash_rows(cols.ctypes.data, w, rows, out.ctypes.data)
    return out


def row_leaves(ext, log_n, log_blowup, c0):
    """the trace tree's leaves of a matrix whose cosets [c0, c0 + nc) are given as (w, nc, n, 2): leaf (k << log_blowup) + c = the row
    of coset c at step k, in logical order over the whole domain; leaves of cosets outside the range are zero"""
    w, nc, n = ext.shape[0], ext.shape[1], ext.shape[2]
    assert n == 1 << log_n
    digests = hash_rows(ext.reshape(w, nc * n, 2))
    leaves = np.zeros((n << log_blowup, 32), dtype=np.uint8)
    c = np.repeat(np.arange(c0, c0 + nc, dtype=np.int64), n)
    k = np.tile(np.arange(n, dtype=np.int64), nc)
    leaves[(k << log_blowup) + c] = digests
    return leaves


def constraint_items(ev, log_n, log_nc):
    """the first level of the constraint tree over one slab of evaluations [c][k] (nc = 2^log_nc cosets of n): item
    (k << (log_nc - 2)) + c4 = blake3(ev[4 c4][k], ev[4 c4 + 1][k], ev[4 c4 + 2][k], ev[4 c4 + 3][k])"""
    n, q = 1 << log_n, 1 << (log_nc - 2)
    ev = vec(ev).reshape(1 << log_nc, n, 2)
    items = np.zeros((n * q, 32), dtype=np.uint8)
    for c4 in range(q):
        items[np.arange(n) * q + c4] = hash_rows(ev[4 * c4:4 * c4 + 4])
    return items


def merkle_nodes(leaves):
    """or_merkle_nodes("blake3"): the heap of one tree, nodes[0] = 0, root = nodes[1]"""
    return np.frombuffer(po.merkle_nodes("blake3", np.ascontiguousarray(leaves).tobytes()), dtype=np.uint8).reshape(-1, 32)
