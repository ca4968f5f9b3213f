"""-m gpu tests of the prover's coefficient-domain stage kernels, one at a time through the test hooks of include/distaff_gpu.h, compared
bit for bit with the oracle's restatement of the reference (tests/poly_stage_refs.py) at the block, batch and size edges of each kernel:

- syn_div_chained_kernel (poly.cu): one block (16 elements) up to 32 768 blocks (2^25), K = 64 vectors behind one ticket counter, both
  power-table layouts, in place and out of place, against polynom::syn_div_in_place;
- strided_suffix_kernel + expanded_stencil_kernel: n up to 2^22 (8n = 2^25), with and without the added boundary quotients;
- eval2_partial_kernel + reduce_partials_kernel: one 4096-element chunk up to 1024 chunks, mixed widths, both forms;
- eval_rows_partial_kernel: one tile up to blocks that walk two tiles, widths 1..128;
- prefold8_kernel and the PK_FOLD_* passes: every coset at b = 8..256, coset ranges, strided batches, the three-pass 2^21 transform;
- coset_interp_finish_kernel: the round trip of 8 coset transforms up to n = 2^21;
- fri_hash_rows_kernel, fri_alpha_kernel, fri_fold_kernel: coset-major, switching and natural layers from 2^10 to 2^25 values.

Vectors hold all-(M-1) values (the longest carry chains and largest unreduced sums) and single coefficients at block boundaries."""
import random

import numpy as np
import pytest

from distaff_b200 import felt
from tests import poly_stage_refs as R

pytestmark = pytest.mark.gpu

M = felt.M
MINUS1 = (M - 1) & (2**64 - 1), (M - 1) >> 64


@pytest.fixture(scope="module")
def lib():
    from distaff_b200 import backend
    backend.device_info()
    return backend.lib()


def _check(lib, rc):
    from distaff_b200 import backend
    if rc != 0:
        raise backend.DgError(rc, lib.dg_last_error().decode(errors="replace"))


def _p(a):
    return None if a is None else a.ctypes.data


def _kinds(n, seed):
    """a random vector, an all-(M-1) vector and one that is zero but for coefficients at block boundaries"""
    rnd = felt.random_elements(n, seed)
    full = np.empty((n, 2), dtype=np.uint64)
    full[:] = MINUS1
    spikes = np.zeros((n, 2), dtype=np.uint64)
    for i in (1, 1023, 1024, 4095, 4096, n - 1):
        if i < n:
            spikes[i] = rnd[i]
    return [rnd, full, spikes]


def _strided(vectors, stride, fill=None):
    n = len(vectors[0])
    buf = np.zeros(((len(vectors) - 1) * stride + n, 2), dtype=np.uint64) if fill is None else fill.copy()
    for q, v in enumerate(vectors):
        buf[q * stride:q * stride + n] = v
    return buf


def _inv(x):
    return pow(x, M - 2, M)


# ---- synthetic division ----------------------------------------------------------------------------------------------------------------
def _syn_div(lib, vectors, points, shared, in_place, in_stride, out_stride, sub0):
    K, n = len(vectors), len(vectors[0])
    src = _strided(vectors, in_stride)
    out = np.zeros(((K - 1) * out_stride + n, 2), dtype=np.uint64)
    b = felt.from_ints(points)
    s = felt.from_ints(sub0)
    _check(lib, lib.dg_test_syn_div(_p(src), _p(out), K, n, in_stride, out_stride, int(in_place), _p(b), int(shared), _p(s)))
    if in_place:                                               # the gaps between the vectors are left as they were
        mask = np.ones(len(out), dtype=bool)
        for q in range(K):
            mask[q * out_stride:q * out_stride + n] = False
        assert np.array_equal(out[mask], src[mask])
    return [out[q * out_stride:q * out_stride + n] for q in range(K)]


@pytest.mark.parametrize("K", [1, 3])
@pytest.mark.parametrize("length", [16, 128, 1024, 2048, 2**15, 2**16, 2**19, 2**23, 2**25])
def test_syn_div(lib, length, K):
    rng = random.Random(length * 7 + K)
    vecs = _kinds(length, length + K)
    groups = [[v] for v in vecs] if K == 1 else [vecs]
    x_last = _inv(felt.root_of_unity(max(length // 8, 1)))
    points = [1, x_last, rng.randrange(M), M - 1]
    gap = length if length <= 2**16 else 1024
    # (shared table, in place, in_stride, out_stride): stage 4 (3E in place, one table), stage 6 (2n in place, a table per proof; E out
    # of place); at the largest sizes two of them
    modes = [(1, True, length + gap, length + gap), (0, False, length + gap, length), (1, False, length, length + gap), (0, True, 2 * length, 2 * length)]
    if length >= 2**23:
        modes = modes[:2]
    for i, b in enumerate(points):
        for vs in groups:
            sub0 = [rng.randrange(M) for _ in vs]                # the quotient does not depend on a[0]
            per_vector = [points[(i + q) % 4] for q in range(len(vs))]
            refs = list(R.POOL.map(lambda qb: R.syn_div(*qb), [(v, b) for v in vs]))
            refs_pv = list(R.POOL.map(lambda qb: R.syn_div(*qb), [(v, p) for v, p in zip(vs, per_vector)]))
            for shared, in_place, si, so in modes:
                got = _syn_div(lib, vs, [b] if shared else per_vector, shared, in_place, si, so, sub0)
                for q, g in enumerate(got):
                    assert np.array_equal(g, (refs if shared else refs_pv)[q]), (b, q, shared, in_place)


def test_syn_div_64_vectors_behind_one_ticket_counter(lib):
    """K = 64 vectors of 2^20 elements: 65 536 blocks in one launch"""
    K, n = 64, 2**20
    rng = random.Random(64)
    vecs = [felt.random_elements(n, 1000 + q) for q in range(K)]
    vecs[5][:] = MINUS1
    vecs[63][:] = 0
    vecs[63][n - 1] = MINUS1
    z = [rng.randrange(M) for _ in range(K)]
    refs = list(R.POOL.map(lambda qb: R.syn_div(*qb), zip(vecs, z)))
    got = _syn_div(lib, vecs, z, 0, False, n, n, [rng.randrange(M) for _ in range(K)])
    for q in range(K):
        assert np.array_equal(got[q], refs[q]), q
    b = rng.randrange(M)
    refs = list(R.POOL.map(lambda v: R.syn_div(v, b), vecs))
    got = _syn_div(lib, vecs, [b], 1, True, n + 512, n + 512, [0] * K)
    for q in range(K):
        assert np.array_equal(got[q], refs[q]), q


# ---- division by (x^n - 1) / (x - x_last), summed with the boundary quotients -----------------------------------------------------------
@pytest.mark.parametrize("K", [1, 5])
@pytest.mark.parametrize("log_n", [4, 10, 16, 22])
def test_syn_div_expanded_sum(lib, log_n, K):
    if log_n == 22 and K > 1:
        pytest.skip("2^25-coefficient vectors: one of them")
    n = 1 << log_n
    E = 8 * n
    x_last = _inv(felt.root_of_unity(n))
    kinds = _kinds(E, log_n)
    a = [kinds[q % 3] if q < 3 else felt.random_elements(E, 50 + q) for q in range(K)]
    add0 = [felt.random_elements(E, 60 + q) for q in range(K)]
    add1 = [kinds[(q + 1) % 3] for q in range(K)]
    quot = list(R.POOL.map(lambda v: R.syn_div_expanded(v, n, x_last), a))
    in_stride = 3 * E if K > 1 else E                          # the prover's [ic | fc | t] slabs
    e = felt.from_ints([x_last])
    for use0, use1 in ((False, False), (True, False), (True, True)):
        src, s0, s1 = _strided(a, in_stride), _strided(add0, in_stride) if use0 else None, _strided(add1, in_stride) if use1 else None
        out = np.zeros(((K - 1) * E + E, 2), dtype=np.uint64)
        _check(lib, lib.dg_test_syn_div_expanded_sum(_p(src), _p(s0), _p(s1), _p(out), K, n, in_stride, E, _p(e)))
        for q in range(K):
            want = quot[q]
            if use0:
                want = R.add(want, add0[q])
            if use1:
                want = R.add(want, add1[q])
            assert np.array_equal(out[q * E:(q + 1) * E], want), (q, use0, use1)


# ---- evaluations at z and z w_n ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n", [4, 12, 13, 20, 22])
def test_eval_polys_at(lib, log_n):
    n = 1 << log_n
    rng = random.Random(log_n)
    widths = (5, 26, 65) if log_n <= 20 else (1, 3, 2)          # three proofs of mixed widths in one call
    cols = []
    for p, w in enumerate(widths):
        kinds = _kinds(n, 100 * log_n + p)
        cols += [kinds[j % 3] if j < 3 else felt.random_elements(n, 1000 * p + j) for j in range(w)]
    col_proof = np.array([p for p, w in enumerate(widths) for _ in range(w)], dtype=np.uint32)
    z = [rng.randrange(M) for _ in widths]
    z[-1] = M - 1
    wn = felt.root_of_unity(n)
    polys = np.ascontiguousarray(np.stack(cols))
    out = np.zeros((2 * len(cols), 2), dtype=np.uint64)
    zb = felt.from_ints(z)
    _check(lib, lib.dg_test_eval_polys_at(_p(polys), len(cols), log_n, _p(zb), len(z), _p(col_proof), _p(out)))
    jobs = []
    for j, c in enumerate(cols):
        zj = z[col_proof[j]]
        jobs += [(c, zj), (c, zj * wn % M)]
    assert felt.to_ints(out) == R.poly_evals(jobs)

    # the one-point form: the constraint polynomial (8n coefficients) of each proof at its own z
    K = 3
    cps = _kinds(8 * n, log_n + 7)
    polys = np.ascontiguousarray(np.stack(cps))
    out = np.zeros((2 * K, 2), dtype=np.uint64)
    _check(lib, lib.dg_test_eval_polys_at(_p(polys), K, log_n, _p(zb), K, None, _p(out)))
    want = R.poly_evals([(cps[q], z[q]) for q in range(K)])
    assert felt.to_ints(out) == [v for q in range(K) for v in (want[q], 0)]


# ---- opened trace rows ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n", [4, 11, 17, 18])
def test_eval_trace_rows(lib, log_n):
    n, W, log_b = 1 << log_n, 128, 4
    N, b = n << log_b, 1 << log_b
    rng = random.Random(log_n)
    kinds = _kinds(n, log_n)
    cols = [kinds[j % 3] if j < 6 else felt.random_elements(n, 7000 + j) for j in range(W)]
    polys = np.ascontiguousarray(np.stack(cols))
    positions = [0, N - 1, b, b * (n - 1), rng.randrange(N), rng.randrange(N)]
    rows = [(pos, rng.randrange(W - w + 1), w) for w in (1, 8, 9, 26, 128) for pos in positions]
    pos = np.array([r[0] for r in rows], dtype=np.uint64)
    col = np.array([r[1] for r in rows], dtype=np.uint32)
    wid = np.array([r[2] for r in rows], dtype=np.uint32)
    out = np.zeros((int(wid.sum()), 2), dtype=np.uint64)
    _check(lib, lib.dg_test_eval_trace_rows(_p(polys), W, log_n, log_n + log_b, _p(pos), _p(col), _p(wid), len(rows), _p(out)))
    wN = felt.root_of_unity(N)
    values = dict(zip([(p, j) for p in positions for j in range(W)],
                      R.poly_evals([(cols[j], pow(wN, p, M)) for p in positions for j in range(W)])))
    got = felt.to_ints(out)
    k = 0
    for p, c0, w in rows:
        assert got[k:k + w] == [values[(p, j)] for j in range(c0, c0 + w)], (p, c0, w)
        k += w
    # a position on the trace domain gives the trace row itself
    trace = [felt.to_ints(R.po.fft(cols[j])) for j in range(3)]
    for p in (0, b, b * (n - 1)):
        assert [values[(p, j)] for j in range(3)] == [trace[j][p // b] for j in range(3)]


# ---- fold-8 extension -------------------------------------------------------------------------------------------------------------------
def _fold8(lib, vectors, log_n, log_b, c0, nc, dst_stride):
    K, n = len(vectors), 1 << log_n
    src = np.ascontiguousarray(np.concatenate(vectors))
    out = np.zeros(((K - 1) * dst_stride + nc * n, 2), dtype=np.uint64)
    _check(lib, lib.dg_test_lde_fold8(_p(src), _p(out), log_n, log_b, c0, nc, K, dst_stride))
    return [out[q * dst_stride:q * dst_stride + nc * n].reshape(nc, n, 2) for q in range(K)], out


def _ranges(b):
    return [(c0, nc) for c0, nc in ((0, 8), (8, 8), (b - 1, 1), (3, 5)) if c0 + nc <= b]


@pytest.mark.parametrize("log_n,log_b", [(4, 3), (4, 4), (4, 5), (4, 8), (10, 3), (10, 4), (10, 5), (10, 8), (11, 3), (11, 4), (11, 5), (11, 8),
                                         (16, 3), (16, 4), (16, 5), (20, 3)])
def test_fold8_extension(lib, log_n, log_b):
    n, b = 1 << log_n, 1 << log_b
    coeffs = felt.random_elements(8 * n, log_n * 16 + log_b)
    coeffs[7 * n:] = MINUS1
    want = R.fold8_extension(coeffs, log_b)
    (full,), _ = _fold8(lib, [coeffs], log_n, log_b, 0, b, b * n)         # all cosets: prefold8_kernel + plain transforms
    assert np.array_equal(full, want)
    for c0, nc in _ranges(b):                                             # coset ranges: the PK_FOLD_* passes
        (part,), _ = _fold8(lib, [coeffs], log_n, log_b, c0, nc, nc * n)
        assert np.array_equal(part, full[c0:c0 + nc]), (c0, nc)


@pytest.mark.parametrize("log_n,log_b", [(4, 4), (10, 5), (11, 3), (16, 4)])
def test_fold8_batch_contiguous_and_strided(lib, log_n, log_b):
    n, b = 1 << log_n, 1 << log_b
    vecs = _kinds(8 * n, log_n + 3 * log_b)
    wants = [R.fold8_extension(v, log_b) for v in vecs]
    contiguous, _ = _fold8(lib, vecs, log_n, log_b, 0, b, b * n)
    strided, raw = _fold8(lib, vecs, log_n, log_b, 0, b, b * n + 48)
    for q in range(3):
        assert np.array_equal(contiguous[q], wants[q]), q
        assert np.array_equal(strided[q], contiguous[q]), q
        assert not raw[q * (b * n + 48) + b * n:(q + 1) * (b * n + 48)].any()      # nothing written between the vectors
    for c0, nc in _ranges(b):
        part, _ = _fold8(lib, vecs, log_n, log_b, c0, nc, nc * n + 16)
        for q in range(3):
            assert np.array_equal(part[q], contiguous[q][c0:c0 + nc]), (q, c0, nc)


def test_fold8_three_pass_extension(lib):
    """log_n = 21: every transform takes three passes; sampled points of every coset against a direct evaluation"""
    log_n, log_b = 21, 4
    n, b = 1 << log_n, 1 << log_b
    coeffs = felt.random_elements(8 * n, 21)
    coeffs[8 * n - 1] = MINUS1
    (full,), _ = _fold8(lib, [coeffs], log_n, log_b, 0, b, b * n)
    rng = random.Random(21)
    picks = [(c, rng.randrange(n)) for c in range(b)] + [(0, 0), (b - 1, n - 1), (3, 1023), (8, 1024)]
    w = felt.root_of_unity(n * b)
    want = R.poly_evals([(coeffs, pow(w, k * b + c, M)) for c, k in picks])
    assert [felt.to_ints(full[c, k])[0] for c, k in picks] == want
    for c0, nc in ((3, 5), (8, 8), (b - 1, 1)):
        (part,), _ = _fold8(lib, [coeffs], log_n, log_b, c0, nc, nc * n)
        assert np.array_equal(part, full[c0:c0 + nc]), (c0, nc)


# ---- coset interpolation --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n,K", [(4, 1), (4, 3), (11, 1), (11, 3), (16, 1), (16, 3), (20, 1), (21, 1)])
def test_coset_interpolation_round_trip(lib, log_n, K):
    n = 1 << log_n
    E = 8 * n
    vecs = _kinds(E, log_n)[:K] if K == 3 else [felt.random_elements(E, log_n)]
    evals = np.ascontiguousarray(np.concatenate([R.coset_evaluations(v).reshape(E, 2) for v in vecs]))
    out_stride = 3 * E                                        # the prover writes into its [ic | fc | t] slabs
    out = np.zeros(((K - 1) * out_stride + E, 2), dtype=np.uint64)
    _check(lib, lib.dg_test_coset_interp(_p(evals), _p(out), log_n, K, out_stride))
    for q in range(K):
        assert np.array_equal(out[q * out_stride:q * out_stride + E], vecs[q]), q
        if q + 1 < K:
            assert not out[q * out_stride + E:(q + 1) * out_stride].any()


# ---- one FRI layer --------------------------------------------------------------------------------------------------------------------
def _fri_layer(lib, values, log_d, log_b, log_N, roots):
    K, D = len(values), 1 << log_d
    Rn = D // 4
    phys = R.phys(np.arange(D), log_d, log_b)
    src = np.zeros((K * D, 2), dtype=np.uint64)
    for q, v in enumerate(values):
        src[q * D + phys] = v
    leaves = np.zeros((K * Rn, 32), dtype=np.uint8)
    alphas = np.zeros((K, 2), dtype=np.uint64)
    copies = np.zeros((K, 32), dtype=np.uint8)
    nxt = np.zeros((K * Rn, 2), dtype=np.uint64)
    rb = np.frombuffer(b"".join(roots), dtype=np.uint8).copy()
    _check(lib, lib.dg_test_fri_layer(_p(src), K, D, log_d, log_b, log_N, _p(rb), 32 * Rn, _p(leaves), _p(alphas), _p(copies), _p(nxt)))
    log_r, rows_b = R.rows_layout(log_d, log_b)
    back = R.phys(np.arange(Rn), log_r, rows_b)
    return leaves.reshape(K, Rn, 32), felt.to_ints(alphas), [bytes(c) for c in copies], [nxt[q * Rn:(q + 1) * Rn][back] for q in range(K)]


def _fri_cases():
    cases = []
    for log_N in range(10, 26):
        lb = 4 + log_N % 5                                    # blowups 16 .. 256
        cases.append((log_N, log_N, lb))                      # first layer: coset-major values and rows
        cases.append((log_N, lb + (log_N - lb) % 2, lb))      # the rows switch to the natural layout (log_r < log_b)
        cases.append((log_N, log_N - 2, -1))                  # a natural layer
    return cases


@pytest.mark.parametrize("log_N,log_d,log_b", _fri_cases())
def test_fri_layer(lib, po, log_N, log_d, log_b):
    D = 1 << log_d
    Rn = D // 4
    K = 4 if log_d <= 20 else 1
    rng = random.Random(log_N * 100 + log_d)
    kinds = _kinds(D, log_N + log_d)
    values = [kinds[q % 3] if q < 3 else felt.random_elements(D, q) for q in range(K)]
    roots = [bytes(rng.randrange(256) for _ in range(32)) for _ in range(K)]
    leaves, alphas, copies, folded = _fri_layer(lib, values, log_d, log_b, log_N, roots)
    assert copies == roots
    assert alphas == [po.prng_vector(r, 1)[0] for r in roots]
    if Rn <= 2**14:
        rows = np.arange(Rn)
    else:                                                     # the edges, every coset boundary near them, and random rows
        edge = [0, 1, Rn // 2 - 1, Rn // 2, Rn - 2, Rn - 1] + [(1 << max(log_b, 0)) * k + d for k in (1, 2, 1000) for d in (-1, 0, 1)]
        rows = np.unique(np.array([r for r in edge if r < Rn] + [rng.randrange(Rn) for _ in range(8192)], dtype=np.int64))
    for q in range(K):
        assert np.array_equal(leaves[q][rows], R.blake3_rows(R.quartic_rows(values[q], rows))), q
        assert np.array_equal(folded[q][rows], R.fri_fold_rows(values[q], rows, log_N, alphas[q])), q


def test_fri_alpha_of_10000_roots(lib, po):
    rng = random.Random(10000)
    K = 10000
    roots = [bytes(rng.randrange(256) for _ in range(32)) for _ in range(K)]
    values = [felt.random_elements(16, q) for q in range(K)]
    _, alphas, copies, _ = _fri_layer(lib, values, 4, -1, 4, roots)
    assert copies == roots
    assert alphas == [po.prng_vector(r, 1)[0] for r in roots]
