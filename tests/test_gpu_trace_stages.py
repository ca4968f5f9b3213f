"""-m gpu tests of the prover's evaluation-domain stage kernels, one at a time through the test hooks of include/distaff_gpu.h, compared
bit for bit with the oracle's restatement of the reference (tests/trace_stage_refs.py):

- stage 1, the trace extension (ntt_batch inverse + extend_trace_columns): every first-pass kind of the fold-1 coset transform at every
  first-pass size it runs at (PK_COSET_ONE at L0 = 2 .. 1024, PK_COSET_TWFULL at L0 = 64 .. 1024, PK_COSET_TW at L0 = 64 .. 1024, the
  three-pass transforms of 2^21 and 2^22 points), coset 0 copied or transformed, coset ranges that start above 0, column strides larger
  than the slab, and batches that cross the 4 GiB chunk of lde_batch and the 1 GiB chunk of ntt_batch;
- stage 2, hash_rows_kernel on coset-major slabs (widths 1 .. 127, coset ranges, a column table of three widths, 2^25 rows) and
  merkle_build (merkle_level_kernel + merkle_top_kernel) for one tree of 2 .. 2^25 leaves and K trees at once;
- stage 5, constraint_items_kernel for 4 .. 256 cosets, n = 16 .. 2^20, K = 1 and 3.

The columns are random, all (M - 1), zero but for coefficients at pass and tile boundaries, and the monomial x^j (closed form at any
size).  Output buffers are zero-filled before the kernels run: what lies outside the written ranges must come back zero."""
import random

import numpy as np
import pytest

from distaff_b200 import felt
from tests import poly_stage_refs as P
from tests import trace_stage_refs as R

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


def _passes(log_n):
    """ntt.cu split_passes: the pass sizes, outermost first"""
    if log_n <= 10:
        return [log_n]
    if log_n <= 20:
        return [(log_n + 1) // 2, log_n // 2]
    return [(log_n + 2) // 3, (log_n + 1) // 3, log_n // 3]


# ---- stage 1: the trace extension ---------------------------------------------------------------------------------------------------
class Columns:
    """register columns of one shape and what their extension must be: random registers, all-(M - 1) registers, spike coefficients
    (zero but at 1, L0 - 1, L0, R1 - 1, R1, n - 1), the monomial x^j, and (small shapes) all-(M - 1) coefficients"""

    def __init__(self, log_n, log_b, seed, kinds=("random", "full", "spikes", "monomial", "full_coeffs")):
        self.log_n, self.log_b = log_n, log_b
        n = self.n = 1 << log_n
        l0 = _passes(log_n)[0]
        L0, R1 = 1 << l0, n >> l0
        rnd = felt.random_elements(n, seed)
        self.kinds, regs, polys = list(kinds), [], []
        self.j = (seed * 7919 + 3) % n
        for kind in self.kinds:
            if kind == "random":
                r = rnd
                p = R.po.fft(r, inverse=True)
            elif kind == "full":
                r = np.empty((n, 2), dtype=np.uint64)
                r[:] = MINUS1
                p = np.zeros((n, 2), dtype=np.uint64)
                p[0] = MINUS1
            elif kind == "spikes":
                p = np.zeros((n, 2), dtype=np.uint64)
                for i in (1, L0 - 1, L0, R1 - 1, R1, n - 1):
                    if 0 <= i < n:
                        p[i] = rnd[i]
                r = R.po.fft(p)
            elif kind == "monomial":
                p = np.zeros((n, 2), dtype=np.uint64)
                p[self.j] = (1, 0)
                r = P.power_series(pow(felt.root_of_unity(n), self.j, M), n)
            else:                                                       # all-(M - 1) coefficients
                p = np.empty((n, 2), dtype=np.uint64)
                p[:] = MINUS1
                r = R.po.fft(p)
            regs.append(r)
            polys.append(p)
        self.regs = np.ascontiguousarray(np.stack(regs))
        self.polys = polys
        self.cache = {}

    def reference(self, q, cosets):
        """[len(cosets)][n]: column q's extension on the given cosets (those of the random and spike columns kept for later calls)"""
        kind = self.kinds[q]
        if kind in ("random", "spikes"):
            todo = [c for c in cosets if (q, c) not in self.cache]
            if todo:
                self.cache.update(((q, c), v) for c, v in zip(todo, R.coset_extension(self.polys[q], self.log_b, todo)))
            return np.stack([self.cache[(q, c)] for c in cosets])
        if kind == "full":
            out = np.empty((len(cosets), self.n, 2), dtype=np.uint64)
            out[:] = MINUS1
            return out
        if kind == "monomial":
            return R.monomial_extension(self.j, self.log_n, self.log_b, cosets)
        return R.coset_extension(self.polys[q], self.log_b, cosets)


def _lde(lib, regs, log_n, log_b, c0, nc, copy, col_stride=None):
    cols, n = regs.shape[0], regs.shape[1]
    col_stride = col_stride or nc * n
    polys = np.zeros((cols, n, 2), dtype=np.uint64)
    ext = np.zeros(((cols - 1) * col_stride + nc * n, 2), dtype=np.uint64)
    _check(lib, lib.dg_test_trace_lde(_p(regs), cols, log_n, log_b, c0, nc, col_stride, int(copy), _p(polys), _p(ext)))
    return polys, ext, col_stride


def _sample(c0, nc, limit, rng, n=1):
    """the cosets of [c0, c0 + nc) a comparison covers: all of them up to `limit` (and 2^21 points), else its edges, its middle and
    random ones"""
    limit = max(6, min(limit, (1 << 21) // n))
    if nc <= limit:
        return list(range(c0, c0 + nc))
    picks = {c0, c0 + 1, c0 + nc // 2 - 1, c0 + nc // 2, c0 + nc - 2, c0 + nc - 1}
    picks |= {rng.randrange(c0, c0 + nc) for _ in range(limit - len(picks))}
    return sorted(picks)


def _compare(cols, polys, ext, col_stride, c0, nc, cosets, chunk=16):
    n = cols.n
    for q in range(len(cols.kinds)):
        assert np.array_equal(polys[q], cols.polys[q]), ("interpolation", cols.kinds[q])
        for i in range(0, len(cosets), chunk):
            part = cosets[i:i + chunk]
            want = cols.reference(q, part)
            for c, w in zip(part, want):
                got = ext[q * col_stride + (c - c0) * n:q * col_stride + (c - c0 + 1) * n]
                assert np.array_equal(got, w), (cols.kinds[q], c)
        gap = ext[q * col_stride + nc * n:(q + 1) * col_stride] if q + 1 < len(cols.kinds) else ext[:0]
        assert not gap.any(), ("written between the columns", q)


def _extension_case(lib, log_n, log_b, limit=64, copy_too=True, kinds=None):
    b = 1 << log_b
    rng = random.Random(log_n * 64 + log_b)
    kinds = kinds or (("random", "full", "spikes", "monomial", "full_coeffs") if log_n <= 10 else ("random", "full", "spikes", "monomial"))
    cols = Columns(log_n, log_b, log_n * 64 + log_b, kinds=kinds)
    cosets = _sample(0, b, limit, rng, cols.n)
    polys, ext, stride = _lde(lib, cols.regs, log_n, log_b, 0, b, False)          # every coset transformed
    _compare(cols, polys, ext, stride, 0, b, cosets)
    if copy_too:                                                                  # coset 0 copied from the registers
        polys2, ext2, _ = _lde(lib, cols.regs, log_n, log_b, 0, b, True)
        assert np.array_equal(ext2, ext) and np.array_equal(polys2, polys)
    return cols, ext


# every first-pass kind at every first-pass size it runs at: (log_n, log_b) -> (kind, L0, passes), see ntt.cu run_transform
TWFULL_TWO = [(log_n, log_b) for log_n in range(11, 21) for log_b in (4, 5)] + [(20, 6), (18, 8)]
TW_TWO = [(20, 7), (19, 8), (17, 10), (14, 13), (12, 15)]
THREE = [(21, 5), (21, 6), (22, 5), (22, 4)]


@pytest.mark.parametrize("log_n", range(1, 11))
def test_one_pass_extension(lib, log_n):
    """PK_COSET_ONE at L = 2 .. 1024, blowups 2 .. 256"""
    for lb in (1, 3, 4, 5, 7, 8):
        _extension_case(lib, log_n, lb, limit=256)


@pytest.mark.parametrize("log_n,log_b", TWFULL_TWO)
def test_two_pass_streamed_table_extension(lib, log_n, log_b):
    """PK_COSET_TWFULL then PK_LAST: L0 = 64 .. 1024, the table up to its 2^26-pair cap (20 x 6, 18 x 8)"""
    assert log_n + log_b <= 26
    _extension_case(lib, log_n, log_b, copy_too=log_n in (11, 16))


def _large_kinds(log_n, log_b):
    """columns of the 2^26- and 2^27-point shapes: fewer of them, so that the extension stays within a few GiB of host memory"""
    return ("random", "spikes", "monomial") if log_n + log_b <= 26 else ("spikes", "monomial")


def _monomial_everywhere(cols, ext, stride, c0, nc, chunk=16):
    """the monomial column (the last one) on every coset of the range, against its closed form"""
    q, n = len(cols.kinds) - 1, cols.n
    for c in range(c0, c0 + nc, chunk):
        part = list(range(c, min(c + chunk, c0 + nc)))
        got = ext[q * stride + (c - c0) * n:q * stride + (part[-1] + 1 - c0) * n]
        assert np.array_equal(got.reshape(len(part), n, 2), cols.reference(q, part)), (c0, nc, c)


def _ranges_above_zero(lib, cols, log_n, log_b, ranges, sample, rng):
    """ranges that start above coset 0 (the pass kernels get the absolute coset): the range's ends and the full run's sampled cosets
    inside it against the reference, the monomial on every coset"""
    for c0, nc in ranges:
        polys, part, stride = _lde(lib, cols.regs, log_n, log_b, c0, nc, False)
        inside = sorted(set([c for c in sample if c0 <= c < c0 + nc] + [c0, c0 + nc - 1]))
        _compare(cols, polys, part, stride, c0, nc, inside)
        _monomial_everywhere(cols, part, stride, c0, nc)
        del part


@pytest.mark.parametrize("log_n,log_b", TW_TWO)
def test_two_pass_two_level_table_extension(lib, log_n, log_b):
    """PK_COSET_TW then PK_LAST (log_n + log_b > 26): L0 = 1024, 512, 128 and 64 (the out-of-line kernel)"""
    assert log_n + log_b > 26
    b, n = 1 << log_b, 1 << log_n
    rng = random.Random(log_n)
    cols = Columns(log_n, log_b, log_n * 64 + log_b, kinds=_large_kinds(log_n, log_b))
    polys, ext, stride = _lde(lib, cols.regs, log_n, log_b, 0, b, False)
    sample = _sample(0, b, 8, rng, n)
    _compare(cols, polys, ext, stride, 0, b, sample)
    _monomial_everywhere(cols, ext, stride, 0, b)
    del ext
    _ranges_above_zero(lib, cols, log_n, log_b, ((1, b - 1), (b - 1, 1), (b // 2 - 5, 9)), sample, rng)


@pytest.mark.parametrize("log_n,log_b", THREE)
def test_three_pass_extension(lib, log_n, log_b):
    """PK_COSET_TWFULL (21 x 5, 22 x 4 at L0 = 128, 256) or PK_COSET_TW (21 x 6, 22 x 5), then PK_TW, then PK_LAST"""
    b, n = 1 << log_b, 1 << log_n
    rng = random.Random(log_n * 10 + log_b)
    cols = Columns(log_n, log_b, log_n * 10 + log_b, kinds=_large_kinds(log_n, log_b))
    polys, ext, stride = _lde(lib, cols.regs, log_n, log_b, 0, b, True)
    sample = _sample(0, b, 6, rng, n)
    _compare(cols, polys, ext, stride, 0, b, sample)
    _monomial_everywhere(cols, ext, stride, 0, b)
    del ext
    _ranges_above_zero(lib, cols, log_n, log_b, ((1, b - 1), (b - 1, 1), (3, 5)), sample, rng)


@pytest.mark.parametrize("log_n,log_b", [(8, 4), (11, 5), (16, 4)])
def test_extension_coset_ranges_and_strides(lib, log_n, log_b):
    """ranges [0, b) by copy, [1, b), [b/2, b), [b - 1, b), an interior one and coset 0 alone, with the slab's column stride and a larger
    one (the gaps stay zero), against the all-cosets result"""
    b, n = 1 << log_b, 1 << log_n
    cols = Columns(log_n, log_b, log_n + log_b)
    _, full, _ = _lde(lib, cols.regs, log_n, log_b, 0, b, False)
    K = len(cols.kinds)
    for c0, nc in ((0, b), (1, b - 1), (b // 2, b // 2), (b - 1, 1), (3, 6), (0, 1), (0, 5)):
        for copy in (False, True):
            for extra in (0, 3 * n + 5):
                polys, part, stride = _lde(lib, cols.regs, log_n, log_b, c0, nc, copy, nc * n + extra)
                for q in range(K):
                    assert np.array_equal(polys[q], cols.polys[q])
                    assert np.array_equal(part[q * stride:q * stride + nc * n], full[q * b * n + c0 * n:q * b * n + (c0 + nc) * n]), (c0, nc, q)
                    if q + 1 < K:
                        assert not part[q * stride + nc * n:(q + 1) * stride].any(), (c0, nc, q)


def test_extension_crosses_the_lde_chunk(lib):
    """9 columns of 2^20 at b = 32 with coset 0 copied: the transform of cosets [1, 32) runs in two launches, 8 vectors and 1"""
    log_n, log_b, K = 20, 5, 9
    n, b = 1 << log_n, 1 << log_b
    cols = Columns(log_n, log_b, 99, kinds=("random", "spikes", "monomial", "random", "full", "random", "spikes", "monomial", "random"))
    for q in (3, 5, 8):                                                          # independent random columns
        cols.regs[q] = felt.random_elements(n, 1000 + q)
        cols.polys[q] = R.po.fft(cols.regs[q], inverse=True)
    polys, ext, stride = _lde(lib, cols.regs, log_n, log_b, 0, b, True)
    _compare(cols, polys, ext, stride, 0, b, [0, 1, 2, 8, 16, 30, 31])


def test_interpolation_crosses_the_ntt_chunk(lib):
    """65 columns of 2^20 on the cosets [5, 7): the interpolation runs in two launches, 64 vectors and 1"""
    log_n, log_b, K = 20, 5, 65
    n = 1 << log_n
    cols = Columns(log_n, log_b, 65, kinds=("random",))
    cols.kinds = ["random"] * K
    cols.regs = np.ascontiguousarray(np.stack([felt.random_elements(n, 2000 + q) for q in range(K)]))
    cols.regs[63][:] = MINUS1
    cols.polys = list(P.POOL.map(lambda r: R.po.fft(r, inverse=True), list(cols.regs)))
    polys, ext, stride = _lde(lib, cols.regs, log_n, log_b, 5, 2, False)
    for q in range(K):                                                           # every interpolation
        assert np.array_equal(polys[q], cols.polys[q]), q
    for q in (0, 1, 62, 63, 64):                                                 # the extension on both sides of the chunk edge
        assert np.array_equal(ext[q * stride:(q + 1) * stride].reshape(2, n, 2), cols.reference(q, [5, 6])), q


# ---- stage 2: row hashing --------------------------------------------------------------------------------------------------------------
def _hash_rows(lib, ext, total_cols, log_n, log_blowup, c0, nc, batch, table=None, leaf_stride=0):
    all_ = 1 << (log_n + log_blowup)
    stride = leaf_stride or all_
    leaves = np.zeros(((batch - 1) * stride + all_, 32), dtype=np.uint8)
    t = None if table is None else np.ascontiguousarray(np.array(table, dtype=np.uint32).reshape(-1))
    _check(lib, lib.dg_test_hash_trace_rows(_p(np.ascontiguousarray(ext)), total_cols, log_n, log_blowup, c0, nc, batch, _p(t), leaf_stride,
                                            _p(leaves)))
    return leaves, stride


def _slab(w, rows, seed):
    a = felt.random_elements(w * rows, seed).reshape(w, rows, 2)
    a[0, :min(rows, 7)] = MINUS1
    return a


@pytest.mark.parametrize("w", [1, 3, 4, 5, 16, 26, 63, 64, 65, 100, 127])
def test_row_hashing(lib, w):
    """one matrix per call and two side by side, on ranges of 2 .. 5120 rows (row counts below and off multiples of 256)"""
    for log_n, log_blowup, c0, nc in ((1, 0, 0, 1), (4, 2, 1, 3), (6, 3, 1, 5), (7, 4, 0, 16), (10, 5, 27, 5)):
        n = 1 << log_n
        ext = _slab(w, nc * n, w * 100 + log_n)
        leaves, _ = _hash_rows(lib, ext, w, log_n, log_blowup, c0, nc, 1)
        assert np.array_equal(leaves, R.row_leaves(ext.reshape(w, nc, n, 2), log_n, log_blowup, c0)), (log_n, c0, nc)
    # two matrices of w columns, their leaves 2^(log_n + log_blowup) + 40 digests apart (the gap stays zero)
    log_n, log_blowup, c0, nc = 5, 3, 2, 4
    n, all_ = 1 << log_n, 1 << (log_n + log_blowup)
    ext = _slab(2 * w, nc * n, w)
    leaves, stride = _hash_rows(lib, ext, 2 * w, log_n, log_blowup, c0, nc, 2, leaf_stride=all_ + 40)
    for q in range(2):
        want = R.row_leaves(ext[q * w:(q + 1) * w].reshape(w, nc, n, 2), log_n, log_blowup, c0)
        assert np.array_equal(leaves[q * stride:q * stride + all_], want), q
    assert not leaves[all_:stride].any()


def test_row_hashing_with_a_column_table(lib):
    """K = 3 matrices of widths 26, 65 and 1 in one launch through the column table, leaves N_loc apart, as the prover's batch"""
    log_n, log_blowup, c0, nc = 9, 4, 4, 8
    n, all_ = 1 << log_n, 1 << (log_n + log_blowup)
    widths = (26, 65, 1)
    first = np.cumsum((0,) + widths)[:-1]
    total = sum(widths) + 3                                    # unused columns after the last matrix
    ext = _slab(total, nc * n, 3)
    leaves, stride = _hash_rows(lib, ext, total, log_n, log_blowup, c0, nc, 3, table=[(f, w) for f, w in zip(first, widths)], leaf_stride=all_)
    for q, (f, w) in enumerate(zip(first, widths)):
        want = R.row_leaves(ext[f:f + w].reshape(w, nc, n, 2), log_n, log_blowup, c0)
        assert np.array_equal(leaves[q * stride:(q + 1) * stride], want), q


def test_row_hashing_2_25_rows(lib):
    """the whole trace commitment's leaves of 4 columns at 2^20 x 32: 2^25 rows"""
    log_n, log_blowup, w = 20, 5, 4
    n, b = 1 << log_n, 1 << log_blowup
    ext = _slab(w, b * n, 25)
    leaves, _ = _hash_rows(lib, ext, w, log_n, log_blowup, 0, b, 1)
    assert np.array_equal(leaves, R.row_leaves(ext.reshape(w, b, n, 2), log_n, log_blowup, 0))


# ---- stages 2 and 5: Merkle trees ----------------------------------------------------------------------------------------------------
def _trees(lib, L, K, seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    leaves = rng.integers(0, 256, size=(K * L, 32), dtype=np.uint8)
    nodes = np.zeros((K * L, 32), dtype=np.uint8)
    _check(lib, lib.dg_test_merkle_batch(_p(leaves), L, K, _p(nodes)))
    for q in range(K):
        assert np.array_equal(nodes[q * L:(q + 1) * L], R.merkle_nodes(leaves[q * L:(q + 1) * L])), q


@pytest.mark.parametrize("L", [2, 4, 1024, 2048, 2**20, 2**25])
def test_merkle_tree(lib, L):
    """L = 2 (one level launch), 1024 (one level launch, then merkle_top_kernel from 512 nodes), 2048 (then the top kernel from 1024 nodes),
    2^20 and 2^25 leaves"""
    _trees(lib, L, 1, L)


@pytest.mark.parametrize("L,K", [(1024, 64), (2**20, 3), (4, 5)])
def test_merkle_trees_of_a_batch(lib, L, K):
    """K trees in one launch per level, the top kernel one block per tree"""
    _trees(lib, L, K, L + K)


# ---- stage 5: constraint items ---------------------------------------------------------------------------------------------------------
CONSTRAINT_SHAPES = [(4, lnc, 3) for lnc in range(2, 9)] + [(11, lnc, 3 if lnc <= 6 else 1) for lnc in range(2, 9)] + [(20, 2, 3), (20, 5, 1)]


@pytest.mark.parametrize("log_n,log_nc,K", CONSTRAINT_SHAPES)
def test_constraint_items(lib, log_n, log_nc, K):
    n = 1 << log_n
    slab = n << log_nc
    ev = felt.random_elements(K * slab, log_n * 16 + log_nc)
    ev[:n] = MINUS1                                            # slab 0, coset 0
    ev[slab - 1] = MINUS1
    items = np.zeros((K * slab // 4, 32), dtype=np.uint8)
    _check(lib, lib.dg_test_constraint_items(_p(ev), log_n, log_nc, K, _p(items)))
    for q in range(K):
        want = R.constraint_items(ev[q * slab:(q + 1) * slab], log_n, log_nc)
        assert np.array_equal(items[q * slab // 4:(q + 1) * slab // 4], want), q
