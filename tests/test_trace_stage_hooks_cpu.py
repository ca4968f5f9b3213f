"""CPU checks of the evaluation-domain test hooks (include/distaff_gpu.h, "test hooks") and of the references test_gpu_trace_stages.py
compares them with:
- every hook rejects a shape the prover never produces with DG_ERR_INVALID and a message, before it looks for a device;
- the references composed from the oracle (tests/trace_stage_refs.py) agree with plain Python-integer restatements at small sizes, and
  the composed extension with the reference's own TraceTable::extend."""
import os
import random

import numpy as np
import pytest

from distaff_b200 import felt
from tests import poly_stage_refs as P
from tests import trace_stage_refs as R

M = felt.M


@pytest.fixture(scope="module")
def lib():
    from distaff_b200 import backend
    if not os.path.exists(backend.LIB_PATH):
        pytest.skip("libdistaff_gpu.so not built (run __graft_entry__.build())")
    return backend.lib()


def _buf(n):
    return np.zeros((max(n, 1), 2), dtype=np.uint64)


def _rejects(lib, rc, words):
    assert rc == -1, (rc, lib.dg_last_error())
    msg = lib.dg_last_error().decode()
    assert words in msg, msg


def _p(a):
    return None if a is None else a.ctypes.data


def _not_canonical(n):
    a = _buf(n)
    a[n - 1] = (M & (2**64 - 1), M >> 64)
    return a


def test_trace_lde_rejects_bad_shapes(lib):
    regs, polys, ext = _buf(64), _buf(64), _buf(1024)

    def call(cols=2, log_n=4, log_b=2, c0=0, nc=4, stride=64, r=regs):
        return lib.dg_test_trace_lde(_p(r), cols, log_n, log_b, c0, nc, stride, 1, _p(polys), _p(ext))
    _rejects(lib, call(c0=2, nc=3), "coset range")                  # a range past b
    _rejects(lib, call(c0=4, nc=1), "coset range")
    _rejects(lib, call(nc=0), "coset range")
    _rejects(lib, call(stride=63), "col_stride")                    # col_stride < ncosets n
    _rejects(lib, call(stride=2**33), "col_stride")
    _rejects(lib, call(log_b=0), "log_b")
    _rejects(lib, call(log_b=17), "log_b")
    _rejects(lib, call(log_n=0), "log_n")
    _rejects(lib, call(log_n=15, log_b=16), "log_n")
    _rejects(lib, call(cols=0), "cols")
    _rejects(lib, call(cols=65536), "cols")
    _rejects(lib, call(r=_not_canonical(32)), "not a field element")
    _rejects(lib, lib.dg_test_trace_lde(None, 1, 4, 2, 0, 4, 64, 0, _p(polys), _p(ext)), "null")


def test_hash_trace_rows_rejects_bad_shapes(lib):
    ext, leaves = _buf(4096), _buf(4096)

    def call(total=4, log_n=4, log_blowup=2, c0=0, nc=4, batch=1, table=None, stride=0, e=ext):
        t = None if table is None else np.array(table, dtype=np.uint32).reshape(-1)
        return lib.dg_test_hash_trace_rows(_p(e), total, log_n, log_blowup, c0, nc, batch, _p(t), stride, _p(leaves))
    _rejects(lib, call(c0=1, nc=4), "coset range")                  # a range past b
    _rejects(lib, call(nc=0), "coset range")
    _rejects(lib, call(table=[(0, 0)]), "width 1..127")             # width 0 or 128 through a column table
    _rejects(lib, call(total=200, table=[(0, 128)]), "width 1..127")
    _rejects(lib, call(total=4, table=[(2, 3)]), "columns out of range")
    _rejects(lib, call(total=128), "width")                         # width 128 without a table
    _rejects(lib, call(total=0), "total_cols")
    _rejects(lib, call(total=5, batch=2), "evenly")
    _rejects(lib, call(batch=0), "batch")
    _rejects(lib, call(batch=65536), "batch")
    _rejects(lib, call(batch=2, total=4, stride=63), "leaf_stride")
    _rejects(lib, call(log_blowup=17), "log_blowup")
    _rejects(lib, call(e=_not_canonical(256)), "not a field element")


def test_merkle_batch_rejects_bad_shapes(lib):
    leaves, nodes = _buf(64), _buf(64)
    for L in (0, 1, 3, 12, 2**31):                                   # L not a power of 2 in 2..2^30
        _rejects(lib, lib.dg_test_merkle_batch(_p(leaves), L, 1, _p(nodes)), "power of 2")
    _rejects(lib, lib.dg_test_merkle_batch(_p(leaves), 4, 0, _p(nodes)), "batch")
    _rejects(lib, lib.dg_test_merkle_batch(_p(leaves), 4, 65536, _p(nodes)), "batch")
    _rejects(lib, lib.dg_test_merkle_batch(None, 4, 1, _p(nodes)), "null")


def test_constraint_items_rejects_bad_shapes(lib):
    ev, items = _buf(1024), _buf(1024)
    _rejects(lib, lib.dg_test_constraint_items(_p(ev), 4, 1, 1, _p(items)), "log_nc")     # log_nc < 2
    _rejects(lib, lib.dg_test_constraint_items(_p(ev), 4, 17, 1, _p(items)), "log_nc")
    _rejects(lib, lib.dg_test_constraint_items(_p(ev), 0, 2, 1, _p(items)), "log_n")
    _rejects(lib, lib.dg_test_constraint_items(_p(ev), 4, 2, 0, _p(items)), "batch")
    _rejects(lib, lib.dg_test_constraint_items(_p(ev), 4, 2, 65536, _p(items)), "batch")
    bad = _not_canonical(128)
    _rejects(lib, lib.dg_test_constraint_items(_p(bad), 4, 3, 1, _p(items)), "not a field element")


# ---- the references against Python integers -----------------------------------------------------------------------------------------------
def _rand(rng, n):
    return [rng.randrange(M) for _ in range(n)]


def _horner(p, x):
    y = 0
    for c in reversed(p):
        y = (y * x + c) % M
    return y


def test_field_mul():
    rng = random.Random(1)
    edge = [0, 1, 2, M - 1, M - 2, 2**64 - 1, 2**64, 2**127, M - 2**64, 45 * 2**40, 2**96 + 1]
    a = edge * len(edge) + _rand(rng, 3000)
    b = [y for y in edge for _ in edge] + _rand(rng, 3000)
    assert felt.to_ints(R.mul(felt.from_ints(a), felt.from_ints(b))) == [x * y % M for x, y in zip(a, b)]
    s = rng.randrange(M)
    assert felt.to_ints(R.mul(felt.from_ints(a), felt.from_ints([s]))) == [x * s % M for x in a]


def test_coset_extension_reference():
    rng = random.Random(2)
    for log_n, log_b in ((1, 1), (3, 2), (4, 3)):
        n, N = 1 << log_n, 1 << (log_n + log_b)
        p = _rand(rng, n)
        p[-1] = M - 1
        w = felt.root_of_unity(N)
        cosets = [0, 1, (1 << log_b) - 1]
        got = R.coset_extension(felt.from_ints(p), log_b, cosets)
        for i, c in enumerate(cosets):
            assert felt.to_ints(got[i]) == [_horner(p, pow(w, (k << log_b) + c, M)) for k in range(n)], (log_n, log_b, c)
        j = rng.randrange(n)
        mono = R.monomial_extension(j, log_n, log_b, cosets)
        for i, c in enumerate(cosets):
            assert felt.to_ints(mono[i]) == [pow(w, j * ((k << log_b) + c), M) for k in range(n)]


def test_coset_extension_is_the_reference_extension():
    """the composed reference read coset by coset equals TraceTable::extend (the zero-padded or_fft of the interpolated registers)"""
    rng = random.Random(3)
    for log_n, log_b in ((4, 4), (10, 3), (7, 5)):
        n, b = 1 << log_n, 1 << log_b
        regs = np.stack([felt.random_elements(n, log_n), felt.from_ints([M - 1] * n), felt.from_ints(_rand(rng, n))])
        lde = R.po.extend(regs, b)
        for q in range(len(regs)):
            poly = R.po.fft(regs[q], inverse=True)
            want = lde[q].reshape(n, b, 2).transpose(1, 0, 2)
            assert np.array_equal(R.coset_extension(poly, log_b, range(b)), want), (log_n, log_b, q)


def test_row_hash_reference(po):
    rng = random.Random(4)
    for w, rows in ((1, 3), (4, 5), (64, 2), (65, 2), (127, 3)):
        cols = felt.from_ints(_rand(rng, w * rows)).reshape(w, rows, 2)
        got = R.hash_rows(cols)
        for i in range(rows):
            row = felt.from_ints([felt.to_ints(cols[j, i])[0] for j in range(w)]).tobytes()
            assert got[i].tobytes() == po.hash("blake3", row), (w, i)
    # leaves in logical order: the row of coset c at step k is leaf (k << log_blowup) + c, cosets outside the range zero
    log_n, log_blowup, c0, nc, w = 2, 3, 5, 2, 3
    n = 1 << log_n
    ext = felt.from_ints(_rand(rng, w * nc * n)).reshape(w, nc, n, 2)
    leaves = R.row_leaves(ext, log_n, log_blowup, c0)
    for i in range(n << log_blowup):
        k, c = i >> log_blowup, i & ((1 << log_blowup) - 1)
        if c0 <= c < c0 + nc:
            assert leaves[i].tobytes() == po.hash("blake3", np.ascontiguousarray(ext[:, c - c0, k]).tobytes()), i
        else:
            assert not leaves[i].any(), i


def test_constraint_item_reference():
    rng = random.Random(5)
    for log_n, log_nc in ((1, 2), (3, 4), (2, 5)):
        n, nc = 1 << log_n, 1 << log_nc
        ev = felt.from_ints(_rand(rng, nc * n)).reshape(nc, n, 2)
        q = nc // 4
        msgs = np.zeros((n * q, 4, 2), dtype=np.uint64)
        for k in range(n):
            for c4 in range(q):
                msgs[k * q + c4] = ev[4 * c4:4 * c4 + 4, k]
        assert np.array_equal(R.constraint_items(ev, log_n, log_nc), P.blake3_rows(msgs)), (log_n, log_nc)


def test_merkle_reference(po):
    rng = np.random.Generator(np.random.PCG64(6))
    leaves = rng.integers(0, 256, size=(8, 32), dtype=np.uint8)
    nodes = R.merkle_nodes(leaves)
    heap = np.concatenate([nodes, leaves])
    assert not nodes[0].any()
    for i in range(1, 8):
        assert nodes[i].tobytes() == po.hash("blake3", heap[2 * i].tobytes() + heap[2 * i + 1].tobytes()), i
