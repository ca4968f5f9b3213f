"""CPU checks of the stage-kernel test hooks (include/distaff_gpu.h, "test hooks") and of the references test_gpu_poly_stages.py compares
them with:
- every hook rejects a shape the prover never produces with DG_ERR_INVALID and a message, before it looks for a device;
- the references composed from the oracle (tests/poly_stage_refs.py) agree with plain Python-integer restatements at small sizes."""
import os
import random

import numpy as np
import pytest

from distaff_b200 import felt
from tests import poly_stage_refs as R

M = felt.M


@pytest.fixture(scope="module")
def lib():
    from distaff_b200 import backend
    if not os.path.exists(backend.LIB_PATH):
        pytest.skip("libdistaff_gpu.so not built (run __graft_entry__.build())")
    return backend.lib()


def _buf(n):
    return np.zeros((max(n, 1), 2), dtype=np.uint64)


def _u32(values):
    return np.array(values, dtype=np.uint32)


def _u64(values):
    return np.array(values, dtype=np.uint64)


def _rejects(lib, rc, words):
    assert rc == -1, (rc, lib.dg_last_error())
    msg = lib.dg_last_error().decode()
    assert words in msg, msg


def _p(a):
    return a.ctypes.data


def test_syn_div_rejects_bad_shapes(lib):
    a, out, b, s = _buf(64), _buf(64), _buf(4), _buf(4)
    b[:, 0] = 3
    call = lambda batch, ln, si, so, inplace=0, shared=0, bb=b: lib.dg_test_syn_div(_p(a), _p(out), batch, ln, si, so, inplace, _p(bb), shared, _p(s))
    _rejects(lib, call(1, 24, 24, 24), "power of 2")
    _rejects(lib, call(1, 1, 1, 1), "power of 2")
    _rejects(lib, call(0, 16, 16, 16), "batch")
    _rejects(lib, call(65536, 16, 16, 16), "batch")
    _rejects(lib, call(2, 16, 8, 16), "in_stride")
    _rejects(lib, call(2, 16, 16, 2**33), "out_stride")
    _rejects(lib, call(2, 16, 32, 16, inplace=1), "one stride")
    _rejects(lib, call(1, 16, 16, 16, bb=_buf(4)), "zero")
    big = _buf(4)
    big[0] = (M & (2**64 - 1), M >> 64)
    _rejects(lib, call(1, 16, 16, 16, bb=big), "not a field element")
    _rejects(lib, lib.dg_test_syn_div(None, _p(out), 1, 16, 16, 16, 0, _p(b), 0, _p(s)), "null")


def test_expanded_division_rejects_bad_shapes(lib):
    a, out, e = _buf(256), _buf(256), _buf(1)
    _rejects(lib, lib.dg_test_syn_div_expanded_sum(_p(a), None, None, _p(out), 1, 12, 96, 96, _p(e)), "power of 2")
    _rejects(lib, lib.dg_test_syn_div_expanded_sum(_p(a), None, None, _p(out), 2, 16, 64, 128, _p(e)), "in_stride")
    _rejects(lib, lib.dg_test_syn_div_expanded_sum(_p(a), None, None, _p(out), 70000, 16, 128, 128, _p(e)), "batch")


def test_evaluations_reject_bad_shapes(lib):
    p, z, out = _buf(4096), _buf(4), _buf(64)
    cp = _u32([0, 2])
    _rejects(lib, lib.dg_test_eval_polys_at(_p(p), 2, 4, _p(z), 2, _p(cp), _p(out)), "names no point")
    _rejects(lib, lib.dg_test_eval_polys_at(_p(p), 3, 4, _p(z), 2, None, _p(out)), "one-point")
    _rejects(lib, lib.dg_test_eval_polys_at(_p(p), 0, 4, _p(z), 1, None, _p(out)), "1..65535")
    _rejects(lib, lib.dg_test_eval_polys_at(_p(p), 1, 27, _p(z), 1, None, _p(out)), "log_n")

    def one(pos, col, w, log_N=8):
        pos, col, w = _u64([pos]), _u32([col]), _u32([w])           # kept alive for the call
        return lib.dg_test_eval_trace_rows(_p(p), 4, 4, log_N, _p(pos), _p(col), _p(w), 1, _p(out))
    _rejects(lib, one(256, 0, 1), "outside the domain")
    _rejects(lib, one(0, 3, 2), "columns out of range")
    _rejects(lib, one(0, 0, 0), "columns out of range")
    _rejects(lib, one(0, 0, 1, log_N=3), "log_N")
    _rejects(lib, one(0, 0, 1, log_N=13), "log_N")


def test_extension_and_interpolation_reject_bad_shapes(lib):
    p, out = _buf(2048), _buf(2048)
    _rejects(lib, lib.dg_test_lde_fold8(_p(p), _p(out), 4, 2, 0, 4, 1, 64), "log_b")
    _rejects(lib, lib.dg_test_lde_fold8(_p(p), _p(out), 4, 9, 0, 4, 1, 64), "log_b")
    _rejects(lib, lib.dg_test_lde_fold8(_p(p), _p(out), 4, 4, 12, 5, 1, 80), "coset range")
    _rejects(lib, lib.dg_test_lde_fold8(_p(p), _p(out), 4, 4, 16, 1, 1, 16), "coset range")
    _rejects(lib, lib.dg_test_lde_fold8(_p(p), _p(out), 4, 4, 0, 0, 1, 16), "coset range")
    _rejects(lib, lib.dg_test_lde_fold8(_p(p), _p(out), 4, 4, 0, 4, 2, 32), "dst_stride")
    _rejects(lib, lib.dg_test_coset_interp(_p(p), _p(out), 0, 1, 8), "log_n")
    _rejects(lib, lib.dg_test_coset_interp(_p(p), _p(out), 4, 2, 64), "out_stride")
    _rejects(lib, lib.dg_test_coset_interp(_p(p), _p(out), 4, 0, 128), "batch")


def test_fri_layer_rejects_bad_shapes(lib):
    v, roots, leaves, alphas, copies, nxt = _buf(4096), _buf(8), _buf(4096), _buf(4), _buf(8), _buf(1024)
    call = lambda log_d, log_b, log_N, stride=None, rs=32, batch=1: lib.dg_test_fri_layer(
        _p(v), batch, stride if stride is not None else 1 << log_d, log_d, log_b, log_N, _p(roots), rs, _p(leaves), _p(alphas), _p(copies), _p(nxt))
    _rejects(lib, call(9, 4, 10), "even number of folds")
    _rejects(lib, call(12, 4, 10), "log_d")
    _rejects(lib, call(2, -1, 10), "log_d")
    _rejects(lib, call(8, 9, 10), "log_b")
    _rejects(lib, call(8, -2, 10), "log_b")
    _rejects(lib, call(8, 4, 10, stride=100), "values_stride")
    _rejects(lib, call(8, 4, 10, rs=16), "root_stride")
    _rejects(lib, call(8, 4, 10, rs=34), "root_stride")
    _rejects(lib, call(8, 4, 10, batch=0), "batch")


# ---- the references against Python integers -----------------------------------------------------------------------------------------------
def _rand(rng, n):
    return [rng.randrange(M) for _ in range(n)]


def _horner(p, x):
    y = 0
    for c in reversed(p):
        y = (y * x + c) % M
    return y


def test_field_add():
    rng = random.Random(1)
    edge = [0, 1, M - 1, M - 2, 2**64 - 1, 2**64, 2**127, M - 2**64]
    a = edge * len(edge) + _rand(rng, 2000)
    b = [y for y in edge for _ in edge] + _rand(rng, 2000)
    assert felt.to_ints(R.add(felt.from_ints(a), felt.from_ints(b))) == [(x + y) % M for x, y in zip(a, b)]


def test_syn_div_reference():
    rng = random.Random(2)
    for n in (2, 16, 64):
        for b in (1, M - 1, rng.randrange(M)):
            a = _rand(rng, n)
            want = [sum(a[j] * pow(b, j - i - 1, M) for j in range(i + 1, n)) % M for i in range(n)]
            assert felt.to_ints(R.syn_div(felt.from_ints(a), b)) == want


def test_expanded_division_reference():
    """a = q (x^n - 1) / (x - e) with e^n = 1 gives back q (the prover's divisions are exact)"""
    rng = random.Random(3)
    for n in (4, 16):
        e = pow(felt.root_of_unity(n), M - 2, M)
        d = [pow(e, n - 1 - i, M) for i in range(n)]                 # (x^n - e^n) / (x - e)
        q = _rand(rng, 7 * n + 1)
        a = [0] * (8 * n)
        for i, qi in enumerate(q):
            for j, dj in enumerate(d):
                a[i + j] = (a[i + j] + qi * dj) % M
        assert felt.to_ints(R.syn_div_expanded(felt.from_ints(a), n, e)) == q + [0] * (n - 1)


def test_evaluation_references():
    rng = random.Random(4)
    p = _rand(rng, 100)
    xs = [0, 1, M - 1] + _rand(rng, 5)
    assert R.poly_evals([(felt.from_ints(p), x) for x in xs]) == [_horner(p, x) for x in xs]
    w = felt.root_of_unity(16)
    assert felt.to_ints(R.power_series(w, 20)) == [pow(w, i, M) for i in range(20)]


def test_extension_references():
    rng = random.Random(5)
    n, log_b = 4, 4
    N = n << log_b
    coeffs = _rand(rng, 8 * n)
    ext = R.fold8_extension(felt.from_ints(coeffs), log_b)
    w = felt.root_of_unity(N)
    for c in range(1 << log_b):
        assert felt.to_ints(ext[c]) == [_horner(coeffs, pow(w, (k << log_b) + c, M)) for k in range(n)]
    ev = R.coset_evaluations(felt.from_ints(coeffs))
    w8n = felt.root_of_unity(8 * n)
    for c in range(8):
        assert felt.to_ints(ev[c]) == [_horner(coeffs, pow(w8n, 8 * k + c, M)) for k in range(n)]


def test_layouts():
    for log_d, log_b in ((6, 2), (6, 6), (5, -1), (8, 4)):
        D = 1 << log_d
        p = R.phys(np.arange(D), log_d, log_b)
        assert sorted(p.tolist()) == list(range(D))
        for i in range(D):
            want = i if log_b < 0 else (i % (1 << log_b)) * (D >> log_b) + (i >> log_b)
            assert p[i] == want
    assert R.rows_layout(10, 4) == (8, 4)
    assert R.rows_layout(6, 5) == (4, -1)
    assert R.rows_layout(10, -1) == (8, -1)


def test_fri_row_references(po):
    rng = random.Random(6)
    log_N, log_d = 8, 6
    D = 1 << log_d
    R4 = D // 4
    v = _rand(rng, D)
    rows = np.array([0, 1, 7, R4 - 1], dtype=np.int64)
    msgs = R.quartic_rows(felt.from_ints(v), rows)
    digests = R.blake3_rows(msgs)
    for k, r in enumerate(rows.tolist()):
        m = felt.from_ints([v[r + j * R4] for j in range(4)]).tobytes()
        assert msgs[k].tobytes() == m
        assert digests[k].tobytes() == po.hash("blake3", m)
    alpha = rng.randrange(M)
    got = felt.to_ints(R.fri_fold_rows(felt.from_ints(v), rows, log_N, alpha))
    wN = felt.root_of_unity(2**log_N)
    for k, r in enumerate(rows.tolist()):
        xs = [pow(wN, (r + j * R4) << (log_N - log_d), M) for j in range(4)]
        ys = [v[r + j * R4] for j in range(4)]
        want = 0
        for i in range(4):                                           # Lagrange form of the cubic through the four points, at alpha
            num, den = 1, 1
            for j in range(4):
                if j != i:
                    num = num * (alpha - xs[j]) % M
                    den = den * (xs[i] - xs[j]) % M
            want = (want + ys[i] * num * pow(den, M - 2, M)) % M
        assert got[k] == want, r

