"""-m gpu tests of the fold-1 trace extension on the shapes the full-table checks of test_gpu_blocks.py do not reach.

- n = 2^19 at blowup 256: the extension domain (2^27 points) is past the streamed first-pass table, so the first pass takes its output
  twiddles from the two-level table.  A transform of 2^27 points on the host is too slow, so the polynomial is sparse: its trace comes
  from the oracle's FFT, and sampled points of every coset are compared with a direct evaluation of its few terms.
- a two-pass trace proven under a memory limit: the prover extends coset ranges that start above 0 and do not cover all cosets."""
import random

import numpy as np
import pytest

from tests.test_gpu_memory_limit import check_limited

pytestmark = pytest.mark.gpu

M = 2**128 - 45 * 2**40 + 1


@pytest.fixture(scope="module")
def dg():
    import distaff_b200
    from distaff_b200 import backend
    backend.device_info()
    yield distaff_b200
    distaff_b200.set_memory_limit(0)


def test_two_level_first_pass_on_every_coset(dg, po):
    log_n, log_b = 19, 8
    n, b = 1 << log_n, 1 << log_b
    rng = random.Random(19)
    terms = {0: rng.randrange(M), 1: rng.randrange(M), n - 1: rng.randrange(M), n // 2 + 1: M - 1}
    while len(terms) < 24:
        terms[rng.randrange(n)] = rng.randrange(M)
    coeffs = np.zeros((n, 2), dtype=np.uint64)
    for j, v in terms.items():
        coeffs[j] = (v & (2**64 - 1), v >> 64)
    trace = po.fft(coeffs)                                   # trace[k] = P(w_n^k)
    ext = dg.lde(trace, b)[0]
    assert np.array_equal(ext[::b], trace)                   # the extension agrees with the trace on the trace domain
    w = po.root_of_unity(n * b)
    assert pow(w, n * b // 2, M) == M - 1
    for c in range(b):
        for k in [0, 1, n - 1] + [rng.randrange(n) for _ in range(3)]:
            i = b * k + c                                    # LDE index of point k of coset c
            x = pow(w, i, M)
            want = sum(v * pow(x, j, M) for j, v in terms.items()) % M
            got = int(ext[i, 0]) | (int(ext[i, 1]) << 64)
            assert got == want, (c, k)


def test_two_pass_coset_ranges_under_a_memory_limit(dg, po):
    from distaff_b200 import hostvm
    tr = hostvm.fibonacci(250)
    assert tr.length == 4096                                 # 64 x 64-point passes
    check_limited(dg, po, tr, dg.ProofOptions(64, 20, 12))
